"""The numpy stand-in of tests/fields_tuple_standin.py with the expression calls of include/dampr_b200.h
(dampr_text_fields_expr, dampr_text_fields_expr_records): the tests of computed keys and values
(test_text_fields_expr_lowering.py) run on it. The other calls behave exactly like the tuple stand-in's.

It also holds a plain-Python evaluator of the programs (eval_program), the statement of which lines the device takes
that the GPU tests compare the kernel's per-line values with."""
import math

from fields_standin import M64, _int18, f64_bits, parse_f64
from fields_tuple_standin import make_tuple_ctx
from fields_where_standin import line_verdict
from fields_ws_standin import WsLine

I64_MIN, I64_MAX, LIM53 = -(1 << 63), (1 << 63) - 1, 1 << 53


def _int64(x):
    return x if I64_MIN <= x <= I64_MAX else None


def eval_program(words, ci, cf, lv, nf):
    """the value of one program (opcode words as lowering.numeric_program builds them) over the load slot values lv
    and the field count nf: an int or a float, or None where the device hands the line to the host (Python raises, or
    an int leaves int64)"""
    from dampr_b200.lowering import _EV
    op_of = {v: k for k, v in _EV.items()}
    st = []
    for w in words:
        op, arg = op_of[w & 0xFF], w >> 8
        if op in ("CI", "CF", "LOAD", "NF"):
            st.append(ci[arg] if op == "CI" else cf[arg] if op == "CF" else lv[arg] if op == "LOAD" else nf)
            continue
        b = st.pop()
        if op in ("I2F", "INEG", "IABS", "FNEG", "FABS", "F2I"):
            if op == "F2I":
                if math.isnan(b) or math.isinf(b):
                    return None
                r = _int64(int(b))
            else:
                r = float(b) if op == "I2F" else -b if op in ("INEG", "FNEG") else abs(b)
                if op in ("INEG", "IABS"):
                    r = _int64(r)
            if r is None:
                return None
            st.append(r)
            continue
        a = st.pop()
        if op in ("IDIV", "IFLOOR", "IMOD", "FDIV") and b == 0:
            return None
        if op == "IDIV" and (abs(a) > LIM53 or abs(b) > LIM53):
            return None
        r = {"IADD": lambda: a + b, "ISUB": lambda: a - b, "IMUL": lambda: a * b, "FADD": lambda: a + b,
             "FSUB": lambda: a - b, "FMUL": lambda: a * b, "FDIV": lambda: a / b, "IDIV": lambda: a / b,
             "IFLOOR": lambda: a // b, "IMOD": lambda: a % b}[op]()
        if type(r) is int and _int64(r) is None:
            return None
        st.append(r)
    assert len(st) == 1
    return st[0]


def expr_line(line, f, expr, spec):
    """(key, value) the device computes for a taken line whose split is f (bytes fields) under expr =
    device.field_expr's tuple and spec = (sep, key field, key kind, value field, op), or None for a line it hands to
    the host (its predicates aside). An int key is an int, a str key bytes."""
    from dampr_b200 import device as dev
    key, val, ci, cf, loads = expr
    _sep, kf, kind, vf, op = spec
    lv = []
    for i, lk in loads:
        if not -len(f) <= i < len(f):
            return None
        x = len(f[i]) if lk == dev.LOAD_LEN else _int18(f[i]) if lk == dev.LOAD_INT else parse_f64(f[i])
        if x is None:
            return None
        lv.append(x)
    flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
    if val is not None:
        v = eval_program(val[1], ci, cf, lv, len(f))
    elif vf == dev.FIELD_VAL_ONE:
        v = 1
    else:
        v = None if not -len(f) <= vf < len(f) else parse_f64(f[vf]) if flt else _int18(f[vf])
    if v is None:
        return None
    if key is not None:
        k = eval_program(key[1], ci, cf, lv, len(f))
        if k is None or k == I64_MIN:
            return None
    else:
        k = None if not -len(f) <= kf < len(f) else f[kf] if kind == dev.FIELD_KEY_STR else _int18(f[kf])
        if k is None:
            return None
    return k, v


def make_expr_ctx(free_bytes=1 << 30):
    """make_tuple_ctx(free_bytes) whose tables also take the expression calls"""
    from dampr_b200 import device as dev
    ctx = make_tuple_ctx(free_bytes)
    Base = type(ctx.table(4))

    class ExprTable(Base):
        def fields_expr(self, tb, lo, hi, spec, expr, cr_is_data=False, preds=()):
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_MIN_I64, dev.OP_MAX_I64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            self._expr_scan(tb, lo, hi, spec, expr, cr_is_data, preds, None)

        def fields_expr_records(self, tb, lo, hi, spec, expr, kv, cr_is_data=False, preds=()):
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_SUM_F64)
            self._expr_scan(tb, lo, hi, spec, expr, cr_is_data, preds, kv)

        def _expr_scan(self, tb, lo, hi, spec, expr, cr_is_data, preds, rec):
            x = dev.field_expr(expr)   # the binding's packing
            assert x.key_type or x.val_type
            dev.fields_spec(spec, cr_is_data, preds)
            data = tb.buf[:tb.n].tobytes()
            pos = 0
            while pos < len(data):
                end = data.find(b"\n", pos)
                end = len(data) if end < 0 else end
                if lo <= pos < hi:
                    line = data[pos:end]
                    self._expr_line(WsLine(line) if spec[0] == dev.FIELD_SEP_WS else line, pos, spec, expr,
                                    cr_is_data, preds, rec)
                pos = end + 1

        def _expr_line(self, line, off, spec, expr, cr_is_data, preds, rec):
            st = self.st
            sep, kf, kind, vf, op = spec
            f = line.split() if sep == dev.FIELD_SEP_WS else line.split(bytes([sep]))
            verdict = line_verdict(line, f, preds, cr_is_data)
            if verdict is False:
                if rec is not None:
                    self._put(rec, 0, 0)
                else:
                    st["raw"] += 1
                return
            kv = expr_line(line, f, expr, spec) if verdict is True else None
            if kv is None:
                self._hand_back(line, off, rec)
                return
            k, v = kv
            st["lines"] += 1
            st["folded"] += 1
            flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            if flt and v == 0 and math.copysign(1.0, v) < 0:
                st["flags"] |= dev.TF_NEGZERO
            if flt and v != v:
                st["flags"] |= dev.TF_NAN
            if not flt:
                self.max_abs = max(self.max_abs, abs(v))
            int_key = expr[0] is not None or kind == dev.FIELD_KEY_INT
            if not int_key and not 1 <= len(k) <= 9:
                st["hashed"] += 1
                self.rep[k] = min(self.rep.get(k, 1 << 62), (off << 20) | len(k))
            if k not in self.code:
                i = len(self.code)
                self.code[k] = ((k ^ (1 << 63)) & M64 if int_key else (1 << 63 | i) if not 1 <= len(k) <= 9 else i + 1)
            if rec is not None:
                self._put(rec, self.code[k], f64_bits(v) if flt else v & M64)
                self.acc[k] = self.acc.get(k, 0) + 1
                return
            if flt:
                b = f64_bits(v)
                enc = b ^ (M64 if b >> 63 else 1 << 63)
            else:
                enc = v & M64 if op == dev.OP_SUM_I64 else (v ^ (1 << 63)) & M64
            if op in (dev.OP_MIN_I64, dev.OP_MIN_F64):
                enc = ~enc & M64
            old = self.acc.get(k, 0)
            self.acc[k] = (old + enc) & M64 if op == dev.OP_SUM_I64 else max(old, enc)

    ctx.table = lambda log2: ExprTable(ctx, log2)
    return ctx

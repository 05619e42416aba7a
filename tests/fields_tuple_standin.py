"""The numpy stand-in of tests/fields_ws_standin.py with the tuple-key calls of include/dampr_b200.h
(dampr_text_fields_tuple, dampr_text_fields_tuple_records, dampr_table_fetch_field_keys): the tests of
`(l.split(S)[i], int(l.split(S)[j]), ...)` keys (test_text_fields_tuple_lowering.py) run on it. The other calls behave
exactly like the whitespace stand-in's.

It also holds a plain-Python statement of the tuple key code, which the GPU tests compare the kernel's codes with."""
from fields_standin import M64, _int18, f64_bits, parse_f64
from fields_where_standin import line_verdict
from fields_ws_standin import WsLine, make_ws_ctx

SEED = 0x243F6A8885A308D3
M32 = (1 << 32) - 1


def mix64(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def tuple_code(parts):
    """the key code of a tuple whose components are `parts`: bytes (a str component) or int (an int() component).
    The field keys' seeded hash is fed each str component's bytes, the 8 little-endian bytes of v ^ 2^63 of each int
    component v, and one 0xFF byte between components; it finishes as for a hashed field key."""
    h1, h2 = (SEED & M32) ^ 0x811C9DC5, (SEED >> 32) ^ 0x9747B28C
    fed = b"\xff".join(p if type(p) is bytes else ((p ^ (1 << 63)) & M64).to_bytes(8, "little") for p in parts)
    for c in fed:
        h1 = ((h1 ^ c) * 16777619) & M32
        h2 = ((h2 ^ c) * 0x85EBCA6B + 0x9E3779B9) & M32
        h2 = ((h2 << 13) | (h2 >> 19)) & M32
    return mix64(((h1 << 32) | h2) ^ ((len(fed) * 0x9E3779B97F4A7C15) & M64)) | (1 << 63)


def tuple_line(line, f, spec, keys, cr_is_data, preds):
    """one line of a tuple-key scan whose fields are f: False (dropped), None (the host's) or (components, value), a
    str component bytes and an int() one an int"""
    from dampr_b200 import device as dev
    _sep, _kf, _kind, vf, op = spec
    verdict = line_verdict(line, f, preds, cr_is_data)
    if verdict is not True:
        return verdict
    flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
    if not all(-len(f) <= i < len(f) for i, _k in keys) or not (vf == dev.FIELD_VAL_ONE or -len(f) <= vf < len(f)):
        return None
    v = 1 if vf == dev.FIELD_VAL_ONE else parse_f64(f[vf]) if flt else _int18(f[vf])
    parts = [f[i] if k == dev.FIELD_KEY_STR else _int18(f[i]) for i, k in keys]
    return None if v is None or None in parts else (parts, v)


def make_tuple_ctx(free_bytes=1 << 30):
    """make_ws_ctx(free_bytes) whose tables also take the tuple-key calls"""
    import numpy as np
    from dampr_b200 import device as dev
    ctx = make_ws_ctx(free_bytes)
    Base = type(ctx.table(4))

    class TupleTable(Base):
        def clear(self):
            Base.clear(self)
            self.tuples = {}   # key code -> the components of its first line (the device's representative)

        def fields_tuple(self, tb, lo, hi, spec, keys, cr_is_data=False, preds=()):
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_MIN_I64, dev.OP_MAX_I64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            self._tuple_scan(tb, lo, hi, spec, keys, cr_is_data, preds, None)

        def fields_tuple_records(self, tb, lo, hi, spec, keys, kv, cr_is_data=False, preds=()):
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_SUM_F64)
            self._tuple_scan(tb, lo, hi, spec, keys, cr_is_data, preds, kv)

        def _tuple_scan(self, tb, lo, hi, spec, keys, cr_is_data, preds, rec):
            assert 1 <= len(keys) <= dev.FIELD_KEYS_MAX
            dev.field_keys(keys), dev.fields_spec(spec, cr_is_data, preds)   # the binding's packing
            data = tb.buf[:tb.n].tobytes()
            pos = 0
            while pos < len(data):
                end = data.find(b"\n", pos)
                end = len(data) if end < 0 else end
                if lo <= pos < hi:
                    line = data[pos:end]
                    self._tuple_line(WsLine(line) if spec[0] == dev.FIELD_SEP_WS else line, pos, spec, keys,
                                     cr_is_data, preds, rec)
                pos = end + 1

        def _tuple_line(self, line, off, spec, keys, cr_is_data, preds, rec):
            st = self.st
            sep, _kf, _kind, vf, op = spec
            f = line.split() if sep == dev.FIELD_SEP_WS else line.split(bytes([sep]))
            got = tuple_line(line, f, spec, keys, cr_is_data, preds)
            if got is False:
                if rec is not None:
                    self._put(rec, 0, 0)
                else:
                    st["raw"] += 1
                return
            if got is None:
                self._hand_back(line, off, rec)
                return
            parts, v = got
            flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            st["lines"] += 1
            st["folded"] += 1
            if flt and v == 0 and str(v).startswith("-"):
                st["flags"] |= dev.TF_NEGZERO
            if not flt:
                self.max_abs = max(self.max_abs, abs(v))
            code = tuple_code(parts)
            if self.tuples.setdefault(code, tuple(parts)) != tuple(parts):
                st["flags"] |= dev.TF_COLLISION
            self.code[code] = code
            self.rep[code] = min(self.rep.get(code, 1 << 62), (off << 20) | len(line))
            if rec is not None:
                self._put(rec, code, f64_bits(v) if flt else v & M64)
                self.acc[code] = self.acc.get(code, 0) + 1
                return
            if flt:
                b = f64_bits(v)
                enc = b ^ (M64 if b >> 63 else 1 << 63)
            else:
                enc = v & M64 if op == dev.OP_SUM_I64 else (v ^ (1 << 63)) & M64
            if op in (dev.OP_MIN_I64, dev.OP_MIN_F64):
                enc = ~enc & M64
            old = self.acc.get(code, 0)
            self.acc[code] = (old + enc) & M64 if op == dev.OP_SUM_I64 else max(old, enc)

        def fetch_field_keys(self, tb, sep, keys):
            codes = list(self.acc)
            cols = []
            for j, (_i, kind) in enumerate(keys):
                xs = [self.tuples[c][j] for c in codes]
                if kind == dev.FIELD_KEY_INT:
                    cols.append(np.array(xs, dtype=np.int64))
                else:
                    cols.append(np.array(xs, dtype="S%d" % max([1] + [len(x) for x in xs])))
            return (cols, np.array([self.acc[c] for c in codes], dtype=np.uint64),
                    np.array(codes, dtype=np.uint64))

    ctx.table = lambda log2: TupleTable(ctx, log2)
    return ctx

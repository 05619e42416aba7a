"""The numpy stand-in of tests/fields_where_standin.py with the JSON-lines calls dampr_text_json_fields and
dampr_text_json_fields_records (include/dampr_b200.h): the tests of `Dampr.json(...)` folds
(test_text_fields_json_lowering.py) run on it. The other calls behave exactly like the WHERE stand-in's.

The device's line rules are restated with Python's own json module: a line is read member by member with
json.decoder.scanstring and JSONDecoder.raw_decode, so each top-level member keeps the raw text of its value, and the
rules the device adds (ASCII only, no text-mode '\\r', under 4 KB, no NaN / Infinity, nesting at most 64 deep, no
escaped top-level name) are checked on top."""
import json
import re

from fields_standin import _int18, parse_f64
from fields_where_standin import _CMPS, make_where_ctx

WS = " \t\n\r"
_INT = re.compile(r"-?(0|[1-9][0-9]*)\Z")
STR, ESC, INT, FLOAT, OTHER = "str", "esc", "int", "float", "other"


def _no_constant(name):
    raise ValueError("NaN / Infinity: the device does not take %s" % name)


_DECODER = json.JSONDecoder(parse_constant=_no_constant)


def _depth(v):
    if isinstance(v, dict):
        return 1 + max((_depth(x) for x in v.values()), default=0)
    if isinstance(v, list):
        return 1 + max((_depth(x) for x in v), default=0)
    return 0


def _kind(raw):
    if raw[0] == '"':
        return ESC if "\\" in raw else STR
    if raw[0] == "-" or raw[0].isdigit():
        return INT if _INT.match(raw) else FLOAT
    return OTHER


def device_members(line, cr_is_data=False):
    """the device's reading of one line (bytes, no '\\n'): None when the device hands it back, else {name: (kind, raw
    text of the value, offset of its bytes in the line)} of the top-level members, the last occurrence of each name;
    a string's raw text and offset are those of the bytes between its quotes"""
    if len(line) >= 4096 or any(c == 0 or c >= 0x80 for c in line) or (not cr_is_data and b"\r" in line):
        return None
    s = line.decode("ascii")
    out = {}
    try:
        i = len(s) - len(s.lstrip(WS))
        if s[i:i + 1] != "{":
            return None
        i += 1
        depth, first = 1, True
        while True:
            i += len(s[i:]) - len(s[i:].lstrip(WS))
            if first and s[i:i + 1] == "}":
                i += 1
                break
            if s[i:i + 1] != '"':
                return None
            name, j = json.decoder.scanstring(s, i + 1)
            if "\\" in s[i + 1:j - 1]:
                return None
            j += len(s[j:]) - len(s[j:].lstrip(WS))
            if s[j:j + 1] != ":":
                return None
            j += 1
            j += len(s[j:]) - len(s[j:].lstrip(WS))
            v, end = _DECODER.raw_decode(s, j)
            depth = max(depth, 1 + _depth(v))
            raw = s[j:end]
            out[name] = (_kind(raw), raw[1:-1], j + 1) if raw[0] == '"' else (_kind(raw), raw, j)
            i = end + len(s[end:]) - len(s[end:].lstrip(WS))
            first = False
            if s[i:i + 1] == ",":
                i += 1
                continue
            if s[i:i + 1] != "}":
                return None
            i += 1
            break
        if s[i:].strip(WS) or depth > 64:
            return None
    except (ValueError, IndexError):
        return None
    assert type(json.loads(s)) is dict   # the reading above takes only what json.loads takes
    return out


def json_where(m, preds, names):
    """the header's JSON WHERE rule over the members m: True, False at the first false predicate, None at the first
    one the device cannot decide"""
    from dampr_b200 import device as dev
    for kind, i, cmp, consts in preds:
        got = m.get(names[i])
        if kind == dev.PRED_MEMBER:
            r = (got is not None) == (cmp == dev.CMP_IN)
        else:
            want = {dev.PRED_STR: (STR,), dev.PRED_INT: (INT,), dev.PRED_F64: (INT, FLOAT)}[kind]
            if got is None or got[0] not in want:
                return None
            raw = got[1].encode("ascii")
            if kind == dev.PRED_STR:
                x, consts = raw, [c.encode("utf-8") for c in consts]
            else:
                x = _int18(raw) if kind == dev.PRED_INT else parse_f64(raw)
                if x is None:
                    return None
            r = (x in consts) == (cmp == dev.CMP_IN) if cmp in (dev.CMP_IN, dev.CMP_NOT_IN) else _CMPS[cmp](x,
                                                                                                         consts[0])
        if not r:
            return False
    return True


def json_line(line, spec, names, cr_is_data, preds):
    """one line of a JSON scan: (outcome, flags). outcome is False (dropped), None (the host's) or (synth, key offset):
    a line of the key's raw bytes, then 0x01 and the value's, which the plain scan reads as field 0 (the key) and
    field 1 (the value, absent under FIELD_VAL_ONE), the key at that offset in the line; flags are the
    DAMPR_TF_JSON_* flags the line raises"""
    from dampr_b200 import device as dev
    _sep, kf, kind, vf, op = spec
    m = device_members(line, cr_is_data)
    verdict = None if m is None else json_where(m, preds, names)
    if verdict is not True:
        return verdict, 0
    flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
    k = m.get(names[kf])
    v = None if vf == dev.FIELD_VAL_ONE else m.get(names[vf])
    flags = 0
    if k is not None and k[0] not in ((INT,) if kind == dev.FIELD_KEY_INT else (STR, ESC)):
        flags |= dev.TF_JSON_KEY_KIND
    if v is not None and v[0] != (FLOAT if flt else INT):
        flags |= dev.TF_JSON_VAL_KIND
    ok = k is not None and k[0] == (INT if kind == dev.FIELD_KEY_INT else STR)
    if vf != dev.FIELD_VAL_ONE:
        ok = ok and v is not None and v[0] in ((INT, FLOAT) if flt else (INT,))
    if ok and kind == dev.FIELD_KEY_INT:
        ok = _int18(k[1].encode()) is not None
    if ok and vf != dev.FIELD_VAL_ONE:
        raw = v[1].encode()
        # float() of a JSON integer is float(int): "-0" is 0.0
        val = (b"0" if raw == b"-0" and flt else raw)
        ok = (parse_f64(val) if flt else _int18(val)) is not None
    if not ok:
        return None, flags
    return (k[1].encode() + (b"" if vf == dev.FIELD_VAL_ONE else b"\x01" + val), k[2]), flags


def make_json_ctx(free_bytes=1 << 30):
    """make_where_ctx(free_bytes) whose tables also take json_fields() and json_fields_records()"""
    from dampr_b200 import device as dev
    ctx = make_where_ctx(free_bytes)
    Where = type(ctx.table(4))
    Plain = next(c for c in Where.__mro__ if c.__name__ == "FieldsTable")

    class JsonTable(Where):
        def json_fields(self, tb, lo, hi, spec, members, cr_is_data=False, preds=()):
            dev.fields_spec(spec, cr_is_data, preds)
            dev.json_members(members)
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_MIN_I64, dev.OP_MAX_I64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            self._json_scan(tb, lo, hi, spec, members, cr_is_data, tuple(preds), None)

        def json_fields_records(self, tb, lo, hi, spec, members, kv, cr_is_data=False, preds=()):
            dev.fields_spec(spec, cr_is_data, preds)
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_SUM_F64)
            self._json_scan(tb, lo, hi, spec, members, cr_is_data, tuple(preds), kv)

        def _json_scan(self, tb, lo, hi, spec, names, cr_is_data, preds, rec):
            assert spec[0] == dev.FIELD_SEP_JSON and 1 <= len(names) <= dev.JSON_MAX_MEMBERS
            data = tb.buf[:tb.n].tobytes()
            pos = 0
            while pos < len(data):
                end = data.find(b"\n", pos)
                end = len(data) if end < 0 else end
                if lo <= pos < hi:
                    self._json_line(data[pos:end], pos, spec, names, cr_is_data, preds, rec)
                pos = end + 1

        def _json_line(self, line, off, spec, names, cr_is_data, preds, rec):
            _sep, _kf, kind, vf, op = spec
            got, flags = json_line(line, spec, names, cr_is_data, preds)
            self.st["flags"] |= flags
            if got is False:
                if rec is not None:
                    self._put(rec, 0, 0)
                else:
                    self.st["raw"] += 1
                return
            if got is None:
                self._hand_back(line, off, rec)
                return
            # the plain stand-in over a line of the key's and the value's raw bytes, the key first at its own offset
            synth, k_off = got
            Plain._line(self, synth, off + k_off, b"\x01", 0, kind, dev.FIELD_VAL_ONE if vf == dev.FIELD_VAL_ONE
                        else 1, op, cr_is_data, rec)

    ctx.table = lambda log2: JsonTable(ctx, log2)
    return ctx

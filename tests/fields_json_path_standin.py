"""The stand-in of tests/fields_json_standin.py for JSON scans whose members are paths r[n1]..[nk]
(dampr_text_json_fields and dampr_text_json_fields_records with DAMPR_JSON_PATH_SEP in a member, include/dampr_b200.h):
the tests of nested `Dampr.json(...)` folds (test_text_fields_json_paths_lowering.py) run on it.

A line is read with Python's json module, recursively through the objects the device compares names in: the
top-level object and every occurrence of a wanted interior name whose value is an object. Each occurrence of a wanted
name replaces the earlier one's subtree, as a later duplicate does in the dict json.loads builds. A name with an
escape in a compared object hands the line back; the device's other line rules are device_members'."""
import json

from fields_filter_standin import leaf as filter_leaf, verdict
from fields_json_standin import FLOAT, INT, STR, ESC, WS, _DECODER, _kind, device_members, json_where, make_json_ctx
from fields_standin import _int18, parse_f64

BAD = "bad"   # a leaf with a missing or non-object node above it: Python raises on reading it


def as_path(member):
    """the path of a member as the binding takes it: a name or a tuple of names"""
    return member if isinstance(member, tuple) else (member,)


def check_paths(paths):
    """the library's argument rules for the paths of one call (AssertionError where it returns DAMPR_ERR_ARG)"""
    from dampr_b200 import device as dev
    assert 1 <= len(paths) <= dev.JSON_MAX_MEMBERS and len(set(paths)) == len(paths)
    for p in paths:
        assert 1 <= len(p) <= dev.JSON_MAX_PATH and (len(p) == 1 or all(p))
    assert len({p[:i] for p in paths for i in range(1, len(p) + 1)}) <= dev.JSON_MAX_NODES


def _skip(s, i):
    return i + len(s[i:]) - len(s[i:].lstrip(WS))


def _members(s, i):
    """the members of the object whose '{' is at s[i], in line order: [(name, escaped, value start, value end)]"""
    out = []
    i = _skip(s, i + 1)
    if s[i] == "}":
        return out
    while True:
        name, j = json.decoder.scanstring(s, i + 1)
        esc = "\\" in s[i + 1:j - 1]
        j = _skip(s, _skip(s, j) + 1)   # past the ':'
        _v, end = _DECODER.raw_decode(s, j)
        out.append((name, esc, j, end))
        i = _skip(s, end)
        if s[i] == "}":
            return out
        i = _skip(s, i + 1)   # past the ','


def device_paths(line, paths, cr_is_data=False):
    """the device's reading of one line (bytes, no '\\n') for the wanted paths (tuples of names): None when the device
    hands it back, else (leaves, nodes). leaves maps each path to (kind, raw text, offset) as device_members gives a
    top-level member, None when its last parent object lacks it, or BAD; nodes maps each interior path to (present,
    is an object) of its last occurrence."""
    if device_members(line, cr_is_data) is None:   # the line rules, the top-level names' escapes included
        return None
    s = line.decode("ascii")
    wanted = {p[:i] for p in paths for i in range(1, len(p) + 1)}
    interior = {p[:i] for p in paths for i in range(1, len(p))}
    last = {}   # path -> its last occurrence's raw text and offset

    def visit(i, prefix):
        for name, esc, j, end in _members(s, i):
            if esc:
                raise LookupError("an escaped name in a compared object")
            p = prefix + (name,)
            if p not in wanted:
                continue
            for q in [q for q in last if q[:len(p)] == p]:
                del last[q]
            last[p] = (s[j:end], j)
            if s[j] == "{" and p in interior:
                visit(j, p)

    try:
        visit(_skip(s, 0), ())
    except LookupError:
        return None
    nodes = {p: (p in last, p in last and last[p][0][0] == "{") for p in interior}
    leaves = {}
    for p in paths:
        if not all(nodes[p[:i]][1] for i in range(1, len(p))):
            leaves[p] = BAD
        elif p not in last:
            leaves[p] = None
        else:
            raw, j = last[p]
            leaves[p] = (_kind(raw), raw[1:-1], j + 1) if raw[0] == '"' else (_kind(raw), raw, j)
    return leaves, nodes


def path_leaf(leaves, names, p):
    """one predicate (device form) over the leaves: True, False or None (undecided)"""
    from dampr_b200 import device as dev
    kind, i, cmp, consts = p
    got = leaves[as_path(names[i])]
    if kind == dev.PRED_MEMBER:
        if got is not BAD:
            return (got is not None) == (cmp == dev.CMP_IN)
        # the container is not an object: Python's `in` on a str container (a member of the call) is the substring
        # test; on anything else it raises
        up = leaves.get(as_path(names[i])[:-1]) if consts else None
        if up is None or up is BAD or up[0] != STR:
            return None
        return (consts[0].encode("utf-8") in up[1].encode("ascii")) == (cmp == dev.CMP_IN)
    if got is None or got is BAD:
        return None
    if kind in (dev.PRED_STR, dev.PRED_INT, dev.PRED_F64) and cmp < dev.CMP_CONTAINS:
        return json_where({"m": got}, [(kind, 0, cmp, consts)], ["m"])
    if got[0] != STR:
        return None
    raw = got[1].encode("ascii")
    return filter_leaf(raw, [raw], (kind, 0, cmp, consts))


def json_path_line(line, spec, names, cr_is_data, preds):
    """fields_json_standin.json_line for members that may be paths: (outcome, flags), outcome False (dropped), None
    (the host's) or (synth, key offset)"""
    from dampr_b200 import device as dev
    _sep, kf, kind, vf, op = spec
    got = device_paths(line, [as_path(n) for n in names], cr_is_data)
    if got is None:
        return None, 0
    leaves = got[0]
    v = verdict(preds, lambda p: path_leaf(leaves, names, p)) if preds else True
    if v is not True:
        return v, 0
    m = {n: None if leaves[as_path(n)] is BAD else leaves[as_path(n)] for n in names}
    flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
    k = m[names[kf]]
    v = None if vf == dev.FIELD_VAL_ONE else m[names[vf]]
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
    val = b""
    if ok and vf != dev.FIELD_VAL_ONE:
        raw = v[1].encode()
        val = b"0" if raw == b"-0" and flt else raw   # float() of a JSON integer is float(int): "-0" is 0.0
        ok = (parse_f64(val) if flt else _int18(val)) is not None
    if not ok:
        return None, flags
    return (k[1].encode() + (b"" if vf == dev.FIELD_VAL_ONE else b"\x01" + val), k[2]), flags


def make_json_path_ctx(free_bytes=1 << 30):
    """make_json_ctx(free_bytes) whose JSON calls also take member paths"""
    from dampr_b200 import device as dev
    ctx = make_json_ctx(free_bytes)
    Json = type(ctx.table(4))
    Plain = next(c for c in Json.__mro__ if c.__name__ == "FieldsTable")

    class JsonPathTable(Json):
        def _json_scan(self, tb, lo, hi, spec, names, cr_is_data, preds, rec):
            check_paths([as_path(n) for n in names])
            self._paths = any(isinstance(n, tuple) and len(n) > 1 for n in names)
            Json._json_scan(self, tb, lo, hi, spec, names, cr_is_data, preds, rec)

        def _json_line(self, line, off, spec, names, cr_is_data, preds, rec):
            if not self._paths:
                return Json._json_line(self, line, off, spec, names, cr_is_data, preds, rec)
            _sep, _kf, kind, vf, op = spec
            got, flags = json_path_line(line, spec, names, cr_is_data, preds)
            self.st["flags"] |= flags
            if got is False:
                if rec is not None:
                    self._put(rec, 0, 0)
                else:
                    self.st["raw"] += 1
            elif got is None:
                self._hand_back(line, off, rec)
            else:
                synth, k_off = got
                Plain._line(self, synth, off + k_off, b"\x01", 0, kind,
                            dev.FIELD_VAL_ONE if vf == dev.FIELD_VAL_ONE else 1, op, cr_is_data, rec)

    ctx.table = lambda log2: JsonPathTable(ctx, log2)
    return ctx

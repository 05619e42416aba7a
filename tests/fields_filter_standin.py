"""The WHERE stand-in of tests/fields_where_standin.py with filter programs (include/dampr_b200.h): and / or / not over
leaves, the string tests (substring, prefix, suffix, length, non-blank) and the whole line as an operand. The tests of
test_text_fields_filter_lowering.py run on it.

Each leaf is True, False or None (the device cannot decide: a missing field, an int() / float() field it does not
parse exactly). Connectives combine left-sequentially, as Python's short circuit does: `a and b` is a when a is False
or None, else b; `a or b` is a when a is True or None, else b; `not` keeps None. The values the program leaves (one
per filter call; a list without connectives leaves one per leaf) are combined the same way with `and`, bottom first.
False drops the line, None hands it to the host, True reads the key and value."""
from fields_standin import device_takes
from fields_where_standin import make_where_ctx, where

WHITESPACE = b"\t\n\x0b\x0c\r\x1c\x1d\x1e\x1f "   # str.split()'s and str.strip()'s ASCII whitespace
_CMPS = [lambda x, c: x == c, lambda x, c: x != c, lambda x, c: x < c, lambda x, c: x <= c, lambda x, c: x > c,
         lambda x, c: x >= c]


def leaf(line, f, p):
    """one leaf over the line (bytes) and its fields f (bytes): True, False or None"""
    from dampr_b200 import device as dev
    kind, i, cmp, consts = p
    if kind not in (dev.PRED_LEN, dev.PRED_NONBLANK) and i != dev.FIELD_LINE and \
            (kind != dev.PRED_STR or cmp < dev.CMP_CONTAINS):
        return where(f, [p])
    if i == dev.FIELD_LINE:
        x = line
    elif not -len(f) <= i < len(f):
        return None
    else:
        x = f[i]
    if kind == dev.PRED_LEN:
        return _CMPS[cmp](len(x), consts[0])
    if kind == dev.PRED_NONBLANK:
        return any(c not in WHITESPACE for c in x)
    if cmp < dev.CMP_CONTAINS:
        return where([x], [(kind, 0, cmp, consts)])
    cs = [c.encode("utf-8") for c in consts]
    if cmp == dev.CMP_CONTAINS:
        return cs[0] in x
    if cmp == dev.CMP_NOT_CONTAINS:
        return cs[0] not in x
    if cmp == dev.CMP_STARTS:
        return any(x.startswith(c) for c in cs)
    return any(x.endswith(c) for c in cs)


def combine(op, a, b=None):
    """left-sequential `and` / `or` of a and b, `not` of a (three values: True, False, None)"""
    if op == "not":
        return None if a is None else not a
    if a is None or a == (op == "or"):
        return a
    return b


def verdict(program, leaf_of):
    """the verdict of a postfix program (device predicates) whose leaves leaf_of(p) decides"""
    from dampr_b200 import device as dev
    names = {dev.PRED_AND: "and", dev.PRED_OR: "or", dev.PRED_NOT: "not"}
    stack = []
    for p in program:
        op = names.get(p[0])
        if op == "not":
            stack.append(combine("not", stack.pop()))
        elif op:
            b = stack.pop()
            stack.append(combine(op, stack.pop(), b))
        else:
            stack.append(leaf_of(p))
    out = True
    for v in stack:
        out = combine("and", out, v)
    return out


def line_verdict(line, f, preds, cr_is_data):
    """the WHERE rule of one line: False (dropped), None (the host's) or True (the key and value decide)"""
    if not device_takes(line, cr_is_data):
        return None
    return verdict(preds, lambda p: leaf(line, f, p)) if preds else True


def make_filter_ctx(free_bytes=1 << 30):
    """make_where_ctx(free_bytes) whose tables take filter programs"""
    ctx = make_where_ctx(free_bytes)
    Where = type(ctx.table(4))
    Base = Where.__mro__[1]

    class FilterTable(Where):
        def _line(self, line, off, sep, kf, kind, vf, op, cr_is_data, rec):
            v = line_verdict(line, line.split(sep), self._preds, cr_is_data)
            if v is False:
                if rec is not None:
                    self._put(rec, 0, 0)
                else:
                    self.st["raw"] += 1
            elif v is None:
                self._hand_back(line, off, rec)
            else:
                Base._line(self, line, off, sep, kf, kind, vf, op, cr_is_data, rec)

    ctx.table = lambda log2: FilterTable(ctx, log2)
    return ctx

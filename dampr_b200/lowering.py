"""Lowering of user lambdas: CPython bytecode -> small expression trees -> closed set of idioms.

The device cannot run Python, and a map left in CPython ingests ~10 MB/s/core (SURVEY §6), so at
graph-run time the planner inspects the user functions of a stage.  A function is lowered only if
its whole body is a straight-line expression over its arguments built from the whitelisted forms
below — anything else (branches, loops, unknown calls, unknown opcodes) returns None and the stage
runs as a host map that feeds the device shuffle.  The analysis is sound by construction: it never
guesses from observed outputs.

Idioms that matter for the five BASELINE configs (SURVEY "Hard parts"):
  x.split()                                   examples/wc.py:12
  set(RX.split(x.lower())), RX = [^\\w]+       benchmarks/tf-idf-dampr.py:12-14
  lambda x: x / lambda x: 1 / x[i] / -x[i]    key and value projections
  lambda x, y: x + y, operator.add, min, max  associative folds (dampr.py:661-708)
  lambda k, it: sum(it) / len(list(it))       group reducers
"""
import builtins
import dis
import operator
import re
import types


class E(object):
    """Expression node."""
    __slots__ = ("op", "a", "b", "c")

    def __init__(self, op, a=None, b=None, c=None):
        self.op, self.a, self.b, self.c = op, a, b, c

    def __repr__(self):
        parts = [repr(x) for x in (self.a, self.b, self.c) if x is not None]
        return "%s(%s)" % (self.op, ", ".join(parts))

    def __eq__(self, other):
        return isinstance(other, E) and (self.op, self.a, self.b, self.c) == (other.op, other.a, other.b, other.c)

    def __hash__(self):
        return hash((self.op, repr(self.a), repr(self.b), repr(self.c)))


# node kinds: arg(i) const(v) obj(pyobject) attr(e, name) call(f, [args]) bin(op, l, r) neg(e)
#             sub(e, idx) tuple([items]) cmp(op, l, r) and(l, r) or(l, r) not(e)
_NULL = object()


_INSTR_CACHE = {}


def _instructions(code):
    """Decoded bytecode of a code object (cached: graphs are rebuilt with fresh lambdas on every run, but
    their code objects are the same, and decoding is the expensive part of the analysis)."""
    ins = _INSTR_CACHE.get(code)
    if ins is None:
        if len(_INSTR_CACHE) > 4096:
            _INSTR_CACHE.clear()
        ins = _INSTR_CACHE[code] = list(dis.get_instructions(code))
    return ins


def analyze(fn):
    """Expression tree of a plain Python function / lambda, or None if it is not a straight-line
    expression over whitelisted opcodes."""
    if not isinstance(fn, types.FunctionType):
        return None
    code = fn.__code__
    if code.co_flags & (0x20 | 0x80 | 0x100 | 0x200):  # generator / coroutine variants
        return None
    if code.co_kwonlyargcount or (code.co_flags & 0x0C):  # *args / **kwargs
        return None
    nargs = code.co_argcount
    argnames = code.co_varnames[:nargs]
    stack = []
    # `a and b` / `a or b` compile to <a> COPY 1; POP_JUMP_IF_FALSE | POP_JUMP_IF_TRUE L; POP_TOP; <b>, merging at L.
    # CPython threads jumps, so several merges can share one L (a and (b or c)) or land on the next COPY ((a and b) or
    # c): pending holds (L, op, a, stack depth) and the merges at L combine innermost first when L is reached.
    pending = []
    ins_list = _instructions(code)
    try:
        for k, ins in enumerate(ins_list):
            while pending and pending[-1][0] == ins.offset:
                _at, bop, lhs, depth = pending.pop()
                if len(stack) != depth + 1:
                    return None
                stack.append(E(bop, lhs, stack.pop()))
            if pending and pending[-1][0] < ins.offset:
                return None
            name = ins.opname
            if name in ("RESUME", "NOP", "COPY_FREE_VARS", "MAKE_CELL", "PRECALL", "CACHE"):
                continue
            if name == "COPY" and ins.arg == 1:
                nxt = ins_list[k + 1] if k + 2 < len(ins_list) else None
                if nxt is None or nxt.opname not in ("POP_JUMP_IF_FALSE", "POP_JUMP_IF_TRUE") or \
                        ins_list[k + 2].opname != "POP_TOP" or not nxt.argval > nxt.offset or \
                        (pending and nxt.argval > pending[-1][0]):
                    return None
                lhs = stack.pop()
                pending.append((nxt.argval, "and" if nxt.opname == "POP_JUMP_IF_FALSE" else "or", lhs, len(stack)))
                continue
            if name in ("POP_JUMP_IF_FALSE", "POP_JUMP_IF_TRUE", "POP_TOP") and k >= 1 and \
                    ins_list[k - 1 if name != "POP_TOP" else k - 2].opname == "COPY" and \
                    ins_list[k - 1 if name != "POP_TOP" else k - 2].arg == 1:
                continue   # the rest of a short-circuit pattern (taken above)
            if name == "UNARY_NOT":
                stack.append(E("not", stack.pop()))
                continue
            if pending and name in ("RETURN_VALUE", "RETURN_CONST"):
                return None
            if name in ("LOAD_FAST", "LOAD_FAST_CHECK"):
                if ins.argval not in argnames:
                    return None
                stack.append(E("arg", argnames.index(ins.argval)))
            elif name == "LOAD_CONST":
                stack.append(E("const", ins.argval))
            elif name == "RETURN_CONST":
                return E("const", ins.argval)
            elif name == "LOAD_GLOBAL":
                if ins.arg & 1:
                    stack.append(_NULL)
                gname = ins.argval
                if gname in fn.__globals__:
                    stack.append(E("obj", fn.__globals__[gname]))
                elif hasattr(builtins, gname):
                    stack.append(E("obj", getattr(builtins, gname)))
                else:
                    return None
            elif name == "LOAD_DEREF":
                idx = (code.co_cellvars + code.co_freevars).index(ins.argval) - len(code.co_cellvars)
                if idx < 0 or fn.__closure__ is None:
                    return None
                stack.append(E("obj", fn.__closure__[idx].cell_contents))
            elif name == "PUSH_NULL":
                stack.append(_NULL)
            elif name == "LOAD_ATTR":
                obj = stack.pop()
                if ins.arg & 1:
                    stack.append(_NULL)
                stack.append(E("attr", obj, ins.argval))
            elif name == "LOAD_METHOD":
                obj = stack.pop()
                stack.append(_NULL)
                stack.append(E("attr", obj, ins.argval))
            elif name == "CALL":
                n = ins.arg
                args = stack[len(stack) - n:] if n else []
                del stack[len(stack) - n:]
                f = stack.pop()
                if stack and stack[-1] is _NULL:
                    stack.pop()
                if any(a is _NULL for a in args) or f is _NULL:
                    return None
                stack.append(E("call", f, tuple(args)))
            elif name == "BINARY_OP":
                r = stack.pop()
                l = stack.pop()
                stack.append(E("bin", ins.argrepr.rstrip("="), l, r))
            elif name == "BINARY_SUBSCR":
                i = stack.pop()
                o = stack.pop()
                stack.append(E("sub", o, i))
            elif name == "UNARY_NEGATIVE":
                stack.append(E("neg", stack.pop()))
            elif name == "BUILD_TUPLE":
                n = ins.arg
                items = tuple(stack[len(stack) - n:]) if n else ()
                del stack[len(stack) - n:]
                stack.append(E("tuple", items))
            elif name == "COMPARE_OP":
                r = stack.pop()
                l = stack.pop()
                stack.append(E("cmp", ins.argval, l, r))
            elif name == "CONTAINS_OP":
                r = stack.pop()
                l = stack.pop()
                stack.append(E("cmp", "not in" if ins.arg else "in", l, r))
            elif name == "RETURN_VALUE":
                out = stack.pop()
                return None if out is _NULL else out
            else:
                return None
    except (IndexError, ValueError, AttributeError):
        return None
    return None


# ---- idiom matchers ----------------------------------------------------------------------------
def _is_arg(e, i=0):
    return isinstance(e, E) and e.op == "arg" and e.a == i


def _const(e):
    """(True, value) if e is a constant."""
    if isinstance(e, E) and e.op == "const":
        return True, e.a
    return False, None


def is_identity(fn):
    e = analyze(fn)
    return e is not None and _is_arg(e, 0) and fn.__code__.co_argcount == 1


def constant_value(fn):
    """(True, v) if fn ignores its argument and returns the constant v."""
    e = analyze(fn)
    if e is None:
        return False, None
    return _const(e)


_NONWORD_PATTERNS = (r"[^\w]+", r"\W+")


def _is_nonword_pattern(obj):
    return isinstance(obj, re.Pattern) and obj.pattern in _NONWORD_PATTERNS and \
        (obj.flags & ~re.UNICODE) == 0


def _is_lower_of_arg(e):
    return isinstance(e, E) and e.op == "call" and e.b == () and isinstance(e.a, E) and \
        e.a.op == "attr" and e.a.b == "lower" and _is_arg(e.a.a)


def _is_nonword_split(e):
    """RX.split(x.lower()) or re.split(PATTERN, x.lower())"""
    if not (isinstance(e, E) and e.op == "call"):
        return False
    f, args = e.a, e.b
    if isinstance(f, E) and f.op == "attr" and f.b == "split" and isinstance(f.a, E) and f.a.op == "obj":
        if _is_nonword_pattern(f.a.a) and len(args) == 1 and _is_lower_of_arg(args[0]):
            return True
        if f.a.a is re and len(args) == 2:
            ok, pat = _const(args[0])
            return ok and pat in _NONWORD_PATTERNS and _is_lower_of_arg(args[1])
    if isinstance(f, E) and f.op == "obj" and f.a is re.split and len(args) == 2:
        ok, pat = _const(args[0])
        return ok and pat in _NONWORD_PATTERNS and _is_lower_of_arg(args[1])
    return False


TOK_WS, TOK_NONWORD_LOWER_SET, TOK_NONWORD_LOWER = 0, 1, 2


def tokenizer_mode(fn):
    """Device tokeniser mode of a flat_map function over a text line, or None."""
    e = analyze(fn)
    if e is None or fn.__code__.co_argcount != 1:
        return None
    # x.split()
    if e.op == "call" and e.b == () and isinstance(e.a, E) and e.a.op == "attr" and e.a.b == "split" \
            and _is_arg(e.a.a):
        return TOK_WS
    if _is_nonword_split(e):
        return TOK_NONWORD_LOWER
    if e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and e.a.a in (set, frozenset) \
            and len(e.b) == 1 and _is_nonword_split(e.b[0]):
        return TOK_NONWORD_LOWER_SET
    return None


FIELD_STR, FIELD_INT, FIELD_FLOAT = "str", "int", "float"


SEP_WS = "<whitespace>"   # the separator of `x.split()`: runs of whitespace (never a one-character separator)


def _split_sep(e, whitespace=False):
    """S if e is `x.split(S)` over the argument with a one-character ASCII separator other than '\\n', '\\r' and NUL
    (the bytes that end or cannot appear in a device line); with `whitespace`, SEP_WS if e is `x.split()` or
    `x.split(None)`; else None. Keyword forms (sep=, maxsplit=) do not reach here: analyze() refuses them."""
    if isinstance(e, E) and e.op == "call" and len(e.b) <= 1 and isinstance(e.a, E) and e.a.op == "attr" \
            and e.a.b == "split" and _is_arg(e.a.a):
        if not e.b:
            return SEP_WS if whitespace else None
        ok, s = _const(e.b[0])
        if ok and s is None:
            return SEP_WS if whitespace else None
        if ok and type(s) is str and len(s) == 1 and s.isascii() and s not in "\n\r\0":
            return s
    return None


def _field_proj(e, record):
    """(kind, i) if e is record(e')[i] (FIELD_STR) or int(record(e')[i]) (FIELD_INT) with a constant int i; record(x)
    says whether x is the split record and returns its separator (any non-None value)"""
    kind = FIELD_STR
    if isinstance(e, E) and e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and e.a.a is int \
            and len(e.b) == 1:
        kind, e = FIELD_INT, e.b[0]
    if not (isinstance(e, E) and e.op == "sub"):
        return None
    ok, i = _const(e.b)
    if not ok or type(i) is not int or not -(1 << 30) <= i < (1 << 30):
        return None
    sep = record(e.a)
    return None if sep is None else (kind, i, sep)


def _value_proj(e, record):
    """(kind, j, sep) if e is int(record(e')[j]) (FIELD_INT) or float(record(e')[j]) (FIELD_FLOAT), else None"""
    if isinstance(e, E) and e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and e.a.a is float \
            and len(e.b) == 1:
        p = _field_proj(e.b[0], record)
        return None if p is None or p[0] != FIELD_STR else (FIELD_FLOAT, p[1], p[2])
    p = _field_proj(e, record)
    return p if p is not None and p[0] == FIELD_INT else None


def _inline_call_of_arg(e):
    """analyze(f) for e = f(x), x the argument and f a one-argument Python function (mean()'s `value(v)`): f's body
    is then already an expression over x"""
    if isinstance(e, E) and e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and len(e.b) == 1 \
            and _is_arg(e.b[0]) and isinstance(e.a.a, types.FunctionType) and e.a.a.__code__.co_argcount == 1:
        return analyze(e.a.a)
    return None


def _is_one(e):
    ok, v = _const(e)
    return ok and type(v) is int and v == 1


FIELD_TUPLE = "tuple"   # a key that is a tuple of field projections
TUPLE_MAX = 4           # components of a tuple key the device takes (DAMPR_FIELD_KEYS_MAX)


def text_fields_spec(key_fn, value_fn, split_fn=None, whitespace=False, tuple_keys=False):
    """Device field-scan spec of a keyed(key_fn, value_fn) over text lines, optionally behind map(split_fn):
    (sep, key_index, key_kind, value_index, value_kind, mean) where the key is l.split(sep)[key_index] (FIELD_STR) or
    its int() (FIELD_INT), and the value is
      the constant 1                                   value_index None, FIELD_INT, mean False
      int() or float() of l.split(sep)[value_index]    FIELD_INT or FIELD_FLOAT, mean False
      mean()'s `(value(v), 1)`, value one of those     FIELD_INT or FIELD_FLOAT, mean True
    Indices may be negative (Python's from-the-end). With `whitespace` the split may also be l.split() / l.split(None),
    sep SEP_WS (a caller that only handles separator characters leaves it off). With `tuple_keys` the key may also be
    a tuple of 1 .. TUPLE_MAX such projections on the same split, e.g. (l.split(S)[0], int(l.split(S)[3])): key_kind
    is then FIELD_TUPLE and key_index the components ((index, FIELD_STR | FIELD_INT), ...). None for any other
    shape."""
    fns = [f for f in (key_fn, value_fn, split_fn) if f is not None]
    if not all(isinstance(f, types.FunctionType) and f.__code__.co_argcount == 1 for f in fns):
        return None
    ke, ve = analyze(key_fn), analyze(value_fn)
    if ke is None or ve is None:
        return None
    if split_fn is None:
        def record(x):                           # the split is inside the key / value functions
            return _split_sep(x, whitespace)
    else:
        sep = _split_sep(analyze(split_fn), whitespace)
        if sep is None:
            return None

        def record(x):                           # key / value functions index the split record
            return sep if _is_arg(x) else None
    k = _field_proj(ke, record)
    if k is None and tuple_keys and ke.op == "tuple" and 1 <= len(ke.a) <= TUPLE_MAX:
        comps = [_field_proj(c, record) for c in ke.a]
        if any(c is None for c in comps) or len({c[2] for c in comps}) != 1:
            return None
        k = FIELD_TUPLE, tuple((i, kind) for kind, i, _sep in comps), comps[0][2]
    if k is None:
        return None
    if _is_one(ve):
        return k[2], k[1], k[0], None, FIELD_INT, False
    mean = ve.op == "tuple" and len(ve.a) == 2
    if mean:
        inner = _inline_call_of_arg(ve.a[0])
        if inner is None or not _is_one(ve.a[1]):
            return None
        ve = inner
    v = _value_proj(ve, record)
    if v is None or v[2] != k[2]:
        return None
    return k[2], k[1], k[0], v[1], v[0], mean


FIELD_COUNT = "nfields"
_FLIP = {"==": "==", "!=": "!=", "<": ">", "<=": ">=", ">": "<", ">=": "<="}
PRED_MAX, PRED_MAX_CONSTS, PRED_MAX_BYTES = 8, 64, 1024   # the device's limits per stage (include/dampr_b200.h)


def _pred_const(e):
    """(True, value) for a constant or a closure / global object"""
    if isinstance(e, E) and e.op in ("const", "obj"):
        return True, e.a
    return False, None


def field_predicate(fn, record=None, whitespace=False):
    """Device WHERE predicate of a `filter(fn)` in front of a field fold, or None. `record` is None when fn takes the
    text line and splits it itself (l.split(S)), else the separator S of the map(lambda l: l.split(S)) fn runs after.
    With `whitespace` fn's own split may also be l.split() / l.split(None) (sep SEP_WS).
    Returns (sep, kind, index, op, constants), with R the split record, for
      F op C, C op F   F = R[i] (FIELD_STR), int(R[i]) (FIELD_INT) or float(R[i]) (FIELD_FLOAT), op one of
                       == != < <= > >= (C op F comes back as F op' C); C a str for a str field, an int in int64 (not a
                       bool) for an int field, a float or an int with |C| <= 2^53 (returned as a float) for a float
                       field
      F in K, F not in K   F = R[i] or int(R[i]); K a tuple / frozenset / set / list, literal or bound to a closure or
                       global name (the members are read now), of 1 .. PRED_MAX_CONSTS members that are all str (a str
                       field) or all int in int64 (an int field); constants is K's members
      len(R) op n      kind FIELD_COUNT, index None, n an int (not a bool)
    Everything else (and / or / not, chained comparisons, methods, raw-line tests, mixed types) is None."""
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return None
    e = analyze(fn)
    if e is None or e.op != "cmp":
        return None
    return _field_leaf(e, _record_of(record, whitespace))


def _record_of(record, whitespace):
    """record(x) of a filter over the line (record None: its own l.split(S)) or over the split record of sep record"""
    if record is None:
        return lambda x: _split_sep(x, whitespace)
    return lambda x: record if _is_arg(x) else None


def _field_leaf(e, rec):
    """field_predicate's result for the comparison tree e"""
    op, l, r = e.a, e.b, e.c
    if op in _FLIP and _pred_const(l)[0] and not _pred_const(r)[0]:
        op, l, r = _FLIP[op], r, l
    ok, c = _pred_const(r)
    if not ok:
        return None
    if isinstance(l, E) and l.op == "call" and isinstance(l.a, E) and l.a.op == "obj" and l.a.a is len \
            and len(l.b) == 1:
        sep = rec(l.b[0])
        if sep is None or op not in _FLIP or type(c) is not int:
            return None
        return sep, FIELD_COUNT, None, op, (c,)
    p = _value_proj(l, rec) or _field_proj(l, rec)
    if p is None:
        return None
    kind, i, sep = p
    if op in ("in", "not in"):
        if kind == FIELD_FLOAT or type(c) not in (tuple, frozenset, set, list) or \
                not 1 <= len(c) <= PRED_MAX_CONSTS:
            return None
        consts = tuple(c)
    elif op in _FLIP:
        consts = (c,)
    else:
        return None
    if kind == FIELD_STR:
        if not all(type(m) is str for m in consts):
            return None
        try:
            if sum(len(m.encode("utf-8")) for m in consts) > PRED_MAX_BYTES:
                return None
        except UnicodeEncodeError:   # a lone surrogate: no UTF-8 bytes to compare
            return None
    elif kind == FIELD_INT:
        if not all(type(m) is int and -(1 << 63) <= m < (1 << 63) for m in consts):
            return None
    else:
        v = consts[0]
        if type(v) is int and abs(v) <= (1 << 53):
            consts = (float(v),)
        elif type(v) is not float:
            return None
    return sep, kind, i, op, consts


# ---- JSON lines: Dampr.json(path) = map(json.loads) in front of the fold ----------------------------------------
FIELD_DATA = "data"       # a bare r["m"]: its Python type is the JSON value's, decided by the data
FIELD_MEMBER = "member"   # "m" in r / "m" not in r


def is_json_loads(fn):
    """True for json.loads itself (Dampr.json's mapper) and for `lambda l: json.loads(l)`"""
    import json
    if fn is json.loads:
        return True
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return False
    e = analyze(fn)
    if e is None or e.op != "call" or len(e.b) != 1 or not _is_arg(e.b[0]) or not isinstance(e.a, E):
        return False
    f = e.a
    if f.op == "attr" and isinstance(f.a, E) and f.a.op == "obj":   # json.loads(l)
        return getattr(f.a.a, f.b, None) is json.loads
    return f.op == "obj" and f.a is json.loads                      # loads(l) after `from json import loads`


def json_member_name(name):
    """True if the device matches member `name` by its bytes: ASCII, at most 64 bytes, no '"', '\\' or control
    character (a JSON line spells every other name with an escape, or cannot hold it)"""
    return type(name) is str and len(name) <= 64 and all(0x20 <= ord(c) < 0x80 for c in name) and \
        '"' not in name and "\\" not in name


def _member(e):
    """(kind, name) if e is r["m"] (FIELD_DATA), int(r["m"]) (FIELD_INT) or float(r["m"]) (FIELD_FLOAT) over the
    argument r with a constant name the device matches, else None"""
    kind = FIELD_DATA
    if isinstance(e, E) and e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and e.a.a in (int, float) \
            and len(e.b) == 1:
        kind, e = FIELD_INT if e.a.a is int else FIELD_FLOAT, e.b[0]
    if not (isinstance(e, E) and e.op == "sub" and _is_arg(e.a)):
        return None
    ok, name = _const(e.b)
    return (kind, name) if ok and json_member_name(name) else None


JSON_MAX_PATH = 4   # names per member path (DAMPR_JSON_MAX_PATH)


def _path(e):
    """(kind, path) if e is r[n1]..[nk] (FIELD_DATA), int() (FIELD_INT) or float() (FIELD_FLOAT) of it over the
    argument r, path the tuple of 1 .. JSON_MAX_PATH constant names the device matches (none empty in a path of two or
    more: the device cannot name them), else None. Array indices (r["a"][0]) and r.get are None."""
    kind = FIELD_DATA
    if isinstance(e, E) and e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and e.a.a in (int, float) \
            and len(e.b) == 1:
        kind, e = FIELD_INT if e.a.a is int else FIELD_FLOAT, e.b[0]
    names = []
    while isinstance(e, E) and e.op == "sub" and len(names) <= JSON_MAX_PATH:
        ok, name = _const(e.b)
        if not ok or not json_member_name(name):
            return None
        names.append(name)
        e = e.a
    if not _is_arg(e) or not 1 <= len(names) <= JSON_MAX_PATH or (len(names) > 1 and not all(names)):
        return None
    return kind, tuple(reversed(names))


def json_fields_spec(key_fn, value_fn):
    """Device JSON-lines spec of a keyed(key_fn, value_fn) behind map(json.loads): (key name, key kind, value name,
    value kind, mean) where the key is r["k"] (FIELD_DATA) or int(r["k"]) (FIELD_INT), and the value is
      the constant 1                                        value name None, FIELD_INT, mean False
      r["v"] (FIELD_DATA), int(r["v"]) or float(r["v"])     mean False
      mean()'s `(value(r), 1)`, value one of those          mean True
    None for any other shape (r.get, r["a"]["b"], tuple keys, float keys, ...)."""
    return _json_spec(key_fn, value_fn, _member)


def json_fields_path_spec(key_fn, value_fn):
    """json_fields_spec over member paths: the key r[n1]..[nk] or int() of it, the value 1, r[n1]..[nk], int() or
    float() of it (or mean()'s pair), 1 <= k <= JSON_MAX_PATH, each name a tuple of names. None unless the key or the
    value is a path of two or more names (json_fields_spec takes the rest)."""
    spec = _json_spec(key_fn, value_fn, _path)
    if spec is None or not any(p is not None and len(p) > 1 for p in (spec[0], spec[2])):
        return None
    return spec


def _json_spec(key_fn, value_fn, member):
    """json_fields_spec's result with member(e) reading the key's and the value's members"""
    fns = (key_fn, value_fn)
    if not all(isinstance(f, types.FunctionType) and f.__code__.co_argcount == 1 for f in fns):
        return None
    ke, ve = analyze(key_fn), analyze(value_fn)
    if ke is None or ve is None:
        return None
    k = member(ke)
    if k is None or k[0] == FIELD_FLOAT:
        return None
    if _is_one(ve):
        return k[1], k[0], None, FIELD_INT, False
    mean = ve.op == "tuple" and len(ve.a) == 2
    if mean:
        inner = _inline_call_of_arg(ve.a[0])
        if inner is None or not _is_one(ve.a[1]):
            return None
        ve = inner
    v = member(ve)
    if v is None:
        return None
    return k[1], k[0], v[1], v[0], mean


def json_predicate(fn):
    """Device WHERE predicate of a `filter(fn)` behind map(json.loads), or None. Returns (kind, name, op, constants):
      "m" in r, "m" not in r   kind FIELD_MEMBER, constants ()
      M op C, C op M           M = r["m"] with C a str (kind FIELD_STR) or an int in int64, not a bool (FIELD_INT);
                               M = int(r["m"]) with C such an int (FIELD_INT); M = float(r["m"]) with C a float or an
                               int with |C| <= 2^53 (FIELD_FLOAT, C returned as a float); op one of == != < <= > >=
      M in K, M not in K       M = r["m"] or int(r["m"]); K a tuple / frozenset / set / list (literal, closure or
                               global) of 1 .. PRED_MAX_CONSTS members, all str (r["m"] only) or all int in int64
    A bare r["m"] against a float constant, and everything field_predicate refuses, is None."""
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return None
    e = analyze(fn)
    if e is None or e.op != "cmp":
        return None
    return _json_leaf(e)


def _json_leaf(e, paths=False):
    """json_predicate's result for the comparison tree e; with `paths` the members are _path's paths, and
    "m" in r[n1]..[nk] (1 <= k < JSON_MAX_PATH) is (FIELD_MEMBER, (n1, .., nk, m), op, ("m",)): Python's `in` on
    whatever r[n1]..[nk] is, membership where it is an object and the substring test where it is a str"""
    op, l, r = e.a, e.b, e.c
    if op in ("in", "not in") and _is_arg(r):
        ok, name = _const(l)
        return (FIELD_MEMBER, name, op, ()) if ok and json_member_name(name) else None
    if paths and op in ("in", "not in"):
        under = _path(r)
        if under is not None and under[0] == FIELD_DATA:
            ok, name = _const(l)
            m = _path(E("sub", r, E("const", name))) if ok else None
            return None if m is None else (FIELD_MEMBER, m[1], op, (name,))
    if op in _FLIP and _pred_const(l)[0] and not _pred_const(r)[0]:
        op, l, r = _FLIP[op], r, l
    ok, c = _pred_const(r)
    m = _path(l) if paths else _member(l)
    if not ok or m is None:
        return None
    kind, name = m
    if op in ("in", "not in"):
        if kind == FIELD_FLOAT or type(c) not in (tuple, frozenset, set, list) or not 1 <= len(c) <= PRED_MAX_CONSTS:
            return None
        consts = tuple(c)
    elif op in _FLIP:
        consts = (c,)
    else:
        return None
    if kind == FIELD_DATA:
        if all(type(x) is str for x in consts):
            kind = FIELD_STR
        elif all(type(x) is int for x in consts):
            kind = FIELD_INT
        else:
            return None
    if kind == FIELD_STR:
        try:
            if sum(len(x.encode("utf-8")) for x in consts) > PRED_MAX_BYTES:
                return None
        except UnicodeEncodeError:   # a lone surrogate: no UTF-8 bytes to compare
            return None
    elif kind == FIELD_INT:
        if not all(type(x) is int and -(1 << 63) <= x < (1 << 63) for x in consts):
            return None
    else:
        v = consts[0]
        if type(v) is int and abs(v) <= (1 << 53):
            consts = (float(v),)
        elif type(v) is not float:
            return None
    return kind, name, op, consts


# ---- filter programs: and / or / not over leaves, string tests, whole-line tests ---------------------------------
LINE = "line"                     # the index of a leaf whose operand is the whole line
FIELD_LEN = "len"                 # len(X) op n
FIELD_NONBLANK = "nonblank"       # X.strip() as a truth value
STR_TESTS = ("contains", "not contains", "startswith", "endswith")
PRED_MAX_OPS = 8                  # connectives per stage (DAMPR_PRED_MAX_OPS)


def _str_consts(consts):
    """consts if every member is a str whose UTF-8 bytes exist (no lone surrogate), else None"""
    if not all(type(c) is str for c in consts):
        return None
    try:
        for c in consts:
            c.encode("utf-8")
    except UnicodeEncodeError:
        return None
    return tuple(consts)


def _str_leaf(e, operand):
    """(op, kind, operand index, consts) for a string test over a str operand: S in X, S not in X, X.startswith(S),
    X.endswith(S) (S a str, or for the last two a tuple of str: a list raises TypeError in Python), len(X) op n /
    n op len(X), and X.strip() as a truth value; operand(x) gives X's index (a field, LINE, a member) or None"""
    if e.op == "cmp" and e.a in ("in", "not in"):
        ok, s = _pred_const(e.b)
        i = operand(e.c)
        if ok and i is not None and type(s) is str and _str_consts((s,)):
            return "contains" if e.a == "in" else "not contains", FIELD_STR, i, (s,)
        return None
    if e.op == "cmp" and e.a in _FLIP:
        op, l, r = e.a, e.b, e.c
        if _pred_const(l)[0] and not _pred_const(r)[0]:
            op, l, r = _FLIP[op], r, l
        ok, n = _pred_const(r)
        if ok and type(n) is int and isinstance(l, E) and l.op == "call" and _callee(l.a) is len and \
                len(l.b) == 1 and -(1 << 63) <= n < (1 << 63):
            i = operand(l.b[0])
            return None if i is None else (op, FIELD_LEN, i, (n,))
        return None
    if e.op == "call" and isinstance(e.a, E) and e.a.op == "attr" and e.a.b in ("startswith", "endswith", "strip"):
        i = operand(e.a.a)
        if i is None:
            return None
        if e.a.b == "strip":
            return (None, FIELD_NONBLANK, i, ()) if e.b == () else None
        if len(e.b) != 1:
            return None
        ok, s = _pred_const(e.b[0])
        if not ok:
            return None
        consts = _str_consts((s,)) if type(s) is str else \
            _str_consts(s) if type(s) is tuple and 1 <= len(s) <= PRED_MAX_CONSTS else None
        return None if consts is None else (e.a.b, FIELD_STR, i, consts)
    return None


def _program(e, leaf):
    """postfix list of a filter's tree: leaf(x) of every leaf ("and" / "or" / "not" for the connectives), or None when
    a leaf is not one, or the program passes the device's limits"""
    out = []

    def walk(x):
        if not isinstance(x, E):
            return False
        if x.op in ("and", "or"):
            if not (walk(x.a) and walk(x.b)):
                return False
            out.append(x.op)
            return True
        if x.op == "not":
            if not walk(x.a):
                return False
            out.append("not")
            return True
        got = leaf(x)
        if got is None:
            return False
        out.append(got)
        return True

    if not walk(e):
        return None
    return out if _within_limits(out) else None


def _within_limits(prog):
    """the leaves, connectives, constants and string bytes of a program (or a stage's) fit the device"""
    leaves = [x for x in prog if not isinstance(x, str)]
    strs = [c for x in leaves for c in x[-1] if type(c) is str]
    return len(leaves) <= PRED_MAX and len(prog) - len(leaves) <= PRED_MAX_OPS and \
        sum(len(x[-1]) for x in leaves) <= PRED_MAX_CONSTS and sum(len(c.encode("utf-8")) for c in strs) <= PRED_MAX_BYTES


def filter_program(fn, record=None, whitespace=False):
    """Device WHERE program of a `filter(fn)` in front of a field fold, or None: the postfix list of its leaves and
    connectives ("and", "or", "not"), fn's body being and / or / not over leaves. A leaf is field_predicate's result
    (sep, kind, index, op, constants) for field_predicate's shapes, and, with X a str field R[i] or (record None: fn
    takes the line) the line itself (index LINE, sep None):
      S in X, S not in X                op "contains" / "not contains", kind FIELD_STR, constants (S,)
      X.startswith(S), X.endswith(S)    op "startswith" / "endswith", FIELD_STR, S a str or a tuple of str
      len(X) op n                       kind FIELD_LEN, constants (n,), n an int (not a bool)
      X.strip() as a truth value        kind FIELD_NONBLANK, op None, constants ()
      X op S, X in K                    the line under field_predicate's str comparisons
    The limits are the device's: PRED_MAX leaves, PRED_MAX_OPS connectives, PRED_MAX_CONSTS constants and
    PRED_MAX_BYTES bytes of str constants. Bare truthiness (lambda l: l), `S in r` over the split record, a field
    inside a str constant (r[0] in "abc"), conditional expressions and chained comparisons are None."""
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return None
    e = analyze(fn)
    if e is None:
        return None
    rec = _record_of(record, whitespace)

    def operand(x):   # (sep, index) of a str operand
        if record is None and _is_arg(x):
            return None, LINE
        p = _field_proj(x, rec)
        return (p[2], p[1]) if p is not None and p[0] == FIELD_STR else None

    def leaf(x):
        if x.op == "cmp":
            p = _field_leaf(x, rec)
            if p is not None:
                return p
            if record is None and x.a in ("in", "not in") + tuple(_FLIP) and \
                    (_is_arg(x.b) or (_is_arg(x.c) and x.a in _FLIP)):
                line = _line_cmp(x)
                if line is not None:
                    return line
        got = _str_leaf(x, operand)
        if got is None:
            return None
        op, kind, (sep, i), consts = got
        return sep, kind, i, op, consts

    return _program(e, leaf)


def _line_cmp(e):
    """(None, FIELD_STR, LINE, op, constants) for the line l compared with str constants: l op S, S op l, l in K"""
    op, l, r = e.a, e.b, e.c
    if op in _FLIP and _pred_const(l)[0] and _is_arg(r):
        op, l, r = _FLIP[op], r, l
    ok, c = _pred_const(r)
    if not ok or not _is_arg(l):
        return None
    if op in ("in", "not in"):
        if type(c) not in (tuple, frozenset, set, list) or not 1 <= len(c) <= PRED_MAX_CONSTS:
            return None
        consts = _str_consts(tuple(c))
    else:
        consts = _str_consts((c,))
    return None if consts is None else (None, FIELD_STR, LINE, op, consts)


def json_filter_program(fn):
    """Device WHERE program of a `filter(fn)` behind map(json.loads), or None: the postfix list of json_predicate's
    leaves (kind, name, op, constants) and of the string tests of filter_program over a member M = r["m"] (the
    member's name in place of an index; the device decides them on a string member without escapes only), with the
    connectives "and", "or", "not" between them"""
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return None
    e = analyze(fn)
    if e is None:
        return None
    return _program(e, _json_program_leaf)


def json_path_filter_program(fn):
    """The program of a filter in a stage that reads member paths: json_filter_program over paths r[n1]..[nk]
    (1 <= k <= JSON_MAX_PATH, each name a tuple of names), its leaves and string tests on paths, and
    "m" in r[n1]..[nk] / "m" not in r[n1]..[nk] for k >= 1 as _json_leaf gives them (the path (n1, .., nk, m) with the
    constant ("m",): the device decides membership where r[n1]..[nk] is an object, the substring test where it is a
    str without escapes). A name the device cannot match keeps json_filter_program's substring leaf on r["a"] and is
    refused deeper. None unless some leaf reads a path of two or more names."""
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return None
    e = analyze(fn)
    if e is None:
        return None

    def leaf(x):
        if x.op == "cmp":
            p = _json_leaf(x, paths=True)
            if p is not None:
                kind, name, op, consts = p
                return kind, name if isinstance(name, tuple) else (name,), op, consts
        p = _json_program_leaf(x)
        if p is not None:
            kind, name, op, consts = p
            return kind, (name,), op, consts
        return _json_program_leaf(x, paths=True)

    prog = _program(e, leaf)
    if prog is None or not any(not isinstance(x, str) and len(x[1]) > 1 for x in prog):
        return None
    return prog


def _json_program_leaf(x, paths=False):
    """a leaf of json_filter_program (kind, name, op, constants), or None; with `paths` over _path's paths"""
    def operand(y):
        m = _path(y) if paths else _member(y)
        return m[1] if m is not None and m[0] == FIELD_DATA else None

    if x.op == "cmp":
        p = _json_leaf(x, paths)
        if p is not None or (paths and x.a in ("in", "not in")):   # S in r[n1]..[nk] is membership, not a substring
            return p
    got = _str_leaf(x, operand)
    if got is None:
        return None
    op, kind, name, consts = got
    return kind, name, op, consts


def field_index(fn):
    """i if fn is `lambda x: x[i]` with a constant non-negative int i, else None."""
    e = analyze(fn)
    return _field(e)


def _field(e):
    if isinstance(e, E) and e.op == "sub" and _is_arg(e.a):
        ok, i = _const(e.b)
        if ok and type(i) is int and i >= 0:
            return i
    return None


def projection(fn):
    """Numeric projection of one record: ('field', i, sign) for x[i] / -x[i], ('ident', None, sign)
    for x / -x, ('const', v, 1) for constants; None otherwise."""
    e = analyze(fn)
    if e is None or fn.__code__.co_argcount != 1:
        return None
    sign = 1
    if e.op == "neg":
        sign, e = -1, e.a
    i = _field(e)
    if i is not None:
        return ("field", i, sign)
    if _is_arg(e):
        return ("ident", None, sign)
    ok, v = _const(e)
    if ok and sign == 1:
        return ("const", v, 1)
    return None


ADD, MIN, MAX, FIRST, LAST = "add", "min", "max", "first", "last"


def binop_kind(fn):
    """Kind of an associative binary operator, or None."""
    if fn is operator.add:
        return ADD
    if fn is min:
        return MIN
    if fn is max:
        return MAX
    e = analyze(fn)
    if e is None or getattr(fn, "__code__", None) is None or fn.__code__.co_argcount != 2:
        return None
    if e.op == "bin" and e.a == "+" and ((_is_arg(e.b, 0) and _is_arg(e.c, 1)) or (_is_arg(e.b, 1) and _is_arg(e.c, 0))):
        return ADD
    if e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and len(e.b) == 2 and \
            {x.a for x in e.b if isinstance(x, E) and x.op == "arg"} == {0, 1}:
        if e.a.a is min:
            return MIN
        if e.a.a is max:
            return MAX
        if e.a.a is operator.add:
            return ADD
    if _is_arg(e, 0):
        return FIRST
    if _is_arg(e, 1):
        return LAST
    return None


def tuple_binop_kinds(fn):
    """[kind per component] of a component-wise binary operator over tuples, e.g. mean()'s
    `lambda x, y: (x[0] + y[0], x[1] + y[1])` (dampr.py:450-467) -> [ADD, ADD]; None otherwise."""
    e = analyze(fn)
    if e is None or getattr(fn, "__code__", None) is None or fn.__code__.co_argcount != 2 or e.op != "tuple":
        return None
    out = []
    for i, comp in enumerate(e.a):
        if not (isinstance(comp, E) and comp.op == "bin" and comp.a == "+"):
            return None
        sides = []
        for side in (comp.b, comp.c):
            if not (isinstance(side, E) and side.op == "sub" and isinstance(side.a, E) and side.a.op == "arg"):
                return None
            ok, j = _const(side.b)
            if not ok or j != i:
                return None
            sides.append(side.a.a)
        if sorted(sides) != [0, 1]:
            return None
        out.append(ADD)
    return out or None


SUM, COUNT = "sum", "count"


def group_reducer_kind(fn):
    """Kind of a group reducer f(key, values_iter): sum(it) / len(list(it)) / min(it) / max(it)."""
    e = analyze(fn)
    if e is None or fn.__code__.co_argcount != 2:
        return None
    if e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and len(e.b) == 1:
        f, a = e.a.a, e.b[0]
        if _is_arg(a, 1):
            if f is sum:
                return SUM
            if f is min:
                return MIN
            if f is max:
                return MAX
        if f is len and isinstance(a, E) and a.op == "call" and isinstance(a.a, E) and a.a.op == "obj" \
                and a.a.a in (list, tuple) and len(a.b) == 1 and _is_arg(a.b[0], 1):
            return COUNT
    return None


def _iter_fold_kind(e, argi):
    """kind of sum(arg) / min(arg) / max(arg) / len(list(arg)) over argument `argi`, else None"""
    if not (isinstance(e, E) and e.op == "call" and isinstance(e.a, E) and e.a.op == "obj" and len(e.b) == 1):
        return None
    f, a = e.a.a, e.b[0]
    if _is_arg(a, argi):
        return {sum: SUM, min: MIN, max: MAX}.get(f) if f in (sum, min, max) else None
    if f is len and isinstance(a, E) and a.op == "call" and isinstance(a.a, E) and a.a.op == "obj" \
            and a.a.a in (list, tuple) and len(a.b) == 1 and _is_arg(a.b[0], argi):
        return COUNT
    return None


PRODUCT = "product"


def join_aggregate_kind(fn):
    """Shape of a join aggregate f(left_values_iter, right_values_iter) (dampr.py:780-820):
      ("folds", kl, kr)   lambda l, r: (K(l), K'(r)) with K, K' in sum / min / max / len(list(.))
      ("product",)        lambda l, r: itertools.product(l, r)   (one output per pair: use with many=True)
    None for anything else (the join then walks Python lists on the host)."""
    import itertools
    e = analyze(fn)
    if e is None or getattr(fn, "__code__", None) is None or fn.__code__.co_argcount != 2:
        return None
    if e.op == "tuple" and len(e.a) == 2:
        kl, kr = _iter_fold_kind(e.a[0], 0), _iter_fold_kind(e.a[1], 1)
        if kl is not None and kr is not None:
            return ("folds", kl, kr)
        return None
    if e.op == "call" and isinstance(e.a, E) and len(e.b) == 2 and _is_arg(e.b[0], 0) and _is_arg(e.b[1], 1):
        f = e.a
        callee = f.a if f.op == "obj" else (
            getattr(f.a.a, f.b, None) if (f.op == "attr" and isinstance(f.a, E) and f.a.op == "obj" and
                                          isinstance(f.a.a, types.ModuleType)) else None)
        if callee is itertools.product:
            return (PRODUCT,)
    return None


def depends_on(e, argi, fields=None):
    """Which fields of argument `argi` an expression reads: set of ints, or None when the argument is
    used whole (or in a way the analysis does not follow)."""
    out = set()

    def walk(x):
        if not isinstance(x, E):
            if isinstance(x, tuple):
                return all(walk(y) for y in x)
            return True
        if x.op == "sub" and _is_arg(x.a, argi):
            ok, i = _const(x.b)
            if ok and type(i) is int:
                out.add(i)
                return True
            return False
        if x.op == "arg":
            return x.a != argi
        if x.op in ("and", "or", "not"):   # boolean structure is not followed
            return False
        return all(walk(y) for y in (x.a, x.b, x.c) if y is not None)

    return out if walk(e) else None


# ---- numeric expressions evaluated natively (dampr_host_eval_f64) -------------------------------------------------
# the opcodes of csrc/common.cuh's EvalOp
_EV = dict(X=0, CI=1, CF=2, I2F=3, IADD=4, ISUB=5, IMUL=6, FADD=7, FSUB=8, FMUL=9, FDIV=10, IDIV=11, LOG=12,
           INEG=13, FNEG=14, LOAD=15, NF=16, IFLOOR=17, IMOD=18, IABS=19, FABS=20, F2I=21)
_EV_BIN = {"+": ("IADD", "FADD"), "-": ("ISUB", "FSUB"), "*": ("IMUL", "FMUL")}
EXPR_MAX_OPS, EXPR_MAX_LOADS, EXPR_MAX_DEPTH, EXPR_MAX_CONSTS = 32, 4, 8, 16   # include/dampr_b200.h


def _callee(f):
    """the Python object a call node calls: a global / builtin, or an attribute of one (math.log)"""
    if isinstance(f, E) and f.op == "obj":
        return f.a
    if isinstance(f, E) and f.op == "attr" and isinstance(f.a, E) and f.a.op == "obj" and isinstance(f.b, str):
        return getattr(f.a.a, f.b, None)
    return None


def numeric_program(e, field, scalar, argi=1, result="f", leaf=None):
    """Postfix program of dampr_host_eval_f64 for a float-valued expression over one int64 field `field` of argument
    `argi` (the column), the other argument as the broadcast value `scalar` (an int or a float) and int / float
    constants, built from + - * /, unary -, float() and math.log — typed as CPython types it (int operands of a float
    operation are converted first, int / int is true division). Returns (program, int constants, float constants),
    or None for anything outside that set (the caller then calls the function in Python).

    With `leaf` (a field scan's program, dampr_field_expr) the arguments are not read as a column or a scalar: leaf(x)
    gives (opcode word, "i" | "f") for a node that is a load or a field count, else None. Such a program may also use
    // and % of ints, abs() and int() of a float, not math.log; it is an int program under result "i", and it stays
    within the device's limits (EXPR_MAX_OPS operations, EXPR_MAX_DEPTH stack values, EXPR_MAX_CONSTS constants of
    each type)."""
    import math
    prog, ci, cf = [], [], []

    def num(v):
        if type(v) is int:
            if not -(1 << 63) <= v < (1 << 63):
                return None
            ci.append(v)
            prog.append(_EV["CI"] | (len(ci) - 1) << 8)
            return "i"
        if type(v) is float:
            cf.append(v)
            prog.append(_EV["CF"] | (len(cf) - 1) << 8)
            return "f"
        return None

    def to_float(t):
        if t == "i":
            prog.append(_EV["I2F"])
        return "f" if t else None

    def walk(x):
        if not isinstance(x, E):
            return None
        if leaf is not None:
            got = leaf(x)
            if got is not None:
                prog.append(got[0])
                return got[1]
            if x.op in ("sub", "arg"):
                return None
        if x.op == "sub" and _is_arg(x.a, argi):
            ok, i = _const(x.b)
            if ok and type(i) is int and i == field:
                prog.append(_EV["X"])
                return "i"
            return None
        if x.op == "arg":
            return num(scalar) if x.a != argi else None
        if x.op == "const":
            return num(x.a)
        if x.op == "neg":
            t = walk(x.a)
            if t:
                prog.append(_EV["INEG" if t == "i" else "FNEG"])
            return t
        if leaf is not None and x.op == "bin" and x.a in ("//", "%"):   # float // and % are not lowered
            if walk(x.b) != "i" or walk(x.c) != "i":
                return None
            prog.append(_EV["IFLOOR" if x.a == "//" else "IMOD"])
            return "i"
        if x.op == "bin" and x.a in ("+", "-", "*", "/"):
            tl = walk(x.b)
            if not tl:
                return None
            at = len(prog)            # where the left operand's conversion goes, if the right one is a float
            tr = walk(x.c)
            if not tr:
                return None
            if x.a == "/" and tl == tr == "i":
                prog.append(_EV["IDIV"])
                return "f"
            if tl == tr == "i":
                prog.append(_EV[_EV_BIN[x.a][0]])
                return "i"
            if tl == "i":
                prog.insert(at, _EV["I2F"])
            to_float(tr)
            prog.append(_EV["FDIV" if x.a == "/" else _EV_BIN[x.a][1]])
            return "f"
        if x.op == "call" and isinstance(x.b, tuple) and len(x.b) == 1:
            f = _callee(x.a)
            if f is float:
                return to_float(walk(x.b[0]))
            if leaf is not None and f is abs:
                t = walk(x.b[0])
                if t:
                    prog.append(_EV["IABS" if t == "i" else "FABS"])
                return t
            if leaf is not None and f is int:
                t = walk(x.b[0])
                if t == "f":
                    prog.append(_EV["F2I"])
                return "i" if t else None
            if leaf is None and f is math.log:
                t = to_float(walk(x.b[0]))
                if t:
                    prog.append(_EV["LOG"])
                return t
        return None

    t = walk(e)
    if t != result or len(prog) > (256 if leaf is None else EXPR_MAX_OPS):
        return None
    if leaf is not None:
        depth = top = 0
        for w in prog:
            op = w & 0xFF
            depth += 1 if op in (_EV["CI"], _EV["CF"], _EV["LOAD"], _EV["NF"]) else 0 if op in _EV_UNARY else -1
            top = max(top, depth)
        if top > EXPR_MAX_DEPTH or len(ci) > EXPR_MAX_CONSTS or len(cf) > EXPR_MAX_CONSTS:
            return None
    return prog, ci, cf


_EV_UNARY = {_EV[k] for k in ("I2F", "LOG", "INEG", "FNEG", "IABS", "FABS", "F2I")}


# ---- computed keys and values of a field fold (dampr_text_fields_expr) --------------------------------------------
EV_CI = _EV["CI"]
FIELD_EXPR = "expr"   # value_index of a text_fields_expr spec whose value is computed by its program
LOAD_INT, LOAD_F64, LOAD_LEN = 0, 1, 2   # load slot kinds (DAMPR_LOAD_*)


class _NoCompose(Exception):
    pass


def _compose(e, m, used):
    """e, a tree over argument 0, with the argument replaced by m, the tree of the map in front (x[i] of a tuple m is
    its element i, whose index goes into `used`; the whole m counts as element -1)"""
    if not isinstance(e, E):
        return e
    op = e.op
    if op == "arg":
        if e.a != 0:
            raise _NoCompose()
        used.add(-1)
        return m
    if op == "sub" and _is_arg(e.a) and isinstance(m, E) and m.op == "tuple":
        ok, i = _const(e.b)
        if not ok or type(i) is not int or not -len(m.a) <= i < len(m.a):
            raise _NoCompose()
        used.add(i % len(m.a))
        return m.a[i]
    if op in ("const", "obj"):
        return e
    if op == "call":
        return E(op, _compose(e.a, m, used), tuple(_compose(x, m, used) for x in e.b))
    if op == "tuple":
        return E(op, tuple(_compose(x, m, used) for x in e.a))
    if op == "attr":
        return E(op, _compose(e.a, m, used), e.b)
    if op in ("bin", "cmp"):
        return E(op, e.a, _compose(e.b, m, used), _compose(e.c, m, used))
    if op == "neg":
        return E(op, _compose(e.a, m, used))
    if op == "sub":
        return E(op, _compose(e.a, m, used), _compose(e.b, m, used))
    raise _NoCompose()


def split_of(fn):
    """the separator of a one-argument `lambda l: l.split(S)` / `l.split()` (SEP_WS), else None"""
    if not (isinstance(fn, types.FunctionType) and fn.__code__.co_argcount == 1):
        return None
    return _split_sep(analyze(fn), True)


def text_fields_expr(key_fn, value_fn, map_fn=None):
    """Device field-scan spec of a keyed(key_fn, value_fn) over text lines, behind an optional map(map_fn), for the
    shapes text_fields_spec refuses: a key that is an int expression (a constant one included, e.g. mean()'s default
    `lambda x: 1`) and / or a value that is an int or float expression, over the leaves int(R[j]), float(R[j]),
    len(R), len(R[j]) and int / float constants, with + - * / // % (// and % of ints), unary -, abs(), float() and
    int() — typed as CPython types them. R is l.split(S) or l.split() of the line.

    map_fn may be l.split(S) / l.split(), or return an expression over the line or a tuple of such; the key and value
    functions are composed with its tree ((...)[i] of its tuple resolves to element i). Every element of such a map
    must be used by the key or the value: the device evaluates only what they read, and an unused element could
    raise in Python.

    Returns (sep, key_index, key_kind, value_index, value_kind, mean, expr) with sep the split's separator (SEP_WS
    for split(); None when no field is read), key_kind FIELD_STR / FIELD_INT (a projection, key_index its field) or
    FIELD_INT with key_index None (a key program), value_index the field of an int() / float() value, None for the
    constant 1 or FIELD_EXPR for a value program, value_kind FIELD_INT / FIELD_FLOAT, mean as text_fields_spec, and
    expr = (key program or None, value program or None, int constants, float constants, loads) with a program
    ("i" | "f", [opcode words]) and loads [(field index, LOAD_*)]. expr is None when the composition left bare
    projections only (the plain scan's spec). None for any other shape."""
    fns = [f for f in (key_fn, value_fn, map_fn) if f is not None]
    if not all(isinstance(f, types.FunctionType) and f.__code__.co_argcount == 1 for f in fns):
        return None
    ke, ve = analyze(key_fn), analyze(value_fn)
    if ke is None or ve is None:
        return None
    mean = ve.op == "tuple" and len(ve.a) == 2
    if mean:
        inner = _inline_call_of_arg(ve.a[0])
        if inner is None or not _is_one(ve.a[1]):
            return None
        ve = inner
    if map_fn is not None:
        me = analyze(map_fn)
        if me is None:
            return None
        used = set()
        try:
            ke, ve = _compose(ke, me, used), _compose(ve, me, used)
        except _NoCompose:
            return None
        if _split_sep(me, True) is None:
            need = set(range(len(me.a))) if me.op == "tuple" else {-1}
            if not need <= used and not (me.op == "tuple" and -1 in used):
                return None

    seps, loads = set(), []

    def record(x):
        sep = _split_sep(x, True)
        if sep is not None:
            seps.add(sep)
        return sep

    def slot(i, kind):
        if (i, kind) not in loads:
            loads.append((i, kind))
        return _EV["LOAD"] | loads.index((i, kind)) << 8

    def leaf(x):
        if not (isinstance(x, E) and x.op == "call" and isinstance(x.b, tuple) and len(x.b) == 1):
            return None
        f = _callee(x.a)
        if f is len:
            if record(x.b[0]) is not None:
                return _EV["NF"], "i"
            p = _field_proj(x.b[0], record)
            return (slot(p[1], LOAD_LEN), "i") if p is not None and p[0] == FIELD_STR else None
        if f in (int, float):
            p = _value_proj(x, record)
            if p is not None:
                return (slot(p[1], LOAD_INT), "i") if p[0] == FIELD_INT else (slot(p[1], LOAD_F64), "f")
        return None

    k = _field_proj(ke, record)
    kprog = None
    if k is None:
        kprog = numeric_program(ke, None, None, result="i", leaf=leaf)
        if kprog is None:
            return None
    vprog, v, vtype = None, None, "i"
    if not (_is_one(ve) and not mean):
        v = _value_proj(ve, record)
        if v is None:
            vprog = numeric_program(ve, None, None, result="i", leaf=leaf)
            if vprog is None:
                vprog, vtype = numeric_program(ve, None, None, result="f", leaf=leaf), "f"
            if vprog is None:
                return None
    if len(seps) > 1 or len(loads) > EXPR_MAX_LOADS:
        return None
    sep = seps.pop() if seps else None
    if kprog is None and vprog is None:   # bare projections after the composition: the plain scan's spec
        return (sep, k[1], k[0], None if v is None else v[1], FIELD_INT if v is None else v[0], mean, None)
    progs, ci, cf = [], [], []
    for p in (kprog, vprog):   # one pool of constants: the value program's indices move past the key program's
        if p is None:
            progs.append(None)
            continue
        words, pci, pcf = p
        out = []
        for w in words:
            op = w & 0xFF
            out.append(op | (w >> 8) + len(ci) << 8 if op == _EV["CI"] else
                       op | (w >> 8) + len(cf) << 8 if op == _EV["CF"] else w)
        progs.append(("i" if p is kprog else vtype, out))
        ci, cf = ci + pci, cf + pcf
    if len(ci) > EXPR_MAX_CONSTS or len(cf) > EXPR_MAX_CONSTS:
        return None
    vkind = (FIELD_INT if v is None else v[0]) if vprog is None else \
        (FIELD_FLOAT if progs[1][0] == "f" else FIELD_INT)
    return (sep, None if kprog else k[1], FIELD_INT if kprog else k[0],
            FIELD_EXPR if vprog else None if v is None else v[1], vkind, mean, (progs[0], progs[1], ci, cf, loads))

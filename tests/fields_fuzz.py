"""Seeded fuzz corpora, stage generators and two per-line oracles of the field-scan kernels (csrc/fields.cu), shared by
test_fields_fuzz_standins.py (the stand-ins against CPython) and test_gpu_fields_fuzz.py (the kernels against both).

Every field scan decides per line: TAKE (fold Python's key and value), DROP (a filter is false) or HOST (hand the line
back, because Python would raise or the device cannot be sure). An outcome here is one of
  ("TAKE", key code, value bits)   the device's real key code (str keys: the field-key code of
                                   test_code_collisions.key_code, int keys v ^ 2^63, tuples fields_tuple_standin.tuple_code)
                                   and the value's int64 or float64 bits
  ("DROP",)
  ("HOST", detail)                 for CPython the name of the exception it raised
The stand-in outcome calls the stand-ins' own per-line rules (plain_line, line_verdict, tuple_line, expr_line,
json_line); the CPython outcome runs the stage's real lambdas."""
import collections
import json
import math
import random

from fields_expr_standin import expr_line
from fields_json_standin import json_line
from fields_standin import M64, f64_bits, plain_line
from fields_tuple_standin import tuple_code, tuple_line
from fields_where_standin import line_verdict
from fields_ws_standin import WsLine, ws_field_offsets
from test_code_collisions import key_code
from test_fparse_host import BOUNDARIES, REJECTED, SPELLINGS
from test_text_fields_expr_lowering import random_lambda

FAMILIES = ("sep", "ws", "json")
TAKE, DROP, HOST = "TAKE", "DROP", "HOST"
# every separator byte the lowering takes: ASCII but NUL, '\n' and '\r'
SEPS = [b for b in range(1, 128) if b not in (10, 13)]

# ---- pools ------------------------------------------------------------------------------------------------------
INT_EDGES = ["", "0", "-0", "+0", "007", "+7", "-", "+", "12345678901234567", "123456789012345678",
             "1234567890123456789", "-123456789012345678", "-1234567890123456789", "999999999999999999",
             "9223372036854775807", "-9223372036854775807", "9223372036854775808", "-9223372036854775808",
             "1_000", " 7", "7 ", "\t7", "0x10", "٣", "7\r"]
FLOAT_EDGES = [s.replace("\n", "") for s in BOUNDARIES + SPELLINGS + REJECTED] + ["nan", "inf", "-0.0", "1e309"]
STR_ALPHA = "abcxyzAB_-.07"
STR_ODD = ["\x01", "\x7f", "é"]
# the kinds of a separated row's fields by position: int, int, float, str, ... (random_lambda reads int(r[0]),
# int(r[1]), float(r[2]), len(r), len(r[3]))
SCHEMA = "iifsisfsiifs"
WS_BYTES = "\t\x0b\x0c\x1c\x1d\x1e\x1f "


def int_spelling(rng, edges=0.12):
    if rng.random() < edges:
        return rng.choice(INT_EDGES)
    return str(rng.choice([rng.randrange(-50, 50), rng.randrange(-10 ** 6, 10 ** 6), rng.randrange(0, 9)]))


def float_spelling(rng, edges=0.12):
    if rng.random() < edges:
        return rng.choice(FLOAT_EDGES)
    return rng.choice(["%.3f", "%g", "%.1e"]) % (rng.randrange(-4000, 4000) / 8.0)


def str_key(rng, sep=""):
    """lengths 0 .. 12 across the 9-byte packed / hashed boundary, some holding 0x01, 0x7F, the separator or é"""
    n = rng.choice([0, 1, 2, 3, 8, 9, 9, 10, 12] if rng.random() < 0.3 else [1, 2, 3])
    s = "".join(rng.choice(STR_ALPHA) for _ in range(n))
    if s and rng.random() < 0.05:
        i = rng.randrange(len(s))
        s = s[:i] + rng.choice(STR_ODD + ([sep] if sep else [])) + s[i + 1:]
    return s


def field(rng, kind, sep=""):
    if rng.random() < 0.06:
        kind = rng.choice("ifs")
    return int_spelling(rng) if kind == "i" else float_spelling(rng) if kind == "f" else str_key(rng, sep)


def mutate(rng, s, alphabet):
    """1-3 random character edits: insert, delete or replace"""
    for _ in range(rng.randint(1, 3)):
        i = rng.randrange(len(s) + 1)
        op = rng.randrange(3)
        c = rng.choice(alphabet)
        s = s[:i] + c + s[i:] if op == 0 else s[:i] + s[i + 1:] if op == 1 else s[:i] + c + s[i + 1:]
    return s


def _long(rng, s, join):
    """s padded to 4094 .. 4098 bytes, around the 4 KB line window"""
    want = rng.randint(4094, 4098)
    pad = want - len(s.encode("utf-8")) - len(join)
    return s + join + "z" * pad if pad > 0 else s


# ---- corpora ----------------------------------------------------------------------------------------------------
def sep_corpus(seed, n, sep, cr=False):
    """n lines of 0 .. 12 fields joined by the separator byte `sep` (an int): typed by SCHEMA, with blank lines,
    leading / trailing / doubled separators, long lines and mutations; '\\r' appears inside fields when `cr`"""
    rng = random.Random(seed)
    S = chr(sep)
    alpha = [S, " ", "\t", "\x0b", "\x0c", "\x1c"] + list("0123456789+-._eE") + ["\x00", "\x7f", "\r", "é"]
    out = []
    for _ in range(n):
        r = rng.random()
        if r < 0.02:
            out.append("")
            continue
        nf = rng.choice([0, 1, 2, 3, 4, 5, 6, 8, 11]) if rng.random() < 0.2 else 12
        line = S.join(field(rng, SCHEMA[i], S) for i in range(nf))
        r = rng.random()
        if r < 0.03:
            line = S + line
        elif r < 0.06:
            line = line + S
        elif r < 0.09 and S in line:
            line = line.replace(S, S + S, 1)
        if rng.random() < 0.002:
            line = _long(rng, line, S)
        if rng.random() < 0.2:
            line = mutate(rng, line, alpha)
        if cr and rng.random() < 0.05:
            i = rng.randrange(len(line) + 1)
            line = line[:i] + "\r" + line[i:]
        out.append(line.replace("\n", ""))
    return finish(rng, out)


def ws_corpus(seed, n, cr=False):
    """n lines of 0 .. 12 fields split by runs of 0x09, 0x0B, 0x0C, 0x1C-0x1F and 0x20 (and 0x0D when `cr`), with
    leading and trailing whitespace and the non-ASCII whitespace \\x85 and \\xa0"""
    rng = random.Random(seed)
    ws = WS_BYTES + ("\r" if cr else "")
    alpha = list(ws) + list("0123456789+-._eE") + ["\x00", "\x7f", "é", "\x85", "\xa0"] + \
        ([] if cr else ["\r"])

    def run():
        if rng.random() < 0.01:
            return rng.choice(["\x85", "\xa0"])
        return "".join(rng.choice(ws if rng.random() < 0.3 else " ") for _ in range(rng.choice([1, 1, 1, 2, 3])))
    out = []
    for _ in range(n):
        if rng.random() < 0.02:
            out.append(rng.choice(["", " ", "\t\x0b"]))
            continue
        nf = rng.choice([0, 1, 2, 3, 4, 6, 11]) if rng.random() < 0.2 else 12
        fs = []
        for i in range(nf):
            f = field(rng, SCHEMA[i])
            fs.append("".join(c for c in f if c not in ws and c not in "\x85\xa0") or "x")
        line = "".join(f + run() for f in fs)[:-1] if fs else ""
        if rng.random() < 0.08:
            line = run() + line
        if rng.random() < 0.08:
            line = line + run()
        if rng.random() < 0.002:
            line = _long(rng, line, " ")
        if rng.random() < 0.2:
            line = mutate(rng, line, alpha)
        out.append(line.replace("\n", ""))
    return finish(rng, out)


NAMES = ["k", "v", "f", "s", "n"]                  # the members stages read
TYPED = {"k": "s", "v": "i", "f": "f", "s": "s", "n": "i"}   # the kind each mostly holds at the top level
DECOYS = ["user", "K", "k2", "vv", "x", "k "]      # other names, some one byte off a wanted one
JSON_NUMBERS = ["-0", "01", "1.", ".5", "1e", "-0.0e-0", "1234567890123456789", "12345678901234567890",
                "-1234567890123456789", "123456789012345678", "1e400", "-", "2E+3", "0.1", "-1.5e-3", "00"]


def json_value(rng, depth=0):
    r = rng.random()
    if r < 0.35:
        return int_spelling(rng, 0).strip() if rng.random() < 0.95 else rng.choice(JSON_NUMBERS)
    if r < 0.55:
        return float_spelling(rng, 0.03).strip() if rng.random() < 0.95 else rng.choice(JSON_NUMBERS)
    if r < 0.75:
        s = str_key(rng)
        if rng.random() < 0.1:
            return '"%s\\n%s"' % (s, rng.choice(["\\\"", "\\u0041", "\\/", "\\\\"]))
        return json.dumps(s, ensure_ascii=rng.random() < 0.9)
    if r < 0.85 and depth < 2:
        return json_object(rng, depth + 1)
    if r < 0.9 and depth < 2:
        return "[%s]" % ", ".join(json_value(rng, depth + 1) for _ in range(rng.randrange(3)))
    return rng.choice(["true", "false", "null", "[]", "{}", "0", "1.5"] * 4 + ["NaN", "Infinity", "-Infinity"])


def _nest(d):
    """an array value nesting a line d deep (its object counts one)"""
    return "[" * (d - 1) + "1" + "]" * (d - 1)


def json_object(rng, depth=0):
    ws = lambda: rng.choice(["", "", "", " ", "\t", "  ", "\r", " \t"])   # noqa: E731
    names = NAMES * 2 + DECOYS
    members = []
    want = [n for n in NAMES if rng.random() < 0.9] if depth == 0 else []
    for _ in range(rng.randrange(0, 7) if depth else rng.randrange(len(want), len(want) + 4)):
        name = want.pop(rng.randrange(len(want))) if want else rng.choice(names)
        qn = json.dumps(name)
        if rng.random() < 0.03:
            qn = '"\\u%04x%s"' % (ord(name[0]), name[1:])   # an escaped name
        val = json_value(rng, depth)
        if depth == 0 and name in TYPED and rng.random() < 0.8:
            kind = TYPED[name] if name != "k" or rng.random() < 0.7 else "i"
            val = json.dumps(str_key(rng)) if kind == "s" else int_spelling(rng, 0) if kind == "i" else \
                float_spelling(rng, 0.03).strip()
        if depth == 0 and rng.random() < 0.01:
            val = _nest(rng.choice([63, 64, 65]))
        members.append(ws() + qn + ws() + ":" + ws() + val + ws())
    if depth == 0 and rng.random() < 0.05 and members:
        members.append(members[0])   # a duplicate name
    return "{" + ",".join(members) + "}"


def json_corpus(seed, n, cr=False):
    """n JSON-lines records over the wanted and decoy names: values of every JSON type, numbers at the grammar's
    edges, duplicate names, escapes, nesting 63 .. 65 deep and ' \\t\\r' between tokens, then mutations"""
    rng = random.Random(seed)
    alpha = list('{}[]":,-+.eE0123456789 \t\r\\/tfnul') + ["\x00", "\x7f", "é"]
    out = []
    for _ in range(n):
        if rng.random() < 0.01:
            out.append(rng.choice(["", " ", "[]", "1", '"a"']))
            continue
        line = json_object(rng)
        if rng.random() < 0.002:
            line = line[:-1] + ', "pad": "' + "z" * (rng.randint(4094, 4098) - len(line) - 11) + '"}'
        if rng.random() < 0.15:
            line = mutate(rng, line, alpha)
        if not cr:
            line = line.replace("\r", " ") if rng.random() < 0.9 else line
        out.append(line.replace("\n", ""))
    return finish(rng, out)


def finish(rng, lines):
    """the corpus's bytes: its lines joined by '\\n', the last line without one half of the time"""
    data = "\n".join(lines) + ("\n" if rng.random() < 0.5 else "")
    return data.encode("utf-8")


def corpus(family, seed, n, cr=False, sep=ord(",")):
    if family == "sep":
        return sep_corpus(seed, n, sep, cr)
    return ws_corpus(seed, n, cr) if family == "ws" else json_corpus(seed, n, cr)


def tame_lines(family, seed, n):
    """n lines of the family whose every field is its SCHEMA kind, without edge spellings or mutations (whole
    pipelines over them run to the end more often than not)"""
    rng = random.Random(seed)
    if family == "json":
        out = []
        for _ in range(n):
            m = {"k": rng.choice(["a", "b", "cc", "abcdefghijk", "é", "a\nb"]), "v": rng.randrange(-99, 99),
                 "f": rng.randrange(-99, 99) / 8.0, "s": rng.choice(["a", "b", "abcdefghijk"]), "n": rng.randrange(9),
                 "user": {"k": 1}}
            out.append(json.dumps(dict(rng.sample(sorted(m.items()), len(m)))))
        return out
    S = "," if family == "sep" else " \t"
    return [S.join(str(rng.randrange(-99, 99)) if k == "i" else "%g" % (rng.randrange(1, 99) / 8.0) if k == "f" else
                   rng.choice(["a", "b", "cc", "abcdefghijk", "é"]) for k in SCHEMA) for _ in range(n)]


def lines_of(data):
    """[(offset, line bytes)] as the scans split data: at every '\\n', the last line ending at the data's end"""
    out, pos = [], 0
    while pos < len(data):
        end = data.find(b"\n", pos)
        end = len(data) if end < 0 else end
        out.append((pos, data[pos:end]))
        pos = end + 1
    return out


# ---- stages -----------------------------------------------------------------------------------------------------
OPS = ["count", "sum", "min", "max", "mean"]
CMPS = ["==", "!=", "<", "<=", ">", ">="]
# a filter's comparison: "!=" and "not in" weighted up, so that chains of filters still pass a share of the lines
CMPS_W = ["==", "!=", "!=", "!=", "<", "<=", ">", ">="]
INS_W = ["in", "not in", "not in"]


def _idx(rng, kind, nmax=12):
    """a field index whose SCHEMA kind is `kind` most of the time, sometimes negative or out of range"""
    i = rng.choice([j for j in range(nmax) if SCHEMA[j] == kind]) if rng.random() < 0.9 else rng.randrange(13)
    return i - nmax if rng.random() < 0.15 else i


def _consts(rng, kind, n):
    pool = {"s": lambda: str_key(rng), "i": lambda: int(int_spelling(rng)) if rng.random() < 0.5 else
            rng.randrange(-50, 50)}[kind]
    out = []
    for _ in range(n):
        try:
            out.append(pool())
        except ValueError:
            out.append(rng.randrange(9) if kind == "i" else "a")
    return out


def text_filter(rng):
    k = rng.random()
    cmp = rng.choice(CMPS_W)
    if k < 0.25:
        c = repr(str_key(rng))
        i = _idx(rng, "s")
        return rng.choice(["r[%d] %s %s" % (i, cmp, c), "%s %s r[%d]" % (c, cmp, i)])
    if k < 0.45:
        return "int(r[%d]) %s %d" % (_idx(rng, "i"), cmp, rng.choice([0, 7, -3, 500, 10 ** 17, rng.randrange(-60, 60)]))
    if k < 0.6:
        return "float(r[%d]) %s %r" % (_idx(rng, "f"), cmp, rng.choice([0.0, -0.0, 1.5, -100.25, 1e300, 3]))
    if k < 0.8:
        kind = rng.choice("si")
        n = rng.choice([1, 2, 3, 8, 30])
        cs = _consts(rng, kind, n)
        x = "r[%d]" % _idx(rng, "s") if kind == "s" else "int(r[%d])" % _idx(rng, "i")
        return "%s %s %s" % (x, rng.choice(INS_W), rng.choice(["(%s,)", "{%s}", "[%s]"]) %
                             ", ".join(map(repr, cs)))
    return "len(r) %s %d" % (cmp, rng.choice([0, 1, 4, 6, 8, 12]))


def json_filter(rng):
    k = rng.random()
    cmp = rng.choice(CMPS_W)
    # mostly a member of the kind the comparison reads (TYPED), else any wanted or decoy name
    pool = {0: "ks", 1: "vn", 2: "vn", 3: "fv", 4: "ksvn"}[0 if k < 0.2 else 1 if k < 0.35 else 2 if k < 0.5 else
                                                           3 if k < 0.62 else 4]
    m = repr(rng.choice(pool if rng.random() < 0.8 else NAMES + ["user"]))
    if k < 0.2:
        return "r[%s] %s %r" % (m, cmp, str_key(rng))
    if k < 0.35:
        return "r[%s] %s %d" % (m, cmp, rng.randrange(-50, 50))
    if k < 0.5:
        return "int(r[%s]) %s %d" % (m, cmp, rng.randrange(-60, 60))
    if k < 0.62:
        return "float(r[%s]) %s %r" % (m, cmp, rng.choice([0.0, 1.5, -100.25, 3]))
    if k < 0.8:
        kind = rng.choice("si")
        cs = _consts(rng, kind, rng.choice([1, 2, 5, 20]))
        x = "r[%s]" % m if kind == "s" or rng.random() < 0.5 else "int(r[%s])" % m
        return "%s %s %s" % (x, rng.choice(INS_W), "(%s,)" % ", ".join(map(repr, cs)))
    return "%s %s r" % (m, rng.choice(INS_W))


def text_key(rng):
    k = rng.random()
    if k < 0.3:
        return "r[%d]" % _idx(rng, "s")
    if k < 0.45:
        return "int(r[%d])" % _idx(rng, "i")
    if k < 0.7:
        comps = []
        for _ in range(rng.randint(1, 4)):
            comps.append("r[%d]" % _idx(rng, "s") if rng.random() < 0.5 else "int(r[%d])" % _idx(rng, "i"))
        if rng.random() < 0.2:
            comps.append(comps[0])   # a repeated index
        return "(%s,)" % ", ".join(comps[:4])
    if k < 0.9:
        return random_lambda(rng)
    return "1"


def text_value(rng):
    k = rng.random()
    return "1" if k < 0.15 else "int(r[%d])" % _idx(rng, "i") if k < 0.4 else \
        "float(r[%d])" % _idx(rng, "f") if k < 0.65 else random_lambda(rng)


def fold_src(op, key, value):
    if op == "count":
        return ".count(lambda r: %s)" % key
    if op == "mean":
        return ".mean(lambda r: %s, lambda r: %s)" % (key, value)
    red = {"sum": ".sum()", "min": ".reduce(min)", "max": ".reduce(max)"}[op]
    return ".a_group_by(lambda r: %s, lambda r: %s)%s" % (key, value, red)


class Stage(object):
    """a generated stage: its pipeline source over P, its real lambdas, and the planner's match of it"""

    def __init__(self, family, map_src, filters, key, value, op):
        self.family, self.filters_src, self.key_src, self.value_src, self.op_name = family, filters, key, value, op
        self.map_src = map_src
        head = "Dampr.json(P)" if family == "json" else "Dampr.text(P).map(%s)" % map_src
        self.src = head + "".join(".filter(lambda r: %s)" % f for f in filters) + fold_src(op, key, value)
        g = {"json": json}
        self.map = json.loads if family == "json" else eval(map_src, g)
        self.filters = [eval("lambda r: " + f, g) for f in filters]
        self.key = eval("lambda r: " + key, g)
        self.value = eval("lambda r: " + (value if op != "count" else "1"), g)
        self.match = None

    def __repr__(self):
        return self.src


def gen_stage(rng, family, sep=None):
    nf = rng.choice([0, 0, 0, 1, 1, 2, 3, 8]) if rng.random() < 0.95 else rng.randint(4, 8)
    op = rng.choice(OPS)
    if family == "json":
        key = rng.choice(['r["k"]', 'int(r["k"])', 'r["s"]', 'r["v"]'])
        value = rng.choice(['r["v"]', 'int(r["v"])', 'float(r["f"])', 'float(r["v"])', '1'])
        return Stage(family, None, [json_filter(rng) for _ in range(nf)], key, value, op)
    map_src = "lambda l: l.split()" if family == "ws" else "lambda l: l.split(%r)" % chr(sep)
    return Stage(family, map_src, [text_filter(rng) for _ in range(nf)], text_key(rng), text_value(rng), op)


def match(stage, path):
    """the planner's match of stage over the (existing) file path, or None; stored on the stage"""
    from dampr_b200 import Dampr, plan
    from dampr_b200.graph import GMap
    pm = eval(stage.src, {"Dampr": Dampr, "P": path, "json": json})
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    ins = [pm.pmer.graph.inputs[st.inputs[0]]]
    stage.match = (plan._match_json_fields if stage.family == "json" else plan._match_text_fields)(st, ins)
    return stage.match


def gen_stages(seed, family, n, path, sep=None):
    """(lowered stages, refused count) of n generated stages"""
    rng = random.Random(seed)
    out, refused = [], 0
    for _ in range(n):
        st = gen_stage(rng, family, sep)
        if match(st, path) is None:
            refused += 1
        else:
            out.append(st)
    return out, refused


def builds_of(family):
    """the build names (Build.name) of a family"""
    kinds = ["json", "json+where"] if family == "json" else \
        ["plain", "where", "tuple", "tuple+where", "expr", "expr+where"]
    return {"%s/%s/%s" % (family, k, v) for k in kinds for v in ("count", "i64", "f64")}


def cover(family, seed, path, per_build, tries=5000):
    """(generated stages, refused count, [(Build, cr_is_data, separator byte)]): generated stages until every build of
    the family has run per_build times with cr_is_data off and per_build times with it on. A generator that stops
    reaching a build fails here."""
    rng = random.Random(seed)
    need = collections.Counter({(name, cr): per_build for name in builds_of(family) for cr in (False, True)})
    out, refused = [], 0
    for j in range(tries):
        if not +need:
            return j, refused, out
        sep = ord(",") if rng.random() < 0.5 else rng.choice(SEPS)
        sts, nref = gen_stages(seed * 100003 + j, family, 1, path, sep)
        refused += nref
        if not sts:
            continue
        b = Build(sts[0])
        cr = next((c for c in (False, True) if need[b.name(), c] > 0), None)
        if cr is None:
            continue
        if len(b.preds) > 2 and need[b.name(), cr] == per_build and rng.random() < 0.9:
            continue   # mostly one or two filters first: a long chain drops or hands back nearly every line
        need[b.name(), cr] -= 1
        out.append((b, cr, sep))
    raise AssertionError("%d generated %s stages reach no %s" % (tries, family, sorted(k for k in +need)))


# ---- the builds of a matched stage ------------------------------------------------------------------------------
class Build(object):
    """the kernel call of a matched stage: kind "plain" / "where" / "tuple" / "expr" / "json", the spec (sep, key,
    key kind, value, op) with the record-mode op, the predicates and the tuple components / programs / members"""

    def __init__(self, stage):
        from dampr_b200 import device as dev, plan
        m = stage.match
        self.stage = stage
        if stage.family == "json":
            _src, spec, op, mean, preds, members, _bare = m
            self.kind, self.extra = "json", members
        else:
            _src, spec, op, mean, preds, expr = m
            if expr is not None:
                self.kind, self.extra = "expr", expr
            elif spec[2] == plan.KEY_TUPLE:
                self.kind, self.extra = "tuple", spec[1]
                spec = (spec[0], 0, dev.FIELD_KEY_STR) + tuple(spec[3:])
            else:
                self.kind, self.extra = ("where" if preds else "plain"), None
        self.table_op = op
        self.flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
        self.spec = tuple(spec) + (dev.OP_SUM_F64 if self.flt else dev.OP_SUM_I64,)
        self.preds = tuple(preds)
        self.int_key = self.kind == "expr" and self.extra[0] is not None or \
            self.kind != "tuple" and spec[2] == dev.FIELD_KEY_INT

    def name(self):
        """family/call/value: the call with "+where" when a tuple, expression or JSON call has filters (its own
        kernel), the value "count" for the constant 1 (table mode only), else the value type"""
        from dampr_b200 import device as dev
        kind = self.kind + ("+where" if self.preds and self.kind != "where" else "")
        value = "count" if self.spec[3] == dev.FIELD_VAL_ONE else "f64" if self.flt else "i64"
        return "%s/%s/%s" % (self.stage.family, kind, value)

    def records(self, tab, tb, lo, hi, kv, cr):
        """the record-mode call of this build"""
        s, x, p = self.spec, self.extra, self.preds
        if self.kind == "json":
            tab.json_fields_records(tb, lo, hi, s, x, kv, cr, p)
        elif self.kind == "expr":
            tab.fields_expr_records(tb, lo, hi, s, x, kv, cr, p)
        elif self.kind == "tuple":
            tab.fields_tuple_records(tb, lo, hi, s, x, kv, cr, p)
        else:
            tab.fields_records(tb, lo, hi, s, kv, cr, p)

    def table(self, tab, tb, lo, hi, op, cr):
        """the table-mode call of this build under op"""
        s, x, p = self.spec[:4] + (op,), self.extra, self.preds
        if self.kind == "json":
            tab.json_fields(tb, lo, hi, s, x, cr, p)
        elif self.kind == "expr":
            tab.fields_expr(tb, lo, hi, s, x, cr, p)
        elif self.kind == "tuple":
            tab.fields_tuple(tb, lo, hi, s, x, cr, p)
        else:
            tab.fields(tb, lo, hi, s, cr, p)


# ---- the oracles ------------------------------------------------------------------------------------------------
def str_code(k):
    return key_code(k, "raw", field_key=True)


def value_bits(v, flt):
    return f64_bits(v) if flt else v & M64


class Out(tuple):
    """an outcome; a stand-in TAKE also carries the key (.key), the value (.value) and the key's offset in the line
    (.key_off, hashed str keys) for the stats and the table checks"""
    key = value = key_off = None
    flags = 0


def _out(*a, **kw):
    o = Out(a)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def standin_outcome(b, line, cr):
    """the stand-ins' outcome of line (bytes) under build b"""
    from dampr_b200 import device as dev
    sp = b.spec
    if b.kind == "json":
        got, flags = json_line(line, sp, b.extra, cr, b.preds)
        if got is False or got is None:
            return _out(DROP, flags=flags) if got is False else _out(HOST, "standin", flags=flags)
        synth, koff = got
        vf = dev.FIELD_VAL_ONE if sp[3] == dev.FIELD_VAL_ONE else 1
        k, v = plain_line(synth, synth.split(b"\x01"), 0, sp[2], vf, b.flt, cr)
        code = (k ^ (1 << 63)) & M64 if b.int_key else str_code(k)
        return _out(TAKE, code, value_bits(v, b.flt), key=k, value=v, key_off=koff, flags=flags)
    ws = sp[0] == dev.FIELD_SEP_WS
    f = WsLine(line).split() if ws else line.split(bytes([sp[0]]))
    if b.kind == "tuple":
        got = tuple_line(line, f, sp, b.extra, cr, b.preds)
        if got is False or got is None:
            return _out(DROP) if got is False else _out(HOST, "standin")
        parts, v = got
        return _out(TAKE, tuple_code(parts), value_bits(v, b.flt), key=tuple(parts), value=v, key_off=0)
    verdict = line_verdict(line, f, b.preds, cr)
    if verdict is not True:
        return _out(DROP) if verdict is False else _out(HOST, "standin")
    kv = expr_line(line, f, b.extra, sp) if b.kind == "expr" else \
        plain_line(line, f, sp[1], sp[2], sp[3], b.flt, cr)
    if kv is None:
        return _out(HOST, "standin")
    k, v = kv
    koff = None
    if not b.int_key and not 1 <= len(k) <= 9:
        kf = sp[1] % len(f)
        koff = ws_field_offsets(line)[kf] if ws else sum(len(x) + 1 for x in f[:kf])
    code = (k ^ (1 << 63)) & M64 if b.int_key else str_code(k)
    return _out(TAKE, code, value_bits(v, b.flt), key=k, value=v, key_off=koff)


def python_outcome(stage, line):
    """CPython's outcome of line (bytes) under the stage's lambdas: ("TAKE", key, value) with Python's own key and
    value, ("DROP",) at the first false filter, ("HOST", exception type name)"""
    try:
        r = stage.map(line.decode("utf-8"))
        for p in stage.filters:
            if not p(r):
                return (DROP,)
        return (TAKE, stage.key(r), stage.value(r))
    except Exception as e:   # noqa: BLE001  the exception is the outcome
        return (HOST, type(e).__name__)


def python_code(k):
    """the device's code of Python's key k, or None where no device code stands for it"""
    if type(k) is str:
        return str_code(k.encode("utf-8"))
    if type(k) is int:
        return (k ^ (1 << 63)) & M64 if -(1 << 63) <= k < (1 << 63) else None
    if type(k) is tuple and all(type(p) in (str, int) for p in k):
        if any(type(p) is int and not -(1 << 63) <= p < (1 << 63) for p in k):
            return None
        return tuple_code([p.encode("utf-8") if type(p) is str else p for p in k])
    return None


def same_bits(py_v, bits, flt):
    if flt:
        return type(py_v) is float and f64_bits(py_v) == bits
    return type(py_v) is int and -(1 << 63) <= py_v < (1 << 63) and py_v & M64 == bits


def sound(b, line, got, py, cr):
    """None if outcome `got` (a stand-in's or the device's) is sound against CPython's `py` on line, else why not"""
    if not cr and b"\r" in line and got[0] != HOST:
        return "a text-mode line holding '\\r' is not the host's"
    if py[0] == HOST and got[0] != HOST:
        return "CPython raises %s" % py[1]
    if got[0] == DROP and py[0] != DROP:
        return "dropped, CPython %s" % (py,)
    if got[0] == TAKE:
        if py[0] != TAKE:
            return "taken, CPython %s" % (py,)
        code = python_code(py[1])
        if b.kind == "tuple" and type(py[1]) is not tuple or b.kind != "tuple" and type(py[1]) is tuple:
            code = None
        if code != got[1]:
            return "key %r: code %x, the device's %x" % (py[1], code or 0, got[1])
        if not same_bits(py[2], got[2], b.flt):
            return "value %r, the device's bits %x" % (py[2], got[2])
    return None


# ---- findings ---------------------------------------------------------------------------------------------------
# the minimal line and stage of every disagreement the fuzzing found, checked first by both test files:
# (family, filters, key, value, op, separator byte or None for split(), line, cr_is_data)
FOUND = []


# ---- the fold of the expected outcomes -------------------------------------------------------------------------
def expected_stats(b, outs):
    """fields_stats() of a record-mode scan whose lines have the stand-in outcomes outs"""
    from dampr_b200 import device as dev
    st = {"records": len(outs), "lines": 0, "folded": 0, "fallback": 0, "hashed": 0, "max_abs": 0, "flags": 0}
    for o in outs:
        st["flags"] |= o.flags
        if o[0] == HOST:
            st["fallback"] += 1
        elif o[0] == TAKE:
            st["lines"] += 1
            st["folded"] += 1
            v = o.value
            if b.flt:
                if v == 0 and math.copysign(1.0, v) < 0:
                    st["flags"] |= dev.TF_NEGZERO
                if v != v and b.kind == "expr":
                    st["flags"] |= dev.TF_NAN
            else:
                st["max_abs"] = max(st["max_abs"], abs(v))
            if b.kind not in ("tuple",) and not b.int_key and not 1 <= len(o.key) <= 9:
                st["hashed"] += 1
    return st


def table_fold(outs, op):
    """{code: the device's accumulator value (int or float bits)} of the TAKE lines under table op"""
    from dampr_b200 import device as dev
    acc = {}
    for o in outs:
        if o[0] != TAKE:
            continue
        c, v = o[1], o.value
        if op == dev.OP_SUM_I64:
            acc[c] = ((acc.get(c, 0) + v + (1 << 63)) & M64) - (1 << 63)
        elif op in (dev.OP_MIN_I64, dev.OP_MAX_I64):
            acc[c] = v if c not in acc else (min if op == dev.OP_MIN_I64 else max)(acc[c], v)
        else:
            # the device orders float bits as their sign-magnitude codes: -0.0 < 0.0, NaN beyond the infinities
            b = f64_bits(v)
            enc = b ^ (M64 if b >> 63 else 1 << 63)
            acc[c] = enc if c not in acc else (min if op == dev.OP_MIN_F64 else max)(acc[c], enc)
    if op in (dev.OP_MIN_F64, dev.OP_MAX_F64):
        return {c: (e ^ (1 << 63) if e >> 63 else ~e & M64) for c, e in acc.items()}
    return acc

"""Computed keys and values of field folds (`int(r[2]) * int(r[3])`, `int(r[0]) // 3600`, `len(l.split())`, constant
keys, dampr_text_fields_expr): the matchers (lowering.text_fields_expr, plan._match_text_fields through one map), the
programs against CPython on seeded rows (the plain-Python evaluator of tests/fields_expr_standin.py), the planner path
on that stand-in, and the results against the REAL reference (Refefer/Dampr), whose outputs are stored in
tests/golden/text_fields_expr.json.gz (DAMPR_REFERENCE=<checkout> records them again). The same pipelines run on the
device in tests/test_gpu_text_fields_expr.py."""
import math
import os
import random

import pytest

from fields_expr_standin import I64_MIN, eval_program, expr_line, make_expr_ctx
from fields_standin import _int18, parse_f64, python_lines, reference_outputs, run_ours, write_files
from test_text_fields_where_lowering import same_up_to_rounding

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_expr.json.gz")
NEEDLE = "device text fields scan+combine"


def ours(src, P, monkeypatch):
    return run_ours(src, P, monkeypatch, ctx=make_expr_ctx())


def _match(pm):
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    return plan._match_text_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]])


# ---- inputs -----------------------------------------------------------------------------------------------------
def csv_text(n, seed, cr=False):
    """`host,start,end,price,qty,latency` rows: timestamps, prices and quantities (ints written 7 / +7 / 07), latencies
    that are multiples of 1/8 (sums exact in any order), blank and short rows, a
    non-ASCII host. cr: some rows hold '\\r' inside"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        r = rng.random()
        if r < 0.03:
            rows.append(rng.choice(["", "x", "a,1"]))
            continue
        start = rng.randrange(0, 90000)
        f = [rng.choice(["h1", "h2", "host-with-a-long-name", "é"]), str(start), str(start + rng.randrange(0, 5000)),
             rng.choice(["%d", "+%d", "0%d"]) % rng.randrange(1, 1000), str(rng.randrange(1, 50)),
             "%.3f" % (rng.randrange(0, 64) / 8.0)]
        line = ",".join(f)
        if cr and i % 17 == 3:
            line = line.replace(",", "\r,", 1)
        rows.append(line)
    return "".join(r + "\n" for r in rows)


def log_text(n, seed):
    """access-log rows split by whitespace: `host - - [ts] "GET /p HTTP/1.1" status bytes`, some with fewer fields"""
    rng = random.Random(seed)
    rows = []
    for _ in range(n):
        if rng.random() < 0.04:
            rows.append(rng.choice(["", "   ", "short line"]))
            continue
        rows.append("%s - - [t%d] \"%s /p%d HTTP/1.1\" %d %d" % (
            rng.choice(["10.0.0.1", "10.0.0.2", "h"]), rng.randrange(100), rng.choice(["GET", "POST"]),
            rng.randrange(9), rng.choice([200, 204, 301, 404, 500]), rng.randrange(0, 1 << 20)))
    return "".join(r + "\n" for r in rows)


def datasets():
    csv = csv_text(300, 31)
    csv_cr = csv_text(200, 32, cr=True)
    return {
        "csv": [["sales.csv", csv]],
        "csv_gz": [["sales.csv.gz", csv_cr.replace("\n", "\r\n")]],
        "ws": [["access.log", log_text(300, 33)]],
        "words": [["words.txt", "a b c\n\nd e\nf\n  g   h i j\n" * 20]],
    }


C = "Dampr.text(P).map(lambda l: l.split(','))"
CF = C + ".filter(lambda r: len(r) == 6)"
CSV = [
    "Dampr.text(P).filter(lambda l: len(l.split(',')) == 6).fold_by(lambda l: l.split(',')[0], "
    "value=lambda l: int(l.split(',')[3]) * int(l.split(',')[4]), binop=lambda a, b: a + b)",
    "Dampr.text(P).filter(lambda l: len(l.split(',')) == 6).map(lambda l: float(l.split(',')[5])).mean()",
    "Dampr.text(P).filter(lambda l: len(l.split(',')) == 6).map(lambda l: int(l.split(',')[1])).count(lambda x: x % 2)",
    CF + ".a_group_by(lambda r: r[0], lambda r: float(r[5]) / 1000).sum()",
    CF + ".a_group_by(lambda r: r[0], lambda r: int(r[2]) - int(r[1])).reduce(max)",
    CF + ".a_group_by(lambda r: int(r[1]) // 3600, lambda r: int(r[3])).sum()",
    CF + ".count(lambda r: len(r[0]))",
    CF + ".mean(lambda r: r[0], lambda r: int(r[3]) / int(r[4]))",
    CF + ".a_group_by(lambda r: r[0], lambda r: -abs(float(r[5]) - 4.0625)).reduce(min)",
    CF + ".filter(lambda r: int(r[4]) > 0).a_group_by(lambda r: int(r[3]) // int(r[4]) % 7, "
         "lambda r: int(float(r[5]) * 10)).sum()",
]
WS = [
    "Dampr.text(P).map(lambda v: len(v.split())).a_group_by(lambda x: 1).sum()",
    "Dampr.text(P).filter(lambda l: len(l.split()) == 10).count(lambda l: int(l.split()[8]) // 100)",
    "Dampr.text(P).filter(lambda l: len(l.split()) == 10).map(lambda l: (l.split()[0], int(l.split()[9])))"
    ".a_group_by(lambda t: t[0], lambda t: t[1]).sum()",
    "Dampr.text(P).filter(lambda l: len(l.split()) == 10).map(lambda l: (l.split()[0], int(l.split()[9]) // 1024))"
    ".a_group_by(lambda t: t[1] % 4, lambda t: len(t[0])).reduce(max)",
]
WORDS = ["Dampr.text(P).map(lambda v: len(v.split())).a_group_by(lambda x: 1).sum()",
         "Dampr.text(P).map(lambda v: len(v.split())).count(lambda n: n // 2)",
         "Dampr.text(P).map(lambda v: float(len(v.split()))).mean()"]
PIPELINES = {"csv": CSV, "csv_gz": CSV[:6], "ws": WS, "words": WORDS}


# ---- the matchers -----------------------------------------------------------------------------------------------
def test_the_issue_examples_are_lowered(tmp_path):
    from dampr_b200 import Dampr, device as dev
    from operator import add
    t = Dampr.text(write_files(tmp_path, [["f.csv", "a,1,2,3,4,5,6,7,8,9\n"]]))
    sp = lambda l: l.split(",")   # noqa: E731
    stages = [
        t.map(lambda v: len(v.split())).a_group_by(lambda x: 1).sum(),
        t.map(lambda l: float(l.split(",")[3])).mean(),
        t.fold_by(lambda l: l.split(",")[0], value=lambda l: int(l.split(",")[3]) * int(l.split(",")[4]), binop=add),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: float(r[5]) / 1000).sum(),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: int(r[9]) // 1024).sum(),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: int(r[2]) - int(r[1])).sum(),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: len(r[1])).sum(),
        t.count(lambda l: int(l.split()[8]) // 100),
        t.map(sp).a_group_by(lambda r: int(r[0]) // 3600, lambda r: int(r[3])).sum(),
        t.map(lambda l: int(l.split(",")[1])).count(lambda x: x % 2),
    ]
    for pm in stages:
        m = _match(pm)
        assert m is not None and m[5] is not None, pm
    # the record-building map: bare projections after the composition, so today's plain spec
    m = _match(t.map(lambda l: (l.split()[0], int(l.split()[9]))).a_group_by(lambda t: t[0], lambda t: t[1]).sum())
    assert m[1] == (dev.FIELD_SEP_WS, 0, dev.FIELD_KEY_STR, 9) and m[5] is None


def test_the_matcher_refuses_what_is_not_lowered(tmp_path):
    from dampr_b200 import Dampr
    t = Dampr.text(write_files(tmp_path, [["f.csv", "a,1,2\n"]]))
    sp = lambda l: l.split(",")   # noqa: E731
    for pm in [
        t.map(sp).count(lambda r: (r[0], int(r[1]) // 2)),                   # expression in a tuple key
        t.map(sp).a_group_by(lambda r: (r[0], r[1]), lambda r: int(r[2]) * 2).sum(),
        t.map(sp).count(lambda r: float(r[1]) * 2),                           # float key
        t.map(sp).a_group_by(lambda r: r[0], lambda r: int(r[1]) ** 2).sum(),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: min(int(r[1]), int(r[2]))).sum(),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: float(r[1]) // 2).sum(),   # float //
        t.map(sp).a_group_by(lambda r: r[0], lambda r: float(r[1]) % 2).sum(),
        t.map(sp).a_group_by(lambda r: r[0], lambda r: len(r[1].strip())).sum(),   # a string method
        t.map(lambda l: int(l.split(",")[1]) * 2).filter(lambda x: x > 3).count(lambda x: x % 2),   # computed filter
        t.map(sp).filter(lambda r: r[0] == "a" and r[1] == "b").count(lambda r: int(r[1]) % 2),
        t.map(lambda x: len(x)).count(lambda n: n // 10),                     # the whole line's length
        t.count(lambda l: len(l) // 10),
        t.map(lambda l: (int(l.split(",")[1]), int(l.split(",")[2]))).count(lambda p: p[0] % 2),   # unused element
        t.map(lambda l: int(l.split(",")[1])).count(lambda x: 1),                                 # unused map
        t.map(sp).count(lambda r: int(r[0]) + int(r[1]) + int(r[2]) + int(r[3]) + int(r[4])),    # 5 loads
        t.map(sp).count(lambda r: int(r[0]) * True),                          # a bool constant
        t.map(sp).count(lambda r: int(r[1]) + (1 << 70)),                      # an int constant outside int64
        Dampr.json(write_files(tmp_path, [["g.jsonl", '{"a": 1}\n']])).count(lambda r: r["a"] % 2),
    ]:
        assert _match(pm) is None, pm


def test_old_shapes_keep_their_spec(tmp_path):
    from dampr_b200 import Dampr, device as dev, lowering
    t = Dampr.text(write_files(tmp_path, [["f.csv", "a,1,2\n"]]))
    sp = lambda l: l.split(",")   # noqa: E731
    m = _match(t.map(sp).filter(lambda r: r[1] != "x").a_group_by(lambda r: r[0], lambda r: int(r[2])).sum())
    assert m[1] == (ord(","), 0, dev.FIELD_KEY_STR, 2) and m[4] == ((dev.PRED_STR, 1, dev.CMP_NE, ("x",)),)
    assert m[5] is None and len(m) == 6
    assert _match(t.count(lambda l: int(l.split()[1])))[5] is None
    # text_fields_spec itself is unchanged: it refuses every computed shape
    assert lowering.text_fields_spec(lambda r: r[0], lambda r: int(r[1]) * 2, sp, whitespace=True) is None
    assert lowering.text_fields_spec(lambda x: 1, lambda r: 1, sp) is None


def test_the_spec_and_programs():
    from dampr_b200 import lowering as L
    sp = lambda l: l.split(",")   # noqa: E731
    EV = L._EV
    got = L.text_fields_expr(lambda r: r[0], lambda r: int(r[3]) * int(r[4]), sp)
    assert got == (",", 0, L.FIELD_STR, L.FIELD_EXPR, L.FIELD_INT, False,
                   (None, ("i", [EV["LOAD"], EV["LOAD"] | 1 << 8, EV["IMUL"]]), [], [],
                    [(3, L.LOAD_INT), (4, L.LOAD_INT)]))
    got = L.text_fields_expr(lambda x: 1, lambda x: x, lambda v: len(v.split()))
    assert got == (L.SEP_WS, None, L.FIELD_INT, L.FIELD_EXPR, L.FIELD_INT, False,
                   (("i", [EV["CI"]]), ("i", [EV["NF"]]), [1], [], []))
    # the value program's constants follow the key program's in the shared pool
    got = L.text_fields_expr(lambda r: int(r[0]) // 60, lambda r: float(r[1]) * 2.5 + 7, sp)
    assert got[6] == (("i", [EV["LOAD"], EV["CI"], EV["IFLOOR"]]),
                      ("f", [EV["LOAD"] | 1 << 8, EV["CF"], EV["FMUL"], EV["CI"] | 1 << 8, EV["I2F"], EV["FADD"]]),
                      [60, 7], [2.5], [(0, L.LOAD_INT), (1, L.LOAD_F64)])
    # limits: 33 operations, a stack of 9
    long_sum = eval("lambda r: " + " + ".join(["int(r[0])"] * 17))
    assert L.text_fields_expr(lambda r: r[1], long_sum, sp) is None
    deep = eval("lambda r: " + "(1 - " * 7 + "int(r[0])" + ")" * 7)
    assert L.text_fields_expr(lambda r: r[1], deep, sp) is not None
    deeper = eval("lambda r: " + "(1 - " * 8 + "int(r[0])" + ")" * 8)
    assert L.text_fields_expr(lambda r: r[1], deeper, sp) is None


# ---- the programs against CPython ------------------------------------------------------------------------------
LEAVES = ["int(r[0])", "int(r[1])", "float(r[2])", "len(r)", "len(r[3])", "3", "-7", "1.5", "0", "-0.0"]


def random_lambda(rng, depth=0):
    """the source of a random expression over the leaves and operations the device takes"""
    if depth > 2 or rng.random() < 0.3:
        return rng.choice(LEAVES)
    k = rng.random()
    a = random_lambda(rng, depth + 1)
    if k < 0.15:
        return rng.choice(["-(%s)", "abs(%s)", "float(%s)"]) % a
    b = random_lambda(rng, depth + 1)
    return "(%s %s %s)" % (a, rng.choice(["+", "-", "*", "/", "//", "%"]), b)


def random_rows(rng, n):
    ints = ["0", "1", "-1", "7", "+7", "07", str(1 << 53), str((1 << 53) + 1), "999999999999999999",
            "-999999999999999999", "3037000499", "-3037000500", "x"]
    floats = ["0.0", "-0.0", "1e308", "-1e308", "5e-324", "2.5", "inf", "1e-300", "3", "x"]
    out = []
    for _ in range(n):
        f = [rng.choice(ints), rng.choice(ints), rng.choice(floats), rng.choice(["", "ab", "abcdefghij"])]
        out.append(",".join(f[:rng.choice([4, 4, 4, 3])]).encode())
    return out


class _HostRule(Exception):
    """a line the header's rules hand to the host although CPython returns a value"""


class _I(int):
    """an int that raises _HostRule when an operation on it leaves int64, or an int / int has an operand beyond 2^53"""


def _checked(r):
    if type(r) is int:
        if not -(1 << 63) <= r < (1 << 63):
            raise _HostRule()
        return _I(r)
    return r


def _int_op(name):
    base = getattr(int, name)

    def op(self, *o):
        if name in ("__truediv__", "__rtruediv__") and type(o[0]) in (int, _I) and \
                max(abs(int(self)), abs(int(o[0]))) > (1 << 53):
            raise _HostRule()
        r = base(int(self), *[int(x) if type(x) is _I else x for x in o])
        return r if r is NotImplemented else _checked(r)
    return op


for _name in ("__add__", "__radd__", "__sub__", "__rsub__", "__mul__", "__rmul__", "__floordiv__", "__rfloordiv__",
              "__mod__", "__rmod__", "__truediv__", "__rtruediv__", "__neg__", "__abs__"):
    setattr(_I, _name, _int_op(_name))


def _load_int(x):
    if type(x) is str and _int18(x.encode()) is None:
        int(x)               # Python's ValueError, if it raises
        raise _HostRule()    # more than 18 digits, blanks, underscores: Python's int, not the device's
    return _checked(int(x))


def _load_float(x):
    if type(x) is str and parse_f64(x.encode()) is None:
        float(x)
        raise _HostRule()    # inf, nan, more than 19 significant digits: Python's float, not the device's
    return float(x)


def _python(src, line):
    """CPython's value of `lambda r: src` over the line's split, its exception, or _HostRule() where the rules name the
    line the host's although Python returns: an int result or intermediate leaving int64, an int / int beyond 2^53,
    a field only Python parses"""
    fn = eval("lambda r: " + src, {"int": _load_int, "float": _load_float, "len": lambda x: _I(len(x))})
    try:
        r = fn(line.decode().split(","))
        return int(r) if type(r) is _I else r
    except (ValueError, ZeroDivisionError, IndexError, OverflowError, TypeError, _HostRule) as e:
        return e


def _same(a, b):
    return type(a) is type(b) and (a == b and (type(a) is not float or math.copysign(1, a) == math.copysign(1, b))
                                   or (type(a) is float and a != a and b != b))


def test_programs_equal_python_bit_for_bit():
    """every line the evaluator takes gives CPython's value and type, and it hands to the host exactly the lines on
    which CPython raises or that the rules name: an int result or intermediate leaving int64, an int / int beyond 2^53,
    a field only Python parses"""
    from dampr_b200 import device as dev, lowering
    rng = random.Random(5)
    rows = random_rows(rng, 200)
    tried = taken = 0
    for _ in range(150):
        src = "lambda r: " + random_lambda(rng)
        fn = eval(src)
        got = lowering.text_fields_expr(lambda r: r[0], fn, lambda l: l.split(","))
        if got is None or got[6] is None:   # a bare projection: the plain scan's
            continue
        tried += 1
        kp, vp, ci, cf, loads = got[6]
        expr = (None, ((dev.EXPR_INT if vp[0] == "i" else dev.EXPR_F64), vp[1]), ci, cf,
                [(i, k) for i, k in loads])
        op = dev.OP_SUM_I64 if vp[0] == "i" else dev.OP_MIN_F64
        for line in rows:
            f = line.split(b",")
            want = _python(src[len("lambda r: "):], line)
            kv = expr_line(line, f, expr, (ord(","), 0, dev.FIELD_KEY_STR, 0, op))
            assert (kv is None) == isinstance(want, Exception), (src, line, kv, want)
            if kv is None:
                continue
            taken += 1
            assert _same(kv[1], want) and _same(kv[1], fn(line.decode().split(","))), (src, line, kv[1], want)
    assert tried > 50 and taken > 1000


@pytest.mark.parametrize("src,line,host", [
    ("int(r[0]) * int(r[1])", b"3037000499,3037000499", False),
    ("int(r[0]) * int(r[1])", b"3037000500,3037000500", True),           # leaves int64
    ("int(r[0]) + int(r[1])", b"999999999999999999,999999999999999999", False),
    ("-(int(r[0]) - int(r[1]) * 10)", b"-999999999999999999,999999999999999999", True),
    ("-(int(r[0]) - int(r[1]) * 10)", b"-99999999999999999,99999999999999999", False),
    ("int(r[0]) * int(r[1]) * 10", b"99999999,999999999", False),
    ("int(r[0]) * int(r[1]) * 10", b"999999999999,999999999", True),
    ("int(r[0]) / int(r[1])", b"9007199254740992,3", False),             # 2^53
    ("int(r[0]) / int(r[1])", b"9007199254740993,3", True),              # 2^53 + 1
    ("int(r[0]) / int(r[1])", b"1,0", True),                             # ZeroDivisionError
    ("int(r[0]) // int(r[1])", b"-7,0", True),
    ("int(r[0]) % int(r[1])", b"-7,2", False),
    ("int(r[0]) // int(r[1])", b"-7,2", False),
    ("float(r[0]) / float(r[1])", b"1,-0.0", True),
    ("float(r[0]) / float(r[1])", b"1e308,1e-308", False),               # inf, as in Python
    ("int(float(r[0]))", b"1e19,1", True),                               # outside int64
    ("int(float(r[0]))", b"inf,1", True),
    ("int(float(r[0]))", b"-9.2e18,1", False),
    ("abs(int(r[0]) * int(r[1]))", b"-3037000499,3037000499", False),
    ("float(r[0]) * 10", b"1e308,1", False),
    ("int(r[2]) + 1", b"1,2", True),                                      # IndexError
])
def test_the_host_rules(src, line, host):
    from dampr_b200 import device as dev, lowering
    fn = eval("lambda r: " + src)
    got = lowering.text_fields_expr(lambda r: r[0], fn, lambda l: l.split(","))
    kp, vp, ci, cf, loads = got[6]
    expr = (None, (dev.EXPR_INT if vp[0] == "i" else dev.EXPR_F64, vp[1]), ci, cf, loads)
    op = dev.OP_SUM_I64 if vp[0] == "i" else dev.OP_SUM_F64
    kv = expr_line(line, line.split(b","), expr, (ord(","), 0, dev.FIELD_KEY_STR, 0, op))
    assert (kv is None) == host, (src, line, kv)
    if not host:
        assert _same(kv[1], fn(line.decode().split(",")))


def test_an_int64_min_key_is_the_hosts():
    from dampr_b200 import device as dev
    assert eval_program([1, 1 | 1 << 8, 5], [-(1 << 62), 1 << 62], [], [], 0) == I64_MIN
    expr = ((dev.EXPR_INT, [1, 1 | 1 << 8, 5]), None, [-(1 << 62), 1 << 62], [], [])
    assert expr_line(b"a", [b"a"], expr, (ord(","), 0, dev.FIELD_KEY_INT, dev.FIELD_VAL_ONE, dev.OP_SUM_I64)) is None


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_expr_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = ours(src, P, monkeypatch)
        same_up_to_rounding(got, e)
        assert NEEDLE in hows[0], (name, src, hows, stages)
        d = stages[0][2]
        assert (" value=expr" in d or " key=expr" in d or " key=const" in d) == (src != WS[2]), (src, d)


def test_details(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.txt", "a b\n\nc d e\n"]])
    got, hows, stages = ours("Dampr.text(P).map(lambda v: len(v.split())).a_group_by(lambda x: 1).sum()", P,
                             monkeypatch)
    assert got == ["(1, 5)"] and stages[0][2] == "op=sum_i64 bytes=11 lines=3 groups=1 host_lines=0 sep=ws value=expr " \
                                                 "key=const"
    got, hows, stages = ours("Dampr.text(P).count(lambda l: len(l.split()) % 2)", P, monkeypatch)
    assert got == ["(0, 2)", "(1, 1)"] and stages[0][2].endswith(" sep=ws key=expr") and "op=count" in stages[0][2]
    P = write_files(tmp_path, [["g.csv", "a,2,3\nb,4,5\na,1,1\n"]])
    got, hows, stages = ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], "
                             "lambda r: int(r[1]) * int(r[2])).sum()", P, monkeypatch)
    assert got == ["('a', 7)", "('b', 20)"] and stages[0][2].endswith(" value=expr")


def test_keys_with_device_and_host_lines_merge(monkeypatch, tmp_path):
    """a key whose lines are split between the device and the host comes back once, folded over both"""
    rows = ["%d,%s,%d" % (i, "é" if i % 3 == 0 else "x", i * 7) for i in range(300)]
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    src = "Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: int(r[0]) % 4, lambda r: int(r[2]) * 3).sum()"
    got, hows, stages = ours(src, P, monkeypatch)
    exp = {}
    for l in python_lines(P):
        r = l.split(",")
        exp[int(r[0]) % 4] = exp.get(int(r[0]) % 4, 0) + int(r[2]) * 3
    assert got == sorted(repr(x) for x in exp.items())
    assert NEEDLE in hows[0] and "host_lines=100" in stages[0][2], stages


def test_host_keys_outside_int64_refuse(monkeypatch, tmp_path):
    """a 20-digit field parses on the host only and its key leaves int64: the stage is the host map's"""
    P = write_files(tmp_path, [["f.csv", "1\n99999999999999999999\n2\n"]])
    got, hows, _s = ours("Dampr.text(P).count(lambda l: int(l.split(',')[0]) * 2)", P, monkeypatch)
    assert got == ["(199999999999999999998, 1)", "(2, 1)", "(4, 1)"] and NEEDLE not in hows[0]


def test_nan_and_negative_zero_under_min_max_refuse(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1e308\na,-1e308\nb,0\n"]])
    for src in ["Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], "
                "lambda r: float(r[1]) * 10 - float(r[1]) * 10).reduce(max)",
                "Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], "
                "lambda r: -float(r[1])).reduce(min)"]:
        got, hows, _s = ours(src, P, monkeypatch)
        assert NEEDLE not in hows[0], src


@pytest.mark.parametrize("src,exc", [
    ("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], lambda r: int(r[1]) // int(r[2])).sum()",
     ZeroDivisionError),
    ("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], lambda r: int(r[1]) * int(r[3])).sum()",
     IndexError),
    ("Dampr.text(P).count(lambda l: float(l.split(',')[1]) / 0)", ZeroDivisionError),
])
def test_raising_lambdas_raise_as_in_python(src, exc, monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1,2,3\nb,2,0,3\nc,3,1\n"]])
    with pytest.raises(exc):
        ours(src, P, monkeypatch)

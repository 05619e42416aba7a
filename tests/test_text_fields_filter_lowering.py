"""Filter programs in front of a field fold: `and` / `or` / `not`, string tests (`"ERROR" in l`, `r[6].startswith(...)`,
`len(r[1]) > 3`, `l.strip()`) and whole-line tests. Covers the bytecode analysis of the short circuit
(lowering.analyze), the program matchers (lowering.filter_program, lowering.json_filter_program), the stage matchers
with and without `programs=True`, the binding's packing, the planner on the numpy stand-in of
tests/fields_filter_standin.py against the REAL reference (tests/golden/text_fields_filter.json.gz; DAMPR_REFERENCE=
<checkout> records it again) and, where a lambda raises, against plain Python (the reference hangs when one of its
workers raises). The same pipelines run on the device in tests/test_gpu_text_fields_filter.py."""
import itertools
import os
import random

import pytest

from fields_filter_standin import combine, make_filter_ctx
from fields_standin import python_lines, reference_outputs, run_ours, write_files

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_filter.json.gz")
NEEDLE = "device text fields scan+combine"
HEADER = "ts,method,status,bytes,latency,host,path"
METHODS = ("GET", "POST")
PREFIX_LIST = ["a", "b"]   # str.startswith / endswith raise TypeError on a list


def log_text(n, seed):
    """a web-log CSV: a header, '#' comments, blank and blank-looking lines, short rows, rows whose status or bytes no
    int() takes, and 7-field rows with paths under /api/, /static/ and /x"""
    rng = random.Random(seed)
    rows = [HEADER]
    for i in range(n):
        r = rng.random()
        if r < 0.04:
            rows.append(rng.choice(["# comment", "#", "", "   ", " \t "]))
        elif r < 0.08:
            rows.append(rng.choice(["short,GET", "s,GET,500", "s,POST,200,7"]))
        elif r < 0.12:
            rows.append("%d,BAD,x%d,oops,0.5,h,/api/v" % (i, i))
        else:
            rows.append("%d,%s,%d,%d,%s,%s,%s" % (
                rng.randrange(100), rng.choice(["GET", "POST", "PUT", "DELETE"]), rng.choice([200, 301, 404, 500, 503]),
                rng.randrange(-50, 5000), rng.choice(["0.25", "1e-3", "nan", "0.0", "2.5"]),
                rng.choice(["a", "bb", "ERROR-host", "timeout", " "]),
                rng.choice(["/api/users", "/api/x", "/static/a.js", "/x", "/", "/xERROR"])))
    return "".join(r + "\n" for r in rows)


def datasets():
    log = log_text(800, 11)
    return {"log": [["log.csv", log]], "log_gz": [["log.csv.gz", log]]}


C = "Dampr.text(P).map(lambda l: l.split(','))"
PIPELINES = {
    "log": [
        "Dampr.text(P).filter(lambda l: 'ERROR' in l).map(lambda l: l.split(',')).filter(lambda r: len(r) == 7)"
        ".count(lambda r: r[1])",
        "Dampr.text(P).filter(lambda l: not l.startswith('#') and l != '" + HEADER + "')" + C[13:] +
        ".filter(lambda r: len(r) == 7 and r[1] == 'GET' and (int(r[2]) >= 500 or r[6].startswith('/api/')))"
        ".a_group_by(lambda r: r[0], lambda r: int(r[3])).sum()",
        "Dampr.text(P).filter(lambda l: l.strip() and len(l) > 10)" + C[13:] +
        ".filter(lambda r: len(r) == 7 and r[1] not in ('BAD', 'method') and "
        "(not r[6].endswith(('.js', '/x')) or r[1] in ('PUT', 'DELETE')))"
        ".a_group_by(lambda r: r[1], lambda r: int(r[3])).reduce(max)",
        C + ".filter(lambda r: len(r) == 7 and not 'api' in r[6] and len(r[5]) <= 2)"
        ".filter(lambda r: r[1] != 'method').mean(lambda r: r[5], lambda r: float(r[4]))",
        "Dampr.text(P).filter(lambda l: l.split(',')[0] != 'ts' and ('ERROR' not in l or l.endswith('x')))"
        ".count(lambda l: l.split(',')[0])",
    ],
}
PIPELINES["log_gz"] = PIPELINES["log"][:2]


def ours(src, P, monkeypatch):
    return run_ours(src, P, monkeypatch, ctx=make_filter_ctx())


# ---- bytecode ------------------------------------------------------------------------------------------------------
def test_analyze_every_nesting_shape():
    from dampr_b200.lowering import analyze
    shapes = {
        "and(c0, c1)": lambda r: r[0] == "a" and r[1] == "b",
        "or(c0, c1)": lambda r: r[0] == "a" or r[1] == "b",
        "and(c0, or(c1, c2))": lambda r: r[0] == "a" and (r[1] == "b" or r[2] == "c"),
        "or(and(c0, c1), c2)": lambda r: (r[0] == "a" and r[1] == "b") or r[2] == "c",
        "not(or(c0, c1))": lambda r: not (r[0] == "a" or r[1] == "b"),
        "or(c0, and(not(c1), c2))": lambda r: r[0] == "a" or not r[1] == "b" and r[2] == "c",
        # CPython jumps from a straight to the end: a and b and c is a and (b and c), the same under the short circuit
        "and(c0, and(c1, c2))": lambda r: r[0] == "a" and r[1] == "b" and r[2] == "c",
        "or(and(c0, c1), and(c2, c3))": lambda r: r[0] == "a" and r[1] == "b" or r[2] == "c" and r[3] == "d",
        "not(not(c0))": lambda r: not not r[0] == "a",
    }

    def shape(e):
        if e.op in ("and", "or"):
            return "%s(%s, %s)" % (e.op, shape(e.a), shape(e.b))
        if e.op == "not":
            return "not(%s)" % shape(e.a)
        assert e.op == "cmp" and e.b.op == "sub"
        return "c%d" % e.b.b.a
    for want, fn in shapes.items():
        assert shape(analyze(fn)) == want
    eight = lambda r: (r[0] == "a" or r[1] == "b") and (r[2] == "c" or not r[3] == "d") and \
        (r[4] == "e" and r[5] == "f" or r[6] == "g" and r[7] == "h")   # noqa: E731
    assert shape(analyze(eight)) == "and(or(c0, c1), and(or(c2, not(c3)), or(and(c4, c5), and(c6, c7))))"


def test_analyze_refuses_other_jumps():
    from dampr_b200.lowering import analyze
    for fn in [lambda r: r[0] if r[1] else r[2], lambda r: 200 <= int(r[2]) < 300, lambda r: (x := r[0]) and x,
               lambda r: any(x == "a" for x in r)]:
        assert analyze(fn) is None, fn


def test_consumers_of_analyze_refuse_the_new_nodes():
    from dampr_b200 import lowering, vexpr
    import numpy as np
    e = lowering.analyze(lambda r: r[0] > 1 and r[1] < 2)
    assert lowering.depends_on(e, 0) is None
    assert lowering.numeric_program(e, 0, 1) is None
    with pytest.raises(vexpr.NotVec):
        vexpr.evaluate(e, [np.arange(3), np.arange(3)], False, 3)
    assert lowering.field_predicate(lambda r: r[0] == "a" and r[1] == "b", ",") is None
    assert lowering.json_predicate(lambda r: r["a"] == "x" or r["b"] == "y") is None
    assert lowering.text_fields_expr(lambda r: r[0] == "a" and r[1] == "b", lambda r: 1, lambda l: l.split(",")) \
        is None


# ---- program matchers ----------------------------------------------------------------------------------------------
def test_filter_program_leaves_and_connectives():
    from dampr_b200.lowering import LINE, filter_program, json_filter_program
    assert filter_program(lambda r: r[1] == "GET" and (int(r[2]) >= 500 or r[6].startswith("/api/")), ",") == [
        (",", "str", 1, "==", ("GET",)), (",", "int", 2, ">=", (500,)), (",", "str", 6, "startswith", ("/api/",)),
        "or", "and"]
    assert filter_program(lambda l: "ERROR" in l) == [(None, "str", LINE, "contains", ("ERROR",))]
    assert filter_program(lambda l: not l.startswith("#")) == [(None, "str", LINE, "startswith", ("#",)), "not"]
    assert filter_program(lambda l: l != HEADER) == [(None, "str", LINE, "!=", (HEADER,))]
    assert filter_program(lambda l: HEADER != l) == [(None, "str", LINE, "!=", (HEADER,))]
    assert filter_program(lambda l: l not in ("a", "b")) == [(None, "str", LINE, "not in", ("a", "b"))]
    assert filter_program(lambda l: len(l) > 0) == [(None, "len", LINE, ">", (0,))]
    assert filter_program(lambda l: 90 < len(l)) == [(None, "len", LINE, ">", (90,))]
    assert filter_program(lambda l: not l.strip()) == [(None, "nonblank", LINE, None, ()), "not"]
    assert filter_program(lambda r: r[6].endswith((".js", ".css")), ",") == [
        (",", "str", 6, "endswith", (".js", ".css"))]
    assert filter_program(lambda r: len(r[1]) <= 3 and "x" not in r[-1], ",") == [
        (",", "len", 1, "<=", (3,)), (",", "str", -1, "not contains", ("x",)), "and"]
    assert filter_program(lambda l: l.split()[0].startswith(METHODS), whitespace=True) == [
        ("<whitespace>", "str", 0, "startswith", METHODS)]
    assert filter_program(lambda r: len(r) == 7 or not float(r[3]) < 1.0, ",") == [
        (",", "nfields", None, "==", (7,)), (",", "float", 3, "<", (1.0,)), "not", "or"]
    assert json_filter_program(lambda r: r["level"] in ("ERROR", "WARN") or "timeout" in r["msg"]) == [
        ("str", "level", "in", ("ERROR", "WARN")), ("str", "msg", "contains", ("timeout",)), "or"]
    assert json_filter_program(lambda r: "a" in r and not r["b"].strip() and len(r["c"]) > 2) == [
        ("member", "a", "in", ()), ("nonblank", "b", None, ()), "not", ("len", "c", ">", (2,)), "and", "and"]


def test_filter_program_refusals():
    from dampr_b200.lowering import filter_program, json_filter_program
    nine = lambda r: r[0] == "a" and r[1] == "b" and r[2] == "c" and r[3] == "d" and r[4] == "e" and \
        r[5] == "f" and r[6] == "g" and r[7] == "h" and r[8] == "i"   # noqa: E731
    nine_ops = lambda r: not not not not not (r[0] == "a" and r[1] == "b" and r[2] == "c" and r[3] == "d" and
                                                r[4] == "e")   # noqa: E731
    big = tuple("k%d" % i for i in range(65))
    for fn, rec in [
        (lambda l: l, None), (lambda r: r[1], ","), (lambda l: "x" in l and l, None),
        (lambda r: "x" in r, ","), (lambda r: r[0] in "abc", ","), (lambda r: r[0] if r[1] else r[2], ","),
        (lambda r: 200 <= int(r[2]) < 300, ","), (nine, ","), (nine_ops, ","),
        (lambda l: l.startswith(big), None), (lambda l: "\ud800" in l, None), (lambda l: l.startswith("#", 1), None),
        (lambda l: l.startswith(()), None), (lambda l: len(l) > True, None), (lambda l: l.strip() == "", None),
        (lambda l: l.lower().startswith("a"), None), (lambda r: "x" in r[0] or r, ","),
        (lambda l: l.startswith(b"#"), None), (lambda l: 5 in l, None), (lambda r: r[0] == "a" and None, ","),
        (lambda l: l.startswith(PREFIX_LIST), None), (lambda r: r[1].endswith(PREFIX_LIST) or r[0] == "a", ","),
    ]:
        assert filter_program(fn, rec) is None, fn
    assert filter_program(lambda r: r[0].startswith("#") or "x" in r[1], ",") is not None
    assert json_filter_program(lambda r: "x" in r) is not None                       # member test
    assert json_filter_program(lambda r: r["a"] or r["b"] == "x") is None            # bare truthiness
    assert json_filter_program(lambda r: "x" in r["a"]["b"]) is None
    assert json_filter_program(lambda r: r["a"].startswith(PREFIX_LIST)) is None


# ---- stage matchers ------------------------------------------------------------------------------------------------
def stage_of(src, **kw):
    from dampr_b200 import Dampr, plan
    pm = eval(src, {"Dampr": Dampr, "P": "/nonexistent/x.csv", "json": __import__("json")})
    st = pm.pmer.graph.stages[-2] if src.endswith(".count()") else pm.pmer.graph.stages[0]
    match = plan._match_json_fields if "json" in src else plan._match_text_fields
    return match(st, [pm.pmer.graph.inputs[st.inputs[0]]], **kw)


def test_stage_matchers_take_programs_only_when_asked():
    from dampr_b200 import device as dev
    src = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[0] == 'a' and r[1] == 'b').count(lambda r: r[0])"
    assert stage_of(src) is None
    m = stage_of(src, programs=True)
    assert m[4] == ((dev.PRED_STR, 0, dev.CMP_EQ, ("a",)), (dev.PRED_STR, 1, dev.CMP_EQ, ("b",)),
                    (dev.PRED_AND, 0, dev.CMP_EQ, ()))
    plain = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[1] == 'b').count(lambda r: r[0])"
    assert stage_of(plain) == stage_of(plain, programs=True)
    line = "Dampr.text(P).filter(lambda l: 'ERROR' in l).map(lambda l: l.split()).count(lambda r: r[3])"
    assert stage_of(line) is None
    m = stage_of(line, programs=True)
    assert m[1][0] == dev.FIELD_SEP_WS and m[4] == ((dev.PRED_STR, dev.FIELD_LINE, dev.CMP_CONTAINS, ("ERROR",)),)
    js = "Dampr.json(P).filter(lambda r: r['level'] in ('ERROR', 'WARN') or 'timeout' in r['msg']).count(lambda r: r['svc'])"
    assert stage_of(js) is None
    m = stage_of(js, programs=True)
    assert m[5] == ("svc", "level", "msg")
    assert m[4] == ((dev.PRED_STR, 1, dev.CMP_IN, ("ERROR", "WARN")), (dev.PRED_STR, 2, dev.CMP_CONTAINS, ("timeout",)),
                    (dev.PRED_OR, 0, dev.CMP_EQ, ()))
    for src in [
        "Dampr.text(P).filter(lambda l: l).map(lambda l: l.split(',')).count(lambda r: r[0])",
        "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: 'x' in r).count(lambda r: r[0])",
        "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[0] == 'a' or r[1].split(';')[0] == 'b')"
        ".count(lambda r: r[0])",
        "Dampr.text(P).filter(lambda l: l.split(';')[0] == 'a' or 'x' in l).map(lambda l: l.split(','))"
        ".count(lambda r: r[0])",   # a field leaf on another separator than the key's
        "Dampr.text(P).map(lambda l: (int(l.split(',')[0]), 1)).filter(lambda t: t[0] > 0 or t[1] > 0)"
        ".count(lambda t: t[0])",   # behind a computing map
    ]:
        assert stage_of(src, programs=True) is None, src


def test_the_binding_packs_programs():
    from dampr_b200 import device as dev
    spec = (ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64)
    s = dev.fields_spec(spec, False, [(dev.PRED_STR, dev.FIELD_LINE, dev.CMP_STARTS, ("#", "//")),
                                      (dev.PRED_NOT, 0, dev.CMP_EQ, ()), (dev.PRED_LEN, 6, dev.CMP_GT, (3,)),
                                      (dev.PRED_NONBLANK, 2, dev.CMP_EQ, ()), (dev.PRED_OR, 0, dev.CMP_EQ, ()),
                                      (dev.PRED_AND, 0, dev.CMP_EQ, ())])
    assert s.npreds == 6 and s.preds[0].field == -(1 << 31) and s.preds[0].n == 2
    assert bytes(s.preds[0].bytes[:3]) == b"#//" and list(s.preds[0].lens[:2]) == [1, 2]
    assert [s.preds[i].kind for i in range(6)] == [dev.PRED_STR, dev.PRED_NOT, dev.PRED_LEN, dev.PRED_NONBLANK,
                                                   dev.PRED_OR, dev.PRED_AND]
    assert s.preds[2].ints[0] == 3 and s.preds[1].n == 0 and s.preds[3].n == 0


def test_left_sequential_logic_is_pythons_short_circuit():
    """a value that would raise is None: for every a, b the stand-in's combination equals Python's `a and b` /
    `a or b` / `not a` when neither raises, and is None exactly when Python's evaluation reaches a raising operand"""
    def py(op, a, b):
        def val(x):
            if x is None:
                raise ValueError
            return x
        try:
            return (not val(a)) if op == "not" else (val(a) and val(b)) if op == "and" else (val(a) or val(b))
        except ValueError:
            return None
    for op, a, b in itertools.product(("and", "or", "not"), (True, False, None), (True, False, None)):
        assert combine(op, a, b) == py(op, a, b), (op, a, b)


# ---- pipelines -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_programs_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, how, stages = ours(src, P, monkeypatch)
        assert got == exp, src
        assert NEEDLE in how[0] and "filtered=" in stages[0][2], (src, how)
        assert "host_lines=0" in stages[0][2] or "ERROR" in src or "nan" in src or "mean" in src, stages[0][2]


def test_u_leaves_never_hide_an_exception(monkeypatch, tmp_path):
    """Python raises only on the lines that reach r[9]; the device drops or takes the others"""
    P = write_files(tmp_path, [["t.csv", "a,x\nb,y\nc,x,1\n"]])
    src = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[1] == 'x' or int(r[9]) > 0).count(lambda r: r[0])"
    with pytest.raises(IndexError):
        ours(src, P, monkeypatch)
    P = write_files(tmp_path, [["u.csv", "a,x\nb,x,1\nc,y,1,2,3,4,5,6,7,10\n"]])
    got, how, stages = ours(src, P, monkeypatch)
    assert got == ["('a', 1)", "('b', 1)", "('c', 1)"] and NEEDLE in how[0]
    assert "host_lines=0" in stages[0][2]
    src = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[1] == 'y' and int(r[9]) > 0).count(lambda r: r[0])"
    got, how, stages = ours(src, P, monkeypatch)
    assert got == ["('c', 1)"] and "filtered=2" in stages[0][2]


def test_a_list_under_startswith_raises_as_in_python(monkeypatch, tmp_path):
    """str.startswith([...]) raises TypeError on every line: the stage stays on the host, which raises it"""
    from fake_device import FakePinned
    from dampr_b200 import Dampr, plan, settings
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: make_filter_ctx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})
    P = write_files(tmp_path, [["p.csv", "a,1\nb,2\nc,3\n"]])
    with pytest.raises(TypeError):
        [l for l in python_lines(P) if l.startswith(PREFIX_LIST)]
    for src in ["Dampr.text(P).filter(lambda l: l.startswith(PREFIX_LIST)).map(lambda l: l.split(','))"
                ".count(lambda r: r[0])",
                "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[0] == 'a' or r[1].endswith(PREFIX_LIST))"
                ".count(lambda r: r[0])"]:
        with pytest.raises(TypeError):
            eval(src, {"Dampr": Dampr, "P": P, "PREFIX_LIST": PREFIX_LIST}).run()


def test_nan_under_not_is_not_a_flipped_comparison(monkeypatch, tmp_path):
    text = "a,1,2,nan\nb,1,2,0.5\nc,1,2,3.0\nd,1,2,-0.0\n"
    P = write_files(tmp_path, [["n.csv", text]])
    src = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: not (float(r[3]) < 1.0)).count(lambda r: r[0])"
    got, how, stages = ours(src, P, monkeypatch)
    exp = sorted(repr((r[0], 1)) for r in (l.split(",") for l in python_lines(P)) if not (float(r[3]) < 1.0))
    assert got == exp == ["('a', 1)", "('c', 1)"] and NEEDLE in how[0]

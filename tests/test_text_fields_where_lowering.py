"""`filter(...)` calls in front of a delimited-field fold (WHERE predicates of dampr_text_fields): the predicate matcher
(lowering.field_predicate), the stage matcher (plan._match_text_fields with filter* [map filter*] keyed chains), the
planner path on the numpy stand-in of tests/fields_where_standin.py, and the results against the REAL reference
(Refefer/Dampr), whose outputs are stored in tests/golden/text_fields_where.json.gz (DAMPR_REFERENCE=<checkout>
records them again). Cases where the user's lambda raises are checked against plain Python: the reference hangs when
one of its workers raises (SURVEY B6). The same pipelines run on the device in tests/test_gpu_text_fields_where.py."""
import ast
import os
import random

import pytest

from fields_standin import python_lines, reference_outputs, run_ours, write_files
from fields_where_standin import make_where_ctx
from test_text_fields_lowering import datasets as int_datasets

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_where.json.gz")
NEEDLE = "device text fields scan+combine"


def ours(src, P, monkeypatch):
    """run_ours on the stand-in that takes WHERE predicates"""
    return run_ours(src, P, monkeypatch, ctx=make_where_ctx())

METHODS = ("GET", "POST")   # a global bound to a tuple: read at plan time


# ---- inputs -----------------------------------------------------------------------------------------------------
def log_text(n, seed):
    """a web-log style CSV `id,method,status,bytes,latency`: a header row, rows with too few fields, BAD rows whose
    bytes and latency no int() / float() takes (status 503, key 'ghost' only there), non-ASCII keys, CRLF rows"""
    rng = random.Random(seed)
    rows = ["id,method,status,bytes,latency"]
    for i in range(n):
        r = rng.random()
        if r < 0.05:
            rows.append("short,GET" if i % 2 else "short,GET,200")
        elif r < 0.15:
            rows.append("%s,BAD,503,x%d,oops" % (rng.choice(["ghost", "a", "b"]), i))
        else:
            rows.append("%s,%s,%d,%d,%s" % (rng.choice(["a", "b", "c", "", "é", "k" * 12, "zz"]),
                                            rng.choice(["GET", "POST", "PUT", "DELETE"]),
                                            rng.choice([200, 201, 301, 404, 500, 503]), rng.randrange(-500, 5000),
                                            rng.choice(["%.3f" % rng.uniform(0, 1), "1e-3", "0.5", "-0.0", " 2.25"])))
    return "".join(r + ("\r\n" if i % 37 == 5 else "\n") for i, r in enumerate(rows))


def datasets():
    d = dict(int_datasets())
    log = log_text(600, 7)
    d["log"] = [["log.csv", log]]
    d["log_gz"] = [["log.csv.gz", log]]
    d["log_issue"] = [["l.csv", "id,method,status,bytes\na,GET,500,1\nb,POST,503,7\nc,GET,200,x\na,PUT,500,9\n"
                                "a,GET,501,2\n"]]
    return d


C3 = "Dampr.text(P).map(lambda l: l.split(','))"
T3 = "Dampr.text(P).map(lambda l: l.split('\\t'))"
LOG = [C3 + ".filter(lambda r: len(r) == 5).filter(lambda r: r[0] != 'id').filter(lambda r: r[1] in ('GET', 'POST'))"
       ".a_group_by(lambda r: r[0], lambda r: int(r[3])).sum()",
       "Dampr.text(P).filter(lambda l: len(l.split(',')) >= 4).filter(lambda l: l.split(',')[1] != 'method')"
       ".map(lambda l: l.split(',')).filter(lambda r: int(r[2]) >= 300).count(lambda r: r[1])",
       C3 + ".filter(lambda r: len(r) == 5).filter(lambda r: r[1] not in ('BAD', 'method'))"
       ".filter(lambda r: float(r[4]) > 0.0).mean(lambda r: r[0], lambda r: float(r[4]))",
       C3 + ".filter(lambda r: len(r) > 4).filter(lambda r: r[1] == 'GET')"
       ".a_group_by(lambda r: r[0], lambda r: int(r[2])).reduce(max)",
       "Dampr.text(P).filter(lambda l: l.split(',')[0] >= 'k').count(lambda l: l.split(',')[0])",
       C3 + ".filter(lambda r: len(r) == 5).filter(lambda r: r[1] in ('GET', 'PUT'))"
       ".filter(lambda r: float(r[4]) != 0.0)"
       ".fold_by(lambda r: r[0], value=lambda r: float(r[4]), binop=lambda a, b: a + b)",
       C3 + ".filter(lambda r: len(r) == 5).filter(lambda r: r[0] != 'id').filter(lambda r: int(r[2]) in (200, 404))"
       ".a_group_by(lambda r: r[0], lambda r: int(r[3])).reduce(min)",
       "Dampr.text(P).filter(lambda l: l.split(',')[1] not in ('BAD', 'method')).map(lambda l: l.split(','))"
       ".filter(lambda r: 5 == len(r)).filter(lambda r: -0.0 < float(r[4]))"
       ".a_group_by(lambda r: r[0], lambda r: float(r[4])).reduce(min)",
       C3 + ".filter(lambda r: len(r) == 5).filter(lambda r: r[1] not in ('method', 'BAD'))"
       ".filter(lambda r: 1000 > int(r[3]))"
       ".mean(lambda r: r[1], lambda r: int(r[3]))"]
PIPELINES = {
    "issue": [C3 + ".filter(lambda r: r[1] != 'z').fold_by(lambda r: r[0], value=lambda r: int(r[2]), "
                   "binop=lambda a, b: a + b)"],
    "mixed": [C3 + ".filter(lambda r: r[1] != 'qq').fold_by(lambda r: r[0], value=lambda r: int(r[2]), "
                   "binop=lambda a, b: a + b)",
              "Dampr.text(P).filter(lambda l: int(l.split(',')[2]) > 0).count(lambda l: l.split(',')[0])",
              C3 + ".filter(lambda r: len(r) == 4).a_group_by(lambda r: r[0], lambda r: int(r[-1])).reduce(max)",
              C3 + ".filter(lambda r: r[0] < 'b').filter(lambda r: r[-2] in ('p', 'é'))"
                   ".a_group_by(lambda r: int(r[2]), lambda r: int(r[2])).reduce(min)"],
    "blank": ["Dampr.text(P).filter(lambda l: len(l.split(',')) >= 2).count(lambda l: l.split(',')[1])",
              "Dampr.text(P).filter(lambda l: l.split(',')[0] not in ('', 'a')).count(lambda l: l.split(',')[0])"],
    "gz": [T3 + ".filter(lambda r: int(r[1]) < 60).fold_by(lambda r: r[0], value=lambda r: int(r[2]), "
                "binop=lambda a, b: a + b)",
           T3 + ".filter(lambda r: r[-1] != '1').count(lambda r: r[0])"],
    "several": [C3 + ".filter(lambda r: r[0] in ('a', 'b', 'k9', '')).count(lambda r: r[0])",
                C3 + ".filter(lambda r: int(r[2]) <= 5).a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()"],
    "wide": [C3 + ".filter(lambda r: int(r[1]) >= 0).a_group_by(lambda r: r[0], lambda r: int(r[1])).sum()",
             C3 + ".filter(lambda r: r[0] == 'a').a_group_by(lambda r: r[0], lambda r: int(r[1])).reduce(max)"],
    "log": LOG,
    "log_gz": LOG,
    "log_issue": [C3 + ".filter(lambda r: r[0] != 'id').filter(lambda r: r[1] in ('GET', 'POST'))"
                       ".filter(lambda r: int(r[2]) >= 500).a_group_by(lambda r: r[0], lambda r: int(r[3])).sum()"],
}
PIPELINES["crlf_text"] = PIPELINES["gz"]


# ---- the predicate matcher --------------------------------------------------------------------------------------
def _pred(fn, sep=None):
    from dampr_b200 import lowering
    return lowering.field_predicate(fn, sep)


def test_predicate_matcher_accepts_the_table():
    from dampr_b200.lowering import FIELD_STR as S, FIELD_INT as I, FIELD_FLOAT as F, FIELD_COUNT as N
    codes = {"GET", "HEAD"}
    limits = [200, 404]
    frozen = frozenset(["a"])
    cases = [
        (lambda r: r[1] == "GET", ",", (",", S, 1, "==", ("GET",))),
        (lambda r: "GET" != r[1], ",", (",", S, 1, "!=", ("GET",))),
        (lambda r: r[-1] < "m", ",", (",", S, -1, "<", ("m",))),
        (lambda r: r[0] <= "é", ";", (";", S, 0, "<=", ("é",))),
        (lambda r: int(r[2]) > -5, ",", (",", I, 2, ">", (-5,))),
        (lambda r: 500 <= int(r[2]), ",", (",", I, 2, ">=", (500,))),
        (lambda r: int(r[2]) >= (1 << 63) - 1, ",", (",", I, 2, ">=", ((1 << 63) - 1,))),
        (lambda r: float(r[3]) < 0.5, ",", (",", F, 3, "<", (0.5,))),
        (lambda r: float(r[3]) == 7, ",", (",", F, 3, "==", (7.0,))),
        (lambda r: -(1 << 53) <= float(r[3]), ",", (",", F, 3, ">=", (-float(1 << 53),))),
        (lambda r: r[1] in ("GET", "POST"), ",", (",", S, 1, "in", ("GET", "POST"))),
        (lambda r: r[1] not in {"a", "b"}, ",", None),
        (lambda r: r[1] in METHODS, ",", (",", S, 1, "in", ("GET", "POST"))),
        (lambda r: r[1] in frozen, ",", (",", S, 1, "in", ("a",))),
        (lambda r: int(r[2]) in limits, ",", (",", I, 2, "in", (200, 404))),
        (lambda r: int(r[2]) not in (1, 2, 3), ",", (",", I, 2, "not in", (1, 2, 3))),
        (lambda r: len(r) == 4, ",", (",", N, None, "==", (4,))),
        (lambda r: 3 < len(r), ",", (",", N, None, ">", (3,))),
        (lambda l: l.split("|")[0] != "id", None, ("|", S, 0, "!=", ("id",))),
        (lambda l: int(l.split("\t")[2]) < 300, None, ("\t", I, 2, "<", (300,))),
        (lambda l: len(l.split(",")) >= 2, None, (",", N, None, ">=", (2,))),
        (lambda l: l.split(",")[1] in codes, None, None),
    ]
    for fn, sep, exp in cases:
        got = _pred(fn, sep)
        if exp is None:   # a set: its members in any order
            assert got is not None and got[:4] == ((",",) + got[1:4]) and got[3] in ("in", "not in"), got
            assert sorted(got[4]) == sorted({"a", "b"} if got[3] == "not in" else codes), got
        else:
            assert got == exp, (exp, got)


def test_predicate_matcher_rejects_the_near_misses():
    big = tuple(range(65))
    long_strs = ("x" * 600, "y" * 600)
    cases = [
        (lambda l: l, None),                                      # truthiness of the line
        (lambda r: r, ","),                                       # truthiness of the record
        (lambda r: r[1], ","),
        (lambda r: r[0] != "id" and r[1] == "GET", ","),          # and / or / not
        (lambda r: r[0] == "a" or r[0] == "b", ","),
        (lambda r: not r[0] == "a", ","),
        (lambda r: 0 < int(r[2]) < 5, ","),                       # chained comparison
        (lambda r: r[1].startswith("G"), ","),
        (lambda r: r[1].strip() == "GET", ","),
        (lambda l: l != "", None),                                # raw-line predicates
        (lambda l: "GET" in l, None),
        (lambda r: r[1] == 5, ","),                               # str against int
        (lambda r: r[1] < 5, ","),
        (lambda r: int(r[2]) == "5", ","),
        (lambda r: int(r[2]) < 5.5, ","),                         # float constant against int()
        (lambda r: int(r[2]) == True, ","),                       # bool constants
        (lambda r: len(r) == True, ","),
        (lambda r: int(r[2]) > (1 << 63), ","),                   # outside int64
        (lambda r: float(r[2]) < (1 << 53) + 1, ","),             # int beyond 2^53 against float()
        (lambda r: float(r[2]) in (1.0, 2.0), ","),               # float sets
        (lambda l: l.split(";")[0] == "a", ","),                  # another split (after map: not the record)
        (lambda r: r[0] in ("a", 1), ","),                        # mixed members
        (lambda r: int(r[0]) in ("1", "2"), ","),
        (lambda r: r[0] in (), ","),
        (lambda r: r[0] in "abc", ","),                           # substring test
        (lambda r: r[0] in big, ","),                             # more than 64 members
        (lambda r: r[0] in long_strs, ","),                       # more than 1 KB of strings
        (lambda r: r[0] == "\ud800", ","),                        # no UTF-8 bytes
        (lambda r: r[0] == r[1], ","),
        (lambda r: len(r[0]) == 3, ","),
        (lambda r: r[1:] == ["a"], ","),
        (lambda r, s=1: r[0] == "a", ","),
    ]
    for fn, sep in cases:
        assert _pred(fn, sep) is None, fn


# ---- the stage matcher -------------------------------------------------------------------------------------------
def _match(pm):
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    return plan._match_text_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]])


def test_stage_matcher_chains(tmp_path):
    from dampr_b200 import Dampr, device as dev
    P = write_files(tmp_path, [["f.csv", "a,GET,1\n"]])
    t = Dampr.text(P)
    key, val = (lambda r: r[0]), (lambda r: int(r[2]))
    sp = lambda l: l.split(",")
    m = _match(t.filter(lambda l: l.split(",")[1] == "GET").a_group_by(lambda l: l.split(",")[0],
                                                                        lambda l: int(l.split(",")[2])).sum())
    assert m is not None and m[4] == ((dev.PRED_STR, 1, dev.CMP_EQ, ("GET",)),)
    m = _match(t.map(sp).filter(lambda r: int(r[2]) >= 0).filter(lambda r: len(r) == 3).a_group_by(key, val).sum())
    assert m[4] == ((dev.PRED_INT, 2, dev.CMP_GE, (0,)), (dev.PRED_NFIELDS, 0, dev.CMP_EQ, (3,)))
    m = _match(t.filter(lambda l: l.split(",")[0] != "id").map(sp).filter(lambda r: float(r[2]) < 1.5)
               .mean(key, lambda r: float(r[2])))
    assert m[4] == ((dev.PRED_STR, 0, dev.CMP_NE, ("id",)), (dev.PRED_F64, 2, dev.CMP_LT, (1.5,))) and m[3]
    assert _match(t.map(sp).a_group_by(key, val).sum())[4] == ()
    for pm in [
        t.filter(lambda l: l).count(lambda l: l.split(",")[0]),                              # truthiness
        t.map(sp).filter(lambda r: r[1] == "GET").filter(lambda r: r).a_group_by(key, val).sum(),
        t.filter(lambda l: l.split(";")[1] == "GET").count(lambda l: l.split(",")[0]),       # another separator
        t.map(sp).filter(lambda r: r[1] == "GET").map(lambda r: r).a_group_by(key, val).sum(),   # two maps
        t.map(sp).filter(lambda r: r[1] == "GET").a_group_by(key, val).first(),
        t.map(sp).filter(lambda r: r[0] in tuple("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"))
         .filter(lambda r: r[1] in ("a", "b", "c")).a_group_by(key, val).sum(),              # 65 constants
        t.map(sp).filter(lambda r: r[0] != "x" * 600).filter(lambda r: r[1] != "y" * 600).a_group_by(key, val).sum(),
    ]:
        assert _match(pm) is None
    many = t.map(sp)
    for i in range(8):
        many = many.filter(lambda r: int(r[2]) != -1)
    assert len(_match(many.a_group_by(key, val).sum())[4]) == 8
    assert _match(many.filter(lambda r: int(r[2]) != -1).a_group_by(key, val).sum()) is None   # 9 predicates


def test_the_binding_refuses_what_the_device_refuses():
    from dampr_b200 import device as dev
    spec = (ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64)
    s = dev.fields_spec(spec, False, [(dev.PRED_STR, 1, dev.CMP_IN, ("a", "bc")), (dev.PRED_F64, -1, dev.CMP_LT, (0.5,)),
                                      (dev.PRED_INT, 2, dev.CMP_GE, (7,)), (dev.PRED_NFIELDS, 0, dev.CMP_EQ, (3,))])
    assert s.npreds == 4 and s.preds[0].n == 2 and list(s.preds[0].lens[:2]) == [1, 2]
    assert bytes(s.preds[0].bytes[:3]) == b"abc" and s.preds[1].f64 == 0.5 and s.preds[2].ints[0] == 7
    assert dev.fields_spec(spec, False, ()).npreds == 0


# ---- against the reference --------------------------------------------------------------------------------------
def same_up_to_rounding(got, exp):
    """sorted reprs equal; float sums and means, which the reference folds in its own combine order, within 2^-40
    relative (the line-order sum bound 4 n 2^-53 sum|v| of these small inputs lies well inside it)"""
    g, e = [ast.literal_eval(x) for x in got], [ast.literal_eval(x) for x in exp]
    assert [k for k, _ in g] == [k for k, _ in e], (got, exp)
    for (k, gv), (_k, ev) in zip(g, e):
        if type(ev) is float and type(gv) is float:
            assert abs(gv - ev) <= 2.0 ** -40 * max(1.0, abs(ev)), (k, gv, ev)
        else:
            assert repr(gv) == repr(ev), (k, gv, ev)


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_where_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = ours(src, P, monkeypatch)
        same_up_to_rounding(got, e)
        assert NEEDLE in hows[0] and "filtered=" in stages[0][2], (name, src, hows)


def test_the_issue_example():
    exp = reference_outputs(datasets()["log_issue"], PIPELINES["log_issue"], GOLDEN)
    assert exp[0] == ["('a', 3)", "('b', 7)"]


# ---- planner paths on the stand-in ------------------------------------------------------------------------------
def test_filtered_count_in_both_modes(monkeypatch, tmp_path):
    """filtered=N: the table-mode slot, and records - folded - host lines in record mode"""
    P = write_files(tmp_path, [["f.csv", "a,GET,1\nb,PUT,2\né,GET,3\na,GET,x\nb,PUT,y\nc,GET,1_0\n"]])
    for red in ("sum()", "reduce(max)"):
        with pytest.raises(ValueError):   # a GET row holds 'x': Python's own error
            ours(C3 + ".filter(lambda r: r[1] == 'GET').a_group_by(lambda r: r[0], lambda r: int(r[2])).%s"
                     % red, P, monkeypatch)
    P = write_files(tmp_path, [["g.csv", "a,GET,1\nb,PUT,2\né,GET,3\na,GET,4\nb,PUT,y\nc,GET,1_0\n"]])
    for src, op in [(C3 + ".filter(lambda r: r[1] == 'GET').a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()",
                     "op=sum_i64"),
                    (C3 + ".filter(lambda r: r[1] == 'GET').mean(lambda r: r[0], lambda r: float(r[2]))", "op=mean_f64")]:
        got, hows, stages = ours(src, P, monkeypatch)
        assert NEEDLE in hows[0] and op in stages[0][2], stages
        assert "filtered=2" in stages[0][2] and "host_lines=2" in stages[0][2] and "lines=4" in stages[0][2], stages
    assert got == ["('a', 2.5)", "('c', 10.0)", "('é', 3.0)"]


def test_rejected_rows_stay_on_the_device(monkeypatch, tmp_path):
    """more rejected rows than the fallback list holds, with keys and values no kernel parses: they are dropped, not
    handed back, and a key seen only on them does not appear"""
    P = write_files(tmp_path, [["f.csv", "ghost\x01,BAD,x\n" * 65600 + "a,GET,1\nb,GET,2\na,GET,3\n"]])
    got, hows, stages = ours(C3 + ".filter(lambda r: r[1] == 'GET').a_group_by(lambda r: r[0], "
                                 "lambda r: int(r[2])).sum()", P, monkeypatch)
    assert got == ["('a', 4)", "('b', 2)"]
    assert NEEDLE in hows[0] and "host_lines=0" in stages[0][2] and "filtered=65600" in stages[0][2], stages


def test_later_index_errors_behind_earlier_filters(monkeypatch, tmp_path):
    """a row an earlier filter rejects never meets a later filter's index or the key's; one it passes raises"""
    P = write_files(tmp_path, [["f.csv", "a,GET,1\nshort\nb,GET,2\n"]])
    src = C3 + ".filter(lambda r: len(r) == 3).filter(lambda r: r[1] == 'GET')" \
               ".a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()"
    got, hows, stages = ours(src, P, monkeypatch)
    assert got == ["('a', 1)", "('b', 2)"] and NEEDLE in hows[0] and "filtered=1" in stages[0][2]
    with pytest.raises(IndexError):
        ours(C3 + ".filter(lambda r: r[1] == 'GET').a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()", P,
                 monkeypatch)
    P = write_files(tmp_path, [["g.csv", "a,GET,1\nb,GET\n"]])
    with pytest.raises(IndexError):   # the filter passes, the value's field is missing
        ours(src.replace("len(r) == 3", "len(r) >= 2"), P, monkeypatch)


def test_nan_inf_and_signed_zero_follow_python(monkeypatch, tmp_path):
    """the float comparisons Python makes: NaN false except under !=, -0.0 == 0.0; inf constants"""
    rows = ["a,nan,1", "a,-0.0,2", "b,0.0,3", "b,inf,4", "c,-inf,5", "c,1e308,6", "d,-0,7", "d,2.5,8"]
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    for cond in ["float(r[1]) == 0.0", "float(r[1]) != 0.0", "float(r[1]) < 1", "float(r[1]) >= -0.0",
                 "float(r[1]) <= INF", "float(r[1]) > NINF", "float(r[1]) != NAN", "float(r[1]) == NAN"]:
        src = C3 + ".filter(lambda r: %s).a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()" % cond
        from dampr_b200 import Dampr
        from fake_device import FakePinned
        from dampr_b200 import settings, plan
        from dampr_b200 import runner as runner_mod
        monkeypatch.setattr(runner_mod, "_CTX", {settings.device: make_where_ctx()})
        monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
        monkeypatch.setattr(plan, "_BUFFERS", {})
        g = {"Dampr": Dampr, "P": P, "INF": float("inf"), "NINF": -float("inf"), "NAN": float("nan")}
        got = sorted(repr(x) for x in eval(src, g).run())
        exp = {}
        f = eval("lambda r: " + cond, g)
        for l in python_lines(P):
            r = l.split(",")
            if f(r):
                exp[r[0]] = exp.get(r[0], 0) + int(r[2])
        assert got == sorted(repr(x) for x in exp.items()), cond
        assert NEEDLE in runner_mod.LAST_STATS.stages[0][1], cond

"""`filter(...)` calls in front of a delimited-field fold on the device (the WHERE build of csrc/fields.cu): the
reference pipelines of tests/test_text_fields_where_lowering.py, every predicate kind and comparison on seeded inputs
against a plain-Python filter-then-fold, rejected rows that no kernel parses, index errors behind earlier filters,
tile seams and long lines, and float sums and means behind filters. Each case asserts which path the stage took."""
import operator
import random

import numpy as np
import pytest

from fields_standin import python_lines, reference_outputs, write_files
from test_text_fields_float_lowering import same_records
from test_text_fields_where_lowering import GOLDEN, NEEDLE, PIPELINES, datasets, same_up_to_rounding

pytestmark = pytest.mark.gpu


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "text_table_log2", settings.text_table_log2)
    monkeypatch.setattr(settings, "ingest_chunk_bytes", settings.ingest_chunk_bytes)
    yield settings
    plan.release_buffers()


def run(src, P, **env):
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    got = sorted(repr(x) for x in eval(src, dict(env, Dampr=Dampr, P=P)).run())
    return got, runner_mod.LAST_STATS.stages[0]


def python_where_fold(P, preds, key, value, binop):
    """plain Python: the records that pass every filter (in order), folded in line order"""
    out = {}
    for l in python_lines(P):
        r = l.split(",")
        if all(p(r) for p in preds):
            k, v = key(r), value(r)
            out[k] = binop(out[k], v) if k in out else v
    return sorted(repr(x) for x in out.items())


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, (_s, how, detail) = run(src, P)
        same_up_to_rounding(got, exp)
        assert NEEDLE in how and "filtered=" in detail, (name, src, how, detail)


def seeded_rows(seed, n=200000):
    """key (0, 1..9 and >= 10 bytes: the hashed path), a method, an int, a float with NaN / -0.0 / inf, and rows
    that hold fewer fields"""
    rng = random.Random(seed)
    keys = ["", "a", "bb", "x" * 9, "y" * 10, "z" * 30] + ["k%d" % i for i in range(200)]
    floats = ["nan", "-0.0", "0.0", "inf", "-inf", "0.5", "-2.25", "1e3", "7", "-0"]
    rows = []
    for i in range(n):
        f = "%r" % rng.uniform(-100, 100) if rng.random() < 0.6 else rng.choice(floats)
        rows.append("%s,%s,%d,%s" % (rng.choice(keys), rng.choice(["GET", "POST", "PUT", "g", ""]),
                                     rng.randrange(-1000, 1000), f))
        if i % 5000 == 7:
            rows[-1] = rows[-1].rsplit(",", 1)[0]
    return "\n".join(rows) + "\n"


OPS = ["==", "!=", "<", "<=", ">", ">="]
PRED_CASES = ([("r[1] %s 'POST'" % op) for op in OPS] + [("r[0] %s 'k5'" % op) for op in OPS] +
              [("int(r[2]) %s 17" % op) for op in OPS] + [("-3 %s int(r[2])" % op) for op in OPS] +
              [("float(r[3]) %s 0.0" % op) for op in OPS] + [("float(r[3]) %s NAN" % op) for op in ("==", "!=")] +
              [("float(r[3]) %s INF" % op) for op in ("<", ">=")] + [("len(r) %s 4" % op) for op in OPS] +
              ["r[1] in ('GET', 'g', '')", "r[1] not in METHODS", "r[0] in KEYS", "int(r[2]) in (1, -1, 999)",
               "int(r[2]) not in INTS"])


@pytest.mark.parametrize("cond", PRED_CASES)
def test_every_predicate_against_python(cond, engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", seeded_rows(len(cond) * 7 + ord(cond[-1]))]])
    env = {"NAN": float("nan"), "INF": float("inf"), "METHODS": ["GET", "PUT"],
           "KEYS": frozenset(["", "a", "y" * 10, "k7", "k150"]), "INTS": {0, 5, -7}}
    guard = "len(r) == 4" if "len(r)" not in cond else "len(r) >= 3"
    src = ("Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: %s).filter(lambda r: %s)"
           ".a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()" % (guard, cond))
    got, (_s, how, detail) = run(src, P, **env)
    g = dict(env)
    preds = [eval("lambda r: " + guard, g), eval("lambda r: " + cond, g)]
    assert got == python_where_fold(P, preds, lambda r: r[0], lambda r: int(r[2]), operator.add), cond
    assert NEEDLE in how and "filtered=" in detail, (how, detail)


@pytest.mark.parametrize("red,binop", [("sum()", operator.add), ("reduce(min)", min), ("reduce(max)", max)])
def test_filters_before_and_after_the_map(red, binop, engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", seeded_rows(11)]])
    src = ("Dampr.text(P).filter(lambda l: len(l.split(',')) == 4).filter(lambda l: l.split(',')[1] != 'g')"
           ".map(lambda l: l.split(',')).filter(lambda r: r[0] >= 'k1').a_group_by(lambda r: r[0], "
           "lambda r: int(r[2])).%s" % red)
    got, (_s, how, detail) = run(src, P)
    preds = [lambda r: len(r) == 4, lambda r: r[1] != "g", lambda r: r[0] >= "k1"]
    assert got == python_where_fold(P, preds, lambda r: r[0], lambda r: int(r[2]), binop)
    assert NEEDLE in how and "host_lines=0" in detail, detail


def test_rejected_rows_stay_on_the_device(engine, tmp_path):
    """more than 65,536 rejected rows whose keys and values no kernel parses: dropped on the device"""
    rows = ["é%d,BAD,x,y" % i if i % 2 else "bad%d\x01,BAD,1_0,z" % i for i in range(70000)]
    rows += ["a,GET,3,1.5", "b,GET,-4,2", "a,GET,5,0.25"]
    P = write_files(tmp_path, [["f.csv", "\n".join(r.replace("é", "e") for r in rows) + "\n"]])
    src = ("Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[1] == 'GET')"
           ".a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()")
    got, (_s, how, detail) = run(src, P)
    assert got == ["('a', 8)", "('b', -4)"]
    assert NEEDLE in how and "host_lines=0" in detail and "filtered=70000" in detail, detail
    got, (_s, how, detail) = run(src.replace("a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()",
                                             "mean(lambda r: r[0], lambda r: float(r[3]))"), P)
    assert got == ["('a', 0.875)", "('b', 2.0)"]
    assert NEEDLE in how and "host_lines=0" in detail and "filtered=70000" in detail, detail


def test_index_errors_behind_earlier_filters(engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,GET,1\n" * 3000 + "short\n" + "b,GET,2\n" * 3000]])
    src = ("Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: len(r) == 3).filter(lambda r: r[1] == 'GET')"
           ".a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()")
    got, (_s, how, detail) = run(src, P)
    assert got == ["('a', 3000)", "('b', 6000)"] and NEEDLE in how and "filtered=1" in detail, detail
    with pytest.raises(IndexError):
        run(src.replace(".filter(lambda r: len(r) == 3)", ""), P)


def test_seams_several_files_and_long_lines(engine, tmp_path):
    """rows across 16 KB tiles with small upload chunks, several files, a row past the 4 KB window (the host applies
    the filter), and a row of 64 KB or more (the whole stage goes to the host)"""
    engine.ingest_chunk_bytes = 1 << 16
    rng = np.random.default_rng(4)
    files = []
    for f in range(3):
        rows = ["k%d|%s|%d" % (rng.integers(0, 500), "p" * int(rng.integers(0, 90)), rng.integers(-50, 50))
                for _ in range(40000)]
        rows[100] = "long|" + "q" * 5000 + "|3"
        rows[101] = "long|" + "q" * 5001 + "|-3"
        rows[200] = "longer|" + "q" * 70000 + "|4"
        files.append(["p%d.txt" % f, "\n".join(rows) + ("" if f == 1 else "\n")])
    src = ("Dampr.text(P).filter(lambda l: int(l.split('|')[2]) >= 0)"
           ".a_group_by(lambda l: l.split('|')[0], lambda l: int(l.split('|')[2])).sum()")

    def exp(P):
        out = {}
        for l in python_lines(P):
            r = l.split("|")
            if int(r[2]) >= 0:
                out[r[0]] = out.get(r[0], 0) + int(r[2])
        return sorted(repr(x) for x in out.items())
    P = write_files(tmp_path, files)
    got, (_s, how, _d) = run(src, P)
    assert got == exp(P) and how.startswith("host-map"), how
    for f in files:
        f[1] = f[1].replace("q" * 70000, "q" * 60000)
    (tmp_path / "b").mkdir()
    P = write_files(tmp_path / "b", files)
    got, (_s, how, detail) = run(src, P)
    assert got == exp(P) and NEEDLE in how and "host_lines=6" in detail, (how, detail)


@pytest.mark.parametrize("red", ["sum()", "mean"])
def test_float_sums_and_means_behind_filters(red, engine, tmp_path):
    rng = random.Random(21)
    rows = []
    for i in range(100000):
        rows.append("%s,%s,%r,%d" % (rng.choice(["a", "b", "q" * 12, "w%d" % rng.randrange(100)]),
                                     rng.choice(["GET", "PUT"]), rng.uniform(-1e4, 1e4), i % 7))
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    base = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[1] == 'GET').filter(lambda r: int(r[3]) != 3)"
    src = base + (".mean(lambda r: r[0], lambda r: float(r[2]))" if red == "mean" else
                  ".a_group_by(lambda r: r[0], lambda r: float(r[2])).sum()")
    got, (_s, how, detail) = run(src, P)
    assert NEEDLE in how and "filtered=" in detail and "host_lines=0" in detail, detail
    keep = [l for l in python_lines(P) if l.split(",")[1] == "GET" and int(l.split(",")[3]) != 3]
    exp = {}
    for l in keep:
        r = l.split(",")
        s, n = exp.get(r[0], (0.0, 0))
        exp[r[0]] = (s + float(r[2]), n + 1)
    exp = {k: (s / float(n) if red == "mean" else s) for k, (s, n) in exp.items()}
    kp = tmp_path / "kept"
    kp.mkdir()
    KP = write_files(kp, [["k.csv", "\n".join(keep) + "\n"]])

    class V(object):
        def __call__(self, l):
            return float(l.split(",")[2])

        def __repr__(self):
            return "mean" if red == "mean" else "sum"
    same_records(got, sorted(repr(x) for x in exp.items()), KP, lambda l: l.split(",")[0], V())

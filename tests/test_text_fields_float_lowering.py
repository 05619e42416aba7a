"""Float columns of delimited text: `float(l.split(S)[j])` sums, minima and maxima and `mean()` of int() or float()
fields. The matcher (lowering.text_fields_spec), the planner's three modes (plan.FieldScan with MIN_F64 / MAX_F64
table codes, float sums and mean() through record mode) on the numpy stand-in for dampr_text_fields and
dampr_text_fields_records in tests/fields_standin.py, and the results against the REAL reference (Refefer/Dampr),
whose outputs are stored in tests/golden/text_fields_float.json.gz (DAMPR_REFERENCE=<checkout> records them again).
Counts, minima and maxima are compared exactly, sums and means within 4·n·2^-53·Σ|v| (DESIGN §9). The same pipelines
run on the device in tests/test_gpu_text_fields_float.py."""
import ast
import math
import os
import random
import re

import pytest

from fields_standin import make_ctx, python_lines, reference_outputs, run_ours, write_files

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_float.json.gz")
NEEDLE = "device text fields scan+combine"

# ---- inputs -----------------------------------------------------------------------------------------------------
FLOAT_POOL = ["1.5", "-2.25", "0.1", "3", "1e3", "2.5E-3", ".5", "7.", "+4.75", " 8.125", "9.5 ", "1_0.5", "12.0",
              "0.30000000000000004", "123456789.123456789", "1.7976931348623157e308", "5e-324", "1e-5",
              "33.333333333333336", "100", "-0.5"]
KEYS = ["a", "b", "", "k9", "abcdefghij", "x" * 20, "é", "7"]


def datasets():
    rng = random.Random(5)
    rows = []
    for i in range(500):
        v = rng.choice(FLOAT_POOL) if rng.random() < 0.6 else "%.6f" % rng.uniform(-1e4, 1e4)
        rows.append("%s,%d,%s,%s" % (rng.choice(KEYS), rng.randrange(-5, 6), v, rng.choice(["1", "-7", "42", "+3"]))
                    + ("\r\n" if rng.random() < 0.04 else "\n"))
    tsv = "".join("%s\t%d\t%s\n" % (rng.choice("abc"), i, repr(rng.uniform(0, 100))) for i in range(200))
    return {
        "issue": [["prices.csv", "a,x,1.5\nb,y,2.25\na,z,0.1\nb,w,-3e2\nc,v,7\n"]],
        "mixed": [["mixed.csv", "".join(rows)]],
        "tsv": [["t.tsv", tsv]],
        "gz": [["t.tsv.gz", tsv.replace("\n", "\r\n", 30)]],
        "several": [["a.csv", "".join(rows[:200])], ["b.csv", "".join(rows[200:400])],
                    ["c.csv.gz", "".join(rows[400:])]],
    }


C4 = "Dampr.text(P).map(lambda l: l.split(','))"
T3 = "Dampr.text(P).map(lambda l: l.split('\\t'))"
PIPELINES = {
    "issue": [C4 + ".fold_by(lambda r: r[0], value=lambda r: float(r[2]), binop=lambda a, b: a + b)",
              C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[2])).reduce(max)",
              C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[2])).reduce(min)",
              C4 + ".mean(lambda r: r[0], lambda r: float(r[2]))"],
    "mixed": [C4 + ".fold_by(lambda r: r[0], value=lambda r: float(r[2]), binop=lambda a, b: a + b)",
              C4 + ".a_group_by(lambda r: int(r[1]), lambda r: float(r[-2])).reduce(max)",
              C4 + ".mean(lambda r: r[0], lambda r: float(r[2]))",
              C4 + ".mean(lambda r: int(r[1]), lambda r: int(r[3]))",
              "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[2])).sum()"],
    "tsv": [T3 + ".mean(lambda r: r[0], lambda r: float(r[2]))",
            T3 + ".fold_by(lambda r: r[0], value=lambda r: float(r[2]), binop=lambda a, b: a + b)",
            T3 + ".a_group_by(lambda r: r[0], lambda r: float(r[2])).reduce(min)",
            T3 + ".mean(lambda r: r[0], lambda r: int(r[1]))"],
    "several": [C4 + ".fold_by(lambda r: r[0], value=lambda r: float(r[2]), binop=lambda a, b: a + b)",
                C4 + ".mean(lambda r: r[0], lambda r: int(r[3]))"],
}
PIPELINES["gz"] = PIPELINES["tsv"]


# ---- comparison -------------------------------------------------------------------------------------------------
def same_records(got, exp, path=None, key=None, value=None):
    """sorted reprs equal, floats within the sum bound of their key: 4 n 2^-53 Σ|v| (+ one rounding for a mean)"""
    g = [ast.literal_eval(x.replace("nan", "None").replace("inf", "1e999")) for x in got]
    e = [ast.literal_eval(x.replace("nan", "None").replace("inf", "1e999")) for x in exp]
    assert [k for k, _ in g] == [k for k, _ in e], (got, exp)
    bound = {}
    if path is not None:
        for l in python_lines(path):
            k, v = key(l), value(l)
            n, a = bound.get(k, (0, 0.0))
            bound[k] = (n + 1, a + abs(v))
    for (k, gv), (_k, ev) in zip(g, e):
        if type(ev) is float and type(gv) is float and gv != ev:
            n, a = bound[k]
            tol = 4 * n * 2.0 ** -53 * a
            if key is not None and n:
                tol = tol / n + abs(ev) * 2.0 ** -52 if "mean" in repr(value) else tol
            assert math.isfinite(ev) and abs(gv - ev) <= 2 * tol, (k, gv, ev, tol)
        else:
            assert repr(gv) == repr(ev), (k, gv, ev)


def _kv_fns(src):
    """(key(line), value(line), is_mean) restated from a pipeline string, for the sum bound"""
    sep = "\t" if "split('\\t')" in src else ","
    m = re.search(r"(?:mean|fold_by|a_group_by)\((lambda [lr]: .+?), (?:value=)?(lambda [lr]: (?:float|int)\(.*?\]\))",
                  src)
    kf, vf = eval(m.group(1)), eval(m.group(2))
    if "map(lambda l: l.split" in src:
        return (lambda l: kf(l.split(sep))), (lambda l: vf(l.split(sep))), "mean" in src
    return kf, vf, "mean" in src


# ---- the matcher ------------------------------------------------------------------------------------------------
def _spec(key, value, split=None):
    from dampr_b200 import lowering
    return lowering.text_fields_spec(key, value, split)


def _mean_value(value):
    return lambda v: (value(v), 1)   # the keyed value mean() builds (dsl.py)


def test_matcher_accepts_float_values_and_means():
    from dampr_b200.lowering import FIELD_STR, FIELD_INT, FIELD_FLOAT
    sp = lambda l: l.split(",")
    assert _spec(lambda r: r[0], lambda r: float(r[4]), sp) == (",", 0, FIELD_STR, 4, FIELD_FLOAT, False)
    assert _spec(lambda l: int(l.split("|")[1]), lambda l: float(l.split("|")[-1])) == \
        ("|", 1, FIELD_INT, -1, FIELD_FLOAT, False)
    assert _spec(lambda r: r[0], _mean_value(lambda r: float(r[2])), lambda l: l.split("\t")) == \
        ("\t", 0, FIELD_STR, 2, FIELD_FLOAT, True)
    assert _spec(lambda r: r[1], _mean_value(lambda r: int(r[2])), sp) == (",", 1, FIELD_STR, 2, FIELD_INT, True)
    assert _spec(lambda l: l.split(";")[0], _mean_value(lambda l: int(l.split(";")[3]))) == \
        (";", 0, FIELD_STR, 3, FIELD_INT, True)
    # the int and count shapes of the same spec
    assert _spec(lambda r: r[0], lambda r: int(r[1]), sp) == (",", 0, FIELD_STR, 1, FIELD_INT, False)
    assert _spec(lambda r: r[0], lambda r: 1, sp) == (",", 0, FIELD_STR, None, FIELD_INT, False)
    assert _spec(lambda r: r[0], lambda r: float(r[1]), sp) == (",", 0, FIELD_STR, 1, FIELD_FLOAT, False)


def test_matcher_rejects_the_near_misses():
    sp = lambda l: l.split(",")
    for key, value, split in [
        (lambda r: float(r[0]), lambda r: float(r[1]), sp),        # float key
        (lambda r: r[0], lambda r: float(r[1].strip()), sp),
        (lambda r: r[0], lambda r: float(r[1]) * 2, sp),
        (lambda r: r[0], _mean_value(lambda r: 1), sp),            # mean of a constant
        (lambda r: (r[0], r[1]), lambda r: float(r[2]), sp),       # tuple key
        (lambda r: r[0], _mean_value(lambda r: r[2]), sp),         # mean of a str
        (lambda r: r[0], _mean_value(lambda r: float(r)), sp),
        (lambda r: r[0], lambda r: (float(r[2]), 2), sp),          # not mean()'s count
        (lambda r: r[0], lambda r: (float(r[2]), 1.0), sp),
        (lambda r: r[0], _mean_value(lambda r: float(r[2])), lambda l: l.split()),
        (lambda l: l.split(",")[0], lambda l: float(l.split(";")[1]), None),   # two separators
        (lambda r: r[0], _mean_value(lambda r, s=1: float(r[2])), sp),
    ]:
        assert _spec(key, value, split) is None, (key, value, split)


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(datasets()))
def test_float_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = run_ours(src, P, monkeypatch)
        k, v, _mean = _kv_fns(src)
        same_records(got, e, P, k, v)
        assert NEEDLE in hows[0], (name, src, hows)


def test_the_issue_example():
    exp = reference_outputs(datasets()["issue"], PIPELINES["issue"], GOLDEN)
    assert exp[1] == ["('a', 1.5)", "('b', 2.25)", "('c', 7.0)"]


# ---- planner paths on the stand-in ------------------------------------------------------------------------------
def test_modes_are_named_in_the_stats(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1.5,2\nb,2.5,3\na,3.25,4\n"]])
    for src, op in [(C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).sum()", "op=sum_f64"),
                    (C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).reduce(max)", "op=max_f64"),
                    (C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).reduce(min)", "op=min_f64"),
                    (C4 + ".a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()", "op=sum_i64"),
                    (C4 + ".a_group_by(lambda r: r[0], lambda r: int(r[2])).reduce(max)", "op=max_i64"),
                    (C4 + ".a_group_by(lambda r: r[0], lambda r: int(r[2])).reduce(min)", "op=min_i64"),
                    ("Dampr.text(P).count(lambda l: l.split(',')[0])", "op=count"),
                    (C4 + ".mean(lambda r: r[0], lambda r: float(r[1]))", "op=mean_f64"),
                    (C4 + ".mean(lambda r: r[0], lambda r: int(r[2]))", "op=mean_i64")]:
        got, hows, stages = run_ours(src, P, monkeypatch)
        assert NEEDLE in hows[0] and op in stages[0][2], (src, stages)
    assert got == ["('a', 3.0)", "('b', 3.0)"]


def test_host_lines_merge_in_line_order(monkeypatch, tmp_path):
    """values only Python parses (underscores, inf, 20 digits, non-ASCII keys) are folded on the host in line order
    and merged as binop(device value, host value)"""
    lines = ["a,1.5", "b,1_0.5", "a,inf", "é,2", "b,0.1", "a,12345678901234567890", "b, 1e-3", "c,-inf", "c,nan"]
    P = write_files(tmp_path, [["f.csv", "\n".join(lines) + "\n"]])
    key, value = (lambda l: l.split(",")[0]), (lambda l: float(l.split(",")[1]))
    src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[1])).sum()"
    got, hows, stages = run_ours(src, P, monkeypatch)
    exp = {}
    for l in lines:
        exp[key(l)] = exp.get(key(l), 0.0) + value(l) if key(l) in exp else value(l)
    same_records(got, sorted(repr(x) for x in exp.items()), P, key, value)
    assert NEEDLE in hows[0] and "host_lines=6" in stages[0][2], stages
    got, hows, stages = run_ours(C4 + ".mean(lambda r: r[0], lambda r: float(r[1]))", P, monkeypatch)
    assert NEEDLE in hows[0]
    m = dict(ast.literal_eval(x.replace("nan", "None").replace("inf", "1e999")) for x in got)
    assert m["a"] == float("inf") and m["b"] == (0.1 + 1e-3 + 10.5) / 3 and m["é"] == 2.0 and m["c"] is None


def test_negative_zero_and_nan_send_min_max_to_the_host(monkeypatch, tmp_path):
    for text, red in [("a,-0.0\na,0.0\n", "reduce(max)"), ("a,0\na,-0\n", "reduce(min)"), ("a,-1e-999\n", "sum()"),
                      ("a,1\na,nan\n", "reduce(max)"), ("a,1\na,-0e5\n", "reduce(min)")]:
        P = write_files(tmp_path, [["f.csv", text]])
        src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[1])).%s" % red
        got, hows, _st = run_ours(src, P, monkeypatch)
        assert hows[0].startswith("host-map"), (text, hows)
        vals = [float(l.split(",")[1]) for l in text.split()]
        r = vals[0]
        for v in vals[1:]:
            r = {"reduce(max)": max, "reduce(min)": min, "sum()": lambda x, y: x + y}[red](r, v)
        assert got == [repr(("a", r))], (text, got)


def test_record_buffer_regrows_once(monkeypatch, tmp_path):
    """more lines than the first guess (one record per 32 bytes + 4096): RECFULL, one rescan at the exact size"""
    from dampr_b200 import plan
    lines = ["%s,%d.25" % ("abc"[i % 3], i % 17) for i in range(9000)]
    P = write_files(tmp_path, [["f.csv", "\n".join(lines) + "\n"]])
    sizes = []
    orig = plan.FieldScan._records_buffer
    monkeypatch.setattr(plan.FieldScan, "_records_buffer", lambda self, n: (sizes.append(n), orig(self, n))[1])
    got, hows, _st = run_ours(C4 + ".mean(lambda r: r[0], lambda r: float(r[1]))", P, monkeypatch)
    assert NEEDLE in hows[0] and len(sizes) == 2 and sizes[0] < 9000 and sizes[1] == 9000, sizes
    exp = {}
    for l in lines:
        k, v = l.split(",")[0], float(l.split(",")[1])
        s, n = exp.get(k, (0.0, 0))
        exp[k] = (s + v, n + 1)
    assert got == sorted(repr((k, s / float(n))) for k, (s, n) in exp.items())


def test_int_mean_is_bit_equal_and_bounded(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,3\na,4\nb,-7\na,1_0\nb,+2\n"]])
    got, hows, _st = run_ours(C4 + ".mean(lambda r: r[0], lambda r: int(r[1]))", P, monkeypatch)
    assert got == [repr(("a", 17 / 3.0)), repr(("b", -5 / 2.0))] and NEEDLE in hows[0]
    P = write_files(tmp_path, [["g.csv", "a,999999999999999999\n" * 6]])
    got, hows, _st = run_ours(C4 + ".mean(lambda r: r[0], lambda r: int(r[1]))", P, monkeypatch)
    assert got == [repr(("a", 999999999999999999 * 6 / 6.0))] and hows[0].startswith("host-map"), hows


def test_records_that_do_not_fit_go_to_the_host(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "".join("a,%d.5\n" % i for i in range(5000))]])
    got, hows, _st = run_ours(C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).sum()", P, monkeypatch,
                              ctx=make_ctx(free_bytes=5000 * 8))
    assert hows[0].startswith("host-map") and got == [repr(("a", sum(i + 0.5 for i in range(5000))))]
    got, hows, _st = run_ours(C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).reduce(max)", P, monkeypatch,
                              ctx=make_ctx(free_bytes=5000 * 8))
    assert NEEDLE in hows[0] and got == ["('a', 4999.5)"]   # the table modes write no records


def test_sort_scratch_that_does_not_fit_goes_to_the_host(monkeypatch, tmp_path):
    """free memory that holds the record buffer (32 B per line) but not the sort's scratch copy and output on top of
    it: the stage is refused before the sort and runs as a host map, instead of failing in the allocation"""
    n = 5000
    P = write_files(tmp_path, [["f.csv", "".join("a,%d.5\n" % i for i in range(n))]])
    got, hows, _st = run_ours(C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).sum()", P, monkeypatch,
                              ctx=make_ctx(free_bytes=40 * n))
    assert hows[0].startswith("host-map") and got == [repr(("a", sum(i + 0.5 for i in range(n))))]
    got, hows, _st = run_ours(C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).sum()", P, monkeypatch,
                              ctx=make_ctx(free_bytes=48 * n))
    assert NEEDLE in hows[0]


def test_float_sum_is_the_same_bits_for_every_chunking(monkeypatch, tmp_path):
    from dampr_b200 import settings
    rng = random.Random(3)
    text = "".join("%s,%r\n" % (rng.choice("ab"), rng.uniform(-1, 1) * 10 ** rng.randrange(-8, 9))
                   for _ in range(20000))
    P = write_files(tmp_path, [["f.csv", text]])
    outs = set()
    for chunk in (4096, 65536, 1 << 22):
        monkeypatch.setattr(settings, "ingest_chunk_bytes", chunk)
        got, hows, _st = run_ours(C4 + ".a_group_by(lambda r: r[0], lambda r: float(r[1])).sum()", P, monkeypatch)
        assert NEEDLE in hows[0]
        outs.add(tuple(got))
    assert len(outs) == 1


def test_distributed_still_raises(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1.5\n"]])
    from dampr_b200 import dist, plan, Dampr
    from dampr_b200.graph import GMap
    monkeypatch.setattr(dist, "active", lambda: True)
    pm = Dampr.text(P).map(lambda l: l.split(",")).mean(lambda r: r[0], lambda r: float(r[1]))
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    with pytest.raises(plan.NotLowerable):
        plan._lower_map(None, st, [pm.pmer.graph.inputs[st.inputs[0]]], 0)

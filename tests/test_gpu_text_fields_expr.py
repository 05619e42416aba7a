"""Computed keys and values of field folds on the device (the expression builds of csrc/fields.cu): the reference
pipelines of tests/test_text_fields_expr_lowering.py, the kernel's per-line values of generated programs and boundary
operands against CPython bit for bit (record mode), every fold under a str key, an int-expression key and a constant
key, with a separator byte and split(), with and without filters, against plain Python, hot keys over 10^7 lines with
device and host lines of one key, a rerun over a dirty table, and the ABI's refusals. Each case asserts which path
the stage took."""
import operator
import random

import numpy as np
import pytest

from fields_expr_standin import expr_line
from fields_standin import python_lines, reference_outputs, write_files
from test_text_fields_expr_lowering import GOLDEN, NEEDLE, PIPELINES, WS, datasets, random_lambda, _same
from test_text_fields_where_lowering import same_up_to_rounding

pytestmark = pytest.mark.gpu


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "ingest_chunk_bytes", settings.ingest_chunk_bytes)
    yield settings
    plan.release_buffers()


def run(src, P):
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P}).run())
    return got, runner_mod.LAST_STATS.stages[0]


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, (_s, how, detail) = run(src, P)
        same_up_to_rounding(got, exp)
        assert NEEDLE in how, (src, how)
        assert (" value=expr" in detail or " key=" in detail) == (src != WS[2]), (src, detail)


# ---- per-line values against CPython ---------------------------------------------------------------------------
def boundary_rows(rng, n):
    ints = ["0", "1", "-1", "7", "-7", str(1 << 53), str((1 << 53) + 1), str(-(1 << 53) - 1), "999999999999999999",
            "-999999999999999999", "3037000499", "-3037000499", "3037000500", "4611686018427387904"[:18], "x"]
    floats = ["0.0", "-0.0", "1e308", "-1e308", "5e-324", "-5e-324", "2.2250738585072014e-308", "2.5", "1e-300",
              "9007199254740993", "0.1", "x"]
    out = []
    for _ in range(n):
        f = [rng.choice(ints), rng.choice(ints), rng.choice(floats), rng.choice(["", "ab", "abcdefghij"])]
        out.append(",".join(f[:rng.choice([4] * 9 + [3])]).encode())
    return out


def test_per_line_values_bit_for_bit(ctx):
    """record mode's per-line values of generated programs over 10^6 lines of boundary operands: every line the
    device takes holds CPython's value to the bit (NaN as NaN), and the device takes exactly the lines the evaluator
    of tests/fields_expr_standin.py takes; zero divisors and IndexErrors are host lines"""
    from dampr_b200 import device as dev, lowering
    rng = random.Random(77)
    rows = boundary_rows(rng, 1000000)
    data = b"\n".join(rows) + b"\n"
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    srcs, done = ["int(r[0]) * int(r[1])", "float(r[2]) / int(r[1])", "int(r[0]) // int(r[1]) - int(r[1]) % 7",
                  "int(float(r[2])) + len(r[3])", "abs(int(r[0])) / int(r[1])", "-float(r[2]) * 3 + len(r)"], 0
    while len(srcs) < 12:
        srcs.append(random_lambda(rng))
    try:
        for src in srcs:
            fn = eval("lambda r: " + src)
            got = lowering.text_fields_expr(lambda r: r[0], fn, lambda l: l.split(","))
            if got is None or got[6] is None:
                continue
            _kp, vp, ci, cf, loads = got[6]
            expr = (None, (dev.EXPR_INT if vp[0] == "i" else dev.EXPR_F64, tuple(vp[1])), tuple(ci), tuple(cf),
                    tuple(loads))
            op = dev.OP_SUM_I64 if vp[0] == "i" else dev.OP_SUM_F64
            spec = (ord(","), 0, dev.FIELD_KEY_STR, 0, op)
            tab = ctx.table(16)
            kv = ctx.kv(len(rows) + 16)
            tab.fields_expr_records(tb, 0, len(data), spec, expr, kv)
            st = tab.fields_stats()
            kv.set_size(st["records"])
            recs = kv.records()
            kv.free()
            tab.free()
            assert st["records"] == len(rows) and not st["flags"] & (dev.TF_RECFULL | dev.TF_TABLEFULL), st
            codes, bits = recs[:, 0], recs[:, 1]
            vals = bits.view(np.int64).tolist() if vp[0] == "i" else bits.view(np.float64).tolist()
            sample = range(len(rows)) if len(rows) <= 200000 else sorted(rng.sample(range(len(rows)), 200000))
            for i in sample:
                want = expr_line(rows[i], rows[i].split(b","), expr, spec)
                assert (codes[i] == 0) == (want is None), (src, rows[i], want)
                if want is not None:
                    assert _same(vals[i], want[1]), (src, rows[i], vals[i], want[1])
                    assert _same(vals[i], fn(rows[i].decode().split(","))), (src, rows[i])
            done += 1
    finally:
        tb.free()
    assert done >= 8


# ---- every fold against Python ----------------------------------------------------------------------------------
def seeded_rows(seed, ws, n=200000):
    rng = random.Random(seed)
    sep = " \t " if ws else ","
    rows = []
    for _ in range(n):
        f = [rng.choice(["a", "bb", "k" * 12] + ["h%d" % i for i in range(50)]), str(rng.randrange(-500, 5000)),
             str(rng.randrange(1, 300)), "%.3f" % (rng.randrange(-64, 64) / 8.0)]
        if rng.random() < 0.01:
            f[0] += "é"   # a host line
        rows.append(sep.join(f))
    return "".join(r + "\n" for r in rows)


KEYS = {"str": "lambda r: r[0]", "expr": "lambda r: int(r[1]) // 100", "const": "lambda r: 1"}
FOLDS = {
    "count": (".count(%s)", None),
    "sum_i64": (".a_group_by(%s, lambda r: int(r[1]) * int(r[2])).sum()", lambda r: int(r[1]) * int(r[2])),
    "min_i64": (".a_group_by(%s, lambda r: int(r[1]) - int(r[2])).reduce(min)", lambda r: int(r[1]) - int(r[2])),
    "max_i64": (".a_group_by(%s, lambda r: int(r[1]) %% 17).reduce(max)", lambda r: int(r[1]) % 17),
    "sum_f64": (".a_group_by(%s, lambda r: float(r[3]) * 2 + 1).sum()", lambda r: float(r[3]) * 2 + 1),
    "min_f64": (".a_group_by(%s, lambda r: float(r[3]) / int(r[2])).reduce(min)", lambda r: float(r[3]) / int(r[2])),
    "max_f64": (".a_group_by(%s, lambda r: float(r[3]) - 100).reduce(max)", lambda r: float(r[3]) - 100),
    "mean": (".mean(%s, lambda r: int(r[1]) / int(r[2]))", lambda r: int(r[1]) / int(r[2])),
}


@pytest.mark.parametrize("fold", sorted(FOLDS))
@pytest.mark.parametrize("key", sorted(KEYS))
@pytest.mark.parametrize("split", ["comma", "ws"])
@pytest.mark.parametrize("filtered", [False, True])
def test_every_fold_against_python(fold, key, split, filtered, engine, tmp_path):
    P = write_files(tmp_path, [["f.txt", seeded_rows(sum(map(ord, fold + key + split)), split == "ws")]])
    sp = "lambda l: l.split()" if split == "ws" else "lambda l: l.split(',')"
    src = "Dampr.text(P).map(%s)" % sp + (".filter(lambda r: r[0] != 'a')" if filtered else "") + \
        FOLDS[fold][0] % KEYS[key]
    got, (_s, how, detail) = run(src, P)
    assert NEEDLE in how, (src, how)
    kf, vf = eval(KEYS[key]), FOLDS[fold][1]
    split_fn = (lambda l: l.split()) if split == "ws" else (lambda l: l.split(","))
    acc = {}
    for l in python_lines(P):
        r = split_fn(l)
        if filtered and r[0] == "a":
            continue
        k = kf(r)
        if fold == "count":
            acc[k] = acc.get(k, 0) + 1
        elif fold == "mean":
            s, c = acc.get(k, (0.0, 0))
            acc[k] = (s + vf(r), c + 1)
        else:
            v = vf(r)
            acc[k] = v if k not in acc else {"sum": operator.add, "min": min, "max": max}[fold[:3]](acc[k], v)
    if fold == "mean":
        exp = sorted(repr((k, s / c)) for k, (s, c) in acc.items())
    else:
        exp = sorted(repr(x) for x in acc.items())
    same_up_to_rounding(got, exp)
    assert ("key=const" in detail) == (key == "const") and ("key=expr" in detail) == (key == "expr"), detail
    assert ("value=expr" in detail) == (fold != "count"), detail


# ---- hot keys -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,nkeys", [("lambda r: 1", 1), ("lambda r: int(r[0]) % 16", 16)])
def test_hot_keys(key, nkeys, engine, tmp_path):
    """10^7 lines into one or 16 keys, ingested in 64 KB chunks, one line in 1000 of every key a host line (a
    non-ASCII field): the warp-aggregated inserts and the host lines merge into Python's sums"""
    engine.ingest_chunk_bytes = 1 << 16
    n = 10 ** 7
    i = np.arange(n, dtype=np.int64)
    nums = (i * 7919) % 100003
    text = "".join("%d,%d,%s\n" % (a, b, "é" if a % 1000 == 999 else "x") for a, b in zip(i.tolist(), nums.tolist()))
    P = write_files(tmp_path, [["f.csv", text]])
    got, (_s, how, detail) = run("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(%s, lambda r: int(r[1]) * 3)"
                                 ".sum()" % key, P)
    assert NEEDLE in how and "host_lines=%d" % (n // 1000) in detail and "groups=%d" % nkeys in detail, detail
    ks = np.ones(n, dtype=np.int64) if nkeys == 1 else i % 16
    exp = {int(k): int(nums[ks == k].sum()) * 3 for k in np.unique(ks).tolist()}
    assert got == sorted(repr(x) for x in exp.items()), got[:3]


# ---- reuse and the ABI ----------------------------------------------------------------------------------------
def test_rerun_over_a_dirty_table_and_a_used_record_buffer(ctx):
    """one record buffer for every scan: it still holds the records of another program's scan when the next one writes
    it; the table still holds a table-mode fold of another op before it is cleared for the next scan (the ABI's
    contract). The two record scans of one program give the same bytes."""
    from dampr_b200 import device as dev, lowering
    rows = ["%d,%d,%s" % (k % 97, k * 31 % 1000, "%.2f" % (k / 8)) for k in range(200000)]
    data = ("\n".join(rows) + "\n").encode()
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))

    def program(key, value):
        kp, vp, ci, cf, loads = lowering.text_fields_expr(key, value, lambda l: l.split(","))[6]
        return (None if kp is None else (dev.EXPR_INT, tuple(kp[1])),
                (dev.EXPR_INT if vp[0] == "i" else dev.EXPR_F64, tuple(vp[1])), tuple(ci), tuple(cf), tuple(loads))
    target = program(lambda r: int(r[0]) // 3, lambda r: float(r[2]) * int(r[1]))
    other = program(lambda r: int(r[1]) % 7, lambda r: float(r[2]) - int(r[0]))
    spec = (ord(","), 0, dev.FIELD_KEY_INT, 0, dev.OP_SUM_F64)
    outs = []
    tab = ctx.table(12)
    kv = ctx.kv(len(rows) + 16)
    try:
        tab.fields_expr_records(tb, 0, len(data), spec, other, kv)   # the buffer now holds other records
        for _ in range(2):
            tab.clear()
            tab.fields_expr(tb, 0, len(data), (ord(","), 0, dev.FIELD_KEY_INT, 0, dev.OP_MAX_F64), other)
            tab.clear()
            tab.fields_expr_records(tb, 0, len(data), spec, target, kv)
            st = tab.fields_stats()
            kv.set_size(st["records"])
            codes, acc, _r = tab.fetch()
            order = np.argsort(codes)
            outs.append((kv.records().tobytes(), codes[order].tobytes(), acc[order].tobytes(), st))
            recs = kv.records()
    finally:
        kv.free()
        tab.free()
        tb.free()
    assert outs[0] == outs[1] and outs[0][3]["lines"] == len(rows)
    want = [((int(r.split(",")[0]) // 3) ^ (1 << 63), float(r.split(",")[2]) * int(r.split(",")[1])) for r in rows]
    assert recs[:, 0].tolist() == [k for k, _v in want]
    assert recs[:, 1].view(np.float64).tolist() == [v for _k, v in want]


def test_reuse_through_the_planner(engine, tmp_path):
    """stages of other ops and key kinds run in between on the planner's cached table and pooled record buffers: the
    same stage gives the same records each time, and Python's"""
    P = write_files(tmp_path, [["f.txt", seeded_rows(91, False)]])
    C = "Dampr.text(P).map(lambda l: l.split(','))"
    srcs = [C + ".mean(lambda r: r[0], lambda r: float(r[3]) * 3)",
            C + ".a_group_by(lambda r: int(r[1]) // 100, lambda r: float(r[3]) / int(r[2])).sum()",
            C + ".a_group_by(lambda r: 1, lambda r: int(r[1]) * int(r[2])).reduce(max)"]
    outs = []
    for src in srcs + srcs[1:] + srcs[:1]:
        got, (_s, how, _d) = run(src, P)
        assert NEEDLE in how, (src, how)
        outs.append(got)
    assert outs[1] == outs[3] and outs[2] == outs[4] and outs[0] == outs[5]
    rows = [l.split(",") for l in python_lines(P)]
    exp = {}
    for r in rows:
        k = int(r[1]) // 100
        exp[k] = exp[k] + float(r[3]) / int(r[2]) if k in exp else float(r[3]) / int(r[2])
    same_up_to_rounding(outs[1], sorted(repr(x) for x in exp.items()))
    assert outs[2] == [repr((1, max(int(r[1]) * int(r[2]) for r in rows)))]


def test_malformed_programs_are_refused(ctx):
    from dampr_b200 import device as dev
    data = b"1,2\n"
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    spec = (ord(","), 0, dev.FIELD_KEY_STR, 0, dev.OP_SUM_I64)
    LOAD, CI, IADD, FADD, X, LOG, NF = 15, 1, 4, 7, 0, 12, 16
    ok = (None, (dev.EXPR_INT, (LOAD, CI, IADD)), (3,), (), ((0, dev.LOAD_INT),))
    try:
        tab.fields_expr(tb, 0, len(data), spec, ok)
        bad = [
            (None, (dev.EXPR_INT, (IADD,)), (), (), ()),                                  # stack underflow
            (None, (dev.EXPR_INT, (CI, CI)), (1,), (), ()),                               # final depth 2
            (None, (dev.EXPR_INT, (99,)), (), (), ()),                                    # unknown opcode
            (None, (dev.EXPR_INT, (X,)), (), (), ()),                                     # the host evaluator's
            (None, (dev.EXPR_INT, (LOAD | 1 << 8,)), (), (), ((0, dev.LOAD_INT),)),      # slot out of range
            (None, (dev.EXPR_INT, (CI | 16 << 8,)), (), (), ()),                          # constant out of range
            (None, (dev.EXPR_F64, (NF,)), (), (), ()),                                    # result type
            (None, (dev.EXPR_INT, (CI, CI, FADD)), (1,), (), ()),                         # operand type
            (None, (dev.EXPR_INT, (CI,) * 9 + (IADD,) * 8), (1,), (), ()),                # depth 9
            (None, (dev.EXPR_INT, (CI,) + (CI, IADD) * 16), (1,), (), ()),                # 33 operations
            (None, None, (), (), ()),                                                     # no program
            (None, (dev.EXPR_INT, (LOAD,)), (), (), ((0, 7),)),                           # slot kind
        ]
        for x in bad:
            with pytest.raises(dev.DeviceError):
                tab.fields_expr(tb, 0, len(data), spec, x)
        for s in [(dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 0, dev.OP_SUM_I64),
                  (ord(","), 0, dev.FIELD_KEY_STR, 0, dev.OP_MIN_F64)]:   # JSON; an int program under a float op
            with pytest.raises(dev.DeviceError):
                tab.fields_expr(tb, 0, len(data), s, ok)
    finally:
        tab.free()
        tb.free()

"""Float keys through the lowered kv and frame stages, against the REAL reference (Refefer/Dampr) whose outputs are
stored in tests/golden/float_keys.json.gz (the ReferenceReplay pattern of test_differential_reference.py).

Python compares keys by value: -0.0 == 0.0 is one key (a sort keeps such rows in input order, a group reports the
key of its first record), every NaN is a key of its own, and negative floats sort below positive ones. The device
orders 64-bit patterns, so every lowering that sorts or groups a float column must normalise it (col + 0.0), sort
it under KEY_F64 and leave a column that holds a NaN to the host. Each case also asserts which path the stage took.
The same pipelines run on the real device in tests/test_gpu_key_orders.py."""
import gzip
import hashlib
import json
import math
import os
import subprocess as _subprocess
import sys

import numpy as np
import pytest

REF = os.environ.get("DAMPR_REFERENCE", "")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "float_keys.json.gz")

DRIVER = r"""
import sys, json
sys.path.insert(0, sys.argv[1])
from dampr import Dampr
recs = [tuple(r) for r in json.loads(sys.argv[2])]; recs2 = [tuple(r) for r in json.loads(sys.argv[4])]
print(json.dumps([[repr(x) for x in eval(src).run()] for src in json.loads(sys.argv[3])]))
"""


def reference_outputs(recs, recs2, srcs):
    """The reference's output records (reprs, in output order) of every pipeline in srcs: recorded in GOLDEN under a
    digest of the driver and its arguments; with DAMPR_REFERENCE set the reference runs and the record is renewed."""
    args = [DRIVER, json.dumps(recs), json.dumps(srcs), json.dumps(recs2)]
    key = hashlib.sha256("\0".join(args).encode()).hexdigest()[:20]
    runs = {}
    if os.path.exists(GOLDEN):
        with gzip.open(GOLDEN, "rb") as f:
            runs = json.loads(f.read())
    if REF:
        env = dict(os.environ)
        env.pop("PYTHONPATH", None)
        p = _subprocess.run([sys.executable, "-c", DRIVER, REF] + args[1:], capture_output=True, text=True, env=env,
                            cwd="/tmp", timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        runs[key] = p.stdout.strip().split("\n")[-1]
        with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
            f.write(json.dumps(runs, sort_keys=True).encode())
    assert key in runs, "no recorded reference output for these inputs: record with DAMPR_REFERENCE=<checkout>"
    return json.loads(runs[key])


# ---- inputs -----------------------------------------------------------------------------------------------------
DBL_MIN_SUB, DBL_MAX_SUB, DBL_MAX = 5e-324, 2.225073858507201e-308, 1.7976931348623157e308
POOL = [0.0, -0.0, -2.5, -1.0, -0.75, 0.5, 1.5, 3.25, 7.0, -7.0, math.inf, -math.inf, DBL_MIN_SUB, -DBL_MIN_SUB,
        DBL_MAX_SUB, -DBL_MAX_SUB, DBL_MAX, -DBL_MAX, 1e-9, -1e-9]


def datasets():
    """name -> (int keys, float values) lists. 'issue' is the smallest input that shows every float-key lowering bug;
    'mixed' has both zeros (0.0 first) and the extremes; 'negzero_first' starts with -0.0; 'nan' holds NaNs;
    'no_negzero' has neither NaN nor -0.0 (the min / max folds may lower there)."""
    rng = np.random.default_rng(2026)
    n = 600
    pool = np.array(POOL)
    mixed = pool[rng.integers(0, len(pool), size=n)]
    mixed[0] = 0.0
    k = rng.integers(-20, 20, size=n).tolist()
    nan = mixed.copy()
    nan[[5, 77, 300, 599]] = np.nan
    no_negzero = np.where(np.signbit(mixed) & (mixed == 0), 0.0, mixed)
    return {
        "issue": (list(range(8)), [0.0, -0.0, 1.5, -0.0, 0.0, -1.0, 0.0, -2.5]),
        "mixed": (k, mixed.tolist()),
        "negzero_first": ([99] + k, [-0.0] + mixed.tolist()),
        "nan": (k, nan.tolist()),
        "no_negzero": (k, no_negzero.tolist()),
    }


def right_side():
    """the right input of the joins: float keys that partly overlap the left's, both zeros (0.0 first)"""
    rng = np.random.default_rng(7)
    v = np.array([0.0, -0.0, -1.0, 3.25, 42.0, -math.inf, DBL_MIN_SUB])[rng.integers(0, 7, size=80)]
    v[0] = 0.0
    return rng.integers(0, 9, size=80).tolist(), v.tolist()


# The reference reads its input as one partition: over several, its threads combine the partial groups in an order
# that varies from run to run, and with it which of 0.0 / -0.0 a merged group reports.
# (pipeline over {A} (and {B}), order, stage, path). The records are compared with the reference's as a multiset;
# order, for a sort, is Python's own stable sort of the input `rows`, which the output must equal in order (the
# reference's threads leave tied records in an order that varies from run to run). stage: the index of the float-keyed stage among the
# stage strings; in a chained sort the second sort gets the rows of the first as a frame (the frame lowering).
# path: a needle of that stage's string when it is lowered.
PIPELINES = [
    ("{A}.sort_by(lambda x: x[1])", "sorted(rows, key=lambda x: x[1])", 0, "device kv partition+sort of whole records"),
    ("{A}.sort_by(lambda x: -x[1])", "sorted(rows, key=lambda x: -x[1])", 0, "device kv partition+sort of whole records"),
    ("{A}.sort_by(lambda x: x[0]).sort_by(lambda x: -x[1])",
     "sorted(sorted(rows, key=lambda x: x[0]), key=lambda x: -x[1])", 1, "device sort of frame rows"),
    ("{A}.sort_by(lambda x: x[0]).sort_by(lambda x: x[1])",
     "sorted(sorted(rows, key=lambda x: x[0]), key=lambda x: x[1])", 1, "device sort of frame rows"),
    ("{A}.a_group_by(lambda x: x[1], lambda x: x[0]).sum()", False, 0, "device kv partition+sort+segmented-reduce"),
    ("{A}.count(lambda x: x[1])", False, 0, "device kv partition+sort+segmented-reduce"),
    ("{A}.group_by(lambda x: x[1], lambda x: x[0]).reduce(lambda k, it: sum(it))", False, 0, "deferred until read"),
    ("{A}.group_by(lambda x: x[1], lambda x: x[0]).reduce(lambda k, it: max(it))", False, 0, "deferred until read"),
    ("{A}.group_by(lambda x: x[1]).reduce(lambda k, it: len(list(it)))", False, 0,
     "device kv partition+sort of whole records"),
    ("{A}.group_by(lambda x: x[1], lambda x: x[0]).join({B}.group_by(lambda x: x[1], lambda x: x[0]))"
     ".reduce(lambda l, r: (sum(l), sum(r)))", False, 0, "deferred until read"),
    ("{A}.group_by(lambda x: x[1], lambda x: x[0]).join({B}.group_by(lambda x: x[1], lambda x: x[0]))"
     ".left_reduce(lambda l, r: (sum(l), sorted(r)))", False, 0, "deferred until read"),
    ("{A}.fold_by(lambda x: x[0], min, lambda x: x[1])", False, 0, "frame keyed fold"),
    ("{A}.fold_by(lambda x: x[0], max, lambda x: x[1])", False, 0, "frame keyed fold"),
    ("{A}.map(lambda x: (x[1], x[0])).count(lambda x: x[0])", False, 0, None),   # a frame's keyed fold on float keys
]


def lowers(src, needle, name):
    """whether the planner must lower the float-keyed stage of pipeline `src` on dataset `name`"""
    if needle is None:
        return False
    if "fold_by" in src:
        return name == "no_negzero"   # min / max over NaN or -0.0: Python's answer depends on the argument order
    if name == "nan":
        return False                  # a NaN key: no device sort or grouping of bit patterns gives Python's answer
    # grouped records whose 0.0 group would have to report its first key, -0.0
    return not (name == "negzero_first" and ".group_by(lambda x: x[1], lambda x: x[0])" in src)


def run_ours(src, ns, make_ctx, monkeypatch):
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    if make_ctx is not None:
        monkeypatch.setattr(runner_mod, "_CTX", {settings.device: make_ctx()})
        monkeypatch.setattr(plan, "_BUFFERS", {})
    env = dict(ns, Dampr=Dampr, ArrayKVInput=ArrayKVInput)
    got = [repr(x) for x in eval(src, env).run()]
    return got, [h for _s, h, _d in runner_mod.LAST_STATS.stages]


def check_all(monkeypatch, make_ctx):
    """every pipeline on every dataset: the same records as the reference (in order for sorts), the expected path"""
    K2, V2 = right_side()
    ref_b = "Dampr.memory(recs2, partitions=1)"
    for name, (K, V) in sorted(datasets().items()):
        # NaN keys: which NaN records meet in a group or a run depends on the order in which the reference's threads
        # compare them, so only the path is checked there
        nan = name == "nan"
        ref = [None] * len(PIPELINES) if nan else reference_outputs(
            list(zip(K, V)), list(zip(K2, V2)), [p.format(A="Dampr.memory(recs, partitions=1)", B=ref_b) for p, _o, _i, _w in PIPELINES])
        ns = {"K": np.array(K, dtype=np.int64), "V": np.array(V, dtype=np.float64),
              "K2": np.array(K2, dtype=np.int64), "V2": np.array(V2, dtype=np.float64)}
        for (p, ordered, i, needle), exp in zip(PIPELINES, ref):
            src = p.format(A="Dampr.read_input(ArrayKVInput(K, V))", B="Dampr.read_input(ArrayKVInput(K2, V2))")
            got, hows = run_ours(src, ns, make_ctx, monkeypatch)
            if not nan:
                assert sorted(got) == sorted(exp), (name, src)
            if ordered and not nan:
                assert got == [repr(x) for x in eval(ordered, {"rows": list(zip(K, V))})], (name, src)
            if lowers(p, needle, name):
                assert needle in hows[i], (name, src, hows)
            else:
                assert hows[i].startswith("host-map"), (name, src, hows)
        # the float column as the first field
        for p, ordered in (("{A}.sort_by(lambda x: x[0])", "sorted(rows, key=lambda x: x[0])"),
                           ("{A}.sort_by(lambda x: -x[0])", "sorted(rows, key=lambda x: -x[0])"),
                           ("{A}.a_group_by(lambda x: x[0], lambda x: x[1]).sum()", None)):
            got, hows = run_ours(p.format(A="Dampr.read_input(ArrayKVInput(V, K))"), ns, make_ctx, monkeypatch)
            assert hows[0].startswith("host-map") == nan, (name, p, hows)
            if nan:
                continue
            exp = reference_outputs([[v, k] for k, v in zip(K, V)], [], [p.format(A="Dampr.memory(recs, partitions=1)")])[0]
            assert sorted(got) == sorted(exp), (name, p)
            if ordered:
                assert got == [repr(x) for x in eval(ordered, {"rows": list(zip(V, K))})], (name, p)


def test_float_keys_agree_with_the_reference(monkeypatch):
    from fake_device import FakeCtx
    check_all(monkeypatch, FakeCtx)


def test_signed_zeros_in_the_issue_example(monkeypatch):
    """sort_by on a float field orders by value and keeps tied zeros in input order; a group of 0.0 and -0.0 is one
    group that reports its first key; the records keep their -0.0 fields"""
    from fake_device import FakeCtx
    K = np.arange(8, dtype=np.int64)
    V = np.array([0.0, -0.0, 1.5, -0.0, 0.0, -1.0, 0.0, -2.5])
    ns = {"K": K, "V": V}
    got, _ = run_ours("Dampr.read_input(ArrayKVInput(K, V)).sort_by(lambda x: x[1])", ns, FakeCtx, monkeypatch)
    assert got == ["(7, -2.5)", "(5, -1.0)", "(0, 0.0)", "(1, -0.0)", "(3, -0.0)", "(4, 0.0)", "(6, 0.0)", "(2, 1.5)"]
    got, _ = run_ours("Dampr.read_input(ArrayKVInput(K, V)).sort_by(lambda x: -x[1])", ns, FakeCtx, monkeypatch)
    assert got == ["(2, 1.5)", "(0, 0.0)", "(1, -0.0)", "(3, -0.0)", "(4, 0.0)", "(6, 0.0)", "(5, -1.0)", "(7, -2.5)"]
    got, _ = run_ours("Dampr.read_input(ArrayKVInput(K, V)).a_group_by(lambda x: x[1], lambda x: x[0]).sum()", ns,
                      FakeCtx, monkeypatch)
    assert sorted(got) == ["(-1.0, 5)", "(-2.5, 7)", "(0.0, 14)", "(1.5, 2)"]
    ns["V"] = np.concatenate(([-0.0], V))
    ns["K"] = np.arange(9, dtype=np.int64)
    got, hows = run_ours("Dampr.read_input(ArrayKVInput(K, V)).count(lambda x: x[1])", ns, FakeCtx, monkeypatch)
    assert sorted(got) == ["(-0.0, 6)", "(-1.0, 1)", "(-2.5, 1)", "(1.5, 1)"]
    assert any("segmented-reduce" in h for h in hows), hows


@pytest.mark.parametrize("kind", ["min", "max"])
def test_float_min_max_fold_declines_on_nan_and_negative_zero(kind):
    """_fold_column groups on the device, where the records of a group meet in an order that is not the input's:
    with NaN or -0.0 among the values Python's min / max depend on that order, so the fold is left to the host"""
    from fake_device import FakeCtx
    from dampr_b200 import lowering, plan

    class R(object):
        ctx = FakeCtx()
    codes = np.array([1, 1, 2], dtype=np.uint64)
    k = lowering.MIN if kind == "min" else lowering.MAX
    for bad in (np.nan, -0.0):
        with pytest.raises(plan.NotLowerable):
            plan._fold_column(R(), codes, 1, np.array([1.0, bad, 2.0]), k)
    rk, rv, _how = plan._fold_column(R(), codes, 1, np.array([1.0, 0.0, -math.inf]), k)
    got = dict(zip(rk.tolist(), rv.tolist()))
    assert got == ({1: 0.0, 2: -math.inf} if kind == "min" else {1: 1.0, 2: -math.inf})

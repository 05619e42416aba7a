"""GPU: float and signed keys through the kv kernels — sort, sort + fold, fold of a sorted run, k-way merge, join
ranges, the spill path — against plain references: numpy's stable argsort of the keys' order domain
(spill._order_domain / mix64), Python left folds over Python ints and floats (math.fsum with the bound
4 n 2^-53 sum|v| for OP_SUM_F64), and the numpy stand-in device (tests/fake_device.py) bit for bit.

Values carry their input position where the order matters, so every check of an order is also a check of stability.
The float keys include +-0.0, +-inf, the smallest and largest subnormals, +-DBL_MAX, quiet NaNs of both signs with
different payloads, exact duplicates, a cluster with a long common bit prefix and a spread over the whole
transformed range; the signed keys include INT64_MIN, INT64_MIN + 1, -1, 0, INT64_MAX and dense runs around zero."""
import functools
import math

import numpy as np
import pytest

from dampr_b200 import device as dev
from fake_device import FakeCtx, FakeKV

pytestmark = pytest.mark.gpu

LEAF = 4096          # records one CTA leaf sorts (csrc/leaf.cuh L_CAP)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
F64_OPS = (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
ALL_OPS = (dev.OP_SUM_I64, dev.OP_SUM_F64, dev.OP_COUNT, dev.OP_MIN_I64, dev.OP_MAX_I64, dev.OP_MIN_F64,
           dev.OP_MAX_F64, dev.OP_FIRST, dev.OP_LAST)


def nan_with(sign, payload):
    return np.array([(sign << 63) | 0x7FF8000000000000 | payload], dtype=np.uint64).view(np.float64)[0]


F64_SPECIAL = np.array([0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.225073858507201e-308, -2.225073858507201e-308,
                        1.7976931348623157e308, -1.7976931348623157e308, nan_with(0, 0), nan_with(1, 0),
                        nan_with(0, 12345), nan_with(1, 0x7FFFF), 1.0, -1.0])
I64_SPECIAL = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX, I64_MAX - 1], dtype=np.int64)


def f64_keys(rng, n):
    """the specials, many exact duplicates, normal values of both signs, a narrow cluster in [1, 1 + 1e-9] and random
    bit patterns over the whole 64-bit range"""
    if n == 0:
        return np.zeros(0)
    pick = rng.integers(0, 5, size=n)
    out = np.empty(n)
    out[pick == 0] = F64_SPECIAL[rng.integers(0, len(F64_SPECIAL), size=int((pick == 0).sum()))]
    dup = rng.standard_normal(64) * 1e3
    out[pick == 1] = dup[rng.integers(0, 64, size=int((pick == 1).sum()))]
    out[pick == 2] = rng.standard_normal(int((pick == 2).sum())) * 10.0 ** rng.integers(-300, 300, size=int((pick == 2).sum()))
    out[pick == 3] = 1.0 + rng.random(int((pick == 3).sum())) * 1e-9
    out[pick == 4] = rng.integers(0, 1 << 64, size=int((pick == 4).sum()), dtype=np.uint64).view(np.float64)
    out[:min(n, len(F64_SPECIAL))] = F64_SPECIAL[:min(n, len(F64_SPECIAL))]
    return out


def i64_keys(rng, n):
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    pick = rng.integers(0, 3, size=n)
    out = rng.integers(I64_MIN, I64_MAX, size=n, dtype=np.int64, endpoint=True)
    out[pick == 0] = I64_SPECIAL[rng.integers(0, len(I64_SPECIAL), size=int((pick == 0).sum()))]
    out[pick == 1] = rng.integers(-300, 300, size=int((pick == 1).sum()))
    out[:min(n, len(I64_SPECIAL))] = I64_SPECIAL[:min(n, len(I64_SPECIAL))]
    return out


def keys_for(xf, rng, n):
    if xf == dev.KEY_F64:
        return f64_keys(rng, n).view(np.uint64)
    if xf == dev.KEY_I64:
        return i64_keys(rng, n).view(np.uint64)
    return rng.integers(0, 1 << 64, size=n, dtype=np.uint64)


def stable_order(keys, xf):
    return np.argsort(FakeKV._order(keys, xf), kind="stable")


def check_sort(ctx, keys, xf):
    vals = np.arange(len(keys), dtype=np.uint64)            # the input position
    kv = ctx.kv_from_columns(keys, vals)
    kv.sort(xf)
    k2, v2 = kv.columns()
    kv.free()
    o = stable_order(keys, xf)
    assert np.array_equal(k2, keys[o])
    assert np.array_equal(v2, o.astype(np.uint64))


# ---- dampr_kv_sort -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, LEAF, LEAF + 1, 27_000, 1_000_000])
@pytest.mark.parametrize("xf", [dev.KEY_F64, dev.KEY_I64])
def test_sort_orders_float_and_signed_keys(ctx, n, xf):
    check_sort(ctx, keys_for(xf, np.random.default_rng(n + 10 * xf), n), xf)


@pytest.mark.parametrize("xf", [dev.KEY_F64, dev.KEY_I64])
def test_sort_two_partition_levels(ctx, xf):
    check_sort(ctx, keys_for(xf, np.random.default_rng(61 + xf), 6_000_000), xf)


@pytest.mark.parametrize("n", [LEAF, 27_000, 1_000_000])
def test_sort_narrow_cluster_next_to_the_whole_range(ctx, n):
    """keys in [1, 1 + 1e-9] share their top ~34 bits: the digits minmax_kernel picks must still split them; then the
    same cluster next to keys spread over the whole transformed range, and the cluster alone"""
    rng = np.random.default_rng(n)
    narrow = 1.0 + rng.random(n) * 1e-9
    wide = rng.integers(0, 1 << 64, size=n // 8, dtype=np.uint64).view(np.float64)
    wide = wide[~np.isnan(wide)]
    check_sort(ctx, narrow.view(np.uint64), dev.KEY_F64)
    both = np.concatenate((narrow, wide, [np.inf, -np.inf, 0.0, -0.0]))
    rng.shuffle(both)
    check_sort(ctx, both.view(np.uint64), dev.KEY_F64)
    ik = np.concatenate((rng.integers(-50, 50, size=n), [I64_MIN, I64_MAX]))
    check_sort(ctx, ik.view(np.uint64), dev.KEY_I64)


# ---- folds ---------------------------------------------------------------------------------------------------
def fold_values(op, rng, n):
    """values for each op: NaN- and -0.0-free floats for MIN / MAX_F64 (the planner sends those to the host), finite
    floats for SUM_F64, int64 extremes for MIN / MAX_I64, sums that stay in 64 bits. SUM_F64 also receives -0.0, +-inf
    and NaN from the planner; those, and the bit-exact checks, are in test_gpu_float_sums.py"""
    if op in (dev.OP_MIN_F64, dev.OP_MAX_F64):
        pool = np.array([0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.225073858507201e-308, -2.5, 1.7976931348623157e308,
                         -1.7976931348623157e308, 3.0])
        v = np.where(rng.random(n) < 0.5, pool[rng.integers(0, len(pool), size=n)], rng.standard_normal(n) * 1e6)
        return v.view(np.uint64)
    if op == dev.OP_SUM_F64:
        return np.where(rng.random(n) < 0.1, 5e-324, rng.standard_normal(n) * 1e3).view(np.uint64)
    if op in (dev.OP_MIN_I64, dev.OP_MAX_I64):
        v = rng.integers(-10 ** 15, 10 ** 15, size=n)
        v[rng.random(n) < 0.05] = I64_MIN
        v[rng.random(n) < 0.05] = I64_MAX
        return v.astype(np.int64).view(np.uint64)
    if op == dev.OP_SUM_I64:
        return rng.integers(-10 ** 12, 10 ** 12, size=n).astype(np.int64).view(np.uint64)
    return np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)   # COUNT / FIRST / LAST: distinct bits


def py_fold(op, vals):
    """Python's left fold of a group's values (uint64 bits, in input order); SUM_F64 returns the exact fsum"""
    if op == dev.OP_COUNT:
        return len(vals)
    if op == dev.OP_FIRST:
        return int(vals[0])
    if op == dev.OP_LAST:
        return int(vals[-1])
    if op == dev.OP_SUM_F64:
        return math.fsum(vals.view(np.float64).tolist())
    if op in (dev.OP_MIN_F64, dev.OP_MAX_F64):
        f = min if op == dev.OP_MIN_F64 else max
        r = functools.reduce(lambda acc, v: f(acc, v), vals.view(np.float64).tolist())
        return int(np.array([r]).view(np.uint64)[0])
    ints = vals.view(np.int64).tolist()
    if op == dev.OP_SUM_I64:
        r = sum(ints)
    else:
        f = min if op == dev.OP_MIN_I64 else max
        r = functools.reduce(lambda acc, v: f(acc, v), ints)
    return r & ((1 << 64) - 1)


def expected_groups(keys, vals, op, xf):
    """(group keys in key order under xf, the fold of each group in input order)"""
    o = stable_order(keys, xf)
    k, v = keys[o], vals[o]
    if len(k) == 0:
        return k, []
    heads = np.flatnonzero(np.concatenate(([True], k[1:] != k[:-1])))
    ends = np.concatenate((heads[1:], [len(k)]))
    return k[heads], [py_fold(op, v[a:b]) for a, b in zip(heads.tolist(), ends.tolist())]


def assert_folds(gk, gv, ek, ev, op, keyed_order, vals=None, keys=None):
    assert len(gk) == len(ek) and len(set(gk.tolist())) == len(gk)
    if not keyed_order:       # the hash-folded integer ops under KEY_MIX: any group order
        o = np.argsort(gk, kind="stable")
        gk, gv = gk[o], gv[o]
        o = np.argsort(ek, kind="stable")
        ek, ev = ek[o], [ev[i] for i in o.tolist()]
    assert np.array_equal(gk, ek)
    if op == dev.OP_SUM_F64:
        got = gv.view(np.float64)
        for k, g, e in zip(gk.tolist(), got.tolist(), ev):
            sel = vals[keys == np.uint64(k)].view(np.float64)
            assert abs(g - e) <= 4 * len(sel) * 2.0 ** -53 * float(np.abs(sel).sum()), (k, g, e)
    else:
        assert gv.tolist() == [int(x) for x in ev]


def keyed_order(op, xf):
    return not (xf == dev.KEY_MIX and op in (dev.OP_SUM_I64, dev.OP_COUNT, dev.OP_MIN_I64, dev.OP_MAX_I64))


def xforms_for(op):
    """F64 ops on F64 and MIX keys; integer ops and FIRST / LAST on I64, F64 and MIX keys"""
    return (dev.KEY_F64, dev.KEY_MIX) if op in F64_OPS else (dev.KEY_I64, dev.KEY_F64, dev.KEY_MIX)


def grouped_keys(xf, rng, n, n_keys):
    pool = keys_for(xf, rng, n_keys)
    return pool[rng.integers(0, len(pool), size=n)]


@pytest.mark.parametrize("op", ALL_OPS)
def test_sort_reduce_and_reduce_by_key_every_op(ctx, op):
    """dampr_kv_sort_reduce at 1 record, one leaf + 1, groups that straddle the 4096-record tiles (20K records of 37
    keys), many groups over a partition level; dampr_kv_reduce_by_key over the same records sorted"""
    for xf in xforms_for(op):
        for n, nk in ((1, 1), (LEAF + 1, 3), (20_000, 37), (300_000, 5000)):
            rng = np.random.default_rng(1000 * op + 10 * xf + nk)
            keys = grouped_keys(xf, rng, n, nk)
            vals = fold_values(op, rng, n)
            ek, ev = expected_groups(keys, vals, op, xf)
            kv = ctx.kv_from_columns(keys, vals)
            out = kv.sort_reduce(op, xf)
            gk, gv = out.columns()
            out.free()
            kv.free()
            assert_folds(gk, gv, ek, ev, op, keyed_order(op, xf), vals, keys)
            # reduce_by_key folds adjacent equal keys of a sorted run, groups in run order
            o = stable_order(keys, xf)
            srt = ctx.kv_from_columns(keys[o], vals[o])
            red = srt.reduce_by_key(op)
            gk, gv = red.columns()
            red.free()
            srt.free()
            assert_folds(gk, gv, ek, ev, op, True, vals, keys)


@pytest.mark.parametrize("op", ALL_OPS)
def test_single_key_larger_than_a_leaf_every_op(ctx, op):
    """every record has the same key: single_group_reduce_kernel folds the range in one CTA. Its lanes combine
    strided partial folds, which for MIN / MAX_F64 must still equal the left fold on the planner's domain"""
    for xf in xforms_for(op):
        for n in (LEAF + 1, 50_000, 1_000_003):
            rng = np.random.default_rng(op * 7 + n)
            key = keys_for(xf, rng, 3)[2]
            keys = np.full(n, key, dtype=np.uint64)
            vals = fold_values(op, rng, n)
            kv = ctx.kv_from_columns(keys, vals)
            out = kv.sort_reduce(op, xf)
            gk, gv = out.columns()
            out.free()
            kv.free()
            assert_folds(gk, gv, keys[:1], [py_fold(op, vals)], op, True, vals, keys)


# ---- merges --------------------------------------------------------------------------------------------------
def sorted_runs(xf, rng, k, op):
    """k runs, each sorted under xf, with empty runs between non-empty ones and keys shared across runs (ties).
    Values: the fold values of op, or (position << 8 | run) when op is None"""
    pool = keys_for(xf, rng, 400)
    runs = []
    for r in range(k):
        n = 0 if (r % 3 == 1) else int(rng.integers(1, 3000))
        keys = pool[rng.integers(0, len(pool), size=n)]
        vals = fold_values(op, rng, n) if op is not None else (np.arange(n, dtype=np.uint64) << np.uint64(8)) | np.uint64(r)
        o = stable_order(keys, xf)
        runs.append((keys[o], vals[o]))
    return runs


@pytest.mark.parametrize("k", [1, 2, 8, 70])
@pytest.mark.parametrize("xf", [dev.KEY_F64, dev.KEY_I64])
def test_merge_and_merge_ranges(ctx, k, xf):
    """dampr_kv_merge and dampr_kv_merge_ranges == the stable sort of the runs' concatenation (ties: run order, then
    position), without and with every op that applies to the values; the numpy stand-in device bit for bit"""
    fake = FakeCtx()
    for op in (None,) + ALL_OPS:
        rng = np.random.default_rng(k * 131 + xf * 7 + (op or 0))
        runs = sorted_runs(xf, rng, k, op)
        allk = np.concatenate([r[0] for r in runs])
        allv = np.concatenate([r[1] for r in runs])
        offs = np.concatenate(([0], np.cumsum([len(r[0]) for r in runs]))).astype(np.uint64)
        dev_runs = [ctx.kv_from_columns(a, b) for a, b in runs]
        flat = ctx.kv_from_columns(allk, allv)
        fake_flat = fake.kv_from_columns(allk, allv)
        code = -1 if op is None else op
        outs = [ctx.kv_merge(dev_runs, xf, code), ctx.kv_merge_ranges(flat, offs, xf, code)]
        want = fake.kv_merge_ranges(fake_flat, offs, xf, code)
        wk, wv = want.columns()
        for out in outs:
            gk, gv = out.columns()
            out.free()
            if op is None:
                o = stable_order(allk, xf)
                assert np.array_equal(gk, allk[o]) and np.array_equal(gv, allv[o]), (k, xf)
            elif op == dev.OP_SUM_F64:
                ek, ev = expected_groups(allk, allv, op, xf)
                assert_folds(gk, gv, ek, ev, op, True, allv, allk)
            else:
                assert np.array_equal(gk, wk) and np.array_equal(gv, wv), (k, xf, op)
                ek, ev = expected_groups(allk, allv, op, xf)
                assert_folds(gk, gv, ek, ev, op, True)
        for x in dev_runs + [flat]:
            x.free()


# ---- joins ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("xf", [dev.KEY_F64, dev.KEY_I64])
def test_join_ranges(ctx, xf):
    """dampr_kv_join_ranges: (left begin, left end, right begin, right end) per left key group, keys on one side
    only, an empty side; the numpy stand-in device bit for bit, up to where an empty right range starts"""
    rng = np.random.default_rng(5 + xf)
    pool = np.unique(keys_for(xf, rng, 3000))
    fake = FakeCtx()
    for nl, nr in ((20_000, 5000), (5000, 0), (0, 5000), (1, 1), (LEAF + 1, 70_000)):
        lk = pool[rng.integers(0, len(pool) * 2 // 3, size=nl)]           # the top third of the pool: right only
        rk = pool[rng.integers(len(pool) // 3, len(pool), size=nr)]       # the bottom third: left only
        sides = []
        for keys in (lk, rk):
            o = stable_order(keys, xf)
            sides.append((keys[o], np.arange(len(keys), dtype=np.uint64)))
        L, R = (ctx.kv_from_columns(*s) for s in sides)
        FL, FR = (fake.kv_from_columns(*s) for s in sides)
        rows = L.join_ranges(R, xf)
        want = FL.join_ranges(FR, xf)
        for r in (rows, want):    # a key without a match: any empty right range (the header's contract)
            r[r[:, 2] == r[:, 3], 2:] = 0
        assert np.array_equal(rows, want), (nl, nr)
        if nl > 1 and nr > 1:   # both kinds of left group occur
            assert (rows[:, 2] < rows[:, 3]).any() and (rows[:, 2] == rows[:, 3]).any()
        L.free()
        R.free()


# ---- the DSL over float keys, on the device ------------------------------------------------------------------
def test_float_key_pipelines_agree_with_the_reference(ctx, monkeypatch):
    """the pipelines of test_float_key_lowering.py (recorded reference outputs) through the real device"""
    import test_float_key_lowering as fkl
    fkl.check_all(monkeypatch, None)


def test_float_keys_through_the_spill_path(ctx):
    """a float sort_by and a float-keyed a_group_by(...).sum() of 1.5M records with a capped device arena: both
    spill, and agree with Python (stable order, one group for 0.0 / -0.0 reporting its first key)"""
    from dampr_b200 import Dampr, settings
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    rng = np.random.default_rng(77)
    n = 1_500_000
    pool = np.concatenate((rng.standard_normal(50_000) * 1e3, [0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324]))
    V = pool[rng.integers(0, len(pool), size=n)]
    V[rng.random(n) < 0.01] = -0.0
    V[rng.random(n) < 0.01] = 0.0
    K = np.arange(n, dtype=np.int64)
    old = settings.device_arena_bytes
    settings.device_arena_bytes = 8 << 20
    try:
        src = Dampr.read_input(ArrayKVInput(K, V))
        got = src.sort_by(lambda x: x[1]).read()
        assert any("[spilled:" in h for _s, h, _d in runner_mod.LAST_STATS.stages)
        o = np.argsort(V, kind="stable")          # numpy's float order: -0.0 == 0.0, stable
        assert [r[0] for r in got] == o.tolist()
        assert np.array_equal(np.array([r[1] for r in got]).view(np.uint64), V[o].view(np.uint64))
        got = src.a_group_by(lambda x: x[1], lambda x: x[0]).sum().read()
        assert any("[spilled:" in h for _s, h, _d in runner_mod.LAST_STATS.stages)
        exp = {}
        for k, v in zip(K.tolist(), V.tolist()):
            exp[v] = exp.get(v, 0) + k
        assert len(got) == len(exp) and dict(got) == exp
        zero = [k for k, _s in got if k == 0]
        first = V[np.flatnonzero(V == 0)[0]]
        assert len(zero) == 1 and math.copysign(1, zero[0]) == math.copysign(1, first)
    finally:
        settings.device_arena_bytes = old

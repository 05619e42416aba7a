"""GPU parity: partition + sort + segmented reduce + join + probe (csrc/kv.cu, ops.cu) vs oracle."""
import numpy as np
import pytest

from dampr_b200 import device as dev
from oracle import gen, refsem

pytestmark = pytest.mark.gpu


def xf_key(keys, xf):
    k = keys.astype(np.uint64)
    if xf == dev.KEY_I64:
        return k ^ np.uint64(1 << 63)
    if xf == dev.KEY_F64:
        neg = (k >> np.uint64(63)).astype(bool)
        return np.where(neg, ~k, k | np.uint64(1 << 63))
    return k


def mix64(x):
    x = x.astype(np.uint64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
    return x


def check_sort(ctx, keys, vals, xf):
    kv = ctx.kv_from_columns(keys, vals)
    kv.sort(xf)
    k2, v2 = kv.columns()
    sk = mix64(keys.view(np.uint64)) if xf == dev.KEY_MIX else xf_key(keys.view(np.uint64), xf)
    order = np.argsort(sk, kind="stable")
    assert np.array_equal(k2, keys.view(np.uint64)[order])
    assert np.array_equal(v2, vals.view(np.uint64)[order])  # stable: ties keep input order
    kv.free()


@pytest.mark.parametrize("n", [0, 1, 2, 31, 1000, 4096, 4097, 50000, 300000])
@pytest.mark.parametrize("xf", [dev.KEY_RAW, dev.KEY_MIX, dev.KEY_I64])
def test_sort_sizes(ctx, n, xf):
    keys, vals = gen.kv(42, n, max(1, n // 3))
    check_sort(ctx, keys, vals, xf)


def test_sort_large_two_levels(ctx):
    keys, vals = gen.kv(7, 6_000_000, 5_000_000)
    check_sort(ctx, keys, vals, dev.KEY_MIX)
    check_sort(ctx, keys, vals, dev.KEY_RAW)


def test_sort_skew_and_duplicates(ctx):
    rng = np.random.default_rng(3)
    n = 400000
    keys = rng.zipf(1.3, size=n).astype(np.uint64)  # heavy hitters
    vals = np.arange(n, dtype=np.int64)
    for xf in (dev.KEY_MIX, dev.KEY_RAW):
        check_sort(ctx, keys, vals, xf)
    keys[:] = 17  # a single key
    check_sort(ctx, keys, vals, dev.KEY_MIX)
    keys = np.arange(n, dtype=np.uint64)[::-1].copy()  # dense small ints, reversed
    check_sort(ctx, keys, vals, dev.KEY_RAW)


def test_sort_signed_and_float(ctx):
    rng = np.random.default_rng(9)
    n = 100000
    ik = rng.integers(-10**12, 10**12, size=n).astype(np.int64)
    vals = np.arange(n, dtype=np.int64)
    kv = ctx.kv_from_columns(ik.view(np.uint64), vals)
    kv.sort(dev.KEY_I64)
    k2, _ = kv.columns()
    assert np.array_equal(k2.view(np.int64), np.sort(ik, kind="stable"))
    fk = rng.standard_normal(n) * 1e6
    kv = ctx.kv_from_columns(fk.view(np.uint64), vals)
    kv.sort(dev.KEY_F64)
    k2, _ = kv.columns()
    assert np.array_equal(k2.view(np.float64), np.sort(fk, kind="stable"))


@pytest.mark.parametrize("n,nk", [(0, 1), (1, 1), (5000, 10), (5000, 5000), (200000, 1000), (3_000_000, 400_000)])
def test_sort_reduce_sum_count(ctx, n, nk):
    keys, vals = gen.kv(11, n, nk)
    kv = ctx.kv_from_columns(keys, vals)
    out = kv.sort_reduce(dev.OP_SUM_I64, dev.KEY_MIX)
    k2, v2 = out.columns()
    got = dict(zip(k2.tolist(), v2.view(np.int64).tolist()))
    assert len(got) == len(k2)
    assert got == refsem.group_sum(keys, vals)
    kv2 = ctx.kv_from_columns(keys, vals)
    out = kv2.sort_reduce(dev.OP_COUNT, dev.KEY_RAW)
    k2, v2 = out.columns()
    assert np.array_equal(k2, np.sort(k2))  # RAW transform returns groups in key order
    assert dict(zip(k2.tolist(), v2.tolist())) == refsem.group_count(keys)


def test_reduce_ops(ctx):
    keys, vals = gen.kv(5, 100000, 300)
    for op, f in ((dev.OP_MIN_I64, min), (dev.OP_MAX_I64, max), (dev.OP_FIRST, lambda a, b: a),
                  (dev.OP_LAST, lambda a, b: b)):
        kv = ctx.kv_from_columns(keys, vals)
        out = kv.sort_reduce(op, dev.KEY_MIX)
        k2, v2 = out.columns()
        assert dict(zip(k2.tolist(), v2.view(np.int64).tolist())) == refsem.group_fold(keys, vals, f)


def test_reduce_float_sum_tolerance(ctx):
    """fp tolerance (SURVEY §8(c)): |x - fsum| <= 4 n 2^-53 sum|v|."""
    import math
    rng = np.random.default_rng(1)
    n = 200000
    keys = rng.integers(0, 50, size=n).astype(np.uint64)
    vals = rng.standard_normal(n) * 1e3
    kv = ctx.kv_from_columns(keys, vals.view(np.uint64))
    out = kv.sort_reduce(dev.OP_SUM_F64, dev.KEY_MIX)
    k2, v2 = out.columns()
    got = dict(zip(k2.tolist(), v2.view(np.float64).tolist()))
    for k in range(50):
        sel = vals[keys == k]
        exact = math.fsum(sel.tolist())
        tol = 4 * len(sel) * 2.0 ** -53 * float(np.abs(sel).sum())
        assert abs(got[k] - exact) <= tol


def test_reduce_consumes_or_keeps_its_input_as_documented(ctx):
    """dampr_kv_sort_reduce consumes its input; dampr_kv_reduce_by_key leaves the sorted run alone, also
    when segments are larger than a leaf (heavy keys) and the sizes force one or two partition levels."""
    for n, nk in ((300_000, 40), (3_000_000, 1500)):
        keys, vals = gen.kv(31, n, nk)
        kv = ctx.kv_from_columns(keys, vals)
        out = kv.sort_reduce(dev.OP_SUM_I64, dev.KEY_RAW)
        assert len(kv) == 0
        k1, v1 = out.columns()
        assert dict(zip(k1.tolist(), v1.view(np.int64).tolist())) == refsem.group_sum(keys, vals)
        kv = ctx.kv_from_columns(keys, vals).sort(dev.KEY_RAW)
        before = kv.records().copy()
        for op, exp in ((dev.OP_SUM_I64, refsem.group_sum(keys, vals)), (dev.OP_COUNT, refsem.group_count(keys))):
            red = kv.reduce_by_key(op)
            rk, rv = red.columns()
            assert dict(zip(rk.tolist(), rv.view(np.int64).tolist())) == exp
            assert len(kv) == n and np.array_equal(kv.records(), before)


def test_heavy_single_key_reduce(ctx):
    n = 1_000_000
    keys = np.full(n, 12345, dtype=np.uint64)
    keys[::1000] = 99
    vals = np.ones(n, dtype=np.int64)
    kv = ctx.kv_from_columns(keys, vals)
    out = kv.sort_reduce(dev.OP_SUM_I64, dev.KEY_MIX)
    k2, v2 = out.columns()
    assert dict(zip(k2.tolist(), v2.tolist())) == {12345: n - 1000, 99: 1000}


def test_group_offsets_and_merge(ctx):
    keys, vals = gen.kv(21, 50000, 700)
    kv = ctx.kv_from_columns(keys, vals).sort(dev.KEY_RAW)
    offs = kv.group_offsets()
    k2, _ = kv.columns()
    heads = np.flatnonzero(np.concatenate(([True], k2[1:] != k2[:-1])))
    assert np.array_equal(offs[:-1], heads) and offs[-1] == len(k2)
    # k-way merge of sorted runs == stable sort of the concatenation; with reduce == group sums
    runs = []
    allk, allv = [], []
    for s in range(5):
        k, v = gen.kv(100 + s, 20000, 900)
        runs.append(ctx.kv_from_columns(k, v).sort(dev.KEY_RAW))
        allk.append(k)
        allv.append(v)
    merged = dev.kv_merge(ctx, runs, dev.KEY_RAW)
    mk, _ = merged.columns()
    assert np.array_equal(mk, np.sort(np.concatenate(allk)))
    red = dev.kv_merge(ctx, runs, dev.KEY_RAW, dev.OP_SUM_I64)
    rk, rv = red.columns()
    assert dict(zip(rk.tolist(), rv.view(np.int64).tolist())) == refsem.group_sum(np.concatenate(allk), np.concatenate(allv))


def test_join_ranges(ctx):
    lk, lv = gen.kv(1, 30000, 2000)
    rk, rv = gen.kv(2, 3000, 4000)
    L = ctx.kv_from_columns(lk, lv).sort(dev.KEY_MIX)
    R = ctx.kv_from_columns(rk, rv).sort(dev.KEY_MIX)
    rows = L.join_ranges(R, dev.KEY_MIX)
    Lk, Lv = L.columns()
    Rk, Rv = R.columns()
    got_inner, got_left = {}, {}
    for lb, le, rb, re_ in rows.tolist():
        k = int(Lk[lb])
        pair = (Lv[lb:le].view(np.int64).tolist(), Rv[rb:re_].view(np.int64).tolist())
        got_left[k] = pair
        if re_ > rb:
            got_inner[k] = pair
    assert got_inner == refsem.inner_join(lk, lv, rk, rv)
    assert got_left == refsem.left_join(lk, lv, rk, rv)


def test_hash_probe(ctx):
    bk = np.unique(gen.kv(3, 20000, 50000)[0])
    bv = np.arange(len(bk), dtype=np.int64)
    pk, pv = gen.kv(4, 100000, 50000)
    B = ctx.kv_from_columns(bk, bv)
    P = ctx.kv_from_columns(pk, pv)
    vals, hit = B.hash_probe(P)
    k2, v2 = vals.columns()
    table = dict(zip(bk.tolist(), bv.tolist()))
    exp_hit = np.array([k in table for k in pk.tolist()], dtype=np.uint8)
    assert np.array_equal(hit, exp_hit)
    exp_val = np.array([table.get(k, 0) for k in pk.tolist()], dtype=np.int64)
    assert np.array_equal(v2.view(np.int64), exp_val)
    assert np.array_equal(k2, pk)


def test_partition_by_owner(ctx):
    keys, vals = gen.kv(8, 100000, 30000)
    kv = ctx.kv_from_columns(keys, vals)
    for nd in (1, 2, 3, 8):
        out, counts = kv.partition_by_owner(nd)
        k2, v2 = out.columns()
        owner = (mix64(keys) % np.uint64(nd)).astype(np.int64)
        order = np.argsort(owner, kind="stable")
        assert np.array_equal(k2, keys[order]) and np.array_equal(v2.view(np.int64), vals[order])
        assert np.array_equal(counts, np.bincount(owner, minlength=nd).astype(np.uint64))


def test_copies_that_straddle_page_locked_regions(ctx):
    """A host range that crosses two separately registered regions (or the end of one) cannot be copied directly
    (cudaErrorInvalidValue): the library sends it through its staging ring (spill.py's run buffer is page-locked
    piecewise). Downloads and uploads, both ends registered, one end registered, none."""
    n = 3_000_000   # 48 MB
    keys, vals = gen.kv(13, n, n)
    kv = ctx.kv_from_columns(keys, vals)
    want = kv.records()
    buf = np.zeros((n, 2), dtype=np.uint64)
    assert dev.host_register(buf[:n // 3]) and dev.host_register(buf[n // 3: 2 * n // 3])
    try:
        for lo, hi in ((0, n), (0, n // 3), (n // 6, n // 2), (n // 2, n), (2 * n // 3, n)):
            buf[:] = 0
            kv.records_into(buf[lo:hi], lo)
            assert np.array_equal(buf[lo:hi], want[lo:hi]), (lo, hi)
            back = ctx.kv(hi - lo)
            back.upload(0, buf[lo:hi], hi - lo)
            ctx.sync()
            assert np.array_equal(back.records(), want[lo:hi]), (lo, hi)
            back.free()
    finally:
        dev.host_unregister(buf[:n // 3])
        dev.host_unregister(buf[n // 3: 2 * n // 3])
    kv.free()


def test_all_to_all_world1_through_the_c_abi(ctx):
    """dampr_kv_all_to_all on a one-rank communicator (csrc/comm.cu; the 2-GPU path is tests/test_gpu_multi.py):
    NCCL binds at run time, the counts + header row comes back, the payload is the stable split by owner."""
    keys, vals = gen.kv(9, 200_000, 30_000)
    kv = ctx.kv_from_columns(keys, vals)
    if getattr(ctx, "comm", None) is None:
        ctx.comm_create(0, 1, ctx.comm_unique_id())
    out, offs, heads = ctx.kv_all_to_all(kv, header=[7, -3, 1 << 40])
    assert offs.tolist() == [0, len(keys)] and heads.tolist() == [[7, -3, 1 << 40]]
    k2, v2 = out.columns()
    assert np.array_equal(k2, keys.view(np.uint64)) and np.array_equal(v2, vals.view(np.uint64))
    assert len(kv) == len(keys)          # the input is left alone
    out.free()
    empty = ctx.kv(1)
    out, offs, heads = ctx.kv_all_to_all(empty)
    assert offs.tolist() == [0, 0] and heads is None and len(out) == 0
    for x in (kv, empty, out):
        x.free()


def test_synth_kv_matches_numpy(ctx):
    kv = ctx.kv(10000)
    ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 42, 10000, 777))
    k2, v2 = kv.columns()
    ek, ev = gen.kv(42, 10000, 777)
    assert np.array_equal(k2, ek) and np.array_equal(v2.view(np.int64), ev)


# ---- partition level + CTA leaf at chosen sizes, recursion on oversized segments ---------------------------
@pytest.mark.parametrize("n", [4097, 9000, 27000, 27600, 60000, 1_000_000])
def test_sort_sizes_around_leaf_and_level_boundaries(ctx, n):
    """4097 is the smallest input that needs a partition level (one leaf holds 4096 records); the larger sizes
    fill the leaf chunks unevenly, up to 1M records in one level; unique-ish and duplicated keys"""
    for nk in (max(1, n // 3), 10 * n):
        keys, vals = gen.kv(77, n, nk)
        check_sort(ctx, keys, vals, dev.KEY_MIX)
        check_sort(ctx, keys, vals, dev.KEY_RAW)


def test_one_key_holding_most_of_a_bucket(ctx):
    """one key holds 70 % of a 20K-record input: its segment outgrows a leaf and is sorted by recursion, where
    the all-equal remainder is copied or folded as one group; the order stays stable and the folds see every
    record"""
    rng = np.random.default_rng(5)
    n = 20000
    keys = rng.integers(0, 1 << 62, size=n).astype(np.uint64)
    keys[rng.random(n) < 0.7] = np.uint64(123456789)
    vals = np.arange(n, dtype=np.int64)
    check_sort(ctx, keys, vals, dev.KEY_MIX)
    check_sort(ctx, keys, vals, dev.KEY_RAW)
    kv = ctx.kv_from_columns(keys, vals)
    out = kv.sort_reduce(dev.OP_COUNT, dev.KEY_RAW)
    k2, v2 = out.columns()
    assert dict(zip(k2.tolist(), v2.tolist())) == refsem.group_count(keys)
    kv = ctx.kv_from_columns(keys, vals)
    out = kv.sort_reduce(dev.OP_FIRST, dev.KEY_MIX)
    k2, v2 = out.columns()
    assert dict(zip(k2.tolist(), v2.view(np.int64).tolist())) == refsem.group_fold(keys, vals, lambda a, b: a)


def test_sort_mixed_and_zipf_keys_and_counts(ctx):
    """a 2.5M-record KEY_MIX sort, a Zipf-skewed KEY_RAW sort and the sort_reduce counts of the Zipf keys"""
    keys, vals = gen.kv(13, 2_500_000, 700_000)
    check_sort(ctx, keys, vals, dev.KEY_MIX)
    keys = (np.random.default_rng(3).zipf(1.2, size=600_000) % 5000).astype(np.uint64)
    check_sort(ctx, keys, np.arange(len(keys), dtype=np.int64), dev.KEY_RAW)
    kv = ctx.kv_from_columns(keys, np.ones(len(keys), dtype=np.int64))
    out = kv.sort_reduce(dev.OP_SUM_I64, dev.KEY_MIX)
    k2, v2 = out.columns()
    assert dict(zip(k2.tolist(), v2.tolist())) == refsem.group_count(keys)


def test_low_cardinality_keys_hot_runs(ctx):
    """few distinct keys: every (tile, bucket) run of the scatter is long (the warp-sorted path)"""
    rng = np.random.default_rng(17)
    n = 1_500_000
    for nk in (1, 3, 200, 5000):
        keys = (rng.integers(0, nk, size=n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        vals = np.arange(n, dtype=np.int64)
        check_sort(ctx, keys, vals, dev.KEY_RAW)
        check_sort(ctx, keys, vals, dev.KEY_MIX)


@pytest.mark.parametrize("n,nk", [(3000, 40), (4096, 1), (4096, 100), (2_000_000, 30_000), (1_000_000, 12_000)])
def test_duplicate_heavy_leaf_bins(ctx, n, nk):
    """K << N: a leaf chunk's bins hold 30..300 records of one key each (leaf.cuh leaf_sort_heavy_bins: a warp
    sorts a single-key bin's record indices through a bitmap) next to bins that several keys share (member walk);
    order among equal keys must stay the input order, through sort, sort+reduce and the merge tiles."""
    rng = np.random.default_rng(n + nk)
    base = rng.integers(0, 1 << 62, size=nk).astype(np.uint64)
    base[: max(1, nk // 10)] = np.arange(max(1, nk // 10), dtype=np.uint64)  # neighbours that share a bin
    keys = base[rng.integers(0, nk, size=n)]
    vals = np.arange(n, dtype=np.int64)
    for xf in (dev.KEY_RAW, dev.KEY_MIX):
        check_sort(ctx, keys, vals, xf)
    u, first = np.unique(keys, return_index=True)
    last = n - 1 - np.unique(keys[::-1], return_index=True)[1]
    for op, exp in ((dev.OP_FIRST, first), (dev.OP_LAST, last)):
        kv = ctx.kv_from_columns(keys, vals)
        red = kv.sort_reduce(op, dev.KEY_RAW)
        rk, rv = red.columns()
        assert np.array_equal(rk, u) and np.array_equal(rv.view(np.int64), exp)
        red.free()
    if n >= 1_000_000:
        half = n // 2
        runs = []
        for lo, hi in ((0, half), (half, n)):
            r = ctx.kv_from_columns(keys[lo:hi], vals[lo:hi])
            r.sort(dev.KEY_RAW)
            runs.append(r)
        out = ctx.kv_merge(runs, dev.KEY_RAW)
        mk, mv = out.columns()
        order = np.argsort(keys, kind="stable")
        assert np.array_equal(mk, keys[order]) and np.array_equal(mv.view(np.int64), vals[order])
        for x in runs + [out]:
            x.free()


def _merge_oracle(runs_k, runs_v, xf):
    """stable k-way merge = stable sort of the concatenation in run order (heapq.merge, dataset.py:571-579)"""
    ak, av = np.concatenate(runs_k), np.concatenate(runs_v)
    sk = mix64(ak) if xf == dev.KEY_MIX else xf_key(ak, xf)
    order = np.argsort(sk, kind="stable")
    return ak[order], av[order]


@pytest.mark.parametrize("k,n,nk", [(2, 50000, 300), (3, 1000, 10 ** 9), (8, 200000, 40000), (8, 5000, 3), (20, 30000, 1000),
                                    (70, 3000, 500)])
def test_merge_kway_stable(ctx, k, n, nk):
    for xf in (dev.KEY_RAW, dev.KEY_MIX):
        runs, rk, rv = [], [], []
        for s in range(k):
            kk, _ = gen.kv(1000 + s, n + 37 * s, nk)
            vv = (np.arange(len(kk), dtype=np.int64) << 8) | s  # value encodes (input position, run)
            kv = ctx.kv_from_columns(kk, vv).sort(xf)
            a, b = kv.columns()
            runs.append(kv)
            rk.append(a.copy())
            rv.append(b.view(np.int64).copy())
        merged = dev.kv_merge(ctx, runs, xf)
        mk, mv = merged.columns()
        ek, ev = _merge_oracle(rk, rv, xf)
        assert np.array_equal(mk, ek)
        assert np.array_equal(mv.view(np.int64), ev)  # ties: run order, then position
        allk, allv = np.concatenate(rk), np.concatenate(rv)
        for op, exp in ((dev.OP_SUM_I64, refsem.group_sum(allk, allv)), (dev.OP_COUNT, refsem.group_count(allk))):
            red = dev.kv_merge(ctx, runs, xf, op)
            gk, gv = red.columns()
            assert len(set(gk.tolist())) == len(gk)
            assert dict(zip(gk.tolist(), gv.view(np.int64).tolist())) == exp
        # FIRST / LAST follow the merge order
        first = dev.kv_merge(ctx, runs, xf, dev.OP_FIRST)
        fk, fv = first.columns()
        heads = np.concatenate(([True], ek[1:] != ek[:-1]))
        assert np.array_equal(fk, ek[heads]) and np.array_equal(fv.view(np.int64), ev[heads])
        last = dev.kv_merge(ctx, runs, xf, dev.OP_LAST)
        lk, lv = last.columns()
        tails = np.concatenate((ek[1:] != ek[:-1], [True]))
        assert np.array_equal(lk, ek[tails]) and np.array_equal(lv.view(np.int64), ev[tails])


def test_merge_edge_cases(ctx):
    empty = ctx.kv_from_columns(np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.int64))
    one = ctx.kv_from_columns(np.array([5], dtype=np.uint64), np.array([7], dtype=np.int64))
    assert len(dev.kv_merge(ctx, [], dev.KEY_RAW)) == 0
    assert len(dev.kv_merge(ctx, [empty, empty], dev.KEY_RAW, dev.OP_SUM_I64)) == 0
    m = dev.kv_merge(ctx, [empty, one, empty, one], dev.KEY_RAW)
    assert m.columns()[0].tolist() == [5, 5]
    r = dev.kv_merge(ctx, [empty, one, empty, one], dev.KEY_RAW, dev.OP_SUM_I64)
    assert [x.tolist() for x in r.columns()] == [[5], [14]]
    # one key spanning many partitions and runs
    n = 40000
    runs = [ctx.kv_from_columns(np.full(n, 9, dtype=np.uint64), np.arange(n, dtype=np.int64) + s * n) for s in range(4)]
    r = dev.kv_merge(ctx, runs, dev.KEY_RAW, dev.OP_SUM_I64)
    assert [x.tolist() for x in r.columns()] == [[9], [sum(range(4 * n))]]
    r = dev.kv_merge(ctx, runs, dev.KEY_RAW, dev.OP_LAST)
    assert [x.tolist() for x in r.columns()] == [[9], [4 * n - 1]]
    m = dev.kv_merge(ctx, runs, dev.KEY_RAW)
    assert np.array_equal(m.columns()[1].view(np.int64), np.arange(4 * n))


def test_reduce_by_key_single_pass(ctx):
    rng = np.random.default_rng(23)
    for n, nk in ((1, 1), (4096, 4096), (4097, 2), (300_000, 7), (2_000_000, 900_000)):
        keys = np.sort(rng.integers(0, nk, size=n).astype(np.uint64))
        vals = rng.integers(-1000, 1000, size=n).astype(np.int64)
        kv = ctx.kv_from_columns(keys, vals)
        for op, f in ((dev.OP_SUM_I64, None), (dev.OP_MIN_I64, min), (dev.OP_FIRST, lambda a, b: a), (dev.OP_LAST, lambda a, b: b)):
            red = kv.reduce_by_key(op)
            gk, gv = red.columns()
            exp = refsem.group_sum(keys, vals) if f is None else refsem.group_fold(keys, vals, f)
            assert np.array_equal(gk, np.unique(keys))
            assert dict(zip(gk.tolist(), gv.view(np.int64).tolist())) == exp
    fl = rng.standard_normal(100000)
    keys = np.sort(rng.integers(0, 20, size=100000).astype(np.uint64))
    red = ctx.kv_from_columns(keys, fl.view(np.uint64)).reduce_by_key(dev.OP_SUM_F64)
    gk, gv = red.columns()
    import math
    for k, got in zip(gk.tolist(), gv.view(np.float64).tolist()):
        sel = fl[keys == k]
        assert abs(got - math.fsum(sel.tolist())) <= 4 * len(sel) * 2.0 ** -53 * float(np.abs(sel).sum())


def test_hash_join_compacts_on_the_device(ctx):
    """dampr_kv_hash_join: the probe records with a partner and (key, build value), in probe order"""
    bk = np.unique(gen.kv(3, 20000, 50000)[0])
    bv = np.arange(len(bk), dtype=np.int64)
    for n in (0, 1, 4095, 4096, 100000, 1_000_000):
        pk, pv = gen.kv(4, n, 50000)
        B = ctx.kv_from_columns(bk, bv)
        P = ctx.kv_from_columns(pk, pv)
        ml, mr = B.hash_join(P)
        table = dict(zip(bk.tolist(), bv.tolist()))
        m = np.array([k in table for k in pk.tolist()], dtype=bool)
        lk, lv = ml.columns()
        rk, rv = mr.columns()
        assert np.array_equal(lk, pk[m]) and np.array_equal(lv.view(np.int64), pv[m])
        assert np.array_equal(rk, pk[m])
        assert np.array_equal(rv.view(np.int64), np.array([table[k] for k in pk[m].tolist()], dtype=np.int64))
        for x in (B, P, ml, mr):
            x.free()

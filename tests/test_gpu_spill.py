"""The out-of-core spill path (dampr_b200/spill.py) on the device and on the numpy stand-in (tests/fake_device.py),
against plain references: Python's left fold of every key group in input order (py_fold; math.fsum with the bound
4 n 2^-53 sum|v| for OP_SUM_F64), numpy's stable argsort of the keys' order domain, and the in-core device fold and
sort of the same records.

The device arena is capped at 4 MB, so a batch holds 65 536 records and 1.2 M records make 19 batches and 24
buckets. The key shapes steer the pipeline into its skew branches: keys crafted through the inverse of mix64 so
that 40 % of the records land in one hash bucket (_merge_runs cuts it into key-range slices), one key holding 70 %
of a sort (the single-key range), and a narrow band of keys the sample misses (external_sort re-splits the range).
Every test also asserts that the branch it names ran, so that a change of the batch size cannot quietly turn it
into a uniform-key test."""
import math

import numpy as np
import pytest

from dampr_b200 import device as dev
from dampr_b200 import settings, spill
from fake_device import FakeCtx, FakeKV
from test_gpu_key_orders import ALL_OPS, F64_SPECIAL, I64_MIN, expected_groups, fold_values, keys_for, py_fold, \
    stable_order

ARENA = 4 << 20
N_GROUP = 1_200_000
N_SORT = 1_000_000
# a heavy key per key transform, at an end of its order: the largest raw key, INT64_MIN, a negative NaN with a payload
DOMINANT = {dev.KEY_RAW: np.uint64((1 << 64) - 1), dev.KEY_I64: np.int64(I64_MIN).view(np.uint64),
            dev.KEY_F64: F64_SPECIAL[13:14].view(np.uint64)[0]}


@pytest.fixture(scope="module", autouse=True)
def _release_run_buffer():
    yield
    spill.release_host_arena()      # no page-locked run buffer outlives this file


@pytest.fixture(autouse=True)
def _capped_arena(monkeypatch):
    monkeypatch.setattr(settings, "device_arena_bytes", ARENA)


@pytest.fixture(params=[pytest.param("device", marks=pytest.mark.gpu), "fake"])
def engine(request):
    return request.getfixturevalue("ctx") if request.param == "device" else FakeCtx()


def kv_class(ctx):
    return FakeKV if isinstance(ctx, FakeCtx) else dev.KV


def chunks(keys, vals, step=100_003):
    """column chunks whose size is no multiple of a batch: _batches has to regroup them"""
    return ((keys[i:i + step], vals[i:i + step]) for i in range(0, len(keys), step))


def columns(pieces):
    if not pieces:
        return np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.uint64)
    return (np.concatenate([np.asarray(p[0]).view(np.uint64) for p in pieces]),
            np.concatenate([np.asarray(p[1]).view(np.uint64) for p in pieces]))


def unmix64(t):
    """the inverse of mix64 (csrc/common.cuh key_unxform, KEY_MIX)"""
    t = np.asarray(t, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        t ^= (t >> np.uint64(31)) ^ (t >> np.uint64(62))
        t *= np.uint64(0x319642B2D24D8EC3)
        t ^= (t >> np.uint64(27)) ^ (t >> np.uint64(54))
        t *= np.uint64(0x96DE1B173F119089)
        t ^= (t >> np.uint64(30)) ^ (t >> np.uint64(60))
    return t


def from_order_domain(d, xf):
    """the inverse of spill._order_domain"""
    if xf == dev.KEY_RAW:
        return d
    if xf == dev.KEY_I64:
        return d ^ np.uint64(1 << 63)
    return np.where((d >> np.uint64(63)).astype(bool), d ^ np.uint64(1 << 63), ~d)


class Spy(object):
    """Wraps spill functions and device methods with monkeypatch and records how they were called."""

    def __init__(self, monkeypatch, ctx):
        self.merge_runs, self.sort_reduce, self.depths, self.cuts, self.leases = [], [], [], [], []
        mr, srd, ext = spill._merge_runs, kv_class(ctx).sort_reduce, spill.external_sort
        take, init = spill._RunArena.take, spill._RunArena.__init__

        def merge_runs(ctx, runs, xform, op, per_batch, sec=None):
            self.merge_runs.append((sum(len(r) for r in runs), per_batch))
            return mr(ctx, runs, xform, op, per_batch, sec)

        def sort_reduce(kv, op, xform=dev.KEY_MIX, sorted_run=False):
            self.sort_reduce.append((op, sorted_run))
            return srd(kv, op, xform, sorted_run=sorted_run)

        def external_sort(ctx, chunk_iter, n_records, xform, sample_keys, _depth=0):
            self.depths.append(_depth)
            return ext(ctx, chunk_iter, n_records, xform, sample_keys, _depth)

        def arena_take(arena, kv):
            self.cuts.append((arena.reg - arena.pos, len(kv)))
            return take(arena, kv)

        def arena_init(arena, n_records, ctx=None):
            init(arena, n_records, ctx)
            self.leases.append(arena.cached)

        monkeypatch.setattr(spill, "_merge_runs", merge_runs)
        monkeypatch.setattr(kv_class(ctx), "sort_reduce", sort_reduce)
        monkeypatch.setattr(spill, "external_sort", external_sort)
        monkeypatch.setattr(spill._RunArena, "take", arena_take)
        monkeypatch.setattr(spill._RunArena, "__init__", arena_init)

    def sliced_a_bucket(self):
        return any(total > per_batch for total, per_batch in self.merge_runs)

    def straddled(self):
        return any(0 < cut < n for cut, n in self.cuts)


# ---- external_group ---------------------------------------------------------------------------------------------
def group_keys(shape, rng, n):
    """n keys drawn from one pool of raw, I64 and F64 key bits (keys_for) in the given shape"""
    pool = np.unique(np.concatenate([keys_for(xf, rng, 100_000) for xf in (dev.KEY_RAW, dev.KEY_I64, dev.KEY_F64)]))
    rng.shuffle(pool)
    if shape == "uniform":
        return pool[rng.integers(0, len(pool), size=n)]
    if shape == "zipf":
        return pool[(rng.zipf(1.2, size=n) - 1) % len(pool)]
    # one bucket: mix64 of 150 K keys in the lowest quarter of bucket 0, 40 % of the records
    per_batch = max(1 << 16, ARENA // spill.RECORD_FOOTPRINT_OVERLAPPED)
    n_buckets = int(np.ceil(1.3 * n / float(per_batch)))
    t = rng.integers(0, (1 << 64) // (4 * n_buckets), size=150_000, dtype=np.uint64)
    crafted = unmix64(t)
    assert np.array_equal(spill._mix64(crafted), t)
    keys = pool[rng.integers(0, len(pool), size=n)]
    hot = rng.random(n) < 0.4
    keys[hot] = crafted[rng.integers(0, len(crafted), size=int(hot.sum()))]
    return keys


def fsum_bounds(keys, vals):
    """4 n 2^-53 sum|v| of every key group, groups in mixed-key order"""
    o = stable_order(keys, dev.KEY_MIX)
    k, a = keys[o], np.abs(vals[o].view(np.float64))
    heads = np.flatnonzero(np.concatenate(([True], k[1:] != k[:-1])))
    return 4 * np.diff(np.append(heads, len(k))) * 2.0 ** -53 * np.add.reduceat(a, heads)


def check_group(gk, gv, keys, vals, op):
    """The spill result is one run in mixed-key order: op=None gives every record, ties in input order; a fold gives
    one record per key holding Python's fold of its values in input order."""
    if op is None:
        o = stable_order(keys, dev.KEY_MIX)
        assert np.array_equal(gk, keys[o]) and np.array_equal(gv, vals[o])
        return
    ek, ev = expected_groups(keys, vals, op, dev.KEY_MIX)
    assert np.array_equal(gk, ek)
    if op == dev.OP_SUM_F64:
        err = np.abs(gv.view(np.float64) - np.array(ev))
        assert (err <= fsum_bounds(keys, vals)).all()
    else:
        assert gv.tolist() == [int(x) for x in ev]


def by_raw_key(k, v):
    o = np.argsort(k, kind="stable")
    return k[o], v[o]


GROUP_SHAPES = ["uniform", "zipf", "one_bucket"]


@pytest.mark.parametrize("op", (None,) + ALL_OPS)
@pytest.mark.parametrize("shape", GROUP_SHAPES)
def test_external_group_every_op(engine, monkeypatch, shape, op):
    """spill.external_group of 1.2 M records: Python's fold per key, the in-core fold of the same records bit for
    bit (but OP_SUM_F64), and on the device the numpy stand-in's spill result bit for bit (but OP_SUM_F64)"""
    rng = np.random.default_rng([GROUP_SHAPES.index(shape), 99 if op is None else op])
    keys = group_keys(shape, rng, N_GROUP)
    vals = fold_values(op, rng, N_GROUP) if op is not None else np.arange(N_GROUP, dtype=np.uint64)
    spy = Spy(monkeypatch, engine)
    pieces, st = spill.external_group(engine, chunks(keys, vals), N_GROUP, op, dev.KEY_MIX)
    gk, gv = columns(pieces)
    check_group(gk, gv, keys, vals, op)
    assert st["batches"] >= 18 and st["buckets"] >= 24
    if op is not None:     # every batch is folded into a sorted run
        assert spy.sort_reduce.count((op, True)) == st["batches"]
    if shape == "one_bucket":
        assert spy.sliced_a_bucket()

    kv = engine.kv_from_columns(keys, vals)
    if op is None:
        ik, iv = kv.sort(dev.KEY_MIX).columns()
    else:
        red = kv.sort_reduce(op, dev.KEY_MIX)
        ik, iv = red.columns()
        red.free()
    kv.free()
    if op != dev.OP_SUM_F64:
        assert all(np.array_equal(a, b) for a, b in zip(by_raw_key(gk, gv), by_raw_key(ik, iv)))
        if not isinstance(engine, FakeCtx):
            fk, fv = columns(spill.external_group(FakeCtx(), chunks(keys, vals), N_GROUP, op, dev.KEY_MIX)[0])
            assert np.array_equal(gk, fk) and np.array_equal(gv, fv)


@pytest.mark.parametrize("op", (None,) + ALL_OPS)
def test_merge_runs_single_key_larger_than_a_batch(engine, monkeypatch, op):
    """_merge_runs over runs of one key that together exceed a batch: no splitter exists, so the runs are folded
    one by one and the partial folds combined (op >= 0), or handed back in run order (op = None)"""
    rng = np.random.default_rng(7 + (op or 0))
    per_batch = 1 << 16
    key = DOMINANT[dev.KEY_F64]         # a negative NaN with a payload: any 64-bit pattern is a key
    sizes = (70_000, 1, 30_000, per_batch, 5)
    vals = fold_values(op, rng, sum(sizes)) if op is not None else np.arange(sum(sizes), dtype=np.uint64)
    edges = np.cumsum((0,) + sizes)
    runs = [np.stack((np.full(b - a, key, dtype=np.uint64), vals[a:b]), axis=1) for a, b in zip(edges[:-1], edges[1:])]
    merges = []
    monkeypatch.setattr(engine, "kv_merge_ranges", lambda *a: merges.append(a))
    k, v = columns(spill._merge_runs(engine, runs, dev.KEY_MIX, -1 if op is None else op, per_batch))
    assert not merges
    assert (k == key).all()
    if op is None:
        assert np.array_equal(v, vals)
        return
    assert len(k) == 1
    if op == dev.OP_SUM_F64:
        a = vals.view(np.float64)
        assert abs(v.view(np.float64)[0] - py_fold(op, vals)) <= 4 * len(a) * 2.0 ** -53 * float(np.abs(a).sum())
    else:
        assert int(v[0]) == py_fold(op, vals)


# ---- external_sort ----------------------------------------------------------------------------------------------
def sort_case(xf, shape, rng, n):
    """(keys, sample keys) of one external_sort input"""
    if shape == "uniform":
        keys = keys_for(xf, rng, n)
    elif shape == "ties":
        keys = keys_for(xf, rng, 40)[rng.integers(0, 40, size=n)]
    elif shape == "dominant":
        keys = keys_for(xf, rng, n)
        keys[rng.random(n) < 0.7] = DOMINANT[xf]
    else:
        # half the records in a band of 10 K neighbouring keys the sample never sees: their range has to be split
        # again on a sample of its own keys
        start = np.array([-1e10]).view(np.uint64) if xf == dev.KEY_F64 else np.array([12345 << 20], dtype=np.uint64)
        d0 = spill._order_domain(start, xf)[0]
        band = from_order_domain(d0 + rng.integers(0, 10_000, size=n // 2).astype(np.uint64), xf)
        assert (spill._order_domain(band, xf) - d0 < 10_000).all()
        other = keys_for(xf, rng, n - n // 2)
        keys = np.concatenate((band, other))
        rng.shuffle(keys)
        return keys, other[rng.integers(0, len(other), size=1 << 16)]
    if xf == dev.KEY_F64:
        keys[rng.integers(0, n, size=64)] = F64_SPECIAL.view(np.uint64)[rng.integers(0, len(F64_SPECIAL), size=64)]
    return keys, keys[rng.integers(0, n, size=1 << 16)]


@pytest.mark.parametrize("shape", ["uniform", "ties", "dominant", "resplit"])
@pytest.mark.parametrize("xf", [dev.KEY_I64, dev.KEY_F64, dev.KEY_RAW])
def test_external_sort_key_shapes(engine, monkeypatch, xf, shape):
    """spill.external_sort of 1 M records with the input position as value: numpy's stable argsort of the order
    domain, bit for bit. A range larger than a batch is split again on a sample of its own keys; at 16 levels it is
    merged whole, past the arena cap, so the re-splits must end well before that."""
    rng = np.random.default_rng(31 * xf + len(shape))
    keys, samp = sort_case(xf, shape, rng, N_SORT)
    vals = np.arange(N_SORT, dtype=np.uint64)
    spy = Spy(monkeypatch, engine)
    pieces, st = spill.external_sort(engine, chunks(keys, vals), N_SORT, xf, samp)
    sk, sv = columns(pieces)
    o = stable_order(keys, xf)
    assert np.array_equal(sk, keys[o]) and np.array_equal(sv, o.astype(np.uint64))
    assert st["batches"] >= 16
    assert max(spy.depths) < 16
    if shape == "resplit":
        assert max(spy.depths) >= 1
    if shape == "dominant":
        # the range that holds nothing but the dominant key is handed back run by run
        only = [p for p in pieces if len(p[0]) and (np.asarray(p[0]).view(np.uint64) == DOMINANT[xf]).all()]
        assert len(only) >= 2 and sum(len(p[0]) for p in only) == int((keys == DOMINANT[xf]).sum())


# ---- the run buffer kept between jobs ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_run_buffer_reused_across_jobs(ctx, monkeypatch):
    """Three jobs on one context share the cached host run buffer. A folds 1.2 M records and spills fewer, after
    which the prefix it wrote is page-locked in the background; B spills a size between A's spilled count and the
    buffer, so its runs straddle the page-locked prefix and are downloaded in two pieces; C is a sort whose skewed
    range is split again while the buffer is leased, so the nested job gets a buffer of its own."""
    spill.release_host_arena()
    spy = Spy(monkeypatch, ctx)
    rng = np.random.default_rng(99)
    pool = keys_for(dev.KEY_I64, rng, 20_000)
    ka = pool[rng.integers(0, len(pool), size=N_GROUP)]
    va = fold_values(dev.OP_SUM_I64, rng, N_GROUP)
    pieces, st = spill.external_group(ctx, chunks(ka, va), N_GROUP, dev.OP_SUM_I64, dev.KEY_MIX)
    check_group(*columns(pieces), ka, va, dev.OP_SUM_I64)
    spilled_a = st["spilled_bytes"] // 16
    assert spilled_a < N_GROUP and spy.leases == [True] and not spy.straddled()

    n_b = (spilled_a + N_GROUP) // 2
    kb = group_keys("uniform", rng, n_b)
    vb = np.arange(n_b, dtype=np.uint64)
    del spy.cuts[:]
    pieces, st = spill.external_group(ctx, chunks(kb, vb), n_b, None, dev.KEY_MIX)
    check_group(*columns(pieces), kb, vb, None)
    assert spill._HOST_ARENA["chunks"][:1] == [(0, spilled_a)]       # A's prefix was page-locked before B ran
    assert spy.leases == [True, True] and spy.straddled()

    keys, samp = sort_case(dev.KEY_F64, "resplit", rng, N_SORT)
    vals = np.arange(N_SORT, dtype=np.uint64)
    del spy.cuts[:]
    pieces, st = spill.external_sort(ctx, chunks(keys, vals), N_SORT, dev.KEY_F64, samp)
    o = stable_order(keys, dev.KEY_F64)
    sk, sv = columns(pieces)
    assert np.array_equal(sk, keys[o]) and np.array_equal(sv, o.astype(np.uint64))
    assert max(spy.depths) >= 1 and spy.leases[2] is True and False in spy.leases[3:]
    assert spy.straddled()


# ---- through the DSL --------------------------------------------------------------------------------------------
def spilled():
    from dampr_b200 import runner as runner_mod
    return any("[spilled:" in how for _s, how, _d in runner_mod.LAST_STATS.stages)


def py_groups(keys, vals):
    out = {}
    for k, v in zip(keys.tolist(), vals.tolist()):
        out.setdefault(k, []).append(v)
    return out


@pytest.mark.gpu
def test_dsl_pipelines_that_spill(ctx):
    """keyed folds, counts, means, grouped value lists and a float sort_by over ArrayKVInput with the capped arena:
    every one spills, and agrees with plain Python over the same rows"""
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    rng = np.random.default_rng(5)
    n = 600_000
    keys = rng.integers(0, 60_000, size=n).astype(np.int64)
    ints = rng.integers(-10 ** 12, 10 ** 12, size=n).astype(np.int64)
    floats = fold_values(dev.OP_MIN_F64, rng, n).view(np.float64)          # +-inf and subnormals, no NaN or -0.0
    finite = fold_values(dev.OP_SUM_F64, rng, n).view(np.float64)
    pick = {"sum": lambda g: sum(g), "min": min, "max": max, "first": lambda g: g[0], "last": lambda g: g[-1]}
    for vals in (ints, floats):
        src = Dampr.read_input(ArrayKVInput(keys, vals))
        grouped = src.a_group_by(lambda x: x[0], lambda x: x[1])
        exp = py_groups(keys, vals)
        pipes = {"min": grouped.reduce(min), "max": grouped.reduce(max), "first": grouped.first(),
                 "last": grouped.reduce(lambda a, b: b)}
        if vals is ints:
            pipes["sum"] = grouped.sum()
        for name, pipe in pipes.items():
            got = dict(pipe.read())
            assert spilled(), name
            want = {k: pick[name](g) for k, g in exp.items()}
            assert got.keys() == want.keys()
            assert all(np.float64(got[k]).view(np.uint64) == np.float64(want[k]).view(np.uint64)
                       if vals is floats else got[k] == want[k] for k in want), name

    # float sums: a_group_by().sum() and fold_by with a float +, within 4 n 2^-53 sum|v| of math.fsum
    src = Dampr.read_input(ArrayKVInput(keys, finite))
    exp = py_groups(keys, finite)
    for pipe in (src.a_group_by(lambda x: x[0], lambda x: x[1]).sum(),
                 src.fold_by(lambda x: x[0], lambda a, b: a + b, lambda x: x[1])):
        got = dict(pipe.read())
        assert spilled() and got.keys() == exp.keys()
        for k, g in exp.items():
            assert abs(got[k] - math.fsum(g)) <= 4 * len(g) * 2.0 ** -53 * sum(abs(x) for x in g), k

    got = dict(Dampr.read_input(ArrayKVInput(keys, ints)).count(lambda x: x[0]).read())
    assert spilled() and got == {k: len(g) for k, g in py_groups(keys, ints).items()}

    got = dict(Dampr.read_input(ArrayKVInput(keys, ints)).mean(lambda x: x[0], lambda x: x[1]).read())
    assert spilled() and got == {k: sum(g) / float(len(g)) for k, g in py_groups(keys, ints).items()}
    got = dict(src.mean(lambda x: x[0], lambda x: x[1]).read())
    assert spilled() and got.keys() == exp.keys()
    for k, g in exp.items():
        assert abs(got[k] - math.fsum(g) / len(g)) <= 4 * 2.0 ** -53 * sum(abs(x) for x in g) + 2.0 ** -52 * abs(got[k])

    # grouped value lists with a dominant key: the spill sort keeps every group's values in input order
    dom = np.where(rng.random(n) < 0.6, 7, keys).astype(np.int64)
    got = dict(Dampr.read_input(ArrayKVInput(dom, ints)).group_by(lambda x: x[0], lambda x: x[1])
               .reduce(lambda k, it: list(it)).read())
    assert getattr(runner_mod.LAST_STATS, "spill", None) is not None
    assert got == py_groups(dom, ints)

    # sort_by on a float field with +-0.0 and +-inf: Python's stable order, in which -0.0 and 0.0 tie
    fv = finite.copy()
    for x in (0.0, -0.0, np.inf, -np.inf):
        fv[rng.random(n) < 0.02] = x
    rows = list(zip(keys.tolist(), fv.tolist()))
    got = Dampr.read_input(ArrayKVInput(keys, fv)).sort_by(lambda x: x[1]).read()
    assert spilled()
    want = sorted(rows, key=lambda r: r[1])
    assert [r[0] for r in got] == [r[0] for r in want]
    assert np.array_equal(np.array([r[1] for r in got]).view(np.uint64), np.array([r[1] for r in want]).view(np.uint64))

"""GPU: OP_SUM_F64, the fold behind every float sum(), mean() and fold_by(..., lambda a, b: a + b) on the device, bit
for bit against Python's left fold of each group's values in input order (np.cumsum(...)[-1], never np.sum, which
sums pairwise).

Exact families. On these values every order of addition gives the same bits, so every path must equal the left
fold exactly, whatever order it adds in:
- integer-valued doubles whose partial sums stay below 2^53, dyadic values m * 2^-e whose partial sums are exact,
  and multiples of the smallest subnormal: every partial sum is exact, so no addition rounds;
- -0.0 alone, and -0.0 among +0.0 and exact values: in round-to-nearest a sum is -0.0 only when every term is -0.0;
- +-inf and NaN among exact values: one sign of infinity gives that infinity, both give NaN, a NaN gives NaN, in
  any order, as long as no finite partial sum overflows. NaNs are compared with isnan, not by their bits.
They run through dampr_kv_sort_reduce under every key transform, dampr_kv_reduce_by_key, the k-way merges and the
spill path, at 1, 4095, 4096, 4097, 50 000 and 10^6 records per key, alone and among many small keys, and through
the DSL paths that reach SUM_F64: runner._combine, plan._fold_column and the field scan's record mode.

Fold order. On values from 1e-8 to 1e8 of both signs the order matters, and the order each path uses is stated here
as Python and compared bit for bit:
- sort_reduce folds a key of at most 4096 records left to right in input order, in one leaf;
- a larger key, or the only key of the input under KEY_RAW, KEY_I64 or KEY_F64 (the key range is empty, so nothing is
  partitioned), goes to single_group_reduce_kernel: 1024 threads each fold their strided records left to right,
  every warp combines its lanes with shuffle-down steps 16, 8, 4, 2, 1, and thread 0 adds the 32 warp sums in order;
- reduce_by_key folds each 4096-record tile of the run left to right, then a key's tile sums left to right;
- a field-scan key of at most 4096 lines is folded in line order.
Merges and the spill path cut at sampled keys and batch sizes, so for them the test checks the bound
4 n 2^-53 sum|v| around math.fsum and that the same call gives the same bits twice."""
import functools
import math
import operator
import struct

import numpy as np
import pytest

from dampr_b200 import device as dev
from dampr_b200 import settings, spill
from test_gpu_key_orders import nan_with, stable_order
from test_gpu_spill import chunks, columns

pytestmark = pytest.mark.gpu

LEAF = 4096            # records of one leaf CTA and of one reduce_by_key tile (csrc/leaf.cuh L_CAP)
THREADS = 1024         # single_group_reduce_kernel's CTA (csrc/kv.cu sort_range)
SIZES = (1, 4095, 4096, 4097, 50_000, 1_000_000)
LAYOUTS = ("alone", "among")
FAMILIES = ("int", "dyadic", "subnormal", "negzero", "zeros", "posinf", "neginf", "bothinf", "nan")
XFORMS = (dev.KEY_RAW, dev.KEY_MIX, dev.KEY_I64, dev.KEY_F64)
MERGE_XF = {1: dev.KEY_RAW, 2: dev.KEY_I64, 8: dev.KEY_F64, 70: dev.KEY_MIX}   # 70 runs: more than one merge pass takes
ARENA = 4 << 20        # the capped spill arena: 65 536 records per batch


@pytest.fixture(scope="module", autouse=True)
def _release_run_buffer():
    yield
    spill.release_host_arena()


@pytest.fixture
def capped_arena(monkeypatch):
    monkeypatch.setattr(settings, "device_arena_bytes", ARENA)


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    yield
    plan.release_buffers()


# ---- references -------------------------------------------------------------------------------------------------
def left_fold(v):
    with np.errstate(invalid="ignore"):      # inf + -inf
        return float(np.cumsum(v)[-1])


def combine(a, b):
    """two partial sums of the tree, None where a partial holds no record"""
    if a is None:
        return b
    return a if b is None else a + b


def tree_fold(v):
    """single_group_reduce_kernel: thread t folds v[t], v[t + 1024], ... left to right; lane i of a warp adds lane
    i + d for d = 16, 8, 4, 2, 1; thread 0 adds the warp sums in warp order. Empty partials are skipped."""
    n = len(v)
    rows = -(-n // THREADS)
    m = np.zeros(rows * THREADS)
    m[:n] = v
    acc = np.add.accumulate(m.reshape(rows, THREADS), axis=0)     # column t: thread t's running sum
    part = [float(acc[(n - 1 - t) // THREADS, t]) if t < n else None for t in range(THREADS)]
    total = None
    for w in range(THREADS // 32):
        lane = part[32 * w:32 * w + 32]
        for d in (16, 8, 4, 2, 1):
            for i in range(d):
                lane[i] = combine(lane[i], lane[i + d])
        total = combine(total, lane[0])
    return total


def tiled_fold(v, start):
    """reduce_by_key of a key whose records v sit at run positions start, start + 1, ...: each 4096-record tile of
    the run is folded left to right, then the key's tile sums left to right"""
    cuts = [0] + [t - start for t in range((start // LEAF + 1) * LEAF, start + len(v), LEAF)] + [len(v)]
    return functools.reduce(operator.add, [left_fold(v[a:b]) for a, b in zip(cuts[:-1], cuts[1:])])


def same(got, want):
    if isinstance(want, float) and math.isnan(want):
        return isinstance(got, float) and math.isnan(got)
    return struct.pack("<d", got) == struct.pack("<d", want)


# ---- data -------------------------------------------------------------------------------------------------------
def key_codes(xf, G):
    """G distinct keys valid under xf: floats (never +-0.0) for KEY_F64, signed ints for KEY_I64, raw bits else"""
    g = np.arange(G, dtype=np.int64)
    if xf == dev.KEY_F64:
        return ((g - G // 2) * 0.75 + 0.125).view(np.uint64)
    if xf == dev.KEY_I64:
        return ((g - G // 2) * 1_000_003).view(np.uint64)
    return (g.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) ^ np.uint64(0x5DEECE66D)


class Groups(object):
    """records in input order: a group id and a value each; want[g] is the left fold of group g in input order"""

    def __init__(self, gid, vals):
        self.gid, self.vals = gid, vals
        self.G = int(gid.max()) + 1
        o = np.argsort(gid, kind="stable")
        bounds = np.searchsorted(gid[o], np.arange(self.G + 1))
        self.members = [o[a:b] for a, b in zip(bounds[:-1], bounds[1:])]
        self.want = [left_fold(vals[m]) for m in self.members]

    def keys(self, xf):
        return key_codes(xf, self.G)[self.gid]

    def check(self, gk, gv, xf, what):
        pos = {k: g for g, k in enumerate(key_codes(xf, self.G).tolist())}
        assert len(gk) == self.G and len(set(gk.tolist())) == self.G, what
        got = [None] * self.G
        for k, v in zip(gk.tolist(), gv.view(np.float64).tolist()):
            got[pos[k]] = v
        bad = [(g, got[g], self.want[g]) for g in range(self.G) if not same(got[g], self.want[g])]
        assert not bad, (what, len(bad), bad[:4])


def group_ids(layout, size, rng):
    """group 0 holds `size` records; among: 500 more groups of 1-11 records, all shuffled together"""
    if layout == "alone":
        return np.zeros(size, dtype=np.int64)
    gid = np.concatenate((np.zeros(size, dtype=np.int64), np.repeat(np.arange(1, 501), rng.integers(1, 12, size=500))))
    rng.shuffle(gid)
    return gid


SPECIALS = {"posinf": [np.inf], "neginf": [-np.inf], "bothinf": [np.inf, -np.inf], "nan": [nan_with(1, 7), np.nan]}


def exact_values(family, rng, gid):
    n = len(gid)
    ints = rng.integers(-2 ** 20, 2 ** 20, size=n).astype(np.float64)      # |partial sums| < 2^40
    if family == "int":
        return ints
    if family == "dyadic":      # multiples of 2^-20 below 2^12: |partial sums| < 2^32, so 52 bits hold them
        return np.ldexp(rng.integers(-2 ** 12, 2 ** 12, size=n).astype(np.float64), -rng.integers(0, 21, size=n))
    if family == "subnormal":   # multiples of 2^-1074 below 2^-1044
        return np.ldexp(rng.integers(-2 ** 30, 2 ** 30, size=n).astype(np.float64), -1074)
    if family == "negzero":
        return np.full(n, -0.0)
    if family == "zeros":       # group 0: +-0.0 only; the small groups also exact values
        v = np.where(rng.random(n) < 0.8, -0.0, 0.0)
        mixed = (gid != 0) & (rng.random(n) < 0.2)
        v[mixed] = ints[mixed]
        return v
    v = ints.copy()
    sp = np.array(SPECIALS[family])
    hit = rng.random(n) < 1e-3
    v[hit] = sp[rng.integers(0, len(sp), size=int(hit.sum()))]
    first, last = np.flatnonzero(gid == 0)[[0, -1]]
    v[first], v[last] = sp[0], sp[-1]
    return v


@functools.lru_cache(maxsize=16)
def exact_groups(family, size, layout):
    rng = np.random.default_rng([FAMILIES.index(family), size, LAYOUTS.index(layout)])
    gid = group_ids(layout, size, rng)
    return Groups(gid, exact_values(family, rng, gid))


def every_exact_case(family, sizes=SIZES):
    for size in sizes:
        for layout in LAYOUTS:
            yield (size, layout), exact_groups(family, size, layout)


# ---- device calls -----------------------------------------------------------------------------------------------
def sort_reduce(ctx, keys, vals, xf):
    kv = ctx.kv_from_columns(keys, vals.view(np.uint64))
    out = kv.sort_reduce(dev.OP_SUM_F64, xf)
    gk, gv = out.columns()
    out.free()
    kv.free()
    return gk, gv


def reduce_by_key(ctx, keys, vals):
    kv = ctx.kv_from_columns(keys, vals.view(np.uint64))
    out = kv.reduce_by_key(dev.OP_SUM_F64)
    gk, gv = out.columns()
    out.free()
    kv.free()
    return gk, gv


def merges(ctx, keys, vals, k, xf):
    """the records cut into k consecutive pieces of the input, each sorted stably under xf: a key's records come out
    of the merge in input order. Returns the folds of dampr_kv_merge and of dampr_kv_merge_ranges."""
    vals = vals.view(np.uint64)
    edges = np.linspace(0, len(keys), k + 1).astype(np.int64)
    runs = []
    for a, b in zip(edges[:-1], edges[1:]):
        o = stable_order(keys[a:b], xf)
        runs.append((keys[a:b][o], vals[a:b][o]))
    dev_runs = [ctx.kv_from_columns(a, b) for a, b in runs]
    flat = ctx.kv_from_columns(np.concatenate([r[0] for r in runs]), np.concatenate([r[1] for r in runs]))
    outs = [ctx.kv_merge(dev_runs, xf, dev.OP_SUM_F64), ctx.kv_merge_ranges(flat, edges.astype(np.uint64), xf,
                                                                             dev.OP_SUM_F64)]
    res = []
    for out in outs:
        res.append(out.columns())
        out.free()
    for x in dev_runs + [flat]:
        x.free()
    return res


def external_group(ctx, keys, vals):
    pieces, st = spill.external_group(ctx, chunks(keys, vals.view(np.uint64)), len(keys), dev.OP_SUM_F64, dev.KEY_MIX)
    return columns(pieces), st


# ---- a. exact families through the kernels ----------------------------------------------------------------------
@pytest.mark.parametrize("family", FAMILIES)
def test_sort_reduce_exact(ctx, family):
    for case, d in every_exact_case(family):
        for xf in XFORMS:
            d.check(*sort_reduce(ctx, d.keys(xf), d.vals, xf), xf, (case, xf))


@pytest.mark.parametrize("family", FAMILIES)
def test_reduce_by_key_exact(ctx, family):
    for case, d in every_exact_case(family):
        keys = d.keys(dev.KEY_RAW)
        o = stable_order(keys, dev.KEY_RAW)
        d.check(*reduce_by_key(ctx, keys[o], d.vals[o]), dev.KEY_RAW, case)


@pytest.mark.parametrize("family", FAMILIES)
def test_merges_exact(ctx, family):
    """group 0 of 10^6 records spans hundreds of merge partitions"""
    for case, d in every_exact_case(family):
        for k, xf in MERGE_XF.items():
            for i, (gk, gv) in enumerate(merges(ctx, d.keys(xf), d.vals, k, xf)):
                d.check(gk, gv, xf, (case, k, ("merge", "merge_ranges")[i]))


@pytest.mark.parametrize("family", FAMILIES)
def test_spill_exact(ctx, capped_arena, family):
    for case, d in every_exact_case(family):
        (gk, gv), st = external_group(ctx, d.keys(dev.KEY_MIX), d.vals)
        d.check(gk, gv, dev.KEY_MIX, case)
        if case[0] == 1_000_000:      # group 0 is larger than a batch
            assert st["batches"] >= 15, st


# ---- b. the DSL paths that reach SUM_F64 ------------------------------------------------------------------------
def stage_paths():
    from dampr_b200 import runner as runner_mod
    return [how for _s, how, _d in runner_mod.LAST_STATS.stages]


def assert_dict(got, want, what):
    assert sorted(got) == sorted(want), what
    bad = [(k, got[k], w) for k, w in want.items() if not same(got[k], w)]
    assert not bad, (what, len(bad), bad[:4])


@pytest.mark.parametrize("family", FAMILIES)
def test_host_map_combine_exact(ctx, monkeypatch, family):
    """Dampr.memory input: the map runs on the host, runner._combine folds the values with sort_reduce(KEY_RAW)"""
    from dampr_b200 import Dampr
    calls = []
    real = dev.KV.sort_reduce

    def spy(kv, op, xform=dev.KEY_MIX, sorted_run=False):
        calls.append(op)
        return real(kv, op, xform, sorted_run)
    monkeypatch.setattr(dev.KV, "sort_reduce", spy)
    for case, d in every_exact_case(family, (1, 4097, 50_000)):
        recs = list(zip(d.gid.tolist(), d.vals.tolist()))
        want = dict(enumerate(d.want))
        for pipe in (Dampr.memory(recs).a_group_by(lambda x: x[0], lambda x: x[1]).sum(),
                     Dampr.memory(recs).fold_by(lambda x: x[0], lambda a, b: a + b, lambda x: x[1])):
            del calls[:]
            got = dict(pipe.read())
            assert "host-map + device shuffle/combine" in stage_paths() and dev.OP_SUM_F64 in calls, case
            assert_dict(got, want, case)


@pytest.mark.parametrize("family", FAMILIES)
def test_kv_input_and_frame_folds_exact(ctx, family):
    """binary kv input: fold_by, a_group_by().sum() and mean() through plan._fold_column; then a fold of a frame
    that an aggregation made"""
    from dampr_b200 import Dampr
    from dampr_b200.inputs import ArrayKVInput
    frame_fold = "frame keyed fold: columns evaluated on the host, groups folded on the device"
    for case, d in every_exact_case(family, (1, 4097, 1_000_000)):
        src = Dampr.read_input(ArrayKVInput(d.gid, d.vals))
        want = dict(enumerate(d.want))
        for pipe in (src.fold_by(lambda x: x[0], lambda a, b: a + b, lambda x: x[1]),
                     src.a_group_by(lambda x: x[0], lambda x: x[1]).sum()):
            got = dict(pipe.read())
            assert frame_fold in stage_paths(), case
            assert_dict(got, want, case)
        got = dict(src.mean(lambda x: x[0], lambda x: x[1]).read())
        assert frame_fold in stage_paths(), case
        assert_dict(got, {g: w / float(len(m)) for g, (w, m) in enumerate(zip(d.want, d.members))}, case)
        # one record per key, then the frame folded by residue
        idx = np.arange(len(d.vals), dtype=np.int64)
        got = dict(Dampr.read_input(ArrayKVInput(idx, d.vals)).a_group_by(lambda x: x[0], lambda x: x[1]).sum()
                   .fold_by(lambda x: x[0] % 7, lambda a, b: a + b, lambda x: x[1]).read())
        assert stage_paths().count(frame_fold) == 2, case
        assert_dict(got, {r: left_fold(d.vals[r::7]) for r in range(min(7, len(d.vals)))}, case)


def field_text(d, path):
    with open(path, "w") as f:
        f.write("".join("k%d,%r\n" % (g, v) for g, v in zip(d.gid.tolist(), d.vals.tolist())))


NEEDLE = "device text fields scan+combine"


@pytest.mark.parametrize("family", [f for f in FAMILIES if f not in ("negzero", "zeros")])
def test_field_scan_exact(ctx, engine, tmp_path, family):
    """float(l.split(',')[1]) with repr spellings: sum() and mean() by key in record mode, and mean() of the
    default key. 'inf' and 'nan' lines go to the host by design and are merged with the device's sums. A parsed
    -0.0 sends the whole stage to the host (Python's min / max depend on the order), so the families with -0.0
    are not field-scan cases."""
    from dampr_b200 import Dampr
    P = str(tmp_path / "v.csv")
    for case, d in every_exact_case(family, (4097, 50_000)):
        field_text(d, P)
        want = {"k%d" % g: w for g, w in enumerate(d.want)}
        got = dict(Dampr.text(P).a_group_by(lambda l: l.split(",")[0], lambda l: float(l.split(",")[1])).sum().read())
        assert NEEDLE in stage_paths()[0], (case, stage_paths())
        assert_dict(got, want, case)
        got = dict(Dampr.text(P).map(lambda l: l.split(",")).mean(lambda r: r[0], lambda r: float(r[1])).read())
        assert NEEDLE in stage_paths()[0], (case, stage_paths())
        assert_dict(got, {"k%d" % g: w / float(len(m)) for g, (w, m) in enumerate(zip(d.want, d.members))}, case)
        if case[1] == "alone":
            got = dict(Dampr.text(P).map(lambda l: float(l.split(",")[1])).mean().read())
            assert NEEDLE in stage_paths()[0], (case, stage_paths())
            assert_dict(got, {1: d.want[0] / float(len(d.vals))}, case)


# ---- c. the fold order ------------------------------------------------------------------------------------------
def order_values(rng, n):
    """magnitudes from 1e-8 to 1e8, both signs: the order of addition changes the result"""
    return rng.choice([-1.0, 1.0], size=n) * 10.0 ** rng.uniform(-8, 8, size=n)


def assert_order_matters(d, groups):
    """reversing a group changes its left fold for most of `groups`: a result in another order would be caught"""
    changed = sum(left_fold(d.vals[d.members[g]]) != left_fold(d.vals[d.members[g]][::-1]) for g in groups)
    assert changed >= 0.75 * len(groups), (changed, len(groups))


def order_groups(seed, sizes):
    rng = np.random.default_rng(seed)
    gid = np.repeat(np.arange(len(sizes)), sizes)
    rng.shuffle(gid)
    return Groups(gid, order_values(rng, len(gid)))


@pytest.mark.parametrize("xf", XFORMS)
def test_sort_reduce_fold_order(ctx, xf):
    """keys of up to 4096 records among others: the left fold in input order; larger keys: the strided tree"""
    rng = np.random.default_rng(3)
    sizes = np.concatenate((rng.integers(64, LEAF + 1, size=150), [1, 2, 3, LEAF - 1, LEAF, LEAF + 1, 50_000]))
    d = order_groups(11 + xf, sizes)
    assert_order_matters(d, [g for g in range(d.G) if sizes[g] >= 64])
    d.want = [left_fold(d.vals[m]) if len(m) <= LEAF else tree_fold(d.vals[m]) for m in d.members]
    assert all(d.want[g] != left_fold(d.vals[d.members[g]]) for g in range(d.G) if sizes[g] > LEAF)
    d.check(*sort_reduce(ctx, d.keys(xf), d.vals, xf), xf, xf)


@pytest.mark.parametrize("xf", XFORMS)
def test_sort_reduce_lone_key_fold_order(ctx, xf):
    """the input's only key: under KEY_MIX one leaf folds up to 4096 records left to right; otherwise the key range
    is empty and single_group_reduce_kernel folds every size, down to one record, by the strided tree"""
    for n in (1, 2, 33, 1000, LEAF, LEAF + 1, 50_000, 1_000_000):
        d = order_groups(n, [n])
        v = d.vals
        if n >= 1000:
            assert tree_fold(v) != left_fold(v) and left_fold(v) != left_fold(v[::-1]), n
        want = left_fold(v) if (xf == dev.KEY_MIX and n <= LEAF) else tree_fold(v)
        gk, gv = sort_reduce(ctx, d.keys(xf), v, xf)
        assert len(gk) == 1 and same(gv.view(np.float64)[0], want), (n, xf, gv.view(np.float64)[0], want)


def test_reduce_by_key_fold_order(ctx):
    """the keys of a sorted run start at offsets that are no multiple of 4096, so the tiles cut them unevenly"""
    sizes = [1234, LEAF + 1, 3, 8191, 100_000, 77, LEAF, 300_000]
    rng = np.random.default_rng(5)
    vals = order_values(rng, sum(sizes))
    keys = np.repeat(key_codes(dev.KEY_RAW, len(sizes)), sizes)
    gk, gv = reduce_by_key(ctx, keys, vals)
    assert np.array_equal(gk, key_codes(dev.KEY_RAW, len(sizes)))
    starts = np.concatenate(([0], np.cumsum(sizes)[:-1]))
    for g, (s, n) in enumerate(zip(starts.tolist(), sizes)):
        v = vals[s:s + n]
        want = tiled_fold(v, s)
        if n > LEAF:
            assert want != left_fold(v) and left_fold(v) != left_fold(v[::-1]), g
        assert same(gv.view(np.float64)[g], want), (g, n, gv.view(np.float64)[g], want)


def test_field_scan_fold_order(ctx, engine, tmp_path):
    """keys of up to 4096 lines: sum() and mean() equal the left fold in line order"""
    from dampr_b200 import Dampr
    rng = np.random.default_rng(8)
    sizes = rng.integers(64, LEAF + 1, size=60)
    sizes[:2] = LEAF - 1, LEAF
    d = order_groups(9, sizes)
    assert_order_matters(d, range(d.G))
    P = str(tmp_path / "v.csv")
    field_text(d, P)
    got = dict(Dampr.text(P).a_group_by(lambda l: l.split(",")[0], lambda l: float(l.split(",")[1])).sum().read())
    assert NEEDLE in stage_paths()[0], stage_paths()
    assert_dict(got, {"k%d" % g: w for g, w in enumerate(d.want)}, "sum")
    got = dict(Dampr.text(P).map(lambda l: l.split(",")).mean(lambda r: r[0], lambda r: float(r[1])).read())
    assert NEEDLE in stage_paths()[0], stage_paths()
    assert_dict(got, {"k%d" % g: w / float(len(m)) for g, (w, m) in enumerate(zip(d.want, d.members))}, "mean")


def test_merges_and_spill_bound_and_repeat(ctx, capped_arena):
    """order-sensitive values through the merges and the spill path: within 4 n 2^-53 sum|v| of math.fsum, and the
    same bits from the same call twice"""
    rng = np.random.default_rng(13)
    sizes = np.concatenate((rng.integers(1, 2000, size=300), [LEAF + 1, 50_000, 700_000]))
    d = order_groups(14, sizes)
    fsum = [math.fsum(d.vals[m].tolist()) for m in d.members]
    bound = [4 * len(m) * 2.0 ** -53 * float(np.abs(d.vals[m]).sum()) for m in d.members]

    def check(gk, gv, xf, what):
        pos = {k: g for g, k in enumerate(key_codes(xf, d.G).tolist())}
        assert len(gk) == d.G, what
        for k, v in zip(gk.tolist(), gv.view(np.float64).tolist()):
            g = pos[k]
            assert abs(v - fsum[g]) <= bound[g], (what, g, v, fsum[g])

    for k, xf in MERGE_XF.items():
        first = merges(ctx, d.keys(xf), d.vals, k, xf)
        again = merges(ctx, d.keys(xf), d.vals, k, xf)
        for i, ((gk, gv), (gk2, gv2)) in enumerate(zip(first, again)):
            check(gk, gv, xf, (k, i))
            assert np.array_equal(gk, gk2) and np.array_equal(gv, gv2), (k, i)
    (gk, gv), st = external_group(ctx, d.keys(dev.KEY_MIX), d.vals)
    (gk2, gv2), _ = external_group(ctx, d.keys(dev.KEY_MIX), d.vals)
    assert st["batches"] >= 15, st
    check(gk, gv, dev.KEY_MIX, "spill")
    assert np.array_equal(gk, gk2) and np.array_equal(gv, gv2)

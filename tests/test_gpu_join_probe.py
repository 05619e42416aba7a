"""The broadcast hash probe and join (dampr_kv_hash_probe / dampr_kv_hash_join), the merge-join ranges
(dampr_kv_join_ranges) and the count dictionary (dampr_count_dictionary) through the C ABI, against plain Python:
dict lookups, the key groups of sorted numpy columns, oracle.refsem's joins and the host's unique_inverse_rows.

The shapes sit on the kernels' seams: probe tables of 1 024 and 2 048 slots (build sides of 511, 512 and 513 keys)
and of 2^21 slots (10^6 keys); build chains that start at slot cap - 3 and wrap past the last slot; probe sides
around the 8-flag words and the 4 096-record tiles of the hit compaction, and of more than 1 024 tiles, where the
single-block tile scan (scan_tiles_kernel) carries its running total from one pass to the next; left sides of more
than 1 024 tiles of 4 096 records with group heads on tile starts; a count column of 2^21 + 1 rows, whose presence
table is at its 2^22 cap with four block counts per thread of the block scan (dict_scan_kernel)."""
import numpy as np
import pytest

from dampr_b200 import device as dev
from dampr_b200 import plan
from dampr_b200 import spill
from oracle import refsem
from test_gpu_spill import unmix64
from test_gpu_tfidf_tail import check as check_dictionary

pytestmark = pytest.mark.gpu

SPECIAL = np.array([0, 1, 1 << 63, (1 << 64) - 1], dtype=np.uint64)
TILE = 4096
PATTERNS = ("none", "all", "alternating", "last", "tile-heads")


def table_slots(n_build):
    cap = 1024
    while cap < 2 * n_build:
        cap <<= 1
    return cap


def build_keys(n, rng):
    """n distinct keys, the special ones (0, 1, 2^63, 2^64 - 1) among them, in no order"""
    special = SPECIAL[:n]
    rest = np.unique(rng.integers(2, (1 << 63) - 1, size=n + n // 8 + 16, dtype=np.int64).view(np.uint64))
    rest = rest[~np.isin(rest, SPECIAL)][:n - len(special)]
    keys = np.concatenate((special, rest + np.uint64(1 << 63) * (rng.random(len(rest)) < 0.5)))
    assert len(np.unique(keys)) == n
    return rng.permutation(keys)


def absent_keys(n, present, rng):
    """n keys (with repeats) none of which is in `present`"""
    k = rng.integers(0, 1 << 62, size=n + 64, dtype=np.int64).view(np.uint64) | np.uint64(1 << 62)
    k = k[~np.isin(k, present)]
    return k[rng.integers(0, len(k), size=n)] if n else k[:0]


def hit_pattern(name, n):
    i = np.arange(n)
    return {"none": np.zeros(n, dtype=bool), "all": np.ones(n, dtype=bool), "alternating": i % 2 == 0,
            "last": i == n - 1, "tile-heads": i % TILE == 0}[name]


def probe_side(bk, want, absent, rng):
    """probe keys: a build key (drawn at random) where `want`, otherwise one of `absent`"""
    pk = absent[rng.integers(0, len(absent), size=len(want))] if len(absent) else np.zeros(len(want), np.uint64)
    if len(bk):
        pk[want] = bk[rng.integers(0, len(bk), size=int(want.sum()))]
    return pk


def expected(bk, bv, pk):
    """Python's dict of the build side: hit flags and the looked-up value, 0 on a miss"""
    d = dict(zip(bk.tolist(), bv.tolist()))
    hit = np.fromiter((k in d for k in pk.tolist()), dtype=bool, count=len(pk))
    val = np.fromiter((d.get(k, 0) for k in pk.tolist()), dtype=np.uint64, count=len(pk))
    return hit, val


def check_probe(ctx, bk, bv, pk, pv, want=None):
    hit_exp, val_exp = expected(bk, bv, pk)
    if want is not None:
        assert np.array_equal(hit_exp, want)
    build = ctx.kv_from_columns(bk, bv)
    probe = ctx.kv_from_columns(pk, pv)
    try:
        vals, hit = build.hash_probe(probe)
        vk, vv = vals.columns()
        vals.free()
        assert hit.dtype == np.uint8 and set(np.unique(hit).tolist()) <= {0, 1}
        bad = np.flatnonzero(hit.astype(bool) != hit_exp)
        assert len(bad) == 0, ("hit flags differ", len(bad), bad[:5], pk[bad[:5]])
        assert np.array_equal(vk, pk), "the probe keys come back aligned with the probe"
        bad = np.flatnonzero(vv != val_exp)
        assert len(bad) == 0, ("values differ (a miss reads 0)", len(bad), bad[:5])
        # hash_join: the matched probe records and (key, build value), compacted in probe order
        jp, jb = build.hash_join(probe)
        (jpk, jpv), (jbk, jbv) = jp.columns(), jb.columns()
        jp.free()
        jb.free()
        assert np.array_equal(jpk, pk[hit_exp]) and np.array_equal(jpv, pv[hit_exp])
        assert np.array_equal(jbk, pk[hit_exp]) and np.array_equal(jbv, val_exp[hit_exp])
    finally:
        build.free()
        probe.free()
    return hit_exp


PROBE_SIZES = (0, 1, 7, 8, 9, 4095, 4096, 4097)


@pytest.mark.parametrize("n_build", [0, 1, 511, 512, 513, 1_000_000])
def test_probe_and_join_against_a_dict(ctx, n_build):
    rng = np.random.default_rng(n_build + 1)
    bk = build_keys(n_build, rng)
    bv = rng.integers(0, 1 << 64, size=n_build, dtype=np.uint64)
    bv[:1] = np.uint64((1 << 64) - 1)
    absent = absent_keys(10_000, bk, rng)
    for n in PROBE_SIZES:
        for pat in PATTERNS:
            want = hit_pattern(pat, n) & (n_build > 0)
            pk = probe_side(bk, want, absent, rng)
            pv = np.arange(n, dtype=np.uint64) * np.uint64(3)
            check_probe(ctx, bk, bv, pk, pv, want)
    # every special key probed where the build side holds it
    pk = np.concatenate((SPECIAL, bk[:100]))
    hit = check_probe(ctx, bk, bv, pk, np.arange(len(pk), dtype=np.uint64))
    assert hit[:min(4, n_build)].all()


@pytest.mark.parametrize("pattern", PATTERNS)
def test_probe_and_join_over_more_than_1024_tiles(ctx, pattern):
    """4 194 307 probe records: 1 025 tiles of 4 096 flags, so the tile scan of hash_join carries between passes"""
    rng = np.random.default_rng(11)
    n = 1024 * TILE + 3
    bk = build_keys(5000, rng)
    bv = rng.integers(0, 1 << 63, size=len(bk), dtype=np.uint64)
    want = hit_pattern(pattern, n)
    pk = probe_side(bk, want, absent_keys(5000, bk, rng), rng)
    check_probe(ctx, bk, bv, pk, np.arange(n, dtype=np.uint64), want)


@pytest.mark.parametrize("n_build", [8, 600])
def test_a_probe_chain_that_wraps_past_the_last_slot(ctx, n_build):
    """Build keys whose mix64 all start at slot cap - 3: the chain runs over the last slots and on from slot 0. Probes
    of present keys, of absent keys that start in the same chain (they walk all of it and stop at its end), and of
    absent keys elsewhere."""
    rng = np.random.default_rng(n_build)
    cap = table_slots(n_build)
    high = rng.choice(np.arange(1, 1 << 20, dtype=np.uint64), size=3 * n_build, replace=False)
    t = (high << np.uint64(int(np.log2(cap)))) | np.uint64(cap - 3)
    crafted = unmix64(t)
    assert np.array_equal(spill._mix64(crafted) & np.uint64(cap - 1), np.full(len(t), cap - 3, dtype=np.uint64))
    bk, same_chain = crafted[:n_build], crafted[n_build:]
    bv = np.arange(n_build, dtype=np.uint64) + np.uint64(1)
    elsewhere = absent_keys(1000, crafted, rng)
    pk = np.concatenate((bk, same_chain, elsewhere, bk[::-1], same_chain[:7], bk[-3:]))
    pk = np.concatenate((pk, rng.permutation(pk)))
    hit = check_probe(ctx, bk, bv, pk, np.arange(len(pk), dtype=np.uint64))
    assert hit.sum() == 2 * (2 * n_build + 3)


def sorted_kv(ctx, keys):
    kv = ctx.kv_from_columns(keys, np.arange(len(keys), dtype=np.uint64))
    kv.sort(dev.KEY_RAW)
    return kv


def expected_ranges(lk, rk):
    """(left begin, left end, number of right records) per left key group of sorted columns"""
    heads = np.flatnonzero(np.concatenate(([True], lk[1:] != lk[:-1]))) if len(lk) else np.zeros(0, np.int64)
    ends = np.append(heads[1:], len(lk))[:len(heads)]
    g = lk[heads]
    rb = np.searchsorted(rk, g, side="left")
    return heads, ends, rb, np.searchsorted(rk, g, side="right") - rb


def check_join_ranges(ctx, lk, rk):
    lk, rk = np.sort(lk), np.sort(rk)
    heads, ends, rb, rn = expected_ranges(lk, rk)
    left, right = sorted_kv(ctx, lk), sorted_kv(ctx, rk)
    try:
        # the group count and offsets first: they come from the same tile scan the join's offsets do
        assert left.count_groups() == len(heads)
        assert np.array_equal(left.group_offsets(), np.append(heads, len(lk)).astype(np.uint64))
        rows = left.join_ranges(right, dev.KEY_RAW).astype(np.int64)
    finally:
        left.free()
        right.free()
    assert rows.shape == (len(heads), 4)
    assert np.array_equal(rows[:, 0], heads) and np.array_equal(rows[:, 1], ends)
    assert np.array_equal(rows[:, 3] - rows[:, 2], rn)
    m = rn > 0
    assert np.array_equal(rows[m, 2], rb[m])
    # the left join these ranges describe (records numbered in sorted order), against oracle.refsem's
    lv, rv = np.arange(len(lk)), np.arange(len(rk))
    got = {int(lk[lb]): (lv[lb:le].tolist(), rv[b:e].tolist() if e > b else []) for lb, le, b, e in rows.tolist()}
    assert got == refsem.left_join(lk, lv, rk, rv)
    return rows


def test_join_ranges_over_more_than_1024_tiles(ctx):
    """a left side of 4 194 305+ records: 64 groups of exactly one tile (heads on tile starts), then groups of 1 to
    3 000 records; right groups for every other left key in the middle, none for the lowest and highest keys"""
    rng = np.random.default_rng(5)
    sizes = [TILE] * 64
    while sum(sizes) < 1024 * TILE + 1:
        sizes.append(int(rng.integers(1, 3000)))
    gk = rng.permutation(np.unique(rng.integers(1, 1 << 40, size=2 * len(sizes), dtype=np.int64)))[:len(sizes)]
    gk = np.sort(gk).view(np.uint64) * np.uint64(4)
    lk = np.repeat(gk, sizes)
    mid = gk[10:-10:2]
    rk = np.concatenate((np.repeat(mid, rng.integers(1, 4, size=len(mid))), gk[11:-10:2] + np.uint64(1)))
    rows = check_join_ranges(ctx, lk, rk)
    assert len(lk) > 1024 * TILE and (rows[:10, 3] == rows[:10, 2]).all() and (rows[-10:, 3] == rows[-10:, 2]).all()
    assert np.count_nonzero(rows[:, 0] % TILE == 0) >= 64


def test_join_ranges_with_an_empty_side(ctx):
    rng = np.random.default_rng(6)
    keys = rng.integers(0, 500, size=20_000, dtype=np.int64).view(np.uint64)
    assert len(check_join_ranges(ctx, keys[:0], keys)) == 0
    rows = check_join_ranges(ctx, keys, keys[:0])
    assert len(rows) == len(np.unique(keys)) and (rows[:, 3] == rows[:, 2]).all()
    check_join_ranges(ctx, keys[:4097], keys[:4096])


def test_count_dictionary_at_the_presence_table_cap(ctx):
    """2^21 + 1 rows: the presence table has its largest size, 2^22 entries, so the block scan runs over 4 096 block
    counts, four per thread. Values B - 1 and B sit on either side of the table's bound."""
    B = 1 << 22
    rng = np.random.default_rng(21)
    n = (1 << 21) + 1
    counts = rng.integers(0, B, size=n, dtype=np.int64)
    counts[rng.integers(0, n, size=5)] = B - 1
    counts[rng.integers(0, n, size=5)] = B
    counts[-1] = B + 12345
    m = check_dictionary(ctx, counts)
    assert m > (1 << 20)
    # a column of every value below 2^12 and a few per block: every block count differs from the next
    check_dictionary(ctx, np.concatenate((np.arange(n - 4096, dtype=np.int64) % (B - 1), np.arange(4096))))


def test_count_dictionary_first_rows_beyond_2_24(ctx):
    """values whose first row is beyond 2^24: the row index of each value is the smallest row holding it"""
    rng = np.random.default_rng(24)
    n = (1 << 24) + 4096
    counts = rng.integers(0, 1000, size=n, dtype=np.int64)
    counts[(1 << 24) + 7] = 5000
    counts[(1 << 24) + 4000] = 1 << 30
    counts[-1] = (1 << 22) - 1
    check_dictionary(ctx, counts)
    plan.forget_count_dictionary()

"""GPU: the kernels over recycled device memory. Every kernel must write every output slot it reports; the engine's
pool (csrc/ctx.cu pool_alloc) hands freed blocks back without clearing them, and the text buffer and combiner table
of plan._cached_textbuf / plan._cached_table live from one scan to the next. Each operation here runs twice, each
time on a fresh context whose pool holds nothing but a ladder of blocks filled with one of two poisons, the second
the bitwise complement of the first, over a text buffer filled with one of two stale texts that share no byte, and
a table left holding another scan's results. The text is uploaded in 64 KB chunks with the kernel launches trailing
the copies (TextScan._count_ready), so a launch runs while the bytes past the uploaded ones are still stale. The two
runs must be byte-identical (an output byte the kernel leaves unwritten differs between them) and both must equal a
plain reference (numpy, Python, the numpy stand-in device tests/fake_device.py, text_contract.py).

Initialisation audit (index = used as an address or offset, count = a size the host or a kernel trusts, bound = a
loop bound). Only buffers that are memset or fully written before they are read are poisoned here; none of the
buffers below is read as an index before it is written.

Pool blocks (pool_alloc / DevBuf):
- kv records (ctx.cu dampr_kv_create): data. Written by the upload, upload_columns (interleave_kernel or the copy
  threads), synth, extract or fold that produces them; only [0, n) is ever read, and n is set by the producer.
- kv alt scratch (kv.cu:906): data. Every sort pass writes [start, start + n) before the next pass reads it.
- kv.cu:594-601 (one partition level): d_tot is a count (memset), d_hist a count (memset when the histogram is split,
  otherwise fully written by part_hist2_kernel), d_seg an index (bucket_scan_kernel writes all nb + 1 entries),
  d_poff an index (column_offsets_kernel writes all NP x nb).
- kv.cu:654-661 (the batched level): d_pieces, d_cta_pb, d_seg_pb, d_seg_off are indices uploaded from the host;
  d_hist a count fully written by part_hist2_kernel; d_poff and d_next indices written by part_scan_kernel.
- kv.cu:828-886 (leaves): d_chunks uploaded; d_estart / d_egroups counts written by leaf_sort_kernel per entry;
  d_off uploaded.
- kv.cu:1046-1073 and ops.cu:288-306 (group offsets): d_cnt a count written per tile, d_base an index written by the
  scan (ntiles + 1 entries), d_offs / offs written at every head (the host appends n).
- ops.cu:361 upload_columns / download_columns staging: data, written by the copy / deinterleave_kernel.
- ops.cu:381-401 join ranges: lo / ro indices from device_group_offsets, d_rows written for every left group.
- ops.cu:418-438 hash probe: used is a bound / slot marker (memset), tk / tv written where used is claimed, hit
  written for every probe record; ops.cu:459-498 hash join adds vals (written per probe record), tcnt (count, per
  tile) and tbase (index, scan).
- merge.cu:234-311: d_runs, d_soff and host cuts are uploaded; d_samples / d_salt written by merge_sample_kernel;
  d_cuts (index) and d_bkeys written by merge_cut_kernel; d_err a flag (memset). merge.cu:320-352: d_tmp written by
  merge_tile_kernel; d_pstart / d_pg / d_contrib / d_cont by merge_cont_kernel; d_poff (index) by the scan.
- ops.cu:512-562 synth_text: uploads and scans, every entry written.
- text.cu:779 dampr_table_fetch: the cursor (memset, text.cu:781) is an index; codes / counts / reps are written at
  every cursor slot below m = stats[0], which equals the number of non-zero keys.
- text.cu:901 fetch_words: the cursor (memset, text.cu:908) is an index; words (NUL-padded to the width by the loop
  at text.cu:877), codes and reps are written at every cursor slot.
- text.cu:1122 count_dictionary: flag (count, memset), first (index sentinel, memset 0xFF), ctr (count, memset),
  bsum (index, written by dict_block_count / dict_scan), extra (uploaded), uniq / rows / inv / big written by the
  rank / inv / mark kernels for every present value.
- text.cu:1914 decode_words: data, every byte of every row written (padding loop text.cu:1903).
Table arrays (cudaMalloc, kept by plan._cached_table between scans):
- keys / counts / reps / stats: table_init_kernel (dampr_table_clear) writes every slot; keys are slot markers,
  stats counters, reps offsets into the text read only for hashed keys, which always store one.
- fb: entries below stats[7] written by the scan that counted them (fallback_lines reads only those).
- tiles (fields.cu:812-826): per-tile line counts, an index in record mode. The count pass writes one entry per
  tile of the range (fields.cu:392), fields_tile_scan_kernel turns them into bases before the record pass reads
  them.
- ext: the count column written by fetch_words for every row below m; ext_n is reset by every clear and fetch.
Context buffers:
- d_scratch (cudaMalloc at context creation): cursors and the minmax pair, memset or uploaded before each use.
- up_tmp[2] (ops.cu:333): upload staging written by the copy stream before interleave_kernel reads it.
Text buffer: the lead-in is memset to '\\n' at creation, dampr_textbuf_set_length memsets everything after n. The
bytes in [uploaded, n) hold the previous scan's text until the copies arrive; TextScan._count_ready launches only
over 4 KB ranges whose halo has been uploaded, which the chunked ingest here exercises."""
import contextlib
import functools
import math
import os
import random
import struct

import numpy as np
import pytest

import text_contract as tc
from dampr_b200 import device as dev
from dampr_b200 import keycodes
from fake_device import FakeCtx
from test_gpu_key_orders import (ALL_OPS, LEAF, assert_folds, expected_groups, fold_values, grouped_keys,
                                 keyed_order, keys_for, sorted_runs, stable_order, xforms_for)

pytestmark = pytest.mark.gpu

POISONS = (0xA5A5, 0x5A5A)
SIZES = [0, 1, LEAF - 1, LEAF, LEAF + 1, 65_537, 1_000_000]
TWO_LEVELS = 6_000_000     # records whose sort needs two radix partition levels
LADDER = [256 << k for k in range(22)]    # 256 B .. 512 MB, doubling
SELF_CHECK = (256, 4096, 1 << 20)


# ---- poison ---------------------------------------------------------------------------------------------------
def poison_pool(ctx, seed):
    """Fill the context's pool with a ladder of blocks that hold synth_kv records: two blocks per size below 64 MB, one
    above (40 blocks, 1.1 GB: inside the pool's 128 blocks and 3 GB that pool_trim keeps). POISONS[1] is the bitwise
    complement of POISONS[0], so the two differ in every byte (synth_kv's values alone are small integers, whose high
    bytes would agree); any other seed is plain synth_kv records of that seed. Fails unless a fresh, unwritten kv
    downloads as the poison."""
    invert = seed == POISONS[1]
    base = POISONS[0] if invert else seed
    kvs, kept = [], {}
    for i, nbytes in enumerate(LADDER):
        for j in range(2 if nbytes < (64 << 20) else 1):
            kv = ctx.synth_kv(base * 1000 + 2 * i + j, nbytes // 16, 1 << 62)
            if invert:
                complement(ctx, kv, nbytes // 8)
            if nbytes in SELF_CHECK:
                kept.setdefault(nbytes, []).append(kv.records())
            kvs.append(kv)
    ctx.sync()
    for kv in kvs:
        kv.free()
    for nbytes, recs in kept.items():
        kv = ctx.kv(nbytes // 16)
        kv.set_size(nbytes // 16)
        got = kv.records()
        kv.free()
        assert any(np.array_equal(got, r) for r in recs), "a fresh kv of %d bytes does not hold the poison" % nbytes


class _DeviceWords(object):
    """n int64 words of device memory at ptr, as a CUDA array (test tooling: torch flips the poison in place)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<i8", "data": (int(ptr), False),
                                         "version": 3, "strides": None, "stream": None}


def complement(ctx, kv, n_words):
    import torch
    ctx.sync()
    t = torch.as_tensor(_DeviceWords(kv.devptr(), n_words), device="cuda:%d" % ctx.device)
    assert t.data_ptr() == kv.devptr()          # a view of the block, not a copy
    t.bitwise_not_()
    torch.cuda.synchronize(ctx.device)


def poison_text(seed, nbytes):
    """stale text: lines of a vocabulary no test corpus uses (z, q, v, digits, ' ', '\\n'), or (POISONS[1] and any
    other seed) one run of word bytes without a newline, made of bytes the first never holds"""
    if seed == POISONS[0]:
        rng = random.Random(seed)
        words = [b"zq%dv" % i for i in range(997)]
        out, n = [], 0
        while n < min(nbytes, 1 << 20):
            line = b" ".join(rng.choice(words) for _ in range(rng.randrange(1, 12))) + b"\n"
            out.append(line)
            n += len(line)
        block = b"".join(out)
        return np.frombuffer((block * (nbytes // len(block) + 1))[:nbytes], dtype=np.uint8)
    return np.frombuffer((b"Qx" * (nbytes // 2 + 1))[:nbytes], dtype=np.uint8)


def poison_textbuf(tb, seed):
    tb.set_length(tb.capacity)
    tb.upload(0, poison_text(seed, tb.capacity))
    tb.ctx.sync()


@contextlib.contextmanager
def poisoned(seed):
    """a fresh context whose pool holds nothing but the poison ladder of `seed`"""
    from dampr_b200 import plan
    c = dev.Ctx(0)
    try:
        poison_pool(c, seed)
        yield c
    finally:
        for b in plan._BUFFERS.pop(id(c), {}).values():   # the cached text buffer and table die with the context
            b.free()
        c.close()


def same_bytes(a, b, where=()):
    if isinstance(a, np.ndarray):
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape, where
        assert a.tobytes() == b.tobytes(), (where, "the two poisons gave different bytes")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            same_bytes(x, y, where + (i,))
    elif isinstance(a, dict):
        assert set(a) == set(b), where
        for k in a:
            same_bytes(a[k], b[k], where + (k,))
    elif isinstance(a, float):
        assert struct.pack("<d", a) == struct.pack("<d", b), where
    else:
        assert a == b, where


def ab(fn):
    """fn(ctx, seed) after each poison; the two results byte-identical; returns the first"""
    outs = []
    for seed in POISONS:
        with poisoned(seed) as c:
            outs.append(fn(c, seed))
    same_bytes(outs[0], outs[1])
    return outs[0]


def canon_reps(codes, reps):
    """reps with a hashed key's text offset dropped: which occurrence a hashed key keeps is the race of its first
    inserts, its length and every other key's rep (0) are not"""
    hashed = (codes >> np.uint64(63)) != 0
    return np.where(hashed, reps & np.uint64(0xFFFFF), reps)


def by_key(k, v):
    o = np.lexsort((v, k))
    return k[o], v[o]


# ---- kv ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
def test_uploads_and_downloads(n):
    rng = np.random.default_rng(n)
    keys = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    vals = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)

    def go(c, _seed):
        a = c.kv_from_columns(keys, vals)
        b = c.kv(n)
        half = n // 2
        b.upload_columns(0, keys[:half], vals[:half])
        b.upload(half, np.ascontiguousarray(np.stack((keys[half:], vals[half:]), axis=1)))
        c.sync()
        out = (a.columns(), a.records(), b.columns(), b.records())
        a.free()
        b.free()
        return out

    (ak, av), arec, (bk, bv), brec = ab(go)
    for k, v, r in ((ak, av, arec), (bk, bv, brec)):
        assert np.array_equal(k, keys) and np.array_equal(v, vals)
        assert np.array_equal(r[:, 0], keys) and np.array_equal(r[:, 1], vals)


@pytest.mark.parametrize("n", SIZES + [TWO_LEVELS])
def test_sort_every_key_transform(n):
    xfs = (dev.KEY_RAW, dev.KEY_MIX, dev.KEY_I64, dev.KEY_F64) if n < TWO_LEVELS else (dev.KEY_F64, dev.KEY_MIX)
    for xf in xfs:
        keys = keys_for(xf, np.random.default_rng(n + xf), n)
        if xf == dev.KEY_MIX:
            keys = keys_for(dev.KEY_RAW, np.random.default_rng(n + xf), n) % np.uint64(max(1, n // 3))
        vals = np.arange(n, dtype=np.uint64)

        def go(c, _seed):
            kv = c.kv_from_columns(keys, vals)
            kv.sort(xf)
            out = kv.columns()
            kv.free()
            return out

        k2, v2 = ab(go)
        if xf == dev.KEY_MIX:     # the mixed order: compare with the stand-in device, which orders by mix64
            fk = FakeCtx().kv_from_columns(keys, vals)
            fk.sort(xf)
            ek, ev = fk.columns()
            assert np.array_equal(k2, ek) and np.array_equal(v2, ev), (n, xf)
        else:
            o = stable_order(keys, xf)
            assert np.array_equal(k2, keys[o]) and np.array_equal(v2, o.astype(np.uint64)), (n, xf)


@pytest.mark.parametrize("op", ALL_OPS)
def test_sort_reduce_and_reduce_by_key_every_op(op):
    for xf in xforms_for(op):
        for n, nk in ((0, 1), (1, 1), (LEAF - 1, 7), (LEAF, 5), (LEAF + 1, 3), (65_537, 501), (1_000_000, 20_000)):
            rng = np.random.default_rng(1000 * op + 10 * xf + nk)
            keys = grouped_keys(xf, rng, n, nk)
            vals = fold_values(op, rng, n)
            o = stable_order(keys, xf)

            def go(c, _seed):
                kv = c.kv_from_columns(keys, vals)
                out = kv.sort_reduce(op, xf)
                got = out.columns()
                out.free()
                kv.free()
                srt = c.kv_from_columns(keys[o], vals[o])
                red = srt.reduce_by_key(op)
                got2 = red.columns()
                red.free()
                srt.free()
                if not keyed_order(op, xf):   # hash-folded groups: their order is the leaves' own
                    got = by_key(*got)
                return got, got2

            (gk, gv), (rk, rv) = ab(go)
            ek, ev = expected_groups(keys, vals, op, xf)
            assert_folds(gk, gv, ek, ev, op, keyed_order(op, xf), vals, keys)
            assert_folds(rk, rv, ek, ev, op, True, vals, keys)


@pytest.mark.parametrize("n", SIZES)
def test_group_offsets(n):
    rng = np.random.default_rng(n + 5)
    keys = np.sort(rng.integers(0, max(1, n // 4), size=n).astype(np.uint64))

    def go(c, _seed):
        kv = c.kv_from_columns(keys, np.zeros(n, dtype=np.uint64))
        out = (kv.group_offsets(), kv.count_groups())
        kv.free()
        return out

    offs, g = ab(go)
    heads = np.flatnonzero(np.concatenate(([True], keys[1:] != keys[:-1]))) if n else np.zeros(0, np.int64)
    assert g == len(heads)
    assert offs.tolist() == heads.tolist() + [n]


@pytest.mark.parametrize("k", [1, 2, 8, 70])
def test_merge_and_merge_ranges(k):
    xf = dev.KEY_F64
    fake = FakeCtx()
    for op in (None, dev.OP_SUM_I64, dev.OP_FIRST, dev.OP_MAX_F64):
        rng = np.random.default_rng(k * 31 + (op or 0))
        runs = sorted_runs(xf, rng, k, op)
        allk = np.concatenate([r[0] for r in runs])
        allv = np.concatenate([r[1] for r in runs])
        offs = np.concatenate(([0], np.cumsum([len(r[0]) for r in runs]))).astype(np.uint64)
        code = -1 if op is None else op

        def go(c, _seed):
            dev_runs = [c.kv_from_columns(a, b) for a, b in runs]
            flat = c.kv_from_columns(allk, allv)
            outs = [c.kv_merge(dev_runs, xf, code), c.kv_merge_ranges(flat, offs, xf, code)]
            got = [o.columns() for o in outs]
            for x in outs + dev_runs + [flat]:
                x.free()
            return got

        want = fake.kv_merge_ranges(fake.kv_from_columns(allk, allv), offs, xf, code).columns()
        for gk, gv in ab(go):
            assert np.array_equal(gk, want[0]) and np.array_equal(gv, want[1]), (k, op)


@pytest.mark.parametrize("n", SIZES)
def test_joins_probes_and_partitions(n):
    rng = np.random.default_rng(n + 11)
    pool = np.unique(rng.integers(0, 1 << 64, size=max(1, n // 2 + 1), dtype=np.uint64))
    lk = np.sort(pool[rng.integers(0, len(pool), size=n)])
    rk = np.sort(pool[rng.integers(0, len(pool), size=max(1, n // 2))])
    build_k = pool[: max(1, len(pool) // 2)]
    build_v = rng.integers(0, 1 << 64, size=len(build_k), dtype=np.uint64)
    probe_k = pool[rng.integers(0, len(pool), size=n)]
    probe_v = np.arange(n, dtype=np.uint64)
    fake = FakeCtx()

    def go(c, _seed):
        L = c.kv_from_columns(lk, np.arange(n, dtype=np.uint64))
        R = c.kv_from_columns(rk, np.arange(len(rk), dtype=np.uint64))
        rows = L.join_ranges(R, dev.KEY_RAW)
        rows[rows[:, 2] == rows[:, 3], 2:] = 0
        B = c.kv_from_columns(build_k, build_v)
        P = c.kv_from_columns(probe_k, probe_v)
        pv, hit = B.hash_probe(P)
        pvals = pv.columns()[1][hit.astype(bool)]
        jp, jb = B.hash_join(P)
        parts = {}
        for nd in (1, 3, 8):
            out, counts = P.partition_by_owner(nd)
            parts[nd] = (out.records(), counts)
            out.free()
        out = (rows, hit, pvals, jp.records(), jb.records(), parts)
        for x in (L, R, B, P, pv, jp, jb):
            x.free()
        return out

    rows, hit, pvals, jp, jb, parts = ab(go)
    FL, FR = fake.kv_from_columns(lk, np.arange(n, dtype=np.uint64)), fake.kv_from_columns(rk, np.arange(len(rk),
                                                                                                          dtype=np.uint64))
    want = FL.join_ranges(FR, dev.KEY_RAW)
    want[want[:, 2] == want[:, 3], 2:] = 0
    assert np.array_equal(rows, want)
    FB, FP = fake.kv_from_columns(build_k, build_v), fake.kv_from_columns(probe_k, probe_v)
    fv, fhit = FB.hash_probe(FP)
    assert np.array_equal(hit, fhit) and np.array_equal(pvals, fv.columns()[1][fhit.astype(bool)])
    fjp, fjb = FB.hash_join(FP)
    assert np.array_equal(jp, fjp.records()) and np.array_equal(jb, fjb.records())
    for nd, (recs, counts) in parts.items():
        fo, fc = FP.partition_by_owner(nd)
        assert np.array_equal(counts, fc)
        frec = fo.records()
        starts = np.concatenate(([0], np.cumsum(fc))).astype(np.int64)
        for d in range(nd):   # each destination's records, as a multiset
            a, b = recs[starts[d]:starts[d + 1]], frec[starts[d]:starts[d + 1]]
            assert np.array_equal(a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])]), (n, nd, d)


def test_all_to_all_at_world_one():
    n = 65_537
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    vals = np.arange(n, dtype=np.uint64)

    def go(c, _seed):
        c.comm_create(0, 1, c.comm_unique_id())
        kv = c.kv_from_columns(keys, vals)
        out, offs, heads = c.kv_all_to_all(kv, header=[7, -3])
        got = (out.records(), offs, heads)
        out.free()
        kv.free()
        return got

    recs, offs, heads = ab(go)
    assert offs.tolist() == [0, n] and heads.tolist() == [[7, -3]]
    assert np.array_equal(recs[:, 0], keys) and np.array_equal(recs[:, 1], vals)


@pytest.mark.parametrize("width", [16, 24, 32, 64, 128, 256])
def test_decode_words(width):
    words = ([b"a", b"ab", b"z" * 9, b"x7_", b"0"] + [b"w%d" % i for i in range(3000)])
    codes = []
    for w in words:                 # 7-bit codes (TOK_WS) of the word, little end first
        c = 0
        for ch in reversed(w):
            c = (c << 7) | ch
        codes.append(c)
    codes += [(1 << 63) | 12345, (1 << 63) | 1]      # hashed codes decode to b''
    keys = np.array(codes, dtype=np.uint64)

    def go(c, _seed):
        kv = c.kv_from_columns(keys, np.zeros(len(keys), dtype=np.uint64))
        out = kv.decode_words(dev.TOK_WS, width)
        kv.free()
        return out.view(np.uint8).reshape(len(keys), width).copy()

    got = ab(go)
    want = [w[:width].ljust(width, b"\0") for w in words] + [b"\0" * width] * 2
    assert [bytes(r) for r in got] == want


# ---- table and text ------------------------------------------------------------------------------------------------
BUILDS = [(2, 4), (2, 3), (2, 2), (1, 2)]
REFUSE = tc.TF_NONASCII | tc.TF_LONGLINE | tc.TF_TABLEFULL
MODES = (dev.TOK_WS, dev.TOK_NONWORD_LOWER_SET, dev.TOK_NONWORD_LOWER)


@functools.lru_cache(maxsize=None)
def zipf_corpus(seed, n_lines):
    from oracle import gen
    return gen.text(seed, n_lines, V=3000) if n_lines else b""


def dirty_corpus(seed, n_lines):
    """Zipf lines with a short non-ASCII line after every 300th: the second-generation kernel's [^\\w]+ modes hand
    those to the host (a non-empty fallback list), the other builds and TOK_WS refuse the scan"""
    lines = zipf_corpus(seed, n_lines).split(b"\n")
    for i in range(len(lines) - 1, 0, -300):
        lines.insert(i, ("Naïve café %d, déjà vu" % i if i % 2 else "ü").encode("utf-8"))
    return b"\n".join(lines)


def long_line_corpus():
    """short lines around lines of 4 to 60 KB, so that many 16 KB tiles hold no line start (ASCII: TOK_WS takes it
    in every build; the [^\\w]+ modes refuse lines that outrun their window)"""
    rng = random.Random(17)
    parts = []
    for i in range(24):
        parts.append(zipf_corpus(100 + i, 40))
        n = rng.randrange(4 << 10, 60 << 10)
        body = b" ".join(b"t%d" % rng.randrange(500) for _ in range(n // 5))[:n]
        parts.append(body + b"\n")
    parts.append(b"Tokens A b, C\n" + b"q" * 40 + b" end\n")
    return b"".join(parts)


TEXT_CORPORA = {"empty": lambda: b"", "one": lambda: b"One line, Of tokens_7 here q%s\n" % (b"q" * 30),
                "zipf": lambda: zipf_corpus(7, 30_000), "dirty": lambda: dirty_corpus(8, 30_000),
                "long": long_line_corpus}
CHUNK = 1 << 16     # the ingest chunk of the unit tests (settings.ingest_chunk_bytes in the end-to-end test)


def dirty_table(c, tab, seed):
    """leave tab holding another scan: record mode over a larger text (more tiles), its fallback list, and the
    extracted count column of a different mode at the widest width"""
    other = zipf_corpus(seed, 120_000) + b"\xff,1\n" * 5
    tb = c.textbuf(len(other) + 64)
    tb.upload_all(other)
    kv = c.kv(len(other) // 2)
    tab.fields_records(tb, 0, len(other), (ord(" "), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64), kv)
    tab.clear()
    tab.count(tb, 0, len(other), dev.TOK_NONWORD_LOWER)
    tab.fetch_words(tb, dev.TOK_NONWORD_LOWER, 256)
    c.sync()
    kv.free()
    tb.free()
    tab.clear()


def ingest_plan(n, halo):
    """[(upload start, upload end, launch range or None)] of a chunked ingest: after each chunk, one launch over the
    4 KB-aligned bytes whose halo has been uploaded (TextScan._count_ready), then the rest"""
    out, counted = [], 0
    for off in range(0, n, CHUNK):
        done = min(off + CHUNK, n)
        hi = max(counted, ((done - halo) // 4096) * 4096 if done > halo else 0)
        out.append((off, done, (counted, hi) if hi > counted else None))
        counted = hi
    if n > counted:
        out.append((n, n, (counted, n)))
    return out


def ingest(tb, data, halo, launch):
    """data into a text buffer that holds stale bytes, launches trailing the copies: a launch waits for the uploads
    queued before it, while the bytes not uploaded yet are still the previous text"""
    arr = np.frombuffer(data, dtype=np.uint8)
    tb.set_length(len(data))
    for a, b, rng in ingest_plan(len(data), halo):
        if b > a:
            tb.upload(a, arr[a:b])
        if rng:
            launch(*rng)


def cached_buffers(c, seed, data):
    """plan's cached text buffer, filled with stale text, and a table left holding another scan"""
    from dampr_b200 import plan
    tb = plan._cached_textbuf(c, len(data) + (1 << 20))
    poison_textbuf(tb, seed)
    tab = c.table(18)
    dirty_table(c, tab, seed)
    return tb, tab


@pytest.fixture(params=BUILDS, ids=["v2-4cta", "v2-3cta", "v2-2cta", "v1"])
def build(request):
    dev.set_option("text_kernel", request.param[0])
    dev.set_option("text_ctas", request.param[1])
    try:
        yield request.param
    finally:
        dev.set_option("text_kernel", 2)
        dev.set_option("text_ctas", 4)


@pytest.mark.parametrize("corpus", sorted(TEXT_CORPORA))
def test_count_fetch_and_dictionary(build, corpus, monkeypatch):
    """dampr_text_count with launches trailing the copies, then every way out of the table. The flags must be the
    ones text_contract.refusals requires; a scan without a refusal flag must equal Python exactly"""
    from dampr_b200 import plan, settings
    monkeypatch.setattr(plan, "_BUFFERS", {})
    data = TEXT_CORPORA[corpus]()
    kernel, ctas = build
    ranges = [r for _a, _b, r in ingest_plan(len(data), plan.TextScan.HALO) if r]
    compared = 0
    for mode in MODES:
        def go(c, seed):
            tb, tab = cached_buffers(c, seed, data)
            ingest(tb, data, plan.TextScan.HALO, lambda a, b: tab.count(tb, a, b, mode))
            st = tab.stats()
            codes, counts, reps = tab.fetch()
            o = np.argsort(codes)
            codes, counts, reps = codes[o], counts[o], reps[o]
            words = keycodes.decode_table(codes, reps, mode, lambda o, n: data[o:o + n])
            out = {"stats": st, "fetch": (codes, counts, canon_reps(codes, reps)), "words": words,
                   "fb": np.sort(tab.fallback_lines())}
            for width in (16, 32, 256):
                for cache in (64 << 20, 0):        # the leased block, then pageable arrays
                    monkeypatch.setattr(settings, "host_result_cache_bytes", cache)
                    w, cn, cd, rp = tab.fetch_words(tb, mode, width)
                    o = np.argsort(cd)
                    rows = np.asarray(w).view(np.uint8).reshape(-1, width)[o].copy()
                    cd, rp = np.array(cd)[o], np.array(rp)[o]
                    out["words", width, cache] = (rows, np.array(cn)[o], cd, canon_reps(cd, rp))
                    ptr, m = tab.extracted_counts()
                    assert m == len(cd)
                    uniq, inv, first = (np.array(x) for x in c.count_dictionary(ptr, m))
                    col = np.array(cn).astype(np.int64)      # the row order of the extracted column
                    eu, einv = np.unique(col, return_inverse=True)
                    assert np.array_equal(uniq, eu) and np.array_equal(inv.astype(np.int64), einv.ravel())
                    assert first.tolist() == [int(np.flatnonzero(col == u)[0]) for u in eu.tolist()]
                    out["dict", width, cache] = (uniq, inv[o])
            kv = tab.to_kv()
            out["kv"] = by_key(*kv.columns())
            kv.free()
            tab.free()
            return out

        out = ab(go)
        st = out["stats"]
        req, allowed = tc.refusals(data, mode, False, ranges, kernel, ctas)
        assert st["flags"] & req == req and st["flags"] & ~allowed == 0, (build, mode, st, req, allowed)
        if st["flags"] & REFUSE:
            continue
        compared += 1
        fb = tc.expected_fallback(data, kernel, mode, False)
        exp = tc.expected_table(data, mode, False, fb)
        assert out["fb"].tolist() == fb
        assert st["fallback"] == len(fb) and st["lines"] == exp["lines"] and st["folded"] == exp["folded"]
        codes, counts, reps = out["fetch"]
        words = out["words"]
        assert dict(zip(words, counts.tolist())) == exp["table"], (build, mode)
        assert np.array_equal(out["kv"][0], codes) and np.array_equal(out["kv"][1], counts)
        for width in (16, 32, 256):
            for cache in (64 << 20, 0):
                rows, cn, cd, rp = out["words", width, cache]
                assert np.array_equal(cd, codes) and np.array_equal(cn, counts)
                assert [bytes(r) for r in rows] == [w.encode()[:width].ljust(width, b"\0") for w in words]
                hashed = (cd >> np.uint64(63)) != 0
                assert np.array_equal(rp[hashed], reps[hashed]) and not rp[~hashed].any()
                uniq, inv = out["dict", width, cache]
                assert np.array_equal(uniq[inv.astype(np.int64)], counts.astype(np.int64))
    # what is compared with Python: every ASCII corpus in TOK_WS, and the fallback list of the second generation
    want = {"dirty": 2 if kernel == 2 else 0, "long": 1}.get(corpus, 3)
    assert compared == want, (corpus, build, compared)


# ---- fields ----------------------------------------------------------------------------------------------------------
def fields_corpus(sep, n_lines):
    """key<sep>value<sep>int<sep>tail lines: short and hashed keys, ints, floats and values the device refuses,
    non-ASCII lines, and lines of 4-60 KB (many tiles without a line start)"""
    rng = random.Random(23 + (sep == dev.FIELD_SEP_WS))
    s = " " if sep == dev.FIELD_SEP_WS else chr(sep)
    lines = []
    for i in range(n_lines):
        k = rng.choice(["a", "bb", "q" * 12, "w%d" % rng.randrange(400), "é", "k7"])
        v = rng.choice(["%d" % rng.randrange(-10 ** 6, 10 ** 6), "%.4f" % (rng.choice((-1, 1)) * rng.uniform(1, 100)),
                        "x", "1_0", repr(rng.random() + 1e-9)])
        tail = "p" * rng.randrange(4 << 10, 60 << 10) if i % 2500 == 7 else "z"
        lines.append(s.join([k, v, "%d" % rng.randrange(100), tail]) + "\n")
    return "".join(lines).encode("utf-8")


def py_records(data, sep):
    """(line start, line bytes, fields) of every line"""
    out, pos = [], 0
    for raw in data.split(b"\n")[:-1]:
        f = raw.split() if sep == dev.FIELD_SEP_WS else raw.split(bytes([sep]))
        out.append((pos, raw, f))
        pos += len(raw) + 1
    return out


def field_fate(raw, f, where, value):
    """what the device must do with a line of key field 0 and value field 1 (dampr_b200.h, text_contract.py): "host"
    (the fallback list), "drop" (a WHERE int(f[2]) >= 30 that is false) or "fold"; value: "int", "f64" or "one" """
    from test_fparse_host import in_grammar
    if len(raw) >= tc.F_HALO or any(c >= 0x80 or c == 0 for c in raw) or b"\r" in raw:
        return "host"
    if where:
        if len(f) < 3 or not tc.INT18.fullmatch(f[2]):
            return "host"
        if int(f[2]) < 30:
            return "drop"
    if len(f) < 2:
        return "host"
    if value == "int" and not tc.INT18.fullmatch(f[1]):
        return "host"
    if value == "f64" and not in_grammar(f[1].decode("ascii")):
        return "host"
    return "fold"


def key_code(kb):
    if 1 <= len(kb) <= 9:
        c = 0
        for ch in reversed(kb):
            c = (c << 7) | ch
        return c
    return None


@pytest.mark.parametrize("n_lines", [0, 1, 60_000])
@pytest.mark.parametrize("sep", [ord(","), dev.FIELD_SEP_WS], ids=["comma", "split"])
@pytest.mark.parametrize("where", [False, True], ids=["plain", "where"])
def test_field_scans(sep, where, n_lines, monkeypatch):
    """table mode (int sum, line count, float max) and record mode (int and float values), launches trailing the
    copies, against Python: the exact fallback list, the fold of the other lines, holes exactly at the host's and
    the dropped lines"""
    from dampr_b200 import plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    data = fields_corpus(sep, n_lines)
    recs = py_records(data, sep)
    preds = [(dev.PRED_INT, 2, dev.CMP_GE, (30,))] if where else []
    TABLE = (("sum", 1, dev.OP_SUM_I64, "int"), ("count", dev.FIELD_VAL_ONE, dev.OP_SUM_I64, "one"),
             ("fmax", 1, dev.OP_MAX_F64, "f64"))
    RECORDS = (("rec_i", dev.OP_SUM_I64, "int"), ("rec_f", dev.OP_SUM_F64, "f64"))

    def go(c, seed):
        tb, tab = cached_buffers(c, seed, data)
        out = {}
        for name, vf, op, _v in TABLE:
            spec = (sep, 0, dev.FIELD_KEY_STR, vf, op)
            poison_textbuf(tb, seed)
            tab.clear()
            ingest(tb, data, dev.FIELDS_HALO, lambda a, b: tab.fields(tb, a, b, spec, preds=preds))
            codes, acc, reps = tab.fetch()     # one fetch: the row order is each extract's own
            vals = dev.decode_fold(acc, op)
            o = np.argsort(codes)
            codes, vals, reps = codes[o], vals[o], reps[o]
            keys = [data[rp >> 20:(rp >> 20) + (rp & 0xFFFFF)] if cd >> 63 else
                    bytes(keycodes.decode_exact(np.array([cd], dtype=np.uint64), dev.TOK_WS)[0], "ascii")
                    for cd, rp in zip(codes.tolist(), reps.tolist())]
            out[name] = (codes, vals, canon_reps(codes, reps), keys, np.sort(tab.fallback_lines()), tab.fields_stats())
        for name, op, _v in RECORDS:
            spec = (sep, 0, dev.FIELD_KEY_STR, 1, op)
            poison_textbuf(tb, seed)
            tab.clear()
            kv = c.kv(len(recs) + 7)
            ingest(tb, data, dev.FIELDS_HALO, lambda a, b: tab.fields_records(tb, a, b, spec, kv, preds=preds))
            st = tab.fields_stats()
            kv.set_size(st["records"])
            out[name] = (kv.records(), np.sort(tab.fallback_lines()), st)
            kv.free()
        tab.free()
        return out

    out = ab(go)
    for name, _vf, op, value in TABLE:
        codes, vals, _reps, keys, fb, st = out[name]
        assert st["flags"] == 0, (name, st)
        fate = [field_fate(raw, f, where, value) for _pos, raw, f in recs]
        assert fb.tolist() == [(pos << 16) | len(raw) for (pos, raw, _f), x in zip(recs, fate) if x == "host"], name
        exp = {}
        for (pos, raw, f), x in zip(recs, fate):
            if x != "fold":
                continue
            v = {"int": lambda s: int(s), "one": lambda s: 1, "f64": float}[value](f[1].decode())
            exp[f[0]] = v if f[0] not in exp else (exp[f[0]] + v if value != "f64" else max(exp[f[0]], v))
        assert dict(zip(keys, vals.tolist())) == exp, name
    for name, op, value in RECORDS:
        rec, fb, st = out[name]
        assert len(rec) == len(recs) and st["flags"] == 0, (name, st)
        fate = [field_fate(raw, f, where, value) for _pos, raw, f in recs]
        assert fb.tolist() == [(pos << 16) | len(raw) for (pos, raw, _f), x in zip(recs, fate) if x == "host"], name
        holes = np.flatnonzero(rec[:, 0] == 0)
        assert holes.tolist() == [i for i, x in enumerate(fate) if x != "fold"], name
        assert not rec[holes].any(), name
        for i, ((pos, raw, f), x) in enumerate(zip(recs, fate)):
            if x != "fold":
                continue
            kc = key_code(f[0])
            if kc is not None:
                assert int(rec[i, 0]) == kc, (name, i)
            v = int(f[1]) if op == dev.OP_SUM_I64 else float(f[1])
            want = (v & ((1 << 64) - 1)) if op == dev.OP_SUM_I64 else struct.unpack("<Q", struct.pack("<d", v))[0]
            assert int(rec[i, 1]) == want, (name, i, f)


# ---- end to end in one process -------------------------------------------------------------------------------------
def test_pipelines_repeat_over_poisoned_memory(monkeypatch, tmp_path):
    """TF-IDF, a field fold, a float mean() and a split() fold against Python, each lowered to the device; then the
    pool, the cached text buffer and the cached table poisoned, and all of them again: the same sink lines, byte for
    byte"""
    import bench
    from dampr_b200 import Dampr, plan, settings
    from dampr_b200 import runner as runner_mod
    from fields_standin import write_files
    from oracle import refsem
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "ingest_chunk_bytes", 1 << 16)
    tf = dirty_corpus(3, 40_000)    # the device tokenises it; its non-ASCII lines go through the fallback list
    rng = random.Random(5)
    csv = "".join("%s,%d,%r\n" % (rng.choice(["a", "b", "q" * 14, "w%d" % rng.randrange(99)]), rng.randrange(-999, 999),
                                  rng.uniform(-5, 5)) for _ in range(120_000))
    ws = "".join("%s  %d\t%d\n" % (rng.choice(["x", "yy", "z" * 11]), rng.randrange(50), rng.randrange(-99, 99))
                 for _ in range(80_000))
    P = write_files(tmp_path, [["f.csv", csv]])
    Q = str(tmp_path / "w.txt")
    with open(Q, "w") as f:
        f.write(ws)
    jobs = {
        "sum": lambda: Dampr.text(P).a_group_by(lambda l: l.split(",")[0], lambda l: int(l.split(",")[1])).sum(),
        "mean": lambda: Dampr.text(P).map(lambda l: l.split(",")).mean(lambda r: r[0], lambda r: float(r[2])),
        "split": lambda: Dampr.text(Q).a_group_by(lambda l: l.split()[0], lambda l: int(l.split()[2])).sum(),
    }
    exp = {}
    for l in csv.splitlines():
        k, v, x = l.split(",")
        exp.setdefault("sum", {})[k] = exp.get("sum", {}).get(k, 0) + int(v)
        exp.setdefault("mean", {}).setdefault(k, []).append(float(x))
    for l in ws.splitlines():
        f = l.split()
        exp.setdefault("split", {})[f[0]] = exp.get("split", {}).get(f[0], 0) + int(f[2])
    want_tf = sorted(refsem.tfidf_sink_lines(tf))

    def run_all(c, seed, tag):
        monkeypatch.setitem(runner_mod._CTX, settings.device, c)
        # the cached buffers the scans will take: a text buffer of stale text, a table left by another scan
        poison_textbuf(plan._cached_textbuf(c, 2 * len(tf) + (4 << 20)), seed)
        dirty_table(c, plan._cached_table(c), seed)
        out = str(tmp_path / ("tf%s" % tag))
        bench.tfidf_job(Dampr, plan.MemoryText(np.frombuffer(tf, dtype=np.uint8)), out)
        lines = sorted(l for fn in os.listdir(out) for l in open(os.path.join(out, fn), encoding="utf-8").read()
                       .splitlines())
        res = {"tfidf": lines}
        hows = [how for _s, how, _d in runner_mod.LAST_STATS.stages]
        assert any(h.startswith("device text tokenise+combine") for h in hows), hows
        for name, job in sorted(jobs.items()):
            res[name] = sorted(job().run())
            assert "device" in runner_mod.LAST_STATS.stages[0][1], (name, runner_mod.LAST_STATS.stages)
        return res

    outs = []
    for rep, seed in enumerate(POISONS):
        with poisoned(seed) as c:
            outs.append(run_all(c, seed, rep))
            poison_pool(c, seed + 1)
            outs.append(run_all(c, seed + 1, "%d-again" % rep))
    for o in outs[1:]:
        same_bytes(outs[0], o)
    res = outs[0]
    assert res["tfidf"] == want_tf
    assert dict(res["sum"]) == exp["sum"]
    assert dict(res["split"]) == exp["split"]
    got = dict(res["mean"])
    assert sorted(got) == sorted(exp["mean"])
    for k, xs in exp["mean"].items():   # the sum's bound against fsum, then one rounding of the division
        want = math.fsum(xs) / len(xs)
        bound = 4 * len(xs) * 2.0 ** -53 * math.fsum(map(abs, xs)) / len(xs) + 2.0 ** -52 * abs(want)
        assert abs(got[k] - want) <= bound, (k, got[k], want)

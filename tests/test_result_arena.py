"""The host side of the step's tail without a device: the lease object numpy views of the result arena hang on, the
sink's persistent worker pool and kept buffers, and the bytes the native joiner and sink write, against a Python
statement of the same rows."""
import gc
import os

import numpy as np
import pytest

from dampr_b200 import device as dev
from dampr_b200 import settings


class StubLib(object):
    def __init__(self):
        self.released = []

    def dampr_result_release(self, h, lease):
        self.released.append(lease)
        return 0


class StubCtx(object):
    def __init__(self):
        self.lib, self.h = StubLib(), 1


def leased(ctx, handle, nbytes):
    """a ResultLease over ordinary memory (kept alive on the lease itself: the stub has no arena)"""
    backing = np.zeros(nbytes, dtype=np.uint8)
    blk = dev.ResultLease(ctx, handle, backing.ctypes.data, nbytes)
    blk.backing = backing
    return blk


def test_views_keep_the_lease_and_the_last_one_releases_it():
    ctx = StubCtx()
    blk = leased(ctx, 7, 64)
    words, counts = blk.array(0, 2, "S16"), blk.array(32, 4, np.uint64)
    counts[:] = [1, 2, 3, 4]
    words[0] = b"kept"
    tail = counts[2:]            # a slice of a view
    del blk, counts
    gc.collect()
    assert ctx.lib.released == []
    # a second lease is taken and filled meanwhile: the first one's bytes are its own
    other = leased(ctx, 8, 64)
    other.array(0, 64, np.uint8)[:] = 0xEE
    assert words[0] == b"kept" and tail.tolist() == [3, 4]
    del words
    gc.collect()
    assert ctx.lib.released == []
    del tail
    gc.collect()
    assert ctx.lib.released == [7]
    del other
    gc.collect()
    assert ctx.lib.released == [7, 8]


def test_a_closed_context_is_not_called():
    ctx = StubCtx()
    blk = leased(ctx, 3, 16)
    ctx.h = None
    del blk
    gc.collect()
    assert ctx.lib.released == []


# ---- the joiner and the sink -----------------------------------------------------------------------------------
def columns(n, seed=0):
    """one column of every kind host_join_tsv takes, and the cells of every row as Python writes them"""
    rng = np.random.default_rng(seed)
    words = np.array([b"w%d" % (i * 7919 % 100003) for i in range(n)], dtype="S16") if n else np.zeros(0, dtype="S16")
    ints = np.unique(np.concatenate(([-5, 0, 1 << 40], rng.integers(-10**9, 10**9, 50)))).astype(np.int64)
    floats = np.unique(np.concatenate(([0.0, 1e-7, 1.5, 1e22, 2.0 / 3], rng.random(40)))).astype(np.float64)
    strs = [b"", b"x", b"a longer cell", "é".encode("utf-8")]
    iv = rng.integers(0, len(ints), n).astype(np.uint32)
    fv = rng.integers(0, len(floats), n).astype(np.uint32)
    sv = rng.integers(0, len(strs), n).astype(np.uint32)
    cols = [words, (iv, ints), (fv, floats), (sv, strs)]
    il = [b"%d" % v for v in ints.tolist()]
    fl = [repr(v).encode() for v in floats.tolist()]
    rows = [b"\t".join((w, il[a], fl[b], strs[c])) + b"\n"
            for w, a, b, c in zip(words.tolist(), iv.tolist(), fv.tolist(), sv.tolist())]
    return cols, rows


SIZES = [0, 1, 32767, 32768, 32769, 3 * 32768 + 5]


def n_files(n):
    return int(min(16, os.cpu_count() or 1, max(1, n // 32768)))


@pytest.mark.parametrize("n", SIZES)
def test_join_and_sink_write_pythons_rows(n, tmp_path):
    cols, rows = columns(n, seed=n)
    want = b"".join(rows)
    assert dev.host_join_tsv(cols).tobytes() == want
    prefix = str(tmp_path / "part-")
    names = dev.host_join_tsv(cols, prefix=prefix, first=3)
    assert names == ["%s%d" % (prefix, 3 + j) for j in range(n_files(n))]
    assert sorted(os.listdir(tmp_path)) == sorted(os.path.basename(x) for x in names)   # no empty extras
    got = [open(x, "rb").read() for x in names]
    assert b"".join(got) == want
    # row ranges n * t / T, whole rows per file
    T = len(names)
    assert [g.count(b"\n") for g in got] == [n * (t + 1) // T - n * t // T for t in range(T)]


def test_formatted_rows_and_a_file_limit(tmp_path):
    n = 70000
    cols, rows = columns(n, seed=5)
    pre, end = [b"[\"", b"\", ", b", ", b", \""], b"\"]\n"
    want = b"".join(b"".join(p + c for p, c in zip(pre, r[:-1].split(b"\t"))) + end for r in rows)
    names = dev.host_join_tsv(cols, prefix=str(tmp_path / "part-"), col_pre=pre, row_end=end)
    assert b"".join(open(x, "rb").read() for x in names) == want
    one = dev.host_join_tsv(cols, prefix=str(tmp_path / "single-"), max_files=1)
    assert len(one) == 1 and open(one[0], "rb").read() == b"".join(rows)


def test_the_pool_is_reused_across_calls_and_directories(tmp_path):
    n = 16 * 32768
    cols, rows = columns(n, seed=9)
    want = b"".join(rows)
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    first = dev.host_join_tsv(cols, prefix=str(tmp_path / "a" / "part-"))
    started = dev.host_pool_threads()
    assert started <= 15          # at most 16 workers, the caller being one
    for d in ("b", "a", "b"):
        names = dev.host_join_tsv(cols, prefix=str(tmp_path / d / "part-"))
        assert len(names) == len(first)
        assert b"".join(open(x, "rb").read() for x in names) == want
    assert dev.host_join_tsv(cols).tobytes() == want
    uniq, inv = dev.host_unique_small(np.arange(n, dtype=np.int64) % 1000)
    assert np.array_equal(uniq[inv], np.arange(n) % 1000)
    assert dev.host_pool_threads() == started
    split = dev.host_sink_timings()
    assert set(split) == {"prep", "start", "open", "format", "write", "close"} and all(v >= 0 for v in split.values())


def test_rows_beyond_the_kept_buffers_are_written_the_same(tmp_path, monkeypatch):
    n = 2 * 32768 + 11
    cols, rows = columns(n, seed=2)
    monkeypatch.setattr(settings, "host_result_cache_bytes", 4096)   # every writer's rows exceed its share
    small = dev.host_join_tsv(cols, prefix=str(tmp_path / "small-"))
    monkeypatch.setattr(settings, "host_result_cache_bytes", 64 << 20)
    kept = dev.host_join_tsv(cols, prefix=str(tmp_path / "kept-"))
    again = dev.host_join_tsv(cols[:1] + cols[3:], prefix=str(tmp_path / "again-"))   # shorter rows, same buffers
    want = b"".join(rows)
    assert b"".join(open(x, "rb").read() for x in small) == want
    assert b"".join(open(x, "rb").read() for x in kept) == want
    assert b"".join(open(x, "rb").read() for x in again) == \
        b"".join(r.split(b"\t")[0] + b"\t" + r.split(b"\t")[3] for r in rows)

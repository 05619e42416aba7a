"""Result downloads through the context's page-locked arena (leases) against the pageable path: the token table, the
count dictionary, tables with hashed tokens and with host lines, back-to-back TF-IDF runs on one context, and results
larger than the arena's bound."""
import gc
import math
import os
import re

import numpy as np
import pytest

from dampr_b200 import Dampr
from dampr_b200 import device as dev
from dampr_b200 import plan, settings
from dampr_b200 import runner as runner_mod
from oracle import gen, refsem

pytestmark = pytest.mark.gpu

RX = re.compile(r"[^\w]+")


@pytest.fixture(scope="module")
def ctx():
    return runner_mod.get_ctx()


def lease_of(arr):
    """the ResultLease an array's memory belongs to, or None"""
    while arr is not None and not isinstance(arr, dev.ResultLease):
        arr = getattr(arr, "base", None)
    return arr


def scan_table(ctx, data, mode=dev.TOK_NONWORD_LOWER_SET):
    tb = dev.TextBuf(ctx, len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = dev.Table(ctx, 20)
    tab.clear()
    tab.count(tb, 0, tb.n, mode)
    return tb, tab


def fetch_both(ctx, tb, tab, mode, width, with_codes, monkeypatch):
    """(leased fetch, pageable fetch) of one table, each with its count dictionary"""
    monkeypatch.setattr(settings, "host_result_cache_bytes", 64 << 20)
    a = tab.fetch_words(tb, mode, width, with_codes)
    da = ctx.count_dictionary(*tab.extracted_counts())
    assert lease_of(a[0]) is not None and lease_of(a[1]) is lease_of(a[0]) and lease_of(da[1]) is not None
    monkeypatch.setattr(settings, "host_result_cache_bytes", 0)
    b = tab.fetch_words(tb, mode, width, with_codes)
    db = ctx.count_dictionary(*tab.extracted_counts())
    assert lease_of(b[0]) is None and lease_of(b[1]) is None and lease_of(db[1]) is None
    return a, da, b, db


def same(a, da, b, db):
    # the extract kernel's row order is its own from launch to launch: compare as sets of rows
    oa, ob = np.argsort(a[0], kind="stable"), np.argsort(b[0], kind="stable")
    for x, y in zip(a, b):
        assert (x is None) == (y is None)
        if x is not None:
            assert x.dtype == y.dtype and np.array_equal(x[oa], y[ob])
    assert np.array_equal(da[0], db[0])
    assert np.array_equal(da[0][da[1]][oa], db[0][db[1]][ob])
    assert da[2].dtype == db[2].dtype == np.int64
    assert np.array_equal(a[1][da[2]].view(np.int64), da[0]) and np.array_equal(b[1][db[2]].view(np.int64), db[0])


def test_zipf_table_through_leases_equals_the_pageable_path(ctx, monkeypatch):
    data = gen.text(7, 60_000, V=50_000)
    tb, tab = scan_table(ctx, data)
    a, da, b, db = fetch_both(ctx, tb, tab, dev.TOK_NONWORD_LOWER_SET, 16, False, monkeypatch)
    assert len(a[0]) > 10_000 and a[2] is None
    same(a, da, b, db)


def test_hashed_tokens_with_codes_and_reps(ctx, monkeypatch):
    longs = [b"x" * 13, b"averyveryverylongtoken_%d" % 5, b"q" * 40]
    lines = [b" ".join([b"short", longs[i % 3], b"w%d" % (i % 97)]) for i in range(5000)]
    data = b"\n".join(lines) + b"\n"
    tb, tab = scan_table(ctx, data)
    assert tab.stats()["hashed"]
    a, da, b, db = fetch_both(ctx, tb, tab, dev.TOK_NONWORD_LOWER_SET, 32, True, monkeypatch)
    same(a, da, b, db)
    assert (b"q" * 32) in a[0].tolist()     # truncated to the width: its length is in reps


def tfidf(source, out):
    docs = Dampr.read_input(source)
    doc_freq = docs.flat_map(lambda x: set(RX.split(x.lower()))).count(reduce_buffer=float("inf"))
    idf = doc_freq.cross_right(docs.len(), lambda df, total: (df[0], df[1], math.log(1 + (float(total) / df[1]))),
                               memory=True)
    idf.sink_tsv(out).run()
    # (the table extract's row order is its own from launch to launch: the lines are compared sorted)
    return sorted(l for fn in os.listdir(out) for l in open(os.path.join(out, fn), "rb").read().splitlines())


def oracle_lines(data):
    return sorted(l.encode("utf-8") for l in refsem.tfidf_sink_lines(data))


def test_long_tokens_and_host_lines_take_the_same_rows(monkeypatch, tmp_path):
    # a token longer than the fetch width (patched from the text) and non-ASCII lines (tokenised on the host)
    base = gen.text(21, 8000, V=4000)
    data = base + (b"tok " + b"z" * 45 + b" end\n") * 3 + "café naïve café\n".encode("utf-8") * 2
    src = plan.MemoryText(np.frombuffer(data, dtype=np.uint8))
    monkeypatch.setattr(settings, "host_result_cache_bytes", 64 << 20)
    a = tfidf(src, str(tmp_path / "a"))
    monkeypatch.setattr(settings, "host_result_cache_bytes", 0)
    b = tfidf(src, str(tmp_path / "b"))
    assert a == b
    assert any(l.startswith(b"z" * 45 + b"\t3\t") for l in a)
    assert any(l.startswith("café\t2\t".encode("utf-8")) for l in a)


def test_two_runs_on_one_context_keep_the_first_runs_words(ctx, monkeypatch, tmp_path):
    monkeypatch.setattr(settings, "host_result_cache_bytes", 64 << 20)
    kept = []
    orig = dev.Table.fetch_words

    def keeping(self, *a, **kw):
        r = orig(self, *a, **kw)
        kept.append((r[0], r[0].copy(), r[1], r[1].copy()))
        return r
    monkeypatch.setattr(dev.Table, "fetch_words", keeping)
    d1, d2 = gen.text(31, 30_000, V=20_000), gen.text(32, 30_000, V=20_000)
    a1 = tfidf(plan.MemoryText(np.frombuffer(d1, dtype=np.uint8)), str(tmp_path / "a1"))
    a2 = tfidf(plan.MemoryText(np.frombuffer(d2, dtype=np.uint8)), str(tmp_path / "a2"))
    b1 = tfidf(plan.MemoryText(np.frombuffer(d1, dtype=np.uint8)), str(tmp_path / "b1"))
    gc.collect()
    assert a1 == b1 and a1 != a2
    assert a2 == oracle_lines(d2)
    assert len(kept) == 3
    for words, wcopy, counts, ccopy in kept:     # every run's arrays still hold what that run fetched
        assert np.array_equal(words, wcopy) and np.array_equal(counts, ccopy)


def test_a_result_larger_than_the_bound_falls_back(ctx, monkeypatch, tmp_path):
    data = gen.text(41, 30_000, V=20_000)
    src = plan.MemoryText(np.frombuffer(data, dtype=np.uint8))
    seen = []
    orig = dev.Table.fetch_words

    def watching(self, *a, **kw):
        r = orig(self, *a, **kw)
        seen.append(lease_of(r[1]) is not None)
        return r
    monkeypatch.setattr(dev.Table, "fetch_words", watching)
    monkeypatch.setattr(settings, "host_result_cache_bytes", 64 << 10)   # smaller than the table's words
    small = tfidf(src, str(tmp_path / "small"))
    monkeypatch.setattr(settings, "host_result_cache_bytes", 64 << 20)
    full = tfidf(src, str(tmp_path / "full"))
    assert seen == [False, True]
    assert small == full and full == oracle_lines(data)


def test_leases_are_reused_and_survive_each_other(ctx):
    lib = ctx.lib
    import ctypes as C
    dev._apply_result_cache()
    p1, l1, p2, l2 = C.c_void_p(), C.c_uint64(), C.c_void_p(), C.c_uint64()
    ctx.check(lib.dampr_result_lease(ctx.h, 3 << 20, C.byref(p1), C.byref(l1)))
    ctx.check(lib.dampr_result_lease(ctx.h, 3 << 20, C.byref(p2), C.byref(l2)))
    assert l1.value and l2.value and l1.value != l2.value and p1.value != p2.value
    ctx.check(lib.dampr_result_release(ctx.h, l1.value))
    p3, l3 = C.c_void_p(), C.c_uint64()
    ctx.check(lib.dampr_result_lease(ctx.h, 2 << 20, C.byref(p3), C.byref(l3)))
    assert p3.value == p1.value          # the free block is taken again
    big, lb = C.c_void_p(), C.c_uint64()
    ctx.check(lib.dampr_result_lease(ctx.h, (64 << 20) + 1, C.byref(big), C.byref(lb)))
    assert not lb.value and not big.value
    ctx.check(lib.dampr_result_release(ctx.h, l2.value))
    ctx.check(lib.dampr_result_release(ctx.h, l3.value))

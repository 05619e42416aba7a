"""The dictionary of a text scan's count column built on the device (dampr_count_dictionary) against the host's
unique_inverse_rows on the same counts, and the TF-IDF graph that uses it against the oracle."""
import math
import re
import tempfile
import os

import numpy as np
import pytest

from dampr_b200 import Dampr
from dampr_b200 import device as dev
from dampr_b200 import plan
from dampr_b200 import runner as runner_mod
from oracle import gen, refsem

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return runner_mod.get_ctx()


def zipf_counts(n, seed=3):
    """document frequencies of a Zipf(1.1) vocabulary of n terms over ~10^8 lines, in table (hash) order"""
    r = np.arange(1, n + 1, dtype=np.float64)
    df = np.maximum(1, (1.5e8 * r ** -1.1)).astype(np.int64)
    return np.random.default_rng(seed).permutation(df)


def check(ctx, counts, extra=()):
    counts = np.asarray(counts, dtype=np.int64)
    full = np.concatenate((counts, np.asarray(extra, dtype=np.int64)))
    plan.forget_count_dictionary()
    uniq, inv, _rep = plan.unique_inverse_rows(full)          # the host's dictionary
    got = ctx.count_dictionary_of(counts, extra)
    assert got is not None
    duniq, dinv, drows = got
    assert duniq.dtype == np.int64 and dinv.dtype == np.uint32 and drows.dtype == np.int64
    assert np.array_equal(duniq, uniq)
    assert np.array_equal(dinv, inv)
    # one row per value: the smallest row holding it
    _u, first = np.unique(full, return_index=True)
    assert np.array_equal(drows, first)
    return len(duniq)


def test_zipf_table(ctx):
    m = check(ctx, zipf_counts(1_000_000))
    assert 5_000 < m < 30_000


def test_all_equal(ctx):
    assert check(ctx, np.full(300_000, 41, dtype=np.int64)) == 1


def test_above_the_presence_table(ctx):
    rng = np.random.default_rng(5)
    # every value beyond the largest presence table (2^22 entries): the sort-and-fold path alone, with repeats
    vals = rng.integers(1 << 23, 1 << 40, 3000)
    counts = vals[rng.integers(0, len(vals), 20_000)]
    check(ctx, counts)
    # mixed: small values plus a few beyond the bound of a small column
    check(ctx, np.concatenate((rng.integers(0, 50, 10_000), rng.integers(1 << 20, 1 << 24, 500))))


def test_empty_token_row_appended(ctx):
    counts = zipf_counts(200_000, seed=11)
    check(ctx, counts, [12345])
    check(ctx, counts, [int(counts[17])])          # a value already present
    check(ctx, counts, [1 << 33])                  # beyond the bound
    check(ctx, np.zeros(0, dtype=np.int64), [7])   # the '' row alone


def test_negative_values_are_left_to_the_host(ctx):
    assert ctx.count_dictionary_of(np.array([3, -1, 5] * 2000, dtype=np.int64)) is None


def test_tfidf_takes_the_device_dictionary(monkeypatch):
    RX = re.compile(r"[^\w]+")
    data = gen.text(99, 40_000, V=20_000)
    calls = []
    orig = dev.Ctx.count_dictionary

    def counted(self, *a, **kw):
        r = orig(self, *a, **kw)
        calls.append(r is not None)
        return r
    monkeypatch.setattr(dev.Ctx, "count_dictionary", counted)
    out = os.path.join(tempfile.mkdtemp(prefix="dampr_tail_"), "idfs")
    docs = Dampr.read_input(plan.MemoryText(np.frombuffer(data, dtype=np.uint8)))
    doc_freq = docs.flat_map(lambda x: set(RX.split(x.lower()))).count(reduce_buffer=float("inf"))
    idf = doc_freq.cross_right(docs.len(), lambda df, total: (df[0], df[1], math.log(1 + (float(total) / df[1]))),
                               memory=True)
    idf.sink_tsv(out).run()
    lines = []
    for fn in os.listdir(out):
        with open(os.path.join(out, fn)) as f:
            lines.extend(l.rstrip("\n") for l in f)
    assert sorted(lines) == refsem.tfidf_sink_lines(data)
    assert calls == [True]

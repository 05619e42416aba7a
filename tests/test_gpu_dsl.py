"""DSL parity on the GPU: the known-answer literals of the reference's own suite
(reference tests/test_dampr.py, cited per test) re-stated against the device runner.  Every shuffle
in here goes through libdampr_b200 (host map + device partition/sort, or a lowered pipeline)."""
import heapq
import itertools
import os
import shutil

import pytest

from dampr_b200 import Dampr, BlockMapper, BlockReducer, Dataset, settings
from dampr_b200.utils import filter_by_count

pytestmark = pytest.mark.gpu


class RangeDataset(Dataset):
    def __init__(self, n):
        self.n = n

    def read(self):
        for i in range(self.n):
            yield i, i


@pytest.fixture
def items(ctx):
    return Dampr.memory(list(range(10, 20)), partitions=2)


def test_identity_and_map(items):  # test_dampr.py:23-29
    assert list(items.run()) == list(range(10, 20))
    assert list(items.map(lambda x: x + 1).run()) == list(range(11, 21))


def test_group_count_and_sum(items):  # :31-61
    res = items.group_by(lambda x: 1, lambda x: 1).reduce(lambda k, it: sum(it)).run()
    assert next(iter(res))[1] == 10
    assert next(iter(items.count(lambda x: None).run())) == (None, 10)
    res = items.group_by(lambda x: 1).reduce(lambda k, it: sum(it)).run()
    assert next(iter(res))[1] == sum(range(10, 20))
    res = items.group_by(lambda v: v % 2).reduce(lambda k, it: sum(it)).run()
    assert [kv[1] for kv in res] == [10 + 12 + 14 + 16 + 18, 11 + 13 + 15 + 17 + 19]


def test_filter_and_sort(items):  # :63-73
    assert list(items.filter(lambda i: i % 2 == 1).run()) == [11, 13, 15, 17, 19]
    assert list(items.sort_by(lambda x: -x).run()) == [19, 18, 17, 16, 15, 14, 13, 12, 11, 10]


def test_reduce_join(items):  # :75-85
    items2 = Dampr.memory(list(range(10)))
    res = items.group_by(lambda x: x % 2).join(items2.group_by(lambda x: x % 2)) \
        .reduce(lambda l, r: list(sorted(itertools.chain(l, r)))).run()
    out = list(res)
    assert out[0] == (0, [0, 2, 4, 6, 8, 10, 12, 14, 16, 18])
    assert out[1] == (1, [1, 3, 5, 7, 9, 11, 13, 15, 17, 19])


def test_disjoint_and_repartition(items):  # :87-106
    items2 = Dampr.memory(list(range(10))).group_by(lambda x: -x)
    assert [v for k, v in items.group_by(lambda x: x).join(items2).run()] == []
    items3 = Dampr.memory(list(range(10))).group_by(lambda x: -x).reduce(lambda k, vs: sum(vs))
    assert [v for k, v in items.group_by(lambda x: x).join(items3).run()] == []


def test_associative_reduce(items):  # :108-116
    out = list(items.a_group_by(lambda x: x % 2).reduce(lambda x, y: x + y).run())
    assert out[0][1] == 10 + 12 + 14 + 16 + 18
    assert out[1][1] == 11 + 13 + 15 + 17 + 19


def test_left_join(items):  # :118-130
    to_remove = Dampr.memory(list(range(10, 13)))
    out = items.group_by(lambda x: x).join(to_remove.group_by(lambda x: x)) \
        .left_reduce(lambda l, r: (list(l), list(r))) \
        .filter(lambda llrs: len(llrs[1][1]) == 0) \
        .map(lambda llrs: llrs[1][0][0]) \
        .sort_by(lambda x: x).run()
    assert list(out) == list(range(13, 20))


def test_multi_output_run(items):  # :132-138
    even = items.filter(lambda x: x % 2 == 0)
    odd = items.filter(lambda x: x % 2 == 1)
    ev, od = Dampr.run(even, odd)
    assert list(ev) == [10, 12, 14, 16, 18]
    assert list(od) == [11, 13, 15, 17, 19]


def test_reduce_many(items):  # :140-159
    even = items.filter(lambda x: x % 2 == 0)
    odd = items.filter(lambda x: x % 2 == 1)

    def cross(x, y):
        y = list(y)
        for xi in x:
            for yi in y:
                yield xi * yi

    results = even.group_by(lambda x: 1).join(odd.group_by(lambda x: 1)).reduce(cross, many=True).run().read()
    e, o = [10, 12, 14, 16, 18], [11, 13, 15, 17, 19]
    assert sorted(results) == sorted((1, ei * oi) for ei in e for oi in o)


def test_fold_by_and_empty(items):  # :161-181
    out = items.fold_by(lambda x: 1, value=lambda x: x % 2, binop=lambda x, y: x + y)
    assert list(out.run()) == [(1, 5)]
    out = items.sample(0.0).fold_by(lambda x: 1, value=lambda x: x % 2, binop=lambda x, y: x + y)
    assert list(out.run()) == []


def test_sink_and_cached(items, tmp_path):  # :183-209
    path = str(tmp_path / "sink")
    sink = items.map(lambda x: str(x)).sink(path=path)
    assert sorted(sink.count().run()) == [("%d" % i, 1) for i in range(10, 20)]
    assert os.path.isdir(path)
    cached = items.map(lambda x: str(x)).cached()
    cached.run()
    assert sorted(cached.count().run()) == [(str(i), 1) for i in range(10, 20)]


def test_cross_joins(items):  # :211-237, :313-330
    total = items.a_group_by(lambda x: 1).sum()
    out = items.cross_right(total, lambda v1, v2: round(v1 / float(v2[1]), 4)).sort_by(lambda x: x)
    count = sum(range(10, 20))
    assert sorted(out.run()) == [round(i / float(count), 4) for i in range(10, 20)]
    out = items.cross_left(items, lambda v1, v2: v1 * v2)
    assert sorted(out.run()) == sorted(i * k for i in range(10, 20) for k in range(10, 20))
    item_counts = items.count()
    tot = items.a_group_by(lambda x: 1, lambda x: 1).sum().map(lambda x: float(x[1]))
    res = item_counts.cross_right(tot, lambda ic, t: (ic[0], ic[1] / t)).read()
    assert sorted(res) == [(i, 1 / float(10)) for i in range(10, 20)]


def test_cross_set_orientation(ctx):
    """Code behaviour, not the docstring, is the contract (SURVEY B4): streams `other`."""
    left = Dampr.memory([1, 2, 3, 4, 5])
    right = Dampr.memory([3, 5])
    assert sorted(left.cross_set(right, lambda x, y: (x, x in y), agg=set).read()) == [(3, True), (5, True)]


def test_blocks(ctx):  # :239-311
    class TopKMapper(BlockMapper):
        def __init__(self, k):
            self.k = k

        def start(self):
            self.heap = []

        def add(self, _k, lc):
            heapq.heappush(self.heap, (lc[1], lc[0]))
            if len(self.heap) > self.k:
                heapq.heappop(self.heap)
            return iter([])

        def finish(self):
            for cl in self.heap:
                yield 1, cl

    class TopKReducer(BlockReducer):
        def __init__(self, k):
            self.k = k

        def add(self, k, it):
            for count, letter in heapq.nlargest(self.k, it):
                yield letter, (letter, count)

    word = Dampr.memory(["supercalifragilisticexpialidociousa"])
    letter_counts = word.flat_map(lambda w: list(w)).count()
    topk = letter_counts.custom_mapper(TopKMapper(2)).custom_reducer(TopKReducer(2))
    assert sorted(topk.run()) == [("a", 4), ("i", 7)]

    def map_topk(it):
        heap = []
        for symbol, count in it:
            heapq.heappush(heap, (count, symbol))
            if len(heap) > 2:
                heapq.heappop(heap)
        return ((1, x) for x in heap)

    def reduce_topk(it):
        counts = (v for k, vit in it for v in vit)
        for count, symbol in heapq.nlargest(2, counts):
            yield symbol, count

    topk = letter_counts.partition_map(map_topk).partition_reduce(reduce_topk)
    assert sorted(topk.run()) == [("a", 4), ("i", 7)]
    top5 = word.flat_map(lambda w: list(w)).count().topk(5, lambda x: x[1])
    assert sorted(top5.run()) == [("a", 4), ("c", 3), ("i", 7), ("l", 3), ("s", 3)]


def test_len(items):  # :332-338
    assert items.len().read() == [10]
    assert Dampr.memory([]).len().read() == [0]


def test_read_input(ctx):  # :358-367
    results = Dampr.read_input(RangeDataset(5), RangeDataset(10)).fold_by(lambda x: 1, lambda x, y: x + y).read()
    assert results[0][1] == sum(range(5)) + sum(range(10))


def test_file_glob_and_links(ctx, tmp_path):  # :380-462
    for i in range(10):
        (tmp_path / ("_test_dampr_%d" % i)).write_text(str(i))
    res = Dampr.text(str(tmp_path / "_test_dampr_[135]")).map(int).fold_by(lambda x: 1, lambda x, y: x + y).read()
    assert res == [(1, 1 + 3 + 5)]
    dirs = []
    for i in range(10):
        d = tmp_path / ("dir_%d" % i)
        d.mkdir()
        (d / "foo").write_text(str(i))
        dirs.append(d)
    base = tmp_path / "links"
    base.mkdir()
    for i in (1, 3, 5):
        os.symlink(str(dirs[i]), str(base / dirs[i].name))
    assert Dampr.text(str(base)).map(int).fold_by(lambda x: 1, lambda x, y: x + y).read() == []
    assert Dampr.text(str(base), followlinks=True).map(int).fold_by(lambda x: 1, lambda x, y: x + y).read() \
        == [(1, 1 + 3 + 5)]


def test_tuple_helpers(items):  # :475-527
    pairs = items.map(lambda item: (item, item))
    assert sorted(pairs.map_values(lambda v: v + 1).read()) == list(zip(range(10, 20), range(11, 21)))
    assert sorted(pairs.map_keys(lambda v: v + 1).read()) == list(zip(range(11, 21), range(10, 20)))
    assert sorted(items.prefix(lambda item: item + 1).read()) == list(zip(range(11, 21), range(10, 20)))
    assert sorted(items.suffix(lambda item: item + 1).read()) == list(zip(range(10, 20), range(11, 21)))


def test_filter_by_count(ctx):  # :529-545
    words = ["one", "two", "three", "four", "five", "six", "seven", "eight", "nine", "ten"]
    pipe = Dampr.memory(words)
    res = filter_by_count(pipe, lambda line: len(line), lambda cnt: cnt >= 4).read()
    assert sorted(res) == sorted(["one", "two", "six", "ten"])
    res = filter_by_count(pipe, lambda line: len(line), lambda cnt: cnt < 4).read()
    assert sorted(res) == sorted(["three", "four", "five", "seven", "eight", "nine"])


# ---- semantics the reference's suite does not pin (SURVEY §4 last bullet) ----------------------
def test_mean_first_unique(ctx):
    ages = [("Andrew", 33), ("Alice", 42), ("Andrew", 12), ("Bob", 51)]
    assert sorted(Dampr.memory(ages).mean(lambda x: x[0], lambda v: v[1]).read()) == \
        [("Alice", 42.0), ("Andrew", 22.5), ("Bob", 51.0)]
    assert sorted(Dampr.memory([1, 2, 3, 4, 5]).a_group_by(lambda x: x % 2).first().read()) == [(0, 2), (1, 1)]
    names = [("Andrew", 1), ("Andrew", 1), ("Andrew", 2), ("Becky", 13)]
    assert sorted(Dampr.memory(names).group_by(lambda x: x[0], lambda x: x[1]).unique().read()) == \
        [("Andrew", [1, 2]), ("Becky", [13])]


def test_mixed_and_big_keys(ctx):
    data = [(2 ** 70, 1), (2 ** 70, 2), ("a", 3), (("t", 1), 4), (("t", 1), 5), (None, 6), (1.5, 7), (1, 8), (1.0, 9)]
    got = dict(Dampr.memory(data).a_group_by(lambda x: x[0], lambda x: x[1]).sum().read())
    assert got == {2 ** 70: 3, "a": 3, ("t", 1): 9, None: 6, 1.5: 7, 1: 17}
    strs = ["pear", "apple", "fig", "apple", "applesauce", "applesauce!", "fig"]
    assert Dampr.memory(strs).count().read() == [("apple", 2), ("applesauce", 1), ("applesauce!", 1), ("fig", 2), ("pear", 1)]
    assert Dampr.memory(strs).sort_by(lambda s: s).read() == sorted(strs)


def test_unknown_kwargs_accepted(items):
    assert items.map(lambda x: x).read(n_partitions=1, n_maps=2, n_reducers=3, max_files_per_stage=7) == list(range(10, 20))


def test_word_stats_example(ctx, tmp_path):
    """The pipeline of the reference's examples/word-stats.py (one shared root, four outputs from one
    Dampr.run, a join of two aggregates) against plain Python on the same file."""
    import collections
    import random
    rng = random.Random(5)
    vocab = ["w%d" % i for i in range(300)] + ["Supercalifragilistic", "naïve", "x", "antidisestablishment"]
    lines = [" ".join(rng.choice(vocab) for _ in range(rng.randint(0, 12))) for _ in range(4000)]
    path = tmp_path / "corpus.txt"
    path.write_text("\n".join(lines) + "\n", encoding="utf-8")

    words = Dampr.text(str(path), 1024 ** 2).flat_map(lambda line: line.split())
    top_words = words.count(lambda x: x).sort_by(lambda wc: -wc[1])
    total_count = top_words.fold_by(key=lambda word: 1, value=lambda x: x[1], binop=lambda x, y: x + y)
    word_lengths = top_words \
        .fold_by(lambda tc: len(tc[0]), value=lambda tc: tc[1], binop=lambda x, y: x + y) \
        .sort_by(lambda cl: cl[0])
    avg = word_lengths \
        .map(lambda wl: wl[0] * wl[1]) \
        .a_group_by(lambda x: 1).sum() \
        .join(total_count) \
        .reduce(lambda awl, tc: next(awl)[1] / float(next(tc)[1]))
    tc, tw, wl, awl = Dampr.run(total_count, top_words, word_lengths, avg, name="word-stats")

    exp = collections.Counter(w for line in lines for w in line.split())
    n = sum(exp.values())
    assert tc.read(1)[0][1] == n
    got = list(tw)
    assert dict(got) == dict(exp)
    hist = collections.Counter()
    for w, c in exp.items():
        hist[len(w)] += c
    assert sorted(wl) == sorted(hist.items())
    assert awl.read(1)[0][1] == sum(k * v for k, v in hist.items()) / float(n)


def test_frame_stages_evaluated_column_at_a_time(ctx):
    """Stages that follow an aggregation (map / filter / map_values / fold_by / mean / sort_by on
    computed keys) run over the aggregate's columns (dampr_b200/vexpr.py) with CPython's results."""
    import numpy as np
    from dampr_b200.inputs import ArrayKVInput
    from dampr_b200 import runner as runner_mod

    def how():
        return [h for _s, h, _d in runner_mod.LAST_STATS.stages]

    rng = np.random.default_rng(11)
    keys = rng.integers(-500, 500, size=60000).astype(np.int64)
    vals = rng.integers(-1000, 1000, size=60000).astype(np.int64)
    agg = Dampr.read_input(ArrayKVInput(keys, vals)).a_group_by(lambda x: x[0], lambda x: x[1]).sum()
    exp = {}
    for k, v in zip(keys.tolist(), vals.tolist()):
        exp[k] = exp.get(k, 0) + v
    rows = sorted(exp.items())

    got = agg.map(lambda kv: (kv[0], kv[1] * 3 - kv[0], kv[1] / 7)).read()
    assert any("column-at-a-time" in h for h in how())
    assert sorted(got) == [(k, v * 3 - k, v / 7) for k, v in rows]

    got = agg.filter(lambda kv: kv[1] > 0).map_values(lambda v: v // 5).read()
    assert any("column-at-a-time" in h for h in how())
    assert sorted(got) == [(k, v // 5) for k, v in rows if v > 0]

    got = agg.fold_by(lambda kv: kv[0] % 7, lambda x, y: x + y, value=lambda kv: kv[1]).read()
    assert any("frame keyed fold" in h for h in how())
    e2 = {}
    for k, v in rows:
        e2[k % 7] = e2.get(k % 7, 0) + v
    assert sorted(got) == sorted(e2.items())

    got = agg.mean(lambda kv: abs(kv[0]) % 5, lambda kv: kv[1]).read()
    assert any("frame keyed fold" in h for h in how())
    e3 = {}
    for k, v in rows:
        s, c = e3.get(abs(k) % 5, (0, 0))
        e3[abs(k) % 5] = (s + v, c + 1)
    assert sorted(got) == sorted((k, s / float(c)) for k, (s, c) in e3.items())

    got = agg.mean(value=lambda kv: float(kv[1])).read()
    tot = 0.0
    # order of the float left fold is the frame's row order: compare with tolerance
    assert len(got) == 1 and got[0][0] == 1
    assert abs(got[0][1] - sum(v for _k, v in rows) / float(len(rows))) < 1e-9

    got = agg.sort_by(lambda kv: kv[1] - 2 * kv[0]).read()
    assert any("device sort of frame rows" in h for h in how())
    assert [r[1] - 2 * r[0] for r in got] == sorted(v - 2 * k for k, v in rows) and sorted(got) == rows

    # a guard trips (division by zero somewhere): the host path must give CPython's behaviour
    with pytest.raises(ZeroDivisionError):
        agg.map(lambda kv: kv[1] / (kv[0] - kv[0])).read()

"""The Dampr DSL on top of the device engine.

Public surface = the reference's (dampr/dampr.py:19-977; SURVEY §8(b) "Python signatures to
keep"): Dampr.memory/read_input/text/json/from_dataset/run, PMap.*, ARReduce.*, PReduce.*,
PJoin.*, ValueEmitter.  Pipelines are lazy and immutable; consecutive record-wise operations are
fused into one Map stage.  Unlike the reference every generated Map carries a structured `Op`
descriptor so the runner can lower the closed set of idioms (tokenise, key/value projections,
associative folds) to CUDA and keep arbitrary Python as a host map in front of the device shuffle.
"""
import heapq
import itertools
import json
import operator
import random
import sys
import time

from . import operators as ops
from .operators import Op, Map, fuse
from .graph import Graph, Source
from .datasets import Chunker, CatDataset
from .inputs import MemoryInput, PathInput


class ValueEmitter(object):
    """Reads the values of a finished computation (dampr.py:19-51)."""

    def __init__(self, datasets):
        self.datasets = datasets

    def stream(self):
        for _k, v in self.datasets.read():
            yield v

    def read(self, k=None):
        it = self.stream()
        return list(it) if k is None else list(itertools.islice(it, k))

    def __iter__(self):
        return self.stream()

    def delete(self):
        self.datasets.delete()


class PBase(object):
    def __init__(self, source, pmer):
        assert isinstance(source, Source)
        self.source = source
        self.pmer = pmer

    def run(self, name=None, **kwargs):
        """Evaluate the graph; returns a ValueEmitter over this node's output (dampr.py:62-74)."""
        if name is None:
            name = "dampr/%s" % random.random()
        out = self.pmer.runner(name, self.pmer.graph, **kwargs).run([self.source])
        return ValueEmitter(out[0])

    def read(self, k=None, **kwargs):
        return self.run(**kwargs).read(k)


def _identity(k, v):
    yield k, v


class PMap(PBase):
    """A collection under construction; record-wise operations accumulate in `agg` and are fused
    when a stage boundary (checkpoint) is needed (dampr.py:85-153)."""

    def __init__(self, source, pmer, agg=None):
        PBase.__init__(self, source, pmer)
        self.agg = list(agg) if agg else []

    # -- plumbing ---------------------------------------------------------------------------
    def run(self, name=None, **kwargs):
        if self.agg:
            return self.checkpoint().run(name, **kwargs)
        return PBase.run(self, name, **kwargs)

    def _add_mapper(self, mapper):
        assert isinstance(mapper, ops.Streamable)
        return PMap(self.source, self.pmer, self.agg + [mapper])

    def _add_map(self, f, op=None):
        return self._add_mapper(Map(f, op))

    def _stage_name(self, aggs):
        return "Stage {}: %s" % " -> ".join(str(a) for a in aggs)

    def checkpoint(self, force=False, combiner=None, options=None):
        """Materialise the pending fused maps as one Map stage (dampr.py:128-153)."""
        if not self.agg and not force:
            return self
        aggs = self.agg if self.agg else [Map(_identity, Op("identity"))]
        source, pmer = self.pmer._add_mapper([self.source], fuse(aggs), combiner=combiner,
                                             name=self._stage_name(aggs), options=options)
        return PMap(source, pmer)

    def custom_mapper(self, mapper, name=None, **options):
        if isinstance(mapper, ops.Streamable):
            return self._add_mapper(mapper)
        assert isinstance(mapper, ops.Mapper)
        me = self.checkpoint()
        source, pmer = me.pmer._add_mapper([me.source], mapper, name=name or str(mapper), options=options)
        return PMap(source, pmer)

    def custom_reducer(self, reducer, name=None, **options):
        assert isinstance(reducer, ops.Reducer)
        me = self.checkpoint(force=True)
        source, pmer = me.pmer._add_reducer([me.source], reducer, name=name or str(reducer), options=options)
        return PMap(source, pmer)

    def partition_map(self, f, **options):
        """f(iterator of values) -> iterator of (key, value) records, once per input chunk."""
        return self.custom_mapper(ops.StreamMapper(f), **options)

    def partition_reduce(self, f):
        """f(iterator of (key, values_iter)) -> iterator of (key, value)."""
        return self.custom_reducer(ops.StreamReducer(f))

    # -- record-wise operations -------------------------------------------------------------
    def map(self, f):
        def _map(k, v):
            yield k, f(v)
        return self._add_map(_map, Op("map", f))

    def filter(self, f):
        def _filter(k, v):
            if f(v):
                yield k, v
        return self._add_map(_filter, Op("filter", f))

    def flat_map(self, f):
        def _flat_map(k, v):
            for vi in f(v):
                yield k, vi
        return self._add_map(_flat_map, Op("flat_map", f))

    def map_values(self, f):
        return self.map(lambda v: (v[0], f(v[1])))

    def map_keys(self, f):
        return self.map(lambda v: (f(v[0]), v[1]))

    def prefix(self, f):
        return self.map(lambda v: (f(v), v))

    def suffix(self, f):
        return self.map(lambda v: (v, f(v)))

    def sample(self, prob):
        assert 0 <= prob <= 1.0

        def _sample(k, v):
            if _rng().random() < prob:
                yield k, v
        return self._add_map(_sample, Op("sample", prob))

    def inspect(self, prefix="", exit=False):
        def _inspect(k, v):
            print("{}: {}".format(prefix, v))
            yield k, v
        ins = self._add_map(_inspect, Op("inspect"))
        if exit:
            ins.run()
            sys.exit(0)
        return ins

    # -- keyed operations -------------------------------------------------------------------
    def _keyed(self, key, vf):
        def _keyed(_k, v):
            yield key(v), vf(v)
        return self._add_map(_keyed, Op("keyed", key, vf))

    def group_by(self, key, vf=lambda x: x):
        pm = self._keyed(key, vf).checkpoint()
        return PReduce(pm.source, pm.pmer)

    def a_group_by(self, key, vf=lambda x: x):
        return ARReduce(self._keyed(key, vf))

    def fold_by(self, key, binop, value=lambda x: x, **options):
        return self.a_group_by(key, value).reduce(binop, **options)

    def sort_by(self, key, **options):
        def _sort_by(_k, v):
            yield key(v), v
        return self._add_map(_sort_by, Op("keyed", key, _ident)).checkpoint(options=options)

    def count(self, key=lambda x: x, **options):
        return self.a_group_by(key, _one).reduce(operator.add, **options)

    def mean(self, key=lambda x: 1, value=lambda x: x, **options):
        def _pair_add(x, y):
            return x[0] + y[0], x[1] + y[1]
        return self.a_group_by(key, lambda v: (value(v), 1)) \
            .reduce(_pair_add, **options) \
            .map(lambda kv: (kv[0], kv[1][0] / float(kv[1][1])))

    def len(self):
        """Number of records, as a one-element collection ([0] for an empty input)."""
        def _map_count(items):
            n = 0
            for _ in items:
                n += 1
            yield 1, n

        def _reduce_count(groups):
            total, seen = 0, False
            for _k, counts in groups:
                seen = True
                for c in counts:
                    total += c
            if seen:
                yield 1, total

        return self.custom_mapper(ops.StreamMapper(_map_count, Op("count_records"))) \
            .custom_reducer(ops.StreamReducer(_reduce_count, Op("sum_counts"))) \
            .map(lambda kv: kv[1])

    def topk(self, k, value=None):
        if value is None:
            value = _ident

        def _map_topk(it):
            heap = []
            for x in it:
                heapq.heappush(heap, (value(x), x))
                if len(heap) > k:
                    heapq.heappop(heap)
            return ((1, x) for x in heap)

        def _reduce_topk(groups):
            cands = (v for _k, vit in groups for v in vit)
            for _score, x in heapq.nlargest(k, cands):
                yield x, 1

        # the descriptor lets the planner take the candidates of a columnar frame with one device sort of the
        # scores (plan._lower_topk); every other input runs _map_topk as written
        sm = ops.StreamMapper(_map_topk)
        sm.op = Op("topk", value, k)
        return self.custom_mapper(sm).partition_reduce(_reduce_topk).map(lambda kv: kv[0])

    def join(self, other):
        assert isinstance(other, PBase)
        me = self.checkpoint(True)
        if isinstance(other, PMap):
            other = other.checkpoint(True)
        return PJoin(me.source, Dampr(me.pmer.graph.union(other.pmer.graph), me.pmer.runner), other.source)

    def cached(self, **options):
        options["memory"] = True
        return self.checkpoint(options=options)

    # -- sinks ------------------------------------------------------------------------------
    def sink(self, path):
        aggs = self.agg if self.agg else [Map(_identity, Op("identity"))]
        source, pmer = self.pmer._add_sink([self.source], fuse(aggs), path=path,
                                           name=self._stage_name(aggs), options=None)
        return PMap(source, pmer)

    def sink_tsv(self, path):
        return self.map(_tsv_line).sink(path)

    def sink_json(self, path):
        return self.map(json.dumps).sink(path)

    # -- map-side joins ---------------------------------------------------------------------
    def cross_right(self, other, cross, memory=False):
        """For every item of self (outer) and every item of other (inner): cross(x, y)."""
        assert isinstance(other, PMap)
        def swapped(xi, yi):
            return cross(yi, xi)
        swapped.swapped_of = cross   # lets the frame lowering call the user's function without the hop
        return other.cross_left(self, swapped, memory)

    def cross_left(self, other, cross, memory=False, **options):
        """Outer loop over `other`, inner over self (cached when `memory`); emits cross(self_item,
        other_item) (dampr.py:560-588)."""
        def _cross(k1, v1, k2, v2):
            yield k1, cross(v2, v1)

        me, other = self.checkpoint(), other.checkpoint()
        pmer = Dampr(me.pmer.graph.union(other.pmer.graph), me.pmer.runner)
        mapper = ops.MapCrossJoin(_cross, cache=memory)
        mapper.user_cross = cross
        source, pmer = pmer._add_mapper([other.source, me.source], mapper, combiner=None,
                                        name="Stage {}: Cross", options=options)
        return PMap(source, pmer)

    def cross_set(self, other, cross, agg=None, **options):
        """Streams `other`, passing every item and agg(all values of self) to cross (the code's
        orientation, which is the contract: dampr.py:610-619, SURVEY B4)."""
        def _cross(k1, v1, table):
            yield k1, cross(v1, table)

        agg = list if agg is None else agg

        def _aggregate(d):
            return agg(v for _k, v in d)

        me, other = self.checkpoint(), other.checkpoint()
        pmer = Dampr(me.pmer.graph.union(other.pmer.graph), me.pmer.runner)
        mapper = ops.MapAllJoin(_cross, _aggregate)
        mapper.user_cross, mapper.user_agg = cross, agg
        source, pmer = pmer._add_mapper([other.source, me.source], mapper, combiner=None,
                                        name="Stage {}: CrossAll", options=options)
        return PMap(source, pmer)


def _ident(x):
    return x


def _one(_x):
    return 1


def _tsv_line(x):
    return u"\t".join(str(p) for p in x)


class ARReduce(object):
    """Associative reductions: a partial fold during the map stage, completed in the reduce
    (dampr.py:654-708)."""

    def __init__(self, pmap):
        self.pmap = pmap

    def reduce(self, binop, reduce_buffer=1000, **options):
        def _fold(_key, vs):
            acc = next(vs)
            for v in vs:
                acc = binop(acc, v)
            return acc

        red = ops.Reduce(_fold)
        red.binop = binop
        options.update({"binop": binop, "reduce_buffer": reduce_buffer})  # reduce_buffer: accepted, unused (B5)
        pm = self.pmap.checkpoint(True, combiner=ops.PartialReduceCombiner(red), options=options)
        folded = PReduce(pm.source, pm.pmer)
        new_source, pmer = folded.pmer._add_reducer([folded.source], _keyed_fold(_fold, binop))
        return PMap(new_source, pmer)

    def first(self, **options):
        return self.reduce(_first, **options)

    def sum(self, **options):
        return self.reduce(operator.add, **options)


def _first(x, _y):
    return x


def _keyed_fold(fold, binop):
    r = ops.KeyedReduce(fold)
    r.binop = binop
    return r


class PReduce(PBase):
    """A grouped collection (dampr.py:711-766)."""

    def reduce(self, f):
        source, pmer = self.pmer._add_reducer([self.source], ops.KeyedReduce(f))
        return PMap(source, pmer)

    def unique(self, key=lambda x: x):
        def _uniq(_k, it):
            seen, out = set(), []
            for v in it:
                fv = key(v)
                if fv not in seen:
                    seen.add(fv)
                    out.append(v)
            return out
        red = ops.KeyedReduce(_uniq)
        red.op = Op("unique", key)   # plan._lower_unique: numeric kv records, identity key
        source, pmer = self.pmer._add_reducer([self.source], red)
        return PMap(source, pmer)

    def join(self, other):
        assert isinstance(other, PBase)
        if isinstance(other, PMap):
            other = other.checkpoint(True)
        return PJoin(self.source, Dampr(self.pmer.graph.union(other.pmer.graph), self.pmer.runner), other.source)

    def partition_reduce(self, f):
        source, pmer = self.pmer._add_reducer([self.source], ops.StreamReducer(f))
        return PMap(source, pmer)


class PJoin(PBase):
    """Joins of two grouped collections (dampr.py:768-829)."""

    def __init__(self, source, pmer, right):
        PBase.__init__(self, source, pmer)
        self.right = right

    def run(self, name=None, **kwargs):
        return self.reduce(lambda l, r: (list(l), list(r))).run(name, **kwargs)

    def _join(self, reducer):
        source, pmer = self.pmer._add_reducer([self.source, self.right], reducer)
        return PMap(source, pmer)

    def reduce(self, aggregate, many=False):
        """Inner join: aggregate(left_values_iter, right_values_iter) per key on both sides."""
        r = ops.KeyedInnerJoin(lambda _k, l, rr: aggregate(l, rr), many)
        r.user_aggregate = aggregate
        return self._join(r)

    def left_reduce(self, aggregate):
        """Left join: every left key; the right iterator is empty when the key is missing."""
        r = ops.KeyedLeftJoin(lambda _k, l, rr: aggregate(l, rr))
        r.user_aggregate = aggregate
        return self._join(r)

    def _cross(self, crosser):
        r = ops.KeyedCrossJoin(lambda k1, v1, k2, v2: (k1, crosser(v1, v2)))
        return self._join(r).map(lambda kv: kv[1])


class Dampr(object):
    """Entry point (dampr.py:831-957). `runner` defaults to the device runner and, unlike the
    reference (SURVEY B7), is carried through every derived graph."""

    def __init__(self, graph=None, runner=None):
        self.graph = Graph() if graph is None else graph
        if runner is None:
            from .runner import B200Runner
            runner = B200Runner
        self.runner = runner

    @classmethod
    def memory(cls, items, partitions=50):
        src, g = Graph().add_input(MemoryInput(list(enumerate(items)), partitions))
        return PMap(src, cls(g))

    @classmethod
    def read_input(cls, *datasets):
        if len(datasets) == 1:
            ds = datasets[0]
        else:
            ds = CatDataset(datasets)
        src, g = Graph().add_input(ds)
        return PMap(src, cls(g))

    @classmethod
    def text(cls, fname, chunk_size=16 * 1024 ** 2, followlinks=False):
        return cls.read_input(PathInput(fname, chunk_size, followlinks))

    @classmethod
    def json(cls, *args, **kwargs):
        return cls.text(*args, **kwargs).map(json.loads)

    @classmethod
    def from_dataset(cls, dataset):
        assert isinstance(dataset, Chunker)
        src, g = Graph().add_input(dataset)
        return PMap(src, cls(g))

    @classmethod
    def run(cls, *pmers, **kwargs):
        """Run several graphs in one pass; one ValueEmitter per argument, in order."""
        assert len(pmers) > 0, "Need at least one graph to run!"
        graph, sources, last = None, [], None
        for pm in pmers:
            if isinstance(pm, PMap):
                pm = pm.checkpoint()
            elif isinstance(pm, PJoin):
                pm = pm.reduce(lambda l, r: (list(l), list(r)))
            graph = pm.pmer.graph if graph is None else graph.union(pm.pmer.graph)
            sources.append(pm.source)
            last = pm
        name = kwargs.pop("name", "dampr/%s" % random.random())
        out = last.pmer.runner(name, graph, **kwargs).run(sources)
        return [ValueEmitter(d) for d in out]

    def _add_mapper(self, *args, **kwargs):
        out, g = self.graph.add_mapper(*args, **kwargs)
        return out, Dampr(g, self.runner)

    def _add_reducer(self, *args, **kwargs):
        out, g = self.graph.add_reducer(*args, **kwargs)
        return out, Dampr(g, self.runner)

    def _add_sink(self, *args, **kwargs):
        out, g = self.graph.add_sink(*args, **kwargs)
        return out, Dampr(g, self.runner)


_RNG = None


def _rng():
    global _RNG
    if _RNG is None:
        _RNG = random.Random(time.time())
    return _RNG

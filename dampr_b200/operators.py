"""Operator library: the objects the DSL puts into the stage graph.

Public names and call contracts follow the reference's operator layer (dampr/base.py:1-433:
Mapper.map(*datasets), Streamable.stream(kvs), Reducer.reduce(*datasets), Combiner.combine,
BlockMapper/BlockReducer start/add/finish) because users subclass them.  What differs is who
executes them: the device runner (runner.py) recognises the structured descriptors (`Op`) that the
DSL attaches to its own Map objects, lowers the closed set of idioms to CUDA pipelines and runs
everything else as a host map that feeds the device shuffle.
"""


class Op(object):
    """Structured description of what a DSL-generated Map does (input to the lowering pass)."""
    __slots__ = ("kind", "fn", "fn2")

    def __init__(self, kind, fn=None, fn2=None):
        self.kind = kind  # map | filter | flat_map | keyed | identity | sample | inspect
        self.fn = fn      # user function (map/filter/flat_map) or key function (keyed)
        self.fn2 = fn2    # value function (keyed)

    def __repr__(self):
        return "Op(%s)" % self.kind


class Splitter(object):
    """Kept for API compatibility (base.py:6-8). The device engine partitions on key-code bits."""

    def partition(self, key, n_partitions):
        return hash(key) % n_partitions


class Mapper(object):
    def map(self, *datasets):
        raise NotImplementedError()


class Streamable(object):
    def stream(self, kvs):
        raise NotImplementedError()


def _name_of(f):
    return getattr(f, "__name__", type(f).__name__)


class Map(Mapper, Streamable):
    """A function (k, v) -> iterable of (k, v) applied to every record (base.py:18-40)."""

    def __init__(self, mapper, op=None):
        assert not isinstance(mapper, Mapper)
        self.mapper = mapper
        self.op = op

    def map(self, *datasets):
        assert len(datasets) == 1
        return self.stream(datasets[0].read())

    def stream(self, kvs):
        f = self.mapper
        for k, v in kvs:
            for out in f(k, v):
                yield out

    def __repr__(self):
        return "Map[%s]" % _name_of(self.mapper)

    __str__ = __repr__


class FusedMapper(Mapper):
    """head.map(...) piped through a chain of Streamables (the reference's ComposedMapper /
    ComposedStreamable, base.py:42-60, flattened into one list so the planner can inspect it)."""

    def __init__(self, head, tail):
        assert isinstance(head, Mapper)
        assert all(isinstance(t, Streamable) for t in tail)
        self.head = head
        self.tail = list(tail)

    def parts(self):
        return [self.head] + self.tail

    def map(self, *datasets):
        it = self.head.map(*datasets)
        for t in self.tail:
            it = t.stream(it)
        return it

    def __repr__(self):
        return " -> ".join(str(p) for p in self.parts())

    __str__ = __repr__


def fuse(aggs):
    return aggs[0] if len(aggs) == 1 else FusedMapper(aggs[0], aggs[1:])


class BlockMapper(Mapper, Streamable):
    """User-defined block mapper: start(), add(key, value) -> iterable, finish() -> iterable
    (base.py:62-101)."""

    def start(self):
        pass

    def add(self, key, value):
        raise NotImplementedError()

    def finish(self):
        return ()

    def map(self, *datasets):
        assert len(datasets) == 1
        return self.stream(datasets[0].read())

    def stream(self, kvs):
        self.start()
        for k, v in kvs:
            for out in self.add(k, v):
                yield out
        for out in self.finish():
            yield out


class StreamMapper(Mapper, Streamable):
    """f(iterator of values) -> iterator of (k, v) records (base.py:103-124)."""

    def __init__(self, streamer_f, op=None):
        self.streamer_f = streamer_f
        self.op = op

    def map(self, *datasets):
        assert len(datasets) == 1
        return self.stream(datasets[0].read())

    def stream(self, kvs):
        return self.streamer_f(v for _k, v in kvs)

    def __repr__(self):
        return "StreamMapper[%s]" % _name_of(self.streamer_f)

    __str__ = __repr__


def as_one_dataset(dataset):
    """A stage input (Chunker, list of datasets or one dataset) as a single readable dataset."""
    from .datasets import Chunker, Dataset, CatDataset, EmptyDataset
    if isinstance(dataset, Dataset):
        return dataset
    if isinstance(dataset, Chunker):
        dataset = list(dataset.chunks())
    if len(dataset) == 0:
        return EmptyDataset()
    return dataset[0] if len(dataset) == 1 else CatDataset(dataset)


class MapCrossJoin(Mapper):
    """Nested-loop cross product, first input outer (base.py:139-163)."""

    def __init__(self, crosser, cache):
        self.crosser = crosser
        self.cache = cache

    def map(self, *datasets):
        assert len(datasets) == 2
        outer, inner = as_one_dataset(datasets[0]), as_one_dataset(datasets[1])
        if self.cache:
            held = list(inner.read())
            read_inner = lambda: held
        else:
            read_inner = inner.read
        for k1, v1 in outer.read():
            for k2, v2 in read_inner():
                for out in self.crosser(k1, v1, k2, v2):
                    yield out


class MapAllJoin(Mapper):
    """Broadcast join: aggregate the whole second input once, stream the first (base.py:165-178)."""

    def __init__(self, crosser, load_f=None):
        self.crosser = crosser
        self.load_f = load_f if load_f is not None else (lambda d: [v for _k, v in d])

    def map(self, *datasets):
        assert len(datasets) == 2
        streamed, whole = as_one_dataset(datasets[0]), as_one_dataset(datasets[1])
        table = self.load_f(whole.read())
        for k, v in streamed.read():
            for out in self.crosser(k, v, table):
                yield out


# ---- reducers -------------------------------------------------------------------------------
class Reducer(object):
    def reduce(self, *datasets):
        raise NotImplementedError()

    def yield_groups(self, dataset):
        return as_one_dataset(dataset).grouped_read()


class Reduce(Reducer):
    """reducer(key, values_iterator) per key group (base.py:197-207)."""

    def __init__(self, reducer):
        self.reducer = reducer

    def reduce(self, *datasets):
        assert len(datasets) == 1
        f = self.reducer
        for k, vs in self.yield_groups(datasets[0]):
            yield k, f(k, vs)


class KeyedReduce(Reduce):
    """Emits (k, (k, result)) so the user reads (key, result) (base.py:254-257)."""

    def reduce(self, *datasets):
        for k, v in Reduce.reduce(self, *datasets):
            yield k, (k, v)


class BlockReducer(Reducer):
    """User-defined block reducer: start(), add(key, values_iter) -> iterable, finish()
    (base.py:209-231)."""

    def start(self):
        pass

    def add(self, k, it):
        raise NotImplementedError()

    def finish(self):
        return ()

    def reduce(self, *datasets):
        assert len(datasets) == 1
        self.start()
        for k, vs in self.yield_groups(datasets[0]):
            for out in self.add(k, vs):
                yield out
        for out in self.finish():
            yield out


class StreamReducer(Reducer):
    """f(iterator of (key, values_iter)) -> iterator of (nk, nv); emits (nk, (nk, nv))
    (base.py:233-252)."""

    def __init__(self, stream_f, op=None):
        self.stream_f = stream_f
        self.op = op

    def reduce(self, *datasets):
        assert len(datasets) == 1
        for nk, nv in self.stream_f(self.yield_groups(datasets[0])):
            yield nk, (nk, nv)

    def __repr__(self):
        return "StreamReducer[%s]" % _name_of(self.stream_f)

    __str__ = __repr__


class JoinReducer(Reducer):
    """Two-input reducers. The runner finds the matching key groups on the device
    (dampr_kv_join_ranges) and calls emit() per key; reduce() is the generic host walk used when a
    user calls it directly with already grouped, key-ordered datasets."""
    left_outer = False
    keyed = False

    def __init__(self, joiner_f, many=False):
        self.joiner_f = joiner_f
        self.many = many

    def emit(self, k, left_it, right_it):
        res = self.joiner_f(k, left_it, right_it)
        for nv in (res if self.many else (res,)):
            yield (k, (k, nv)) if self.keyed else (k, nv)

    def reduce(self, *datasets):
        assert len(datasets) == 2
        g1, g2 = self.yield_groups(datasets[0]), self.yield_groups(datasets[1])
        left, right = next(g1, None), next(g2, None)
        while left is not None:
            if right is not None and right[0] < left[0]:
                right = next(g2, None)
                continue
            if right is not None and right[0] == left[0]:
                for out in self.emit(left[0], left[1], right[1]):
                    yield out
                right = next(g2, None)
            elif self.left_outer:
                for out in self.emit(left[0], left[1], iter(())):
                    yield out
            left = next(g1, None)


class InnerJoin(JoinReducer):
    """base.py:259-283"""


class KeyedInnerJoin(InnerJoin):
    keyed = True


class LeftJoin(JoinReducer):
    """base.py:290-315"""
    left_outer = True

    def __init__(self, joiner_f, default=None):
        JoinReducer.__init__(self, joiner_f, many=False)


class KeyedLeftJoin(LeftJoin):
    keyed = True


class CrossJoin(Reducer):
    """Reduce-side cross product (base.py:322-331)."""

    def __init__(self, joiner_f):
        self.joiner_f = joiner_f

    def reduce(self, *datasets):
        assert len(datasets) == 2
        right = list(as_one_dataset(datasets[1]).read())
        for lk, lv in as_one_dataset(datasets[0]).read():
            for rk, rv in right:
                yield self.joiner_f(lk, lv, rk, rv)


class KeyedCrossJoin(CrossJoin):
    def reduce(self, *datasets):
        for k, v in CrossJoin.reduce(self, *datasets):
            yield k, (k, v)


# ---- combiners ----------------------------------------------------------------------------------
class Combiner(object):
    """Marker of a map-side combine (base.py:373-382). The device engine does the combining: the
    runner reads `reducer`/`binop` off the stage instead of calling combine()."""

    def combine(self, datasets):
        raise NotImplementedError()


class NoopCombiner(Combiner):
    def combine(self, datasets):
        from .datasets import CatDataset
        return CatDataset(datasets)


class UnorderedCombiner(NoopCombiner):
    pass


class PartialReduceCombiner(Combiner):
    """Associative partial reduce during the map stage (base.py:393-402)."""

    def __init__(self, reducer):
        self.reducer = reducer

    def combine(self, datasets):
        from .datasets import StreamDataset
        ds = as_one_dataset(datasets)
        f = self.reducer.reducer
        return StreamDataset((k, f(k, vs)) for k, vs in ds.grouped_read())

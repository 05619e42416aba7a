"""CPU: host-side logic of the engine (no device): key codec, lambda lowering, text chunk ownership,
graph IR, token key-code decoding, C-ABI surface."""
import ctypes
import math
import operator
import os
import re
import subprocess

import numpy as np
import pytest

from dampr_b200 import keycodec, keycodes, lowering
from dampr_b200 import device as dev
from dampr_b200.datasets import TextLineDataset
from dampr_b200.inputs import TextInput, MemoryInput
from oracle import gen, refsem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_keycodec_ints_floats_order_and_roundtrip():
    keys = [5, -3, 0, 2 ** 62, -2 ** 63, 7]
    codes, codec = keycodec.encode(keys)
    assert codec.kind == keycodec.INT and codec.exact
    assert [keys[i] for i in np.argsort(codes, kind="stable")] == sorted(keys)
    assert keycodec.decode_exact(codes, codec) == keys
    fk = [1.5, -0.0, -2.25, 3e300, -1e-300, 2]
    codes, codec = keycodec.encode(fk)
    assert codec.kind == keycodec.FLOAT
    assert [fk[i] for i in np.argsort(codes, kind="stable")] == sorted(fk)
    assert keycodec.decode_exact(codes, codec) == [float(x) for x in fk]


def test_keycodec_strings_prefix_order_and_refine():
    keys = ["pear", "apple", "applesauce!", "applesauce", "fig", "apple"]
    codes, codec = keycodec.encode(keys)
    assert codec.kind == keycodec.STR and not codec.exact and codec.ordered
    order = np.argsort(codes, kind="stable")
    ks = [keys[i] for i in order]
    vs = list(order)
    ks, vs = keycodec.refine_runs(ks, vs, codes[order], codec)
    assert ks == sorted(keys)
    assert [keys[i] for i in vs] == ks


def test_keycodec_hash_class_groups_equal_keys():
    keys = [None, (1, "a"), (1, "a"), 2 ** 70, (1.0, "a"), None, "x"]
    codes, codec = keycodec.encode(keys)
    assert codec.kind == keycodec.HASH
    assert codes[0] == codes[5] and codes[1] == codes[2] == codes[4]
    assert len({int(c) for c in codes}) == 4
    with pytest.raises(TypeError):
        keycodec.encode([None, 1], need_order=True)
    codes, codec = keycodec.encode([(2, "b"), (1, "z"), (1, "a")], need_order=True)
    assert codec.kind == keycodec.TUPLE and codes[1] == codes[2] < codes[0]


def test_lowering_idioms():
    RX = re.compile(r"[^\w]+")
    assert lowering.tokenizer_mode(lambda x: x.split()) == lowering.TOK_WS
    assert lowering.tokenizer_mode(lambda x: set(RX.split(x.lower()))) == lowering.TOK_NONWORD_LOWER_SET
    assert lowering.tokenizer_mode(lambda x: RX.split(x.lower())) == lowering.TOK_NONWORD_LOWER
    assert lowering.tokenizer_mode(lambda x: re.split(r"\W+", x.lower())) == lowering.TOK_NONWORD_LOWER
    assert lowering.tokenizer_mode(lambda x: x.split(",")) is None
    assert lowering.tokenizer_mode(lambda x: set(RX.split(x))) is None  # no lower(): not the idiom
    RXI = re.compile(r"[^\w]+", re.I)
    assert lowering.tokenizer_mode(lambda x: set(RXI.split(x.lower()))) is None
    assert lowering.is_identity(lambda x: x) and not lowering.is_identity(lambda x: x + 0)
    assert lowering.constant_value(lambda x: 1) == (True, 1)
    assert lowering.projection(lambda x: -x[1]) == ("field", 1, -1)
    assert lowering.binop_kind(operator.add) == lowering.ADD
    assert lowering.binop_kind(lambda x, y: y + x) == lowering.ADD
    assert lowering.binop_kind(lambda x, y: x * y) is None
    assert lowering.binop_kind(lambda x, _y: x) == lowering.FIRST
    assert lowering.group_reducer_kind(lambda k, it: sum(it)) == lowering.SUM

    def branchy(x):
        if x:
            return 1
        return 2
    assert lowering.analyze(branchy) is None
    e = lowering.analyze(lambda df, total: (df[0], df[1], math.log(1 + (float(total) / df[1]))))
    assert [lowering.depends_on(c, 0) for c in e.a] == [{0}, {1}, {1}]


def test_text_chunk_ownership_every_line_once(tmp_path):
    """SURVEY B2: every line belongs to exactly one chunk, for any chunk size (also float)."""
    datas = [gen.dirty_text(3, 400, 700), b"a\nbb\n\nccc", b"\n\n", b"x" * 100 + b"\n" + b"y" * 5,
             b"one\r\ntwo\rthree\n"]
    for di, data in enumerate(datas):
        p = tmp_path / ("f%d.txt" % di)
        p.write_bytes(data)
        want = [l for _o, l in refsem.text_lines(data)]
        for cs in (1, 2, 3, 7, 64, 1000, 33.7, len(data) / 3.0 + 1, 10 ** 9):
            got = []
            for ch in TextInput(str(p), cs).chunks():
                got.extend(ch.read())
            assert [l for _o, l in got] == want, (di, cs)
            assert [o for o, _l in got] == sorted(o for o, _l in got)


def test_memory_input_chunks_cover_everything():
    items = list(enumerate(range(103)))
    got = [kv for ch in MemoryInput(items, 50).chunks() for kv in ch.read()]
    assert got == items
    assert [kv for ch in MemoryInput([], 50).chunks() for kv in ch.read()] == []


def test_token_code_decoding():
    def enc38(w):
        sym = {c: i + 1 for i, c in enumerate("0123456789_abcdefghijklmnopqrstuvwxyz")}
        code = 0
        for ch in reversed(w):
            code = code * 38 + sym[ch]
        return code

    words = ["a", "zz", "hello_world9", "0", "_"]
    codes = np.array([enc38(w) for w in words], dtype=np.uint64)
    assert keycodes.decode_exact(codes, dev.TOK_NONWORD_LOWER_SET) == words
    ws = ["Hi!", "a", "x" * 9, "~"]
    codes = np.array([sum(ord(c) << (7 * i) for i, c in enumerate(w)) for w in ws], dtype=np.uint64)
    assert keycodes.decode_exact(codes, dev.TOK_WS) == ws


def test_abi_exports_every_declared_symbol():
    """The library loads on a CPU-only box and exports every function include/dampr_b200.h declares."""
    hdr = open(os.path.join(ROOT, "include", "dampr_b200.h")).read()
    declared = set(re.findall(r"\b(dampr_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"dampr_ctx", "dampr_textbuf", "dampr_table", "dampr_kv"}
    assert len(declared) > 40
    lib = ctypes.CDLL(dev.LIB_PATH)
    missing = [n for n in sorted(declared) if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.dampr_abi_version() == 1
    dev.load_library()


def test_set_option_accepts_only_the_live_switches():
    """The partition/sort kernel variants and their switches are gone: their names are unknown options. The
    switches that remain accept their defaults (setting them leaves the process as it was). Each removed name
    is tried with the value that was its default."""
    for name, old_default in (("kv_scatter", 1), ("kv_hist", 2), ("kv_cluster", 0), ("kv_hints", 1),
                              ("kv_max_bits", 12), ("kv_leaf_target", 2600), ("scatter_tma", 1)):
        with pytest.raises(dev.DeviceError):
            dev.set_option(name, old_default)
    for name, default in (("text_ctas", 4), ("text_kernel", 2), ("host_threads", 16), ("file_cufile", 0),
                          ("cufile_threads", 8)):
        dev.set_option(name, default)


def test_no_gpu_fails_loudly():
    if dev.device_count() > 0:
        pytest.skip("GPU present")
    from dampr_b200 import Dampr
    with pytest.raises(dev.DeviceError):
        Dampr.memory([1, 2, 3]).map(lambda x: x).read()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "dampr_b200")
    for dirpath, _d, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_host_join_tsv_native():
    """Pure-host sink formatter of the library (no device needed)."""
    words = np.array([b"alpha", b"b", b"", b"x" * 8], dtype="S8")
    inv = np.array([2, 0, 1, 0], dtype=np.uint32)
    strs = [b"1.5", b"", b"-3"]
    out = dev.host_join_tsv([words, (inv, strs)]).tobytes()
    assert out == b"alpha\t-3\nb\t1.5\n\t\nxxxxxxxx\t1.5\n"
    n = 200000
    w = np.array([b"w%d" % i for i in range(n)], dtype="S12")
    iv = (np.arange(n) % 7).astype(np.uint32)
    ss = [str(i * 0.5).encode() for i in range(7)]
    out = dev.host_join_tsv([w, (iv, ss), (iv, ss)]).tobytes()
    assert out == b"".join(b"w%d\t%s\t%s\n" % (i, ss[i % 7], ss[i % 7]) for i in range(n))


def test_frame_cross_and_sink_lowering_exact_python_values(tmp_path):
    """plan._lower_cross evaluates the user's own lambda once per distinct field value: the floats
    are Python's (math.log), and the sink lines equal str() of the tuples."""
    import math
    from dampr_b200 import plan
    from dampr_b200.datasets import RecordsDataset

    class FakeRunner(object):
        class stats(object):
            @staticmethod
            def add(*a, **k):
                pass

    words = np.array([b"a", b"bb", b"ccc", b"dd"], dtype="S32")
    counts = np.array([3, 1, 3, 7], dtype=np.int64)
    fr = plan.Frame(words, [words, counts], scalar=False, combined=True)
    user = lambda df, total: (df[0], df[1], math.log(1 + (float(total) / df[1])))

    class Stage(object):
        pass
    st = Stage()
    st.mapper = Stage()
    st.mapper.user_cross = lambda xi, yi: user(yi, xi)
    out = plan._lower_cross(FakeRunner, st, [fr, RecordsDataset([0], [10])])
    exp = [user((w.decode(), int(c)), 10) for w, c in zip(words.tolist(), counts.tolist())]
    assert out.values() == exp
    cols = [plan._sink_column(c) for c in out.cols]
    blob = dev.host_join_tsv(cols).tobytes().decode()
    assert blob == "".join(u"\t".join(str(p) for p in row) + "\n" for row in exp)


def test_vexpr_matches_cpython_row_by_row():
    """Column-at-a-time evaluation of lowered lambdas (dampr_b200/vexpr.py) gives exactly what CPython
    gives per row, and refuses (NotVec) whenever that cannot be guaranteed."""
    import math
    import numpy as np
    import pytest
    from dampr_b200 import lowering, vexpr
    rng = np.random.default_rng(3)
    n = 5000
    a = rng.integers(-10**6, 10**6, size=n).astype(np.int64)
    b = rng.integers(1, 1000, size=n).astype(np.int64)
    f = rng.normal(size=n) * 1e3
    w = np.array([b"x" * int(k) for k in rng.integers(1, 20, size=n)], dtype="S32")
    cols = [a, b, f, w]
    rows = list(zip(a.tolist(), b.tolist(), f.tolist(), [x.decode() for x in w.tolist()]))
    fns = [
        lambda x: x[0] + x[1] * 3 - 7,
        lambda x: (x[0], x[0] / x[1], x[0] // x[1], x[0] % x[1]),
        lambda x: -x[0] * x[1],
        lambda x: x[2] * x[0] + 0.5,
        lambda x: float(x[0]) / x[2],
        lambda x: len(x[3]) * x[1],
        lambda x: abs(x[0]) - abs(x[2]),
        lambda x: (x[0] < x[1], x[2] >= 0.0, x[0] == x[1], x[0] != 5),
        lambda x: (x[1], (x[0], 1)),
    ]
    for fn in fns:
        e = lowering.analyze(fn)
        assert e is not None
        v = vexpr.evaluate(e, cols, False, n)

        def pyl(c):
            if isinstance(c, vexpr.Tup):
                return list(zip(*[pyl(x) for x in c.items]))
            return vexpr.broadcast(c, n).tolist()
        got = pyl(v)
        exp = [fn(r) for r in rows]
        assert got == exp, fn
    big = np.full(n, 1 << 61, dtype=np.int64)
    for fn, cs in [(lambda x: x[0] * x[1], [big, b]), (lambda x: x[0] + x[0], [big]), (lambda x: x[0] / x[1], [big, b]),
                   (lambda x: x[0] / (x[1] - x[1]), [a, b]), (lambda x: math.sqrt(x[0]), [b]), (lambda x: x[0] + "s", [b])]:
        with pytest.raises(vexpr.NotVec):
            vexpr.evaluate(lowering.analyze(fn), cs, False, n)
    assert lowering.tuple_binop_kinds(lambda x, y: (x[0] + y[0], x[1] + y[1])) == [lowering.ADD, lowering.ADD]
    assert lowering.tuple_binop_kinds(lambda x, y: (x[0] + y[1], x[1] + y[0])) is None


def test_native_host_helpers(tmp_path):
    """Host-side entry points of the library (no device work): sink formatting into part files, decimal
    formatting of int dictionaries, dictionary encoding of count columns."""
    import numpy as np
    from dampr_b200 import device as dev
    from dampr_b200 import plan
    rng = np.random.default_rng(4)
    for n, W in ((0, 16), (7, 16), (70000, 24), (150000, 32)):
        vals = np.array([0, -1, 5, 123456789, -42, 10, 100, -9223372036854775808, 9223372036854775807], dtype=np.int64)
        inv = rng.integers(0, len(vals), size=n).astype(np.uint32)
        words = np.array([b"x" * int(l) for l in rng.integers(0, W + 1, size=n)], dtype="S%d" % W)
        fl = [repr(float(i) / 7).encode() for i in range(40)]
        inv2 = rng.integers(0, 40, size=n).astype(np.uint32)
        exp = b"".join(b"%s\t%d\t%s\n" % (words[i], vals[inv[i]], fl[inv2[i]]) for i in range(n))
        cols = [words, (inv, vals), (inv2, fl)]
        if n:
            assert dev.host_join_tsv(cols).tobytes() == exp
            d = tmp_path / ("s%d" % n)
            d.mkdir()
            names = dev.host_join_tsv(cols, prefix=str(d / "part-"), first=16)
            assert names[0].endswith("part-16") and len(names) == max(1, min(16, n // 32768))
            assert b"".join(open(f, "rb").read() for f in names) == exp
    for trial in range(4):
        x = rng.integers(0, 3000, size=60000).astype(np.int64)
        if trial >= 1:
            x[rng.integers(0, len(x), size=200)] = rng.integers(1 << 30, 1 << 40, size=200)
        if trial == 3:
            x[11] = -5   # negative value: the presence table does not apply, numpy path
        u, inv, rows = plan.unique_inverse_rows(x)
        assert np.array_equal(u, np.unique(x)) and np.array_equal(u[inv], x) and np.array_equal(x[rows], u)
        u2, inv2 = plan.unique_inverse(x)
        assert np.array_equal(u2, u) and np.array_equal(u2[inv2], x)


def test_frame_take_and_tuple_columns():
    import numpy as np
    from dampr_b200 import plan, vexpr
    n = 1000
    rng = np.random.default_rng(2)
    words = np.array([b"w%d" % i for i in range(n)], dtype="S16")
    counts = rng.integers(0, 50, size=n).astype(np.int64)
    uq, inv = np.unique(counts, return_inverse=True)
    fr = plan.Frame(words, [words, plan.DictCol(inv.astype(np.uint32), uq), vexpr.Tup([counts, counts * 2])], scalar=False)
    perm = rng.permutation(n)[:300]
    out = fr.take(perm)
    assert out.cols[0] is out.keys                      # the shared column object is gathered once
    exp = [(words[i].decode(), int(counts[i]), (int(counts[i]), int(2 * counts[i]))) for i in perm]
    assert out.values() == exp and list(k for k, _v in out.read()) == [words[i].decode() for i in perm]
    empty = fr.take(np.zeros(0, dtype=np.int64))
    assert empty.values() == [] and len(empty) == 0


def test_parallel_host_map_matches_sequential(tmp_path):
    """hostmap.parallel (forked workers over contiguous chunk ranges, optional in-worker fold) gives the
    sequential record order / the same folds, and re-raises the user's exception."""
    import pytest
    from dampr_b200 import hostmap
    from dampr_b200 import operators as ops
    from dampr_b200.inputs import TextInput
    lines = ["Line %d has the words alpha beta %s gamma" % (i, "delta" * (i % 3)) for i in range(20000)]
    p = tmp_path / "t.txt"
    p.write_text("\n".join(lines) + "\n")
    chunks = list(TextInput(str(p), 64 * 1024).chunks())
    assert len(chunks) > 8

    def fm(k, v):
        for w in v.upper().split():     # .upper(): not a lowered idiom
            yield w, 1
    mapper = ops.Map(fm)
    k1, v1 = hostmap.sequential(mapper, chunks, ())
    k2, v2 = hostmap.parallel(mapper, chunks, (), None, 4)
    assert (k1, v1) == (k2, v2)
    k3, v3 = hostmap.parallel(mapper, chunks, (), lambda a, b: a + b, 3)
    exp = {}
    for k in k1:
        exp[k] = exp.get(k, 0) + 1
    got = {}
    for k, v in zip(k3, v3):
        got[k] = got.get(k, 0) + v
    assert got == exp and len(k3) <= 3 * len(exp)

    def bad(k, v):
        if "Line 777 " in v:
            raise ZeroDivisionError("boom")
        yield k, v
    with pytest.raises(ZeroDivisionError):
        hostmap.parallel(ops.Map(bad), chunks, (), None, 4)

    def unpicklable(k, v):
        yield k, (lambda: v)            # a record that cannot cross a process boundary
    k4, v4 = hostmap.parallel(ops.Map(unpicklable), chunks, (), None, 4)
    assert len(k4) == len(lines) and [f() for f in v4] == lines


def test_parallel_host_reduce_matches_sequential():
    from dampr_b200 import hostmap
    from dampr_b200 import operators as ops
    from dampr_b200.datasets import RecordsDataset
    keys, vals = [], []
    for k in range(3000):
        for j in range(1 + (k * 7) % 23):
            keys.append("k%05d" % k)
            vals.append(k * 1000 + j)
    red = ops.KeyedReduce(lambda k, it: sum(it) - len(k))
    seq = list(red.reduce(RecordsDataset(keys, vals)))
    for nproc in (1, 2, 5, 16):
        ks, vs = hostmap.parallel_reduce(red, RecordsDataset(keys, vals), nproc)
        assert list(zip(ks, vs)) == seq
    one = RecordsDataset(["a"] * 50, list(range(50)))       # a single group cannot be split
    assert hostmap.parallel_reduce(red, one, 4) == (["a"], [("a", sum(range(50)) - 1)])


def test_vexpr_random_expressions_agree_with_cpython():
    """Seeded random arithmetic over the whitelisted forms: column-at-a-time evaluation either raises
    NotVec or gives, row for row, exactly what CPython gives (value and type)."""
    import random
    import numpy as np
    from dampr_b200 import lowering, vexpr
    rng = random.Random(12345)
    nrng = np.random.default_rng(99)
    n = 400
    a = nrng.integers(-50, 50, size=n).astype(np.int64)
    b = nrng.integers(-3, 4, size=n).astype(np.int64)          # has zeros: division guards must trip
    c = (nrng.normal(size=n) * 10).astype(np.float64)
    cols = [a, b, c]
    rows = list(zip(a.tolist(), b.tolist(), c.tolist()))

    def gen(depth):
        if depth == 0 or rng.random() < 0.25:
            return rng.choice(["x[0]", "x[1]", "x[2]", str(rng.randint(-5, 5)), repr(round(rng.uniform(-3, 3), 2))])
        k = rng.random()
        if k < 0.6:
            return "(%s %s %s)" % (gen(depth - 1), rng.choice(["+", "-", "*", "/", "//", "%"]), gen(depth - 1))
        if k < 0.7:
            return "(-%s)" % gen(depth - 1)
        if k < 0.8:
            return "abs(%s)" % gen(depth - 1)
        if k < 0.9:
            return "float(%s)" % gen(depth - 1)
        return "(%s %s %s)" % (gen(depth - 1), rng.choice(["<", "<=", "==", "!=", ">", ">="]), gen(depth - 1))

    checked = refused = 0
    for _ in range(400):
        src = "lambda x: " + gen(3)
        fn = eval(src)
        e = lowering.analyze(fn)
        if e is None:
            continue
        try:
            exp = [fn(r) for r in rows]
        except (ZeroDivisionError, OverflowError):
            exp = None
        try:
            v = vexpr.evaluate(e, cols, False, n)
        except vexpr.NotVec:
            refused += 1
            continue
        assert exp is not None, src     # CPython raised for some row: the evaluation must have refused
        got = vexpr.broadcast(v, n).tolist()
        for g, x in zip(got, exp):
            assert type(g) is type(x) and (g == x or (g != g and x != x)), (src, g, x)
        checked += 1
    assert checked > 50 and refused > 20


from fake_device import FakeCtx as _FakeCtx, FakeKV as _FakeKV  # noqa: E402


def test_spill_host_logic_with_a_numpy_device(monkeypatch):
    """external_group / external_sort (dampr_b200/spill.py) against numpy, with an arena so small that
    batches, buckets, splitter ties, heavy single keys and the recursive re-split all occur."""
    from dampr_b200 import settings, spill
    from dampr_b200 import device as dev
    ctx = _FakeCtx()
    monkeypatch.setattr(settings, "device_arena_bytes", 48 * 70000)     # 70 000 records per batch
    rng = np.random.default_rng(8)
    n = 400000

    def chunks(k, v, step=30000):
        return ((k[i:i + step], v[i:i + step]) for i in range(0, len(k), step))

    # grouping (hash buckets): sums and first-by-input-order
    keys = rng.integers(0, 5000, size=n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    vals = rng.integers(-1000, 1000, size=n).astype(np.int64)
    for op in (dev.OP_SUM_I64, dev.OP_FIRST):
        pieces, st = spill.external_group(ctx, chunks(keys, vals), n, op, dev.KEY_MIX)
        assert st["buckets"] > 2 and st["batches"] > 2
        gk = np.concatenate([p[0] for p in pieces])
        gv = np.concatenate([p[1] for p in pieces]).view(np.int64)
        assert len(np.unique(gk)) == len(gk)
        u, first_idx, inv = np.unique(keys, return_index=True, return_inverse=True)
        exp = np.zeros(len(u), dtype=np.int64)
        if op == dev.OP_SUM_I64:
            np.add.at(exp, inv, vals)
        else:
            exp = vals[first_idx]
        o = np.argsort(gk)
        assert np.array_equal(gk[o], u) and np.array_equal(gv[o], exp)

    # sorting (range buckets): stable global order, for uniform keys, heavy ties and one dominant key
    for name, k in (("uniform", rng.integers(-10**9, 10**9, size=n).astype(np.int64)),
                    ("ties", rng.integers(-20, 20, size=n).astype(np.int64)),
                    ("dominant", np.where(rng.random(n) < 0.7, 5, rng.integers(-1000, 1000, size=n)).astype(np.int64))):
        v = np.arange(n, dtype=np.int64)
        samp = k[rng.integers(0, n, size=4096)]
        pieces, st = spill.external_sort(ctx, chunks(k.view(np.uint64), v), n, dev.KEY_I64, samp)
        sk = np.concatenate([p[0] for p in pieces]).view(np.int64)
        sv = np.concatenate([p[1] for p in pieces]).view(np.int64)
        o = np.argsort(k, kind="stable")
        assert np.array_equal(sk, k[o]) and np.array_equal(sv, v[o]), name


def test_frame_general_lowering_with_a_numpy_device():
    """plan._lower_frame_general (map / filter chains, keyed folds incl. mean's pair fold, single-group
    folds, sort_by on a computed key) against plain Python, on the numpy stand-in for the device."""
    from dampr_b200 import operators as ops
    from dampr_b200 import plan
    from dampr_b200.operators import Op

    class Ctx(_FakeCtx):
        def kv_from_columns(self, keys, vals=None):
            kv = _FakeKV(self, max(1, len(keys)))
            kv.upload_columns(0, keys, vals if vals is not None else np.zeros(len(keys), dtype=np.int64))
            return kv

    class Runner(object):
        ctx = Ctx()

        class stats(object):
            @staticmethod
            def add(*a, **k):
                pass

    def stage(opsl, binop=None):
        class S(object):
            pass
        st = S()
        maps = [ops.Map(lambda k, v: [(k, v)], op=o) for o in opsl]
        st.mapper = maps[0] if len(maps) == 1 else ops.FusedMapper(maps[0], maps[1:])
        st.combiner = ops.PartialReduceCombiner(None) if binop is not None else None
        st.options = {"binop": binop} if binop is not None else {}
        st.output = "test"
        return st

    rng = np.random.default_rng(6)
    n = 5000
    words = np.array([b"w" * int(l) for l in rng.integers(1, 12, size=n)], dtype="S16")
    counts = rng.integers(1, 500, size=n).astype(np.int64)
    fr = plan.Frame(words, [words, counts], scalar=False, combined=True)
    rows = list(zip([w.decode() for w in words.tolist()], counts.tolist()))

    # fold_by(len(word), count, +)  (examples/word-stats.py:24-28)
    out = plan._lower_frame_general(Runner, stage([Op("keyed", lambda tc: len(tc[0]), lambda tc: tc[1])], lambda x, y: x + y), fr)
    exp = {}
    for w, c in rows:
        exp[len(w)] = exp.get(len(w), 0) + c
    assert out is not None and out.combined and dict(zip(out.keys.tolist(), out.values())) == exp

    # fold with a constant key: one group, folded on the host
    out = plan._lower_frame_general(Runner, stage([Op("keyed", lambda x: 1, lambda x: x[1])], lambda x, y: x + y), fr)
    assert out.values() == [sum(c for _w, c in rows)] and out.keys.tolist() == [1]

    # mean(): (value, 1) pairs under a component-wise add
    out = plan._lower_frame_general(
        Runner, stage([Op("keyed", lambda tc: tc[1] % 7, lambda tc: (tc[1] * 2, 1))], lambda x, y: (x[0] + y[0], x[1] + y[1])), fr)
    e2 = {}
    for _w, c in rows:
        s0, s1 = e2.get(c % 7, (0, 0))
        e2[c % 7] = (s0 + 2 * c, s1 + 1)
    assert dict(zip(out.keys.tolist(), out.values())) == e2

    # map + filter chain, then sort_by on a computed key (stable)
    st = stage([Op("map", lambda tc: (tc[0], tc[1] * 3, tc[1] / 4)), Op("filter", lambda r: r[1] > 300),
                Op("keyed", lambda r: -r[1] + len(r[0]), lambda r: r)])
    out = plan._lower_frame_general(Runner, st, fr)
    exp_rows = [(w, c * 3, c / 4) for w, c in rows if c * 3 > 300]
    exp_rows.sort(key=lambda r: -r[1] + len(r[0]))
    assert out.values() == exp_rows

    # a guard trips (possible int64 overflow): not lowered
    big = plan.Frame(words, [words, np.full(n, 1 << 61, dtype=np.int64)], scalar=False)
    assert plan._lower_frame_general(Runner, stage([Op("map", lambda tc: tc[1] * 4)]), big) is None


def test_device_fold_guards_keep_python_semantics():
    """ADVICE r1: bools folded with min / max / first / last stay bools (host fold), float min / max with NaN or -0.0
    stay on the host, uint64 values >= 2^63 are not handed to the signed device folds."""
    import numpy as np
    from dampr_b200 import lowering, runner
    col, op = runner._numeric_column([True, False, True], lowering.MAX)
    assert col is None
    col, op = runner._numeric_column([True, 2, False], lowering.ADD)
    assert col is not None and col.tolist() == [1, 2, 0]
    assert runner._numeric_column([1.0, float("nan")], lowering.MIN)[0] is None
    assert runner._numeric_column([0.0, -0.0], lowering.MAX)[0] is None
    assert runner._numeric_column([1.5, -2.0], lowering.MAX)[0] is not None
    assert runner._numeric_column([3, 4], lowering.MIN)[0] is not None


def test_topk_over_a_frame_takes_its_candidates_with_one_device_sort(monkeypatch):
    """topk(k, value) over a columnar frame (plan._lower_topk, dampr.py:621-652): the k largest by the reference's
    (value(x), x) tuple order, ties at the boundary included; NaN scores and non-projection value functions fall
    back to the generic partition_map."""
    import heapq
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: _FakeCtx()})
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 5000, size=60000).astype(np.int64)
    vals = rng.integers(0, 4, size=60000).astype(np.int64)    # few distinct sums: many ties
    base = Dampr.read_input(ArrayKVInput(keys, vals)).a_group_by(lambda x: x[0], lambda x: x[1]).sum()
    rows = base.read()
    for k in (0, 1, 7, 100, 6000):
        for value in (lambda x: x[1], lambda x: -x[1], lambda x: x[0]):
            got = base.topk(k, value).read()
            assert any("top-k" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
            exp = [x for _s, x in heapq.nlargest(k, [(value(x), x) for x in rows])]
            assert sorted(got) == sorted(exp), k
    got = base.topk(5, lambda x: x[1] * 2 + x[0]).read()   # not a projection: host path, same answer
    assert not any("top-k" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    assert sorted(got) == sorted(x for _s, x in heapq.nlargest(5, [(x[1] * 2 + x[0], x) for x in rows]))


def test_unique_over_kv_records_keeps_first_appearance_order(monkeypatch):
    """group_by(k, v).unique() over binary kv records (plan._lower_unique, dampr.py:727-746): per key the distinct
    values in first-appearance order, Python ints / floats; NaN values and non-numeric key functions stay on the host."""
    from dampr_b200 import Dampr, settings
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: _FakeCtx()})
    rng = np.random.default_rng(3)

    def ref(keys, vals):
        d = {}
        for k, v in zip(keys.tolist(), vals.tolist()):
            seen = d.setdefault(k, [])
            if v not in seen:
                seen.append(v)
        return d

    def lowered():
        return any("device unique" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    for kd, vd in ((np.int64, np.int64), (np.uint64, np.float64), (np.int64, np.uint64)):
        keys = rng.integers(0, 500, size=20000).astype(kd)
        vals = (rng.integers(-20, 40, size=20000) if vd != np.uint64 else rng.integers(0, 40, size=20000)).astype(vd)
        if vd == np.float64:
            vals = vals / 4.0 + 0.25
        got = dict(Dampr.read_input(ArrayKVInput(keys, vals)).group_by(lambda x: x[0], lambda x: x[1]).unique().read())
        assert lowered()
        assert got == ref(keys, vals)
        assert all(type(x) is (float if vd == np.float64 else int) for l in got.values() for x in l)
    vals = rng.integers(-20, 40, size=20000).astype(np.float64)
    vals[5] = float("nan")
    vals[6] = -0.0
    got = dict(Dampr.read_input(ArrayKVInput(keys, vals)).group_by(lambda x: x[0], lambda x: x[1]).unique().read())
    assert not lowered()
    # a vectorisable key function: "the same" = equal key(v); the first v of every class is kept
    ivals = rng.integers(-20, 40, size=20000).astype(np.int64)

    def ref_by(keys, vals, f):
        d, seen = {}, {}
        for k, v in zip(keys.tolist(), vals.tolist()):
            if f(v) not in seen.setdefault(k, set()):
                seen[k].add(f(v))
                d.setdefault(k, []).append(v)
        return d
    for f in (lambda v: v % 3, lambda v: v > 5, lambda v: v * 0.5, lambda v: -v):
        got = dict(Dampr.read_input(ArrayKVInput(keys, ivals)).group_by(lambda x: x[0], lambda x: x[1]).unique(f).read())
        assert lowered()
        assert got == ref_by(keys, ivals, f)
    got = dict(Dampr.read_input(ArrayKVInput(keys, ivals)).group_by(lambda x: x[0], lambda x: x[1]).unique(lambda v: str(v)[0]).read())
    assert not lowered()   # not a numeric expression: the host reducer over device-grouped records
    assert got == ref_by(keys, ivals, lambda v: str(v)[0])


def test_native_float_repr_is_pythons_repr():
    """dampr_host_format_f64 (the formatter behind the float dictionaries of the native sink): bit-for-bit
    repr(float) — shortest round-trip digits, fixed notation for -4 < decpt <= 16, two-digit exponents, '.0',
    signed zeros, inf / nan — on edge cases, the tf-idf value range and random bit patterns."""
    lib = dev.load_library()
    rng = np.random.default_rng(1)
    cases = [0.0, -0.0, 1.0, -1.0, 0.1, 1e16, 1e15, 123456789012345678.0, 1234567890123456.0, 9999999999999998.0, 1e-4, 1e-5,
             0.0001234, 1.5e-7, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, float("inf"), float("-inf"),
             float("nan"), 1e22, 1e23, 1e100, 1e-100, 123.456, 0.30000000000000004, 2.5, 100.0, 1e21, 12345678901234567890.0]
    cases += [math.log(1 + 1e8 / d) for d in range(1, 5000)]
    cases += (rng.random(50000) * 10.0 ** rng.integers(-30, 30, size=50000)).tolist()
    vals = np.concatenate([np.array(cases, dtype=np.float64), rng.integers(0, 1 << 64, size=200000, dtype=np.uint64).view(np.float64)])
    n = len(vals)
    slots = np.zeros(n * 24, dtype=np.uint8)
    lens = np.zeros(n, dtype=np.uint8)
    assert lib.dampr_host_format_f64(vals.ctypes.data_as(ctypes.c_void_p), n, slots.ctypes.data_as(ctypes.c_void_p),
                                     lens.ctypes.data_as(ctypes.c_void_p)) == 0
    blob = slots.tobytes()
    for i, v in enumerate(vals.tolist()):
        assert blob[i * 24:i * 24 + int(lens[i])].decode() == repr(v), (v, i)
    # through the join: a float dictionary column next to an int dictionary and a fixed-width string column
    inv = rng.integers(0, 1000, size=5000).astype(np.uint32)
    fu = np.array([math.log(1 + 1e6 / (j + 1)) for j in range(1000)], dtype=np.float64)
    iu = np.arange(1000, dtype=np.int64) * 7 - 50
    words = np.array([("w%d" % j).encode() for j in inv.tolist()], dtype="S8")
    rows = dev.host_join_tsv([words, (inv, iu), (inv, fu)]).tobytes().decode().split("\n")[:-1]
    assert rows == ["w%d\t%d\t%r" % (j, iu[j], float(fu[j])) for j in inv.tolist()]


def test_cross_components_with_placeholder_rows_fall_back_when_needed(monkeypatch):
    """plan._lower_cross evaluates a component that reads one field on representative rows whose OTHER fields are
    placeholders; when another component of the user's function cannot digest a placeholder (None + 1) the full
    rows are used — the results are Python's either way."""
    from dampr_b200 import Dampr, settings
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: _FakeCtx()})
    rng = np.random.default_rng(5)
    keys = rng.integers(0, 3000, size=40000).astype(np.int64)
    vals = rng.integers(1, 9, size=40000).astype(np.int64)
    sums = Dampr.read_input(ArrayKVInput(keys, vals)).a_group_by(lambda x: x[0], lambda x: x[1]).sum()
    rows = sums.read()
    n = len(rows)
    got = sums.cross_right(sums.len(), lambda kv, total: (kv[0] + 1, kv[1], math.log(1 + float(total) / kv[1]))).read()
    assert any("frame cross" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    assert sorted(got) == sorted((k + 1, v, math.log(1 + float(n) / v)) for k, v in rows)
    got = sums.cross_right(sums.len(), lambda kv, total: (kv[0], kv[1], math.log(1 + float(total) / kv[1]))).read()
    assert sorted(got) == sorted((k, v, math.log(1 + float(n) / v)) for k, v in rows)


def test_spill_pipeline_propagates_upload_errors_and_releases_the_run_buffer():
    """The next batch is uploaded by a host thread (spill._Upload): an error there must surface in the caller, leave
    no thread behind and give the process-wide run buffer back."""
    from dampr_b200 import settings, spill
    ctx = _FakeCtx()
    old = settings.device_arena_bytes
    settings.device_arena_bytes = 1 << 20
    rng = np.random.default_rng(0)
    keys = rng.integers(0, 1000, size=200000).astype(np.uint64)
    vals = np.ones(200000, dtype=np.int64)
    orig = _FakeKV.upload_columns
    try:
        for fail_at in (1, 2, 4):
            calls = {"n": 0}

            def boom(self, off, k, v):
                calls["n"] += 1
                if calls["n"] == fail_at:
                    raise RuntimeError("upload failed")
                return orig(self, off, k, v)
            _FakeKV.upload_columns = boom
            with pytest.raises(RuntimeError, match="upload failed"):
                spill.external_group(ctx, iter([(keys, vals)]), len(keys), dev.OP_SUM_I64, dev.KEY_MIX)
            assert spill._HOST_ARENA["leased"] is False
        _FakeKV.upload_columns = orig
        pieces, st = spill.external_group(ctx, iter([(keys, vals)]), len(keys), dev.OP_SUM_I64, dev.KEY_MIX)
        got = dict(zip(np.concatenate([p[0] for p in pieces]).tolist(), np.concatenate([p[1] for p in pieces]).view(np.int64).tolist()))
        exp = {}
        for k in keys.tolist():
            exp[k] = exp.get(k, 0) + 1
        assert got == exp and st["batches"] == 4
    finally:
        _FakeKV.upload_columns = orig
        settings.device_arena_bytes = old
        spill.release_host_arena()


def test_overflow_bound_evaluated_next_to_the_device_work_still_vetoes(monkeypatch):
    """a_group_by(...).sum() over many records checks the 64-bit overflow bound on a host thread while the device
    folds (plan._lower_kv_map); sums that leave the 64-bit range must still come back as Python's exact integers
    (host path), sums that do not are the device's."""
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: _FakeCtx()})
    monkeypatch.setattr(plan, "_LATE_OVERFLOW_MIN", 1000)
    keys = (np.arange(6000) % 50).astype(np.int64)
    big = np.full(6000, (1 << 62) - 3, dtype=np.int64)
    got = dict(Dampr.read_input(ArrayKVInput(keys, big)).a_group_by(lambda x: x[0], lambda x: x[1]).sum().read())
    assert got == {k: 120 * ((1 << 62) - 3) for k in range(50)}
    assert not any("segmented-reduce" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    small = np.arange(6000, dtype=np.int64)
    got = dict(Dampr.read_input(ArrayKVInput(keys, small)).a_group_by(lambda x: x[0], lambda x: x[1]).sum().read())
    assert got == {k: int(small[keys == k].sum()) for k in range(50)}
    assert any("segmented-reduce" in how for _s, how, _d in runner_mod.LAST_STATS.stages)


def test_sink_json_over_frames_is_json_dumps_per_record(monkeypatch, tmp_path):
    """sink_json over a frame (plan._json_columns + dampr_host_sink_fmt): every line is json.dumps(value) — arrays
    for tuple rows, quoted strings, decimal ints, repr floats; values the native writer does not take (strings that
    need escaping in an 'S' column, non-finite floats) go through the host sink and give the same lines."""
    import json
    from fake_device import FakeTextCtx, FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: FakeTextCtx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})

    def lines_of(d):
        out = []
        for fn in sorted(os.listdir(d)):
            with open(os.path.join(d, fn)) as f:
                out.extend(l.rstrip("\n") for l in f)
        return out

    def native():
        return any("native frame sink" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    data = gen.text(5, 3000, V=800)
    p = tmp_path / "c.txt"
    p.write_bytes(data)
    counts = Dampr.text(str(p)).flat_map(lambda x: x.split()).count()
    rows = counts.read()
    n = len(rows)
    idf = counts.cross_right(counts.len(), lambda df, total: (df[0], df[1], math.log(1 + float(total) / df[1])))
    idf.sink_json(str(tmp_path / "j1")).run()
    assert native()
    assert sorted(lines_of(str(tmp_path / "j1"))) == sorted(json.dumps((w, c, math.log(1 + float(n) / c))) for w, c in rows)
    counts.sink_json(str(tmp_path / "j2")).run()
    assert native()
    assert sorted(lines_of(str(tmp_path / "j2"))) == sorted(json.dumps((w, c)) for w, c in rows)
    counts.map(lambda x: x[0]).sink_json(str(tmp_path / "j3")).run()       # scalar string rows
    assert sorted(lines_of(str(tmp_path / "j3"))) == sorted(json.dumps(w) for w, _c in rows)
    # tokens with a quote / a backslash: not what the native writer copies verbatim -> host sink, same lines
    q = tmp_path / "q.txt"
    q.write_bytes(b'say "hi" to\\ back\\slash "hi"\nplain words only\n')
    qc = Dampr.text(str(q)).flat_map(lambda x: x.split()).count()
    qc.sink_json(str(tmp_path / "j4")).run()
    assert not native()
    assert sorted(lines_of(str(tmp_path / "j4"))) == sorted(json.dumps(r) for r in qc.read())
    # non-finite floats: json.dumps writes NaN / Infinity
    keys = np.arange(6, dtype=np.int64)
    vals = np.array([1, 2, 0, 4, 5, 6], dtype=np.int64)
    fr = Dampr.read_input(ArrayKVInput(keys, vals)).a_group_by(lambda x: x[0], lambda x: x[1]).sum()
    inf = fr.map(lambda x: (x[0], x[1] * 1e308 * 10))
    inf.sink_json(str(tmp_path / "j5")).run()
    assert sorted(lines_of(str(tmp_path / "j5"))) == sorted(json.dumps(r) for r in inf.read())


def test_plain_sink_of_tuple_rows_is_print_of_the_tuple(monkeypatch, tmp_path):
    """sink(path) over tuple rows (plan._tuple_repr_columns): every line is str(value) = repr of the tuple, written by
    the native row writer; strings with quotes fall back to the host sink and give the same lines."""
    from fake_device import FakeTextCtx, FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: FakeTextCtx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})

    def lines_of(d):
        out = []
        for fn in sorted(os.listdir(d)):
            with open(os.path.join(d, fn)) as f:
                out.extend(l.rstrip("\n") for l in f)
        return out

    def native():
        return any("native frame sink" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    data = gen.text(6, 2500, V=700)
    p = tmp_path / "c.txt"
    p.write_bytes(data)
    counts = Dampr.text(str(p)).flat_map(lambda x: x.split()).count()
    rows = counts.read()
    counts.sink(str(tmp_path / "s1")).run()
    assert native()
    assert sorted(lines_of(str(tmp_path / "s1"))) == sorted(str(r) for r in rows)
    n = len(rows)
    idf = counts.cross_right(counts.len(), lambda df, total: (df[0], df[1], math.log(1 + float(total) / df[1])))
    idf.sink(str(tmp_path / "s2")).run()
    assert native()
    assert sorted(lines_of(str(tmp_path / "s2"))) == sorted(str((w, c, math.log(1 + float(n) / c))) for w, c in rows)
    counts.map(lambda x: (x[1],)).sink(str(tmp_path / "s3")).run()       # 1-tuples: "(3,)"
    assert native()
    assert sorted(lines_of(str(tmp_path / "s3"))) == sorted(str((c,)) for _w, c in rows)
    q = tmp_path / "q.txt"
    q.write_bytes(b"it's a \"quoted\" line\nplain words only\n")
    qc = Dampr.text(str(q)).flat_map(lambda x: x.split()).count()
    qc.sink(str(tmp_path / "s4")).run()
    assert not native()
    assert sorted(lines_of(str(tmp_path / "s4"))) == sorted(str(r) for r in qc.read())

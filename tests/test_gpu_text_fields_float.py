"""Float columns of delimited text on the device (csrc/fields.cu with csrc/fparse.cuh): float() minima and maxima
through the table, float sums and mean() through record mode (dampr_text_fields_records). Parse exactness through
the public path, record order across range cuts, and sums, minima, maxima and means against Python, asserting which
path each stage took."""
import math
import os
import random
import struct
import zlib

import numpy as np
import pytest

from fields_standin import python_lines, reference_outputs, write_files
from test_fparse_host import corpus, in_grammar
from test_text_fields_float_lowering import GOLDEN, NEEDLE, PIPELINES, datasets, same_records, _kv_fns

pytestmark = pytest.mark.gpu


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "text_table_log2", settings.text_table_log2)
    monkeypatch.setattr(settings, "ingest_chunk_bytes", settings.ingest_chunk_bytes)
    yield settings
    plan.release_buffers()


def run(src, P):
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P}).run())
    return got, runner_mod.LAST_STATS.stages[0]


def bits(v):
    return struct.pack("<d", v)


@pytest.mark.parametrize("name", sorted(datasets()))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, (_s, how, _d) = run(src, P)
        k, v, _m = _kv_fns(src)
        same_records(got, exp, P, k, v)
        assert NEEDLE in how, (name, src, how)


def test_parse_exactness_through_the_public_path(engine, tmp_path):
    """the parser corpus as lines `i,<s>` under max: every device value is float(s) bit for bit, and the strings the
    device refuses come back as host lines (Python's value, or its ValueError for the rejected ones)"""
    cases = [s for _k, s in corpus()[::4] if "\n" not in s and "\r" not in s and "," not in s and s.isascii()]
    good = [s for s in cases if _float_or_none(s) is not None]
    text = "".join("%d,%s\n" % (i, s) for i, s in enumerate(good))
    P = write_files(tmp_path, [["f.csv", text]])
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    out = dict(Dampr.text(P).map(lambda l: l.split(",")).fold_by(lambda r: int(r[0]), value=lambda r: float(r[1]),
                                                                 binop=max).run())
    _s, how, detail = runner_mod.LAST_STATS.stages[0]
    assert NEEDLE in how, how
    assert len(out) == len(good)
    for i, s in enumerate(good):
        assert bits(out[i]) == bits(float(s)), (s, out[i])
    refused = sum(1 for s in good if not in_grammar(s))
    assert "host_lines=%d" % refused in detail, (refused, detail)


def _float_or_none(s):
    try:
        v = float(s)
    except ValueError:
        return None
    return None if v != v or (v == 0 and math.copysign(1.0, v) < 0) else v


def test_record_order_is_the_same_for_every_range_cut(ctx, engine):
    """dampr_text_fields_records over one text cut three ways: identical records, in line order, holes exactly at the
    lines the device leaves to the host"""
    from dampr_b200 import device as dev
    rng = random.Random(9)
    lines = []
    for i in range(60000):
        v = rng.choice(["%.3f" % rng.uniform(-50, 50), "1_0", "x", repr(rng.random()), "%d" % i])
        lines.append("%s,%s" % (rng.choice(["a", "bb", "é", "k" * 12, ""]), v) + ("\n" * rng.randrange(1, 3)))
    data = "".join(lines).encode()
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    n = len(data)
    spec = (ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_F64)
    outs = []
    for cuts in ([0, n], [0, n // 48 * 16, n // 24 * 16, n], [0] + sorted(rng.randrange(0, n // 16) * 16
                                                                     for _ in range(40)) + [n]):
        tab = ctx.table(16)
        kv = ctx.kv(len(data))
        for a, b in zip(cuts[:-1], cuts[1:]):
            if b > a:
                tab.fields_records(tb, a, b, spec, kv)
        st = tab.fields_stats()
        kv.set_size(st["records"])
        recs = kv.records()
        fb = set((np.sort(tab.fallback_lines()) >> np.uint64(16)).tolist())
        outs.append((recs, st, fb))
        kv.free()
        tab.free()
    tb.free()
    starts = [0] + [i + 1 for i, c in enumerate(data[:-1]) if c == 10]
    for recs, st, fb in outs:
        assert np.array_equal(recs, outs[0][0])
        assert len(recs) == len(starts) and st["records"] == len(starts)
        assert not st["flags"] & (dev.TF_RECFULL | dev.TF_COLLISION)
    recs = outs[0][0]
    holes = np.flatnonzero(recs[:, 0] == 0)
    assert set(np.array(starts)[holes].tolist()) == outs[0][2]
    for i in range(0, len(starts), 997):   # line order: record i is line i
        end = data.find(b"\n", starts[i])
        f = data[starts[i]:end].split(b",")
        if recs[i, 0]:
            assert recs[i, 1] == struct.unpack("<Q", struct.pack("<d", float(f[1])))[0]


@pytest.mark.parametrize("red", ["sum()", "reduce(min)", "reduce(max)", "mean"])
def test_folds_against_python(red, engine, tmp_path):
    """str keys (hashed ones too), CRLF text and .gz, several files, long lines, many host lines"""
    rng = random.Random(zlib.crc32(red.encode()))
    rows = []
    for i in range(30000):
        k = rng.choice(["a", "b", "q" * 12, "w%d" % rng.randrange(300), "long" * 300 if i % 997 == 0 else "c"])
        v = rng.choice(["%.6f" % rng.uniform(-1e5, 1e5), repr(rng.uniform(-1, 1)), "1_5.5", "%d" % i])
        rows.append("%s,%s,%d" % (k, v, i) + ("\r\n" if i % 101 == 0 else "\n"))
    files = [["a.csv", "".join(rows[:10000])], ["b.csv.gz", "".join(rows[10000:20000])],
             ["c.csv", "".join(rows[20000:])]]
    P = write_files(tmp_path, files)
    if red == "mean":
        src = "Dampr.text(P).map(lambda l: l.split(',')).mean(lambda r: r[0], lambda r: float(r[1]))"
    else:
        src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[1])).%s" % red
    got, (_s, how, detail) = run(src, P)
    assert NEEDLE in how, (how, detail)
    key, value = (lambda l: l.split(",")[0]), (lambda l: float(l.split(",")[1]))
    exp = {}
    for l in python_lines(P):
        k, v = key(l), value(l)
        if red == "mean":
            s, n = exp.get(k, (0.0, 0))
            exp[k] = (s + v, n + 1)
        elif k in exp:
            exp[k] = {"sum()": lambda a, b: a + b, "reduce(min)": min, "reduce(max)": max}[red](exp[k], v)
        else:
            exp[k] = v
    if red == "mean":
        exp = {k: s / float(n) for k, (s, n) in exp.items()}
    same_records(got, sorted(repr(x) for x in exp.items()), P, key, (lambda l: value(l)) if red != "mean" else
                 _MeanValue(value))


class _MeanValue(object):
    """a value function whose repr marks a mean (one more rounding in same_records' bound)"""
    def __init__(self, f):
        self.f = f

    def __call__(self, l):
        return self.f(l)

    def __repr__(self):
        return "mean"


def test_int_mean_is_bit_equal(engine, tmp_path):
    rng = random.Random(4)
    lines = ["%d\t%s\t%d" % (rng.randrange(-20, 20), rng.choice("xyz"), rng.randrange(-10 ** 12, 10 ** 12))
             for _ in range(50000)]
    P = write_files(tmp_path, [["f.tsv", "\n".join(lines) + "\n"]])
    got, (_s, how, detail) = run("Dampr.text(P).map(lambda l: l.split('\\t')).mean(lambda r: int(r[0]), "
                                 "lambda r: int(r[2]))", P)
    exp = {}
    for l in lines:
        f = l.split("\t")
        s, n = exp.get(int(f[0]), (0, 0))
        exp[int(f[0])] = (s + int(f[2]), n + 1)
    assert got == sorted(repr((k, s / float(n))) for k, (s, n) in exp.items())
    assert NEEDLE in how and "op=mean_i64" in detail


def test_regrow_rescan_and_reproducibility(engine, monkeypatch, tmp_path):
    """short lines overflow the first record buffer (RECFULL, one rescan), many keys regrow the table, and the float
    sums are the same bits over three runs and three chunk sizes"""
    from dampr_b200 import plan
    sizes = []
    orig = plan.FieldScan._records_buffer
    monkeypatch.setattr(plan.FieldScan, "_records_buffer", lambda self, n: (sizes.append(n), orig(self, n))[1])
    engine.text_table_log2 = 12
    rng = random.Random(8)
    text = "".join("k%d,%r\n" % (rng.randrange(5000), rng.uniform(-1, 1) * 10 ** rng.randrange(-6, 7))
                   for _ in range(400000))
    P = write_files(tmp_path, [["f.csv", text]])
    src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[1])).sum()"
    outs = set()
    for chunk in (1 << 16, 1 << 20, 1 << 26, 1 << 26):
        engine.ingest_chunk_bytes = chunk
        del sizes[:]
        got, (_s, how, _d) = run(src, P)
        assert NEEDLE in how
        # the first guess is too small for these short lines: RECFULL, then one buffer of exactly the line count
        assert len(sizes) == 2 and sizes[0] < 400000 and sizes[1] == 400000, sizes
        outs.add(tuple(got))
    assert len(outs) == 1 and engine.text_table_log2 > 12
    key, value = (lambda l: l.split(",")[0]), (lambda l: float(l.split(",")[1]))
    exp = {}
    for l in text.splitlines():
        exp[key(l)] = exp[key(l)] + value(l) if key(l) in exp else value(l)
    same_records(list(outs)[0], sorted(repr(x) for x in exp.items()), P, key, value)


@pytest.mark.parametrize("text,red", [("a,-0.0\na,0.0\n", "reduce(max)"), ("a,1\na,-0\n", "reduce(min)"),
                                      ("a,1\na,-1e-999\n", "sum()"), ("a,1\na,nan\n", "reduce(max)")])
def test_negative_zero_and_nan_refusals(text, red, engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", text]])
    src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[1])).%s" % red
    got, (_s, how, _d) = run(src, P)
    assert how.startswith("host-map"), how
    vals = [float(l.split(",")[1]) for l in text.split()]
    r = vals[0]
    for v in vals[1:]:
        r = {"reduce(max)": max, "reduce(min)": min, "sum()": lambda x, y: x + y}[red](r, v)
    assert got == [repr(("a", r))]


def test_downstream_sort_and_sink(engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,3.5\nb,5.25\na,4\nc,1e-3\n"]])
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    out = str(tmp_path / "out")
    Dampr.text(P).map(lambda l: l.split(",")).mean(lambda r: r[0], lambda r: float(r[1])) \
        .sort_by(lambda x: -x[1]).sink_tsv(out).run()
    lines = []
    for fn in sorted(os.listdir(out)):
        with open(os.path.join(out, fn)) as f:
            lines.extend(l.rstrip("\n") for l in f)
    assert lines == ["b\t5.25", "a\t3.75", "c\t0.001"]
    assert NEEDLE in runner_mod.LAST_STATS.stages[0][1]

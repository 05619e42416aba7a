"""The field-scan kernels (csrc/fields.cu) line by line against their stand-ins and CPython, over the fuzzed corpora
and generated stages of tests/fields_fuzz.py.

Per-line record mode: each family (separator byte, split(), JSON) runs generated stages until every build it has
(fields_fuzz.builds_of: plain, WHERE, tuple and expression calls, the last two with and without filters; counts, int
and float values) has run PER_BUILD times with cr_is_data off and on, over LINES lines each. Counts have no record
mode: their per-line outcomes are checked through the table's counts, fallback list and dropped count. A line's device outcome is TAKE when its record has a nonzero code, HOST when
its hole's `offset << 16 | length` is in fallback_lines(), DROP otherwise. It must equal the stand-in's (class, code,
value bits) and be sound against CPython, and fields_stats() must equal the stand-in's. The same stage then runs in
table mode under every table op of its value type (fold per code, hashed keys' representatives, the fallback list and
the dropped count) and as 3-6 ranges cut at random byte offsets (the records and the fallback list byte for byte).

Separator sweep: all 125 separator bytes through the plain and WHERE record builds, SWEEP_LINES lines each.
End to end: E2E pipelines per family through Dampr.text / Dampr.json over fuzzed files, one gzipped, against plain
Python, exceptions included.

The Python oracles set the time (about 0.1 ms per line for both): 3 x 36 stages x 5000 lines + 125 x 2 x 1500 lines,
about 9 x 10^5 oracle lines. The file ran in 64 s on one H100 80GB HBM3 (700 W power limit)."""
import collections
import gzip
import json
import operator
import os
import random

import numpy as np
import pytest

import fields_fuzz as fz
from fields_standin import python_lines
from test_text_fields_where_lowering import same_up_to_rounding

pytestmark = pytest.mark.gpu

LINES, SWEEP_LINES, E2E = 5000, 1500, 30
# stages per (build, cr_is_data), fields_fuzz.builds_of: 18 text and 6 JSON builds, so 36 stages per family
PER_BUILD = {"sep": 1, "ws": 1, "json": 3}
NEEDLE = "device text fields scan+combine"


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "ingest_chunk_bytes", settings.ingest_chunk_bytes)
    yield settings
    plan.release_buffers()


@pytest.fixture(scope="module")
def path(tmp_path_factory):
    p = tmp_path_factory.mktemp("fzg") / "f.txt"
    p.write_bytes(b"a,1\n")
    return str(p)


class Text(object):
    """a corpus uploaded to the device"""

    def __init__(self, ctx, data):
        self.data, self.lines = data, fz.lines_of(data)
        self.tb = ctx.textbuf(len(data) + 64)
        self.tb.upload_all(np.frombuffer(data, dtype=np.uint8))


def scan_records(ctx, b, text, cr, cuts=None):
    """(records uint64 [n, 2], sorted fallback list, fields_stats()) of b's record call over text, as one range or
    cut at the byte offsets `cuts`"""
    tab, kv = ctx.table(17), ctx.kv(len(text.lines) + 16)
    try:
        bounds = [0] + list(cuts or []) + [len(text.data)]
        for lo, hi in zip(bounds, bounds[1:]):
            b.records(tab, text.tb, lo, hi, kv, cr)
        st = tab.fields_stats()
        kv.set_size(st["records"])
        return kv.records(), sorted(tab.fallback_lines().tolist()), st
    finally:
        kv.free()
        tab.free()


def device_outcomes(text, recs, fb):
    fb = set(fb)
    out = []
    for i, (off, line) in enumerate(text.lines):
        code, bits = int(recs[i, 0]), int(recs[i, 1])
        out.append((fz.TAKE, code, bits) if code else (fz.HOST,) if (off << 16 | len(line)) in fb else (fz.DROP,))
    return out


def check_count(ctx, b, text, cr, tally, rng):
    """a count (value 1, no record mode): the table's counts per code, its fallback list and dropped count against the
    stand-in's outcomes and CPython's, as one range and cut into ranges"""
    from dampr_b200 import device as dev
    want = [fz.standin_outcome(b, line, cr) for _off, line in text.lines]
    for (off, line), w in zip(text.lines, want):
        py = fz.python_outcome(b.stage, line)
        why = fz.sound(b, line, w, py, cr)
        assert why is None, (b.stage.src, cr, line, w, py, why)
        tally[b.name(), cr][w[0]] += 1
    exp_fb = sorted(off << 16 | len(line) for (off, line), w in zip(text.lines, want) if w[0] == fz.HOST)
    exp = fz.expected_stats(b, want)
    cuts = sorted(rng.sample(range(16, len(text.data), 16), max(0, min(rng.randint(2, 5), len(text.data) // 16 - 1))))
    for bounds in ([0, len(text.data)], [0] + cuts + [len(text.data)]):
        tab = ctx.table(17)
        try:
            for lo, hi in zip(bounds, bounds[1:]):
                b.table(tab, text.tb, lo, hi, dev.OP_SUM_I64, cr)
            codes, vals = tab.fields_fetch(dev.OP_SUM_I64)
            st = tab.fields_stats()
            fb = sorted(tab.fallback_lines().tolist())
        finally:
            tab.free()
        assert dict(zip(codes.tolist(), vals.tolist())) == fz.table_fold(want, dev.OP_SUM_I64), b.stage.src
        assert fb == exp_fb, (b.stage.src, bounds)
        assert st["records"] == sum(w[0] == fz.DROP for w in want), (b.stage.src, st)
        assert all(st[k] == exp[k] for k in exp if k != "records"), (b.stage.src, st, exp)


def check_build(ctx, b, text, cr, tally, rng):
    """the record, table and range-cut checks of build b over text"""
    from dampr_b200 import device as dev
    if b.spec[3] == dev.FIELD_VAL_ONE:
        return check_count(ctx, b, text, cr, tally, rng)
    recs, fb, st = scan_records(ctx, b, text, cr)
    assert st["records"] == len(text.lines), st
    assert not st["flags"] & (dev.TF_NONASCII | dev.TF_LONGLINE | dev.TF_RECFULL | dev.TF_TABLEFULL), st
    want = [fz.standin_outcome(b, line, cr) for _off, line in text.lines]
    got = device_outcomes(text, recs, fb)
    for (off, line), g, w in zip(text.lines, got, want):
        assert g == (tuple(w) if w[0] != fz.HOST else (fz.HOST,)), (b.stage.src, cr, off, line, g, w)
        py = fz.python_outcome(b.stage, line)
        why = fz.sound(b, line, g, py, cr)
        assert why is None, (b.stage.src, cr, line, g, py, why)
        tally[b.name(), cr][g[0]] += 1
    exp = fz.expected_stats(b, want)
    assert {k: st[k] for k in exp} == exp, (b.stage.src, st, exp)

    # table mode under every table op of the value type
    ops = [dev.OP_MIN_F64, dev.OP_MAX_F64] if b.flt else [dev.OP_SUM_I64, dev.OP_MIN_I64, dev.OP_MAX_I64]
    for op in ops:
        tab = ctx.table(17)
        try:
            b.table(tab, text.tb, 0, len(text.data), op, cr)
            codes, vals = tab.fields_fetch(op)
            _c, _n, reps = tab.fetch()
            tst = tab.fields_stats()
            tfb = sorted(tab.fallback_lines().tolist())
        finally:
            tab.free()
        vals = vals.view(np.uint64) if b.flt else vals
        assert dict(zip(codes.tolist(), vals.tolist())) == fz.table_fold(want, op), (b.stage.src, op)
        assert tfb == fb and tst["records"] == sum(w[0] == fz.DROP for w in want), (b.stage.src, op, tst)
        if op == ops[0] and b.kind != "expr":
            lows = {}
            for (off, line), w in zip(text.lines, want):
                if w[0] == fz.TAKE and (b.kind == "tuple" or not b.int_key and not 1 <= len(w.key) <= 9):
                    rep = (off << 20 | len(line)) if b.kind == "tuple" else (off + w.key_off) << 20 | len(w.key)
                    lows[w[1]] = min(lows.get(w[1], rep), rep)
            got_reps = dict(zip(_c.tolist(), reps.tolist()))
            assert all(got_reps[c] == r for c, r in lows.items()), b.stage.src

    # range cuts, some inside lines
    # (the calls take ranges on 16-byte boundaries)
    cuts = sorted(rng.sample(range(16, len(text.data), 16), max(0, min(rng.randint(2, 5), len(text.data) // 16 - 1))))
    recs2, fb2, st2 = scan_records(ctx, b, text, cr, cuts)
    assert recs2.tobytes() == recs.tobytes() and fb2 == fb, (b.stage.src, cuts)


def test_found(ctx, path):
    """the minimal lines of earlier findings, first"""
    for family, filters, key, value, op, sep, line, cr in fz.FOUND:
        st = fz.Stage(family, None if family == "json" else "lambda l: l.split()" if sep is None else
                      "lambda l: l.split(%r)" % chr(sep), filters, key, value, op)
        assert fz.match(st, path) is not None, st
        text = Text(ctx, line + b"\n")
        try:
            check_build(ctx, fz.Build(st), text, cr, collections.defaultdict(collections.Counter), random.Random(0))
        finally:
            text.tb.free()


@pytest.mark.parametrize("family", fz.FAMILIES)
def test_per_line_against_the_standin_and_cpython(family, ctx, path):
    rng = random.Random(sum(map(ord, family)) + 1)
    generated, refused, stages = fz.cover(family, 2, path, PER_BUILD[family])
    tally = collections.defaultdict(collections.Counter)
    texts = {}
    try:
        for j, (b, cr, sep) in enumerate(stages):
            key = (sep if family == "sep" else 0, cr)
            if key not in texts:
                texts[key] = Text(ctx, fz.corpus(family, 11 * j, LINES, cr, sep))
            check_build(ctx, b, texts[key], cr, tally, rng)
    finally:
        for t in texts.values():
            t.tb.free()
    print("\n%s: %d stages (%d generated, %d refused)" % (family, len(stages), generated, refused))
    for k, c in sorted(tally.items()):
        print("  %-22s cr=%d %s" % (k[0], k[1], dict(c)))
    assert set(tally) == {(name, cr) for name in fz.builds_of(family) for cr in (False, True)}
    per_build = collections.defaultdict(collections.Counter)
    for (name, _cr), c in tally.items():
        per_build[name].update(c)
    for name, c in per_build.items():   # every build reaches both sides of its decision
        assert c[fz.TAKE] >= 50 and c[fz.HOST] >= 50, (name, c)
        assert "where" not in name or c[fz.DROP] >= 50, (name, c)


def test_every_separator_byte(ctx, path):
    """all 125 separator bytes through the plain and the WHERE record builds"""
    tally = collections.defaultdict(collections.Counter)
    rng = random.Random(3)
    for sep in fz.SEPS:
        cr = sep % 2 == 0
        text = Text(ctx, fz.corpus("sep", 20000 + sep, SWEEP_LINES, cr, sep))
        try:
            seen = set()
            for k in range(60):
                sts, _n = fz.gen_stages(30000 + 100 * sep + k, "sep", 1, path, sep)
                if not sts:
                    continue
                b = fz.Build(sts[0])
                if b.kind in ("plain", "where") and b.kind not in seen:
                    seen.add(b.kind)
                    check_build(ctx, b, text, cr, tally, rng)
                if len(seen) == 2:
                    break
            assert seen == {"plain", "where"}, sep
        finally:
            text.tb.free()
    total = collections.Counter()
    for c in tally.values():
        total.update(c)
    print("\nseparator sweep: %s" % dict(total))
    assert total[fz.TAKE] > 50000 and total[fz.DROP] > 5000 and total[fz.HOST] > 20000, total


# ---- end to end ---------------------------------------------------------------------------------------------------
def python_run(st, P):
    """plain Python of the stage over the reader's lines of P: sorted reprs of its records"""
    binop = {"count": operator.add, "sum": operator.add, "min": min, "max": max}
    out = {}
    for l in python_lines(P):
        r = st.map(l)
        if all(p(r) for p in st.filters):
            k, v = st.key(r), st.value(r)
            if st.op_name == "mean":
                s, c = out.get(k, (None, 0))
                out[k] = (v if s is None else s + v, c + 1)
            else:
                out[k] = binop[st.op_name](out[k], v) if k in out else v
    if st.op_name == "mean":
        return sorted(repr((k, s / c)) for k, (s, c) in out.items())
    return sorted(repr(x) for x in out.items())


def outcome(fn):
    """fn()'s value, or the type of the exception it raised"""
    try:
        return fn()
    except Exception as e:   # noqa: BLE001  the exception is the result under test
        return type(e)


@pytest.mark.parametrize("family", fz.FAMILIES)
def test_end_to_end(family, engine, tmp_path, caplog):
    """E2E generated stages through the planner over a fuzzed file and its gzipped copy (cr_is_data), against plain
    Python; a stage the planner matched runs on the device unless Python raises or the planner names a reason"""
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    rng = random.Random(sum(map(ord, family)) + 2)
    sep = ord(",")
    # t.txt: lines every stage reads, some of them host lines; f.txt: t.txt's and 20 fuzzed ones; g.txt.gz: t.txt's
    # with '\r\n' line ends, '\r' being data in a .gz file
    tame = fz.tame_lines(family, 5, 600)
    lines = list(tame)
    for _off, l in fz.lines_of(fz.corpus(family, 6, 20, False, sep)):
        lines.insert(rng.randrange(len(lines) + 1), l.decode("utf-8"))
    d = str(tmp_path)
    for name, ls in (("t.txt", tame), ("f.txt", lines)):
        with open(os.path.join(d, name), "w", newline="") as f:
            f.write("\n".join(ls) + "\n")
    with gzip.open(os.path.join(d, "g.txt.gz"), "wb") as f:
        f.write("\r\n".join(tame).encode("utf-8") + b"\n")
    stats = collections.Counter()
    n = 0
    while n < E2E:
        st = fz.gen_stage(rng, family, sep)
        st.filters_src = st.filters_src[:2]
        st = fz.Stage(family, st.map_src, st.filters_src, st.key_src, st.value_src, st.op_name)
        P = os.path.join(d, ["t.txt", "f.txt", "t.txt", "g.txt.gz"][n % 4])
        if fz.match(st, P) is None:
            continue
        n += 1
        exp = outcome(lambda: python_run(st, P))
        caplog.clear()
        got = outcome(lambda: sorted(repr(x) for x in eval(st.src, {"Dampr": Dampr, "P": P, "json": json}).run()))
        if isinstance(exp, type):
            assert got is exp, (st.src, P, got, exp)
            stats["raises"] += 1
            continue
        assert not isinstance(got, type), (st.src, P, got, exp)
        same_up_to_rounding(got, exp)
        output, how, _detail = runner_mod.LAST_STATS.stages[0]
        # a fallback of the field stage itself names its reason (plan.try_lower); another stage's does not count
        reasons = [r.getMessage() for r in caplog.records if "stage %s not lowered" % output in r.getMessage()]
        assert NEEDLE in how or reasons, (st.src, how)
        stats["device" if NEEDLE in how else "host"] += 1
        if NEEDLE not in how:
            print("host: %s: %s" % (st.src, reasons[0]))
    print("\n%s end to end: %s" % (family, dict(stats)))
    assert stats["device"] >= 5, stats

"""The WHERE builds of csrc/fields.cu with filter programs, line by line against the stand-in of
tests/fields_filter_standin.py and CPython, over the fuzzed corpora of tests/fields_fuzz.py and the random programs of
tests/fields_filter_fuzz.py (the expression record build: a constant key and value, so a kept line is always taken).
A line's device outcome is TAKE when its record has a nonzero code, HOST when its hole is on the fallback list, DROP
otherwise; it must equal the stand-in's, be sound against CPython, and the dropped count must match. Also: malformed
programs are refused by the library."""
import collections

import numpy as np
import pytest

import fields_filter_fuzz as ff

pytestmark = pytest.mark.gpu

STAGES, LINES = 40, 3000


@pytest.fixture(scope="module")
def path(tmp_path_factory):
    p = tmp_path_factory.mktemp("fffg") / "f.txt"
    p.write_bytes(b"a,1\n")
    return str(p)


@pytest.mark.parametrize("family", ["sep", "ws"])
def test_kernels_match_the_standin_and_python(family, path, ctx):
    sts, _refused = ff.stages(23, family, STAGES, path)
    tally = collections.Counter()
    for k, st in enumerate(sts):
        cr = k % 2 == 1
        data, lines = ff.corpus_lines(family, 300 + k, LINES, cr)
        tb = ctx.textbuf(len(data) + 64)
        tab, kv = ctx.table(12), ctx.kv(len(lines) + 16)
        try:
            tb.upload_all(np.frombuffer(data, dtype=np.uint8))
            tab.fields_expr_records(tb, 0, len(data), tuple(st.spec) + (st.op,), st.expr, kv, cr, st.preds)
            stats = tab.fields_stats()
            kv.set_size(stats["records"])
            recs, fb = kv.records(), set(tab.fallback_lines().tolist())
        finally:
            kv.free()
            tab.free()
            tb.free()
        assert stats["records"] == len(lines), (st.src, stats)
        drops = 0
        for i, (off, line) in enumerate(lines):
            got = ff.TAKE if int(recs[i, 0]) else ff.HOST if (off << 16 | len(line)) in fb else ff.DROP
            want, py = ff.standin_outcome(st, line, cr), ff.python_outcome(st, line)
            assert got == want, (st.src, cr, line, got, want, py)
            assert got == ff.HOST or got == py, (st.src, cr, line, got, py)
            drops += got == ff.DROP
            tally[got] += 1
        assert stats["records"] - stats["lines"] - stats["fallback"] == drops, (st.src, stats)
    assert min(tally[x] for x in (ff.TAKE, ff.DROP, ff.HOST)) > 1000, tally


def test_malformed_programs_are_refused(ctx):
    from dampr_b200 import device as dev
    data = b"a,1,x\nb,2,y\n"
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    spec = (ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64)
    js = (dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64)
    S, AND, OR, NOT = (dev.PRED_STR, 0, dev.CMP_EQ, ("a",)), (dev.PRED_AND, 0, 0, ()), (dev.PRED_OR, 0, 0, ()), \
        (dev.PRED_NOT, 0, 0, ())
    try:
        for preds in [
            [AND], [S, AND], [NOT], [S, S, AND, AND],                       # stack underflow
            [S, S, (dev.PRED_AND, 0, 0, (1,))],                             # a connective with a constant
            [S] + [NOT] * 9,                                                # 9 connectives
            [S] * 9 + [AND] * 7,                                            # 9 leaves among 16 entries
            [(dev.PRED_NFIELDS, dev.FIELD_LINE, dev.CMP_EQ, (2,))],          # NFIELDS of the line
            [(dev.PRED_LEN, 1, dev.CMP_IN, (2, 3))],                        # LEN with IN
            [(dev.PRED_NONBLANK, 1, dev.CMP_EQ, (1,))],                     # NONBLANK with a constant
            [(dev.PRED_INT, 1, dev.CMP_CONTAINS, (1,))],                    # CONTAINS on INT
            [(dev.PRED_LEN, 1, dev.CMP_STARTS, (1,))],                      # STARTS on LEN
            [(dev.PRED_MEMBER, 0, dev.CMP_IN, ())],                         # MEMBER in a field call
        ]:
            with pytest.raises(dev.DeviceError):
                tab.fields(tb, 0, len(data), spec, preds=preds)
        for preds in [[(dev.PRED_STR, dev.FIELD_LINE, dev.CMP_CONTAINS, ("a",))], [S, AND]]:
            with pytest.raises(dev.DeviceError):
                tab.json_fields(tb, 0, len(data), js, ["a", "b"], preds=preds)
        tab.clear()   # the same call with a well-formed program runs
        tab.fields(tb, 0, len(data), spec, preds=[S, (dev.PRED_STR, dev.FIELD_LINE, dev.CMP_CONTAINS, ("y",)), OR, NOT])
        st = tab.fields_stats()
        assert st["lines"] == 0 and st["records"] == 2, st   # (a or contains 'y') holds on both lines: both dropped
    finally:
        tab.free()
        tb.free()

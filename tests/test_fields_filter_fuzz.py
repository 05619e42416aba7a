"""The filter-program stand-in (tests/fields_filter_standin.py) line by line against CPython, over the fuzzed corpora
of tests/fields_fuzz.py and random programs of 1 .. 8 leaves (tests/fields_filter_fuzz.py): a line the stand-in takes
must pass every filter in Python without an exception, a line it drops must fail one without an exception. This is
the check that an undecided leaf never hides an exception. The kernels run the same stages in
test_gpu_fields_filter_fuzz.py."""
import collections

import pytest

import fields_filter_fuzz as ff

STAGES, LINES = 40, 1500


@pytest.fixture(scope="module")
def path(tmp_path_factory):
    p = tmp_path_factory.mktemp("fff") / "f.txt"
    p.write_bytes(b"a,1\n")
    return str(p)


@pytest.mark.parametrize("family", ["sep", "ws"])
def test_standin_is_sound_against_python(family, path):
    sts, refused = ff.stages(11, family, STAGES, path)
    assert refused < STAGES, refused   # most generated programs lower
    tally = collections.Counter()
    for k, st in enumerate(sts):
        cr = k % 2 == 1
        _data, lines = ff.corpus_lines(family, 100 + k, LINES, cr)
        for _off, line in lines:
            got, py = ff.standin_outcome(st, line, cr), ff.python_outcome(st, line)
            assert got == ff.HOST or got == py, (st.src, cr, line, got, py)
            tally[got, py] += 1
    # every outcome occurs, and the device decides most lines Python decides
    assert tally[ff.TAKE, ff.TAKE] > 1000 and tally[ff.DROP, ff.DROP] > 1000 and tally[ff.HOST, ff.HOST] > 1000, tally
    assert tally[ff.HOST, ff.TAKE] + tally[ff.HOST, ff.DROP] < tally[ff.TAKE, ff.TAKE] + tally[ff.DROP, ff.DROP], tally


def test_programs_use_every_leaf_kind(path):
    from dampr_b200 import device as dev
    kinds = collections.Counter()
    for family in ("sep", "ws"):
        for st in ff.stages(11, family, STAGES, path)[0]:
            for p in st.preds:
                kinds[p[0], p[2] if p[0] == dev.PRED_STR else None, p[1] == dev.FIELD_LINE] += 1
    for k in [(dev.PRED_STR, dev.CMP_CONTAINS, True), (dev.PRED_STR, dev.CMP_STARTS, False), (dev.PRED_LEN, None, True),
              (dev.PRED_NONBLANK, None, False), (dev.PRED_AND, None, False), (dev.PRED_OR, None, False),
              (dev.PRED_NOT, None, False), (dev.PRED_INT, None, False)]:
        assert kinds[k] > 0, (k, kinds)

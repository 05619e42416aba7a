"""Delimited-field folds over text (`l.split(S)[i]` keys with counts and int sums / minima / maxima): the matcher
(lowering.text_fields_spec), the planner path (plan.FieldScan) on the numpy stand-in for dampr_text_fields in
tests/fields_standin.py, and the results against the REAL reference (Refefer/Dampr), whose outputs are stored in
tests/golden/text_fields.json.gz (the ReferenceReplay pattern of test_float_key_lowering.py; DAMPR_REFERENCE=<checkout>
records them again). Cases where the user's lambda raises are checked against plain Python: the reference hangs
when one of its workers raises (SURVEY B6). The same pipelines run on the device in tests/test_gpu_text_fields.py."""
import operator
import os
import random

import pytest

from fields_standin import make_ctx, python_fold, reference_outputs, run_ours, write_files

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields.json.gz")
NEEDLE = "device text fields scan+combine"

# ---- inputs -----------------------------------------------------------------------------------------------------
# (|v| <= 10^16: 400 records stay below the 64-bit sum bound; the 'wide' input holds 18 and 19 digits)
INT_POOL = ["3", "-4", "007", "+5", " 42", "1_0", "-0", "0", "12 ", "9999999999999999", "-9999999999999999",
            "+0", "-00012", "5\t"]
KEY_POOL = ["", "a", "b", "k9", "abcdefghi", "abcdefghij", "x" * 41, "ключ", " sp ", "a\tb", "Zz", "0"]


def datasets():
    """name -> [[file name, text]]. Every line of 'mixed' has an int()-able third field (and fourth, when present);
    'blank' holds blank lines and lines with one field, for counts only."""
    rng = random.Random(11)
    mixed = []
    for i in range(400):
        f = [rng.choice(KEY_POOL), rng.choice(["p", "", "qq", "é"]), rng.choice(INT_POOL)]
        if rng.random() < 0.3:
            f.append(rng.choice(INT_POOL))
        mixed.append(",".join(f) + ("\r\n" if rng.random() < 0.05 else "\n"))
    blank = []
    for i in range(300):
        blank.append(",".join(rng.choice(KEY_POOL) for _ in range(rng.randint(1, 3))) if rng.random() > 0.1 else "")
    tsv = "\n".join("%s\t%d\t%s" % (rng.choice(["a", "b", "c", ""]), i, rng.choice(["1", "2", "-3"])) +
                    ("\r" if i % 7 == 0 else "") for i in range(120)) + "\n"
    return {
        "issue": [["events.csv", "a,x,3\nb,y,-4\n,z,007\na,w,+5\r\nb,v,1_0\n"]],
        "wide": [["wide.csv", "a,999999999999999999\nb,-999999999999999999\na,1234567890123456789\n"]],
        "mixed": [["mixed.csv", "".join(mixed).rstrip("\n")]],
        "blank": [["blank.csv", "\n".join(blank)]],
        "gz": [["t.tsv.gz", tsv]],
        "crlf_text": [["t.tsv", tsv]],
        "several": [["a.csv", "".join(mixed[:150])], ["b.csv", "".join(mixed[150:300]).rstrip("\n")],
                    ["c.csv.gz", "".join(mixed[300:])]],
    }


C3 = "Dampr.text(P).map(lambda l: l.split(','))"
PIPELINES = {
    "issue": [C3 + ".fold_by(lambda r: r[0], value=lambda r: int(r[2]), binop=lambda a, b: a + b)",
              "Dampr.text(P).count(lambda l: l.split(',')[0])",
              C3 + ".a_group_by(lambda r: r[0], lambda r: int(r[-1])).reduce(min)",
              C3 + ".a_group_by(lambda r: r[0], lambda r: int(r[-1])).reduce(max)",
              "Dampr.text(P).count(lambda l: int(l.split(',')[2]))"],
    "mixed": [C3 + ".fold_by(lambda r: r[0], value=lambda r: int(r[2]), binop=lambda a, b: a + b)",
              "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[-1])).sum()",
              C3 + ".a_group_by(lambda r: r[1], lambda r: int(r[2])).reduce(min)",
              C3 + ".a_group_by(lambda r: r[-3], lambda r: int(r[2])).reduce(max)",
              C3 + ".fold_by(lambda r: int(r[2]), value=lambda r: int(r[2]), binop=max)",
              "Dampr.text(P).count(lambda l: l.split(',')[1])",
              "Dampr.text(P).count(lambda l: int(l.split(',')[2]))"],
    "blank": ["Dampr.text(P).count(lambda l: l.split(',')[0])",
              "Dampr.text(P).count(lambda l: l.split(',')[-1])"],
    "gz": ["Dampr.text(P).map(lambda l: l.split('\\t')).fold_by(lambda r: r[0], value=lambda r: int(r[2]), "
           "binop=lambda a, b: a + b)",
           "Dampr.text(P).count(lambda l: l.split('\\t')[-1])"],
    "several": [C3 + ".fold_by(lambda r: r[0], value=lambda r: int(r[2]), binop=lambda a, b: a + b)",
                "Dampr.text(P).count(lambda l: l.split(',')[0])"],
}
PIPELINES["crlf_text"] = PIPELINES["gz"]
PIPELINES["wide"] = [C3 + ".fold_by(lambda r: r[0], value=lambda r: int(r[1]), binop=lambda a, b: a + b)",
                     C3 + ".a_group_by(lambda r: r[0], lambda r: int(r[1])).reduce(min)",
                     C3 + ".a_group_by(lambda r: r[0], lambda r: int(r[1])).reduce(max)",
                     "Dampr.text(P).count(lambda l: int(l.split(',')[1]))"]


# ---- the matcher ------------------------------------------------------------------------------------------------
def _spec(key, value, split=None):
    from dampr_b200 import lowering
    return lowering.text_fields_spec(key, value, split)


def test_matcher_accepts_the_field_shapes():
    from dampr_b200.lowering import FIELD_STR, FIELD_INT, FIELD_FLOAT
    one = lambda l: 1
    assert _spec(lambda l: l.split(",")[0], one) == (",", 0, FIELD_STR, None, FIELD_INT, False)
    assert _spec(lambda l: int(l.split("\t")[-2]), one) == ("\t", -2, FIELD_INT, None, FIELD_INT, False)
    assert _spec(lambda l: l.split(";")[3], lambda l: int(l.split(";")[-1])) == \
        (";", 3, FIELD_STR, -1, FIELD_INT, False)
    assert _spec(lambda l: int(l.split("|")[1]), lambda l: int(l.split("|")[1])) == \
        ("|", 1, FIELD_INT, 1, FIELD_INT, False)
    sp = lambda l: l.split(" ")
    assert _spec(lambda r: r[2], lambda r: int(r[5]), sp) == (" ", 2, FIELD_STR, 5, FIELD_INT, False)
    assert _spec(lambda r: int(r[-1]), one, sp) == (" ", -1, FIELD_INT, None, FIELD_INT, False)
    assert _spec(lambda r: r[0], lambda r: int(r[0]), sp) == (" ", 0, FIELD_STR, 0, FIELD_INT, False)
    assert _spec(lambda l: l.split(",")[0], lambda l: float(l.split(",")[1])) == \
        (",", 0, FIELD_STR, 1, FIELD_FLOAT, False)


def test_matcher_rejects_the_near_misses():
    one = lambda l: 1
    sp = lambda l: l.split(",")
    for key, value, split in [
        (lambda l: l.split()[0], one, None),                       # split() without a separator
        (lambda l: l.split(",", 1)[0], one, None),                 # maxsplit
        (lambda l: l.split("::")[0], one, None),                   # multi-character separator
        (lambda l: l.split("\n")[0], one, None),
        (lambda l: l.split("\r")[0], one, None),
        (lambda l: l.split("\0")[0], one, None),
        (lambda l: l.split("é")[0], one, None),                    # non-ASCII separator
        (lambda l: l.split(",")[0].strip(), one, None),
        (lambda l: (l.split(",")[0], l.split(",")[1]), one, None),  # tuple key
        (lambda l: l.split(",")[0], lambda l: 2, None),
        (lambda l: l.split(",")[0], lambda l: True, None),
        (lambda l: l.split(",")[0], lambda l: l.split(",")[1], None),   # str value
        (lambda l: l.split(",")[0], lambda l: int(l.split(";")[1]), None),   # two separators
        (lambda l: l.split(",")[True], one, None),
        (lambda l: l.split(",")[1:], one, None),
        (lambda l: l, one, None),
        (lambda r: r, one, sp),
        (lambda r: r[0], one, lambda l: l.split()),
        (lambda r: r[0], one, lambda l: l.lower().split(",")),
        (lambda r: r.split(",")[0], one, sp),
        (lambda r: float(r[0]), one, sp),
        (lambda r, s=1: r[0], one, sp),
    ]:
        assert _spec(key, value, split) is None, (key, value, split)


def test_tokenizer_mode_is_unchanged():
    from dampr_b200 import lowering
    assert lowering.tokenizer_mode(lambda x: x.split(",")) is None


def test_stage_matcher_rejects_filters_first_and_distributed(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1\nb,2\na,3\n"]])
    for src, lowered in [
        ("Dampr.text(P).count(lambda l: l.split(',')[0])", True),
        ("Dampr.text(P).filter(lambda l: l).count(lambda l: l.split(',')[0])", False),
        ("Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).first()", False),
        ("Dampr.text(P).map(lambda l: l.split(',')).group_by(lambda r: r[0], lambda r: int(r[1]))"
         ".reduce(lambda k, it: sum(it))", False),
    ]:
        got, hows, _stages = run_ours(src, P, monkeypatch)
        assert (NEEDLE in hows[0]) == lowered, (src, hows)
    from dampr_b200 import dist
    monkeypatch.setattr(dist, "active", lambda: True)
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    from dampr_b200 import Dampr
    pm = Dampr.text(P).count(lambda l: l.split(",")[0])
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    with pytest.raises(plan.NotLowerable):
        plan._lower_map(None, st, [pm.pmer.graph.inputs[st.inputs[0]]], 0)


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(datasets()))
def test_field_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, _stages = run_ours(src, P, monkeypatch)
        assert got == e, (name, src)
        assert NEEDLE in hows[0], (name, src, hows)


def test_the_issue_example():
    files = datasets()["issue"]
    exp = reference_outputs(files, PIPELINES["issue"], GOLDEN)
    assert exp[0] == ["('', 7)", "('a', 8)", "('b', 6)"]


# ---- planner paths on the stand-in ------------------------------------------------------------------------------
def test_host_lines_merge_and_stats(monkeypatch, tmp_path):
    """lines the device hands back (non-ASCII, CR, int() fields only Python parses) are folded on the host and
    merged; the stats line counts them"""
    text = "a,1\nb, 2\né,3\na,4\r\nb,1_0\nc,+7\n"
    P = write_files(tmp_path, [["f.csv", text]])
    for binop, red in ((operator.add, "sum()"), (min, "reduce(min)"), (max, "reduce(max)")):
        src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).%s" % red
        got, hows, _stages = run_ours(src, P, monkeypatch)
        assert got == python_fold(P, lambda l: l.split(",")[0], lambda l: int(l.split(",")[1]), binop), red
        assert NEEDLE in hows[0]
    from dampr_b200 import runner as runner_mod
    detail = runner_mod.LAST_STATS.stages[0][2]
    assert "host_lines=4" in detail and "lines=6" in detail and "groups=4" in detail, detail


def test_min_max_identities(monkeypatch, tmp_path):
    """MIN / MAX start from their identity, not from the cleared 0: all-positive minima, all-negative maxima"""
    P = write_files(tmp_path, [["f.csv", "a,5\na,9\nb,-3\nb,-8\nc,0\n"]])
    got, _hows, _stages = run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], lambda r: int(r[1]))"
                      ".reduce(min)", P, monkeypatch)
    assert got == ["('a', 5)", "('b', -8)", "('c', 0)"]
    got, _hows, _stages = run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], lambda r: int(r[1]))"
                      ".reduce(max)", P, monkeypatch)
    assert got == ["('a', 9)", "('b', -3)", "('c', 0)"]


def test_empty_key_and_int_key_equality(monkeypatch, tmp_path):
    """'' is a key (blank lines, empty fields); 007, 7 and +7 are one int key, -0 and 0 another"""
    P = write_files(tmp_path, [["f.csv", "\n,1\n007,1\n7,2\n+7,3\n-0,4\n0,5\n"]])
    got, hows, _stages = run_ours("Dampr.text(P).count(lambda l: l.split(',')[0])", P, monkeypatch)
    assert got == ["('', 2)", "('+7', 1)", "('-0', 1)", "('0', 1)", "('007', 1)", "('7', 1)"]
    with pytest.raises(ValueError):     # int('') of the blank line: the user's own exception
        run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: int(r[0]), "
                 "lambda r: int(r[-1])).sum()", P, monkeypatch)
    P = write_files(tmp_path, [["g.csv", "007,1\n7,2\n+7,3\n-0,4\n0,5\n"]])
    got, hows, _stages = run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: int(r[0]), "
                         "lambda r: int(r[1])).sum()", P, monkeypatch)
    assert got == ["(0, 9)", "(7, 6)"] and NEEDLE in hows[0]


def test_overflow_bound_refuses_and_the_host_sums_exactly(monkeypatch, tmp_path):
    """records x max|v| >= 2^62: the device sum is refused, the host path gives Python's unbounded sum"""
    P = write_files(tmp_path, [["f.csv", "".join("a,999999999999999999\n" for _ in range(10)) + "b,1\n"]])
    src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).sum()"
    got, hows, _stages = run_ours(src, P, monkeypatch)
    assert got == ["('a', 9999999999999999990)", "('b', 1)"]
    assert NEEDLE not in hows[0] and hows[0].startswith("host-map"), hows
    # a 19-digit value is the host's (Python int): its sum is checked with the same bound
    P = write_files(tmp_path, [["g.csv", "a,1234567890123456789\na,1234567890123456789\na,1234567890123456789\n"
                                         "a,1234567890123456789\n"]])
    got, hows, _stages = run_ours(src, P, monkeypatch)
    assert got == ["('a', 4938271560493827156)"] and NEEDLE not in hows[0]
    P = write_files(tmp_path, [["h.csv", "a,1234567890123456789\nb,-5\n"]])
    got, hows, _stages = run_ours(src, P, monkeypatch)
    assert got == ["('a', 1234567890123456789)", "('b', -5)"] and NEEDLE in hows[0]


def test_host_values_outside_int64_send_min_max_to_the_host(monkeypatch, tmp_path):
    """a 20-digit host value sends the stage to the host map even where the merge would keep the device value of
    its key"""
    for red, big in (("reduce(min)", "12345678901234567890"), ("reduce(max)", "-12345678901234567890")):
        P = write_files(tmp_path, [["f.csv", "a,5\na,%s\nb,1\n" % big]])
        src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).%s" % red
        got, hows, _stages = run_ours(src, P, monkeypatch)
        assert got == ["('a', 5)", "('b', 1)"] and hows[0].startswith("host-map"), (red, hows)


def test_user_exceptions_reach_the_caller(monkeypatch, tmp_path):
    """a missing field raises IndexError, a non-numeric field ValueError, as plain Python does"""
    P = write_files(tmp_path, [["f.csv", "a,1\nb\n"]])
    with pytest.raises(IndexError):
        run_ours("Dampr.text(P).map(lambda l: l.split(',')).fold_by(lambda r: r[0], value=lambda r: int(r[1]), "
                 "binop=lambda a, b: a + b)", P, monkeypatch)
    P = write_files(tmp_path, [["g.csv", "a,1\nb,x\n"]])
    with pytest.raises(ValueError):
        run_ours("Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).sum()", P,
                 monkeypatch)


def test_too_many_host_lines_send_the_stage_to_the_host(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "é,1\n" * 65537 + "a,2\n"]])
    got, hows, _stages = run_ours("Dampr.text(P).count(lambda l: l.split(',')[0])", P, monkeypatch)
    assert got == ["('a', 1)", "('é', 65537)"]
    assert hows[0].startswith("host-map"), hows


def test_table_regrow_and_long_keys(monkeypatch, tmp_path):
    """more distinct keys than half the table: a 4x table and a second scan; keys longer than the fetch width are
    read back from their representative occurrence"""
    from dampr_b200 import settings
    monkeypatch.setattr(settings, "text_table_log2", 10)
    lines = ["%s,%d" % (("k%d" % i) * (1 + i % 9), i % 5) for i in range(1500)]
    P = write_files(tmp_path, [["f.csv", "\n".join(lines + lines[:100])]])
    src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).sum()"
    got, hows, _stages = run_ours(src, P, monkeypatch)
    assert got == python_fold(P, lambda l: l.split(",")[0], lambda l: int(l.split(",")[1]), operator.add)
    assert NEEDLE in hows[0] and settings.text_table_log2 == 12


def test_downstream_sort_and_sink(monkeypatch, tmp_path):
    """the frame a field fold returns feeds sort_by and sink_tsv unchanged"""
    P = write_files(tmp_path, [["f.csv", "a,3\nb,5\na,4\nc,1\n"]])
    from fake_device import FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: make_ctx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})
    out = str(tmp_path / "out")
    Dampr.text(P).a_group_by(lambda l: l.split(",")[0], lambda l: int(l.split(",")[1])).sum() \
        .sort_by(lambda x: -x[1]).sink_tsv(out).run()
    lines = []
    for fn in sorted(os.listdir(out)):
        with open(os.path.join(out, fn)) as f:
            lines.extend(l.rstrip("\n") for l in f)
    assert lines == ["a\t7", "b\t5", "c\t1"]
    assert NEEDLE in runner_mod.LAST_STATS.stages[0][1]

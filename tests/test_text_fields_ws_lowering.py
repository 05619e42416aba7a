"""Whitespace-split field folds (`line.split()[i]`, DAMPR_FIELD_SEP_WS of dampr_text_fields): the matchers
(lowering.text_fields_spec, lowering.field_predicate and plan._match_text_fields with split() in key, value, filter and
map positions), the planner path on the numpy stand-in of tests/fields_ws_standin.py, and the results against the REAL
reference (Refefer/Dampr), whose outputs are stored in tests/golden/text_fields_ws.json.gz (DAMPR_REFERENCE=<checkout>
records them again). Cases where the user's lambda raises are checked against plain Python: the reference hangs when
one of its workers raises (SURVEY B6). The same pipelines run on the device in tests/test_gpu_text_fields_ws.py."""
import os
import random

import pytest

from fields_standin import python_lines, reference_outputs, run_ours, write_files
from fields_ws_standin import WsLine, make_ws_ctx, ws_field_offsets
from test_text_fields_where_lowering import same_up_to_rounding

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_ws.json.gz")
NEEDLE = "device text fields scan+combine"


def ours(src, P, monkeypatch):
    """run_ours on the stand-in that takes the whitespace split"""
    return run_ours(src, P, monkeypatch, ctx=make_ws_ctx())


# ---- inputs -----------------------------------------------------------------------------------------------------
RUNS = [" ", " ", " ", "  ", "\t", " \t", "\t\t ", "\x0b", "\x0c", "\x1c", "\x1d", "\x1e", "\x1f", "   "]
EDGES = ["", "", "", " ", "\t", " \x0c", "\x1f "]
UNICODE_WS = ["\u00a0", "\u2003", "\u3000"]


def log_text(n, seed, cr=False):
    """web-log style rows `host method path status bytes latency` joined by mixed runs of ASCII whitespace (the
    0x1C-0x1F bytes among them) with leading and trailing blanks; rows with too few fields, blank and all-whitespace
    lines, BAD rows whose bytes and latency no int() / float() takes, non-ASCII keys, and rows split only by non-ASCII
    whitespace (NBSP, U+2003, U+3000). cr: some rows hold '\\r' inside and end in '\\r\\n'"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        r = rng.random()
        if r < 0.04:
            rows.append(rng.choice(["", " ", "\t \x0b", "\x1c\x1d"]))
            continue
        if r < 0.08:
            f = ["short", "GET"][:rng.randint(1, 2)]
        elif r < 0.16:
            f = [rng.choice(["ghost", "h1", "h2"]), "BAD", "/x", "503", "x%d" % i, "oops"]
        else:
            # latencies are multiples of 1/8: their sums are exact in any order, so the reference's means are too
            f = [rng.choice(["h1", "h2", "h3", "10.0.0.%d" % rng.randrange(4), "k" * 12, "é",
                             "node-%d" % rng.randrange(9)]),
                 rng.choice(["GET", "POST", "PUT", "DELETE"]), rng.choice(["/", "/a", "/b/c", "/index.html"]),
                 str(rng.choice([200, 201, 301, 404, 500, 503])), str(rng.randrange(-500, 5000)),
                 rng.choice(["%.3f" % (rng.randrange(0, 64) / 8.0), "5e-1", "0.5", "+2.25", "7", "1.25E1"])]
        if r > 0.97:
            line = rng.choice(UNICODE_WS).join(f)
        else:
            line = rng.choice(EDGES) + "".join(x + rng.choice(RUNS) for x in f[:-1]) + f[-1] + rng.choice(EDGES)
        if cr and i % 23 == 5:
            line = line.replace(" ", "\r", 1) + "\r"
        rows.append(line)
    return "".join(r + "\n" for r in rows)


def blank_text(n, seed):
    rng = random.Random(seed)
    rows = []
    for _ in range(n):
        k = rng.randint(0, 4)
        rows.append(rng.choice(EDGES) + rng.choice(RUNS).join(rng.choice(["a", "b", "cc", "d" * 11, "0"])
                                                             for _ in range(k)) + rng.choice(EDGES + ["  \t"]))
    return "\n".join(rows) + "\n"


def double_text(n, seed):
    """rows of single- and double-spaced fields, some with a leading space: split(' ') sees '' fields, split() not"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        sp = rng.choice([" ", "  "])
        rows.append(rng.choice(["", "", " "]) + sp.join([rng.choice(["a", "b", "c"]), rng.choice(["x", "y"]),
                                                         str(rng.randrange(-50, 50))]))
    return "\n".join(rows) + "\n"


def datasets():
    log = log_text(600, 3)
    log_cr = log_text(400, 5, cr=True)
    return {
        "log": [["access.log", log]],
        "log_gz": [["access.log.gz", log_cr]],
        "crlf_text": [["access.log", log_cr.replace("\n", "\r\n")]],
        "several": [["a.log", log[:len(log) // 3]], ["b.log.gz", log_cr], ["c.log", log[len(log) // 3:]]],
        "blank": [["b.txt", blank_text(300, 9)]],
        "double": [["d.txt", double_text(300, 13)]],
    }


W = "Dampr.text(P).map(lambda l: l.split())"
LOG = [W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] != 'BAD')"
       ".a_group_by(lambda r: r[0], lambda r: int(r[4])).sum()",
       "Dampr.text(P).filter(lambda l: len(l.split()) >= 4).count(lambda l: l.split()[1])",
       W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] in ('GET', 'POST'))"
       ".mean(lambda r: r[0], lambda r: float(r[-1]))",
       W + ".filter(lambda r: len(r) > 5).filter(lambda r: r[1] != 'BAD')"
       ".a_group_by(lambda r: r[-6], lambda r: int(r[3])).reduce(max)",
       "Dampr.text(P).filter(lambda l: len(l.split(None)) == 6).filter(lambda l: l.split()[1] != 'BAD')"
       ".a_group_by(lambda l: int(l.split()[3]), lambda l: int(l.split(None)[-2])).reduce(min)",
       W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] != 'BAD')"
       ".a_group_by(lambda r: r[2], lambda r: float(r[5])).reduce(min)",
       W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] not in ('BAD', 'PUT'))"
       ".a_group_by(lambda r: r[0], lambda r: float(r[5])).reduce(max)",
       W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] != 'BAD')"
       ".fold_by(lambda r: r[1], value=lambda r: float(r[5]), binop=lambda a, b: a + b)",
       W + ".filter(lambda r: len(r) >= 1).count(lambda r: r[0])",
       "Dampr.text(P).filter(lambda l: len(l.split()) == 6).filter(lambda l: int(l.split()[3]) >= 400)"
       ".count(lambda l: l.split()[0])",
       W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] != 'BAD').mean(lambda r: r[1], lambda r: int(r[4]))"]
PIPELINES = {
    "log": LOG,
    "log_gz": LOG,
    "crlf_text": LOG,
    "several": LOG[:3],
    "blank": ["Dampr.text(P).filter(lambda l: len(l.split()) >= 2).count(lambda l: l.split()[1])",
              W + ".filter(lambda r: len(r) >= 1).count(lambda r: r[-1])",
              W + ".filter(lambda r: 3 <= len(r)).count(lambda r: r[-3])"],
    "double": ["Dampr.text(P).count(lambda l: l.split()[1])",
               "Dampr.text(P).count(lambda l: l.split(' ')[1])",
               "Dampr.text(P).a_group_by(lambda l: l.split()[0], lambda l: int(l.split()[-1])).sum()",
               "Dampr.text(P).a_group_by(lambda l: l.split(' ')[0], lambda l: int(l.split(' ')[-1])).sum()",
               "Dampr.text(P).map(lambda l: l.split()).filter(lambda r: int(r[2]) > 0).count(lambda r: r[1])"],
}


# ---- the matchers -----------------------------------------------------------------------------------------------
def test_spec_matcher_accepts_split_and_split_none():
    from dampr_b200 import lowering
    from dampr_b200.lowering import SEP_WS, FIELD_STR as S, FIELD_INT as I, FIELD_FLOAT as F

    def mv(value):
        return lambda v: (value(v), 1)   # the keyed value mean() builds (dsl.py)
    sp, spn = (lambda l: l.split()), (lambda l: l.split(None))
    cases = [
        ((lambda l: l.split()[0], lambda l: 1), (SEP_WS, 0, S, None, I, False)),
        ((lambda l: l.split(None)[-1], lambda l: int(l.split()[2])), (SEP_WS, -1, S, 2, I, False)),
        ((lambda l: int(l.split()[1]), lambda l: float(l.split(None)[-2])), (SEP_WS, 1, I, -2, F, False)),
        ((lambda r: r[0], lambda r: int(r[3]), sp), (SEP_WS, 0, S, 3, I, False)),
        ((lambda r: r[-1], lambda r: float(r[1]), spn), (SEP_WS, -1, S, 1, F, False)),
        ((lambda r: r[2], mv(lambda r: float(r[4])), sp), (SEP_WS, 2, S, 4, F, True)),
        ((lambda l: l.split()[0], mv(lambda l: int(l.split()[1]))), (SEP_WS, 0, S, 1, I, True)),
    ]
    for args, exp in cases:
        assert lowering.text_fields_spec(*args, whitespace=True) == exp, (args, exp)
        assert lowering.text_fields_spec(*args) is None   # a caller that only handles separator characters
    assert SEP_WS != " " and len(SEP_WS) != 1


def test_spec_matcher_refuses_other_forms():
    from dampr_b200 import lowering
    for args in [
        (lambda l: l.split(sep=None)[0], lambda l: 1),                   # keyword forms
        (lambda l: l.split(maxsplit=2)[0], lambda l: 1),
        (lambda l: l.split(None, 2)[0], lambda l: 1),                    # maxsplit
        (lambda l: l.split(None, -1)[0], lambda l: 1),
        (lambda l: l.strip().split()[0], lambda l: 1),                   # .strip() first
        (lambda l: l.split()[0], lambda l: int(l.split(" ")[1])),        # two separators
        (lambda l: l.split(",")[0], lambda l: int(l.split()[1])),
        (lambda r: r[0], lambda r: 1, lambda l: l.split(None, 1)),
        (lambda r: r[0], lambda r: 1, lambda l: l.rsplit()),
        (lambda r: r[0], lambda r: 1, lambda l: l.split("  ")),          # multi-character separator
    ]:
        assert lowering.text_fields_spec(*args, whitespace=True) is None, args


def test_predicate_matcher_with_split():
    from dampr_b200 import lowering
    from dampr_b200.lowering import SEP_WS, FIELD_STR as S, FIELD_INT as I, FIELD_FLOAT as F, FIELD_COUNT as N
    cases = [
        (lambda l: len(l.split()) >= 3, None, (SEP_WS, N, None, ">=", (3,))),
        (lambda l: l.split(None)[1] in ("GET", "POST"), None, (SEP_WS, S, 1, "in", ("GET", "POST"))),
        (lambda l: int(l.split()[-3]) < 400, None, (SEP_WS, I, -3, "<", (400,))),
        (lambda r: float(r[-1]) > 0.5, SEP_WS, (SEP_WS, F, -1, ">", (0.5,))),
        (lambda r: 0 == len(r), SEP_WS, (SEP_WS, N, None, "==", (0,))),
    ]
    for fn, rec, exp in cases:
        assert lowering.field_predicate(fn, rec, whitespace=True) == exp, exp
    for fn, rec in [(lambda l: len(l.split(maxsplit=1)) == 2, None), (lambda l: l.split(None, 1)[0] == "a", None),
                    (lambda l: l.split()[0] == "a", SEP_WS)]:   # after the map the argument is the record
        assert lowering.field_predicate(fn, rec, whitespace=True) is None


def _match(pm):
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    return plan._match_text_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]])


def test_stage_matcher_and_the_binding(tmp_path):
    from dampr_b200 import Dampr, device as dev
    t = Dampr.text(write_files(tmp_path, [["f.log", "a GET 1\n"]]))
    key, val = (lambda r: r[0]), (lambda r: int(r[2]))
    m = _match(t.filter(lambda l: len(l.split()) == 3).map(lambda l: l.split()).filter(lambda r: r[1] != "x")
               .a_group_by(key, val).sum())
    assert m[1] == (dev.FIELD_SEP_WS, 0, dev.FIELD_KEY_STR, 2)
    assert m[4] == ((dev.PRED_NFIELDS, 0, dev.CMP_EQ, (3,)), (dev.PRED_STR, 1, dev.CMP_NE, ("x",)))
    m = _match(t.count(lambda l: int(l.split(None)[-1])))
    assert m[1] == (dev.FIELD_SEP_WS, -1, dev.FIELD_KEY_INT, dev.FIELD_VAL_ONE) and m[4] == ()
    assert _match(t.map(lambda l: l.split(",")).a_group_by(key, val).sum())[1][0] == ord(",")
    for pm in [
        t.filter(lambda l: l.split(" ")[1] == "GET").map(lambda l: l.split()).a_group_by(key, val).sum(),
        t.filter(lambda l: len(l.split(" ")) == 3).count(lambda l: l.split()[0]),
        t.filter(lambda l: len(l.split()) == 3).count(lambda l: l.split(" ")[0]),
        t.filter(lambda l: l.split()[1] == "GET").map(lambda l: l.split(",")).a_group_by(key, val).sum(),
        t.map(lambda l: l.split(None, 2)).a_group_by(key, val).sum(),
        t.map(lambda l: l.split(maxsplit=2)).a_group_by(key, val).sum(),
        t.map(lambda l: l.split(sep=None)).a_group_by(key, val).sum(),
    ]:
        assert _match(pm) is None
    s = dev.fields_spec((dev.FIELD_SEP_WS, 0, dev.FIELD_KEY_STR, 2, dev.OP_SUM_I64), False, ())
    assert s.sep == 256 == dev.FIELD_SEP_WS and s.npreds == 0


# ---- the stand-in -----------------------------------------------------------------------------------------------
def test_the_standin_splits_like_str_split():
    line = b" \x1ca\x1fbb \t c\x0b\x0c"
    assert WsLine(line).split() == [b"a", b"bb", b"c"] and line.split() == [b"\x1ca\x1fbb", b"c"]
    assert ws_field_offsets(line) == [2, 4, 9] and WsLine(b" \t ").split() == []


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_ws_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = ours(src, P, monkeypatch)
        same_up_to_rounding(got, e)
        assert NEEDLE in hows[0], (name, src, hows)
        assert ("sep=ws" in stages[0][2]) == ("split(' ')" not in src), (src, stages[0][2])


def test_split_and_split_space_stay_different():
    """the same double-spaced rows folded both ways: both match Python, and they differ from each other"""
    exp = reference_outputs(datasets()["double"], PIPELINES["double"], GOLDEN)
    lines = python_lines_of(datasets()["double"][0][1])
    for i, (sp, j) in enumerate([(None, 1), (" ", 1)]):
        counts = {}
        for l in lines:
            k = l.split(sp)[j]
            counts[k] = counts.get(k, 0) + 1
        assert exp[i] == sorted(repr(x) for x in counts.items())
    assert exp[0] != exp[1] and exp[2] != exp[3]


def python_lines_of(text):
    return text.split("\n")[:-1]


def test_detail_of_a_separator_byte_is_unchanged(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1\nb,2\na,3\n"]])
    got, hows, stages = ours("Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1]))"
                             ".sum()", P, monkeypatch)
    assert got == ["('a', 4)", "('b', 2)"] and NEEDLE in hows[0]
    assert stages[0][2] == "op=sum_i64 bytes=12 lines=3 groups=2 host_lines=0"


# ---- planner paths on the stand-in ------------------------------------------------------------------------------
def test_long_keys_blank_lines_and_host_lines(monkeypatch, tmp_path):
    """hashed keys (longer than 9 bytes) decoded from their real offset, blank lines behind a len() filter, '\\r' in a
    text file and non-ASCII whitespace on the host"""
    rows = ["  %s\t%d " % ("key-%s" % ("x" * (i % 40)), i) for i in range(200)] + ["", " \t", "a\u00a0 5", "b\r7"]
    P = write_files(tmp_path, [["f.txt", "\n".join(rows) + "\n"]])
    src = W + ".filter(lambda r: len(r) == 2).a_group_by(lambda r: r[0], lambda r: int(r[1])).sum()"
    got, hows, stages = ours(src, P, monkeypatch)
    exp = {}
    for l in python_lines(P):
        r = l.split()
        if len(r) == 2:
            exp[r[0]] = exp.get(r[0], 0) + int(r[1])
    assert got == sorted(repr(x) for x in exp.items())
    assert NEEDLE in hows[0] and "sep=ws" in stages[0][2] and "filtered=2" in stages[0][2], stages
    # 'a\xa0 5' holds two fields for Python; 'b\r7' is the lines 'b' and '7' in text mode, both filtered on the host
    assert "host_lines=1" in stages[0][2], stages


@pytest.mark.parametrize("src,exc", [
    ("Dampr.text(P).count(lambda l: l.split()[0])", IndexError),
    (W + ".filter(lambda r: len(r) >= 1).a_group_by(lambda r: r[0], lambda r: int(r[-1])).sum()", ValueError),
    (W + ".filter(lambda r: r[0] != 'z').count(lambda r: r[0])", IndexError),
    (W + ".filter(lambda r: len(r) == 2).mean(lambda r: r[0], lambda r: float(r[1]))", ValueError),
])
def test_raising_lambdas_raise_as_in_python(src, exc, monkeypatch, tmp_path):
    """a blank line under an unguarded index, an int() / float() of a word: Python's own error"""
    P = write_files(tmp_path, [["f.txt", "a 1\n\nb  2\n \t\nc x\n"]])
    with pytest.raises(exc):
        ours(src, P, monkeypatch)

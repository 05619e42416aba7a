"""Tuple keys of field folds (`(l.split(S)[i], int(l.split(S)[j]), ...)`, dampr_text_fields_tuple): the matchers
(lowering.text_fields_spec with tuple_keys, plan._match_text_fields), the planner path on the numpy stand-in of
tests/fields_tuple_standin.py, the host merge of keys with device and host lines, and the results against the REAL
reference (Refefer/Dampr), whose outputs are stored in tests/golden/text_fields_tuple.json.gz (DAMPR_REFERENCE=
<checkout> records them again). Also the plain-Python statement of the tuple key code against the real 64-bit
collisions of tests/golden/code_collisions.json. The same pipelines run on the device in
tests/test_gpu_text_fields_tuple.py."""
import os
import random

import pytest

from fields_standin import python_lines, reference_outputs, run_ours, write_files
from fields_tuple_standin import make_tuple_ctx, tuple_code
from test_code_collisions import PAIRS, hash_state, long_code
from test_text_fields_where_lowering import same_up_to_rounding
from test_text_fields_ws_lowering import log_text

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_tuple.json.gz")
NEEDLE = "device text fields scan+combine"


def ours(src, P, monkeypatch):
    """run_ours on the stand-in that takes tuple keys"""
    return run_ours(src, P, monkeypatch, ctx=make_tuple_ctx())


# ---- inputs -----------------------------------------------------------------------------------------------------
def csv_text(n, seed, cr=False):
    """`host,method,path,status,bytes,latency` rows: hosts of 1..9 bytes and longer (hashed lengths), '' methods and
    paths, statuses written 200 / +200 / 0200, non-ASCII paths (a non-key field), BAD rows whose status no int()
    takes, short rows. Latencies are multiples of 1/8, so sums and means are exact in any order. cr: some rows hold
    '\\r' inside"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        r = rng.random()
        if r < 0.03:
            rows.append(rng.choice(["", "x", "a,b"]))
            continue
        st = rng.choice([200, 201, 404, 500, 7])
        f = [rng.choice(["h1", "h2", "10.0.0.%d" % rng.randrange(3), "host-with-a-long-name", ""]),
             rng.choice(["GET", "POST", "", "PUT"]),
             rng.choice(["/", "/a", "", "/b/c", "/é"]),
             rng.choice(["%d" % st, "+%d" % st, "0%d" % st]) if r > 0.08 else "BAD",
             str(rng.randrange(-500, 5000)),
             "%.3f" % (rng.randrange(0, 64) / 8.0)]
        line = ",".join(f)
        if cr and i % 19 == 4:
            line = line.replace(",", "\r,", 1)
        rows.append(line)
    return "".join(r + "\n" for r in rows)


def datasets():
    csv = csv_text(300, 11)
    csv_cr = csv_text(200, 12, cr=True)
    return {
        "csv": [["log.csv", csv]],
        "csv_gz": [["log.csv.gz", csv_cr]],
        "crlf_text": [["log.csv", csv_cr.replace("\n", "\r\n")]],
        "several": [["a.csv", csv[:len(csv) // 3]], ["b.csv.gz", csv_cr], ["c.csv", csv[len(csv) // 3:]]],
        "ws": [["access.log", log_text(300, 21)]],
    }


C = "Dampr.text(P).map(lambda l: l.split(','))"
CF = C + ".filter(lambda r: len(r) == 6).filter(lambda r: r[3] != 'BAD')"
CSV = [C + ".filter(lambda r: len(r) == 6).count(lambda r: (r[0], r[1]))",
       "Dampr.text(P).filter(lambda l: len(l.split(',')) == 6).filter(lambda l: l.split(',')[3] != 'BAD')"
       ".a_group_by(lambda l: (l.split(',')[0], int(l.split(',')[3])), lambda l: int(l.split(',')[4])).sum()",
       CF + ".a_group_by(lambda r: (r[0], r[1], int(r[3])), lambda r: float(r[5])).reduce(max)",
       CF + ".mean(lambda r: (r[-6], r[2], int(r[-3]), r[1]), lambda r: float(r[5]))",
       CF + ".fold_by(lambda r: (int(r[3]), r[0]), min, lambda r: int(r[4]))",
       C + ".filter(lambda r: len(r) == 6).count(lambda r: (r[1],))",
       CF + ".a_group_by(lambda r: (r[0], r[0], int(r[4])), lambda r: int(r[4])).sum()",
       CF + ".filter(lambda r: int(r[3]) >= 404).mean(lambda r: (r[1], int(r[3])), lambda r: int(r[4]))",
       CF + ".fold_by(lambda r: (r[2], r[1]), lambda a, b: a + b, lambda r: float(r[5]))",
       CF + ".a_group_by(lambda r: (int(r[3]), r[-1]), lambda r: float(r[-1])).reduce(min)"]
W = "Dampr.text(P).map(lambda l: l.split())"
WF = W + ".filter(lambda r: len(r) == 6).filter(lambda r: r[1] != 'BAD')"
WS = [WF + ".count(lambda r: (r[0], r[1]))",
      "Dampr.text(P).filter(lambda l: len(l.split()) == 6).filter(lambda l: l.split()[1] != 'BAD')"
      ".a_group_by(lambda l: (l.split()[0], int(l.split()[3])), lambda l: int(l.split()[4])).sum()",
      WF + ".mean(lambda r: (r[0], r[-4], int(r[3]), r[1]), lambda r: float(r[5]))",
      WF + ".filter(lambda r: r[1] in ('GET', 'POST')).a_group_by(lambda r: (r[1], r[2], int(r[-3])),"
      " lambda r: int(r[4])).reduce(max)"]
PIPELINES = {"csv": CSV, "csv_gz": CSV, "crlf_text": CSV[:5], "several": CSV[:4], "ws": WS}


# ---- the matchers -----------------------------------------------------------------------------------------------
def test_spec_matcher_accepts_tuples_of_projections():
    from dampr_b200 import lowering
    from dampr_b200.lowering import SEP_WS, FIELD_STR as S, FIELD_INT as I, FIELD_FLOAT as F, FIELD_TUPLE as T

    def mv(value):
        return lambda v: (value(v), 1)   # the keyed value mean() builds (dsl.py)
    sp = lambda l: l.split(",")   # noqa: E731
    cases = [
        ((lambda r: (r[0], r[3]), lambda r: 1, sp), (",", ((0, S), (3, S)), T, None, I, False)),
        ((lambda l: (l.split(",")[0], int(l.split(",")[-1])), lambda l: int(l.split(",")[2])),
         (",", ((0, S), (-1, I)), T, 2, I, False)),
        ((lambda r: (r[1],), lambda r: float(r[2]), sp), (",", ((1, S),), T, 2, F, False)),
        ((lambda r: (r[0], r[0], int(r[4]), r[-2]), mv(lambda r: int(r[4])), sp),
         (",", ((0, S), (0, S), (4, I), (-2, S)), T, 4, I, True)),
        ((lambda l: (l.split()[0], int(l.split(None)[3])), lambda l: 1), (SEP_WS, ((0, S), (3, I)), T, None, I, False)),
        ((lambda r: (int(r[2]), r[1]), mv(lambda r: float(r[-1])), lambda l: l.split()),
         (SEP_WS, ((2, I), (1, S)), T, -1, F, True)),
    ]
    for args, exp in cases:
        assert lowering.text_fields_spec(*args, whitespace=True, tuple_keys=True) == exp, (args, exp)
        assert lowering.text_fields_spec(*args, whitespace=True) is None   # a caller that does not opt in
    # a single key reads as before with the option on
    assert lowering.text_fields_spec(lambda r: r[0], lambda r: 1, sp, tuple_keys=True) == (",", 0, S, None, I, False)


def test_spec_matcher_refuses_other_tuples():
    from dampr_b200 import lowering
    sp = lambda l: l.split(",")   # noqa: E731
    for args in [
        (lambda r: (r[0], float(r[1])), lambda r: 1, sp),                # float() component
        (lambda r: (r[0], (r[1], r[2])), lambda r: 1, sp),               # nested tuple
        (lambda r: (r[0].lower(), r[1]), lambda r: 1, sp),               # not a bare projection
        (lambda r: (r[0], "x"), lambda r: 1, sp),                        # a constant
        (lambda r: (r[0] + r[1], r[2]), lambda r: 1, sp),
        (lambda r: (r[0], r[1], r[2], r[3], r[4]), lambda r: 1, sp),     # more than 4 components
        (lambda l: (l.split(",")[0], l.split(";")[1]), lambda l: 1, None),   # different separators
        (lambda l: (l.split(",")[0], l.split()[1]), lambda l: 1, None),
        (lambda l: (l.split(",")[0], l.split(",")[1]), lambda l: int(l.split()[2]), None),
        (lambda r: (), lambda r: 1, sp),                                 # no component
        (lambda r: [r[0], r[1]], lambda r: 1, sp),                       # a list is not hashable
        (lambda r: (r[0], r[int(r[1])]), lambda r: 1, sp),               # an index that is not a constant
    ]:
        assert lowering.text_fields_spec(*args, whitespace=True, tuple_keys=True) is None, args


def _match(pm):
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    return plan._match_text_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]])


def test_stage_matcher(tmp_path):
    from dampr_b200 import Dampr, plan, device as dev
    t = Dampr.text(write_files(tmp_path, [["f.csv", "a,1,2\n"]]))
    m = _match(t.map(lambda l: l.split(",")).filter(lambda r: r[1] != "x").count(lambda r: (r[0], int(r[-1]))))
    assert m[1] == (ord(","), ((0, dev.FIELD_KEY_STR), (-1, dev.FIELD_KEY_INT)), plan.KEY_TUPLE, dev.FIELD_VAL_ONE)
    assert m[2] == dev.OP_SUM_I64 and m[4] == ((dev.PRED_STR, 1, dev.CMP_NE, ("x",)),)
    m = _match(t.filter(lambda l: len(l.split()) == 3).a_group_by(lambda l: (l.split()[1], l.split()[0]),
                                                                    lambda l: float(l.split()[2])).reduce(min))
    assert m[1] == (dev.FIELD_SEP_WS, ((1, dev.FIELD_KEY_STR), (0, dev.FIELD_KEY_STR)), plan.KEY_TUPLE, 2)
    assert m[2] == dev.OP_MIN_F64
    for pm in [t.map(lambda l: l.split(",")).count(lambda r: (r[0], float(r[1]))),
               t.filter(lambda l: l.split(";")[0] == "a").count(lambda l: (l.split(",")[0], l.split(",")[1])),
               t.count(lambda l: (l.split(",")[0], l.split(",")[1], l.split(",")[2], l.split(",")[0],
                                  l.split(",")[1]))]:
        assert _match(pm) is None
    k = dev.field_keys(((0, dev.FIELD_KEY_STR), (-2, dev.FIELD_KEY_INT)))
    assert k.n == 2 and list(k.field)[:2] == [0, -2] and list(k.kind)[:2] == [0, 1]


# ---- the key code -----------------------------------------------------------------------------------------------
def test_the_code_statement():
    """one component of bytes is the hashed field key's code; int components and the 0xFF joints feed the stream"""
    for b in [b"", b"a", b"abcdefghijklmnop"]:
        assert tuple_code([b]) == long_code(b, "raw")
    assert tuple_code([b"a", 7]) == long_code(b"a\xff" + (7 ^ (1 << 63)).to_bytes(8, "little"), "raw")
    assert tuple_code([-1, b""]) == long_code((((-1) ^ (1 << 63)) & ((1 << 64) - 1)).to_bytes(8, "little") + b"\xff",
                                              "raw")
    assert len({tuple_code(p) for p in [[b"a", b"b"], [b"ab", b""], [b"", b"ab"], [b"ab"]]}) == 4
    assert all(tuple_code(p) >> 63 for p in [[0], [b"x", 5, b"y"]])


def test_raw_collisions_collide_as_first_components():
    """a raw pair shares the whole hash state, so any common suffix keeps the codes equal"""
    for a, b, state, code in PAIRS["raw"]:
        assert hash_state(a, "raw") == hash_state(b, "raw") == state
        for rest in [[b"GET"], [200], [b"x", -7, b""]]:
            assert tuple_code([a] + rest) == tuple_code([b] + rest)
        assert tuple_code([a]) == code and tuple_code([b, b"GET"]) != tuple_code([b, b"PUT"])


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_tuple_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = ours(src, P, monkeypatch)
        same_up_to_rounding(got, e)
        assert NEEDLE in hows[0] and " key=tuple" in stages[0][2], (name, src, hows, stages)
        assert ("sep=ws" in stages[0][2]) == (name == "ws")


def test_the_inputs_cover_the_cases():
    """hashed-length and '' components, int components written +200 / 0200 (the same key as 200), non-ASCII in a
    non-key field (its lines are the host's)"""
    csv = datasets()["csv"][0][1]
    assert "+200," in csv and ",0200," in csv and ",/é," in csv and ",," in csv and "host-with-a-long-name" in csv
    exp = reference_outputs(datasets()["csv"], PIPELINES["csv"], GOLDEN)
    assert "('h1', 200)" in " ".join(exp[1]) and "'+200'" not in " ".join(exp[1])


# ---- planner paths on the stand-in ------------------------------------------------------------------------------
def test_detail_and_int_normalisation(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,7\na,+7\na,07\nb,-0\nb,0\n"]])
    got, hows, stages = ours("Dampr.text(P).count(lambda l: (l.split(',')[0], int(l.split(',')[1])))", P,
                             monkeypatch)
    assert got == ["(('a', 7), 3)", "(('b', 0), 2)"] and NEEDLE in hows[0]
    assert stages[0][2] == "op=count bytes=23 lines=5 groups=2 host_lines=0 key=tuple2"
    got, hows, stages = ours("Dampr.text(P).count(lambda l: l.split(',')[0])", P, monkeypatch)
    assert stages[0][2] == "op=count bytes=23 lines=5 groups=2 host_lines=0"   # a single key's detail is unchanged


def test_keys_with_device_and_host_lines_merge(monkeypatch, tmp_path):
    """a key whose lines are split between the device and the host comes back once, folded over both"""
    rows = ["k%d,GET,%d,/p%s" % (i % 5, i, "é" if i % 3 == 0 else "") for i in range(300)] + ["k1,GET,9,\r"]
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    for src, binop in [(C + ".a_group_by(lambda r: (r[0], r[1]), lambda r: int(r[2])).sum()", lambda a, b: a + b),
                       (C + ".a_group_by(lambda r: (r[0], int(r[2]) // 100), lambda r: int(r[2])).reduce(max)", max)]:
        got, hows, stages = ours(src, P, monkeypatch)
        if "//" in src:   # a component that is not a bare projection: the host map's stage
            assert NEEDLE not in hows[0]
            continue
        exp = {}
        for l in python_lines(P):
            r = l.split(",")
            k = (r[0], r[1])
            exp[k] = binop(exp[k], int(r[2])) if k in exp else int(r[2])
        assert got == sorted(repr(x) for x in exp.items())
        assert NEEDLE in hows[0] and "host_lines=101" in stages[0][2], stages


def test_host_int_components_outside_int64_refuse(monkeypatch, tmp_path):
    """a 20-digit component parses on the host only; the merged column could not hold it, so the stage is the host
    map's and the answer is Python's"""
    P = write_files(tmp_path, [["f.csv", "a,1\na,99999999999999999999\nb,2\n"]])
    got, hows, _s = ours("Dampr.text(P).count(lambda l: (l.split(',')[0], int(l.split(',')[1])))", P, monkeypatch)
    assert got == ["(('a', 1), 1)", "(('a', 99999999999999999999), 1)", "(('b', 2), 1)"]
    assert NEEDLE not in hows[0]


def test_collisions_send_the_stage_to_the_host(monkeypatch, tmp_path):
    a, b, _s, _c = PAIRS["raw"][0]
    rows = ["%s,GET,1" % a.decode(), "%s,GET,2" % b.decode(), "%s,GET,3" % a.decode()]
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    got, hows, _s = ours(C + ".a_group_by(lambda r: (r[0], r[1]), lambda r: int(r[2])).sum()", P, monkeypatch)
    assert got == sorted(["((%r, 'GET'), 4)" % a.decode(), "((%r, 'GET'), 2)" % b.decode()])
    assert NEEDLE not in hows[0]


@pytest.mark.parametrize("src,exc", [
    ("Dampr.text(P).count(lambda l: (l.split(',')[0], l.split(',')[2]))", IndexError),
    ("Dampr.text(P).count(lambda l: (l.split(',')[0], int(l.split(',')[1])))", ValueError),
])
def test_raising_lambdas_raise_as_in_python(src, exc, monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,1,x\nb,2\nc,x,y\n"]])
    with pytest.raises(exc):
        ours(src, P, monkeypatch)

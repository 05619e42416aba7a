"""JSON-lines field folds (`Dampr.json(path)` = map(json.loads), dampr_text_json_fields): the matchers
(lowering.json_fields_spec, lowering.json_predicate, lowering.is_json_loads and plan._match_json_fields), the planner
path on the numpy stand-in of tests/fields_json_standin.py, and the results against the REAL reference
(Refefer/Dampr), whose outputs are stored in tests/golden/text_fields_json.json.gz (DAMPR_REFERENCE=<checkout> records
them again). Lines json.loads rejects, and lambdas that raise, are checked against plain Python: the reference hangs
when one of its workers raises (SURVEY B6). The same pipelines run on the device in tests/test_gpu_text_fields_json.py."""
import json
import os
import random

import pytest

from fields_json_standin import device_members, make_json_ctx
from fields_standin import reference_outputs, write_files
from test_text_fields_where_lowering import same_up_to_rounding

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_json.json.gz")
NEEDLE = "device text fields scan+combine"


def ours(src, P, monkeypatch):
    """run_ours on the stand-in that takes the JSON calls, with `json` in the pipeline's globals"""
    from fake_device import FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: make_json_ctx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P, "json": json}).run())
    return got, [h for _s, h, _d in runner_mod.LAST_STATS.stages], runner_mod.LAST_STATS.stages


# ---- inputs -----------------------------------------------------------------------------------------------------
def event(rng, i):
    """one event row: string user / host / method / endpoint, int bytes, int-or-string status, float latency (a
    multiple of 1/8: sums are exact in any order), an int zone, and a nested object holding decoy members named like
    the keys"""
    return {"user": "u%d" % rng.randrange(40), "host": rng.choice(["h1", "h2", "h3", "node-%d" % rng.randrange(5),
                                                                   "k" * 12]),
            "method": rng.choice(["GET", "POST", "PUT"]), "endpoint": rng.choice(["/", "/a", "/b/c"]),
            "status": rng.choice([200, 201, 404, 500, 503, "404", "500"]), "bytes": rng.randrange(-500, 5000),
            "latency": rng.randrange(0, 64) / 8.0, "zone": rng.randrange(-3, 4), "code": rng.choice([7, 8, 9]),
            "ratio": rng.choice([0.5, 1.25, -2.0, 3e-3]),
            "meta": {"user": "decoy", "host": ["h9", {"bytes": 1}]}}


def event_text(n, seed, cr=False):
    """JSON lines the device takes, and valid lines it hands back: escapes in values, names and keys, non-ASCII
    values, duplicate members, a wanted name spelt with an escape, NaN / Infinity, 20-digit ints in a nested object,
    nesting one past the device's limit, odd whitespace. cr: '\\r' between tokens (a .gz source keeps it, CRLF text drops it)"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        e = event(rng, i)
        r = rng.random()
        if r < 0.03:
            e["user"] = "ué%d" % (i % 3)            # non-ASCII: a host line
        elif r < 0.06:
            line = json.dumps(e)
            rows.append(line.replace('"user": "', '"user": "\\u0075', 1))   # an escaped key value
            continue
        elif r < 0.08:
            line = json.dumps(e)
            rows.append(line.replace('"host"', '"\\u0068ost"', 1))           # a wanted name with an escape
            continue
        elif r < 0.10:
            line = json.dumps(e)
            rows.append(line[:-1] + ', "host": "dup", "bytes": 7}')          # duplicates: the last one counts
            continue
        elif r < 0.11:
            e["meta"] = json.loads("[" * 64 + "]" * 64)                     # nesting 65 deep
        elif r < 0.12:
            e["meta"] = {"bytes": 10 ** 19 + i, "user": -(10 ** 25)}          # ints the device does not parse
        elif r < 0.13:
            e["meta"] = {"x": float("nan"), "y": float("inf")}               # NaN / Infinity
        line = json.dumps(e, separators=rng.choice([(",", ":"), (", ", ": "), (" ,\t", " :  ")]))
        if cr and i % 7 == 3:
            line = line.replace(",", "\r,", 2)
        rows.append(rng.choice(["", " ", "\t"]) + line + rng.choice(["", " ", "  \t"]))
    return "".join(r + "\n" for r in rows)


def datasets():
    ev = event_text(220, 3)
    ev_cr = event_text(120, 5, cr=True)
    cut = ev.index("\n", len(ev) // 3) + 1   # every file holds whole lines
    return {
        "events": [["events.jsonl", ev]],
        "events_gz": [["events.jsonl.gz", ev_cr]],
        "crlf_text": [["events.jsonl", ev.replace("\n", "\r\n")]],
        "several": [["a.jsonl", ev[:cut]], ["b.jsonl.gz", ev_cr], ["c.jsonl", ev[cut:]]],
    }


J = "Dampr.json(P)"
EVENTS = [
    J + ".count(lambda r: r['user'])",
    J + ".filter(lambda r: int(r['status']) >= 500).a_group_by(lambda r: r['host'], lambda r: r['bytes']).sum()",
    J + ".mean(lambda r: r['endpoint'], lambda r: float(r['latency']))",
    J + ".a_group_by(lambda r: r['host'], lambda r: r['bytes']).reduce(min)",
    J + ".filter(lambda r: r['method'] != 'PUT').a_group_by(lambda r: r['user'], lambda r: r['latency']).reduce(max)",
    J + ".filter(lambda r: 'meta' in r).filter(lambda r: r['method'] in ('GET', 'POST'))"
        ".fold_by(lambda r: r['host'], value=lambda r: float(r['latency']), binop=lambda a, b: a + b)",
    J + ".filter(lambda r: 'nope' not in r).mean(lambda r: r['method'], lambda r: r['bytes'])",
    J + ".count(lambda r: r['code'])",
    J + ".a_group_by(lambda r: r['host'], lambda r: r['ratio']).sum()",
    J + ".filter(lambda r: float(r['latency']) < 4.0).a_group_by(lambda r: int(r['zone']), "
        "lambda r: int(r['bytes'])).reduce(max)",
    "Dampr.text(P).map(lambda l: json.loads(l)).filter(lambda r: r['zone'] >= 0).count(lambda r: r['endpoint'])",
]
PIPELINES = {
    "events": EVENTS,
    "events_gz": EVENTS,
    "crlf_text": EVENTS[:4],
    "several": EVENTS[:3],
}


# ---- the matchers -----------------------------------------------------------------------------------------------
def test_spec_matcher_accepts_member_reads():
    from dampr_b200 import lowering
    from dampr_b200.lowering import FIELD_DATA as D, FIELD_INT as I, FIELD_FLOAT as F

    def mv(value):
        return lambda v: (value(v), 1)   # the keyed value mean() builds (dsl.py)
    cases = [
        ((lambda r: r["user"], lambda r: 1), ("user", D, None, I, False)),
        ((lambda r: r["h"], lambda r: r["b"]), ("h", D, "b", D, False)),
        ((lambda r: int(r["z"]), lambda r: float(r["l"])), ("z", I, "l", F, False)),
        ((lambda r: r["e"], mv(lambda r: float(r["l"]))), ("e", D, "l", F, True)),
        ((lambda r: r["e"], mv(lambda r: r["b"])), ("e", D, "b", D, True)),
        ((lambda r: r[""], lambda r: int(r["x y"])), ("", D, "x y", I, False)),
    ]
    for args, exp in cases:
        assert lowering.json_fields_spec(*args) == exp, (args, exp)


def test_spec_matcher_refuses_other_forms():
    from dampr_b200 import lowering
    for args in [
        (lambda r: r.get("a"), lambda r: 1),
        (lambda r: r["a"]["b"], lambda r: 1),
        (lambda r: len(r), lambda r: 1),
        (lambda r: (r["a"], r["b"]), lambda r: 1),
        (lambda r: float(r["a"]), lambda r: 1),           # float keys
        (lambda r: r[0], lambda r: 1),                    # not a member name
        (lambda r: r['a"b'], lambda r: 1),                # names the device does not match by their bytes
        (lambda r: r["a\\b"], lambda r: 1),
        (lambda r: r["é"], lambda r: 1),
        (lambda r: r["x" * 65], lambda r: 1),
        (lambda r: r["a"], lambda r: str(r["b"])),
        (lambda r: r["a"], lambda r: r["b"] + 1),
    ]:
        assert lowering.json_fields_spec(*args) is None, args


def test_predicate_matcher():
    from dampr_b200 import lowering
    from dampr_b200.lowering import FIELD_STR as S, FIELD_INT as I, FIELD_FLOAT as F, FIELD_MEMBER as M
    allowed = {"GET", "POST"}
    cases = [
        (lambda r: "m" in r, (M, "m", "in", ())),
        (lambda r: "m" not in r, (M, "m", "not in", ())),
        (lambda r: r["s"] >= 500, (I, "s", ">=", (500,))),
        (lambda r: 500 > r["s"], (I, "s", "<", (500,))),
        (lambda r: r["m"] == "GET", (S, "m", "==", ("GET",))),
        (lambda r: r["m"] in ("GET", "POST"), (S, "m", "in", ("GET", "POST"))),
        (lambda r: r["m"] not in [1, 2], (I, "m", "not in", (1, 2))),
        (lambda r: int(r["s"]) != 404, (I, "s", "!=", (404,))),
        (lambda r: float(r["l"]) < 0.5, (F, "l", "<", (0.5,))),
        (lambda r: float(r["l"]) <= 2, (F, "l", "<=", (2.0,))),
        (lambda r: r["m"] in allowed, (S, "m", "in", tuple(allowed))),
    ]
    for fn, exp in cases:
        assert lowering.json_predicate(fn) == exp, exp
    for fn in [lambda r: r["l"] < 0.5,                 # a bare member against a float
               lambda r: r["m"] in ("a", 1),           # mixed constants
               lambda r: r["m"] == True,               # noqa: E712  a bool
               lambda r: r["m"] is None,
               lambda r: int(r["s"]) == "a",
               lambda r: float(r["l"]) in (1.0, 2.0),
               lambda r: len(r) == 3,
               lambda r: r.get("m") == "a",
               lambda r: r["a"]["b"] == 1,
               lambda r: "m" in r["a"],
               lambda r: "m\\" in r,
               lambda l: "m" in l.split(",")[0],
               lambda r: r["a"] == "x" and r["b"] == "y"]:
        assert lowering.json_predicate(fn) is None


def test_mapper_matcher():
    from dampr_b200 import lowering
    assert lowering.is_json_loads(json.loads) and lowering.is_json_loads(lambda l: json.loads(l))
    for fn in [json.dumps, lambda l: json.loads(l.strip()), lambda l: json.loads(l)["a"], lambda l, x=1: l, len]:
        assert not lowering.is_json_loads(fn), fn


def _match(pm):
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    return plan._match_json_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]])


def test_stage_matcher_and_the_binding(tmp_path):
    from dampr_b200 import Dampr, device as dev
    P = write_files(tmp_path, [["f.jsonl", '{"a": "x", "b": 1}\n']])
    t = Dampr.json(P)
    m = _match(t.filter(lambda r: "c" in r).filter(lambda r: r["a"] != "y").a_group_by(lambda r: r["a"],
                                                                                       lambda r: r["b"]).sum())
    src, spec, op, mean, preds, members, bare = m
    assert spec == (dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1) and op == dev.OP_SUM_I64 and not mean
    assert members == ("a", "b", "c") and bare == (True, True)
    assert preds == ((dev.PRED_MEMBER, 2, dev.CMP_IN, ()), (dev.PRED_STR, 0, dev.CMP_NE, ("y",)))
    m = _match(t.mean(lambda r: int(r["k"]), lambda r: float(r["v"])))
    assert m[1] == (dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_INT, 1) and m[2] == dev.OP_SUM_F64 and m[3]
    assert m[6] == (False, False)
    assert _match(t.count(lambda r: r["a"]))[1][3] == dev.FIELD_VAL_ONE
    for pm in [
        Dampr.text(P).map(json.dumps).count(lambda r: r["a"]),
        Dampr.text(P).filter(lambda l: "x" in l).map(json.loads).count(lambda r: r["a"]),   # a raw-line filter
        t.map(lambda r: r).count(lambda r: r["a"]),
        t.count(lambda r: r.get("a")),
        t.a_group_by(lambda r: r["a"], lambda r: r["b"]).reduce(lambda a, b: a * b),
    ]:
        assert _match(pm) is None
    s = dev.fields_spec((dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64), False,
                        [(dev.PRED_MEMBER, 2, dev.CMP_NOT_IN, ())])
    assert s.sep == 257 and s.npreds == 1 and s.preds[0].n == 0
    m = dev.json_members(["a", "", "bc"])
    assert m.n == 3 and m.bytes == b"abc" and [m.len[i] for i in range(3)] == [1, 0, 2]


def test_nine_members_stay_on_the_host(tmp_path):
    from dampr_b200 import Dampr
    P = write_files(tmp_path, [["f.jsonl", '{"a": "x"}\n']])
    pm = Dampr.json(P)
    for n in ["m%d" % i for i in range(8)]:
        pm = pm.filter(eval("lambda r: %r in r" % n))
    assert _match(pm.count(lambda r: r["m0"])) is not None
    assert _match(pm.filter(lambda r: "m8" in r).count(lambda r: r["m0"])) is None


# ---- the stand-in's line rules ----------------------------------------------------------------------------------
@pytest.mark.parametrize("line,takes", [
    (b'{"a": 1}', True), (b' {"a":"x" , "b" :[1,{"c":null}]}\t', True), (b"{}", True),
    (b'{"a": 1', False), (b'{"a": 1}}', False), (b'{"a": 1} x', False), (b'[1, 2]', False), (b'"a"', False),
    (b"", False), (b'{"a": 01}', False), (b'{"a": 1.}', False), (b'{"a": .5}', False), (b'{"a": +1}', False),
    (b'{"a": NaN}', False), (b'{"a": -Infinity}', False), (b'{"a": tru}', False), (b'{"a": "\\x"}', False),
    (b'{"a": "\t"}', False), (b'{"\\u0061": 1}', False), (b'{"a": [1,]}', False), (b'{"a" 1}', False),
    (b'{"a": 1,}', False), (b'{"a": "\xc3\xa9"}', False), (b'{"a": 1}\r', False),
    (b'{"a": ' + b"[" * 63 + b"]" * 63 + b"}", True), (b'{"a": ' + b"[" * 64 + b"]" * 64 + b"}", False),
])
def test_the_standin_reads_lines_as_the_header_says(line, takes):
    assert (device_members(line) is not None) == takes, line


def test_the_standin_keeps_the_last_top_level_member():
    m = device_members(b'{"a": {"k": "in"}, "k": "x", "b": "y\\n", "k": 12, "c": 1e3}')
    assert m["k"] == ("int", "12", 46) and m["b"][0] == "esc" and m["c"][0] == "float" and m["a"][0] == "other"
    assert device_members(b'{"a":\r1}', cr_is_data=True) == {"a": ("int", "1", 6)}


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_json_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = ours(src, P, monkeypatch)
        same_up_to_rounding(got, e)
        assert NEEDLE in hows[0] and "sep=json" in stages[0][2], (name, src, hows)


def test_mixed_kinds_go_to_the_host(monkeypatch, tmp_path):
    """str and int keys, or int and float values, of one bare member: the host map's (the reference cannot sort such
    keys, so plain Python is the yardstick)"""
    rows = [json.dumps({"tag": t, "v": v}) for t, v in zip(["a", 1, "b", 2, "a"] * 20, [1, 2.5, 3, 4.0, 5] * 20)]
    P = write_files(tmp_path, [["m.jsonl", "\n".join(rows) + "\n"]])
    # behind the filter only str tags and int values remain: the int tags are host lines the host's filter drops
    for src, key, val, device in [(J + ".count(lambda r: r['tag'])", "tag", None, False),
                                  (J + ".a_group_by(lambda r: r['tag'], lambda r: r['v']).sum()", "tag", "v", False),
                                  (J + ".filter(lambda r: r['tag'] in ('a', 'b')).a_group_by(lambda r: r['tag'], "
                                       "lambda r: r['v']).sum()", "tag", "v", True)]:
        exp = {}
        for r in map(json.loads, rows):
            if "filter" in src and r["tag"] not in ("a", "b"):
                continue
            v = 1 if val is None else r[val]
            exp[r[key]] = exp[r[key]] + v if r[key] in exp else v
        got, hows, _stages = ours(src, P, monkeypatch)
        assert got == sorted(repr(x) for x in exp.items()) and (NEEDLE in hows[0]) == device, (src, hows)


def test_kind_retries_on_the_standin(monkeypatch, tmp_path):
    """int keys and float values read bare: the scan is repeated once with the other kind"""
    P = write_files(tmp_path, [["f.jsonl", "".join('{"k": %d, "v": %r}\n' % (i % 5, i / 4.0) for i in range(100))]])
    got, hows, stages = ours(J + ".a_group_by(lambda r: r['k'], lambda r: r['v']).sum()", P, monkeypatch)
    exp = {}
    for i in range(100):
        exp[i % 5] = exp.get(i % 5, 0) + i / 4.0
    assert got == sorted(repr(x) for x in exp.items())
    assert NEEDLE in hows[0] and "op=sum_f64" in stages[0][2] and "host_lines=0" in stages[0][2], stages


def test_host_lines_with_another_type_send_the_stage_to_the_host(monkeypatch, tmp_path):
    """a bare value that is a str on a line the predicates leave to the host: Python folds it, so must the stage"""
    rows = ['{"k": "a", "s": 500, "v": 1}', '{"k": "b", "s": "500", "v": "x"}', '{"k": "a", "s": 501, "v": 2}']
    P = write_files(tmp_path, [["f.jsonl", "\n".join(rows) + "\n"]])
    src = J + ".filter(lambda r: int(r['s']) >= 500).a_group_by(lambda r: r['k'], lambda r: r['v']).sum()"
    got, hows, _stages = ours(src, P, monkeypatch)
    assert got == ["('a', 3)", "('b', 'x')"] and NEEDLE not in hows[0]


def test_details_and_host_lines(monkeypatch, tmp_path):
    rows = ['{"k": "a", "v": 1}', '{"k": "a\\u0062", "v": 2}', '{"k": "é", "v": 3}', '{"k": "a", "v": 4}',
            '{"k": "b", "v": 5, "k": "c"}', '{"k": "long-key-of-many-bytes", "v": 6}']
    P = write_files(tmp_path, [["f.jsonl", "\n".join(rows) + "\n"]])
    got, hows, stages = ours(J + ".a_group_by(lambda r: r['k'], lambda r: r['v']).sum()", P, monkeypatch)
    assert got == ["('a', 5)", "('ab', 2)", "('c', 5)", "('long-key-of-many-bytes', 6)", "('é', 3)"]
    assert stages[0][2] == "op=sum_i64 bytes=%d lines=6 groups=5 host_lines=2 sep=json" % os.path.getsize(P)


@pytest.mark.parametrize("src,exc,rows", [
    (J + ".count(lambda r: r['a'])", json.JSONDecodeError, ['{"a": "x"}', '{"a": 1,}']),   # json.loads rejects it
    (J + ".count(lambda r: r['a'])", json.JSONDecodeError, ['{"a": "x"}', '', '{"a": "y"}']),   # a blank line
    (J + ".filter(lambda r: 'a' in r).count(lambda r: r['b'])", KeyError, None),            # a missing member
    (J + ".filter(lambda r: 'a' in r).a_group_by(lambda r: r['a'], lambda r: int(r['a'])).sum()", ValueError, None),
    (J + ".filter(lambda r: 'a' in r).filter(lambda r: r['a'] > 1).count(lambda r: r['a'])", TypeError, None),
])
def test_raising_lambdas_raise_as_in_python(src, exc, rows, monkeypatch, tmp_path):
    rows = rows or ['{"a": "x", "b": 1}', '{"a": "y"}', '{"c": 1}', '{"a": "x", "b": 2}', '{"a": 1,}']
    P = write_files(tmp_path, [["f.jsonl", "\n".join(rows) + "\n"]])
    with pytest.raises(exc):
        ours(src, P, monkeypatch)

"""JSON-lines field folds over member paths (`Dampr.json(path)` with r["actor"]["login"] keys, r["payload"]["size"]
values and filters on paths up to four names deep): the matchers (lowering.json_fields_path_spec,
lowering.json_path_filter_program, plan._match_json_fields(paths=True)) and the binding's packing, the stand-in of
tests/fields_json_path_standin.py against CPython on an adversarial line set and a fuzzed nested corpus, and the
planner on the stand-in against the REAL reference (Refefer/Dampr), whose outputs are stored in
tests/golden/text_fields_json_paths.json.gz (DAMPR_REFERENCE=<checkout> records them again). Pipelines that raise are
checked against plain Python: the reference hangs when one of its workers raises (SURVEY B6). The same pipelines run
on the device in tests/test_gpu_text_fields_json_paths.py."""
import json
import os
import random

import pytest

from fields_json_path_standin import BAD, device_paths, make_json_path_ctx
from fields_standin import reference_outputs, write_files
from test_text_fields_where_lowering import same_up_to_rounding

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields_json_paths.json.gz")
NEEDLE = "device text fields scan+combine"


def ours(src, P, monkeypatch):
    """run_ours on the stand-in that takes JSON paths"""
    from fake_device import FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: make_json_path_ctx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P, "json": json}).run())
    return got, [h for _s, h, _d in runner_mod.LAST_STATS.stages], runner_mod.LAST_STATS.stages


# ---- inputs: GitHub Archive-shaped events -----------------------------------------------------------------------
TYPES = ["PushEvent", "WatchEvent", "IssuesEvent", "ForkEvent"]


def gh_event(rng, i):
    """one event: actor / repo / payload objects, a depth-3 float (a multiple of 1/8: sums are exact in any order)
    and decoy members named like the wanted ones at other depths"""
    return {"id": i, "type": rng.choice(TYPES),
            "actor": {"id": rng.randrange(-5, 30), "login": "user%d" % rng.randrange(25), "login_decoy": "x"},
            "repo": {"id": rng.randrange(100), "name": rng.choice(["org/a", "org/b", "me/c", "you/d-%d" % (i % 4)])},
            "payload": {"size": rng.randrange(0, 9), "push": {"commits": {"n": 1}} if rng.random() < 0.6 else {},
                        "stats": {"ratio": rng.randrange(-16, 64) / 8.0, "login": "decoy"}},
            "meta": {"actor": {"login": "decoy"}, "size": -1}, "login": "top-decoy"}


def gh_text(n, seed, cr=False):
    """events the device takes and valid lines it hands back, none of which makes a golden pipeline raise: non-ASCII
    values, an escaped wanted name, escaped names in decoy subtrees (the device takes those), duplicate interior
    objects that carry every wanted member, a 65-deep decoy, an escaped key value, odd whitespace. cr: '\\r' between tokens"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        e = gh_event(rng, i)
        r = rng.random()
        line = None
        if r < 0.03:
            e["actor"]["login"] = "ü%d" % (i % 3)
        elif r < 0.06:
            line = json.dumps(e).replace('"login": "user', '"\\u006cogin": "user', 1)   # a wanted name, escaped
        elif r < 0.10:
            line = json.dumps(e)[:-1] + ', "meta": {"\\u0061ctor": 1}}'              # an escape in a decoy
        elif r < 0.14:
            dup = dict(e["actor"], login="dup%d" % (i % 5))
            line = json.dumps(e)[:-1] + ', "actor": %s}' % json.dumps(dup)          # the last actor wins
        elif r < 0.16:
            e["meta"] = json.loads("[" * 64 + "]" * 64)                             # nesting 65 deep
        elif r < 0.18:
            line = json.dumps(e).replace('"login": "user', '"login": "\\u0075ser', 1)   # an escaped key value
        if line is None:
            line = json.dumps(e, separators=rng.choice([(",", ":"), (", ", ": "), (" ,\t", " :  ")]))
        if cr and i % 7 == 3:
            line = line.replace(",", "\r,", 2)
        rows.append(rng.choice(["", " "]) + line + rng.choice(["", "\t"]))
    return "".join(r + "\n" for r in rows)


def datasets():
    ev = gh_text(110, 3)
    ev_cr = gh_text(60, 5, cr=True)
    cut = ev.index("\n", len(ev) // 3) + 1
    return {
        "events": [["events.jsonl", ev]],
        "events_gz": [["events.jsonl.gz", ev_cr]],
        "crlf_text": [["events.jsonl", ev.replace("\n", "\r\n")]],
        "several": [["a.jsonl", ev[:cut]], ["b.jsonl.gz", ev_cr], ["c.jsonl", ev[cut:]]],
    }


J = "Dampr.json(P)"
EVENTS = [
    J + ".filter(lambda r: r['type'] == 'PushEvent').count(lambda r: r['repo']['name'])",
    J + ".a_group_by(lambda r: r['actor']['login'], lambda r: r['payload']['size']).sum()",
    J + ".mean(lambda r: r['type'], lambda r: float(r['payload']['stats']['ratio']))",
    J + ".a_group_by(lambda r: int(r['actor']['id']), lambda r: r['payload']['size']).reduce(max)",
    J + ".filter(lambda r: r['payload']['size'] >= 2 and not r['type'] == 'WatchEvent')"
        ".count(lambda r: r['actor']['login'])",
    J + ".filter(lambda r: 'commits' in r['payload']['push']).a_group_by(lambda r: r['repo']['name'], "
        "lambda r: r['payload']['size']).reduce(min)",
    J + ".filter(lambda r: 'size' in r['payload']).count(lambda r: r['repo']['name'])",
    J + ".filter(lambda r: r['actor']['login'].startswith('user1') or r['repo']['id'] < 10)"
        ".a_group_by(lambda r: r['type'], lambda r: float(r['payload']['stats']['ratio'])).sum()",
]
PIPELINES = {
    "events": EVENTS,
    "events_gz": EVENTS,
    "crlf_text": EVENTS[:4],
    "several": EVENTS[:3],
}


# ---- the adversarial line set -----------------------------------------------------------------------------------
NAMES = ("a", "b", "c", "d")


def _nest(names, inner):
    """'{"n1": {"n2": .. {inner}}}' as text"""
    out = "{%s}" % inner
    for n in reversed(names):
        out = '{"%s": %s}' % (n, out)
    return out


def adversarial(depth):
    """lines against the key path NAMES[:depth] and the value path NAMES[:depth - 1] + ("v",): [(label, line)]"""
    kp = NAMES[:depth]
    up, leaf = kp[:-1], kp[-1]
    good = '"%s": "x", "v": 1' % leaf
    out = [("ok", _nest(up, good)), ("ok spaced", " " + _nest(up, ' "v" : 2 , "%s" : "y" ' % leaf) + "\t")]
    for i in range(1, depth):   # level i: the object of up[:i] holds up[i - 1]
        pre, rest = up[:i - 1], up[i - 1:]
        body = _nest(rest[1:], good)
        for what, val in [("str", '"s"'), ("list", "[1, {\"b\": 1}]"), ("number", "5"), ("null", "null"),
                          ("true", "true")]:
            out.append(("parent %d is %s" % (i, what), _nest(pre, '"%s": %s' % (rest[0], val))))
        out.append(("parent %d missing" % i, _nest(pre, '"zz": %s' % body)))
        out.append(("dup parent %d replaced by an object" % i, _nest(pre, '"%s": %s, "%s": {"q": 1}' % (rest[0], body,
                                                                                                       rest[0]))))
        out.append(("dup parent %d replaced by a scalar" % i, _nest(pre, '"%s": %s, "%s": 7' % (rest[0], body,
                                                                                               rest[0]))))
        out.append(("dup parent %d replaced by a full one" % i,
                    _nest(pre, '"%s": {"q": 1}, "%s": %s' % (rest[0], rest[0], body))))
        out.append(("escaped parent %d" % i, _nest(pre, '"\\u00%02x%s": %s' % (ord(rest[0][0]), rest[0][1:], body))))
        out.append(("escape in a decoy next to parent %d" % i,
                    _nest(pre, '"%s": %s, "dec": {"\\u0062": {"\\u0061": 1}}' % (rest[0], body))))
    out.append(("dup leaf", _nest(up, '"%s": "x1", "v": 1, "%s": "x2", "v": 3' % (leaf, leaf))))
    out.append(("leaf is an object", _nest(up, '"%s": {"x": 1}, "v": 1' % leaf)))
    out.append(("leaf is a number", _nest(up, '"%s": 12, "v": 1' % leaf)))
    out.append(("escaped leaf", _nest(up, '"\\u00%02x": "x", "v": 1' % ord(leaf))))
    out.append(("escaped leaf value", _nest(up, '"%s": "x\\n", "v": 1' % leaf)))
    out.append(("leaf too deep", _nest(up, '"q": {"%s": "x"}, "v": 1' % leaf)))
    out.append(("leaf too shallow", '{"%s": "x", "v": 1, %s' % (leaf, _nest(up, '"v": 1')[1:])))
    out.append(("value is a float", _nest(up, '"%s": "x", "v": 1.5' % leaf)))
    out.append(("value missing", _nest(up, '"%s": "x"' % leaf)))
    for deep in (64 - depth, 65 - depth):   # a decoy whose nesting puts the line at depth 64, then 65
        out.append(("decoy %d deep" % (deep + depth),
                    _nest(up, good + ', "deep": ' + "[" * deep + "]" * deep)))
    out.append(("key and value in a 64-deep line", _nest(up, good + ', "deep": ' + "[" * (64 - depth) + "1" +
                                                         "]" * (64 - depth))))
    return out


def python_read(r, path):
    """r[n1]..[nk] in Python: its value, or the exception type"""
    try:
        for n in path:
            r = r[n]
        return r
    except Exception as e:   # noqa: BLE001  the exception is the result under test
        return type(e)


def _kind_of(v):
    if isinstance(v, bool) or v is None or isinstance(v, (dict, list)):
        return "other"
    return {str: ("str", "esc"), int: ("int",), float: ("float",)}[type(v)]


def check_reading(line, paths, cr_is_data=False):
    """the stand-in's reading of one line against CPython's dict; returns whether the device takes the line"""
    got = device_paths(line.encode("ascii") if isinstance(line, str) else line, paths, cr_is_data)
    if got is None:
        return False
    leaves, nodes = got
    r = json.loads(line)
    for p, (present, is_obj) in nodes.items():
        v = python_read(r, p)
        assert present == (v is not KeyError and v is not TypeError) and is_obj == isinstance(v, dict), (line, p)
    for p, leaf in leaves.items():
        v = python_read(r, p)
        above_objects = all(isinstance(python_read(r, p[:i]), dict) for i in range(1, len(p)))
        if leaf is BAD:
            assert not above_objects and v in (KeyError, TypeError), (line, p)
        elif leaf is None:
            assert above_objects and v is KeyError, (line, p)
        else:
            kind, raw, off = leaf
            assert above_objects and kind in _kind_of(v), (line, p, leaf)
            text = line if isinstance(line, str) else line.decode("ascii")
            if kind in ("str", "esc"):
                assert json.loads('"%s"' % raw) == v and text[off:off + len(raw)] == raw, (line, p)
            elif kind != "other":
                assert json.loads(raw) == v and text[off:off + len(raw)] == raw, (line, p)
        # "m" in r[n1]..[nk]: the device decides it where r[n1]..[nk] is an object
        if len(p) > 1:
            host = python_read(r, p[:-1])
            assert (leaf is BAD) == (not isinstance(host, dict)), (line, p)
    return True


@pytest.mark.parametrize("depth", [2, 3, 4])
def test_the_standin_reads_the_adversarial_set_as_cpython(depth):
    kp = NAMES[:depth]
    paths = [kp, kp[:-1] + ("v",)]
    taken = {}
    for label, line in adversarial(depth):
        taken[label] = check_reading(line, paths)
    assert taken["ok"] and taken["ok spaced"] and taken["dup leaf"]
    assert not taken["escaped leaf"] and taken["escaped leaf value"]
    assert taken["decoy %d deep" % 64] and not taken["decoy %d deep" % 65]
    for i in range(1, depth):
        assert not taken["escaped parent %d" % i] and taken["escape in a decoy next to parent %d" % i]
        assert taken["dup parent %d replaced by a scalar" % i] and taken["parent %d is list" % i]
    leaves = device_paths(_nest(kp[:-1], '"%s": "x", "v": 1' % kp[-1]).encode(), paths)[0]
    assert leaves[kp] == ("str", "x", leaves[kp][2])


def test_the_standin_follows_every_occurrence_of_an_interior_name():
    """an escape in an earlier, replaced occurrence of a wanted object still hands the line back (the device compares
    names in every occurrence); one in a leaf's object value does not (it is not searched)"""
    assert device_paths(b'{"a": {"\\u0062": 1}, "a": {"b": 2}}', [("a", "b")]) is None
    assert device_paths(b'{"a": {"b": {"\\u0063": 1}}}', [("a", "b")]) is not None
    leaves, nodes = device_paths(b'{"a": {"b": 1}, "a": {"c": 2}}', [("a", "b"), ("a", "c")])
    assert leaves == {("a", "b"): None, ("a", "c"): ("int", "2", 27)} and nodes == {("a",): (True, True)}
    leaves, _ = device_paths(b'{"a": {"b": 1}, "a": 5}', [("a", "b"), ("a",)])
    assert leaves[("a", "b")] is BAD and leaves[("a",)] == ("int", "5", 21)


def fuzz_line(rng, depth=0):
    """a random JSON object text whose names come from a small alphabet, so wanted paths, duplicates, non-object
    parents and escaped spellings all occur"""
    parts = []
    for _ in range(rng.randrange(0, 5)):
        name = rng.choice(NAMES + ("v", "q"))
        qn = json.dumps(name) if rng.random() < 0.93 else '"\\u00%02x"' % ord(name)
        r = rng.random()
        if r < 0.4 and depth < 5:
            val = fuzz_line(rng, depth + 1)
        elif r < 0.55:
            val = json.dumps("x%d" % rng.randrange(5)) if rng.random() < 0.9 else '"e\\n"'
        elif r < 0.75:
            val = str(rng.randrange(-50, 50))
        elif r < 0.85:
            val = rng.choice(["1.5", "-0", "1e3", "null", "true", "[]", "[{}]"])
        else:
            val = "[" * 62 + "]" * 62 if rng.random() < 0.1 else '"s"'
        parts.append(qn + rng.choice([":", ": ", " : "]) + val)
    return "{" + rng.choice([",", ", "]).join(parts) + "}"


def test_the_standin_is_sound_on_a_fuzzed_nested_corpus():
    rng = random.Random(2024)
    taken = 0
    path_sets = [[("a", "b"), ("a", "v")], [("a", "b", "c"), ("a", "b", "v"), ("a",)],
                 [("a", "b", "c", "d"), ("a", "b", "c", "v"), ("q", "v"), ("a", "b")], [("b",), ("a", "a", "a")]]
    for i in range(6000):
        line = fuzz_line(rng)
        taken += check_reading(line, path_sets[i % len(path_sets)])
    assert taken > 2000


# ---- the matchers -----------------------------------------------------------------------------------------------
def test_spec_matcher_accepts_paths():
    from dampr_b200 import lowering
    from dampr_b200.lowering import FIELD_DATA as D, FIELD_INT as I, FIELD_FLOAT as F

    def mv(value):
        return lambda v: (value(v), 1)
    cases = [
        ((lambda r: r["a"]["b"], lambda r: 1), (("a", "b"), D, None, I, False)),
        ((lambda r: r["actor"]["login"], lambda r: r["payload"]["size"]), (("actor", "login"), D, ("payload", "size"),
                                                                          D, False)),
        ((lambda r: int(r["a"]["b"]["c"]["d"]), lambda r: float(r["v"])), (("a", "b", "c", "d"), I, ("v",), F, False)),
        ((lambda r: r["k"], mv(lambda r: float(r["s"]["x"]["y"]))), (("k",), D, ("s", "x", "y"), F, True)),
        ((lambda r: r["a"]["x y"], lambda r: int(r["a"]["b"])), (("a", "x y"), D, ("a", "b"), I, False)),
    ]
    for args, exp in cases:
        assert lowering.json_fields_path_spec(*args) == exp, (args, exp)
        assert lowering.json_fields_spec(*args) is None


def test_spec_matcher_refuses_other_paths():
    from dampr_b200 import lowering
    for args in [
        (lambda r: r["a"], lambda r: r["b"]),                    # no path: json_fields_spec's
        (lambda r: r["a"]["b"]["c"]["d"]["e"], lambda r: 1),     # a fifth name
        (lambda r: r["a"][0], lambda r: 1),                      # an array index
        (lambda r: r["a"][0]["b"], lambda r: 1),
        (lambda r: r.get("a")["b"], lambda r: 1),
        (lambda r: r["a"].get("b"), lambda r: 1),
        (lambda r: r["a"][""], lambda r: 1),                     # an empty name inside a path
        (lambda r: r["a"]['b"'], lambda r: 1),                   # names the device cannot match
        (lambda r: r["a\\"]["b"], lambda r: 1),
        (lambda r: r["a"]["é"], lambda r: 1),
        (lambda r: r["a"]["x" * 65], lambda r: 1),
        (lambda r: float(r["a"]["b"]), lambda r: 1),             # float keys
        (lambda r: (r["a"]["b"], r["c"]), lambda r: 1),          # tuple keys
        (lambda r: r["a"]["b"], lambda r: r["c"]["d"] + 1),      # expressions
        (lambda r: r["a"]["b"], lambda r: str(r["c"]["d"])),
    ]:
        assert lowering.json_fields_path_spec(*args) is None, args


def test_filter_matcher_takes_paths():
    from dampr_b200 import lowering
    from dampr_b200.lowering import FIELD_STR as S, FIELD_INT as I, FIELD_FLOAT as F, FIELD_MEMBER as M, \
        FIELD_LEN as L
    cases = [
        (lambda r: r["a"]["b"] == 1, [(I, ("a", "b"), "==", (1,))]),
        (lambda r: 5 > int(r["a"]["b"]["c"]), [(I, ("a", "b", "c"), "<", (5,))]),
        (lambda r: float(r["a"]["b"]) <= 2, [(F, ("a", "b"), "<=", (2.0,))]),
        (lambda r: r["a"]["b"] in ("x", "y"), [(S, ("a", "b"), "in", ("x", "y"))]),
        (lambda r: "m" in r["a"]["b"], [(M, ("a", "b", "m"), "in", ("m",))]),
        (lambda r: "m" not in r["a"]["b"]["c"], [(M, ("a", "b", "c", "m"), "not in", ("m",))]),
        (lambda r: "m" in r["a"], [(M, ("a", "m"), "in", ("m",))]),   # membership or substring, by r["a"]'s type
        (lambda r: r["a"]["b"].endswith(("x", "y")), [(S, ("a", "b"), "endswith", ("x", "y"))]),
        (lambda r: len(r["a"]["b"]) > 3, [(L, ("a", "b"), ">", (3,))]),
        (lambda r: r["t"] == "P" and not r["a"]["b"] >= 2 or "m" in r,
         [(S, ("t",), "==", ("P",)), (I, ("a", "b"), ">=", (2,)), "not", "and", (M, ("m",), "in", ()), "or"]),
        (lambda r: "x" in r["s"] and r["a"]["b"] == 1,
         [(M, ("s", "x"), "in", ("x",)), (I, ("a", "b"), "==", (1,)), "and"]),
        (lambda r: "é" in r["s"] and r["a"]["b"] == 1,           # no member named "é": the substring test alone
         [("str", ("s",), "contains", ("é",)), (I, ("a", "b"), "==", (1,)), "and"]),
    ]
    for fn, exp in cases:
        assert lowering.json_path_filter_program(fn) == exp, exp
    for fn in [lambda r: r["a"] == 1,                            # no path: json_filter_program's
               lambda r: "é" in r["a"],
               lambda r: "m" in r["a"]["b"]["c"]["d"],            # a fifth name
               lambda r: "" in r["a"]["b"],
               lambda r: r["a"][0] == 1,
               lambda r: r.get("a")["b"] == 1,
               lambda r: r["a"]["b"]["c"]["d"]["e"] == 1,
               lambda r: r["a"]["b"] == 1.5,                     # a bare member against a float
               lambda r: r["a"]["b"] + 1 == 2]:
        assert lowering.json_path_filter_program(fn) is None


def test_the_old_matchers_still_refuse_paths():
    from dampr_b200 import lowering
    assert lowering.json_fields_spec(lambda r: r["a"]["b"], lambda r: 1) is None
    assert lowering.json_predicate(lambda r: r["a"]["b"] == 1) is None
    assert lowering.json_predicate(lambda r: "m" in r["a"]) is None
    assert lowering.json_filter_program(lambda r: "x" in r["a"]["b"]) is None


def _match(pm, **kw):
    from dampr_b200 import plan
    from dampr_b200.graph import GMap
    st = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
    return plan._match_json_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]], **kw)


def test_stage_matcher_and_the_binding(tmp_path):
    from dampr_b200 import Dampr, device as dev
    P = write_files(tmp_path, [["f.jsonl", '{"a": {"b": "x"}, "c": 1}\n']])
    t = Dampr.json(P)
    pm = t.filter(lambda r: "m" in r["a"]["b"]).filter(lambda r: r["c"] != 2 and r["a"]["b"] == "y") \
        .a_group_by(lambda r: r["a"]["b"], lambda r: r["c"]).sum()
    assert _match(pm) is None and _match(pm, programs=True) is None   # the defaults: what they matched before
    src, spec, op, mean, preds, members, bare = _match(pm, programs=True, paths=True)
    assert spec == (dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1) and op == dev.OP_SUM_I64 and not mean
    assert members == (("a", "b"), "c", ("a", "b", "m")) and bare == (True, True)   # de-duplicated by path
    assert preds == ((dev.PRED_MEMBER, 2, dev.CMP_IN, ("m",)), (dev.PRED_INT, 1, dev.CMP_NE, (2,)),
                     (dev.PRED_STR, 0, dev.CMP_EQ, ("y",)), (dev.PRED_AND, 0, dev.CMP_EQ, ()))
    # a top-level stage matches as before, names and all, "x" in r["a"] a substring test on the top-level build
    for top in [t.filter(lambda r: "c" in r).a_group_by(lambda r: r["a"], lambda r: r["c"]).sum(),
                t.filter(lambda r: "x" in r["a"]).count(lambda r: r["c"])]:
        assert _match(top, programs=True, paths=True) == _match(top, programs=True) is not None
    # in a stage that reads a path, "x" in r["s"] is the member test of ("s", "x") that also lists its container
    m = _match(t.filter(lambda r: "x" in r["s"]).count(lambda r: r["a"]["b"]), programs=True, paths=True)
    assert m[5] == (("a", "b"), ("s", "x"), "s") and m[4] == ((dev.PRED_MEMBER, 1, dev.CMP_IN, ("x",)),)
    # 17 path nodes do not fit
    wide = t
    for n in ["p%d" % i for i in range(7)]:
        wide = wide.filter(eval("lambda r: r[%r]['x']['y'] == 1" % n))
    assert _match(wide.count(lambda r: r["a"]["b"]), programs=True, paths=True) is None
    assert _match(t.filter(lambda r: r["p"]["x"]["y"] == 1).count(lambda r: r["a"]["b"]), paths=True) is not None
    s = dev.fields_spec((dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64), False,
                        [(dev.PRED_MEMBER, 2, dev.CMP_IN, ("xy",))])
    assert s.preds[0].n == 1 and s.preds[0].lens[0] == 2 and bytes(s.preds[0].bytes[:2]) == b"xy"
    m = dev.json_members([("a", "b"), "", ("c", "d", "e", "f"), ("g",)])
    assert m.n == 4 and m.bytes == b"a\x1fbc\x1fd\x1fe\x1ffg" and [m.len[i] for i in range(4)] == [3, 0, 7, 1]


# ---- against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_path_folds_agree_with_the_reference(name, monkeypatch, tmp_path):
    files = datasets()[name]
    exp = reference_outputs(files, PIPELINES[name], GOLDEN)
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows, stages = ours(src, P, monkeypatch)
        same_up_to_rounding(got, e)
        took_lines(hows[0], stages[0][2], name != "crlf_text")


def took_lines(how, detail, some=True):
    """the stage ran the path scan and (some) the device took at least one line; a text-mode file whose lines end in
    '\r\n' has none to take: '\r' ends a line in text mode, so every line is the host's"""
    assert NEEDLE in how and "sep=json path=" in detail, (how, detail)
    stats = dict(x.split("=", 1) for x in detail.split())
    assert (int(stats["host_lines"]) < int(stats["lines"])) == some, detail


def test_membership_of_an_object_or_a_str_member(monkeypatch, tmp_path):
    """"m" in r["p"]: membership where r["p"] is an object, the substring test where it is a str, both on the device;
    a list, a number, null, a missing r["p"] or an escaped str are the host's (Python raises on the scalars)"""
    rows = ['{"k": {"n": "a"}, "p": {"size": 1}}', '{"k": {"n": "a"}, "p": {"other": 1}}',
            '{"k": {"n": "b"}, "p": "the size"}', '{"k": {"n": "b"}, "p": "none"}',
            '{"k": {"n": "c"}, "p": ["size"]}', '{"k": {"n": "c"}, "p": "s\\u0069ze"}']
    P = write_files(tmp_path, [["f.jsonl", "\n".join(rows * 3) + "\n"]])
    # the host folds the list and escaped-str lines Python keeps: all 6 under `in`, none under `not in`
    for src, exp, host in [(J + ".filter(lambda r: 'size' in r['p']).count(lambda r: r['k']['n'])",
                            ["('a', 3)", "('b', 3)", "('c', 6)"], 6),
                           (J + ".filter(lambda r: 'size' not in r['p']).count(lambda r: r['k']['n'])",
                            ["('a', 3)", "('b', 3)"], 0)]:
        got, hows, stages = ours(src, P, monkeypatch)
        assert got == exp, (src, got)
        took_lines(hows[0], stages[0][2])
        assert "lines=%d groups" % (6 + host) in stages[0][2] and "host_lines=%d filtered=6" % host in stages[0][2], \
            stages
    for bad in ['{"k": {"n": "d"}, "p": 5}', '{"k": {"n": "d"}, "p": null}', '{"k": {"n": "d"}}']:
        P = write_files(tmp_path, [["g.jsonl", rows[0] + "\n" + bad + "\n"]])
        with pytest.raises((TypeError, KeyError)):
            ours(J + ".filter(lambda r: 'size' in r['p']).count(lambda r: r['k']['n'])", P, monkeypatch)


def test_details_and_host_lines(monkeypatch, tmp_path):
    rows = ['{"u": {"id": "a"}, "s": {"n": 1}}', '{"u": {"id": "a"}, "s": {"n": 2}}', '{"u": {"id": "é"}, "s": {"n": 3}}',
            '{"u": {"id": "b"}, "s": {"n": 4}, "u": {"id": "c"}}', '{"u": {"\\u0069d": "d"}, "s": {"n": 5}}']
    P = write_files(tmp_path, [["f.jsonl", "\n".join(rows) + "\n"]])
    got, hows, stages = ours(J + ".a_group_by(lambda r: r['u']['id'], lambda r: r['s']['n']).sum()", P, monkeypatch)
    assert got == ["('a', 3)", "('c', 4)", "('d', 5)", "('é', 3)"]
    assert stages[0][2] == "op=sum_i64 bytes=%d lines=5 groups=4 host_lines=2 sep=json path=u.id" % os.path.getsize(P)


def test_kind_retry_of_bare_nested_members(monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.jsonl", "".join('{"m": {"k": %d}, "s": {"x": {"v": %r}}}\n' % (i % 5, i / 4.0)
                                                   for i in range(100))]])
    got, hows, stages = ours(J + ".a_group_by(lambda r: r['m']['k'], lambda r: r['s']['x']['v']).sum()", P,
                             monkeypatch)
    exp = {}
    for i in range(100):
        exp[i % 5] = exp.get(i % 5, 0) + i / 4.0
    assert got == sorted(repr(x) for x in exp.items())
    assert NEEDLE in hows[0] and "op=sum_f64" in stages[0][2] and "host_lines=0" in stages[0][2], stages


@pytest.mark.parametrize("src,exc,rows", [
    (J + ".count(lambda r: r['a']['b'])", KeyError, ['{"a": {"b": 1}}', '{"a": {"c": 1}}']),
    (J + ".count(lambda r: r['a']['b'])", TypeError, ['{"a": {"b": 1}}', '{"a": {"b": 1}, "a": 5}']),
    (J + ".count(lambda r: r['a']['b'])", TypeError, ['{"a": {"b": 1}}', '{"a": [1]}']),
    (J + ".filter(lambda r: 'b' in r['a']['x']).count(lambda r: r['a']['b'])", TypeError,
     ['{"a": {"b": 1, "x": {"b": 1}}}', '{"a": {"b": 1, "x": 3}}']),
    (J + ".filter(lambda r: r['a']['b'] > 0).count(lambda r: r['c'])", TypeError, ['{"a": {"b": "s"}, "c": 1}']),
])
def test_raising_lambdas_raise_as_in_python(src, exc, rows, monkeypatch, tmp_path):
    P = write_files(tmp_path, [["f.jsonl", "\n".join(rows) + "\n"]])
    with pytest.raises(exc):
        ours(src, P, monkeypatch)


def _sub(path):
    return "".join("[%r]" % n for n in path)


def adversarial_runs(tmp_path):
    """(pipeline, path, expected, where) runs over the adversarial set: per depth, the lines on which Python does not
    raise together behind valid ones (where "device"), each line that gives a bare member another kind alone behind
    them (where "host map": a bare key or value of two kinds is the host map's), then each raising line alone behind
    them (where None). The fold reads the key path and the value path behind a filter on "v" in the value's parent."""
    from fields_standin import python_lines
    out = []
    for depth in (2, 3, 4):
        kp = NAMES[:depth]
        vp = kp[:-1] + ("v",)
        flt = "lambda r: 'v' in r%s" % _sub(kp[:-1])
        key, val = eval("lambda r: r%s" % _sub(kp)), eval("lambda r: r%s" % _sub(vp))
        keep = eval(flt) if flt else (lambda r: True)
        src = J + (".filter(%s)" % flt if flt else "") + \
            ".a_group_by(lambda r: r%s, lambda r: r%s).reduce(max)" % (_sub(kp), _sub(vp))

        def python(P):
            try:
                acc = {}
                for l in python_lines(P):
                    r = json.loads(l)
                    if keep(r):
                        k, v = key(r), val(r)
                        acc[k] = max(acc[k], v) if k in acc else v
                return sorted(repr(x) for x in acc.items())
            except Exception as e:   # noqa: BLE001  the exception is the result under test
                return type(e)

        base = [_nest(kp[:-1], '"%s": "k%d", "v": %d' % (kp[-1], i % 7, i)) for i in range(200)]
        calm, mixed, raising = [], [], []
        for label, line in adversarial(depth):
            if label == "leaf is an object":   # an unhashable key: the host map's concern, not the scan's
                continue
            P = write_files(tmp_path, [["one.jsonl", line + "\n"]])
            (raising if isinstance(python(P), type) else
             mixed if label in ("leaf is a number", "value is a float") else calm).append(line)
        runs = [(calm, "device")] + [([x], "host map") for x in mixed] + [([x], None) for x in raising]
        for i, (extra, where) in enumerate(runs):
            P = write_files(tmp_path, [["adv%d_%d.jsonl" % (depth, i), "\n".join(base + extra) + "\n"]])
            out.append((src, P, python(P), where))
    return out


def test_adversarial_set_end_to_end_on_the_standin(monkeypatch, tmp_path):
    """every adversarial line behind valid ones, through a filtered path fold: Python's result or its exception, on
    the path each run expects"""
    for src, P, exp, where in adversarial_runs(tmp_path):
        try:
            got, hows, stages = ours(src, P, monkeypatch)
        except Exception as e:   # noqa: BLE001  the exception is the result under test
            got, hows, stages = type(e), None, None
        assert got == exp, (src, open(P).read()[-300:], got, exp)
        if where == "device":
            took_lines(hows[0], stages[0][2])
        elif where == "host map":
            assert NEEDLE not in hows[0], (src, stages)

"""JSON-lines field folds over member paths on the device (the path builds of csrc/fields.cu, `Dampr.json(path)` with
r["a"]["b"] keys, values and filters): the library's answers to bad paths, the reference pipelines of
tests/test_text_fields_json_paths_lowering.py, every fold with and without filters on seeded inputs against json.loads
and plain Python, the adversarial line set end to end (Python's result or Python's exception), every path build line
by line against the stand-in of tests/fields_json_path_standin.py and CPython with cr_is_data off and on, the kind
retry of bare nested members, tile seams and the 4 KB window, more host lines than the fallback list holds, a
long-key collision as a nested key, and one scan over poisoned memory. Each end-to-end case asserts that its stage
took the device path and names its longest path in the stats."""
import collections
import json
import operator
import random

import numpy as np
import pytest

import fields_fuzz as fz
from fields_json_path_standin import json_path_line
from fields_standin import python_lines, reference_outputs, write_files
from test_code_collisions import PAIRS
from test_gpu_fields_fuzz import Text, check_build
from test_gpu_poisoned_memory import ab, dirty_table, poison_textbuf
from test_text_fields_json_paths_lowering import GOLDEN, NEEDLE, PIPELINES, adversarial_runs, datasets, took_lines
from test_text_fields_where_lowering import same_up_to_rounding

pytestmark = pytest.mark.gpu


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "ingest_chunk_bytes", settings.ingest_chunk_bytes)
    yield settings
    plan.release_buffers()


def run(src, P):
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P, "json": json}).run())
    return got, runner_mod.LAST_STATS.stages[0]


def on_device(stage):
    """the stage ran the path scan and the device took at least one line"""
    _s, how, detail = stage
    took_lines(how, detail)


def python_fold(P, preds, key, value, binop):
    out = {}
    for l in python_lines(P):
        r = json.loads(l)
        if all(p(r) for p in preds):
            k, v = key(r), value(r)
            out[k] = binop(out[k], v) if k in out else v
    return sorted(repr(x) for x in out.items())


def test_the_library_refuses_bad_paths(ctx):
    from dampr_b200 import device as dev
    data = b'{"a": {"b": "x"}, "c": 2}\n'
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    js = (dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64)
    wide = [("p%d" % i, "x", "y") for i in range(5)] + [("q", "r", "s")]   # 18 nodes
    try:
        for members in [[("a", ""), "c"], [("", "b"), "c"], [("a", "b", "c", "d", "e"), "c"], wide,
                        [("a", "b"), ("a", "b")], [("a", "b"), "c\x1f"], [("a", 'b"'), "c"]]:
            with pytest.raises(dev.DeviceError):
                tab.json_fields(tb, 0, len(data), js, members)
        # a member test's substring constant: one, and only in a call over paths
        for members, preds in [(["a", "c"], [(dev.PRED_MEMBER, 0, dev.CMP_IN, ("x",))]),
                               ([("a", "b"), "c", ("a", "m")], [(dev.PRED_MEMBER, 2, dev.CMP_IN, ("m", "n"))])]:
            with pytest.raises(dev.DeviceError):
                tab.json_fields(tb, 0, len(data), js, members, preds=preds)
        tab.clear()
        tab.json_fields(tb, 0, len(data), js, [("a", "b"), "c"])
        st = tab.fields_stats()
        assert st["lines"] == 1 and st["fallback"] == 0 and st["flags"] == 0, st
        assert tab.fields_fetch(dev.OP_SUM_I64)[1].tolist() == [2]
        tab.clear()   # "x" in r["a"]["b"], a str: the substring test
        tab.json_fields(tb, 0, len(data), js, [("a", "b"), "c", ("a", "b", "x")],
                        preds=[(dev.PRED_MEMBER, 2, dev.CMP_IN, ("x",))])
        st = tab.fields_stats()
        assert st["lines"] == 1 and st["fallback"] == 0, st
    finally:
        tb.free()
        tab.free()


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, stage = run(src, P)
        same_up_to_rounding(got, exp)
        took_lines(stage[1], stage[2], name != "crlf_text")


def event(rng, i):
    return {"user": {"id": "u%03d" % rng.randrange(60), "org": {"team": "t%d" % rng.randrange(6)}},
            "stats": {"n": rng.randrange(-500, 5000), "latency": rng.randrange(0, 64) / 8.0,
                      "deep": {"x": {"ratio": rng.choice([0.5, 1.25, -2.0, 3e-3])}}, "zone": rng.randrange(-3, 4)},
            "meta": {"user": {"id": "decoy"}, "n": 1}, "method": rng.choice(["GET", "POST", "PUT"])}


def events_file(tmp_path, n, seed):
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        e = event(rng, i)
        if i % 97 == 5:
            e["user"]["id"] = "ü%d" % (i % 4)   # non-ASCII: a host line under every fold
        if i % 89 == 7:
            e["stats"]["latency"] = 7          # an int among the floats: float() takes it
        rows.append(json.dumps(e, separators=(",", ":") if i % 3 else (", ", ": "), ensure_ascii=False))
    P = str(tmp_path / "ev.jsonl")
    with open(P, "w", encoding="utf-8") as f:
        f.write("\n".join(rows) + "\n")
    return P


FOLDS = {
    "count": ("count(lambda r: r['user']['id'])", lambda r: r["user"]["id"], lambda r: 1, operator.add),
    "int_sum": ("a_group_by(lambda r: r['user']['org']['team'], lambda r: r['stats']['n']).sum()",
                lambda r: r["user"]["org"]["team"], lambda r: r["stats"]["n"], operator.add),
    "int_min": ("a_group_by(lambda r: r['user']['id'], lambda r: int(r['stats']['n'])).reduce(min)",
                lambda r: r["user"]["id"], lambda r: int(r["stats"]["n"]), min),
    "int_max": ("a_group_by(lambda r: int(r['stats']['zone']), lambda r: r['stats']['n']).reduce(max)",
                lambda r: int(r["stats"]["zone"]), lambda r: r["stats"]["n"], max),
    "float_min": ("a_group_by(lambda r: r['method'], lambda r: float(r['stats']['deep']['x']['ratio'])).reduce(min)",
                  lambda r: r["method"], lambda r: float(r["stats"]["deep"]["x"]["ratio"]), min),
    "float_max": ("a_group_by(lambda r: r['user']['id'], lambda r: float(r['stats']['latency'])).reduce(max)",
                  lambda r: r["user"]["id"], lambda r: float(r["stats"]["latency"]), max),
    "float_sum": ("a_group_by(lambda r: r['user']['id'], lambda r: float(r['stats']['latency'])).sum()",
                  lambda r: r["user"]["id"], lambda r: float(r["stats"]["latency"]), operator.add),
    "mean_int": ("mean(lambda r: r['method'], lambda r: r['stats']['n'])", lambda r: r["method"],
                 lambda r: r["stats"]["n"], None),
    "mean_float": ("mean(lambda r: r['user']['org']['team'], lambda r: float(r['stats']['latency']))",
                   lambda r: r["user"]["org"]["team"], lambda r: float(r["stats"]["latency"]), None),
}
FILTERS = [(".filter(lambda r: int(r['stats']['n']) >= 0)", lambda r: int(r["stats"]["n"]) >= 0),
           (".filter(lambda r: r['method'] in ('GET', 'PUT') and 'team' in r['user']['org'])",
            lambda r: r["method"] in ("GET", "PUT") and "team" in r["user"]["org"]),
           (".filter(lambda r: not r['user']['id'].endswith('7') or float(r['stats']['latency']) <= 6.5)",
            lambda r: not r["user"]["id"].endswith("7") or float(r["stats"]["latency"]) <= 6.5)]


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("fold", sorted(FOLDS))
def test_every_fold_against_python(fold, filtered, engine, tmp_path):
    P = events_file(tmp_path, 200_000, 11)
    body, key, value, binop = FOLDS[fold]
    flt = FILTERS if filtered else []
    got, stage = run("Dampr.json(P)" + "".join(f for f, _p in flt) + "." + body, P)
    if binop is None:   # mean(): (sum, count) folded, then divided
        sums = dict(eval(x) for x in python_fold(P, [p for _f, p in flt], key, lambda r: (value(r), 1),
                                                 lambda a, b: (a[0] + b[0], a[1] + b[1])))
        exp = sorted(repr((k, s / c)) for k, (s, c) in sums.items())
    else:
        exp = python_fold(P, [p for _f, p in flt], key, value, binop)
    same_up_to_rounding(got, exp)
    on_device(stage)
    assert "host_lines=0" not in stage[2], stage


def test_adversarial_set_end_to_end(engine, tmp_path):
    """each adversarial line (missing and non-object parents, replaced subtrees, duplicate leaves, escaped names on
    and off the wanted paths, wrong depths, the 64-deep limit) gives Python's result or Python's exception; the runs
    without a raising line take lines on the device, those whose bare member has a second kind run on the host map"""
    for src, P, exp, where in adversarial_runs(tmp_path):
        try:
            got, stage = run(src, P)
        except Exception as e:   # noqa: BLE001  the exception is the result under test
            got, stage = type(e), None
        assert got == exp, (src, got, exp)
        if where == "device":
            on_device(stage)
        elif where == "host map":
            assert NEEDLE not in stage[1], stage


# ---- line by line against the stand-in --------------------------------------------------------------------------
def nested_corpus(seed, n, cr):
    """rows the path builds take, and mutations of them: a missing or non-object parent, a replaced subtree, a
    duplicate leaf, escaped names on and off the wanted paths, a str where a filter tests membership, other kinds at
    the leaves, '\\r' between tokens"""
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        k = rng.choice(['"k%d"' % rng.randrange(30), '"k\\n"', '"%s"' % ("long-key-" * rng.randrange(1, 3)),
                        str(rng.randrange(-9, 9)), "1.5", "null"])
        v = rng.choice([str(rng.randrange(-999, 999)), "%r" % (rng.randrange(-64, 64) / 8.0), "-0", "1e3", '"7"',
                        "12345678901234567890"])
        u = '{"k": %s, "x": {"m": 1}, "k2": "d"}' % k
        s = '{"v": %s, "w": {"f": %s}}' % (v, v)
        r = rng.random()
        if r < 0.05:
            u = rng.choice(['"s"', "[1]", "5", "null", "{}"])
        elif r < 0.10:
            s = rng.choice(['"s"', "[{\"v\": 1}]", "{}", '{"w": 3, "v": 1}'])
        elif r < 0.14:
            u = u + ', "u": ' + rng.choice(['{"k": "z"}', "7", '{"q": 1}'])
        elif r < 0.17:
            u = '{"k": "a", "\\u006b": "b"}' if rng.random() < 0.5 else '{"k": "a", "d": {"\\u006b": 1}}'
        elif r < 0.20:
            s = '{"v": 1, "v": %s, "w": {"f": 1, "f": 2.5}}' % v
        elif r < 0.26:   # "m" in r["u"]["x"] over a str: the substring test (an escaped str is the host's)
            u = '{"k": %s, "x": "%s", "k2": "d"}' % (k, rng.choice(["m", "q", "none", "mq", "e\\u006d"]))
        line = '{"u": %s, "s": %s, "t": "%s", "n": %d}' % (u, s, rng.choice("ab"), i)
        if rng.random() < 0.05:
            line = line.replace(", ", ",\r ", 1)
        rows.append(line.replace(": ", rng.choice([":", ": ", " : "])))
    return "".join(r + "\n" for r in rows).encode()


STAGES = [
    ([], 'r["u"]["k"]', 'r["s"]["v"]', "sum"),
    ([], 'r["u"]["k"]', 'float(r["s"]["w"]["f"])', "sum"),
    ([], 'int(r["u"]["k"])', '1', "count"),
    (['r["t"] == "a" or "m" in r["u"]["x"]', 'int(r["s"]["v"]) > -500'], 'r["u"]["k"]', 'int(r["s"]["v"])', "max"),
    (['not r["u"]["k2"] == "e" and r["s"]["w"]["f"] != 3'], 'r["u"]["k"]', 'float(r["s"]["v"])', "min"),
    (['"q" not in r["u"]["x"]'], 'r["u"]["k"]', '1', "count"),
]


@pytest.mark.parametrize("cr", [False, True])
def test_every_path_build_line_by_line(cr, ctx, tmp_path, monkeypatch):
    """int and float values, table and record mode, plain and WHERE, against the stand-in (class, key code, value
    bits) and CPython"""
    from dampr_b200 import Dampr, plan
    from dampr_b200.graph import GMap
    monkeypatch.setattr(fz, "json_line", json_path_line)   # the stand-in outcome of a path member
    P = str(tmp_path / "f.jsonl")
    with open(P, "w") as f:
        f.write('{"u": {"k": "a"}}\n')
    text = Text(ctx, nested_corpus(5 + cr, 5000, cr))
    tally = collections.defaultdict(collections.Counter)
    try:
        for filters, key, value, op in STAGES:
            st = fz.Stage("json", None, filters, key, value, op)
            pm = eval(st.src, {"Dampr": Dampr, "P": P, "json": json})
            g = [s for s in pm.pmer.graph.stages if isinstance(s, GMap)][0]
            st.match = plan._match_json_fields(g, [pm.pmer.graph.inputs[g.inputs[0]]], programs=True, paths=True)
            assert st.match is not None and any(isinstance(m, tuple) for m in st.match[5]), st.src
            check_build(ctx, fz.Build(st), text, cr, tally, random.Random(3))
    finally:
        text.tb.free()
    for k, c in sorted(tally.items()):
        print("  %-22s cr=%d %s" % (k[0], k[1], dict(c)))
        assert c[fz.TAKE] >= 50 and c[fz.HOST] >= 50, (k, c)


def test_kind_retry_of_bare_nested_members(engine, tmp_path):
    rows = [json.dumps({"m": {"k": i % 7 - 3}, "s": {"x": {"v": i / 8.0}}}) for i in range(50_000)]
    P = write_files(tmp_path, [["n.jsonl", "\n".join(rows) + "\n"]])
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['m']['k'], lambda r: r['s']['x']['v']).sum()", P)
    same_up_to_rounding(got, python_fold(P, [], lambda r: r["m"]["k"], lambda r: r["s"]["x"]["v"], operator.add))
    on_device(stage)
    assert "host_lines=0" in stage[2] and "op=sum_f64" in stage[2], stage


def test_tile_seams_window_and_long_lines(engine, tmp_path):
    rng = random.Random(7)
    rows = []
    for i in range(3000):
        pad = rng.choice([0, 1, 2, 3, 5, 100, 4000, 4040, 4050, 4060, 4070, 5000, 9000])
        rows.append(json.dumps({"p": {"x": "x" * pad}, "a": {"k": "k%d" % (i % 13), "b": {"v": i}}},
                               separators=(",", ":")))
    P = write_files(tmp_path, [["seams.jsonl", "\n".join(rows) + "\n"]])
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['a']['k'], lambda r: r['a']['b']['v']).sum()", P)
    assert got == python_fold(P, [], lambda r: r["a"]["k"], lambda r: r["a"]["b"]["v"], operator.add)
    on_device(stage)
    assert "host_lines=0" not in stage[2], stage


def test_more_host_lines_than_the_list_holds(engine, tmp_path):
    rows = ['{"a": {"k": "é%d", "v": %d}}' % (i % 3, i) for i in range(70_000)] + \
        ['{"a": {"k": "a", "v": %d}}' % i for i in range(1000)]
    P = write_files(tmp_path, [["h.jsonl", "\n".join(rows) + "\n"]])
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['a']['k'], lambda r: r['a']['v']).sum()", P)
    assert got == python_fold(P, [], lambda r: r["a"]["k"], lambda r: r["a"]["v"], operator.add)
    assert NEEDLE not in stage[1], stage


def test_long_key_collision_falls_back(engine, tmp_path):
    a, b, _s, _c = PAIRS["raw"][0]
    rows = [json.dumps({"x": {"k": [a.decode(), b.decode(), "short"][i % 3]}, "v": {"n": i}}) for i in range(3000)]
    P = write_files(tmp_path, [["c.jsonl", "\n".join(rows) + "\n"]])
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['x']['k'], lambda r: r['v']['n']).sum()", P)
    assert got == python_fold(P, [], lambda r: r["x"]["k"], lambda r: r["v"]["n"], operator.add)
    assert NEEDLE not in stage[1], stage


def test_a_path_scan_over_poisoned_memory(monkeypatch, tmp_path):
    """a filtered int fold and a float mean() over nested members, on a poisoned pool, a stale text buffer and a
    dirty table: byte-identical runs, equal to Python"""
    from dampr_b200 import Dampr, plan, settings
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "ingest_chunk_bytes", 1 << 16)
    P = events_file(tmp_path, 60_000, 4)
    jobs = {"sum": lambda: Dampr.json(P).filter(lambda r: r["method"] != "PUT")
            .a_group_by(lambda r: r["user"]["org"]["team"], lambda r: r["stats"]["n"]).sum(),
            "mean": lambda: Dampr.json(P).mean(lambda r: r["user"]["id"], lambda r: float(r["stats"]["latency"]))}

    def go(c, seed):
        monkeypatch.setitem(runner_mod._CTX, settings.device, c)
        poison_textbuf(plan._cached_textbuf(c, 2 * (60_000 * 400) + (4 << 20)), seed)
        dirty_table(c, plan._cached_table(c), seed)
        out = {}
        for name, job in sorted(jobs.items()):
            out[name] = sorted(job().run())
            on_device(runner_mod.LAST_STATS.stages[0])
        return out
    res = ab(go)
    exp = python_fold(P, [lambda r: r["method"] != "PUT"], lambda r: r["user"]["org"]["team"],
                      lambda r: r["stats"]["n"], operator.add)
    assert sorted(repr(x) for x in res["sum"]) == exp
    sums = dict(eval(x) for x in python_fold(P, [], lambda r: r["user"]["id"],
                                             lambda r: (float(r["stats"]["latency"]), 1),
                                             lambda a, b: (a[0] + b[0], a[1] + b[1])))
    same_up_to_rounding(sorted(repr(x) for x in res["mean"]), sorted(repr((k, s / c)) for k, (s, c) in sums.items()))

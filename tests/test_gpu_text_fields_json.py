"""JSON-lines field folds on the device (the JSON builds of csrc/fields.cu, `Dampr.json(path)`): the reference pipelines
of tests/test_text_fields_json_lowering.py, every fold with and without filters on seeded inputs against json.loads and
plain Python, an adversarial line set (each line gives Python's result or Python's exception), the kind retries and the
mixed-kind fallback, tile seams and the 4 KB window, more host lines than the fallback list holds, a long-key collision,
and one scan over poisoned memory. Each case asserts which path the stage took."""
import json
import operator
import random

import pytest

from fields_standin import python_lines, reference_outputs, write_files
from test_code_collisions import PAIRS
from test_gpu_poisoned_memory import ab, dirty_table, poison_textbuf
from test_text_fields_json_lowering import GOLDEN, NEEDLE, PIPELINES, datasets, event
from test_text_fields_where_lowering import same_up_to_rounding

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
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P, "json": json}).run())
    return got, runner_mod.LAST_STATS.stages[0]


def outcome(fn):
    """fn()'s value, or the type of the exception it raised"""
    try:
        return fn()
    except Exception as e:   # noqa: BLE001  the exception is the result under test
        return type(e)


def python_fold(P, preds, key, value, binop):
    """plain Python: json.loads of every line, the records that pass every filter, folded in line order"""
    out = {}
    for l in python_lines(P):
        r = json.loads(l)
        if all(p(r) for p in preds):
            k, v = key(r), value(r)
            out[k] = binop(out[k], v) if k in out else v
    return sorted(repr(x) for x in out.items())


def on_device(stage):
    _s, how, detail = stage
    assert NEEDLE in how and "sep=json" in detail, (how, detail)


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, stage = run(src, P)
        same_up_to_rounding(got, exp)
        on_device(stage)


def events_file(tmp_path, n, seed):
    rng = random.Random(seed)
    rows = []
    for i in range(n):
        e = event(rng, i)
        if i % 97 == 5:
            e["user"] = "ü%d" % (i % 4)            # a non-ASCII byte: a host line under every fold
        if i % 89 == 7:
            e["latency"] = 7                        # an int among the floats: float() takes it
        rows.append(json.dumps(e, separators=(",", ":") if i % 3 else (", ", ": "), ensure_ascii=False))
    P = str(tmp_path / "ev.jsonl")
    with open(P, "w", encoding="utf-8") as f:
        f.write("\n".join(rows) + "\n")
    return P


FOLDS = {
    "count": ("count(lambda r: r['user'])", lambda r: r["user"], lambda r: 1, operator.add),
    "int_sum": ("a_group_by(lambda r: r['host'], lambda r: r['bytes']).sum()", lambda r: r["host"],
                lambda r: r["bytes"], operator.add),
    "int_min": ("a_group_by(lambda r: r['user'], lambda r: int(r['bytes'])).reduce(min)", lambda r: r["user"],
                lambda r: int(r["bytes"]), min),
    "int_max": ("a_group_by(lambda r: int(r['zone']), lambda r: r['bytes']).reduce(max)", lambda r: int(r["zone"]),
                lambda r: r["bytes"], max),
    "float_min": ("a_group_by(lambda r: r['host'], lambda r: float(r['ratio'])).reduce(min)", lambda r: r["host"],
                  lambda r: float(r["ratio"]), min),
    "float_max": ("a_group_by(lambda r: r['endpoint'], lambda r: float(r['ratio'])).reduce(max)",
                  lambda r: r["endpoint"], lambda r: float(r["ratio"]), max),
    "float_sum": ("a_group_by(lambda r: r['user'], lambda r: float(r['latency'])).sum()", lambda r: r["user"],
                  lambda r: float(r["latency"]), operator.add),
    "mean_int": ("mean(lambda r: r['method'], lambda r: r['bytes'])", None, None, None),
    "mean_float": ("mean(lambda r: r['endpoint'], lambda r: float(r['latency']))", None, None, None),
}
FILTERS = [(".filter(lambda r: int(r['status']) >= 404)", lambda r: int(r["status"]) >= 404),
           (".filter(lambda r: r['method'] in ('GET', 'PUT'))", lambda r: r["method"] in ("GET", "PUT")),
           (".filter(lambda r: 'meta' in r)", lambda r: "meta" in r),
           (".filter(lambda r: float(r['latency']) <= 6.5)", lambda r: float(r["latency"]) <= 6.5)]


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("fold", sorted(FOLDS))
def test_every_fold_against_python(fold, filtered, engine, tmp_path):
    P = events_file(tmp_path, 200_000, 11)
    body, key, value, binop = FOLDS[fold]
    flt = FILTERS if filtered else []
    src = "Dampr.json(P)" + "".join(f for f, _p in flt) + "." + body
    got, stage = run(src, P)
    if key is None:   # mean(): (sum, count) folded, then divided
        k = (lambda r: r["method"]) if "method" in body else (lambda r: r["endpoint"])
        v = (lambda r: r["bytes"]) if "bytes" in body else (lambda r: float(r["latency"]))
        sums = dict(eval(x) for x in python_fold(P, [p for _f, p in flt], k, lambda r: (v(r), 1),
                                                 lambda a, b: (a[0] + b[0], a[1] + b[1])))
        exp = sorted(repr((kk, s / c)) for kk, (s, c) in sums.items())
    else:
        exp = python_fold(P, [p for _f, p in flt], key, value, binop)
    same_up_to_rounding(got, exp)
    on_device(stage)
    assert "host_lines=0" not in stage[2], stage


ADVERSARIAL = [
    # valid lines: each gives a result
    '{"k": "a", "v": 1}', '{"k":"a","v":2}', ' {"k" : "b" , "v" : 3 } ', '{"k": "a\\"b", "v": 4}',
    '{"k": "{[\\"", "v": 5}', '{"k": "a\\\\", "v": 6}', '{"k": "\\u0061", "v": 7}', '{"\\u006b": "x", "v": 8}',
    '{"k": "b", "v": 9, "k": "c"}', '{"n": {"k": "decoy"}, "k": "d", "v": 10}', '{"k": "e", "v": -0}',
    '{"k": "e", "v": 123456789012345678}', '{"k": "e", "v": 1234567890123456789}',
    '{"k": "e", "v": 1, "big": -12345678901234567890}', '{"k": "f", "v": 1, "x": 1e5, "y": -2.5E-3, "z": 0.0}',
    '{"k": "f", "v": 1, "t": true, "u": false, "w": null, "a": [], "o": {}}',
    '{"k": "g", "v": 1, "x": NaN}', '{"k": "g", "v": 1, "x": Infinity}', '{"k": "g", "v": 1, "x": -Infinity}',
    '{"k": "h", "v": 1, "d": ' + "[" * 63 + "]" * 63 + "}", '{"k": "h", "v": 2, "d": ' + "[" * 64 + "]" * 64 + "}",
    '{"k": "i\x7f", "v": 1}', '{"k": "é", "v": 1}', '\t{"k": "j", "v": 1}\t ', '{"v": 1, "k": "z"}',
]
BAD = [
    '{"k": "a", "v": 01}', '{"k": "a", "v": 1.}', '{"k": "a", "v": .5}', '{"k": "a", "v": +1}', '{"k": "a", "v": 1}x',
    '[1, 2]', '"k"', '5', '', '{"k": "a", "v": tru}', '{"k": "a\tb", "v": 1}', '{"k": "a\x01", "v": 1}',
    '{"k": "a", "v": [1,}', '{"k": "a" "v": 1}', '{"k": "a", "v": 1,}', '{"k": "\\x", "v": 1}', '{"k": "\\u12", "v": 1}',
    '{"v": 1}', '{"k": "a", "v": "1"}', '{"k": "a", "v": true}', '{"k": "a", "v": 1.5}', '{"k": 1, "v": 1}',
]


def test_adversarial_lines(engine, tmp_path):
    """the valid lines together, then each line of BAD behind them: Python's result or Python's exception"""
    # max: an 18-digit value would trip the 64-bit sum bound and send every run to the host
    src = "Dampr.json(P).a_group_by(lambda r: r['k'], lambda r: r['v']).reduce(max)"
    base = [json.dumps({"k": "a", "v": i}) for i in range(300)]
    for extra in [[]] + [[b] for b in BAD]:
        rows = base + ADVERSARIAL + extra
        P = str(tmp_path / "adv.jsonl")
        with open(P, "w", encoding="utf-8", newline="") as f:
            f.write("\n".join(rows) + "\n")
        exp = outcome(lambda: python_fold(P, [], lambda r: r["k"], lambda r: r["v"], max))
        got = outcome(lambda: run(src, P))
        if not extra:
            on_device(got[1])
        assert (got[0] if isinstance(got, tuple) else got) == exp, (extra, got, exp)
    for gz in (False, True):   # '\r' between tokens: whitespace in a .gz source, a line end in a text file
        rows = ['{"k":\r"a", "v": 1}', '{"k": "b",\r"v": 2}\r', '{"k": "c", "v": 3}']
        P = write_files(tmp_path, [["cr.jsonl" + (".gz" if gz else ""), "\n".join(rows) + "\n"]])
        exp = outcome(lambda: python_fold(P, [], lambda r: r["k"], lambda r: r["v"], max))
        assert outcome(lambda: run(src, P)[0]) == exp, gz


def test_kind_retries_and_the_mixed_fallback(engine, tmp_path):
    rows = [json.dumps({"k": i % 7 - 3, "v": i / 8.0, "s": "x%d" % (i % 3)}) for i in range(50_000)]
    P = str(tmp_path / "n.jsonl")
    with open(P, "w") as f:
        f.write("\n".join(rows) + "\n")
    for src, key, val, binop in [
        ("Dampr.json(P).a_group_by(lambda r: r['k'], lambda r: r['v']).sum()", "k", "v", operator.add),
        ("Dampr.json(P).a_group_by(lambda r: r['k'], lambda r: r['v']).reduce(max)", "k", "v", max),
        ("Dampr.json(P).count(lambda r: r['k'])", "k", None, operator.add),
        ("Dampr.json(P).a_group_by(lambda r: r['s'], lambda r: r['v']).reduce(min)", "s", "v", min),
    ]:
        got, stage = run(src, P)
        same_up_to_rounding(got, python_fold(P, [], lambda r: r[key], (lambda r: r[val]) if val else (lambda r: 1),
                                             binop))
        on_device(stage)
        assert "host_lines=0" in stage[2], stage
    rows[100] = json.dumps({"k": "str", "v": 1.5, "s": 3})
    with open(P, "w") as f:
        f.write("\n".join(rows) + "\n")
    for src, key in [("Dampr.json(P).count(lambda r: r['k'])", "k"), ("Dampr.json(P).count(lambda r: r['s'])", "s")]:
        got, stage = run(src, P)
        assert got == python_fold(P, [], lambda r: r[key], lambda r: 1, operator.add)
        assert NEEDLE not in stage[1], stage


def test_tile_seams_window_and_long_lines(engine, tmp_path):
    """lines whose padding puts their start, their members and their end on every side of the 16 KB tile seams and
    at the 4 KB window, plus lines longer than the window"""
    rng = random.Random(7)
    rows = []
    for i in range(3000):
        pad = rng.choice([0, 1, 2, 3, 5, 100, 4000, 4060, 4070, 4080, 4090, 5000, 9000])
        rows.append(json.dumps({"p": "x" * pad, "k": "k%d" % (i % 13), "v": i}, separators=(",", ":")))
    P = str(tmp_path / "seams.jsonl")
    with open(P, "w") as f:
        f.write("\n".join(rows) + "\n")
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['k'], lambda r: r['v']).sum()", P)
    assert got == python_fold(P, [], lambda r: r["k"], lambda r: r["v"], operator.add)
    on_device(stage)
    assert "host_lines=0" not in stage[2], stage


def test_more_host_lines_than_the_list_holds(engine, tmp_path):
    rows = [json.dumps({"k": "é%d" % (i % 3), "v": i}, ensure_ascii=False) for i in range(70_000)]
    rows += [json.dumps({"k": "a", "v": i}) for i in range(1000)]
    P = write_files(tmp_path, [["h.jsonl", "\n".join(rows) + "\n"]])
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['k'], lambda r: r['v']).sum()", P)
    assert got == python_fold(P, [], lambda r: r["k"], lambda r: r["v"], operator.add)
    assert NEEDLE not in stage[1], stage


def test_long_key_collision_falls_back(engine, tmp_path):
    """two 13-byte keys with the same 64-bit code (tests/golden/code_collisions.json) as string values"""
    a, b, _s, _c = PAIRS["raw"][0]
    rows = [json.dumps({"k": [a.decode(), b.decode(), "short"][i % 3], "v": i}) for i in range(3000)]
    P = write_files(tmp_path, [["c.jsonl", "\n".join(rows) + "\n"]])
    got, stage = run("Dampr.json(P).a_group_by(lambda r: r['k'], lambda r: r['v']).sum()", P)
    assert got == python_fold(P, [], lambda r: r["k"], lambda r: r["v"], operator.add)
    assert NEEDLE not in stage[1], stage


def test_a_json_scan_over_poisoned_memory(monkeypatch, tmp_path):
    """a filtered int fold and a float mean() over JSON lines, on a poisoned pool, a stale text buffer and a dirty
    table: byte-identical runs, equal to Python"""
    from dampr_b200 import Dampr, plan, settings
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "ingest_chunk_bytes", 1 << 16)
    P = events_file(tmp_path, 60_000, 4)
    jobs = {"sum": lambda: Dampr.json(P).filter(lambda r: r["method"] != "PUT")
            .a_group_by(lambda r: r["host"], lambda r: r["bytes"]).sum(),
            "mean": lambda: Dampr.json(P).mean(lambda r: r["user"], lambda r: float(r["latency"]))}

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
    exp = python_fold(P, [lambda r: r["method"] != "PUT"], lambda r: r["host"], lambda r: r["bytes"], operator.add)
    assert sorted(repr(x) for x in res["sum"]) == exp
    sums = dict(eval(x) for x in python_fold(P, [], lambda r: r["user"], lambda r: (float(r["latency"]), 1),
                                             lambda a, b: (a[0] + b[0], a[1] + b[1])))
    same_up_to_rounding(sorted(repr(x) for x in res["mean"]),
                        sorted(repr((k, s / c)) for k, (s, c) in sums.items()))


def test_the_binding_checks_its_arguments(ctx):
    import numpy as np
    from dampr_b200 import device as dev
    data = b'{"a": "x", "b": 2}\n{"a": "x", "b": 3}\n'
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    js = (dev.FIELD_SEP_JSON, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64)
    try:
        for spec, members, preds in [
            ((ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64), ["a", "b"], ()),   # a separator byte
            ((dev.FIELD_SEP_JSON, 2, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64), ["a", "b"], ()),   # no member 2
            (js, ["a", 'b"'], ()),
            (js, ["a"] * 9, ()),
            (js, ["a", "b"], [(dev.PRED_NFIELDS, 0, dev.CMP_EQ, (2,))]),
            (js, ["a", "b"], [(dev.PRED_MEMBER, 0, dev.CMP_EQ, ())]),
            (js, ["a", "b"], [(dev.PRED_MEMBER, 2, dev.CMP_IN, ())]),
        ]:
            with pytest.raises(dev.DeviceError):
                tab.json_fields(tb, 0, len(data), spec, members, preds=preds)
        with pytest.raises(dev.DeviceError):   # the field call does not take the JSON separator or MEMBER
            tab.fields(tb, 0, len(data), js)
        with pytest.raises(dev.DeviceError):
            tab.fields(tb, 0, len(data), (ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64),
                       preds=[(dev.PRED_MEMBER, 0, dev.CMP_IN, ())])
        tab.clear()
        tab.json_fields(tb, 0, len(data), js, ["a", "b"])
        st = tab.fields_stats()
        assert st["lines"] == 2 and st["fallback"] == 0 and st["flags"] == 0, st
        assert tab.fields_fetch(dev.OP_SUM_I64)[1].tolist() == [5]
    finally:
        tb.free()
        tab.free()

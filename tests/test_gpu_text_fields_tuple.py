"""Tuple keys of field folds on the device (the tuple-key builds of csrc/fields.cu, `(r[i], int(r[j]), ...)`): the
reference pipelines of tests/test_text_fields_tuple_lowering.py, every fold with 2 and 4 components under a separator
byte and split(), with and without filters, on seeded inputs against plain Python, keys whose lines are split between
the device and the host, the kernel's codes against the Python statement, real 64-bit code collisions, tile seams, the
4 KB window, more host lines than the fallback list holds, and the consumers of a tuple-keyed result. Each case
asserts which path the stage took."""
import json
import operator
import os
import random

import numpy as np
import pytest

from fields_standin import python_lines, reference_outputs, write_files
from fields_tuple_standin import tuple_code
from test_code_collisions import PAIRS
from test_text_fields_float_lowering import same_records
from test_text_fields_tuple_lowering import GOLDEN, NEEDLE, PIPELINES, datasets
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
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P}).run())
    return got, runner_mod.LAST_STATS.stages[0]


def on_device(how, detail, n):
    assert NEEDLE in how and " key=tuple%d" % n in detail, (how, detail)


def python_fold(P, split, preds, key, value, binop):
    out = {}
    for l in python_lines(P):
        r = split(l)
        if all(p(r) for p in preds):
            k, v = key(r), value(r)
            out[k] = binop(out[k], v) if k in out else v
    return sorted(repr(x) for x in out.items())


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, (_s, how, detail) = run(src, P)
        same_up_to_rounding(got, exp)
        assert NEEDLE in how and " key=tuple" in detail and ("sep=ws" in detail) == (name == "ws"), (src, detail)


# ---- every fold against Python ----------------------------------------------------------------------------------
WS_RUNS = [" ", "  ", "\t", " \t ", "\x0b", "\x1f"]


def seeded_rows(seed, sep, n=200000):
    """`host method status bytes latency tag` rows: hosts of 1..9 bytes and longer (hashed lengths), statuses written
    404 / +404 / 0404, int and float columns, a few non-ASCII tags (host lines); under split() mixed whitespace runs
    and leading and trailing blanks"""
    rng = random.Random(seed)
    hosts = ["a", "bb", "x" * 9, "y" * 10, "z" * 40, ""] + ["h%d" % i for i in range(300)]
    rows = []
    for i in range(n):
        st = rng.choice([200, 301, 404, 500, -7])
        f = [rng.choice(hosts) or ("q" if sep is None else ""), rng.choice(["GET", "POST", "PUT"]),
             rng.choice(["%d" % st, "%+d" % st, "0%d" % st if st > 0 else "-0%d" % -st]),
             str(rng.randrange(-1000, 100000)),
             "%r" % rng.uniform(-100, 100) if rng.random() < 0.7 else rng.choice(["0.5", "7", "-2.25", "1e3"]),
             "t%d" % rng.randrange(4) if i % 1009 else "é"]
        if sep is None:
            rows.append(rng.choice(["", " ", "\t"]) + "".join(x + rng.choice(WS_RUNS) for x in f[:-1]) + f[-1] +
                        rng.choice(["", " "]))
        else:
            rows.append(sep.join(f))
    return "\n".join(rows) + "\n"


KEYS = {   # components: (key source, Python key)
    2: ("(r[0], int(r[2]))", lambda r: (r[0], int(r[2]))),
    4: ("(r[1], r[0], int(r[-4]), r[5])", lambda r: (r[1], r[0], int(r[-4]), r[5])),
}
FOLDS = {   # name: (pipeline tail with K for the key, value, binop, float value)
    "count": (".count(lambda r: K)", lambda r: 1, operator.add, False),
    "sum_i64": (".a_group_by(lambda r: K, lambda r: int(r[3])).sum()", lambda r: int(r[3]), operator.add, False),
    "min_i64": (".a_group_by(lambda r: K, lambda r: int(r[3])).reduce(min)", lambda r: int(r[3]), min, False),
    "max_i64": (".fold_by(lambda r: K, max, lambda r: int(r[-3]))", lambda r: int(r[-3]), max, False),
    "min_f64": (".a_group_by(lambda r: K, lambda r: float(r[4])).reduce(min)", lambda r: float(r[4]), min, False),
    "max_f64": (".a_group_by(lambda r: K, lambda r: float(r[4])).reduce(max)", lambda r: float(r[4]), max, False),
    "sum_f64": (".a_group_by(lambda r: K, lambda r: float(r[4])).sum()", lambda r: float(r[4]), operator.add, True),
    "mean_i64": (".mean(lambda r: K, lambda r: int(r[3]))", lambda r: int(r[3]), None, True),
    "mean_f64": (".mean(lambda r: K, lambda r: float(r[4]))", lambda r: float(r[4]), None, True),
}


class _Named(object):
    """a value function whose repr tells same_records a mean from a sum"""
    def __init__(self, f, name):
        self.f, self.name = f, name

    def __call__(self, l):
        return self.f(l)

    def __repr__(self):
        return self.name


@pytest.fixture(scope="module")
def seeded(tmp_path_factory):
    d = tmp_path_factory.mktemp("seeded")
    out = {}
    for name, sep in ((",", ","), ("ws", None)):
        (d / name).mkdir()
        out[name] = write_files(d / name, [["f.txt", seeded_rows(len(name), sep)]])
    return out


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("sep", [",", "ws"])
@pytest.mark.parametrize("n", sorted(KEYS))
@pytest.mark.parametrize("fold", sorted(FOLDS))
def test_every_fold_against_python(fold, n, sep, filtered, seeded, engine, tmp_path):
    tail, value, binop, flt = FOLDS[fold]
    ksrc, key = KEYS[n]
    P = seeded[sep]
    split = (lambda l: l.split(",")) if sep == "," else (lambda l: l.split())
    src = "Dampr.text(P).map(lambda l: l.split(%s))" % ("','" if sep == "," else "")
    preds = []
    if filtered:
        preds = [lambda r: r[1] != "PUT", lambda r: int(r[3]) >= -500]
        src += ".filter(lambda r: r[1] != 'PUT').filter(lambda r: int(r[3]) >= -500)"
    got, (_s, how, detail) = run(src + tail.replace("K", ksrc), P)
    on_device(how, detail, n)
    assert "host_lines=%d" % sum(1 for l in python_lines(P) if "é" in l and all(p(split(l)) for p in preds)) in detail
    if not flt:
        assert got == python_fold(P, split, preds, key, value, binop), fold
        return
    kept = [l for l in python_lines(P) if all(p(split(l)) for p in preds)]
    acc = {}
    for l in kept:
        r = split(l)
        s, c = acc.get(key(r), (0, 0))
        acc[key(r)] = (s + value(r), c + 1)
    exp = sorted(repr((k, s / float(c) if fold.startswith("mean") else s)) for k, (s, c) in acc.items())
    (tmp_path / "kept").mkdir()
    KP = write_files(tmp_path / "kept", [["k.txt", "\n".join(kept) + "\n"]])
    same_records(got, exp, KP, lambda l: key(split(l)), _Named(lambda l: value(split(l)), fold))


# ---- the merge, the codes, collisions ---------------------------------------------------------------------------
def test_keys_with_device_and_host_lines(engine, tmp_path):
    """every key has lines the device takes and lines only the host can read (non-ASCII, text-mode '\\r'): each key
    comes back once, folded over both"""
    rows = []
    for i in range(20000):
        tail = "é" if i % 7 == 0 else "\r" if i % 11 == 0 else "x"
        rows.append("k%d,%s,%d,%s" % (i % 13, ["GET", "PUT"][i % 2], i % 97 - 40, tail))
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    for tail, value, binop in [(".a_group_by(lambda r: (r[0], r[1]), lambda r: int(r[2])).sum()",
                                lambda r: int(r[2]), operator.add),
                               (".a_group_by(lambda r: (r[0], int(r[2]) ), lambda r: int(r[2])).reduce(min)",
                                lambda r: int(r[2]), min)]:
        got, (_s, how, detail) = run("Dampr.text(P).map(lambda l: l.split(','))" + tail, P)
        key = (lambda r: (r[0], r[1])) if "r[1])" in tail else (lambda r: (r[0], int(r[2])))
        assert got == python_fold(P, lambda l: l.split(","), [], key, value, binop)
        on_device(how, detail, 2)
        assert "host_lines=0" not in detail, detail
    got, (_s, how, detail) = run("Dampr.text(P).map(lambda l: l.split(',')).mean(lambda r: (r[1], r[0]),"
                                 " lambda r: float(r[2]))", P)
    on_device(how, detail, 2)
    acc = {}
    for l in python_lines(P):
        r = l.split(",")
        s, c = acc.get((r[1], r[0]), (0.0, 0))
        acc[(r[1], r[0])] = (s + float(r[2]), c + 1)
    same_up_to_rounding(got, sorted(repr((k, s / c)) for k, (s, c) in acc.items()))


def test_kernel_codes_equal_the_statement(ctx):
    from dampr_b200 import device as dev
    rows = [b"a,7,xyz", b"a,+7,xyz", b"long-key-of-many-bytes,-3,", b",0,q", b"b,123456789012345678,\x1f"]
    data = b"\n".join(rows) + b"\n"
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    keys = ((0, dev.FIELD_KEY_STR), (1, dev.FIELD_KEY_INT), (-1, dev.FIELD_KEY_STR))
    try:
        tab.fields_tuple(tb, 0, len(data), (ord(","), 0, dev.FIELD_KEY_STR, dev.FIELD_VAL_ONE, dev.OP_SUM_I64), keys)
        st = tab.fields_stats()
        assert st["lines"] == 5 and st["fallback"] == 0 and st["flags"] == 0 and st["hashed"] == 0, st
        cols, counts, codes = tab.fetch_field_keys(tb, ord(","), keys)
        got = {(a.decode(), int(b), c.decode()): (int(n), int(code))
               for a, b, c, n, code in zip(cols[0].tolist(), cols[1].tolist(), cols[2].tolist(), counts, codes)}
        exp = {}
        for r in rows:
            f = r.split(b",")
            k = (f[0].decode(), int(f[1]), f[2].decode())
            exp[k] = (exp.get(k, (0, 0))[0] + 1, tuple_code([f[0], int(f[1]), f[2]]))
        assert got == exp
        assert cols[0].dtype == np.dtype("S22") and cols[1].dtype == np.int64
        for bad in ((), ((0, dev.FIELD_KEY_STR),) * 5, ((0, 2),)):   # n outside 1 .. 4, a kind
            with pytest.raises(dev.DeviceError):
                tab.fields_tuple(tb, 0, len(data), (ord(","), 0, 0, dev.FIELD_VAL_ONE, dev.OP_SUM_I64), bad)
        with pytest.raises(dev.DeviceError):
            tab.fields_tuple(tb, 0, len(data), (dev.FIELD_SEP_JSON, 0, 0, dev.FIELD_VAL_ONE, dev.OP_SUM_I64), keys)
    finally:
        tb.free()
        tab.free()


def test_real_collisions_fall_back(ctx, engine, tmp_path):
    """the raw pairs of tests/golden/code_collisions.json as first components share the tuple's code: the kernel
    flags DAMPR_TF_COLLISION and the stage returns Python's answer through the host map; with one of each pair only,
    it stays on the device"""
    from dampr_b200 import device as dev
    rows = []
    for i, (a, b, _s, _c) in enumerate(PAIRS["raw"][:8]):
        rows += [b"%s,GET,%d" % (a, i), b"%s,GET,%d" % (b, i + 100), b"%s,PUT,1" % a]
    data = b"\n".join(rows) + b"\n"
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    try:
        tab.fields_tuple(tb, 0, len(data), (ord(","), 0, 0, 2, dev.OP_SUM_I64),
                         ((0, dev.FIELD_KEY_STR), (1, dev.FIELD_KEY_STR)))
        assert tab.fields_stats()["flags"] & dev.TF_COLLISION
    finally:
        tb.free()
        tab.free()
    src = "Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: (r[0], r[1]), lambda r: int(r[2])).sum()"
    for keep_b, device in ((True, False), (False, True)):
        text = "".join(r.decode() + "\n" for r in rows
                       if keep_b or not any(r.startswith(p[1]) for p in PAIRS["raw"][:8]))
        (tmp_path / str(keep_b)).mkdir()
        P = write_files(tmp_path / str(keep_b), [["f.csv", text * 50]])
        got, (_s, how, detail) = run(src, P)
        assert got == python_fold(P, lambda l: l.split(","), [], lambda r: (r[0], r[1]), lambda r: int(r[2]),
                                  operator.add)
        if device:
            on_device(how, detail, 2)
        else:
            assert how.startswith("host-map"), how


# ---- seams, window, host lines ----------------------------------------------------------------------------------
def test_tile_seams_and_the_window(engine, tmp_path):
    """components of every length at every offset across 16 KB tiles and small upload chunks, and lines just under
    and over the 4 KB window (the longer ones are host lines)"""
    engine.ingest_chunk_bytes = 1 << 16
    rng = random.Random(8)
    rows = []
    for i in range(60000):
        rows.append("%s %s\t%d %s" % ("k" * rng.randint(1, 12), "m" * rng.randint(1, 5), rng.randrange(-99, 99),
                                      "p" * rng.randint(0, 40)))
    rows[1000] = "long x 1 " + "p" * 4086           # 4095 bytes: its newline is the window's last byte
    rows[1001] = "long x 1 " + "p" * 4087           # 4096 bytes: a host line
    rows[30000] = "long y 2 " + "p" * 5000
    P = write_files(tmp_path, [["f.txt", "\n".join(rows) + "\n"]])
    src = "Dampr.text(P).map(lambda l: l.split()).a_group_by(lambda r: (r[1], r[0], int(r[2])), lambda r: len(r)).sum()"
    got, (_s, how, detail) = run(src.replace("lambda r: len(r)", "lambda r: 1"), P)
    on_device(how, detail, 3)
    assert "host_lines=2" in detail, detail
    assert got == python_fold(P, lambda l: l.split(), [], lambda r: (r[1], r[0], int(r[2])), lambda r: 1,
                              operator.add)


def test_more_host_lines_than_the_list_holds(engine, tmp_path):
    rows = ["k%d,é,%d" % (i % 7, i) for i in range(70000)] + ["a,b,1"]
    P = write_files(tmp_path, [["f.txt", "\n".join(rows) + "\n"]])
    got, (_s, how, _d) = run("Dampr.text(P).map(lambda l: l.split(',')).count(lambda r: (r[0], r[1]))", P)
    assert how.startswith("host-map"), how
    assert got == python_fold(P, lambda l: l.split(","), [], lambda r: (r[0], r[1]), lambda r: 1, operator.add)


# ---- downstream consumers ---------------------------------------------------------------------------------------
def test_consumers_of_a_tuple_keyed_result(engine, tmp_path):
    from dampr_b200 import Dampr
    rng = random.Random(3)
    rows = ["h%d,%s,%d,%d" % (rng.randrange(40), rng.choice(["GET", "POST"]), rng.choice([200, 404]),
                              rng.randrange(1000)) for _ in range(30000)]
    P = write_files(tmp_path, [["f.csv", "\n".join(rows) + "\n"]])
    lines = python_lines(P)
    exp = {}
    for l in lines:
        r = l.split(",")
        k = (r[0], int(r[2]))
        exp[k] = exp.get(k, 0) + int(r[3])
    hits = {}
    for l in lines:
        r = l.split(",")
        k = (r[0], int(r[2]))
        hits[k] = hits.get(k, 0) + 1

    def folded():
        return Dampr.text(P).map(lambda l: l.split(",")).a_group_by(lambda r: (r[0], int(r[2])),
                                                                     lambda r: int(r[3])).sum()
    from dampr_b200 import runner as runner_mod
    assert sorted(folded().run()) == sorted(exp.items())
    on_device(runner_mod.LAST_STATS.stages[0][1], runner_mod.LAST_STATS.stages[0][2], 2)
    assert sorted(folded().sort_by(lambda kv: (kv[1], kv[0])).run()) == sorted(exp.items())
    top = list(folded().topk(5, lambda kv: kv[1]).run())
    assert sorted(v for _k, v in top) == sorted(exp.values())[-5:]
    assert sorted(folded().map(lambda kv: (kv[0][1], kv[0][0], kv[1])).run()) == \
        sorted((k[1], k[0], v) for k, v in exp.items())
    other = Dampr.text(P).map(lambda l: l.split(",")).count(lambda r: (r[0], int(r[2])))
    # a fold's records (key, value) are the values of the join under its key
    joined = sorted(folded().join(other).reduce(lambda a, b: ([v for _k, v in a], [v for _k, v in b])).run())
    assert joined == sorted((k, ([v], [hits[k]])) for k, v in exp.items())
    for kind in ("sink", "sink_tsv", "sink_json"):
        out = str(tmp_path / kind)
        getattr(folded(), kind)(out).run()
        text = []
        for fn in sorted(os.listdir(out)):
            with open(os.path.join(out, fn)) as f:
                text += [l.rstrip("\n") for l in f]
        if kind == "sink_json":
            assert sorted(json.dumps(json.loads(t)) for t in text) == sorted(json.dumps([k, v]) for k, v in exp.items())
        elif kind == "sink_tsv":
            assert sorted(text) == sorted("%s\t%s" % (k, v) for k, v in exp.items())
        else:
            assert sorted(text) == sorted(str((k, v)) for k, v in exp.items())

"""Whitespace-split field folds on the device (the WS builds of csrc/fields.cu, `line.split()[i]`): the reference
pipelines of tests/test_text_fields_ws_lowering.py, every fold with and without filters on seeded inputs against plain
Python, whitespace runs and fields at every offset of the 4-byte steps, tile seams, the 4 KB window and the 64 KB limit,
more host lines than the fallback list holds, and a long-key code collision. Each case asserts which path the stage
took."""
import operator
import random
import zlib

import numpy as np
import pytest

from fields_standin import python_lines, reference_outputs, write_files
from test_code_collisions import PAIRS
from test_text_fields_float_lowering import same_records
from test_text_fields_where_lowering import same_up_to_rounding
from test_text_fields_ws_lowering import GOLDEN, NEEDLE, PIPELINES, datasets

pytestmark = pytest.mark.gpu

RUNS = [" ", " ", "  ", "\t", " \t ", "\x0b", "\x0c", "\x1c", "\x1d", "\x1e", "\x1f", "     "]


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


def on_device(how, detail):
    assert NEEDLE in how and "sep=ws" in detail, (how, detail)


def python_fold(P, preds, key, value, binop):
    """plain Python: split() of every line, the records that pass every filter, folded in line order"""
    out = {}
    for l in python_lines(P):
        r = l.split()
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
        assert NEEDLE in how and ("sep=ws" in detail) == ("split(' ')" not in src), (name, src, how, detail)


def seeded_rows(seed, n=200000):
    """`key method int float` rows joined by mixed whitespace runs, leading and trailing blanks; keys of 1..9 bytes
    and longer (the hashed path); blank, all-whitespace and short rows"""
    rng = random.Random(seed)
    keys = ["a", "bb", "x" * 9, "y" * 10, "z" * 40] + ["k%d" % i for i in range(200)]
    rows = []
    for i in range(n):
        if i % 997 == 3:
            rows.append(rng.choice(["", "   ", "\t\x0b", "short"]))
            continue
        f = [rng.choice(keys), rng.choice(["GET", "POST", "PUT"]), str(rng.randrange(-1000, 1000)),
             "%r" % rng.uniform(-100, 100) if rng.random() < 0.7 else rng.choice(["0.5", "7", "-2.25", "1e3"])]
        rows.append(rng.choice(["", "", " ", "\t "]) + "".join(x + rng.choice(RUNS) for x in f[:-1]) + f[-1] +
                    rng.choice(["", "", " ", "\x1f"]))
    return "\n".join(rows) + "\n"


FOLDS = {   # name: (pipeline tail, key, value, binop, float value)
    "count": (".count(lambda r: r[0])", lambda r: r[0], lambda r: 1, operator.add, False),
    "sum_i64": (".a_group_by(lambda r: r[0], lambda r: int(r[2])).sum()", lambda r: r[0], lambda r: int(r[2]),
                operator.add, False),
    "min_i64": (".a_group_by(lambda r: r[1], lambda r: int(r[-2])).reduce(min)", lambda r: r[1],
                lambda r: int(r[-2]), min, False),
    "max_i64": (".a_group_by(lambda r: int(r[2]), lambda r: int(r[2])).reduce(max)", lambda r: int(r[2]),
                lambda r: int(r[2]), max, False),
    "min_f64": (".a_group_by(lambda r: r[-4], lambda r: float(r[3])).reduce(min)", lambda r: r[-4],
                lambda r: float(r[3]), min, False),
    "max_f64": (".a_group_by(lambda r: r[0], lambda r: float(r[-1])).reduce(max)", lambda r: r[0],
                lambda r: float(r[-1]), max, False),
    "sum_f64": (".a_group_by(lambda r: r[0], lambda r: float(r[3])).sum()", lambda r: r[0], lambda r: float(r[3]),
                operator.add, True),
    "mean": (".mean(lambda r: r[1], lambda r: float(r[3]))", lambda r: r[1], lambda r: float(r[3]), None, True),
}


class _Named(object):
    """a value function whose repr tells same_records a mean from a sum"""
    def __init__(self, f, name):
        self.f, self.name = f, name

    def __call__(self, l):
        return self.f(l)

    def __repr__(self):
        return self.name


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("fold", sorted(FOLDS))
def test_every_fold_against_python(fold, filtered, engine, tmp_path):
    tail, key, value, binop, flt = FOLDS[fold]
    P = write_files(tmp_path, [["f.log", seeded_rows(zlib.crc32(fold.encode()) + filtered)]])
    preds = [lambda r: len(r) == 4]
    src = "Dampr.text(P).map(lambda l: l.split()).filter(lambda r: len(r) == 4)"
    if filtered:
        preds += [lambda r: r[1] != "PUT", lambda r: int(r[2]) >= -500]
        src += ".filter(lambda r: r[1] != 'PUT').filter(lambda r: int(r[2]) >= -500)"
    got, (_s, how, detail) = run(src + tail, P)
    on_device(how, detail)
    assert "host_lines=0" in detail and "filtered=" in detail, detail
    if not flt:
        assert got == python_fold(P, preds, key, value, binop), fold
        return
    kept = [l for l in python_lines(P) if all(p(l.split()) for p in preds)]
    acc = {}
    for l in kept:
        r = l.split()
        s, n = acc.get(key(r), (0.0, 0))
        acc[key(r)] = (s + value(r), n + 1)
    exp = sorted(repr((k, s / float(n) if fold == "mean" else s)) for k, (s, n) in acc.items())
    (tmp_path / "kept").mkdir()
    KP = write_files(tmp_path / "kept", [["k.log", "\n".join(kept) + "\n"]])
    same_records(got, exp, KP, lambda l: key(l.split()), _Named(lambda l: value(l.split()), fold))


def test_runs_and_fields_at_every_offset(engine, tmp_path):
    """leading blanks, whitespace runs and fields of 1..6 bytes in every combination: field starts and ends, and the
    class carried between 4-byte steps, at every offset mod 4, in lines that start at every offset mod 4"""
    ws = " \t\x0b\x0c\x1c\x1d\x1e\x1f"
    rows = []
    rng = random.Random(5)
    for lead in range(6):
        for run_len in range(1, 7):
            for flen in range(1, 7):
                for t in range(4):
                    sep = "".join(rng.choice(ws) for _ in range(run_len))
                    f = ["k" * flen, str(rng.randrange(10 ** (flen - 1), 10 ** flen)), "v" * ((flen + t) % 6 + 1)]
                    rows.append("".join(rng.choice(ws) for _ in range(lead)) + sep.join(f) +
                                " " * ((lead + t) % 3))
    P = write_files(tmp_path, [["f.log", "\n".join(rows * 20) + "\n"]])
    for src, key, value in [
            ("Dampr.text(P).a_group_by(lambda l: l.split()[0], lambda l: int(l.split()[1])).sum()",
             lambda r: r[0], lambda r: int(r[1])),
            ("Dampr.text(P).a_group_by(lambda l: l.split()[-1], lambda l: int(l.split()[-2])).sum()",
             lambda r: r[-1], lambda r: int(r[-2])),
            ("Dampr.text(P).filter(lambda l: l.split()[2] >= 'vvv').count(lambda l: l.split()[1])",
             lambda r: r[1], lambda r: 1)]:
        got, (_s, how, detail) = run(src, P)
        on_device(how, detail)
        assert "host_lines=0" in detail, detail
        preds = [lambda r: r[2] >= "vvv"] if "filter" in src else []
        assert got == python_fold(P, preds, key, value, operator.add), src
    # '\r' is whitespace in a .gz source (binary mode): the same rows with it in their runs
    rows = [r.replace("\x1d", "\r") for r in rows]
    (tmp_path / "gz").mkdir()
    P = write_files(tmp_path / "gz", [["f.log.gz", "\n".join(rows * 20) + "\n"]])
    got, (_s, how, detail) = run("Dampr.text(P).a_group_by(lambda l: l.split()[0], lambda l: int(l.split()[1])).sum()",
                                 P)
    on_device(how, detail)
    assert "host_lines=0" in detail and got == python_fold(P, [], lambda r: r[0], lambda r: int(r[1]), operator.add)


def test_tile_seams_window_and_long_lines(engine, tmp_path):
    """rows across 16 KB tiles with small upload chunks, several files, rows just under and over the 4 KB window (the
    host runs the stage's functions on the longer ones), a row under 64 KB (a host line) and one over it (the whole
    stage on the host)"""
    engine.ingest_chunk_bytes = 1 << 16
    rng = np.random.default_rng(4)
    files = []
    for f in range(3):
        rows = ["  k%d %s %d" % (rng.integers(0, 500), "p" * int(rng.integers(1, 90)), rng.integers(-50, 50))
                for _ in range(40000)]
        rows[100] = "long " + " " * 4088 + " 3"      # 4095 bytes: its newline is the window's last byte
        rows[101] = "long " + " " * 4088 + "\t-3"    # 4096 bytes: a host line
        rows[102] = "\t" * 4093 + "w 1"               # 4096 bytes
        rows[200] = "longer " + " " * 70000 + " 4"
        files.append(["p%d.txt" % f, "\n".join(rows) + ("" if f == 1 else "\n")])
    src = "Dampr.text(P).a_group_by(lambda l: l.split()[0], lambda l: int(l.split()[-1])).sum()"

    def exp(P):
        return python_fold(P, [], lambda r: r[0], lambda r: int(r[-1]), operator.add)
    P = write_files(tmp_path, files)
    got, (_s, how, _d) = run(src, P)
    assert got == exp(P) and how.startswith("host-map"), how
    for f in files:
        f[1] = f[1].replace(" " * 70000, " " * 60000)
    (tmp_path / "b").mkdir()
    P = write_files(tmp_path / "b", files)
    got, (_s, how, detail) = run(src, P)
    assert got == exp(P), detail
    on_device(how, detail)
    assert "host_lines=9" in detail, detail   # rows 101, 102 and 200 of each file


def test_more_host_lines_than_the_list_holds(engine, tmp_path):
    """70,000 rows split by NBSP (non-ASCII: host lines) send the whole stage to the host; 70,000 blank rows behind a
    len() filter are dropped on the device"""
    rows = ["k%d %d" % (i % 7, i) for i in range(70000)] + ["a 1", "b\t2", "a  3"]
    P = write_files(tmp_path, [["f.txt", "\n".join(rows) + "\n"]])
    src = "Dampr.text(P).map(lambda l: l.split()).a_group_by(lambda r: r[0], lambda r: int(r[1])).sum()"
    got, (_s, how, _d) = run(src, P)
    assert how.startswith("host-map"), how
    assert got == python_fold(P, [], lambda r: r[0], lambda r: int(r[1]), operator.add)
    rows = [" \t" * (i % 3) for i in range(70000)] + ["a 1", "b\t2", "a  3"]
    (tmp_path / "b").mkdir()
    P = write_files(tmp_path / "b", [["f.txt", "\n".join(rows) + "\n"]])
    got, (_s, how, detail) = run(src.replace(".a_group_by", ".filter(lambda r: len(r) >= 2).a_group_by"), P)
    assert got == ["('a', 4)", "('b', 2)"]
    on_device(how, detail)
    assert "host_lines=0" in detail and "filtered=70000" in detail, detail


def test_long_key_collision_falls_back(engine, tmp_path):
    """two keys of 13 bytes with the same 64-bit code (tests/golden/code_collisions.json): the stage runs on the host
    and equals Python; the same rows with one key only stay on the device"""
    a, b, _s, _c = PAIRS["raw"][0]
    a, b = a.decode(), b.decode()
    assert not any(c.isspace() for c in a + b)
    src = "Dampr.text(P).map(lambda l: l.split()).a_group_by(lambda r: r[1], lambda r: int(r[2])).sum()"
    for second, device in ((b, False), (a, True)):
        rows = ["  x\t%s  %d" % (a if i % 3 else "k%d" % (i % 5), i) for i in range(3000)]
        rows[1700] = "y %s\x1f7 " % second
        (tmp_path / second).mkdir()
        P = write_files(tmp_path / second, [["f.txt", "\n".join(rows) + "\n"]])
        got, (_s, how, detail) = run(src, P)
        assert got == python_fold(P, [], lambda r: r[1], lambda r: int(r[2]), operator.add)
        if device:
            on_device(how, detail)
        else:
            assert how.startswith("host-map"), how


def test_the_binding_refuses_other_separators(ctx):
    from dampr_b200 import device as dev
    data = b"a 1\n"
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(10)
    try:
        for sep in (257, 255, 0x80, 0, 10, 13, -1):
            with pytest.raises(dev.DeviceError):
                tab.fields(tb, 0, len(data), (sep, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64))
        tab.fields(tb, 0, len(data), (dev.FIELD_SEP_WS, 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64))
        st = tab.fields_stats()
        assert st["lines"] == 1 and st["fallback"] == 0 and st["flags"] == 0, st
    finally:
        tb.free()
        tab.free()

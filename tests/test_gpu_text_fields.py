"""Delimited-field folds (`l.split(S)[i]` keys with counts, int sums, minima and maxima) on the device
(dampr_text_fields, csrc/fields.cu): every case is compared with a plain-Python restatement, the shared inputs also
with the reference's stored outputs (tests/test_text_fields_lowering.py), and each asserts which path the stage took."""
import gzip
import operator
import os

import numpy as np
import pytest

from fields_standin import python_fold, reference_outputs, write_files
from test_text_fields_lowering import GOLDEN, NEEDLE, PIPELINES, datasets

pytestmark = pytest.mark.gpu


@pytest.fixture
def engine(monkeypatch):
    """the real device context for the runner, fresh scan buffers, the settings a case may change restored"""
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


SUM = "Dampr.text(P).a_group_by(lambda l: l.split('%s')[%d], lambda l: int(l.split('%s')[%d])).%s"


@pytest.mark.parametrize("name", sorted(datasets()))
def test_reference_inputs(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, (_s, how, _d) = run(src, P)
        assert got == exp, (name, src)
        assert NEEDLE in how, (name, src, how)


@pytest.mark.parametrize("red,binop", [("sum()", operator.add), ("reduce(min)", min), ("reduce(max)", max)])
@pytest.mark.parametrize("ki,vi", [(0, 2), (-1, 1), (1, -2), (2, 2)])
def test_str_keys_indices_and_ops(red, binop, ki, vi, engine, tmp_path):
    """str keys of 0, 1, 2, 9, 10 and 45 bytes at the first, a middle and the last field; sums, minima, maxima"""
    rng = np.random.default_rng((ki + 3) * 11 + vi + 3)
    lines = []
    for i in range(20000):
        k = ["", "a", "bb", "x" * 9, "y" * 10, "z" * 45, "w%d" % rng.integers(0, 500)][rng.integers(0, 7)]
        lines.append("%s,%d,%d,%s" % (k, rng.integers(-10 ** 6, 10 ** 6), rng.integers(-99, 99), k))
    P = write_files(tmp_path, [["f.csv", "\n".join(lines)]])
    got, (_s, how, detail) = run(SUM % (",", ki, ",", vi, red), P)
    assert got == python_fold(P, lambda l: l.split(",")[ki], lambda l: int(l.split(",")[vi]), binop)
    assert NEEDLE in how and "host_lines=0" in detail, (how, detail)


def test_int_keys_and_counts(engine, tmp_path):
    vals = ["0", "-0", "+0", "007", "7", "+7", "-7", "999999999999999999", "-999999999999999999", "12"]
    lines = ["%s\t%s" % (vals[i % len(vals)], vals[(i * 3) % len(vals)]) for i in range(5000)]
    P = write_files(tmp_path, [["f.tsv", "\n".join(lines)]])   # the last line has no '\n'
    got, (_s, how, _d) = run("Dampr.text(P).count(lambda l: int(l.split('\\t')[0]))", P)
    assert got == python_fold(P, lambda l: int(l.split("\t")[0]), lambda l: 1, operator.add)
    assert NEEDLE in how
    got, (_s, how, _d) = run("Dampr.text(P).map(lambda l: l.split('\\t')).fold_by(lambda r: int(r[1]), "
                             "value=lambda r: int(r[0]), binop=min)", P)
    assert got == python_fold(P, lambda l: int(l.split("\t")[1]), lambda l: int(l.split("\t")[0]), min)
    assert NEEDLE in how


def test_host_lines_and_exceptions(engine, tmp_path):
    """non-ASCII lines, int() fields only Python parses, CRLF in text mode (host) against CRLF in .gz (data)"""
    body = "".join("%s,%s\r\n" % (k, v) for k, v in [("a", " 4"), ("é", "1"), ("b", "1_0"), ("a", "+3"), ("c", "-00"),
                                                      ("b", "-999"), ("d", "5 ")] * 50)
    for name in ("f.csv", "f.csv.gz"):
        P = write_files(tmp_path, [[name, body]])
        got, (_s, how, detail) = run(SUM % (",", 0, ",", -1, "sum()"), P)
        assert got == python_fold(P, lambda l: l.split(",")[0], lambda l: int(l.split(",")[-1]), operator.add)
        assert NEEDLE in how and "host_lines=0" not in detail, (how, detail)
        got, _ = run("Dampr.text(P).count(lambda l: l.split(',')[-1])", P)
        assert got == python_fold(P, lambda l: l.split(",")[-1], lambda l: 1, operator.add)
    P = write_files(tmp_path, [["g.csv", "a,1\n" * 1000 + "b\n"]])
    with pytest.raises(IndexError):
        run(SUM % (",", 0, ",", 1, "sum()"), P)
    P = write_files(tmp_path, [["h.csv", "a,1\n" * 1000 + "b,x\n"]])
    with pytest.raises(ValueError):
        run(SUM % (",", 0, ",", 1, "sum()"), P)


def test_seams_several_files_and_long_lines(engine, tmp_path):
    """keys across the 16 KB tiles and small upload chunks, files back to back, lines past the device window"""
    engine.ingest_chunk_bytes = 1 << 20
    rng = np.random.default_rng(3)
    files = []
    for f in range(3):
        lines = []
        for i in range(60000):
            k = "k%d" % rng.integers(0, 3000)
            lines.append("%s|%s|%d" % (k, "p" * int(rng.integers(0, 60)), rng.integers(-50, 50)))
        lines[100] = "long|" + "q" * 5000 + "|3"          # longer than the 4 KB window: a host line
        lines[200] = "longer|" + "q" * 70000 + "|4"       # 64 KB or more: the whole stage goes to the host
        files.append(["p%d.txt" % f, "\n".join(lines) + ("" if f == 1 else "\n")])
    P = write_files(tmp_path, files)
    src = SUM % ("|", 0, "|", 2, "sum()")
    exp = python_fold(P, lambda l: l.split("|")[0], lambda l: int(l.split("|")[2]), operator.add)
    got, (_s, how, _d) = run(src, P)
    assert got == exp and how.startswith("host-map"), how
    for f in files:
        f[1] = f[1].replace("q" * 70000, "q" * 60000)
    (tmp_path / "b").mkdir()
    P = write_files(tmp_path / "b", files)
    exp = python_fold(P, lambda l: l.split("|")[0], lambda l: int(l.split("|")[2]), operator.add)
    got, (_s, how, detail) = run(src, P)
    assert got == exp and NEEDLE in how and "host_lines=6" in detail, (how, detail)


def test_too_many_host_lines(engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", "é,1\na,2\n" * 66000]])
    got, (_s, how, _d) = run("Dampr.text(P).count(lambda l: l.split(',')[0])", P)
    assert got == ["('a', 66000)", "('é', 66000)"] and how.startswith("host-map"), how


def test_table_regrow(engine, tmp_path):
    """more distinct keys than half the table (2^20 at the default 2^21 entries): a 4x table, one more scan"""
    n = (1 << 20) + 50000
    P = str(tmp_path / "f.csv")
    with open(P, "w") as f:
        f.write("".join("u%d,%d\n" % (i, i % 13) for i in range(n)))
        f.write("".join("u%d,1\n" % i for i in range(0, n, 97)))
    log2 = engine.text_table_log2
    got, (_s, how, detail) = run(SUM % (",", 0, ",", 1, "sum()"), P)
    assert got == python_fold(P, lambda l: l.split(",")[0], lambda l: int(l.split(",")[1]), operator.add)
    assert NEEDLE in how and engine.text_table_log2 > log2, (how, detail)


def test_overflow_bound(engine, tmp_path):
    P = write_files(tmp_path, [["f.csv", "a,999999999999999999\n" * 6 + "b,-1\n"]])
    got, (_s, how, _d) = run(SUM % (",", 0, ",", 1, "sum()"), P)
    assert got == ["('a', 5999999999999999994)", "('b', -1)"] and how.startswith("host-map"), how


def test_downstream_sort_and_sink(engine, tmp_path):
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    rng = np.random.default_rng(5)
    lines = ["%s,%d" % ("k%d" % rng.integers(0, 300), rng.integers(0, 1000)) for _ in range(30000)]
    P = write_files(tmp_path, [["f.csv", "\n".join(lines) + "\n"]])
    out = str(tmp_path / "out")
    Dampr.text(P).a_group_by(lambda l: l.split(",")[0], lambda l: int(l.split(",")[1])).sum() \
        .sort_by(lambda x: -x[1]).sink_tsv(out).run()
    assert NEEDLE in runner_mod.LAST_STATS.stages[0][1]
    rows = []
    for fn in sorted(os.listdir(out)):
        with open(os.path.join(out, fn)) as f:
            rows.extend(l.rstrip("\n").split("\t") for l in f)
    exp = {}
    for l in lines:
        k, v = l.split(",")
        exp[k] = exp.get(k, 0) + int(v)
    assert sorted((k, int(v)) for k, v in rows) == sorted(exp.items())
    assert [int(v) for _k, v in rows] == sorted(exp.values(), reverse=True)


def test_memory_and_device_texts(engine, tmp_path):
    """MemoryText (page-locked host memory) and DeviceText (HBM) inputs take the same scan"""
    from dampr_b200 import Dampr, device, plan, runner as runner_mod
    data = ("a,1\nb,2\n,3\n" * 1000 + "c,4").encode()
    pin = device.PinnedBuffer(len(data))
    pin.array[:] = np.frombuffer(data, dtype=np.uint8)
    tb = runner_mod.get_ctx().textbuf(len(data) + 64)
    tb.upload_all(data)
    for ds in (plan.MemoryText(pin.array), plan.DeviceText(tb)):
        got = sorted(repr(x) for x in Dampr.read_input(ds).a_group_by(
            lambda l: l.split(",")[0], lambda l: int(l.split(",")[1])).sum().run())
        assert got == ["('', 3000)", "('a', 1000)", "('b', 2000)", "('c', 4)"]
        assert NEEDLE in runner_mod.LAST_STATS.stages[0][1]

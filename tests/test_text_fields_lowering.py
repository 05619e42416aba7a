"""Delimited-field folds over text (`l.split(S)[i]` keys with counts and int sums / minima / maxima): the matcher
(lowering.text_fields_spec), the planner path (plan.FieldScan) on a numpy stand-in for dampr_text_fields defined
here, and the results against the REAL reference (Refefer/Dampr), whose outputs are stored in
tests/golden/text_fields.json.gz (the ReferenceReplay pattern of test_float_key_lowering.py; DAMPR_REFERENCE=<checkout>
records them again). Cases where the user's lambda raises are checked against plain Python: the reference hangs
when one of its workers raises (SURVEY B6). The same pipelines run on the device in tests/test_gpu_text_fields.py."""
import gzip
import hashlib
import json
import operator
import os
import random
import subprocess as _subprocess
import sys

import numpy as np
import pytest

REF = os.environ.get("DAMPR_REFERENCE", "")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_fields.json.gz")
NEEDLE = "device text fields scan+combine"

DRIVER = r"""
import sys, json, os, gzip, tempfile
sys.path.insert(0, sys.argv[1])
from dampr import Dampr
d = tempfile.mkdtemp()
for name, text in json.loads(sys.argv[2]):
    with (gzip.open if name.endswith(".gz") else open)(os.path.join(d, name), "wb") as f:
        f.write(text.encode("utf-8"))
P = d if len(json.loads(sys.argv[2])) > 1 else os.path.join(d, json.loads(sys.argv[2])[0][0])
print(json.dumps([sorted(repr(x) for x in eval(src).run()) for src in json.loads(sys.argv[3])]))
"""


def reference_outputs(files, srcs):
    """The reference's output records (sorted reprs) of every pipeline in srcs over the text files `files`
    ([name, text]); `P` in a pipeline is the file (one) or the directory holding them (several)."""
    args = [DRIVER, json.dumps(files), json.dumps(srcs)]
    key = hashlib.sha256("\0".join(args).encode()).hexdigest()[:20]
    runs = {}
    if os.path.exists(GOLDEN):
        with gzip.open(GOLDEN, "rb") as f:
            runs = json.loads(f.read())
    if REF:
        env = dict(os.environ)
        env.pop("PYTHONPATH", None)
        p = _subprocess.run([sys.executable, "-c", DRIVER, REF] + args[1:], capture_output=True, text=True, env=env,
                            cwd="/tmp", timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        runs[key] = p.stdout.strip().split("\n")[-1]
        with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
            f.write(json.dumps(runs, sort_keys=True).encode())
    assert key in runs, "no recorded reference output for these inputs: record with DAMPR_REFERENCE=<checkout>"
    return json.loads(runs[key])


def write_files(d, files):
    for name, text in files:
        with (gzip.open if name.endswith(".gz") else open)(os.path.join(str(d), name), "wb") as f:
            f.write(text.encode("utf-8"))
    return str(d) if len(files) > 1 else os.path.join(str(d), files[0][0])


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


# ---- numpy stand-in for dampr_text_fields ------------------------------------------------------------------------
def _int18(b):
    s = b[1:] if b[:1] in (b"+", b"-") else b
    if not (1 <= len(s) <= 18 and s.isdigit()):
        return None
    return -int(s) if b[:1] == b"-" else int(s)


def make_ctx():
    """FakeTextCtx whose tables also take dampr_text_fields (restating its header's contract with numpy)"""
    from fake_device import FakeTextCtx, FakeTable
    from dampr_b200 import device as dev

    class FieldsTable(FakeTable):
        def clear(self):
            FakeTable.clear(self)
            self.acc, self.rep, self.max_abs = {}, {}, 0

        def fields(self, tb, lo, hi, spec, cr_is_data=False):
            sep, kf, kind, vf, op = spec
            data = tb.buf[:tb.n].tobytes()
            pos = 0
            while pos < len(data):
                end = data.find(b"\n", pos)
                end = len(data) if end < 0 else end
                if lo <= pos < hi:
                    self._line(data[pos:end], pos, bytes([sep]), kf, kind, vf, op, cr_is_data)
                pos = end + 1

        def _line(self, line, off, sep, kf, kind, vf, op, cr_is_data):
            st = self.st
            f = line.split(sep)
            ok = len(line) < 4096 and all(0 < c < 0x80 for c in line) and (cr_is_data or b"\r" not in line)
            ok = ok and -len(f) <= kf < len(f) and (vf == dev.FIELD_VAL_ONE or -len(f) <= vf < len(f))
            v = 1 if vf == dev.FIELD_VAL_ONE else (_int18(f[vf]) if ok else None)
            k = f[kf] if ok else None
            if ok and kind == dev.FIELD_KEY_INT:
                k = _int18(k)
            if not ok or v is None or k is None:
                if len(line) > 0xFFFF:
                    st["flags"] |= dev.TF_LONGLINE
                elif len(self.fb) < (1 << 16):
                    self.fb.append((off << 16) | len(line))
                    st["fallback"] += 1
                else:
                    st["flags"] |= dev.TF_NONASCII
                return
            st["lines"] += 1
            st["folded"] += 1
            self.max_abs = max(self.max_abs, abs(v))
            if kind == dev.FIELD_KEY_STR and not 1 <= len(k) <= 9:
                st["hashed"] += 1
                off_k = off + sum(len(x) + 1 for x in f[:kf if kf >= 0 else len(f) + kf])
                self.rep[k] = min(self.rep.get(k, 1 << 62), (off_k << 20) | len(k))
            enc = v & ((1 << 64) - 1) if op == dev.OP_SUM_I64 else (v ^ (1 << 63)) & ((1 << 64) - 1)
            if op == dev.OP_MIN_I64:
                enc = ~enc & ((1 << 64) - 1)
            old = self.acc.get(k, 0)
            self.acc[k] = (old + enc) & ((1 << 64) - 1) if op == dev.OP_SUM_I64 else max(old, enc)

        def stats(self):
            d = dict(self.st, entries=len(self.acc), empty=self.max_abs)
            if len(self.acc) * 2 > self.capacity and len(self.acc) >= self.capacity:
                d["flags"] |= dev.TF_TABLEFULL
            return d

        def fields_stats(self):
            st = self.stats()
            return {"entries": st["entries"], "lines": st["lines"], "max_abs": st["empty"], "folded": st["folded"],
                    "flags": st["flags"], "hashed": st["hashed"], "fallback": st["fallback"]}

        def fetch(self):
            ks = list(self.acc)
            codes = np.array([(k ^ (1 << 63)) & ((1 << 64) - 1) for k in ks], dtype=np.uint64)
            return codes, np.array([self.acc[k] for k in ks], dtype=np.uint64), np.zeros(len(ks), dtype=np.uint64)

        def fetch_words(self, tb, mode, width=32, with_codes=True):
            ks = list(self.acc)
            words = np.array([k[:width] for k in ks], dtype="S%d" % width) if ks else np.zeros(0, dtype="S%d" % width)
            counts = np.array([self.acc[k] for k in ks], dtype=np.uint64)
            if not with_codes:
                return words, counts, None, None
            codes = np.array([(1 << 63 | i) if k in self.rep else i + 1 for i, k in enumerate(ks)], dtype=np.uint64)
            reps = np.array([self.rep.get(k, 0) for k in ks], dtype=np.uint64)
            return words, counts, codes, reps

    class Ctx(FakeTextCtx):
        def table(self, log2):
            return FieldsTable(self, log2)
    return Ctx()


def run_ours(src, P, monkeypatch, ctx=None):
    """records (sorted reprs) of pipeline src over path P and the stage strings of the run"""
    from fake_device import FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: ctx or make_ctx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P}).run())
    return got, [h for _s, h, _d in runner_mod.LAST_STATS.stages]


# ---- the matcher ------------------------------------------------------------------------------------------------
def _spec(key, value, split=None):
    from dampr_b200 import lowering
    return lowering.text_fields_spec(key, value, split)


def test_matcher_accepts_the_field_shapes():
    from dampr_b200.lowering import FIELD_STR, FIELD_INT
    one = lambda l: 1
    assert _spec(lambda l: l.split(",")[0], one) == (",", 0, FIELD_STR, None)
    assert _spec(lambda l: int(l.split("\t")[-2]), one) == ("\t", -2, FIELD_INT, None)
    assert _spec(lambda l: l.split(";")[3], lambda l: int(l.split(";")[-1])) == (";", 3, FIELD_STR, -1)
    assert _spec(lambda l: int(l.split("|")[1]), lambda l: int(l.split("|")[1])) == ("|", 1, FIELD_INT, 1)
    sp = lambda l: l.split(" ")
    assert _spec(lambda r: r[2], lambda r: int(r[5]), sp) == (" ", 2, FIELD_STR, 5)
    assert _spec(lambda r: int(r[-1]), one, sp) == (" ", -1, FIELD_INT, None)
    assert _spec(lambda r: r[0], lambda r: int(r[0]), sp) == (" ", 0, FIELD_STR, 0)


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
        (lambda l: l.split(",")[0], lambda l: float(l.split(",")[1]), None),
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
        got, hows = run_ours(src, P, monkeypatch)
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
    exp = reference_outputs(files, PIPELINES[name])
    P = write_files(tmp_path, files)
    for src, e in zip(PIPELINES[name], exp):
        got, hows = run_ours(src, P, monkeypatch)
        assert got == e, (name, src)
        assert NEEDLE in hows[0], (name, src, hows)


def test_the_issue_example():
    files = datasets()["issue"]
    exp = reference_outputs(files, PIPELINES["issue"])
    assert exp[0] == ["('', 7)", "('a', 8)", "('b', 6)"]


# ---- planner paths on the stand-in ------------------------------------------------------------------------------
def python_fold(path, key, value, binop):
    """plain-Python restatement: text-mode lines (universal newlines), .gz lines split at '\\n' only"""
    paths = [os.path.join(path, f) for f in sorted(os.listdir(path))] if os.path.isdir(path) else [path]
    out = {}
    for p in paths:
        if p.endswith(".gz"):
            with gzip.open(p, "rb") as f:
                lines = [l.decode("utf-8").rstrip("\n") for l in f]
        else:
            with open(p) as f:
                lines = [l.rstrip("\n") for l in f]
        for l in lines:
            k, v = key(l), value(l)
            out[k] = binop(out[k], v) if k in out else v
    return sorted(repr(x) for x in out.items())


def test_host_lines_merge_and_stats(monkeypatch, tmp_path):
    """lines the device hands back (non-ASCII, CR, int() fields only Python parses) are folded on the host and
    merged; the stats line counts them"""
    text = "a,1\nb, 2\né,3\na,4\r\nb,1_0\nc,+7\n"
    P = write_files(tmp_path, [["f.csv", text]])
    for binop, red in ((operator.add, "sum()"), (min, "reduce(min)"), (max, "reduce(max)")):
        src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).%s" % red
        got, hows = run_ours(src, P, monkeypatch)
        assert got == python_fold(P, lambda l: l.split(",")[0], lambda l: int(l.split(",")[1]), binop), red
        assert NEEDLE in hows[0]
    from dampr_b200 import runner as runner_mod
    detail = runner_mod.LAST_STATS.stages[0][2]
    assert "host_lines=4" in detail and "lines=6" in detail and "groups=4" in detail, detail


def test_min_max_identities(monkeypatch, tmp_path):
    """MIN / MAX start from their identity, not from the cleared 0: all-positive minima, all-negative maxima"""
    P = write_files(tmp_path, [["f.csv", "a,5\na,9\nb,-3\nb,-8\nc,0\n"]])
    got, _ = run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], lambda r: int(r[1]))"
                      ".reduce(min)", P, monkeypatch)
    assert got == ["('a', 5)", "('b', -8)", "('c', 0)"]
    got, _ = run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: r[0], lambda r: int(r[1]))"
                      ".reduce(max)", P, monkeypatch)
    assert got == ["('a', 9)", "('b', -3)", "('c', 0)"]


def test_empty_key_and_int_key_equality(monkeypatch, tmp_path):
    """'' is a key (blank lines, empty fields); 007, 7 and +7 are one int key, -0 and 0 another"""
    P = write_files(tmp_path, [["f.csv", "\n,1\n007,1\n7,2\n+7,3\n-0,4\n0,5\n"]])
    got, hows = run_ours("Dampr.text(P).count(lambda l: l.split(',')[0])", P, monkeypatch)
    assert got == ["('', 2)", "('+7', 1)", "('-0', 1)", "('0', 1)", "('007', 1)", "('7', 1)"]
    with pytest.raises(ValueError):     # int('') of the blank line: the user's own exception
        run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: int(r[0]), "
                 "lambda r: int(r[-1])).sum()", P, monkeypatch)
    P = write_files(tmp_path, [["g.csv", "007,1\n7,2\n+7,3\n-0,4\n0,5\n"]])
    got, hows = run_ours("Dampr.text(P).map(lambda l: l.split(',')).a_group_by(lambda r: int(r[0]), "
                         "lambda r: int(r[1])).sum()", P, monkeypatch)
    assert got == ["(0, 9)", "(7, 6)"] and NEEDLE in hows[0]


def test_overflow_bound_refuses_and_the_host_sums_exactly(monkeypatch, tmp_path):
    """records x max|v| >= 2^62: the device sum is refused, the host path gives Python's unbounded sum"""
    P = write_files(tmp_path, [["f.csv", "".join("a,999999999999999999\n" for _ in range(10)) + "b,1\n"]])
    src = "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).sum()"
    got, hows = run_ours(src, P, monkeypatch)
    assert got == ["('a', 9999999999999999990)", "('b', 1)"]
    assert NEEDLE not in hows[0] and hows[0].startswith("host-map"), hows
    # a 19-digit value is the host's (Python int): its sum is checked with the same bound
    P = write_files(tmp_path, [["g.csv", "a,1234567890123456789\na,1234567890123456789\na,1234567890123456789\n"
                                         "a,1234567890123456789\n"]])
    got, hows = run_ours(src, P, monkeypatch)
    assert got == ["('a', 4938271560493827156)"] and NEEDLE not in hows[0]
    P = write_files(tmp_path, [["h.csv", "a,1234567890123456789\nb,-5\n"]])
    got, hows = run_ours(src, P, monkeypatch)
    assert got == ["('a', 1234567890123456789)", "('b', -5)"] and NEEDLE in hows[0]


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
    got, hows = run_ours("Dampr.text(P).count(lambda l: l.split(',')[0])", P, monkeypatch)
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
    got, hows = run_ours(src, P, monkeypatch)
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

"""Shared helpers of the delimited-field tests (test_text_fields_lowering.py, test_text_fields_float_lowering.py and
their GPU twins): the REAL reference's recorded outputs, plain-Python restatements of a field fold, and a numpy
stand-in for dampr_text_fields and dampr_text_fields_records that restates include/dampr_b200.h.

tests/text_contract.py restates the same contract on its own, on purpose: it is the independent oracle the kernel
seam tests compare against."""
import gzip
import hashlib
import json
import math
import os
import re
import struct
import subprocess as _subprocess
import sys

import numpy as np

REF = os.environ.get("DAMPR_REFERENCE", "")

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


def reference_outputs(files, srcs, golden):
    """The reference's output records (sorted reprs) of every pipeline in srcs over the text files `files`
    ([name, text]), as stored in the gzipped JSON file `golden`; `P` in a pipeline is the file (one) or the directory
    holding them (several). DAMPR_REFERENCE=<checkout> runs the reference and records them again."""
    args = [DRIVER, json.dumps(files), json.dumps(srcs)]
    key = hashlib.sha256("\0".join(args).encode()).hexdigest()[:20]
    runs = {}
    if os.path.exists(golden):
        with gzip.open(golden, "rb") as f:
            runs = json.loads(f.read())
    if REF:
        env = dict(os.environ)
        env.pop("PYTHONPATH", None)
        p = _subprocess.run([sys.executable, "-c", DRIVER, REF] + args[1:], capture_output=True, text=True, env=env,
                            cwd="/tmp", timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        runs[key] = p.stdout.strip().split("\n")[-1]
        with gzip.GzipFile(golden, "wb", mtime=0) as f:
            f.write(json.dumps(runs, sort_keys=True).encode())
    assert key in runs, "no recorded reference output for these inputs: record with DAMPR_REFERENCE=<checkout>"
    return json.loads(runs[key])


def write_files(d, files):
    for name, text in files:
        with (gzip.open if name.endswith(".gz") else open)(os.path.join(str(d), name), "wb") as f:
            f.write(text.encode("utf-8"))
    return str(d) if len(files) > 1 else os.path.join(str(d), files[0][0])


# ---- plain Python -----------------------------------------------------------------------------------------------
def python_lines(path):
    """the reader's lines: text-mode files with universal newlines, .gz files split at '\\n' only"""
    paths = [os.path.join(path, f) for f in sorted(os.listdir(path))] if os.path.isdir(path) else [path]
    out = []
    for p in paths:
        if p.endswith(".gz"):
            with gzip.open(p, "rb") as f:
                out += [l.decode("utf-8").rstrip("\n") for l in f]
        else:
            with open(p) as f:
                out += [l.rstrip("\n") for l in f]
    return out


def python_fold(path, key, value, binop):
    """plain-Python restatement of a field fold over the reader's lines: sorted reprs of its (key, value) records"""
    out = {}
    for l in python_lines(path):
        k, v = key(l), value(l)
        out[k] = binop(out[k], v) if k in out else v
    return sorted(repr(x) for x in out.items())


# ---- numpy stand-in for dampr_text_fields and dampr_text_fields_records -----------------------------------------
GRAMMAR = re.compile(rb"[ \t]*[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?[ \t]*\Z")
M64 = (1 << 64) - 1


def parse_f64(b):
    """the header's float() rule: Python's value of the strings the device takes, else None"""
    m = GRAMMAR.match(b)
    if not m or len(m.group(1).replace(b".", b"").lstrip(b"0")) > 19:
        return None
    return float(b)


def _int18(b):
    """the header's int() rule: [+-]?[0-9]{1,18}, else None"""
    s = b[1:] if b[:1] in (b"+", b"-") else b
    if not (1 <= len(s) <= 18 and s.isdigit()):
        return None
    return -int(s) if b[:1] == b"-" else int(s)


def device_takes(line, cr_is_data):
    """the header's rule of the lines a field scan may take: under 4 KB, ASCII without NUL, no text-mode '\\r'"""
    return len(line) < 4096 and all(0 < c < 0x80 for c in line) and (cr_is_data or b"\r" not in line)


def plain_line(line, f, kf, kind, vf, flt, cr_is_data):
    """(key, value) the plain scan folds for a line whose fields are f (bytes), or None for a line it hands to the
    host: a str key is bytes, an int key an int; the value 1 (vf FIELD_VAL_ONE), a float (flt) or an int"""
    from dampr_b200 import device as dev
    ok = device_takes(line, cr_is_data) and -len(f) <= kf < len(f) and \
        (vf == dev.FIELD_VAL_ONE or -len(f) <= vf < len(f))
    if not ok:
        return None
    v = 1 if vf == dev.FIELD_VAL_ONE else parse_f64(f[vf]) if flt else _int18(f[vf])
    k = _int18(f[kf]) if kind == dev.FIELD_KEY_INT else f[kf]
    return None if v is None or k is None else (k, v)


def f64_bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def make_ctx(free_bytes=1 << 30):
    """FakeTextCtx whose tables also take dampr_text_fields (TABLE mode: SUM / MIN / MAX of I64, MIN / MAX of F64) and
    dampr_text_fields_records (RECORDS mode: SUM of I64 or F64), and whose kv buffers count against `free_bytes`"""
    from fake_device import FakeTextCtx, FakeTable, FakeKV
    from dampr_b200 import device as dev

    class RecKV(FakeKV):
        """a kv whose buffers count against the context's free memory, as device allocations do"""
        def __init__(self, ctx, capacity):
            FakeKV.__init__(self, ctx, capacity)
            ctx.live[id(self)] = 16 * capacity

        def set_size(self, n):
            assert n <= len(self.rec)
            self.n = int(n)

        def sort_reduce(self, op, xform, sorted_run=False):
            # dampr_kv_sort_reduce: a scratch copy at the capacity and an output of n records, or DAMPR_ERR_NOMEM
            if 16 * (len(self.rec) + self.n) > self.ctx.mem_info()[0]:
                raise dev.DeviceError("libdampr_b200 status -3: out of device memory")
            return FakeKV.sort_reduce(self, op, xform, sorted_run)

        def free(self):
            self.ctx.live.pop(id(self), None)

    class FieldsTable(FakeTable):
        def clear(self):
            FakeTable.clear(self)
            self.acc, self.rep, self.code, self.max_abs = {}, {}, {}, 0

        def _scan(self, tb, lo, hi, spec, cr_is_data, rec):
            sep, kf, kind, vf, op = spec
            data = tb.buf[:tb.n].tobytes()
            pos = 0
            while pos < len(data):
                end = data.find(b"\n", pos)
                end = len(data) if end < 0 else end
                if lo <= pos < hi:
                    self._line(data[pos:end], pos, bytes([sep]), kf, kind, vf, op, cr_is_data, rec)
                pos = end + 1

        def fields(self, tb, lo, hi, spec, cr_is_data=False):
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_MIN_I64, dev.OP_MAX_I64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            self._scan(tb, lo, hi, spec, cr_is_data, None)

        def fields_records(self, tb, lo, hi, spec, kv, cr_is_data=False):
            assert spec[4] in (dev.OP_SUM_I64, dev.OP_SUM_F64)
            self._scan(tb, lo, hi, spec, cr_is_data, kv)

        def _line(self, line, off, sep, kf, kind, vf, op, cr_is_data, rec):
            st = self.st
            f = line.split(sep)
            flt = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
            kv = plain_line(line, f, kf, kind, vf, flt, cr_is_data)
            if kv is None:
                if len(line) > 0xFFFF:
                    st["flags"] |= dev.TF_LONGLINE
                elif len(self.fb) < (1 << 16):
                    self.fb.append((off << 16) | len(line))
                    st["fallback"] += 1
                else:
                    st["flags"] |= dev.TF_NONASCII
                if rec is not None:
                    self._put(rec, 0, 0)
                return
            k, v = kv
            st["lines"] += 1
            st["folded"] += 1
            if flt and v == 0 and math.copysign(1.0, v) < 0:
                st["flags"] |= dev.TF_NEGZERO
            if not flt:
                self.max_abs = max(self.max_abs, abs(v))
            if kind == dev.FIELD_KEY_STR and not 1 <= len(k) <= 9:
                st["hashed"] += 1
                off_k = off + sum(len(x) + 1 for x in f[:kf if kf >= 0 else len(f) + kf])
                self.rep[k] = min(self.rep.get(k, 1 << 62), (off_k << 20) | len(k))
            if k not in self.code:
                i = len(self.code)
                self.code[k] = ((k ^ (1 << 63)) & M64 if kind == dev.FIELD_KEY_INT else
                                (1 << 63 | i) if kind == dev.FIELD_KEY_STR and not 1 <= len(k) <= 9 else i + 1)
            if rec is not None:
                self._put(rec, self.code[k], f64_bits(v) if flt else v & M64)
                self.acc[k] = self.acc.get(k, 0) + 1
                return
            if flt:
                b = f64_bits(v)
                enc = b ^ (M64 if b >> 63 else 1 << 63)
            else:
                enc = v & M64 if op == dev.OP_SUM_I64 else (v ^ (1 << 63)) & M64
            if op in (dev.OP_MIN_I64, dev.OP_MIN_F64):
                enc = ~enc & M64
            old = self.acc.get(k, 0)
            self.acc[k] = (old + enc) & M64 if op == dev.OP_SUM_I64 else max(old, enc)

        def _put(self, kv, code, bits):
            i = self.st["raw"]
            self.st["raw"] += 1
            if i < len(kv.rec):
                kv.rec[i] = (code, bits)
            else:
                self.st["flags"] |= dev.TF_RECFULL

        def stats(self):
            d = dict(self.st, entries=len(self.acc), empty=self.max_abs)
            if len(self.acc) * 2 > self.capacity and len(self.acc) >= self.capacity:
                d["flags"] |= dev.TF_TABLEFULL
            return d

        def fields_stats(self):
            st = self.stats()
            return {"entries": st["entries"], "lines": st["lines"], "max_abs": st["empty"], "folded": st["folded"],
                    "flags": st["flags"], "hashed": st["hashed"], "fallback": st["fallback"], "records": st["raw"]}

        def fetch(self):
            ks = list(self.acc)
            return (np.array([self.code[k] for k in ks], dtype=np.uint64),
                    np.array([self.acc[k] for k in ks], dtype=np.uint64), np.zeros(len(ks), dtype=np.uint64))

        def fetch_words(self, tb, mode, width=32, with_codes=True):
            ks = list(self.acc)
            words = np.array([k[:width] for k in ks], dtype="S%d" % width) if ks else np.zeros(0, dtype="S%d" % width)
            counts = np.array([self.acc[k] for k in ks], dtype=np.uint64)
            if not with_codes:
                return words, counts, None, None
            codes = np.array([self.code[k] for k in ks], dtype=np.uint64)
            reps = np.array([self.rep.get(k, 0) for k in ks], dtype=np.uint64)
            return words, counts, codes, reps

    class Ctx(FakeTextCtx):
        live = None

        def table(self, log2):
            return FieldsTable(self, log2)

        def kv(self, capacity):
            return RecKV(self, capacity)

        def mem_info(self):
            return (free_bytes - sum(self.live.values()), 1 << 34)
    c = Ctx()
    c.live = {}
    return c


def run_ours(src, P, monkeypatch, ctx=None):
    """(records (sorted reprs) of pipeline src over path P, the stage strings of the run, its (stage, how, detail)
    triples) on the stand-in"""
    from fake_device import FakePinned
    from dampr_b200 import Dampr, settings, plan
    from dampr_b200 import runner as runner_mod
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: ctx or make_ctx()})
    monkeypatch.setattr(plan, "_pinned_ring", lambda n, b: [FakePinned(b) for _ in range(n)])
    monkeypatch.setattr(plan, "_BUFFERS", {})
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P}).run())
    return got, [h for _s, h, _d in runner_mod.LAST_STATS.stages], runner_mod.LAST_STATS.stages

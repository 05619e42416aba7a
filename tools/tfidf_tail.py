"""Where the serial tail of the TF-IDF step goes:
python tools/tfidf_tail.py [--gb 10] [--steps 5] [--warmup 2] [--source resident|host]

Runs bench.tfidf_job on text already resident in HBM (the bench's corpus: Zipf(1.1), V = 1e6, seed 1234) and reports
the wall milliseconds of every phase after the tokenise kernel. Each phase is a call of the engine wrapped here and
closed by a device synchronise, so a phase holds its own kernels and copies and nothing of its neighbours':

  tokenise            the tokenise+combine kernel (not part of the tail; for scale)
  stats               the table's counters (a 64-byte download)
  extract_decode      the table extract + word decode kernel (its CUDA-event time)
  download            words and counts to the host (fetch_words wall time minus the kernel)
  df_dictionary       distinct document frequencies, their inverse and one row each
  idf_eval            the rest of the cross stage: the idf of every distinct document frequency
  sink                the native sink: dictionary formatting, row formatting and the part-file writes
  rewrite             not part of the step, for scale: the same bytes written once more afterwards from Python, one
                      thread per file
  sink.*              the library's own host clocks inside that sink call (dampr_host_sink_timings): dictionary
                      preparation on the calling thread, then the largest value any writer thread saw for its start
                      delay, open(), row formatting, write() and close()
  other               the step's wall time minus every phase above: Python planning, frames, stage glue

--source host takes the text from page-locked host memory, as the headline does. The chunked upload and the tokenise
launches that trail it are then one phase, `ingest`, which ends when the table's counters have arrived (the first
point at which the host knows the last launch is done); `tokenise` and `stats` are not reported apart, and the tail
is everything after `ingest`.

The step times printed last are taken without the wrappers. Prints one JSON line on stdout."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

import numpy as np

import bench
from dampr_b200 import Dampr, synth
from dampr_b200 import device as dev
from dampr_b200 import plan
from dampr_b200 import runner as runner_mod
from dampr_b200.plan import DeviceText, MemoryText


def gpu_name_and_power():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


class Phases(object):
    """Wraps engine calls: every call runs between two device synchronises and its wall time is added to a phase."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.ms = {}
        self.saved = []

    def add(self, name, ms):
        self.ms[name] = self.ms.get(name, 0.0) + ms

    def wrap(self, owner, attr, name):
        fn = getattr(owner, attr, None)
        if fn is None:
            return
        self.saved.append((owner, attr, fn))
        ph = self

        def timed(*a, **kw):
            ph.ctx.sync()
            t0 = time.perf_counter()
            try:
                return fn(*a, **kw)
            finally:
                ph.ctx.sync()
                ph.add(name, 1e3 * (time.perf_counter() - t0))
        setattr(owner, attr, timed)

    def install(self, host):
        if host:
            self.wrap(plan.TextScan, "_ingest", "ingest")
        else:
            self.wrap(dev.Table, "count", "tokenise")
            self.wrap(dev.Table, "stats", "stats")
        self.wrap(dev.Table, "fetch_words", "fetch_words")
        # the df dictionary: built on the host, or handed over from the device (Ctx.count_dictionary)
        self.wrap(plan, "unique_inverse_rows", "df_dictionary")
        self.wrap(plan, "_lower_cross", "cross")
        self.wrap(dev, "host_join_tsv", "sink")

    def uninstall(self):
        for owner, attr, fn in reversed(self.saved):
            setattr(owner, attr, fn)
        self.saved = []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=10.0)
    ap.add_argument("--vocab", type=int, default=1000000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--source", choices=("resident", "host"), default="resident")
    args = ap.parse_args()
    host = args.source == "host"

    ctx = runner_mod.get_ctx()
    vocab, cdf = synth.make_vocab(args.vocab), synth.make_cdf(args.vocab)
    tb = ctx.synth_text(1234, int(int(args.gb * 1e9) / bench.MEAN_LINE), vocab[0], vocab[1], cdf)
    if host:
        pin = dev.PinnedBuffer(tb.n)
        ctx.check(ctx.lib.dampr_textbuf_download(ctx.h, tb.h, 0, pin.array.ctypes.data, tb.n))
        source = MemoryText(pin.array[:tb.n])
    else:
        source = DeviceText(tb)
    out_root = tempfile.mkdtemp(prefix="dampr_tail_")
    rctx = runner_mod.get_ctx()

    def step(i, keep=False):
        d = os.path.join(out_root, "o%d" % i)
        t0 = time.perf_counter()
        bench.tfidf_job(Dampr, source, d)
        ms = 1e3 * (time.perf_counter() - t0)
        if not keep:
            shutil.rmtree(d, ignore_errors=True)
        return ms, d

    def rewrite(d):
        """wall ms of writing the part files of `d` once more (same sizes, one thread per file)"""
        from concurrent.futures import ThreadPoolExecutor
        blobs = []
        for fn in sorted(os.listdir(d)):
            with open(os.path.join(d, fn), "rb") as f:
                blobs.append(f.read())
        shutil.rmtree(d, ignore_errors=True)
        os.makedirs(d)

        def write(j):
            fd = os.open(os.path.join(d, "part-%d" % j), os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
            try:
                mv = memoryview(blobs[j])
                while len(mv):
                    mv = mv[os.write(fd, mv):]
            finally:
                os.close(fd)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(len(blobs)) as ex:
            list(ex.map(write, range(len(blobs))))
        ms = 1e3 * (time.perf_counter() - t0)
        shutil.rmtree(d, ignore_errors=True)
        return ms, sum(len(b) for b in blobs)

    try:
        for i in range(args.warmup):
            step(-1 - i)
        rctx.timing_enable(True)
        rows = []
        for i in range(args.steps):
            ph = Phases(rctx)
            ph.install(host)
            rctx.timings_reset()
            try:
                total, d = step(i, keep=True)
            finally:
                ph.uninstall()
            extract = sum(ms for name, ms in rctx.timings() if name == "table_extract")
            write, out_bytes = rewrite(d)
            sink_split = dev.host_sink_timings()
            m = ph.ms
            head = "ingest" if host else "tokenise"
            r = {head: m.get(head, 0.0)}
            if not host:
                r["stats"] = m.get("stats", 0.0)
            r.update({"extract_decode": extract,
                      "download": m.get("fetch_words", 0.0) - extract, "df_dictionary": m.get("df_dictionary", 0.0),
                      "idf_eval": m.get("cross", 0.0) - m.get("df_dictionary", 0.0),
                      "sink": m.get("sink", 0.0)})
            r["tail"] = sum(v for k, v in r.items() if k != head)
            r["other"] = total - r[head] - r["tail"]
            r["tail_with_other"] = total - r[head]
            r["rewrite"] = write
            r.update(("sink." + k, v) for k, v in sink_split.items())
            r["step_profiled"] = total
            rows.append(r)
        plain = [step(100 + i)[0] for i in range(args.steps)]
    finally:
        shutil.rmtree(out_root, ignore_errors=True)
    keys = list(rows[0])
    med = {k: round(float(np.median([r[k] for r in rows])), 2) for k in keys}
    print("phase            median ms   (every step)", file=sys.stderr)
    for k in keys:
        print("  %-16s %8.2f   %s" % (k, med[k], [round(r[k], 1) for r in rows]), file=sys.stderr)
    print("  gpu: %s" % gpu_name_and_power(), file=sys.stderr)
    print("  step (no wrappers) %s ms" % [round(x, 1) for x in plain], file=sys.stderr)
    print(json.dumps({"gpu": gpu_name_and_power(), "source": args.source, "gb": args.gb, "vocab": args.vocab,
                      "steps": args.steps,
                      "median_ms": med, "step_ms_unwrapped": [round(x, 2) for x in plain],
                      "sink_bytes": out_bytes}))
    return 0


if __name__ == "__main__":
    sys.exit(main())

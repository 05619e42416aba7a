"""Delimited-field fold benchmark: `map(l.split(",")).fold_by(r[0], int(r[2]), +)` over seeded CSV text.

Prints one JSON line: the card and its power limit (read in the same run), the bytes scanned, the field kernel's time
from CUDA events (dampr_ctx_timings, DAMPR_K_TEXT_FIELDS) with its GB/s and share of the HBM data-sheet bandwidth
(the kernel needs 1 byte read per input byte), end-to-end MB/s from page-locked memory (MemoryText) and from a
page-cache-warm file, the host-map MB/s on a sample, and whether the device and the host results agree there.

    python tools/fields_bench.py [--gb 2] [--keys 1000000] [--reps 3] [--sample-mb 32] [--out DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s
LINE = 100           # bytes per line: "u%07d," key, an 83-letter field, ",%+06d" value, '\n'


def csv_text(seed, n_lines, n_keys):
    """n_lines seeded CSV lines of LINE bytes: key u0000000..u{n_keys-1} (uniform), a lowercase filler field, a
    signed 5-digit value"""
    rng = np.random.default_rng(seed)
    out = np.empty((n_lines, LINE), dtype=np.uint8)
    keys = rng.integers(0, n_keys, size=n_lines)
    out[:, 0] = ord("u")
    for p in range(7):
        out[:, 7 - p] = 48 + (keys // 10 ** p) % 10
    out[:, 8] = ord(",")
    out[:, 9:92] = rng.integers(97, 123, size=(n_lines, 83), dtype=np.uint8)
    out[:, 92] = ord(",")
    vals = rng.integers(-99999, 100000, size=n_lines)
    out[:, 93] = np.where(vals < 0, ord("-"), ord("+"))
    av = np.abs(vals)
    for p in range(5):
        out[:, 98 - p] = 48 + (av // 10 ** p) % 10
    out[:, 99] = ord("\n")
    return out.reshape(-1)


def job(Dampr, src):
    return Dampr.read_input(src).map(lambda l: l.split(",")) \
        .fold_by(lambda r: r[0], value=lambda r: int(r[2]), binop=lambda a, b: a + b)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return q[0], q[1]
    except Exception as e:   # the numbers are still the device's; say what could not be read
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--keys", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample-mb", type=float, default=32)
    ap.add_argument("--out", default=None, help="directory for the text file (default: a temporary one)")
    a = ap.parse_args()

    from dampr_b200 import Dampr, device as dev, plan
    from dampr_b200 import runner as runner_mod
    ctx = runner_mod.get_ctx()
    name, power = card()
    n_lines = int(a.gb * 1e9) // LINE
    text = csv_text(2026, n_lines, a.keys)
    nbytes = len(text)
    pin = dev.PinnedBuffer(nbytes)
    pin.array[:] = text
    tmpdir = a.out or tempfile.mkdtemp(prefix="fields_bench_")
    path = os.path.join(tmpdir, "events.csv")
    text.tofile(path)
    del text

    def timed(src):
        ctx.timings_reset()
        t0 = time.perf_counter()
        n = len(list(job(Dampr, src).run()))
        dt = time.perf_counter() - t0
        stages = runner_mod.LAST_STATS.stages
        assert "device text fields scan+combine" in stages[0][1], stages
        ms = sum(m for k, m in ctx.timings() if k == "text_fields")
        return dt, ms, n, stages[0][2]

    ctx.timing_enable(True)
    timed(plan.MemoryText(pin.array))          # warm-up: module load, buffers, table size
    mem = [timed(plan.MemoryText(pin.array)) for _ in range(a.reps)]
    with open(path, "rb") as f:                # page cache warm
        while f.read(64 << 20):
            pass
    from dampr_b200.inputs import PathInput
    fil = [timed(PathInput(path)) for _ in range(a.reps)]
    ctx.timing_enable(False)

    # host map on a sample: the stage as plain Python (the same lambdas), and the device result of the same bytes
    sample_lines = max(1, int(a.sample_mb * 1e6) // LINE)
    sample = pin.array[:sample_lines * LINE].tobytes()
    t0 = time.perf_counter()
    host = {}
    for l in sample.decode("ascii").split("\n")[:-1]:
        r = l.split(",")
        k, v = r[0], int(r[2])
        host[k] = host[k] + v if k in host else v
    host_s = time.perf_counter() - t0
    spin = dev.PinnedBuffer(len(sample))
    spin.array[:] = np.frombuffer(sample, dtype=np.uint8)
    got = dict(job(Dampr, plan.MemoryText(spin.array)).run())

    kernel_ms = min(m[1] for m in mem)
    res = {
        "bench": "text_fields",
        "card": name, "power_limit": power,
        "bytes": nbytes, "lines": n_lines, "distinct_keys": mem[0][2],
        "kernel_ms": round(kernel_ms, 3),
        "kernel_GBps": round(nbytes / kernel_ms / 1e6, 1),
        "kernel_share_of_hbm_peak": round(nbytes / (kernel_ms / 1e3) / HBM_PEAK, 4),
        "e2e_pinned_MBps": round(nbytes / min(m[0] for m in mem) / 1e6, 1),
        "e2e_pinned_s": [round(m[0], 3) for m in mem],
        "e2e_file_warm_MBps": round(nbytes / min(f[0] for f in fil) / 1e6, 1),
        "e2e_file_warm_s": [round(f[0], 3) for f in fil],
        "file_kernel_ms": round(min(f[1] for f in fil), 3),
        "host_map_MBps": round(len(sample) / host_s / 1e6, 1),
        "host_sample_bytes": len(sample),
        "sample_equal": got == host,
        "stats": mem[0][3],
    }
    if a.out is None:
        shutil.rmtree(tmpdir, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

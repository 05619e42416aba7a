"""Delimited-field fold benchmark: `map(l.split(",")).fold_by(r[0], int(r[2]), +)` over seeded CSV text.

Prints one JSON line: the card and its power limit (read in the same run), the bytes scanned, the field kernel's time
from CUDA events (dampr_ctx_timings, DAMPR_K_TEXT_FIELDS) with its GB/s and share of the HBM data-sheet bandwidth
(the kernel needs 1 byte read per input byte), end-to-end MB/s from page-locked memory (MemoryText) and from a
page-cache-warm file, the host-map MB/s on a sample, and whether the device and the host results agree there.

    python tools/fields_bench.py [--gb 2] [--keys 1000000] [--reps 3] [--sample-mb 32] [--out DIR]
                                 [--value int|float] [--op sum|min|max|mean] [--where none|str|int|float|set|contains|prefix|or|line]
                                 [--sep comma|ws] [--key-fields 1|2|3] [--expr none|product|ratio|nfields]
                                 [--key field|const|bucket]

--value float writes the value field as float text (even lines "%.6f", odd lines repr() of the double, right-aligned
in a 24-byte field) and folds float(r[2]); --op picks `+` (fold_by), min / max (a_group_by().reduce) or mean(). A run
other than the default also reports every kernel's time by name (the record modes' count pass, fold and sort), and
for float sums and means whether the sample agrees with Python within 4·n·2^-53·Σ|v| per key (plus one rounding for
a mean); the default run prints exactly the fields it always printed.

--where adds one `filter` in front of the fold and runs the stage both ways in the same invocation: the unfiltered
figures under their usual names, the filtered ones as where_* (kernel ms and GB/s over the same bytes, end-to-end
MB/s, the stats line with filtered=N, and whether the host-map sample of the filtered stage agrees). The filters:
  str    r[0] < 'u0500000'        (about half the lines at the default --keys)
  int    int(r[2]) >= 0           (the signed value field: about half; --value int only)
  float  float(r[2]) >= 0         (about half)
  set    r[0] not in <64 keys>    (keeps almost every line: each one is compared with all 64 members)
  contains  'ab' in l             (a substring of the whole line, in front of the split: about one line in nine)
  prefix    not r[1].startswith('x')                   (about 25 lines in 26)
  or        r[0] < 'u0500000' or float(r[2]) >= 0      (about three quarters)
  line      l.startswith('u0') and len(l) > 90         (every line at the default --keys, in front of the split)

--sep ws writes the same rows with their fields joined by runs of 1-3 spaces or tabs instead of commas, a blank in
front of about a quarter of them and behind another quarter (the filler field gives up the bytes, so every line keeps
its LINE bytes), and runs the same pipelines with `l.split()`. The JSON line then also holds "sep": "ws".

--key-fields 2 groups by the tuple (r[0], r[1]) and 3 by (r[0], r[1], r[-3]) (the key field again, counted from
the end). The filler field then holds one of two strings (a lowercase run with 'a' or 'b' in its middle), so a tuple
key has about twice as many groups as the single key (under --sep ws the filler's length also varies with the blank
runs around it, which multiplies the groups; "distinct_keys" says how many). It works with every other option of the CSV rows, and the JSON
line also holds "key_fields" and "fetch_to_frame_ms" (the time from the table fetch to the key column of Python
tuples, best run).

--expr and --key fold computed values and keys (the expression builds of the field kernel). product and ratio carve a
quantity field of 1-999 ("%03d") out of the filler, behind the value, so every line keeps its LINE bytes and
r[2] is the value, r[3] the quantity:
  product  int(r[2]) * int(r[3])
  ratio    int(r[2]) / int(r[3])      (a float value)
  nfields  map(lambda l: len(l.split())) in front of the keyed functions, the README's stage; --key const only
--key const groups everything under `lambda r: 1`, bucket under int(r[2]) // 1000 (about 200 keys), field under r[0]
(the default). They take --sep comma and ws (nfields: ws only), --op, and --value int; the JSON line then also holds
"expr" and "key", and whether the host-map sample agrees (float values: within the sum bound above).

--format json writes JSON lines of JLINE bytes instead: {"user": "u%07d", "n": int, "status": an int or a string,
"latency": float, "meta": {"user": "decoy", ...}, "pad": filler}, padded with JSON whitespace after the numbers, and
runs `Dampr.json`-style stages: `map(json.loads).fold_by(r["user"], value=r["n"], +)` (--value float:
float(r["latency"])), min / max / mean() the same way. The host-map rate is then json.loads plus the lambdas. The JSON
line holds "format": "json"; --where is not taken. --nested moves the key and the value one or two levels down:
{"user": {"id": "u%07d"}, "stats": {"n": int, "status": .., "latency": float}, "meta": {"user": {"id": "decoy"}, ..},
"pad": filler}, read as r["user"]["id"] and r["stats"]["n"] (float(r["stats"]["latency"])), and adds "nested": true.
"""
import argparse
import json
import os
import random
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


FVAL = 24           # bytes of the float value field (--value float)


def float_text(seed, n_lines, n_keys):
    """the same layout with a 24-byte float value field: key, a 65-letter filler field, the value right-aligned in
    spaces (Python's float() takes them), '\n'; even lines "%.6f", odd lines repr()"""
    rng = np.random.default_rng(seed)
    out = np.empty((n_lines, LINE), dtype=np.uint8)
    keys = rng.integers(0, n_keys, size=n_lines)
    out[:, 0] = ord("u")
    for p in range(7):
        out[:, 7 - p] = 48 + (keys // 10 ** p) % 10
    out[:, 8] = ord(",")
    vstart = LINE - 1 - FVAL
    out[:, 9:vstart - 1] = rng.integers(97, 123, size=(n_lines, vstart - 10), dtype=np.uint8)
    out[:, vstart - 1] = ord(",")
    vals = rng.uniform(-1e5, 1e5, size=n_lines)
    step = 1 << 20
    for a in range(0, n_lines, step):
        v = vals[a:a + step].tolist()
        s = [("%.6f" % x if (a + i) % 2 == 0 else repr(x)).rjust(FVAL) for i, x in enumerate(v)]
        out[a:a + len(s), vstart:LINE - 1] = np.frombuffer("".join(s).encode("ascii"), dtype=np.uint8).reshape(-1, FVAL)
    out[:, LINE - 1] = ord("\n")
    return out.reshape(-1)


def whitespace_rows(text, seed, vwidth):
    """the rows of csv_text / float_text (value field of vwidth bytes) rewritten in place with whitespace runs for
    separators: [blank?] key [1-3 blanks] filler [1-3 blanks] value [blank?] '\n', LINE bytes each"""
    rows = text.reshape(-1, LINE)
    rng = np.random.default_rng(seed)
    step = 1 << 20
    for a in range(0, len(rows), step):
        t = rows[a:a + step]
        n = len(t)
        key, val = t[:, 0:8].copy(), t[:, LINE - 1 - vwidth:LINE - 1].copy()
        lead = (rng.random(n) < 0.25).astype(np.int64)
        trail = ((rng.random(n) < 0.33) & (lead == 0)).astype(np.int64)
        r1, r2 = rng.integers(1, 4, size=n), rng.integers(1, 4, size=n)
        blank = np.array([ord(" "), ord("\t")], dtype=np.uint8)
        i = np.arange(n)
        t[:, 0] = np.where(lead == 1, ord(" "), t[:, 0])
        for j in range(8):
            t[i, lead + j] = key[:, j]
        for j in range(3):
            m = j < r1
            t[i[m], (lead + 8 + j)[m]] = blank[rng.integers(0, 2, size=int(m.sum()))]
        vstart = LINE - 1 - trail - vwidth
        for j in range(vwidth):
            t[i, vstart + j] = val[:, j]
        for j in range(1, 4):
            m = j <= r2
            t[i[m], (vstart - j)[m]] = blank[rng.integers(0, 2, size=int(m.sum()))]
        t[:, LINE - 2] = np.where(trail == 1, ord(" "), t[:, LINE - 2])
    return text


JLINE = 176         # bytes per JSON line (--format json)


JROW = '{"user":"u0000000","n":%s,"status":%s,"latency":%s,"meta":{"user":"decoy","ids":[%d,%d]},"pad":"'
JROW_NESTED = '{"user":{"id":"u0000000"},"stats":{"n":%s,"status":%s,"latency":%s},' \
    '"meta":{"user":{"id":"decoy"},"ids":[%d,%d]},"pad":"'


def json_text(seed, n_lines, n_keys, nested=False):
    """n_lines seeded JSON lines of JLINE bytes: rows drawn from a pool of 4096 (int n, int-or-string status, float
    latency, a nested decoy member named "user", a filler string), the user key u0000000..u{n_keys-1} (uniform);
    nested: the rows of JROW_NESTED, the same members one level down"""
    prng = random.Random(seed)
    pool = np.empty((4096, JLINE), dtype=np.uint8)
    for i in range(len(pool)):
        row = (JROW_NESTED if nested else JROW) % (
            str(prng.randrange(-99999, 100000)).ljust(7), str(prng.choice([200, 201, 404, 500, '"404"', '"503"'])).ljust(6),
            repr(prng.uniform(0, 1e3)).ljust(23), prng.randrange(1000), prng.randrange(1000))
        row += "".join(prng.choice("abcdefghij") for _ in range(JLINE - 3 - len(row))) + '"}\n'
        pool[i] = np.frombuffer(row.encode("ascii"), dtype=np.uint8)
    at = row.index("u0000000") + 1
    rng = np.random.default_rng(seed)
    out = np.empty((n_lines, JLINE), dtype=np.uint8)
    step = 1 << 20
    for a in range(0, n_lines, step):
        t = out[a:a + step]
        t[:] = pool[rng.integers(0, len(pool), size=len(t))]
        keys = rng.integers(0, n_keys, size=len(t))
        for p in range(7):
            t[:, at + 6 - p] = 48 + (keys // 10 ** p) % 10
    return out.reshape(-1)


SET_KEYS = tuple("u%07d" % (i * 7919) for i in range(64))
WHERE = {"str": lambda r: r[0] < "u0500000", "int": lambda r: int(r[2]) >= 0, "float": lambda r: float(r[2]) >= 0,
         "set": lambda r: r[0] not in SET_KEYS, "prefix": lambda r: not r[1].startswith("x"),
         "or": lambda r: r[0] < "u0500000" or float(r[2]) >= 0}
LINE_WHERE = {"contains": lambda l: "ab" in l, "line": lambda l: l.startswith("u0") and len(l) > 90}   # on the line


def rewrite_filler(text, seed, key_fields):
    """--key-fields 2 and 3: the filler field of every row becomes one of two strings ('f' letters with 'a' or 'b' at
    byte 50, which lies inside the filler of both layouts and is not touched by whitespace_rows)"""
    if key_fields > 1:
        rows = text.reshape(-1, LINE)
        rng = np.random.default_rng(seed)
        step = 1 << 20
        for a in range(0, len(rows), step):
            t = rows[a:a + step]
            fill_end = 92 if t[0, 92] == ord(",") else LINE - 2 - FVAL
            t[:, 9:fill_end] = ord("f")
            t[:, 50] = ord("a") + rng.integers(0, 2, size=len(t), dtype=np.uint8)
    return text


KEY_FNS = {1: lambda r: r[0], 2: lambda r: (r[0], r[1]), 3: lambda r: (r[0], r[1], r[-3])}
EXPR_KEYS = {"field": lambda r: r[0], "const": lambda r: 1, "bucket": lambda r: int(r[2]) // 1000}
EXPR_VALUES = {"none": lambda r: int(r[2]), "product": lambda r: int(r[2]) * int(r[3]),
               "ratio": lambda r: int(r[2]) / int(r[3])}


def carve_quantity(text, seed, ws):
    """--expr product / ratio: the rows of csv_text with the filler 4 bytes shorter and a quantity field of 1-999
    behind the value: key ',' filler ',' value ',' qty '\\n', LINE bytes each (ws: a blank before the quantity,
    which whitespace_rows keeps)"""
    rows = text.reshape(-1, LINE)
    rng = np.random.default_rng(seed)
    step = 1 << 20
    for a in range(0, len(rows), step):
        t = rows[a:a + step]
        t[:, 89:95] = t[:, 93:99].copy()
        t[:, 88] = ord(",")
        t[:, 95] = ord(" " if ws else ",")
        q = rng.integers(1, 1000, size=len(t))
        for p in range(3):
            t[:, 98 - p] = 48 + (q // 10 ** p) % 10
    return text


def expr_job(Dampr, src, expr, key, op, sep):
    """the --expr / --key stage"""
    d = Dampr.read_input(src)
    if expr == "nfields":
        d = d.map(lambda v: len(v.split()))
        kf, vf = (lambda x: 1), (lambda x: x)
    else:
        d = d.map(splitter(sep))
        kf, vf = EXPR_KEYS[key], EXPR_VALUES[expr]
    if op == "mean":
        return d.mean(kf, vf)
    if op in ("min", "max"):
        return d.a_group_by(kf, vf).reduce(min if op == "min" else max)
    return d.fold_by(kf, value=vf, binop=lambda a, b: a + b)


def expr_fold(sample, expr, key, op, sep):
    """the --expr / --key stage as plain Python over the sample's lines: ({key: result}, {key: (lines, sum |v|)})"""
    out, mag = {}, {}
    lines = sample.decode("ascii").split("\n")[:-1]
    if expr == "nfields":
        rows = ((1, len(l.split())) for l in lines)
    else:
        kf, vf = EXPR_KEYS[key], EXPR_VALUES[expr]
        rows = ((kf(r), vf(r)) for r in map(splitter(sep), lines))
    for k, v in rows:
        n, m = mag.get(k, (0, 0.0))
        mag[k] = (n + 1, m + abs(v))
        if op == "mean":
            s, c = out.get(k, (0, 0))
            out[k] = (s + v, c + 1)
        elif k in out:
            out[k] = out[k] + v if op == "sum" else (min if op == "min" else max)(out[k], v)
        else:
            out[k] = v
    if op == "mean":
        out = {k: s / float(c) for k, (s, c) in out.items()}
    return out, mag


def splitter(sep):
    return (lambda l: l.split()) if sep == "ws" else (lambda l: l.split(","))


def json_job(Dampr, src, value, op, nested=False):
    d = Dampr.read_input(src).map(json.loads)
    if nested:
        key = lambda r: r["user"]["id"]   # noqa: E731
        val = (lambda r: r["stats"]["n"]) if value == "int" else (lambda r: float(r["stats"]["latency"]))
    else:
        key = lambda r: r["user"]   # noqa: E731
        val = (lambda r: r["n"]) if value == "int" else (lambda r: float(r["latency"]))
    if op == "mean":
        return d.mean(key, val)
    if op in ("min", "max"):
        return d.a_group_by(key, val).reduce(min if op == "min" else max)
    return d.fold_by(key, value=val, binop=lambda a, b: a + b)


def json_rows(sample, value, nested=False):
    """(key, value) of the sample's JSON lines, as the stage's lambdas read them"""
    for l in sample.decode("ascii").split("\n")[:-1]:
        r = json.loads(l)
        if nested:
            r = dict(r["stats"], user=r["user"]["id"])
        yield r["user"], (r["n"] if value == "int" else float(r["latency"]))


def job(Dampr, src, value="int", op="sum", where="none", sep="comma", key_fields=1, nested=False):
    if sep == "json":
        return json_job(Dampr, src, value, op, nested)
    conv = int if value == "int" else float
    key = KEY_FNS[key_fields]
    d = Dampr.read_input(src)
    if where in LINE_WHERE:
        d = d.filter(LINE_WHERE[where])
    d = d.map(splitter(sep))
    if where in WHERE:
        d = d.filter(WHERE[where])
    if op == "mean":
        return d.mean(key, lambda r: conv(r[2]))
    if op in ("min", "max"):
        return d.a_group_by(key, lambda r: conv(r[2])).reduce(min if op == "min" else max)
    return d.fold_by(key, value=lambda r: conv(r[2]), binop=lambda a, b: a + b)


def python_fold(sample, value, op, where="none", sep="comma", key_fields=1, nested=False):
    """the stage as plain Python over the sample's lines: {key: result}"""
    conv = int if value == "int" else float
    keep = WHERE.get(where, lambda r: True)
    split = splitter(sep)
    key = KEY_FNS[key_fields]
    out = {}
    if sep == "json":
        rows = json_rows(sample, value, nested)
    else:
        lines = [l for l in sample.decode("ascii").split("\n")[:-1] if LINE_WHERE.get(where, lambda l: True)(l)]
        rows = ((key(r), conv(r[2])) for r in map(split, lines) if keep(r))
    for k, v in rows:
        if op == "mean":
            s, n = out.get(k, (0, 0))
            out[k] = (s + v, n + 1)
        elif k in out:
            out[k] = out[k] + v if op == "sum" else (min if op == "min" else max)(out[k], v)
        else:
            out[k] = v
    if op == "mean":
        out = {k: s / float(n) for k, (s, n) in out.items()}
    return out


def magnitudes(sample, sep="comma", key_fields=1, nested=False):
    """{key: (lines, sum of |float value|)} of the sample: the scale of the sum bound"""
    mag = {}
    split = splitter(sep)
    key = KEY_FNS[key_fields]
    rows = json_rows(sample, "float", nested) if sep == "json" else \
        ((key(r), r[2]) for r in map(split, sample.decode("ascii").split("\n")[:-1]))
    for k, v in rows:
        n, a = mag.get(k, (0, 0.0))
        mag[k] = (n + 1, a + abs(float(v)))
    return mag


def within_bound(got, host, mag, op):
    """every key's device result within 4·n·2^-53·Σ|v| of Python's (plus one rounding of the result for a mean)"""
    if set(got) != set(host):
        return False
    for k, hv in host.items():
        n, a = mag[k]
        tol = 4 * n * 2.0 ** -53 * a
        if op == "mean":
            tol = tol / n + abs(hv) * 2.0 ** -52
        if abs(got[k] - hv) > 2 * tol:
            return False
    return True


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
    ap.add_argument("--value", choices=("int", "float"), default="int")
    ap.add_argument("--op", choices=("sum", "min", "max", "mean"), default="sum")
    ap.add_argument("--where", choices=("none", "str", "int", "float", "set", "contains", "prefix", "or", "line"),
                    default="none")
    ap.add_argument("--sep", choices=("comma", "ws", ","), default="comma")
    ap.add_argument("--format", choices=("csv", "json"), default="csv")
    ap.add_argument("--nested", action="store_true", help="--format json: the key and value one or two levels down")
    ap.add_argument("--key-fields", type=int, choices=(1, 2, 3), default=1)
    ap.add_argument("--expr", choices=("none", "product", "ratio", "nfields"), default="none")
    ap.add_argument("--key", choices=("field", "const", "bucket"), default="field")
    a = ap.parse_args()
    computed = a.expr != "none" or a.key != "field"
    if computed and (a.format != "csv" or a.value != "int" or a.where != "none" or a.key_fields != 1):
        ap.error("--expr and --key take neither --format json, --value float, --where nor --key-fields")
    if a.expr == "nfields" and (a.sep != "ws" or a.key != "const"):
        ap.error("--expr nfields is the README's stage: --sep ws --key const")
    if a.sep == ",":
        a.sep = "comma"
    if a.format == "json":
        if a.where != "none" or a.sep != "comma" or a.key_fields != 1:
            ap.error("--format json takes neither --where, --sep nor --key-fields")
        a.sep = "json"
    elif a.nested:
        ap.error("--nested takes --format json")
    if a.where == "int" and a.value != "int":
        ap.error("--where int needs --value int (int() of a float field raises)")
    default = a.value == "int" and a.op == "sum" and a.key_fields == 1 and not computed
    K = a.key_fields

    from dampr_b200 import Dampr, device as dev, plan
    from dampr_b200 import runner as runner_mod
    ctx = runner_mod.get_ctx()
    name, power = card()
    line = JLINE if a.sep == "json" else LINE
    n_lines = int(a.gb * 1e9) // line
    if a.sep == "json":
        text = json_text(2026, n_lines, a.keys, a.nested)
    else:
        text = csv_text(2026, n_lines, a.keys) if a.value == "int" else float_text(2026, n_lines, a.keys)
        text = rewrite_filler(text, 2028, K)
        if a.expr in ("product", "ratio"):
            text = carve_quantity(text, 2029, a.sep == "ws")
    if a.sep == "ws":
        text = whitespace_rows(text, 2027, 10 if a.expr in ("product", "ratio") else 6 if a.value == "int" else FVAL)
    nbytes = len(text)
    pin = dev.PinnedBuffer(nbytes)
    pin.array[:] = text
    tmpdir = a.out or tempfile.mkdtemp(prefix="fields_bench_")
    path = os.path.join(tmpdir, "events.csv")
    text.tofile(path)
    del text

    fetch_s = []   # --key-fields: seconds from the table fetch to the list of key tuples, per scan
    if K > 1:
        fetch = plan.FieldScan._fetch_tuple_keys

        def timed_fetch(scan, tab, tb):
            t = time.perf_counter()
            out = fetch(scan, tab, tb)
            fetch_s.append(time.perf_counter() - t)
            return out
        plan.FieldScan._fetch_tuple_keys = timed_fetch

    def timed(src, where="none"):
        ctx.timings_reset()
        t0 = time.perf_counter()
        stage = expr_job(Dampr, src, a.expr, a.key, a.op, a.sep) if computed else \
            job(Dampr, src, a.value, a.op, where, a.sep, K, a.nested)
        n = len(list(stage.run()))
        dt = time.perf_counter() - t0
        stages = runner_mod.LAST_STATS.stages
        assert "device text fields scan+combine" in stages[0][1], stages
        tm = ctx.timings()
        ms = sum(m for k, m in tm if k == "text_fields")
        by_name = {}
        for k, m in tm:
            by_name[k] = by_name.get(k, 0.0) + m
        return dt, ms, n, stages[0][2], by_name

    ctx.timing_enable(True)
    timed(plan.MemoryText(pin.array))          # warm-up: module load, buffers, table size
    mem = [timed(plan.MemoryText(pin.array)) for _ in range(a.reps)]
    with open(path, "rb") as f:                # page cache warm
        while f.read(64 << 20):
            pass
    from dampr_b200.inputs import PathInput
    fil = [timed(PathInput(path)) for _ in range(a.reps)]
    if a.where != "none":
        timed(plan.MemoryText(pin.array), a.where)
        wmem = [timed(plan.MemoryText(pin.array), a.where) for _ in range(a.reps)]
        wfil = [timed(PathInput(path), a.where) for _ in range(a.reps)]
    ctx.timing_enable(False)

    # host map on a sample: the stage as plain Python (the same lambdas), and the device result of the same bytes
    sample_lines = max(1, int(a.sample_mb * 1e6) // line)
    sample = pin.array[:sample_lines * line].tobytes()
    t0 = time.perf_counter()
    if computed:
        host, host_mag = expr_fold(sample, a.expr, a.key, a.op, a.sep)
    elif default and a.sep != "json":
        host = {}
        split = splitter(a.sep)
        for l in sample.decode("ascii").split("\n")[:-1]:
            r = split(l)
            k, v = r[0], int(r[2])
            host[k] = host[k] + v if k in host else v
    else:
        host = python_fold(sample, a.value, a.op, sep=a.sep, key_fields=K, nested=a.nested)
    host_s = time.perf_counter() - t0
    spin = dev.PinnedBuffer(len(sample))
    spin.array[:] = np.frombuffer(sample, dtype=np.uint8)
    got = dict((expr_job(Dampr, plan.MemoryText(spin.array), a.expr, a.key, a.op, a.sep) if computed else
                job(Dampr, plan.MemoryText(spin.array), a.value, a.op, sep=a.sep, key_fields=K, nested=a.nested)).run())

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
    if not default:
        best = min(mem, key=lambda m: m[0])
        res.update({"value": a.value, "op": a.op,
                    "kernels_ms": {k: round(v, 3) for k, v in sorted(best[4].items())}})
        if a.value == "float" and a.op in ("sum", "mean"):
            res["sample_within_bound"] = within_bound(got, host, magnitudes(sample, a.sep, K, a.nested), a.op)
        if computed:
            res.update({"expr": a.expr, "key": a.key})
            if a.expr == "ratio" or a.op == "mean":
                res["sample_within_bound"] = within_bound(got, host, host_mag, a.op)
    if K > 1:
        res.update({"key_fields": K, "fetch_to_frame_ms": round(1e3 * min(fetch_s[1:1 + a.reps]), 3)})
    if a.where != "none":
        t0 = time.perf_counter()
        whost = python_fold(sample, a.value, a.op, a.where, a.sep, K)
        whost_s = time.perf_counter() - t0
        wgot = dict(job(Dampr, plan.MemoryText(spin.array), a.value, a.op, a.where, a.sep, K).run())
        wk = min(m[1] for m in wmem)
        res.update({
            "where": a.where,
            "where_kernel_ms": round(wk, 3),
            "where_kernel_GBps": round(nbytes / wk / 1e6, 1),
            "where_e2e_pinned_MBps": round(nbytes / min(m[0] for m in wmem) / 1e6, 1),
            "where_e2e_pinned_s": [round(m[0], 3) for m in wmem],
            "where_e2e_file_warm_MBps": round(nbytes / min(f[0] for f in wfil) / 1e6, 1),
            "where_host_map_MBps": round(len(sample) / whost_s / 1e6, 1),
            "where_sample_equal": wgot == whost if not (a.value == "float" and a.op in ("sum", "mean")) else
            within_bound(wgot, whost, magnitudes(sample, a.sep, K), a.op),
            "where_stats": wmem[0][3],
        })
    if a.sep == "ws":
        res["sep"] = "ws"
    if a.sep == "json":
        res["format"] = "json"
    if a.nested:
        res["nested"] = True
    if a.out is None:
        shutil.rmtree(tmpdir, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Planner: recognises stages whose functions belong to the closed idiom set (lowering.py) and runs
them as device pipelines over columnar data; returns None for everything else (host-map path).

Lowered pipelines and the reference code they replace:
  TextCount     Dampr.text(..).flat_map(tokenise).count()/fold_by(identity, +)  — MapStageRunner.medium_map
                (stagerunner.py:79-129) with ReducedWriter (dataset.py:84-117): K0+K1+K2 in one kernel
  KeyedFold     the KeyedReduce that completes an associative fold (dampr.py:678-691) over an
                already fully combined frame: a relabelling, no work
  LineCount     .len() over a text input (dampr.py:245-275): by-product of the tokenise kernel
  KVFold        a_group_by(x[0], x[1]).sum()/min/max over binary kv records: K3+K4+K5
  KVGroup       group_by(x[0], x[1]) + reduce(sum(it)/len/min/max): K3+K4 (+K5)
  FrameSort     sort_by(+-x[i]) over a columnar frame: K3+K4 on (code, row) records
  FrameCross    cross_left/right against a one-row collection with an analysable function,
                evaluated once per distinct value of the fields it reads (exact Python results)
  FrameSink     sink / sink_tsv of a frame: vectorised formatting
"""
import logging
import math
import json
import os
import re
import threading

import numpy as np

from . import device as dev
from . import dist, keycodes, lowering, settings, vexpr
from . import operators as ops
from .datasets import Dataset, RecordsDataset, TextLineDataset, CatDataset, EmptyDataset
from .graph import GMap, GReduce, GSink
from .inputs import PathInput, TextInput, KVInput, ArrayKVInput

log = logging.getLogger("dampr_b200")


class NotLowerable(Exception):
    pass


# ---- columnar stage output -----------------------------------------------------------------------
class DictCol(object):
    """Dictionary-encoded column: value[i] = uniq[inv[i]] (uniq: numpy array or list)."""

    def __init__(self, inv, uniq):
        self.inv = inv
        self.uniq = uniq

    def __len__(self):
        return len(self.inv)

    def materialize(self):
        if isinstance(self.uniq, np.ndarray):
            return self.uniq[self.inv]
        il = self.inv.tolist()
        u = self.uniq
        return [u[j] for j in il]


# The dictionary of the count column of the last device text scan, built on the device when first asked for:
# (the column object, a function returning (uniq, inv, rows) or None, its result once known)
_COUNT_DICT = [None, None, None]


def remember_count_dictionary(col, build):
    _COUNT_DICT[:] = [col, build, None]


def forget_count_dictionary():
    _COUNT_DICT[:] = [None, None, None]


def _known_dictionary(col):
    if _COUNT_DICT[0] is not col:
        return None
    if _COUNT_DICT[2] is None and _COUNT_DICT[1] is not None:
        build, _COUNT_DICT[1] = _COUNT_DICT[1], None
        _COUNT_DICT[2] = build()
    return _COUNT_DICT[2]


def unique_inverse_rows(col):
    """unique_inverse plus one row index per distinct value (any row holding it)."""
    known = _known_dictionary(col)
    if known is not None:
        return known
    n = len(col)
    if n >= 4096 and col.dtype == np.int64:
        r = dev.host_unique_small(col, with_rows=True)
        if r is not None:
            return r
    uniq, inv = unique_inverse(col)
    rep = np.empty(len(uniq), dtype=np.int64)
    rep[inv] = np.arange(n, dtype=np.int64)
    return uniq, inv, rep


def unique_inverse(col):
    """(sorted unique values, inverse index uint32) of an int64/float64 column. Small non-negative
    ints (the bulk of count columns) go through a counting pass instead of a sort."""
    known = _known_dictionary(col)
    if known is not None:
        return known[0], known[1]
    n = len(col)
    if n >= 4096 and col.dtype == np.int64:
        r = dev.host_unique_small(col)   # native presence-table pass; None if the values do not suit it
        if r is not None:
            return r
    if n and col.dtype.kind in "iu":
        # counting table sized by the bulk of the values (99.9th percentile, capped at 4 M entries)
        T = int(min(1 << 22, max(1024, int(np.partition(col, max(0, n - 1 - n // 1000))[max(0, n - 1 - n // 1000)]) + 1)))
        small = col < T
        if col.min() >= 0 and small.mean() > 0.99:
            cs = col[small].astype(np.int64)
            present = np.zeros(T, dtype=bool)
            present[cs] = True
            us = np.flatnonzero(present)
            rank = np.zeros(T, dtype=np.uint32)
            rank[us] = np.arange(len(us), dtype=np.uint32)
            inv = np.empty(n, dtype=np.uint32)
            inv[small] = rank[cs]
            if not small.all():
                ul, il = np.unique(col[~small], return_inverse=True)
                inv[~small] = il.astype(np.uint32) + np.uint32(len(us))
                uniq = np.concatenate((us.astype(col.dtype), ul))
            else:
                uniq = us.astype(col.dtype)
            return uniq, inv
    uniq, inv = np.unique(col, return_inverse=True)
    return uniq, inv.astype(np.uint32)


class Frame(Dataset):
    """Columnar collection. `keys` is the routing/sort key column (what read() yields as k), `cols`
    are the value columns; the user-visible value is cols[0][i] when `scalar` else the tuple of the
    columns. Columns are numpy arrays (numeric) or Python lists (strings / objects)."""

    def __init__(self, keys, cols, scalar, combined=False):
        self.keys = keys
        self.cols = list(cols)
        self.scalar = scalar
        self.combined = combined  # every key appears once (map-side combine already complete)
        self.n = len(cols[0]) if cols else 0
        self.meta = {}

    def __len__(self):
        return self.n

    @staticmethod
    def _pylist(col):
        if isinstance(col, vexpr.Tup):   # tuple-valued column (e.g. mean()'s (sum, count) pairs)
            return list(zip(*[Frame._pylist(c) for c in col.items]))
        if isinstance(col, DictCol):
            col = col.materialize()
        if isinstance(col, np.ndarray):
            if col.dtype.kind == "S":  # device-decoded ASCII keys
                return [b.decode("ascii") for b in col.tolist()]
            return col.tolist()
        return col

    def values(self):
        if self.scalar:
            return self._pylist(self.cols[0])
        return list(zip(*[self._pylist(c) for c in self.cols]))

    def read(self):
        keys = self._pylist(self.keys) if self.keys is not None else range(self.n)
        return zip(keys, self.values())

    def take(self, perm):
        done = {}   # a column object that appears twice (keys == cols[0] after a relabel) is gathered once

        def tk(c):
            if id(c) not in done:
                done[id(c)] = tk1(c)
            return done[id(c)]

        def tk1(c):
            if isinstance(c, vexpr.Tup):
                return vexpr.Tup([tk(x) for x in c.items])
            if isinstance(c, DictCol):
                return DictCol(c.inv[perm], c.uniq)
            if isinstance(c, np.ndarray):
                if c.dtype.kind == "S" and c.dtype.itemsize % 8 == 0 and c.flags["C_CONTIGUOUS"] and c.ndim == 1:
                    # fixed-width strings gather faster as rows of 8-byte words than as 'S' elements
                    w = c.dtype.itemsize // 8
                    return np.take(c.view(np.uint64).reshape(len(c), w), perm, axis=0).view(c.dtype).ravel()
                return c[perm]
            pl = perm.tolist()
            return [c[i] for i in pl]
        f = Frame(tk(self.keys) if self.keys is not None else None, [tk(c) for c in self.cols], self.scalar,
                  self.combined)
        return f

    def delete(self):
        self.keys, self.cols, self.n = None, [[]], 0


# ---- text sources ----------------------------------------------------------------------------------
class MemoryText(Dataset):
    """Text held in host memory (a numpy uint8 array, ideally page-locked): the "file in pinned host
    memory" starting point of the end-to-end metric (SURVEY §8(d)). read() yields lines like
    TextLineDataset."""

    def __init__(self, array):
        self.array = array

    def read(self):
        from .datasets import _iter_lines
        return _iter_lines(self.array.tobytes(), 0)


class DeviceText(Dataset):
    """Text already resident in HBM (a device.TextBuf): the starting point of the device-resident
    throughput figure."""

    def __init__(self, tb):
        self.tb = tb

    def read(self):
        from .datasets import _iter_lines
        return _iter_lines(self.tb.download(0, self.tb.n).tobytes(), 0)


def _text_files(ds):
    """[(kind, payload)] if the dataset is plain text the device can ingest, else None."""
    if isinstance(ds, MemoryText):
        return [("mem", ds.array)]
    if isinstance(ds, DeviceText):
        return [("dev", ds.tb)]
    if isinstance(ds, PathInput):
        files = ds.files()
    elif isinstance(ds, TextInput):
        files = [ds.path]
    elif isinstance(ds, TextLineDataset) and ds.start == 0 and ds.end is None:
        files = [ds.path]
    elif isinstance(ds, CatDataset) and ds.datasets and all(
            isinstance(d, TextLineDataset) and d.start == 0 and d.end is None for d in ds.datasets):
        files = [d.path for d in ds.datasets]
    else:
        return None
    # .gz inputs (TextInput on a gzip file: one unsplittable chunk, inputs.py:43-46 / dataset.py:484-499 in
    # the reference) are inflated on the host and ingested like in-memory text
    return [("gz" if f.endswith(".gz") else "file", f) for f in files]


_NONWORD_RX = re.compile(r"[^\w]+")   # what lowering.tokenizer_mode matched ([^\w]+ or \W+, default flags)


def _tokens_present(words, tokens):
    """the subset of `tokens` (str) that the token table `words` holds"""
    if isinstance(words, np.ndarray):
        W = words.dtype.itemsize
        fit = [k for k in tokens if k.isascii() and 0 < len(k) <= W and "\0" not in k]
        if not fit or not len(words):
            return set()
        arr = np.array([k.encode("ascii") for k in fit], dtype=words.dtype)
        return set(b.decode("ascii") for b in arr[np.isin(arr, words)].tolist())
    have = set(words)
    return set(k for k in tokens if k in have)


def merge_token_counts(words, counts, extra):
    """(words, counts) of a device token table plus {token: count} of host-tokenised lines. `words` is a
    fixed-width 'S' array (ASCII tokens) or a list of str; tokens the array cannot hold (non-ASCII, longer than
    its width) turn it into a list."""
    if not extra:
        return words, counts
    counts = np.array(counts, dtype=np.int64, copy=True)
    keys = list(extra)
    if isinstance(words, np.ndarray):
        W = words.dtype.itemsize
        fit = [k for k in keys if k.isascii() and 0 < len(k) <= W and "\0" not in k]
        pos = {}
        if fit and len(words):
            arr = np.array([k.encode("ascii") for k in fit], dtype=words.dtype)
            hit = np.flatnonzero(np.isin(words, arr))
            pos = {w: int(i) for w, i in zip(words[hit].tolist(), hit.tolist())}
        new = []
        for k in keys:
            i = pos.get(k.encode("ascii")) if (k.isascii() and len(k) <= W) else None
            if i is not None:
                counts[i] += extra[k]
            else:
                new.append(k)
        if not new:
            return words, counts
        if all(k.isascii() and 0 < len(k) <= W and "\0" not in k for k in new):
            words = np.concatenate((words, np.array([k.encode("ascii") for k in new], dtype=words.dtype)))
        else:
            words = [b.decode("ascii") for b in words.tolist()] + new
        return words, np.concatenate((counts, np.array([extra[k] for k in new], dtype=np.int64)))
    pos = {w: i for i, w in enumerate(words)}
    new = []
    for k in keys:
        i = pos.get(k)
        if i is not None:
            counts[i] += extra[k]
        else:
            new.append(k)
    return list(words) + new, np.concatenate((counts, np.array([extra[k] for k in new], dtype=np.int64)))


def _inflate(paths):
    """Decompressed bytes of gzip files as uint8 arrays (zlib releases the GIL: one thread per file)."""
    import gzip
    from concurrent.futures import ThreadPoolExecutor

    def one(p):
        with gzip.open(p, "rb") as f:
            return np.frombuffer(f.read(), dtype=np.uint8)
    if len(paths) == 1:
        return [one(paths[0])]
    with ThreadPoolExecutor(min(len(paths), max(1, int(settings.max_processes)))) as ex:
        return list(ex.map(one, paths))


_PIN_RING = {}


def _pinned_ring(nslots, slot_bytes):
    key = (nslots, slot_bytes)
    ring = _PIN_RING.get(key)
    if ring is None:
        ring = [dev.PinnedBuffer(slot_bytes) for _ in range(nslots)]
        _PIN_RING.clear()
        _PIN_RING[key] = ring
    return ring


_BUFFERS = {}


def _cached_textbuf(ctx, capacity):
    """Device text buffer reused across scans of one context (grow-only): a 10 GB cudaMalloc/cudaFree
    per run costs tens of milliseconds."""
    slot = _BUFFERS.setdefault(id(ctx), {})
    tb = slot.get("tb")
    if tb is None or tb.ctx.h is None or tb.capacity < capacity:
        if tb is not None and tb.ctx.h is not None:
            tb.free()
        tb = ctx.textbuf(capacity)
        slot["tb"] = tb
    return tb


def _cached_table(ctx):
    slot = _BUFFERS.setdefault(id(ctx), {})
    tab = slot.get("tab")
    log2 = int(settings.text_table_log2)
    if tab is None or tab.ctx.h is None or tab.capacity != (1 << log2):
        if tab is not None and tab.ctx.h is not None:
            tab.free()
        tab = ctx.table(log2)
        slot["tab"] = tab
    else:
        tab.clear()
    return tab


def release_buffers():
    for slot in _BUFFERS.values():
        for b in slot.values():
            try:
                if b.ctx.h is not None:
                    b.free()
            except Exception:
                pass
    _BUFFERS.clear()


def resident_retry_block(scan):
    """Bound the table-growth retries of one scan."""
    scan._grow = getattr(scan, "_grow", 0) + 1
    return scan._grow > 4


class TextScan(object):
    """One pass of the tokenise+combine kernel over a set of files (or a memory text), with the
    host->device copies pipelined against the kernel chunk by chunk."""

    HALO = 16384   # bytes past a launch's range that must be uploaded before it (the kernel's window)

    def __init__(self, runner, sources, mode):
        self.runner = runner
        self.sources = sources
        self.mode = mode
        self.words = None
        self.counts = None
        self.n_lines = 0
        self.empty = 0
        self.nbytes = 0
        self.has_cr = False   # '\r' seen: n_lines counts '\n' only and is not the universal-newline line count

    def _launch(self, tab, tb, lo, hi):
        """the kernel over the lines that start in [lo, hi)"""
        tab.count(tb, lo, hi, self.mode, getattr(self, "_cr_is_data", False))

    def _ingest(self):
        """Upload the sources (or take the resident text), run _launch over all of it: (ctx, tb, table, stats)."""
        ctx = self.runner.ctx
        resident = len(self.sources) == 1 and self.sources[0][0] == "dev"
        tab = None
        self._tab = None
        if resident:
            tb = self.sources[0][1]
            self.nbytes = tb.n
        else:
            gz = [p for kind, p in self.sources if kind == "gz"]
            # the reference reads .gz files in BINARY mode (GzipLineDataset, dataset.py:488-493): only '\n' ends a
            # line and a '\r' stays in it, where it is an ordinary separator of the \w tokenisers and whitespace
            # for str.split. The kernels treat it exactly like that; the CR flag (universal newlines of text-mode
            # files) does not apply when every source of the scan is a .gz file.
            if gz and len(gz) == len(self.sources):
                self._cr_is_data = True
            if not hasattr(self, "_binary_src"):   # (a repeated scan sees the inflated .gz sources as memory texts)
                self._binary_src = [kind == "gz" for kind, _p in self.sources]
            if gz:
                if dist.active():
                    raise NotLowerable("gzip inputs are not sharded across ranks")
                texts = iter(_inflate(gz))
                self.sources = [("mem", next(texts)) if kind == "gz" else (kind, p) for kind, p in self.sources]
            sizes = []
            for kind, p in self.sources:
                sizes.append(len(p) if kind == "mem" else os.path.getsize(p))
            total = sum(sizes) + len(sizes)
            self.nbytes = sum(sizes)
            tb = _cached_textbuf(ctx, total + 64)
        # buffers are cached per context (see _cached_textbuf): nothing to release here
        if resident:
            self._tab = _cached_table(ctx)
            self._launch(self._tab, tb, 0, tb.n)
        else:
            self._upload_and_count(ctx, tb, sizes)
        tab = self._tab
        st = tab.stats()
        if getattr(self, "_cr_is_data", False):
            st = dict(st, flags=st["flags"] & ~dev.TF_CR)
        return ctx, tb, tab, st

    def _grow_table(self, tab, st):
        """True when the table was made 4x larger for a repeated scan: it is full or over half full, below 2^28
        entries, and the scan has retries left. ReducedWriter would flush a run here (dataset.py:107-113); with HBM
        to spare the table is simply made larger (later scans start at the new size)."""
        if (st["flags"] & dev.TF_TABLEFULL or st["entries"] * 2 > tab.capacity) and settings.text_table_log2 < 28 \
                and not resident_retry_block(self):
            settings.text_table_log2 = int(settings.text_table_log2) + 2
            return True
        return False

    def run(self):
        ctx, tb, tab, st = self._ingest()
        flags = st["flags"]
        if dist.active():
            return self._finish_distributed(ctx, tb, tab, st)
        if self._grow_table(tab, st):
            return self.run()
        if flags & dev.TF_TABLEFULL:
            raise NotLowerable("combiner table overflow")
        if flags & (dev.TF_NONASCII | dev.TF_LONGTOKEN):
            raise NotLowerable("non-ASCII text or oversized token: device tokeniser is ASCII-only")
        if self.mode != dev.TOK_WS and flags & dev.TF_LONGLINE and not flags & dev.TF_CR \
                and not getattr(self, "_retry_v1", False):
            # a line with too many distinct tokens for the default build of the kernel (64 remembered per
            # straddling line at 4 CTAs/SM): the 2-CTA build remembers 256 ...
            if not getattr(self, "_retry_2cta", False):
                self._retry_2cta = True
                dev.set_option("text_ctas", 2)
                try:
                    return self.run()
                finally:
                    dev.set_option("text_ctas", int(settings.text_kernel_ctas))
            # ... and a line too long for the warp-autonomous kernel altogether goes to the first-generation
            # kernel (4 KB line window, no per-line token limit)
            self._retry_v1 = True
            dev.set_option("text_kernel", 1)
            try:
                return self.run()
            finally:
                dev.set_option("text_kernel", 2)
        if self.mode != dev.TOK_WS and flags & (dev.TF_CR | dev.TF_LONGLINE):
            raise NotLowerable("carriage returns or a line longer than the device window")
        if st["hashed"] and getattr(self, "_retry_v1", False):
            # the first-generation kernel verifies long tokens in a second pass; the v2 kernel
            # compares every long token with its entry's representative while counting
            tab.verify(tb, 0, tb.n, self.mode)
            flags = tab.stats()["flags"]
        if flags & dev.TF_COLLISION:
            raise NotLowerable("64-bit key-code collision between two long tokens")
        words, counts = self._fetch_words(tab, tb, st, self.mode)
        self._fetched = (getattr(tab, "fetches", None), len(counts))   # the table still holds this column on the device
        self.words = words
        self.counts = counts.view(np.int64)
        self.n_lines = int(st["lines"])
        self.empty = int(st["empty"])
        self.has_cr = bool(flags & dev.TF_CR)
        extra, extra_empty, extra_lines = self._host_lines(tb, tab, st)
        if extra_lines:
            self.words, self.counts = merge_token_counts(self.words, self.counts, extra)
            self.empty += extra_empty
            self.n_lines += extra_lines
        self.host_lines = extra_lines
        return self

    def _fetch_words(self, tab, tb, st, mode, want_codes=False):
        """(keys, counts) of the table: keys are materialised on the device (K9) as fixed-width ASCII; only tokens
        longer than the width (rare) are patched on the host from their representative occurrence.
        want_codes: (keys, counts, key codes)"""
        # exact codes hold at most 12 characters: without hashed tokens 16 bytes per key are enough and
        # neither codes nor representatives are needed on the host
        hashed = bool(st["hashed"])
        W = 32 if hashed else 16
        words, counts, codes, reps = tab.fetch_words(tb, mode, W, with_codes=hashed or want_codes)
        too_long = np.flatnonzero(((codes >> np.uint64(63)) != 0) & ((reps & np.uint64(0xFFFFF)) > W)) if hashed else ()
        if len(too_long):
            wl = [b.decode("ascii") for b in words.tolist()]
            for i in too_long.tolist():
                rep = int(reps[i])
                s = tb.download(rep >> 20, rep & 0xFFFFF).tobytes().decode("ascii")
                wl[i] = s if mode == dev.TOK_WS else s.lower()
            words = wl
        return (words, counts, codes) if want_codes else (words, counts)

    def count_dictionary(self, extra=()):
        """unique_inverse_rows of the count column followed by the rows `extra`, computed on the device from the
        column the table still holds; None when the table has moved on (another scan, another fetch) or host-
        tokenised lines changed the column."""
        tab = self._tab
        fetched = getattr(self, "_fetched", None)
        if tab is None or fetched is None or fetched[0] is None or fetched[0] != tab.fetches or self.host_lines:
            return None
        ptr, n = tab.extracted_counts()
        if n != fetched[1]:
            return None
        return self.runner.ctx.count_dictionary(ptr, n, 1, extra)

    def _fallback_lines(self, tb, tab):
        """(offset, line) of every line on the table's fallback list, split by the reference's reader rules"""
        from .datasets import _iter_lines
        import bisect
        fb = np.sort(tab.fallback_lines())
        starts = getattr(self, "_layout_starts", None)
        binary = getattr(self, "_binary_src", None)
        for e in fb.tolist():
            off, ln = e >> 16, e & 0xFFFF
            raw = tb.download(off, ln).tobytes()
            # a .gz source is read in binary mode by the reference ('\r' stays in the line), a text file with
            # universal newlines: the line's offset tells which source it came from
            universal = not getattr(self, "_cr_is_data", False)
            if starts and binary and len(binary) == len(starts):
                universal = not binary[max(0, bisect.bisect_right(starts, off) - 1)]
            for item in _iter_lines(raw, off, universal=universal):
                yield item

    def _host_lines(self, tb, tab, st):
        """Per-line fallback (SURVEY §8(a) T1/T2, VERDICT r1 #5): the lines the kernel could not tokenise the way
        Python does — a non-ASCII byte (Unicode \\w and lower()), a '\\r' in a text-mode source (universal
        newlines split the line) — were left out of the table; they are read back, split and tokenised here with
        the reference's own rules (TextLineDataset.read dataset.py:458-476, the matched tokeniser idiom) and the
        counts are merged. Returns ({token: count}, count of the '' token, number of lines)."""
        if self.mode == dev.TOK_WS or not st.get("fallback"):
            return {}, 0, 0
        extra, empty, nlines = {}, 0, 0
        dedup = self.mode == dev.TOK_NONWORD_LOWER_SET
        for _o, line in self._fallback_lines(tb, tab):
            nlines += 1
            toks = _NONWORD_RX.split(line.lower())
            for t in (set(toks) if dedup else toks):
                if t == "":
                    empty += 1
                else:
                    extra[t] = extra.get(t, 0) + 1
        return extra, empty, nlines

    def _finish_distributed(self, ctx, tb, tab, st):
        """world > 1: this rank scanned its shard; move every term to its owner with one all-to-all
        (dist.shuffle_kv), finish the fold there (merge + segmented reduce), sum the line counts."""
        rank, n = dist.world()
        flags = int(st["flags"])
        bad = flags & (dev.TF_TABLEFULL | dev.TF_NONASCII | dev.TF_LONGTOKEN)
        if self.mode != dev.TOK_WS:
            bad |= flags & (dev.TF_CR | dev.TF_LONGLINE)
        hashed_words = {}
        if flags & dev.TF_COLLISION:
            bad |= dev.TF_COLLISION
        if st["hashed"] and not bad:
            codes, _counts, reps = tab.fetch()
            hs = np.flatnonzero((codes & keycodes.HASHED_BIT) != 0)
            ws = keycodes.decode_table(codes[hs], reps[hs], self.mode,
                                       lambda off, ln: tb.download(off, ln).tobytes())
            hashed_words = dict(zip(codes[hs].tolist(), ws))
        # the local table as ONE SORTED RUN, one exchange (dampr_kv_all_to_all: the line counts and flags of every
        # rank travel with the record counts, so the scan needs no collective of its own), then the owner merges
        # the sorted runs of all source ranks and folds equal keys while merging (MergeDataset.read + the
        # combiner, dataset.py:571-579, base.py:393-402): one read + one write instead of a second sort
        header = [int(st["lines"]), int(st["empty"]), 1 if bad else 0, len(hashed_words), 1 if flags & dev.TF_CR else 0,
                  int(st.get("fallback", 0))]
        local = tab.to_kv() if not bad else ctx.kv(1)   # a rank that cannot lower still takes part in the exchange
        try:
            if not bad:
                local.sort(dev.KEY_MIX)
            recv, offs, heads = dist.shuffle_kv(ctx, local, header)
        finally:
            local.free()
        lines, empty, anybad, any_hashed, any_cr, any_fb = [int(x) for x in np.asarray(heads).sum(axis=0).tolist()]
        self.has_cr = bool(any_cr)
        if anybad:
            recv.free()
            raise RuntimeError("distributed text scan cannot be lowered on every rank (flags=%d); the "
                               "host-map path is single-process only" % flags)
        merged = {}
        for d in (dist.all_gather_objects(hashed_words) if any_hashed else ()):
            for c, w in d.items():
                if merged.setdefault(c, w) != w:
                    raise RuntimeError("64-bit key-code collision between two long tokens across ranks")
        red = ctx.kv_merge_ranges(recv, offs, dev.KEY_MIX, dev.OP_SUM_I64)
        recv.free()
        codes, counts = red.columns()
        W = 32 if any_hashed else 16             # exact codes hold at most 12 characters
        words = red.decode_words(self.mode, W)   # exact codes decoded on the device
        red.free()
        hs = np.flatnonzero((codes & keycodes.HASHED_BIT) != 0)
        if len(hs):
            strs = [merged[int(codes[i])] for i in hs.tolist()]
            if max(len(x) for x in strs) <= W:
                words[hs] = np.array([x.encode("ascii") for x in strs], dtype=words.dtype)
            else:
                wl = [b.decode("ascii") for b in words.tolist()]
                for i, x in zip(hs.tolist(), strs):
                    wl[i] = x
                words = wl
        self.words = words
        self.counts = counts.view(np.int64)
        self.n_lines = int(lines)
        self.empty = int(empty) if rank == 0 else 0
        # per-line fallback across ranks: every rank tokenises the lines its shard handed back; the counts of all
        # ranks are added up, a token goes to the rank whose table already holds it, otherwise to rank 0
        self.host_lines = 0
        if any_fb:   # (known from the exchange's header: no extra collective when no rank handed lines back)
            extra, extra_empty, extra_lines = self._host_lines(tb, tab, st)
            tot = dist.all_reduce_sum_int([extra_lines, extra_empty])
            self.host_lines = int(tot[0])
            merged_extra = {}
            for d in dist.all_gather_objects(extra):
                for k, v in d.items():
                    merged_extra[k] = merged_extra.get(k, 0) + v
            mine = _tokens_present(self.words, list(merged_extra))
            owners = dist.all_gather_objects(sorted(mine))
            taken = set()
            for o in owners:
                taken.update(o)
            take = {k: v for k, v in merged_extra.items() if k in mine or (rank == 0 and k not in taken)}
            self.words, self.counts = merge_token_counts(self.words, self.counts, take)
            self.n_lines += int(tot[0])
            if rank == 0:
                self.empty += int(tot[1])
        return self

    def _upload_and_count(self, ctx, tb, sizes):
        chunk = int(settings.ingest_chunk_bytes)
        chunk -= chunk % 4096
        # layout: files back to back; a file that does not end in '\n' gets one (its last line is a
        # line either way), so line and token semantics of the concatenation equal the per-file ones
        self._tab = _cached_table(ctx)
        tab = self._tab
        # the total length must be known before the first kernel: files are stat'ed, the optional
        # separator is reserved and patched if not needed (a spare '\n' after a terminated file would
        # add an empty line, so the layout is decided by peeking at each file's last byte)
        layout = []
        pos = 0
        for (kind, p), sz in zip(self.sources, sizes):
            need_nl = False
            if sz:
                if kind == "mem":
                    need_nl = p[sz - 1] != 10
                else:
                    with open(p, "rb") as f:
                        f.seek(sz - 1)
                        need_nl = f.read(1) != b"\n"
            layout.append((pos, sz, need_nl))
            pos += sz + (1 if need_nl else 0)
        total = pos
        self._layout_starts = [a for a, _sz, _nl in layout]
        tb.set_length(total)
        # files are a global input: under torch.distributed every rank owns one 4 KB-aligned byte range
        # of the concatenation (line ownership at the seams is the kernel's rule); in-memory texts are
        # rank-local shards already
        self._own = (0, total)
        if dist.active() and all(k == "file" for k, _p in self.sources):
            r, n = dist.world()
            lo = (total * r // n) // 4096 * 4096
            hi = total if r == n - 1 else (total * (r + 1) // n) // 4096 * 4096
            self._own = (lo, hi)
        nl = np.frombuffer(b"\n", dtype=np.uint8)
        done = 0      # bytes uploaded
        counted = 0   # bytes handed to the kernel
        ring = None
        for (kind, p), (base, sz, need_nl) in zip(self.sources, layout):
            if kind == "mem":
                off = 0
                while off < sz:
                    ln = min(chunk, sz - off)
                    tb.upload(base + off, p[off:off + ln], ln)
                    off += ln
                    done = base + off
                    counted = self._count_ready(tab, tb, counted, done, total, final=False)
            else:
                self._upload_file(ctx, tb, p, base, sz, ring, chunk, tab, counted, total)
                done = base + sz
                counted = self._counted
            if need_nl:
                tb.upload(base + sz, nl, 1)
                done = base + sz + 1
        self._count_ready(tab, tb, counted, total, total, final=True)
        return layout

    def _count_ready(self, tab, tb, counted, done, total, final):
        """Launch the kernel over every 4 KB-aligned range whose halo has been uploaded."""
        HALO = self.HALO
        hi = total if final else max(counted, ((done - HALO) // 4096) * 4096 if done > HALO else 0)
        if hi > counted:
            a, b = max(counted, self._own[0]), min(hi, self._own[1])
            if b > a:
                self._launch(tab, tb, a, b)
            counted = hi
        self._counted = counted
        return counted

    def _upload_file(self, ctx, tb, path, base, sz, ring, chunk, tab, counted, total):
        """page cache -> the library's page-locked ring (its copy threads pread() 1 MB pieces in parallel) -> device,
        chunk by chunk, kernel launches trailing the copies (dampr_textbuf_upload_file)."""
        self._counted = counted
        off = 0
        while off < sz:
            ln = min(chunk, sz - off)
            tb.upload_file(base + off, path, off, ln)
            off += ln
            self._count_ready(tab, tb, self._counted, base + off, total, final=False)


class FieldScan(TextScan):
    """One pass of the delimited-field kernel (dampr_text_fields) over a text input: TextScan's ingest with the field
    fold as the per-range launch. The lines the device hands back go through the stage's own functions.

    Float sums and mean() run the kernel's record mode (dampr_text_fields_records): one {key code, value} record per
    line in line order, folded by a stable device sort + segmented reduce, so a float sum is the same bits whatever
    the chunking; the table counts the lines of each key (mean()'s count)."""

    HALO = dev.FIELDS_HALO   # a line longer than the kernel's window is measured up to 64 KB past its start
    REC_BYTES = 32           # per record: the record and the sort's scratch copy

    def __init__(self, runner, sources, spec, op, stage, mean, preds=(), expr=None):
        TextScan.__init__(self, runner, sources, None)
        self.expr = expr     # computed key / value programs (device.field_expr) for dampr_text_fields_expr, or None
        self.spec = spec     # (separator byte or FIELD_SEP_WS, key index, key kind, value index or FIELD_VAL_ONE)
        # a tuple key (key kind KEY_TUPLE): its components go to the tuple calls, the spec's key field is not read
        self.key_comps = spec[1] if spec[2] == KEY_TUPLE else None
        self.preds = preds   # the stage's filters as device WHERE predicates (device.fields_spec)
        self._where = {"preds": preds} if preds else {}
        self.filtered = 0    # lines the predicates dropped on the device
        self.op = op
        self.stage = stage
        self.mean = mean     # values are mean()'s (sum, count) pairs
        self.records = mean or op == dev.OP_SUM_F64
        self.float_values = op in (dev.OP_SUM_F64, dev.OP_MIN_F64, dev.OP_MAX_F64)
        self.keys = self.values = None
        self.groups = self.host_lines = 0
        self._rec = None     # record buffer (KV) and its capacity
        self._rec_cap = 0
        self._rec_regrown = False

    def _launch(self, tab, tb, lo, hi):
        spec = tuple(self.spec) + (self.op,)
        cr = getattr(self, "_cr_is_data", False)
        if self.key_comps is not None:
            spec = (spec[0], 0, dev.FIELD_KEY_STR) + spec[3:]
        if not self.records:
            # a stage without filters makes exactly the plain call
            if self.expr is not None:
                tab.fields_expr(tb, lo, hi, spec, self.expr, cr, **self._where)
            elif self.key_comps is not None:
                tab.fields_tuple(tb, lo, hi, spec, self.key_comps, cr, **self._where)
            else:
                tab.fields(tb, lo, hi, spec, cr, **self._where)
            return
        if self._rec is None:
            # a first guess of one record per 32 bytes of text; a scan with more lines is repeated once with a
            # buffer of the exact size (DAMPR_TF_RECFULL)
            self._records_buffer(min(tb.n // 32 + 4096, self._free_bytes() // (2 * self.REC_BYTES)))
        if self.expr is not None:
            tab.fields_expr_records(tb, lo, hi, spec, self.expr, self._rec, cr, **self._where)
        elif self.key_comps is not None:
            tab.fields_tuple_records(tb, lo, hi, spec, self.key_comps, self._rec, cr, **self._where)
        else:
            tab.fields_records(tb, lo, hi, spec, self._rec, cr, **self._where)

    def _free_bytes(self):
        return int(self.runner.ctx.mem_info()[0])

    def _records_buffer(self, n):
        """a record buffer of n records, refused when it and the sort's scratch do not fit in device memory"""
        held = self._rec_cap * 16
        self._free_records()
        if self.REC_BYTES * n > self._free_bytes() + held:
            raise NotLowerable("field records and sort scratch (%d B per line) exceed free device memory"
                               % self.REC_BYTES)
        self._rec = self.runner.ctx.kv(max(1, n))
        self._rec_cap = max(1, n)

    def _free_records(self):
        if self._rec is not None:
            self._rec.free()
        self._rec, self._rec_cap = None, 0

    def run(self):
        try:
            return self._run()
        finally:
            self._free_records()

    def _run(self):
        _ctx, tb, tab, _st = self._ingest()
        st = tab.fields_stats()
        flags = st["flags"]
        if self._grow_table(tab, st):
            return self._run()
        if self._kind_retry(st):
            return self._run()
        if flags & dev.TF_TABLEFULL:
            raise NotLowerable("combiner table overflow")
        if flags & (dev.TF_NONASCII | dev.TF_LONGLINE):
            raise NotLowerable("more lines for the host than the fallback list holds, or a line of 64 KB or more")
        if flags & dev.TF_COLLISION:
            raise NotLowerable("64-bit key-code collision between two long keys")
        if self.float_values and flags & dev.TF_NEGZERO:
            raise NotLowerable("-0.0 among the float() values: Python's result depends on the order of the arguments")
        if self.float_values and self.op != dev.OP_SUM_F64 and flags & dev.TF_NAN:
            raise NotLowerable("a computed NaN under min/max: Python's result depends on the order of the arguments")
        if self.records and flags & dev.TF_RECFULL:
            if self._rec_regrown:
                raise NotLowerable("field records overflow their buffer")
            self._rec_regrown = True
            self._records_buffer(int(st["records"]))   # the exact line count of the scan
            return self._run()
        if self.key_comps is not None:
            keys, acc, codes = self._fetch_tuple_keys(tab, tb)
        elif self.spec[2] == dev.FIELD_KEY_INT:
            codes, acc, _reps = tab.fetch()
            keys = (codes ^ np.uint64(1 << 63)).view(np.int64)
        elif self.records:
            keys, acc, codes = self._fetch_words(tab, tb, st, dev.TOK_WS, want_codes=True)
        else:
            keys, acc = self._fetch_words(tab, tb, st, dev.TOK_WS)   # 7-bit codes: the str.split decoding
        # the lines the device handed back: the stage's own mapper functions, folded with its binop in line order
        binop = self.stage.options.get("binop")
        extra, nrec, max_abs = {}, 0, 0
        if st["fallback"]:
            it = iter(self._fallback_lines(tb, tab))
            for p in _parts(self.stage.mapper):
                it = p.stream(it)
            for k, v in it:
                nrec += 1
                self._check_host_kinds(k, v)
                if not self.float_values:
                    max_abs = max(max_abs, abs(v[0] if self.mean else v))
                elif self.op != dev.OP_SUM_F64 and (v != v or (v == 0 and math.copysign(1.0, v) < 0)):
                    raise NotLowerable("NaN or -0.0 under min/max")   # the result depends on the argument order
                extra[k] = binop(extra[k], v) if k in extra else v
        # Python's ints are unbounded, the table's are 64-bit (SURVEY B12): the bound of _may_overflow
        if self.op == dev.OP_SUM_I64 and (int(st["folded"]) + nrec) * max(int(st["max_abs"]), max_abs) >= (1 << 62):
            raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
        if not self.records:
            self.keys, (self.values,) = _merge_fold_cols(keys, [dev.decode_fold(acc, self.op)], extra, binop)
        else:
            sums = self._record_sums(codes, int(st["records"]))
            if self.mean:
                self.keys, cols = _merge_fold_cols(keys, [sums, acc.view(np.int64)], extra, binop)
                self.values = vexpr.Tup(cols)
            else:
                self.keys, (self.values,) = _merge_fold_cols(keys, [sums], extra, binop)
        self.groups = len(self.keys)
        self.n_lines = int(st["lines"]) + nrec   # one record per line
        self.host_lines = nrec
        if self.preds:   # the table-mode slot, or the records that are neither folded nor handed back
            self.filtered = int(st["records"]) - (int(st["lines"]) + int(st["fallback"]) if self.records else 0)
        return self

    def _fetch_tuple_keys(self, tab, tb):
        """(list of key tuples, accumulators, key codes) of a tuple-key table: one column per component decoded on the
        device, the tuples built in one zip"""
        cols, acc, codes = tab.fetch_field_keys(tb, self.spec[0], self.key_comps)
        cols = [c.astype("U%d" % c.dtype.itemsize).tolist() if c.dtype.kind == "S" else c.tolist() for c in cols]
        return list(zip(*cols)), acc, codes

    def _kind_retry(self, st):
        """True when the scan is to be repeated with other key or value kinds (JSON scans)"""
        return False

    def _check_host_kinds(self, k, v):
        """raise NotLowerable when a host line's key or value would give the device's column another type"""

    def _record_sums(self, codes, n):
        """per table key code (in `codes` order): the sum of its records' values by the stable sort + segmented reduce
        (float64 under OP_SUM_F64, else int64): in line order for a key of at most 4096 lines, by the fixed strided
        tree of single_group_reduce_kernel for a larger one"""
        # dampr_kv_sort_reduce allocates its scratch copy at the buffer's capacity and an output of n records
        if 16 * (self._rec_cap + n) > self._free_bytes():
            raise NotLowerable("the sort scratch of the field records exceeds free device memory")
        kv, self._rec, self._rec_cap = self._rec, None, 0
        try:
            kv.set_size(n)
            # KEY_MIX: packed str codes are far from uniform in their raw bits, and the sort's partitions follow the
            # bits it sorts by. 2*10^7 records of 10^6 "u%07d" keys on an H100: leaf sort 153 ms under KEY_RAW,
            # 1.6 ms under KEY_MIX. The stable sort keeps each key's records in line order either way.
            red = kv.sort_reduce(self.op, dev.KEY_MIX)   # consumes kv
        finally:
            kv.free()
        try:
            rk, rv = red.columns()
        finally:
            red.free()
        real = rk != 0                                  # the holes: key code 0
        rk, rv = rk[real], rv[real]
        order = np.argsort(rk)
        rk, rv = rk[order], rv[order]
        pos = np.searchsorted(rk, codes)
        if len(codes) != len(rk) or (len(codes) and not np.array_equal(rk[np.minimum(pos, len(rk) - 1)], codes)):
            raise NotLowerable("field records and table keys disagree")
        return rv[pos].view(np.float64 if self.op == dev.OP_SUM_F64 else np.int64)


class JsonFieldScan(FieldScan):
    """FieldScan over JSON lines (dampr_text_json_fields): the members of json.loads(line) instead of split fields.

    A bare r["k"] or r["v"] gives whatever Python type the JSON value has. The scan starts with str keys and int values;
    when the device took no line and saw only the other kind (DAMPR_TF_JSON_KEY_KIND / DAMPR_TF_JSON_VAL_KIND), it is
    repeated once with int keys or float values. A bare member of mixed kinds, or a host line whose bare key or value
    has another type than the device's column, sends the stage to the host map."""

    _FLOAT_OPS = {dev.OP_SUM_I64: dev.OP_SUM_F64, dev.OP_MIN_I64: dev.OP_MIN_F64, dev.OP_MAX_I64: dev.OP_MAX_F64}

    def __init__(self, runner, sources, spec, op, stage, mean, preds, members, bare):
        FieldScan.__init__(self, runner, sources, spec, op, stage, mean, preds)
        self.members = members              # the member names the spec and the predicates index
        self.bare_key, self.bare_val = bare
        self._kinds_retried = False

    def _launch(self, tab, tb, lo, hi):
        spec = tuple(self.spec) + (self.op,)
        cr = getattr(self, "_cr_is_data", False)
        if not self.records:
            tab.json_fields(tb, lo, hi, spec, self.members, cr, self.preds)
            return
        if self._rec is None:
            self._records_buffer(min(tb.n // 32 + 4096, self._free_bytes() // (2 * self.REC_BYTES)))
        tab.json_fields_records(tb, lo, hi, spec, self.members, self._rec, cr, self.preds)

    def _fallback_lines(self, tb, tab):
        """the host lines in offset order, a blank one included: it is the empty line json.loads('') raises on (the
        reader's split of a zero-length piece yields no line)"""
        blank = sorted(e >> 16 for e in tab.fallback_lines().tolist() if e & 0xFFFF == 0)
        i = 0
        for off, line in FieldScan._fallback_lines(self, tb, tab):
            while i < len(blank) and blank[i] < off:
                yield blank[i], ""
                i += 1
            yield off, line
        for off in blank[i:]:
            yield off, ""

    def _kind_retry(self, st):
        key = self.bare_key and st["flags"] & dev.TF_JSON_KEY_KIND
        val = self.bare_val and st["flags"] & dev.TF_JSON_VAL_KIND
        if not (key or val):
            return False
        if self._kinds_retried or st["lines"]:
            raise NotLowerable("a bare JSON member of more than one kind")
        self._kinds_retried = True
        sep, ki, kkind, vi = self.spec
        if key:
            kkind = dev.FIELD_KEY_INT
        if val:
            self.op = self._FLOAT_OPS[self.op]
            self.records = self.mean or self.op == dev.OP_SUM_F64
            self.float_values = True
        self.spec = (sep, ki, kkind, vi)
        self._free_records()
        self._rec_regrown = False
        return True

    def _check_host_kinds(self, k, v):
        if self.bare_key and type(k) is not (int if self.spec[2] == dev.FIELD_KEY_INT else str):
            raise NotLowerable("a host line's JSON key has another type than the device's keys")
        if self.bare_val and type(v[0] if self.mean else v) is not (float if self.float_values else int):
            raise NotLowerable("a host line's JSON value has another type than the device's values")


def _key_positions(keys, extra):
    """{key: index into keys} for the keys of `extra` that a device fold's `keys` ('S' array, int64 array or list of
    str) holds"""
    if isinstance(keys, np.ndarray) and keys.dtype.kind == "S":
        W = keys.dtype.itemsize
        fit = [k for k in extra if type(k) is str and k.isascii() and len(k) <= W and "\0" not in k]
        probe = np.array([k.encode("ascii") for k in fit], dtype=keys.dtype)
        hit = np.flatnonzero(np.isin(keys, probe)) if fit and len(keys) else np.zeros(0, dtype=np.int64)
        return {b.decode("ascii"): i for b, i in zip(keys[hit].tolist(), hit.tolist())}
    if isinstance(keys, np.ndarray):
        fit = [k for k in extra if type(k) is int]
        probe = np.array(fit, dtype=np.int64)
        hit = np.flatnonzero(np.isin(keys, probe)) if fit and len(keys) else np.zeros(0, dtype=np.int64)
        return dict(zip(keys[hit].tolist(), hit.tolist()))
    return {k: i for i, k in enumerate(keys)}


def _append_keys(keys, new):
    """keys (as _key_positions) followed by the keys `new`, in the cheapest representation that holds them all"""
    if isinstance(keys, np.ndarray) and keys.dtype.kind == "S" and \
            all(type(k) is str and k.isascii() and len(k) <= keys.dtype.itemsize and "\0" not in k for k in new):
        return np.concatenate((keys, np.array([k.encode("ascii") for k in new], dtype=keys.dtype)))
    if isinstance(keys, np.ndarray) and keys.dtype.kind == "i" and all(type(k) is int for k in new):
        return np.concatenate((keys, np.array(new, dtype=np.int64)))
    return Frame._pylist(keys) + new


def _merge_fold_cols(keys, cols, extra, binop):
    """(keys, value columns) of a device fold plus {key: value} folded on the host: a key present in both gets
    binop(device value, host value). The columns are one int64 or float64 column, or mean()'s (sum, count) pairs
    (int64 or float64 sums, int64 counts); `keys` is an 'S' array, an int64 array, or a list of str or of tuples of
    str and int. An int64 column must hold every host-folded value as well as every merged one, and every int key or
    key component must be an int64."""
    if not extra:
        return keys, cols
    if any(type(c) is int and not -(1 << 63) <= c < (1 << 63) for k in extra for c in (k if type(k) is tuple else (k,))):
        raise NotLowerable("a host-folded key outside int64")
    cols = [np.array(c, copy=True) for c in cols]

    def parts(v):
        return tuple(v) if len(cols) > 1 else (v,)

    def fits(xs, c):
        if c.dtype == np.float64:
            return all(type(x) is float for x in xs)
        return all(type(x) is int and -(1 << 63) <= x < (1 << 63) for x in xs)

    # checked before the merge: a 20-digit host value under min or max sends the stage to the host even when the
    # device value of its key is the one the merge keeps
    if not all(fits([x], c) for v in extra.values() for x, c in zip(parts(v), cols) if c.dtype == np.int64):
        raise NotLowerable("a host-folded value outside int64")
    pos = _key_positions(keys, extra)
    new = []
    for k, v in extra.items():
        i = pos.get(k) if type(k) in (str, int) or (type(k) is tuple and all(type(c) in (str, int) for c in k)) \
            else None
        if i is None:
            new.append(k)
            continue
        dv = cols[0][i].item() if len(cols) == 1 else tuple(c[i].item() for c in cols)
        r = parts(binop(dv, v))
        if len(r) != len(cols) or not all(fits([x], c) for x, c in zip(r, cols)):
            raise NotLowerable("a merged value the device columns do not hold")
        for x, c in zip(r, cols):
            c[i] = x
    if not new:
        return keys, cols
    nv = [[parts(extra[k])[j] for k in new] for j in range(len(cols))]
    if not all(len(parts(extra[k])) == len(cols) for k in new) or not all(fits(x, c) for x, c in zip(nv, cols)):
        raise NotLowerable("a host-folded value the device columns do not hold")
    return _append_keys(keys, new), [np.concatenate((c, np.array(x, dtype=c.dtype))) for c, x in zip(cols, nv)]


def _source_key(sources):
    out = []
    for kind, p in sources:
        if kind == "mem":
            out.append(("mem", id(p), len(p)))
        elif kind == "dev":
            out.append(("dev", id(p), p.n))
        else:
            st = os.stat(p)
            out.append(("file", p, st.st_size, st.st_mtime_ns))
    return tuple(out)


# ---- stage matchers -----------------------------------------------------------------------------------
def _parts(mapper):
    if isinstance(mapper, ops.FusedMapper):
        return mapper.parts()
    return [mapper]


def _opkinds(mapper):
    """[(kind, Op)] for a mapper made only of DSL-generated Maps, else None."""
    out = []
    for p in _parts(mapper):
        op = getattr(p, "op", None)
        if not isinstance(p, (ops.Map, ops.StreamMapper)) or op is None:
            return None
        out.append((op.kind, op))
    return out


def _match_text_count(stage, inputs):
    """flat_map(tokeniser) -> keyed(identity, const 1) + PartialReduceCombiner(add) over text."""
    if not isinstance(stage, GMap) or len(inputs) != 1:
        return None
    src = _text_files(inputs[0])
    if src is None:
        return None
    ks = _opkinds(stage.mapper)
    if ks is None or [k for k, _ in ks] != ["flat_map", "keyed"]:
        return None
    mode = lowering.tokenizer_mode(ks[0][1].fn)
    if mode is None:
        return None
    keyed = ks[1][1]
    if not lowering.is_identity(keyed.fn):
        return None
    ok, v = lowering.constant_value(keyed.fn2)
    if not ok or v != 1 or type(v) is not int:
        return None
    if not isinstance(stage.combiner, ops.PartialReduceCombiner):
        return None
    if lowering.binop_kind(stage.options.get("binop")) != lowering.ADD:
        return None
    return src, mode


KEY_TUPLE = "tuple"   # the key kind of a field scan's spec whose key is a tuple of fields


def _match_text_fields(stage, inputs, programs=False):
    """filter* [map(l.split(S) | l.split()) filter*] keyed(field key, 1 | int(field) | float(field)) +
    PartialReduceCombiner(+ | min | max), or mean()'s keyed(field key, (int(field) | float(field), 1)) + component-wise
    (+, +), over text, each filter one lowering.field_predicate on the key's separator: (sources, (sep byte or
    FIELD_SEP_WS, key index, key kind, value index or FIELD_VAL_ONE), op, mean, device predicates) or None. A tuple
    key of field projections has key kind KEY_TUPLE and, as its key index, the components ((index, FIELD_KEY_STR |
    FIELD_KEY_INT), ...). A sixth element is the stage's computed key / value programs (lowering.text_fields_expr, in
    device.field_expr form) for the shapes text_fields_spec refuses, else None: the map may then also compute an
    expression or a tuple of them (no filter may follow such a map), a key program's keys are FIELD_KEY_INT keys.
    With `programs` each filter may be a lowering.filter_program (and / or / not, string tests, whole-line tests): the
    device predicates are then the stage's postfix program (_device_program), the same 4-tuples as without it when no
    filter needs more than one leaf of field_predicate's shapes."""
    if not isinstance(stage, GMap) or len(inputs) != 1:
        return None
    src = _text_files(inputs[0])
    if src is None:
        return None
    ks = _opkinds(stage.mapper)
    kinds = [k for k, _ in ks] if ks is not None else []
    if not kinds or kinds[-1] != "keyed" or any(k not in ("filter", "map") for k in kinds[:-1]) or \
            kinds.count("map") > 1:
        return None
    if not isinstance(stage.combiner, ops.PartialReduceCombiner):
        return None
    keyed = ks[-1][1]
    at = kinds.index("map") if "map" in kinds else None
    mapfn = ks[at][1].fn if at is not None else None
    spec = lowering.text_fields_spec(keyed.fn, keyed.fn2, mapfn, whitespace=True, tuple_keys=True)
    expr = None
    if spec is None:
        spec = lowering.text_fields_expr(keyed.fn, keyed.fn2, mapfn)
        if spec is None:
            return None
        msep = lowering.split_of(mapfn) if at is not None else None
        if at is not None and msep is None and "filter" in kinds[at + 1:]:
            return None   # a filter over the computed record of the map: not a field predicate
        spec, expr = spec[:6], spec[6]
        if spec[0] is None and msep is not None:
            spec = (msep,) + spec[1:]
    sep, ki, kkind, vi, vkind, mean = spec
    if kkind == lowering.FIELD_TUPLE:
        ki = tuple((i, dev.FIELD_KEY_INT if k == lowering.FIELD_INT else dev.FIELD_KEY_STR) for i, k in ki)
    preds = []
    for i, (k, o) in enumerate(ks[:-1]):
        if k == "filter":
            rec = sep if at is not None and i > at else None
            p = lowering.field_predicate(o.fn, rec, whitespace=True)
            prog = [p] if p is not None else lowering.filter_program(o.fn, rec, whitespace=True) if programs else None
            if prog is None:
                return None
            for p in prog:
                if isinstance(p, str) or p[2] == lowering.LINE:
                    continue
                if sep is None:   # a computed key and value that read no field: the filters' split
                    sep = p[0]
                if p[0] != sep:
                    return None
            preds += _device_program(prog)
    if not _preds_fit(preds):
        return None
    binop = stage.options.get("binop")
    if mean:
        if lowering.tuple_binop_kinds(binop) != [lowering.ADD, lowering.ADD]:
            return None
        op = dev.OP_SUM_F64 if vkind == lowering.FIELD_FLOAT else dev.OP_SUM_I64
    else:
        kind = lowering.binop_kind(binop)
        if kind not in (lowering.ADD, lowering.MIN, lowering.MAX):
            return None
        op = (_FOLD_OPS_F64 if vkind == lowering.FIELD_FLOAT else _FOLD_OPS)[kind]
    if expr is not None:
        kp, vp, ci, cf, loads = expr
        types = {"i": dev.EXPR_INT, "f": dev.EXPR_F64}
        expr = (None if kp is None else (types[kp[0]], tuple(kp[1])), None if vp is None else (types[vp[0]], tuple(vp[1])),
                tuple(ci), tuple(cf), tuple(loads))
        ki = 0 if ki is None else ki      # (the programs replace the spec's key and value fields)
        vi = 0 if vi == lowering.FIELD_EXPR else vi
        sep = "," if sep is None else sep   # nothing is split: any separator
    return src, (dev.FIELD_SEP_WS if sep == lowering.SEP_WS else ord(sep), ki,
                 KEY_TUPLE if kkind == lowering.FIELD_TUPLE else
                 dev.FIELD_KEY_INT if kkind == lowering.FIELD_INT else dev.FIELD_KEY_STR,
                 dev.FIELD_VAL_ONE if vi is None else vi), op, mean, tuple(preds), expr


def _match_json_fields(stage, inputs, programs=False, paths=False):
    """map(json.loads) filter* keyed(r["k"] | int(r["k"]), 1 | r["v"] | int(r["v"]) | float(r["v"])) +
    PartialReduceCombiner(+ | min | max), or mean()'s keyed(key, (value, 1)) + component-wise (+, +), over text, each
    filter one lowering.json_predicate: (sources, (FIELD_SEP_JSON, key member, key kind, value member or FIELD_VAL_ONE),
    op, mean, device predicates, member names, (bare key, bare value)) or None. With `programs` each filter may be a
    lowering.json_filter_program, as _match_text_fields takes filter programs. With `paths`, a stage that does not
    match so may read member paths in its key, value and filters (lowering.json_fields_path_spec,
    lowering.json_path_filter_program, which every filter of such a stage prefers): a member is then the tuple of its
    names (a one-name path is its name), at most dev.JSON_MAX_NODES distinct path nodes. "m" in r[n1]..[nk] also lists
    its container r[n1]..[nk], whose str the device tests for the substring."""
    m = _match_json_stage(stage, inputs, programs, False)
    return m if m is not None or not paths else _match_json_stage(stage, inputs, programs, True)


def _match_json_stage(stage, inputs, programs, nested):
    """_match_json_fields' match of stage: of the top-level members only, or (nested) of member paths"""
    if not isinstance(stage, GMap) or len(inputs) != 1:
        return None
    src = _text_files(inputs[0])
    if src is None:
        return None
    ks = _opkinds(stage.mapper)
    kinds = [k for k, _ in ks] if ks is not None else []
    if len(kinds) < 2 or kinds[0] != "map" or kinds[-1] != "keyed" or any(k != "filter" for k in kinds[1:-1]):
        return None
    if not lowering.is_json_loads(ks[0][1].fn) or not isinstance(stage.combiner, ops.PartialReduceCombiner):
        return None
    keyed = ks[-1][1]
    spec = lowering.json_fields_spec(keyed.fn, keyed.fn2)
    if spec is None and nested:
        spec = lowering.json_fields_path_spec(keyed.fn, keyed.fn2)
    if spec is None:
        return None
    kname, kkind, vname, vkind, mean = spec
    members = []

    def member(name):
        if isinstance(name, tuple) and len(name) == 1:
            name = name[0]
        if name not in members:
            members.append(name)
        return members.index(name)

    ki = member(kname)
    vi = dev.FIELD_VAL_ONE if vname is None else member(vname)
    preds = []
    for _k, o in ks[1:-1]:
        prog = lowering.json_path_filter_program(o.fn) if nested else None
        if prog is None:
            p = lowering.json_predicate(o.fn)
            prog = [p] if p is not None else lowering.json_filter_program(o.fn) if programs else None
        if prog is None:
            return None
        for p in prog:
            if isinstance(p, str):
                preds.append((_PRED_OPS[p], 0, dev.CMP_EQ, ()))
                continue
            kind, name, cmp, consts = p
            preds.append((dev.PRED_MEMBER if kind == lowering.FIELD_MEMBER else _PRED_KINDS[kind], member(name),
                          _PRED_CMPS.get(cmp, dev.CMP_EQ), consts))
            if kind == lowering.FIELD_MEMBER and consts:   # the container, for the substring test of a str
                member(name[:-1])
    if nested and not any(isinstance(m, tuple) for m in members):
        return None
    if len(members) > dev.JSON_MAX_MEMBERS or not _preds_fit(preds) or \
            len({m[:i] for m in members if isinstance(m, tuple) for i in range(1, len(m) + 1)} |
                {(m,) for m in members if isinstance(m, str)}) > dev.JSON_MAX_NODES:
        return None
    binop = stage.options.get("binop")
    if mean:
        if lowering.tuple_binop_kinds(binop) != [lowering.ADD, lowering.ADD]:
            return None
        op = dev.OP_SUM_F64 if vkind == lowering.FIELD_FLOAT else dev.OP_SUM_I64
    else:
        kind = lowering.binop_kind(binop)
        if kind not in (lowering.ADD, lowering.MIN, lowering.MAX):
            return None
        op = (_FOLD_OPS_F64 if vkind == lowering.FIELD_FLOAT else _FOLD_OPS)[kind]
    return src, (dev.FIELD_SEP_JSON, ki, dev.FIELD_KEY_INT if kkind == lowering.FIELD_INT else dev.FIELD_KEY_STR,
                 vi), op, mean, tuple(preds), tuple(members), \
        (kkind == lowering.FIELD_DATA, vkind == lowering.FIELD_DATA)


_PRED_KINDS = {lowering.FIELD_STR: dev.PRED_STR, lowering.FIELD_INT: dev.PRED_INT, lowering.FIELD_FLOAT: dev.PRED_F64,
               lowering.FIELD_COUNT: dev.PRED_NFIELDS, lowering.FIELD_LEN: dev.PRED_LEN,
               lowering.FIELD_NONBLANK: dev.PRED_NONBLANK}
_PRED_CMPS = {"==": dev.CMP_EQ, "!=": dev.CMP_NE, "<": dev.CMP_LT, "<=": dev.CMP_LE, ">": dev.CMP_GT, ">=": dev.CMP_GE,
              "in": dev.CMP_IN, "not in": dev.CMP_NOT_IN, "contains": dev.CMP_CONTAINS,
              "not contains": dev.CMP_NOT_CONTAINS, "startswith": dev.CMP_STARTS, "endswith": dev.CMP_ENDS}
_PRED_OPS = {"and": dev.PRED_AND, "or": dev.PRED_OR, "not": dev.PRED_NOT}


def _device_pred(p):
    """(PRED_*, field, CMP_*, constants) of a lowering.field_predicate or a filter_program leaf"""
    _sep, kind, i, op, consts = p
    return _PRED_KINDS[kind], dev.FIELD_LINE if i == lowering.LINE else 0 if i is None else i, \
        _PRED_CMPS.get(op, dev.CMP_EQ), consts


def _device_program(prog):
    """device predicates of a lowering.filter_program (connectives as PRED_AND / PRED_OR / PRED_NOT entries)"""
    return [(_PRED_OPS[p], 0, dev.CMP_EQ, ()) if isinstance(p, str) else _device_pred(p) for p in prog]


def _preds_fit(preds):
    """a stage's device predicates are within the device's limits per call"""
    ops = sum(p[0] in (dev.PRED_AND, dev.PRED_OR, dev.PRED_NOT) for p in preds)
    return len(preds) - ops <= dev.PRED_MAX and ops <= dev.PRED_MAX_OPS and \
        sum(len(p[3]) for p in preds) <= dev.PRED_MAX_CONSTS and \
        sum(len(c.encode("utf-8")) for p in preds if p[0] == dev.PRED_STR for c in p[3]) <= dev.PRED_MAX_BYTES


_FIELD_OP_NAMES = {dev.OP_SUM_I64: "sum_i64", dev.OP_MIN_I64: "min_i64", dev.OP_MAX_I64: "max_i64",
                   dev.OP_SUM_F64: "sum_f64", dev.OP_MIN_F64: "min_f64", dev.OP_MAX_F64: "max_f64"}


def _match_line_count(stage, inputs):
    if not isinstance(stage, GMap) or len(inputs) != 1:
        return None
    ks = _opkinds(stage.mapper)
    if ks is None or [k for k, _ in ks] != ["count_records"]:
        return None
    return True


def text_scan(runner, src, mode):
    # memoised per graph execution only: the same file is scanned once for len() and count()
    cache = runner.__dict__.setdefault("_scan_cache", {})
    key = (_source_key(src), mode)
    hit = cache.get(key)
    if hit is not None:
        return hit
    scan = TextScan(runner, src, mode).run()
    cache[key] = scan
    return scan


def _future_text_count(runner, si, source):
    """A later stage that tokenises the same text: its scan also yields the line count."""
    for st in runner.graph.stages[si + 1:]:
        if isinstance(st, GMap) and len(st.inputs) == 1 and st.inputs[0] == source:
            inp = [runner.graph.inputs.get(st.inputs[0])]
            if inp[0] is None:
                continue
            m = _match_text_count(st, inp)
            if m is not None:
                return m
    return None


def try_lower(runner, stage, inputs, si, data):
    try:
        if isinstance(stage, GMap):
            return _lower_map(runner, stage, inputs, si)
        if isinstance(stage, GReduce):
            if len(inputs) == 2:
                return _lower_join(runner, stage, inputs)
            return _lower_reduce(runner, stage, inputs)
        if isinstance(stage, GSink):
            return _lower_sink(runner, stage, inputs)
    except NotLowerable as e:
        log.warning("stage %s not lowered (%s): running as host map + device shuffle", stage.output, e)
    return None


# ---- map stages ------------------------------------------------------------------------------------------
def _lower_map(runner, stage, inputs, si):
    m = _match_text_count(stage, inputs)
    if m is not None:
        src, mode = m
        scan = text_scan(runner, src, mode)
        words, counts = scan.words, scan.counts
        extra = []
        if mode != dev.TOK_WS and scan.empty:
            if isinstance(words, np.ndarray):
                words = np.concatenate((words, np.array([b""], dtype=words.dtype)))
            else:
                words = words + [""]
            extra = [scan.empty]
            counts = np.concatenate((counts, np.array(extra, dtype=np.int64)))
        # a cross or a sink that dictionary-encodes this column gets the dictionary built on the device
        remember_count_dictionary(counts, lambda: scan.count_dictionary(extra))
        f = Frame(words, [counts], scalar=True, combined=True)
        runner.stats.add(stage, "device text tokenise+combine",
                         "bytes=%d terms=%d lines=%d" % (scan.nbytes, len(words), scan.n_lines))
        return f
    m = _match_text_fields(stage, inputs, programs=True)
    if m is not None:
        if dist.active():
            raise NotLowerable("the field scan runs on one process")
        src, spec, op, mean, preds, expr = m
        scan = FieldScan(runner, src, spec, op, stage, mean, preds, expr).run()
        opname = ("mean_f64" if op == dev.OP_SUM_F64 else "mean_i64") if mean else \
            "count" if spec[3] == dev.FIELD_VAL_ONE and op == dev.OP_SUM_I64 and (expr is None or expr[1] is None) \
            else _FIELD_OP_NAMES[op]
        detail = "op=%s bytes=%d lines=%d groups=%d host_lines=%d" % (opname, scan.nbytes, scan.n_lines, scan.groups,
                                                                      scan.host_lines)
        if preds:
            detail += " filtered=%d" % scan.filtered
        if spec[0] == dev.FIELD_SEP_WS:
            detail += " sep=ws"
        if spec[2] == KEY_TUPLE:
            detail += " key=tuple%d" % len(spec[1])
        if expr is not None and expr[1] is not None:
            detail += " value=expr"
        if expr is not None and expr[0] is not None:
            detail += " key=const" if len(expr[0][1]) == 1 and expr[0][1][0] & 0xFF == lowering.EV_CI else " key=expr"
        runner.stats.add(stage, "device text fields scan+combine", detail)
        return Frame(scan.keys, [scan.values], scalar=True, combined=True)
    m = _match_json_fields(stage, inputs, programs=True, paths=True)
    if m is not None:
        if dist.active():
            raise NotLowerable("the JSON field scan runs on one process")
        src, spec, op, mean, preds, members, bare = m
        scan = JsonFieldScan(runner, src, spec, op, stage, mean, preds, members, bare).run()
        op, spec = scan.op, scan.spec   # after a kind retry
        opname = ("mean_f64" if op == dev.OP_SUM_F64 else "mean_i64") if mean else \
            "count" if spec[3] == dev.FIELD_VAL_ONE and op == dev.OP_SUM_I64 else _FIELD_OP_NAMES[op]
        detail = "op=%s bytes=%d lines=%d groups=%d host_lines=%d" % (opname, scan.nbytes, scan.n_lines, scan.groups,
                                                                      scan.host_lines)
        if preds:
            detail += " filtered=%d" % scan.filtered
        detail += " sep=json"
        nested = [p for p in members if isinstance(p, tuple)]
        if nested:   # the longest member path, its names joined by '.'
            detail += " path=" + ".".join(max(nested, key=len))
        runner.stats.add(stage, "device text fields scan+combine", detail)
        return Frame(scan.keys, [scan.values], scalar=True, combined=True)
    if _match_line_count(stage, inputs):
        ds = inputs[0]
        src = _text_files(ds)
        if src is not None:
            fut = _future_text_count(runner, si, stage.inputs[0])
            mode = fut[1] if fut is not None else dev.TOK_WS
            scan = text_scan(runner, src, mode)
            if scan.has_cr:
                # text mode reads with universal newlines (dataset.py:458-476): '\r' and '\r\n' end lines too
                raise NotLowerable("carriage returns: the line count needs universal-newline semantics")
            runner.stats.add(stage, "device line count (tokenise kernel by-product)", "lines=%d" % scan.n_lines)
            if scan.nbytes == 0:
                # no bytes, no chunks, no count record: len() of an empty text input is an empty collection in
                # the reference (dampr.py:245-275), not [0]
                return RecordsDataset([], [], replicated=True)
            return RecordsDataset([1], [scan.n_lines], replicated=True)
        kvc = _kv_columns(ds)
        if kvc is not None:
            # binary (key, value) records: the input is the same on every rank, its length needs no pass at all
            n = len(kvc[0])
            runner.stats.add(stage, "record count of a columnar input", "records=%d" % n)
            return RecordsDataset([1], [n], replicated=True) if n else RecordsDataset([], [], replicated=True)
        if isinstance(ds, (Frame, RecordsDataset)):
            n = len(ds)
            if dist.active():
                # results are owner-partitioned over the ranks: the length is the sum of the shards
                n = int(dist.all_reduce_sum_int([n])[0])
            runner.stats.add(stage, "frame length", "records=%d" % n)
            return RecordsDataset([1], [n], replicated=True)
        return None
    kv = _lower_kv_map(runner, stage, inputs)
    if kv is not None:
        return kv
    if len(inputs) == 1 and not isinstance(inputs[0], Frame) and not dist.active():
        # binary (key, value) records under a stage _lower_kv_map does not take (a map / filter chain in front of the
        # fold, mean(), topk ...): the two columns are a frame of (key, value) rows, and whatever a frame can do
        # column-at-a-time applies — no per-record Python over hundreds of millions of records
        kvc = _kv_columns(inputs[0])
        if kvc is not None and len(kvc[0]):
            fr = Frame(None, [kvc[0], kvc[1]], scalar=False)
            out = _lower_frame_map(runner, stage, fr)
            if out is None:
                out = _lower_frame_general(runner, stage, fr)
            if out is not None:
                return out
    if len(inputs) == 1 and isinstance(inputs[0], Frame):
        out = _lower_frame_map(runner, stage, inputs[0])
        if out is None and not isinstance(inputs[0], LazyKVFrame):
            out = _lower_frame_general(runner, stage, inputs[0])
        return out
    if isinstance(stage.mapper, ops.MapCrossJoin) and len(inputs) == 2 and isinstance(inputs[0], Frame):
        return _lower_cross(runner, stage, inputs)
    if isinstance(stage.mapper, ops.MapAllJoin) and len(inputs) == 2:
        return _lower_probe(runner, stage, inputs)
    return None


def _kv_columns(ds):
    if isinstance(ds, (KVInput, ArrayKVInput)) or hasattr(ds, "columns"):
        try:
            return ds.columns()
        except Exception:
            return None
    return None


_FOLD_OPS = {lowering.ADD: dev.OP_SUM_I64, lowering.MIN: dev.OP_MIN_I64, lowering.MAX: dev.OP_MAX_I64,
             lowering.FIRST: dev.OP_FIRST, lowering.LAST: dev.OP_LAST}


def _key_xform_for(col):
    if col.dtype == np.int64:
        return dev.KEY_I64
    return dev.KEY_F64 if col.dtype == np.float64 else dev.KEY_RAW


def _float_keys(col):
    """A float64 key column as Python compares keys: (col + 0.0, the key its 0.0 group reports), or None when the
    column holds a NaN (NaN != NaN: no sort or grouping of bit patterns gives Python's answer). -0.0 == 0.0 are
    one key, and a group reports the key of its first record in input order, as the reference does."""
    if np.isnan(col).any():
        return None
    zero = np.flatnonzero(col == 0)
    return col + 0.0, (col[zero[0]] if len(zero) else np.float64(0.0))


def _report_zero(keys, rep):
    """group keys of a column normalised by _float_keys, with the 0.0 group relabelled to the key it reports"""
    if np.signbit(rep):
        keys = keys.copy()
        keys[keys == 0] = rep
    return keys


def _lower_kv_map(runner, stage, inputs):
    """keyed(x[0], x[1]) over binary (key, value) records."""
    if len(inputs) != 1:
        return None
    cols = _kv_columns(inputs[0])
    if cols is None:
        return None
    ks = _opkinds(stage.mapper)
    if ks is None or [k for k, _ in ks] != ["keyed"]:
        return None
    kp = lowering.projection(ks[0][1].fn)
    vp = lowering.projection(ks[0][1].fn2)
    if kp is None or vp is None or kp[0] != "field" or kp[1] not in (0, 1):
        return None
    if vp[0] == "ident":
        # sort_by(lambda x: +-x[i]) (or group_by with the whole record as value): one device sort of the
        # records on that field; rows come back as a two-column frame in key order (stable)
        if stage.combiner is not None:
            return None
        col, other = cols[kp[1]], cols[1 - kp[1]]
        if col.dtype == np.float64:
            # sorted on the normalised key with the record positions as values: -0.0 and 0.0 tie (input order
            # kept), and the rows are gathered from the input, so a -0.0 field stays -0.0
            fk = _float_keys(-col if kp[2] < 0 else col)
            if fk is None:
                return None
            kn, rep = fk
            _k, perm, how = _device_group(runner, kn.view(np.uint64), np.arange(len(col), dtype=np.uint64), None,
                                          dev.KEY_F64)
            perm = perm.view(np.int64)
            rk, ro = col[perm], other[perm]
            f = Frame(_report_zero(kn[perm], rep), [rk, ro] if kp[1] == 0 else [ro, rk], scalar=False, combined=False)
            runner.stats.add(stage, "device kv partition+sort of whole records" + how, "records=%d" % len(col))
            return f
        if kp[2] < 0:
            if col.dtype != np.int64 or (len(col) and int(col.min()) == -(1 << 63)):
                return None
            kcol = -col
        else:
            kcol = col
        rk, rv, how = _device_group(runner, kcol, other, None, _key_xform_for(kcol))
        rk, rv = rk.view(kcol.dtype), rv.view(other.dtype)
        orig = -rk if kp[2] < 0 else rk
        f = Frame(rk, [orig, rv] if kp[1] == 0 else [rv, orig], scalar=False, combined=False)
        runner.stats.add(stage, "device kv partition+sort of whole records" + how, "records=%d" % len(col))
        return f
    if kp[2] != 1:
        return None
    keys = cols[kp[1]]
    rep = None
    if keys.dtype == np.float64:
        fk = _float_keys(keys)
        if fk is None:
            return None
        keys, rep = fk
    count_only = False
    if vp[0] == "field" and vp[2] == 1 and vp[1] in (0, 1):
        vals = cols[vp[1]]
    elif vp[0] == "const" and type(vp[1]) is int:
        vals = np.full(len(keys), vp[1], dtype=np.int64)
        count_only = vp[1] == 1
    else:
        return None
    ctx = runner.ctx
    binop = stage.options.get("binop")
    n = len(keys)
    if isinstance(stage.combiner, ops.PartialReduceCombiner) and callable(binop):
        kind = lowering.binop_kind(binop)
        if kind not in _FOLD_OPS or vals.dtype not in (np.int64, np.uint64):
            return None
        if vals.dtype == np.uint64 and len(vals) and int(vals.max()) >= (1 << 63):
            return None   # the device folds are signed 64-bit: values >= 2^63 would compare / add as negatives
        # the overflow bound of a sum scans every value (numpy, GIL released): on a large input it runs on a host
        # thread next to the upload + device fold and vetoes the result afterwards
        late = kind == lowering.ADD and n >= _LATE_OVERFLOW_MIN and not count_only and not dist.active()
        if kind == lowering.ADD and n and not late and _may_overflow(vals):
            raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
        op = dev.OP_COUNT if (count_only and kind == lowering.ADD) else _FOLD_OPS[kind]
        chk = _Background(_may_overflow, vals) if late else None
        try:
            rk, rv, how = _device_group(runner, keys, vals, op, dev.KEY_MIX)
        finally:
            overflow = chk.result() if chk is not None else False
        if overflow:
            raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
        rk = rk.view(keys.dtype)
        f = Frame(rk if rep is None else _report_zero(rk, rep), [rv.view(np.int64)], scalar=True, combined=True)
        runner.stats.add(stage, "device kv partition+sort+segmented-reduce" + how, "records=%d groups=%d" % (n, len(rk)))
        return f
    if stage.combiner is None:
        # group_by: the partition + sort is deferred until somebody reads the grouped records; when the
        # only consumer is a lowered reduce (sum(it), len, min, max) the sort and the fold run as ONE
        # device pass (or one spill pipeline) over the original columns. Its consumers (fused reduces, unique,
        # joins) report the normalised keys, so a 0.0 group whose first key is -0.0 is left to the host
        if rep is not None and np.signbit(rep):
            return None
        f = LazyKVFrame(runner, keys, vals, _key_xform_for(keys))
        f.meta["sorted_kv"] = True
        runner.stats.add(stage, "device kv partition+sort (deferred until read; fused into a lowered reduce)",
                         "records=%d" % n)
        return f
    return None


class LazyKVFrame(Frame):
    """Grouped kv records whose device sort happens on first access."""

    def __init__(self, runner, keys, vals, xform):
        self._runner, self._rk, self._rv, self._xf = runner, keys, vals, xform
        self._done = False
        self.scalar, self.combined, self.meta = True, False, {}
        self.n = len(keys)

    def raw(self):
        return self._rk, self._rv

    def _materialise(self):
        if not self._done:
            rk, rv, how = _device_group(self._runner, self._rk, self._rv, None, self._xf)
            self._keys = rk.view(self._rk.dtype)
            self._cols = [rv.view(self._rv.dtype)]
            self._done = True
            self.meta["how"] = how

    @property
    def keys(self):
        self._materialise()
        return self._keys

    @keys.setter
    def keys(self, v):
        self._keys = v

    @property
    def cols(self):
        self._materialise()
        return self._cols

    @cols.setter
    def cols(self, v):
        self._cols = v

    def delete(self):
        self._rk = self._rv = None
        self._keys, self._cols, self._done, self.n = None, [[]], True, 0


_LATE_OVERFLOW_MIN = 1 << 24   # records from which the overflow bound of a sum runs next to the device work


class _Background(object):
    """fn(*args) on a host thread (numpy reductions release the GIL); result() joins."""

    def __init__(self, fn, *args):
        import threading
        self._out, self._err = None, None

        def work():
            try:
                self._out = fn(*args)
            except BaseException as e:
                self._err = e
        self._th = threading.Thread(target=work, name="dampr-background")
        self._th.start()

    def result(self):
        self._th.join()
        if self._err is not None:
            raise self._err
        return self._out


def _may_overflow(vals):
    """Cheap bound for Python-int semantics (SURVEY B12): n * max|v| must stay far below 2^63."""
    n = len(vals)
    if n > (1 << 24):
        # numpy reductions release the GIL: a few threads keep this memory-bound scan off the critical path
        from concurrent.futures import ThreadPoolExecutor
        step = -(-n // 8)
        with ThreadPoolExecutor(8) as ex:
            parts = list(ex.map(lambda i: (int(vals[i:i + step].min()), int(vals[i:i + step].max())), range(0, n, step)))
        lo, hi = min(p[0] for p in parts), max(p[1] for p in parts)
    else:
        lo, hi = int(vals.min()), int(vals.max())
    return n * max(abs(lo), abs(hi)) >= (1 << 62)


def _device_group(runner, keys, vals, op, xform):
    """Group (and fold, when op is given) kv columns on the device: in core when the records fit the
    device arena, otherwise through the spill path (spill.py). Returns (keys, vals, how)."""
    from . import spill
    ctx = runner.ctx
    n = len(keys)
    if op is not None and dist.active():
        # kv inputs are global: every rank folds its record range, one all-to-all moves each key to its
        # owner (dist.shuffle_kv), the owner finishes the fold. Runs arrive in rank order and the device
        # sort is stable, so FIRST/LAST keep their input-order meaning.
        r, w = dist.world()
        lo, hi = n * r // w, n * (r + 1) // w
        kv = ctx.kv_from_columns(keys[lo:hi], vals[lo:hi])
        try:
            part = kv.sort_reduce(op, dev.KEY_MIX, sorted_run=True)
        finally:
            kv.free()
        recv, offs, _h = dist.shuffle_kv(ctx, part)   # `part` is sorted by the mixed key: sorted runs arrive
        part.free()
        op2 = dev.OP_SUM_I64 if op == dev.OP_COUNT else op
        red = ctx.kv_merge_ranges(recv, offs, dev.KEY_MIX, op2)   # runs in rank order: FIRST / LAST keep their meaning
        recv.free()
        try:
            rk, rv = red.columns()
        finally:
            red.free()
        return rk, rv, " [rank %d/%d: local fold, all-to-all, owner fold]" % (r, w)
    if n and spill.needs_spill(ctx, n):
        step = 1 << 24
        chunks = ((keys[i:i + step], vals[i:i + step]) for i in range(0, n, step))
        if op is None and xform != dev.KEY_MIX:
            samp = keys[np.random.default_rng(0).integers(0, n, size=min(n, 1 << 16))]
            pieces, st = spill.external_sort(ctx, chunks, n, xform, samp)
        else:
            pieces, st = spill.external_group(ctx, chunks, n, op, xform if op is None else dev.KEY_MIX)
        if len(pieces) == 1:    # external_group writes its result columns in place: nothing to concatenate
            rk, rv = pieces[0]
        else:
            rk = np.concatenate([p[0] for p in pieces]) if pieces else np.zeros(0, dtype=np.uint64)
            rv = np.concatenate([p[1] for p in pieces]) if pieces else np.zeros(0, dtype=np.uint64)
        runner.stats.spill = st
        return rk, rv, " [spilled: %d buckets, %d batches, arena %d MB]" % (
            st["buckets"], st["batches"], st["arena_bytes"] >> 20)
    kv = ctx.kv_from_columns(keys, vals)
    try:
        if op is None:
            kv.sort(xform)
            rk, rv = kv.columns()
        else:
            red = kv.sort_reduce(op, xform)
            try:
                rk, rv = red.columns()
            finally:
                red.free()
    finally:
        kv.free()
    return rk, rv, ""


def _numeric(col):
    return isinstance(col, np.ndarray) and col.dtype.kind in "iuf" and col.dtype.itemsize == 8


def _lower_topk(runner, stage, frame, op):
    """topk(k, value) over a columnar frame (dampr.py:621-652): value = +-x[i] / +-x on a numeric column. One
    device sort of (score, row) finds the k-th largest score; the rows at or above it (a superset of the answer
    when scores tie at the boundary) become the candidates, cut to k by the reference's own (value(x), x) tuple
    order on the host. Emits what map_topk emits: (1, (value(x), x)) for the surviving rows — the stage's
    partition_reduce (heapq.nlargest over all candidates) then runs unchanged on at most k records."""
    import heapq
    value, k = op.fn, op.fn2
    if dist.active() or not isinstance(k, int) or isinstance(k, bool) or stage.combiner is not None:
        return None
    kp = lowering.projection(value)
    if kp is None:
        return None
    if kp[0] == "field" and not frame.scalar and kp[1] < len(frame.cols):
        col = frame.cols[kp[1]]
    elif kp[0] == "ident" and frame.scalar:
        col = frame.cols[0]
    else:
        return None
    if isinstance(col, DictCol):
        col = col.materialize()
    if not _numeric(col) or col.dtype.kind not in "if" or (col.dtype.kind == "f" and np.isnan(col).any()):
        return None   # NaN scores make the heap order depend on the arrival order
    n = frame.n
    if k <= 0 or n == 0:
        runner.stats.add(stage, "device top-k candidates", "records=%d k=%d candidates=0" % (n, k))
        return RecordsDataset([], [])
    sign = kp[2]
    if col.dtype.kind == "f":
        if sign < 0 and (col == 0).any():
            return None   # -0.0 == 0.0 but the codes differ
        score = (col * sign) if sign < 0 else col
        codes, xf = score.view(np.uint64), dev.KEY_F64
    else:
        c64 = col.astype(np.int64)
        if sign < 0 and len(c64) and int(c64.min()) == -(1 << 63):
            return None
        score = -c64 if sign < 0 else c64
        codes, xf = score.view(np.uint64), dev.KEY_I64
    if n > k:
        kv = runner.ctx.kv_from_columns(codes, np.arange(n, dtype=np.uint64))
        try:
            kv.sort(xf)
            sk, perm = kv.columns()
        finally:
            kv.free()
        sk = sk.view(score.dtype)
        lo = int(np.searchsorted(sk, sk[n - k], side="left"))   # every row tied with the k-th largest score
        cand = np.sort(perm[lo:].view(np.int64))
    else:
        cand = np.arange(n, dtype=np.int64)
    rows = frame.take(cand).values()
    scored = [(value(x), x) for x in rows]
    if len(scored) > k:
        scored = heapq.nlargest(k, scored)
    runner.stats.add(stage, "device top-k candidates (one sort of the scores; ties cut by the tuple order on the host)",
                     "records=%d k=%d candidates=%d" % (n, k, len(cand)))
    return RecordsDataset([1] * len(scored), scored)


def _lower_frame_map(runner, stage, frame):
    """sort_by(+-x[i]) / sort_by(+-x) over a frame."""
    ks = _opkinds(stage.mapper)
    if ks is None:
        return None
    kinds = [k for k, _ in ks]
    if kinds == ["topk"]:
        return _lower_topk(runner, stage, frame, ks[0][1])
    if kinds == ["keyed"] and stage.combiner is None:
        op = ks[0][1]
        if not lowering.is_identity(op.fn2):
            return None
        kp = lowering.projection(op.fn)
        if kp is None:
            return None
        if kp[0] == "field" and not frame.scalar and kp[1] < len(frame.cols):
            col = frame.cols[kp[1]]
        elif kp[0] == "ident" and frame.scalar:
            col = frame.cols[0]
        else:
            return None
        if not _numeric(col):
            return None
        sign = kp[2]
        if col.dtype.kind == "f":
            fk = _float_keys(-col if sign < 0 else col)
            if fk is None:
                return None
            kcol = _report_zero(*fk)
            codes, xf = fk[0].view(np.uint64), dev.KEY_F64
        else:
            kcol = (-col.astype(np.int64)) if sign < 0 else col.astype(np.int64)
            codes, xf = kcol.view(np.uint64), dev.KEY_I64
        n = frame.n
        ctx = runner.ctx
        kv = ctx.kv_from_columns(codes, np.arange(n, dtype=np.uint64))
        try:
            kv.sort(xf)
            _k, perm = kv.columns()
        finally:
            kv.free()
        perm = perm.view(np.int64)
        out = frame.take(perm)
        out.keys = kcol[perm]
        out.combined = False
        runner.stats.add(stage, "device sort of frame rows", "records=%d" % n)
        return out
    return None


_FOLD_OPS_F64 = {lowering.ADD: dev.OP_SUM_F64, lowering.MIN: dev.OP_MIN_F64, lowering.MAX: dev.OP_MAX_F64,
                 lowering.FIRST: dev.OP_FIRST, lowering.LAST: dev.OP_LAST}


def _fold_single_group(vals, kind):
    """binop-fold of a whole column in record order (a constant key: one group)."""
    if kind == lowering.ADD:
        if vals.dtype == np.int64:
            if _may_overflow(vals):
                raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
            return int(vals.sum())
        return float(np.cumsum(vals)[-1])   # the left fold binop(acc, v) in record order, exactly
    if kind in (lowering.MIN, lowering.MAX):
        if vals.dtype == np.float64 and (np.isnan(vals).any() or (vals == 0).any()):
            raise NotLowerable("NaN or signed zeros under min/max")   # which of -0.0 / 0.0 wins depends on the order
        r = vals.min() if kind == lowering.MIN else vals.max()
        return r.item()
    return (vals[0] if kind == lowering.FIRST else vals[-1]).item()


def _fold_column(runner, kcodes, xf, vals, kind):
    """Group `vals` by the 64-bit key codes on the device; returns (group key codes, folded values)."""
    opmap = _FOLD_OPS if vals.dtype == np.int64 else _FOLD_OPS_F64
    if kind not in opmap:
        raise NotLowerable("fold %s" % kind)
    if kind == lowering.ADD and vals.dtype == np.int64 and len(vals) and _may_overflow(vals):
        raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
    if kind in (lowering.MIN, lowering.MAX) and vals.dtype == np.float64 and \
            (np.isnan(vals).any() or (np.signbit(vals) & (vals == 0)).any()):
        raise NotLowerable("NaN or -0.0 under min/max")   # Python's answer depends on the order of the arguments
    rk, rv, how = _device_group(runner, kcodes, vals.view(np.uint64), opmap[kind], xf)
    return rk, rv.view(vals.dtype), how


def _apply_chain(frame, body):
    """A fused map / filter chain ([(kind, Op)]) over a frame, evaluated column-at-a-time (vexpr: CPython's exact
    results); the resulting Frame, or None when a step is not vectorisable (or a filter leaves nothing: the host
    path then produces the empty result). May raise vexpr.NotVec."""
    keys, cols, scalar, n = frame.keys, list(frame.cols), frame.scalar, frame.n
    for kind, op in body:
        if kind == "identity":
            continue
        e = _inline(op.fn)
        if e is None:
            return None
        v = vexpr.evaluate(e, cols, scalar, n)
        if kind == "map":
            if isinstance(v, vexpr.Tup):
                cols, scalar = [vexpr.broadcast(c, n) for c in v.items], False
            else:
                cols, scalar = [vexpr.broadcast(v, n)], True
        elif kind == "filter":
            if not (isinstance(v, np.ndarray) and v.dtype == np.bool_):
                return None   # truthiness of a non-boolean: host path
            idx = np.flatnonzero(v)
            tmp = Frame(keys, cols, scalar).take(idx)
            keys, cols, n = tmp.keys, tmp.cols, len(idx)
            if n == 0:
                return None
        else:
            return None
    out = Frame(keys, cols, scalar)
    out.n = n
    return out


def _lower_frame_general(runner, stage, frame):
    """map / filter chains and keyed folds over a frame whose lambdas evaluate column-at-a-time
    (vexpr): the stages after an aggregation in examples/word-stats.py:24-37, mean(), map_values() ..."""
    ks = _opkinds(stage.mapper)
    if not ks or frame.n == 0 or dist.active():   # frames are rank-local under torch.distributed
        return None
    body, last, topk_op = ks, None, None
    if ks[-1][0] == "keyed":
        body, last = ks[:-1], ks[-1][1]
    elif ks[-1][0] == "topk":       # map / filter chain fused in front of a topk: evaluate it, then take the candidates
        body, topk_op = ks[:-1], ks[-1][1]
    try:
        chained = _apply_chain(frame, body)
        if chained is None:
            return None
        keys, cols, scalar, n = chained.keys, list(chained.cols), chained.scalar, chained.n
        if topk_op is not None:
            return _lower_topk(runner, stage, Frame(keys, cols, scalar), topk_op)
        if last is None:
            out = Frame(keys, cols, scalar)
            runner.stats.add(stage, "frame map/filter evaluated column-at-a-time", "records=%d" % n)
            return out
        ke, ve = _inline(last.fn), _inline(last.fn2)
        if ke is None or ve is None:
            return None
        kv = vexpr.evaluate(ke, cols, scalar, n)
        vv = vexpr.evaluate(ve, cols, scalar, n)
        binop = stage.options.get("binop")
        if isinstance(stage.combiner, ops.PartialReduceCombiner) and callable(binop):
            comp_kinds = None
            if isinstance(vv, vexpr.Tup):
                comp_kinds = lowering.tuple_binop_kinds(binop)
                if comp_kinds is None or len(comp_kinds) != len(vv.items):
                    return None
                vcols = [vexpr.broadcast(c, n) for c in vv.items]
            else:
                k1 = lowering.binop_kind(binop)
                if k1 is None:
                    return None
                comp_kinds, vcols = [k1], [vexpr.broadcast(vv, n)]
            if not all(isinstance(c, np.ndarray) and c.dtype in (np.int64, np.float64) for c in vcols):
                return None
            if isinstance(kv, vexpr.Const):
                res = [_fold_single_group(c, k) for c, k in zip(vcols, comp_kinds)]
                rcols = [np.array([r]) for r in res]
                okeys, how = np.array([kv.v]), " [one group, folded on the host]"
            else:
                if not (isinstance(kv, np.ndarray) and kv.dtype in (np.int64, np.uint64)):
                    return None   # float / string keys: equality is not bit equality
                rk = None
                rcols = []
                for c, k in zip(vcols, comp_kinds):
                    rk2, rv, how = _fold_column(runner, kv.view(np.uint64), dev.KEY_MIX, c, k)
                    if len(vcols) > 1:
                        # the group order of a hash-aggregated fold is not defined: bring every
                        # component into key order (a device sort of the few group records)
                        g = runner.ctx.kv_from_columns(rk2, rv.view(np.uint64))
                        try:
                            g.sort(dev.KEY_RAW)
                            rk2, rv2 = g.columns()
                        finally:
                            g.free()
                        rv = rv2.view(rv.dtype)
                    if rk is not None and not np.array_equal(rk, rk2):
                        raise NotLowerable("component folds disagree on the groups")
                    rk = rk2
                    rcols.append(rv)
                okeys = rk.view(kv.dtype)
            val = vexpr.Tup(rcols) if isinstance(vv, vexpr.Tup) else rcols[0]
            out = Frame(okeys, [val], scalar=True, combined=True)
            runner.stats.add(stage, "frame keyed fold: columns evaluated on the host, groups folded on the device" + how,
                             "records=%d groups=%d" % (n, len(okeys)))
            return out
        if stage.combiner is None and lowering.is_identity(last.fn2):
            # sort_by(expr): device sort of (key code, row index)
            kc = vexpr.broadcast(kv, n)
            if not (isinstance(kc, np.ndarray) and kc.dtype in (np.int64, np.float64)):
                return None
            if kc.dtype == np.float64 and np.isnan(kc).any():
                return None
            if kc.dtype == np.float64:
                kc = kc + 0.0   # -0.0 and 0.0 are one key for Python's sort
            xf = dev.KEY_I64 if kc.dtype == np.int64 else dev.KEY_F64
            kvh = runner.ctx.kv_from_columns(kc.view(np.uint64), np.arange(n, dtype=np.uint64))
            try:
                kvh.sort(xf)
                _k, perm = kvh.columns()
            finally:
                kvh.free()
            perm = perm.view(np.int64)
            out = Frame(keys, cols, scalar).take(perm)
            out.keys = kc[perm]
            runner.stats.add(stage, "device sort of frame rows", "records=%d" % n)
            return out
    except vexpr.NotVec as why:
        log.debug("stage %s not vectorised: %s", stage.output, why)
    return None


def _lower_cross(runner, stage, inputs):
    """MapCrossJoin(outer=frame, inner=one row), cross analysable: evaluate the user's function once
    per distinct value of the outer fields each output component reads."""
    mapper = stage.mapper
    cross = getattr(mapper, "user_cross", None)
    if cross is None:
        return None
    outer = inputs[0]
    inner_rows = [v for _k, v in ops.as_one_dataset(inputs[1]).read()]
    if len(inner_rows) != 1 or outer.n == 0:
        return None
    inner = inner_rows[0]
    e = _inline(cross)
    if e is None:
        return None
    # cross(v_inner, v_outer): arg0 = inner value, arg1 = outer value
    comps = e.a if e.op == "tuple" else (e,)
    out_cols = []
    dict_cache = {}
    for ci, comp in enumerate(comps):
        f = lowering._field(_swap_to_arg0(comp, 1))
        if f is not None and not outer.scalar and f < len(outer.cols):
            src = outer.cols[f]
            if _numeric(src) and src.dtype.kind in "iu":
                # share the dictionary with the components computed from this field (and with the sink)
                uq = dict_cache.get(f) or unique_inverse_rows(src)
                dict_cache[f] = uq
                src = DictCol(uq[1], uq[0])
            out_cols.append(src)
            continue
        deps = lowering.depends_on(comp, 1)
        if deps is None or outer.scalar or not deps or any(d >= len(outer.cols) for d in deps):
            return None
        dep = sorted(deps)
        if len(dep) != 1 or not (isinstance(outer.cols[dep[0]], DictCol) or _numeric(outer.cols[dep[0]])):
            return None
        col = outer.cols[dep[0]]
        # one representative row per distinct value (any row holding it)
        if isinstance(col, DictCol):
            uniq, inv = col.uniq, col.inv
            rep = np.empty(len(uniq), dtype=np.int64)
            rep[inv] = np.arange(outer.n, dtype=np.int64)
        else:
            uniq, inv, rep = dict_cache.get(dep[0]) or unique_inverse_rows(col)
            dict_cache[dep[0]] = (uniq, inv, rep)
        direct = getattr(cross, "swapped_of", None)
        pick = ci if e.op == "tuple" else None

        def evaluate(rep_cols):
            out = []
            if direct is not None:   # cross_right's argument swap, without the extra call per value
                for row in zip(*rep_cols):
                    r = direct(row, inner)
                    out.append(r if pick is None else r[pick])
            else:
                for row in zip(*rep_cols):
                    r = cross(inner, row)
                    out.append(r if pick is None else r[pick])
            return out
        # representative rows, gathered column-wise (no per-cell Python dispatch). This component reads only the
        # fields in `dep`: the other fields of the representative rows are placeholders (no gather, no string
        # decoding of thousands of keys nobody looks at). The user's function still evaluates its other
        # components on them; if one of those chokes on a placeholder the full rows are used instead.
        m = len(rep)
        res = _native_eval(comp, dep[0], inner, uniq)
        if res is None and pick is not None and len(outer.cols) > len(dep):
            try:
                res = evaluate([_gather(c, rep) if j in dep else [None] * m for j, c in enumerate(outer.cols)])
            except Exception:
                res = None
        if res is None:
            res = evaluate([_gather(c, rep) for c in outer.cols])
        kinds = set(type(x) for x in res) if isinstance(res, list) else None
        if kinds == {float}:
            res = np.array(res, dtype=np.float64)
        elif kinds == {int}:
            res = np.array(res, dtype=np.int64)
        out_cols.append(DictCol(inv, res))
    f = Frame(outer.keys, out_cols, scalar=(e.op != "tuple"))
    runner.stats.add(stage, "frame cross with a 1-row broadcast (memoised per distinct field value)",
                     "records=%d" % outer.n)
    return f


def _native_eval(comp, field, inner, uniq):
    """float64 values of one cross component at the distinct values `uniq` of the int field it reads, computed by
    the library (dampr_host_eval_f64, CPython's results to the bit), or None: the component is outside the lowered
    numeric set (lowering.numeric_program), or CPython would raise or leave the IEEE path for some value."""
    if not (isinstance(uniq, np.ndarray) and uniq.dtype == np.int64):
        return None
    prog = lowering.numeric_program(comp, field, inner)
    if prog is None:
        return None
    return dev.host_eval_f64(uniq, *prog)


def _gather(col, idx):
    """Python values of rows idx (numpy int array) of a frame column, as a list."""
    if isinstance(col, DictCol):
        sub = col.inv[idx]
        if isinstance(col.uniq, np.ndarray):
            return _gather(col.uniq, sub)
        return [col.uniq[j] for j in sub.tolist()]
    if isinstance(col, np.ndarray):
        v = col[idx]
        if v.dtype.kind == "S":
            return [b.decode("ascii") for b in v.tolist()]
        return v.tolist()
    return [col[i] for i in idx.tolist()]


def _lower_probe(runner, stage, inputs):
    """small.cross_set(big, lambda b, table: (..., b[i] in table, ...), agg=set): the broadcast join of
    MapAllJoin.map (base.py:165-178) as a device hash build + probe (dampr_kv_hash_probe). Streams the
    kv records of `big`; the table is the set of (integer) values of `small`."""
    mapper = stage.mapper
    cross, agg = getattr(mapper, "user_cross", None), getattr(mapper, "user_agg", None)
    if cross is None or agg not in (set, frozenset):
        return None
    cols = _kv_columns(inputs[0])
    if cols is None:
        return None
    e = lowering.analyze(cross)
    if e is None or cross.__code__.co_argcount != 2:
        return None
    comps = e.a if e.op == "tuple" else (e,)
    plan_ = []
    for comp in comps:
        f = lowering._field(comp)
        if f is not None and f in (0, 1):
            plan_.append(("col", f))
            continue
        if comp.op == "cmp" and comp.a in ("in", "not in") and lowering._is_arg(comp.c, 1):
            f = lowering._field(comp.b)
            if f in (0, 1):
                plan_.append(("probe", f, comp.a == "not in"))
                continue
        return None
    small_vals = [v for _k, v in ops.as_one_dataset(inputs[1]).read()]
    if not all(type(v) is int and -(1 << 63) <= v < (1 << 64) for v in small_vals):
        return None
    ctx = runner.ctx
    build_keys = np.unique(np.array([v & 0xFFFFFFFFFFFFFFFF for v in small_vals], dtype=np.uint64))
    build = ctx.kv_from_columns(build_keys, np.ones(len(build_keys), dtype=np.uint64))
    hits = {}
    try:
        for item in plan_:
            if item[0] == "probe" and item[1] not in hits:
                probe = ctx.kv_from_columns(cols[item[1]].view(np.uint64), np.zeros(len(cols[item[1]]), dtype=np.uint64))
                try:
                    vals, hit = build.hash_probe(probe)
                    vals.free()
                finally:
                    probe.free()
                hits[item[1]] = hit.astype(bool)
    finally:
        build.free()
    out_cols = []
    for item in plan_:
        if item[0] == "col":
            out_cols.append(cols[item[1]])
        else:
            h = hits[item[1]]
            out_cols.append(~h if item[2] else h)
    n = len(cols[0])
    f = Frame(np.arange(n, dtype=np.int64), out_cols, scalar=(e.op != "tuple"))
    runner.stats.add(stage, "device broadcast hash build+probe", "build=%d probe=%d" % (len(build_keys), n))
    return f


def _swap_to_arg0(e, argi):
    """Rewrite arg(argi) as arg(0) so that lowering._field can test `x[i]` patterns."""
    E = lowering.E
    if not isinstance(e, E):
        return e
    if e.op == "arg":
        return E("arg", 0) if e.a == argi else E("arg", 99)
    if e.op in ("const", "obj"):
        return e

    def sw(x):
        if isinstance(x, tuple):
            return tuple(sw(y) for y in x)
        return _swap_to_arg0(x, argi) if isinstance(x, E) else x
    return E(e.op, sw(e.a), sw(e.b), sw(e.c))


def _inline(fn, depth=0):
    """analyze(fn) with calls to analysable Python functions substituted (DSL wrappers such as
    cross_right's `lambda xi, yi: cross(yi, xi)`)."""
    E = lowering.E
    e = lowering.analyze(fn)
    if e is None or depth > 3:
        return e

    def subst(x, args):
        if isinstance(x, tuple):
            return tuple(subst(y, args) for y in x)
        if not isinstance(x, E):
            return x
        if x.op == "arg":
            return args[x.a]
        if x.op in ("const", "obj"):
            return x
        return E(x.op, subst(x.a, args), subst(x.b, args), subst(x.c, args))

    def walk(x):
        if isinstance(x, tuple):
            return tuple(walk(y) for y in x)
        if not isinstance(x, E):
            return x
        if x.op in ("const", "obj", "arg"):
            return x
        y = E(x.op, walk(x.a), walk(x.b), walk(x.c))
        if y.op == "call" and isinstance(y.a, E) and y.a.op == "obj":
            import types
            target = y.a.a
            if isinstance(target, types.FunctionType) and target.__code__.co_argcount == len(y.b):
                inner = _inline(target, depth + 1)
                if inner is not None:
                    return subst(inner, list(y.b))
        return y

    return walk(e)


# ---- reduce stages ----------------------------------------------------------------------------------------
def _device_perm(runner, codes, xf, payload=None):
    """Stable device sort of 64-bit codes under `xf`; returns the payload (default: the positions) in sorted order."""
    n = len(codes)
    kv = runner.ctx.kv_from_columns(codes, np.arange(n, dtype=np.uint64) if payload is None else payload)
    try:
        kv.sort(xf)
        _k, perm = kv.columns()
    finally:
        kv.free()
    return perm.view(np.int64)


def _lower_unique(runner, stage, fr, key_fn=None):
    """group_by(k, v).unique() over binary kv records (dampr.py:727-746): per key, the distinct values in the
    order of their first appearance. Three stable device sorts and linear host passes over the columns:
      by key                      -> the records of every key, in input order;
      by value, then by key       -> equal (key, value) pairs adjacent, earliest first => the first occurrence of
                                     every distinct pair is the head of its run;
    the by-key order filtered to first occurrences is the answer. The value lists are Python lists (the
    reducer's return type), built per group at the end."""
    from . import spill
    keys, vals = fr.raw()
    n = len(keys)
    if dist.active() or n == 0 or spill.needs_spill(runner.ctx, 2 * n):
        return None
    if vals.dtype.itemsize != 8 or vals.dtype.kind not in "iuf":
        return None
    # what makes two values "the same": key(v) — the identity, or a straight-line numeric expression evaluated
    # column-at-a-time with CPython's results (vexpr)
    fv = vals
    if key_fn is not None and not lowering.is_identity(key_fn):
        ke = _inline(key_fn)
        if ke is None:
            return None
        try:
            fv = vexpr.evaluate(ke, [vals], True, n)
        except vexpr.NotVec:
            return None
        if isinstance(fv, vexpr.Const):
            fv = vexpr.broadcast(fv, n)
        if not isinstance(fv, np.ndarray) or fv.dtype.kind not in "iufb" or len(fv) != n:
            return None
        if fv.dtype.kind == "b":
            fv = fv.astype(np.int64)     # True == 1, False == 0 (and hash alike)
        elif fv.dtype.itemsize != 8:
            return None
    if fv.dtype.kind == "f":
        if np.isnan(fv).any() or (np.signbit(fv) & (fv == 0)).any():
            return None   # NaN != NaN keeps every NaN; -0.0 == 0.0 are one value: leave those to the set()
        vxf = dev.KEY_F64
    else:
        vxf = _key_xform_for(fv)
    kxf = _key_xform_for(keys)
    ku, vu = keys.view(np.uint64), np.ascontiguousarray(fv).view(np.uint64)
    by_key = _device_perm(runner, ku, kxf)
    p1 = _device_perm(runner, vu, vxf)
    p2 = _device_perm(runner, ku[p1], kxf, p1.view(np.uint64))
    k2, v2 = ku[p2], vu[p2]
    head = np.empty(n, dtype=np.bool_)
    head[0] = True
    np.logical_or(k2[1:] != k2[:-1], v2[1:] != v2[:-1], out=head[1:])
    first = np.zeros(n, dtype=np.bool_)
    first[p2[head]] = True
    sel = by_key[first[by_key]]
    ks, vs = keys[sel], vals[sel]
    cut = np.flatnonzero(ks[1:] != ks[:-1]) + 1
    starts = np.concatenate(([0], cut))
    ends = np.concatenate((cut, [len(ks)]))
    vl = vs.tolist()
    lists = [vl[a:b] for a, b in zip(starts.tolist(), ends.tolist())]
    gk = ks[starts]
    out = Frame(gk, [gk, lists], scalar=False, combined=True)
    runner.stats.add(stage, "device unique: three stable sorts (by key; by value then key), first occurrences kept in input order",
                     "records=%d groups=%d distinct pairs=%d" % (n, len(gk), len(ks)))
    return out


def _lower_reduce(runner, stage, inputs):
    red = stage.reducer
    if len(inputs) == 1 and isinstance(inputs[0], Frame):
        fr = inputs[0]
        binop = getattr(red, "binop", None)
        uop = getattr(red, "op", None)
        if isinstance(red, ops.KeyedReduce) and uop is not None and uop.kind == "unique" \
                and isinstance(fr, LazyKVFrame) and not fr._done:
            out = _lower_unique(runner, stage, fr, uop.fn)
            if out is not None:
                return out
        if isinstance(red, ops.KeyedReduce) and binop is not None and fr.combined and fr.scalar:
            # fully combined on the map side: the fold of a one-element group is the element
            out = Frame(fr.keys, [fr.keys, fr.cols[0]], scalar=False, combined=True)
            runner.stats.add(stage, "keyed fold over a fully combined frame (relabel)", "records=%d" % fr.n)
            return out
        if isinstance(red, ops.KeyedReduce) and isinstance(fr, LazyKVFrame) and not fr._done:
            kind = lowering.group_reducer_kind(red.reducer)
            opmap = {lowering.SUM: dev.OP_SUM_I64, lowering.COUNT: dev.OP_COUNT, lowering.MIN: dev.OP_MIN_I64,
                     lowering.MAX: dev.OP_MAX_I64}
            keys, vals = fr.raw()
            from . import spill as _spill
            # the overflow bound (SURVEY B12) scans every value: on an input large enough to spill (tens of GB) it runs
            # on a host thread NEXT TO the device pipeline and vetoes the result afterwards, instead of in front of it
            late = kind == lowering.SUM and vals.dtype.kind in "iu" and len(vals) and _spill.needs_spill(runner.ctx, len(vals)) \
                and not dist.active()
            if kind in opmap and vals.dtype.kind in "iu" and not (kind == lowering.SUM and len(vals) and not late and _may_overflow(vals)) \
                    and not (vals.dtype == np.uint64 and len(vals) and int(vals.max()) >= (1 << 63)):
                chk = _Background(_may_overflow, vals) if late else None
                try:
                    rk, rv, how = _device_group(runner, keys, vals, opmap[kind], dev.KEY_MIX)
                finally:
                    overflow = chk.result() if chk is not None else False
                if overflow:
                    raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
                rk = rk.view(keys.dtype)
                out = Frame(rk, [rk, rv.view(np.int64)], scalar=False, combined=True)
                runner.stats.add(stage, "device kv partition+sort+segmented-reduce (fused group_by + reduce)" + how,
                                 "records=%d groups=%d" % (len(keys), len(rk)))
                return out
        if isinstance(red, ops.KeyedReduce) and fr.meta.get("sorted_kv") and fr.scalar and _numeric(fr.cols[0]):
            kind = lowering.group_reducer_kind(red.reducer)
            opmap = {lowering.SUM: dev.OP_SUM_I64, lowering.COUNT: dev.OP_COUNT, lowering.MIN: dev.OP_MIN_I64,
                     lowering.MAX: dev.OP_MAX_I64}
            if kind in opmap and fr.cols[0].dtype.kind in "iu" and isinstance(fr.keys, np.ndarray):
                vals = fr.cols[0]
                if kind == lowering.SUM and fr.n and _may_overflow(vals):
                    return None
                rk, rv, how = _device_group(runner, fr.keys, vals, opmap[kind], _key_xform_for(fr.keys))
                rk = rk.view(fr.keys.dtype)
                out = Frame(rk, [rk, rv.view(np.int64)], scalar=False, combined=True)
                runner.stats.add(stage, "device segmented reduce of sorted kv" + how, "records=%d groups=%d" % (fr.n, len(rk)))
                return out
    return None


# ---- reduce-side joins -----------------------------------------------------------------------------------------
def _exchange_raw(runner, keys, vals):
    """world > 1: this rank's record range of a global kv input, every record moved to the owner of its key
    (the same owner function on both join sides = the reference's requirement that both sides use one Splitter
    and partition count, base.py:264-283). Returns host columns of the records this rank owns."""
    ctx = runner.ctx
    r, w = dist.world()
    n = len(keys)
    lo, hi = n * r // w, n * (r + 1) // w
    kv = ctx.kv_from_columns(keys[lo:hi], np.asarray(vals[lo:hi]).view(np.uint64))
    try:
        recv, _offs, _h = dist.shuffle_kv(ctx, kv)
    finally:
        kv.free()
    try:
        k, v = recv.columns()
    finally:
        recv.free()
    return k.view(keys.dtype), v.view(vals.dtype)


def _lower_join(runner, stage, inputs):
    """Columnar reduce-side join (InnerJoin / LeftJoin, base.py:264-315; PJoin.reduce dampr.py:780-820) of two
    grouped binary-kv inputs when the aggregate is one of the idioms of lowering.join_aggregate_kind:
      folds    lambda l, r: (sum(l), len(list(r)))...  both sides are folded per key on the device
               (partition + sort + segmented reduce; across ranks: local fold, all-to-all, owner fold) and the two
               sets of unique keys are matched by the hash build + probe kernels;
      product  lambda l, r: itertools.product(l, r) with many=True and unique right keys (a dimension table): every
               left record looks its partner up in the hash table built from the right side — no sort at all.
    Records never become Python objects; the result is a frame (K, (fl, fr)) / (K, (lv, rv))."""
    red = stage.reducer
    if not isinstance(red, (ops.InnerJoin, ops.LeftJoin)) or not getattr(red, "keyed", False):
        return None
    agg = getattr(red, "user_aggregate", None)
    L, R = inputs
    if agg is None or not (isinstance(L, LazyKVFrame) and isinstance(R, LazyKVFrame)) or L._done or R._done:
        return None
    kind = lowering.join_aggregate_kind(agg)
    if kind is None:
        return None
    lk, lv = L.raw()
    rk, rv = R.raw()
    if lk.dtype != rk.dtype or lv.dtype.kind not in "iu" or rv.dtype.kind not in "iu":
        return None
    left_outer = isinstance(red, ops.LeftJoin)
    ctx = runner.ctx
    opmap = {lowering.SUM: dev.OP_SUM_I64, lowering.COUNT: dev.OP_COUNT, lowering.MIN: dev.OP_MIN_I64,
             lowering.MAX: dev.OP_MAX_I64}
    if kind[0] == "folds":
        if bool(getattr(red, "many", False)):
            return None
        _k, kl, kr = kind
        if left_outer and kr not in (lowering.SUM, lowering.COUNT):
            return None   # min / max of an empty right group raise in Python
        for col, kk in ((lv, kl), (rv, kr)):
            if kk == lowering.SUM and len(col) and _may_overflow(col):
                raise NotLowerable("64-bit sum could overflow (SURVEY B12)")
        gk_l, gv_l, how = _device_group(runner, lk, lv, opmap[kl], dev.KEY_MIX)
        gk_r, gv_r, _h = _device_group(runner, rk, rv, opmap[kr], dev.KEY_MIX)
        build = ctx.kv_from_columns(gk_r, gv_r)
        probe = ctx.kv_from_columns(gk_l, gv_l)
        try:
            if left_outer:
                vals, hit = build.hash_probe(probe)
                try:
                    _pk, fr = vals.columns()
                finally:
                    vals.free()
                keys = gk_l.view(lk.dtype)
                fl = gv_l.view(np.int64)
                fr = np.where(hit.astype(bool), fr.view(np.int64), 0)   # sum / len of an empty right group
            else:
                # matched groups are compacted on the device: only the joined rows come back
                ml, mr = build.hash_join(probe)
                try:
                    keys, fl = ml.columns()
                    _k2, fr = mr.columns()
                finally:
                    ml.free()
                    mr.free()
                keys, fl, fr = keys.view(lk.dtype), fl.view(np.int64), fr.view(np.int64)
        finally:
            build.free()
            probe.free()
        out = Frame(keys, [keys, vexpr.Tup([fl, fr])], scalar=False, combined=True)
        runner.stats.add(stage, "device join: per-side partition+sort+fold, hash build+probe of the group keys" + how,
                         "left=%d right=%d left groups=%d right groups=%d rows=%d" % (len(lk), len(rk), len(gk_l), len(gk_r), len(keys)))
        return out
    # ---- product with a unique right side --------------------------------------------------------------------
    if left_outer or not bool(getattr(red, "many", False)):
        return None
    how = ""
    if dist.active():
        lk, lv = _exchange_raw(runner, lk, lv)
        rk, rv = _exchange_raw(runner, rk, rv)
        how = " [rank %d/%d: both sides exchanged by key owner]" % dist.world()
    build = ctx.kv_from_columns(rk, np.asarray(rv).view(np.uint64))
    try:
        cnt = ctx.kv_from_columns(rk, np.ones(len(rk), dtype=np.int64)).sort_reduce(dev.OP_COUNT, dev.KEY_MIX)
        unique = len(cnt) == len(rk)
        cnt.free()
        if dist.active():
            unique = dist.all_reduce_sum_int([0 if unique else 1])[0] == 0
        if not unique:
            raise NotLowerable("product join: the right side has duplicate keys")
        probe = ctx.kv_from_columns(lk, np.asarray(lv).view(np.uint64))
        try:
            ml, mr = build.hash_join(probe)   # matched rows compacted on the device, probe order kept
            try:
                keys, plv = ml.columns()
                _k2, prv = mr.columns()
            finally:
                ml.free()
                mr.free()
        finally:
            probe.free()
    finally:
        build.free()
    keys = keys.view(lk.dtype)
    out = Frame(keys, [keys, vexpr.Tup([plv.view(lv.dtype), prv.view(rv.dtype)])], scalar=False, combined=False)
    runner.stats.add(stage, "device join: broadcast hash build + probe (unique right keys)" + how,
                     "left=%d right=%d rows=%d" % (len(lk), len(rk), len(keys)))
    return out


# ---- sinks ---------------------------------------------------------------------------------------------------
def _sink_column(col):
    """A frame column in the form dampr_host_join_tsv takes: an 'S' array, or (inv, [bytes per distinct
    value]) with Python's own str() of every distinct value (exact float repr); None if unsupported."""
    if isinstance(col, DictCol):
        if isinstance(col.uniq, np.ndarray) and col.uniq.dtype in (np.int64, np.float64):
            # decimal text of the distinct ints / Python's repr of the distinct floats is produced natively
            # (dampr_host_format_f64: bit-for-bit repr(float), tests/test_host_logic.py)
            return (col.inv, col.uniq)
        u = col.uniq.tolist() if isinstance(col.uniq, np.ndarray) else col.uniq
        return (col.inv, [str(x).encode("utf-8") for x in u])
    if isinstance(col, np.ndarray):
        if col.dtype.kind == "S":
            return col
        if col.dtype.kind in "iuf":
            uniq, inv = unique_inverse(col)
            if uniq.dtype in (np.int64, np.float64):
                return (inv, uniq)
            return (inv, [str(x).encode("utf-8") for x in uniq.tolist()])
        return None
    if isinstance(col, list) and all(type(x) is str for x in col):
        uniq = sorted(set(col))
        idx = {w: i for i, w in enumerate(uniq)}
        inv = np.fromiter((idx[w] for w in col), dtype=np.uint32, count=len(col))
        return (inv, [w.encode("utf-8") for w in uniq])
    return None


def _tuple_repr_columns(fr):
    """sink(path) over tuple rows: print(value) writes str(tuple) = "('w', 3, 1.5)" — the repr of every element.
    'S' strings go out between single quotes when they are printable ASCII without quotes and backslashes (what
    repr(str) writes for them), ints in decimal, floats by repr (any float: repr is what print uses). Other cells
    -> None: the host sink."""
    cols, kinds = [], []
    for c in fr.cols:
        if isinstance(c, DictCol) and isinstance(c.uniq, np.ndarray) and c.uniq.dtype in (np.int64, np.float64):
            cols.append((c.inv, c.uniq)); kinds.append("n")
        elif isinstance(c, np.ndarray) and c.dtype.kind == "S":
            b = np.ascontiguousarray(c).view(np.uint8)
            if ((b != 0) & ((b < 0x20) | (b > 0x7e) | (b == 0x22) | (b == 0x27) | (b == 0x5c))).any():
                return None
            cols.append(c); kinds.append("s")
        elif isinstance(c, np.ndarray) and c.dtype in (np.int64, np.float64):
            sc = _sink_column(c)
            if sc is None:
                return None
            cols.append(sc); kinds.append("n")
        else:
            return None
    pre = []
    for i, k in enumerate(kinds):
        p = b"(" if i == 0 else (b"'" if kinds[i - 1] == "s" else b"") + b", "
        if k == "s":
            p += b"'"
        pre.append(p)
    end = (b"'" if kinds[-1] == "s" else b"") + (b",)" if len(kinds) == 1 else b")") + b"\n"
    return cols, pre, end


def _json_columns(fr):
    """sink_json over a frame (json.dumps(value) per record, dampr.py:531-539): the columns in the form the native
    row writer takes plus the byte strings it puts in front of every column and at the end of a row — `["w", 3, 1.5]`
    for tuple rows, the bare value for scalar rows. Strings of an 'S' column go out as they are between quotes when
    they are printable ASCII without '"' and '\\' (what json.dumps would write); dictionary strings are escaped
    per distinct value by json.dumps itself; ints in decimal; floats by repr() — json.dumps does the same for
    finite floats. Anything else (non-finite floats, bools, None, nested tuples) -> None: the host sink."""
    cols, kinds = [], []
    for c in fr.cols:
        if isinstance(c, DictCol):
            u = c.uniq
            if isinstance(u, np.ndarray) and u.dtype == np.int64:
                cols.append((c.inv, u)); kinds.append("n")
            elif isinstance(u, np.ndarray) and u.dtype == np.float64:
                if not np.isfinite(u).all():
                    return None
                cols.append((c.inv, u)); kinds.append("n")
            elif isinstance(u, list) and all(type(x) is str for x in u):
                cols.append((c.inv, [json.dumps(x).encode("ascii") for x in u])); kinds.append("n")
            else:
                return None
        elif isinstance(c, np.ndarray) and c.dtype.kind == "S":
            b = np.ascontiguousarray(c).view(np.uint8)
            if ((b != 0) & ((b < 0x20) | (b > 0x7e) | (b == 0x22) | (b == 0x5c))).any():
                return None
            cols.append(c); kinds.append("s")
        elif isinstance(c, np.ndarray) and c.dtype in (np.int64, np.float64):
            if c.dtype == np.float64 and not np.isfinite(c).all():
                return None
            sc = _sink_column(c)
            if sc is None:
                return None
            cols.append(sc); kinds.append("n")
        elif isinstance(c, list) and all(type(x) is str for x in c):
            uniq = sorted(set(c))
            idx = {w: i for i, w in enumerate(uniq)}
            inv = np.fromiter((idx[w] for w in c), dtype=np.uint32, count=len(c))
            cols.append((inv, [json.dumps(w).encode("ascii") for w in uniq])); kinds.append("n")
        else:
            return None
    pre = []
    for i, k in enumerate(kinds):
        p = b""
        if i == 0:
            p += b"" if fr.scalar else b"["
        else:
            p += (b'"' if kinds[i - 1] == "s" else b"") + b", "
        if k == "s":
            p += b'"'
        pre.append(p)
    end = (b'"' if kinds[-1] == "s" else b"") + (b"" if fr.scalar else b"]") + b"\n"
    return cols, pre, end


def _lower_sink(runner, stage, inputs):
    if len(inputs) != 1 or not isinstance(inputs[0], Frame):
        return None
    fr = inputs[0]
    parts = _parts(stage.mapper)
    from .dsl import _tsv_line
    cols = None
    col_pre = row_end = None
    ks = _opkinds(stage.mapper)
    if not ks:
        return None
    # the last step formats (sink_tsv's / sink_json's map, or nothing: print(value)); whatever is fused in front of
    # it (x.map(f).sink(...)) is a map / filter chain, evaluated column-at-a-time first
    last_kind, last_op = ks[-1]
    if last_kind == "identity" or (last_kind == "map" and (last_op.fn is _tsv_line or last_op.fn is json.dumps)):
        chain, fmt = ks[:-1], last_op
    else:
        chain, fmt = ks, None
    if any(k != "identity" for k, _o in chain):
        if not fr.n or dist.active():
            return None
        try:
            fr = _apply_chain(fr, chain)
        except vexpr.NotVec:
            fr = None
        if fr is None:
            return None
    if fmt is not None and fmt.kind == "map" and fmt.fn is _tsv_line:
        if not fr.scalar:
            cols = [_sink_column(c) for c in fr.cols]
    elif fmt is not None and fmt.kind == "map" and fmt.fn is json.dumps:
        js = _json_columns(fr)    # sink_json: one JSON value (an array for tuple rows) per line
        if js is not None:
            cols, col_pre, row_end = js
    elif fr.scalar:
        cols = [_sink_column(fr.cols[0])]
    else:
        tp = _tuple_repr_columns(fr)   # sink(path) of tuple rows: print(value) writes repr(tuple)
        if tp is not None:
            cols, col_pre, row_end = tp
    if cols is None or any(c is None for c in cols):
        return None
    os.makedirs(stage.path, exist_ok=True)
    # part files: up to 16 per process (row ranges written in parallel), numbered after the rank
    first = 16 * dist.world()[0] if dist.active() else 0
    prefix = os.path.join(stage.path, "part-")
    if fr.n:
        # formatted and written by native threads
        names = dev.host_join_tsv(cols, prefix=prefix, first=first, col_pre=col_pre, row_end=row_end)
    else:
        names = ["%s%d" % (prefix, first)]
        open(names[0], "wb").close()
    lines = range(fr.n)
    runner.stats.add(stage, "native frame sink (per-distinct-value formatting)", "records=%d" % len(lines))
    return CatDataset([TextLineDataset(fn) for fn in names])

"""ctypes binding of libdampr_b200.so (the C-ABI declared in include/dampr_b200.h).

This is the only door between the Python host side and the device: every shuffle / sort /
combine / reduce of the engine goes through these calls.  There is no CPU fallback — if the
library or a CUDA device is missing the calls raise.

Reference interfaces replaced (see the header for per-function citations): the process pool of
``StageRunner.run`` (stagerunner.py:15-43), the writers/datasets of dataset.py and the combiner of
``ReducedWriter`` (dataset.py:84-117).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdampr_b200.so")

# tokeniser modes
TOK_WS = 0
TOK_NONWORD_LOWER_SET = 1
TOK_NONWORD_LOWER = 2
# key transforms
KEY_RAW, KEY_MIX, KEY_I64, KEY_F64 = 0, 1, 2, 3
# reduce ops
OP_SUM_I64, OP_SUM_F64, OP_COUNT, OP_MIN_I64, OP_MAX_I64, OP_MIN_F64, OP_MAX_F64, OP_FIRST, OP_LAST = range(9)
# table flags
TF_NONASCII, TF_CR, TF_LONGLINE, TF_TABLEFULL, TF_LONGTOKEN, TF_COLLISION = 1, 2, 4, 8, 16, 32
TOK_FLAG_CR_DATA = 0x100

KERNEL_NAMES = {
    1: "text_count", 2: "table_extract", 3: "text_verify", 4: "part_hist", 5: "part_scatter",
    6: "leaf_sort", 7: "seg_reduce", 8: "merge", 9: "join", 10: "probe", 11: "synth", 12: "misc",
}


class DeviceError(RuntimeError):
    pass


_lib = None


def _sig(lib, name, *argtypes, restype=C.c_int32):
    fn = getattr(lib, name)
    fn.argtypes = list(argtypes)
    fn.restype = restype
    return fn


def load_library():
    """Load the shared library (raises if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DeviceError(
            "libdampr_b200.so is not built: run `python -m dampr_b200.build` (needs nvcc); "
            "the engine has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int32, C.c_uint32
    pvp, pu64 = C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)
    _sig(lib, "dampr_abi_version")
    _sig(lib, "dampr_device_count", C.POINTER(i32))
    _sig(lib, "dampr_set_option", C.c_char_p, C.c_int64)
    _sig(lib, "dampr_ctx_create", i32, pvp)
    _sig(lib, "dampr_ctx_destroy", vp)
    _sig(lib, "dampr_ctx_sync", vp)
    _sig(lib, "dampr_ctx_sync_copy", vp)
    _sig(lib, "dampr_last_error", vp, restype=C.c_char_p)
    _sig(lib, "dampr_ctx_timings", vp, C.POINTER(C.c_double), C.POINTER(i32), i32, C.POINTER(i32))
    _sig(lib, "dampr_ctx_timings_reset", vp)
    _sig(lib, "dampr_ctx_timing_enable", vp, i32)
    _sig(lib, "dampr_ctx_launches", vp, pu64)
    _sig(lib, "dampr_ctx_mem_info", vp, pu64, pu64)
    _sig(lib, "dampr_ctx_num_sms", vp, C.POINTER(i32))
    _sig(lib, "dampr_ctx_stream", vp, pu64)
    _sig(lib, "dampr_host_alloc", u64, pvp)
    _sig(lib, "dampr_host_free", vp)
    _sig(lib, "dampr_host_format_f64", vp, u64, vp, vp)
    _sig(lib, "dampr_host_register", vp, u64)
    _sig(lib, "dampr_host_unregister", vp)
    _sig(lib, "dampr_textbuf_create", vp, u64, pvp)
    _sig(lib, "dampr_textbuf_destroy", vp, vp)
    _sig(lib, "dampr_textbuf_set_length", vp, vp, u64)
    _sig(lib, "dampr_textbuf_upload_file", vp, vp, u64, C.c_char_p, u64, u64)
    _sig(lib, "dampr_textbuf_upload", vp, vp, u64, vp, u64)
    _sig(lib, "dampr_textbuf_download", vp, vp, u64, vp, u64)
    _sig(lib, "dampr_textbuf_devptr", vp, vp, pu64)
    _sig(lib, "dampr_table_create", vp, u32, pvp)
    _sig(lib, "dampr_table_destroy", vp, vp)
    _sig(lib, "dampr_table_clear", vp, vp)
    _sig(lib, "dampr_text_count", vp, vp, vp, u64, u64, i32)
    _sig(lib, "dampr_text_verify", vp, vp, vp, u64, u64, i32)
    _sig(lib, "dampr_table_stats", vp, vp, pu64)
    _sig(lib, "dampr_table_fallback_lines", vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_table_fetch", vp, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_table_to_kv", vp, vp, pvp)
    _sig(lib, "dampr_table_fetch_words", vp, vp, vp, i32, u32, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_kv_decode_words", vp, vp, i32, u32, vp)
    _sig(lib, "dampr_host_join_tsv", u64, i32, vp, vp, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_host_sink_tsv", C.c_char_p, C.c_uint32, C.c_uint32, u64, i32, vp, vp, vp, vp, vp, pu64,
         C.POINTER(C.c_uint32))
    _sig(lib, "dampr_host_sink_fmt", C.c_char_p, C.c_uint32, C.c_uint32, u64, i32, vp, vp, vp, vp, vp, vp, C.c_char_p, pu64,
         C.POINTER(C.c_uint32))
    _sig(lib, "dampr_host_unique_small", vp, u64, u64, vp, pu64, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_kv_create", vp, u64, pvp)
    _sig(lib, "dampr_kv_destroy", vp, vp)
    _sig(lib, "dampr_kv_size", vp, vp, pu64)
    _sig(lib, "dampr_kv_set_size", vp, vp, u64)
    _sig(lib, "dampr_kv_devptr", vp, vp, pu64)
    _sig(lib, "dampr_kv_upload", vp, vp, u64, vp, u64)
    _sig(lib, "dampr_kv_download", vp, vp, u64, vp, u64)
    _sig(lib, "dampr_kv_upload_columns", vp, vp, u64, vp, vp, u64)
    _sig(lib, "dampr_kv_download_columns", vp, vp, u64, vp, vp, u64)
    _sig(lib, "dampr_kv_sort", vp, vp, i32)
    _sig(lib, "dampr_kv_reduce_by_key", vp, vp, i32, pvp)
    _sig(lib, "dampr_kv_group_offsets", vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_kv_merge", vp, pvp, i32, i32, i32, pvp)
    _sig(lib, "dampr_kv_merge_ranges", vp, vp, vp, i32, i32, i32, pvp)
    _sig(lib, "dampr_kv_sort_reduce", vp, vp, i32, i32, pvp)
    _sig(lib, "dampr_kv_join_ranges", vp, vp, vp, i32, vp, u64, pu64)
    _sig(lib, "dampr_kv_hash_join", vp, vp, vp, pvp, pvp)
    _sig(lib, "dampr_kv_hash_probe", vp, vp, vp, pvp, vp)
    _sig(lib, "dampr_kv_partition_by_owner", vp, vp, i32, pvp, vp)
    _sig(lib, "dampr_comm_unique_id", vp, u32)
    _sig(lib, "dampr_comm_create", vp, i32, i32, vp, u32, pvp)
    _sig(lib, "dampr_comm_destroy", vp)
    _sig(lib, "dampr_kv_all_to_all", vp, vp, vp, vp, i32, pvp, vp, vp)
    _sig(lib, "dampr_synth_text", vp, vp, u64, u64, vp, vp, u32, vp, pu64)
    _sig(lib, "dampr_synth_kv", vp, vp, u64, u64, u64)
    _lib = lib
    return lib


def device_count():
    lib = load_library()
    n = C.c_int32(0)
    rc = lib.dampr_device_count(C.byref(n))
    return n.value if rc == 0 else 0


def set_option(name, value):
    rc = load_library().dampr_set_option(name.encode(), int(value))
    if rc:
        raise DeviceError("unknown option %r" % name)


def _ptr(a):
    """Host pointer of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


COMM_ID_BYTES = 128


class PinnedBuffer(object):
    """Page-locked host memory exposed as a numpy uint8 array (ingest staging / spill ring)."""

    def __init__(self, nbytes):
        lib = load_library()
        p = C.c_void_p()
        rc = lib.dampr_host_alloc(int(nbytes), C.byref(p))
        if rc:
            raise DeviceError("pinned allocation of %d bytes failed" % nbytes)
        self._p = p
        self.nbytes = int(nbytes)
        buf = (C.c_uint8 * max(1, self.nbytes)).from_address(p.value)
        self.array = np.frombuffer(buf, dtype=np.uint8, count=self.nbytes)

    def free(self):
        if self._p is not None:
            self.array = None
            load_library().dampr_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def host_register(arr):
    """Page-lock the memory of a C-contiguous numpy array (cudaHostRegister). True on success; the caller must
    host_unregister() before the array is released."""
    return load_library().dampr_host_register(_ptr(arr), int(arr.nbytes)) == 0


def host_unregister(arr):
    load_library().dampr_host_unregister(_ptr(arr))


class Ctx(object):
    """One GPU: a compute stream, a copy stream and the kernels' event timings."""

    def __init__(self, device=0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.dampr_ctx_create(int(device), C.byref(h))
        if rc:
            raise DeviceError(
                "cannot create a device context on cuda:%d (status %d): the engine needs a "
                "CUDA device and has no CPU fallback" % (device, rc))
        self.h = h
        self.device = device

    # -- plumbing ---------------------------------------------------------------------------
    def check(self, rc):
        if rc:
            msg = self.lib.dampr_last_error(self.h)
            raise DeviceError("libdampr_b200 status %d: %s" % (rc, msg.decode() if msg else "?"))

    def sync(self):
        self.check(self.lib.dampr_ctx_sync(self.h))

    def sync_copy_stream(self):
        self.check(self.lib.dampr_ctx_sync_copy(self.h))

    def close(self):
        if self.h is not None:
            if getattr(self, "comm", None) is not None:
                self.lib.dampr_comm_destroy(self.comm)
                self.comm = None
            self.lib.dampr_ctx_destroy(self.h)
            self.h = None

    def num_sms(self):
        n = C.c_int32(0)
        self.check(self.lib.dampr_ctx_num_sms(self.h, C.byref(n)))
        return n.value

    def mem_info(self):
        f, t = C.c_uint64(0), C.c_uint64(0)
        self.check(self.lib.dampr_ctx_mem_info(self.h, C.byref(f), C.byref(t)))
        return f.value, t.value

    def launches(self):
        n = C.c_uint64(0)
        self.check(self.lib.dampr_ctx_launches(self.h, C.byref(n)))
        return n.value

    def stream(self):
        s = C.c_uint64(0)
        self.check(self.lib.dampr_ctx_stream(self.h, C.byref(s)))
        return s.value

    def timing_enable(self, on):
        self.check(self.lib.dampr_ctx_timing_enable(self.h, 1 if on else 0))

    def timings_reset(self):
        self.check(self.lib.dampr_ctx_timings_reset(self.h))

    def timings(self, cap=65536):
        """[(kernel name, ms)] of every timed launch since the last reset (blocks)."""
        ms = (C.c_double * cap)()
        ids = (C.c_int32 * cap)()
        n = C.c_int32(0)
        self.check(self.lib.dampr_ctx_timings(self.h, ms, ids, cap, C.byref(n)))
        return [(KERNEL_NAMES.get(ids[i], str(ids[i])), ms[i]) for i in range(n.value)]

    # -- factories --------------------------------------------------------------------------
    def textbuf(self, capacity):
        return TextBuf(self, capacity)

    def table(self, capacity_log2=22):
        return Table(self, capacity_log2)

    def kv(self, capacity):
        return KV(self, capacity)

    def kv_from_columns(self, keys, vals=None):
        keys = np.ascontiguousarray(keys).view(np.uint64)
        kv = KV(self, len(keys))
        if vals is not None:
            vals = np.ascontiguousarray(vals)
            assert vals.dtype.itemsize == 8 and len(vals) == len(keys)
            vals = vals.view(np.uint64)
        self.check(self.lib.dampr_kv_upload_columns(self.h, kv.h, 0, _ptr(keys), _ptr(vals), len(keys)))
        self.sync()  # the host arrays may be temporaries
        return kv

    def synth_text(self, seed, n_lines, vocab_bytes, vocab_off, cdf, capacity=None):
        """Device-side synthetic corpus (bench/test tooling; same algorithm as oracle/gen.py)."""
        cap = int(capacity) if capacity else int(n_lines) * 120 + (1 << 20)
        tb = TextBuf(self, cap)
        out = C.c_uint64(0)
        self.check(self.lib.dampr_synth_text(self.h, tb.h, int(seed), int(n_lines), _ptr(vocab_bytes),
                                             _ptr(vocab_off), len(vocab_off) - 1, _ptr(cdf), C.byref(out)))
        tb.n = out.value
        return tb

    def kv_merge(self, runs, xform, op=-1):
        """k-way merge (op < 0) or merge + fold of key-sorted KVs -> new KV (stable: run order, then position)"""
        arr = (C.c_void_p * len(runs))(*[r.h for r in runs])
        h = C.c_void_p()
        self.check(self.lib.dampr_kv_merge(self.h, arr, len(runs), int(xform), int(op), C.byref(h)))
        return KV(self, None, handle=h)

    def kv_merge_ranges(self, kv, offsets, xform, op=-1):
        """the same over the sorted runs kv[offsets[i]:offsets[i+1]] of one KV"""
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        h = C.c_void_p()
        self.check(self.lib.dampr_kv_merge_ranges(self.h, kv.h, offs.ctypes.data_as(C.c_void_p), len(offs) - 1,
                                                  int(xform), int(op), C.byref(h)))
        return KV(self, None, handle=h)

    # ---- the shuffle exchange inside the C-ABI (csrc/comm.cu) --------------------------------------------
    @staticmethod
    def comm_unique_id():
        """128 bytes rank 0 creates and every rank passes to comm_create (ncclGetUniqueId)."""
        buf = (C.c_uint8 * COMM_ID_BYTES)()
        if load_library().dampr_comm_unique_id(buf, COMM_ID_BYTES):
            raise DeviceError("NCCL is not available (dampr_comm_unique_id)")
        return bytes(buf)

    def comm_create(self, rank, world, unique_id):
        """This context's NCCL communicator (one per process / GPU); kept on the context."""
        assert len(unique_id) >= COMM_ID_BYTES
        idb = (C.c_uint8 * len(unique_id)).from_buffer_copy(unique_id)
        h = C.c_void_p()
        self.check(self.lib.dampr_comm_create(self.h, int(rank), int(world), idb, len(unique_id), C.byref(h)))
        self.comm, self.comm_world = h, int(world)
        return h

    def kv_all_to_all(self, kv, header=None):
        """Every record to the owner of its key (owner = mix(key) % world). Returns (received KV, offsets, headers):
        the records of source rank s are recv[offsets[s]:offsets[s+1]] in the order rank s held them; headers is
        the (world, len(header)) int64 matrix of every rank's header values (None without a header)."""
        assert getattr(self, "comm", None) is not None, "comm_create first"
        w = self.comm_world
        hdr = np.ascontiguousarray(header if header is not None else [], dtype=np.int64)
        allh = np.zeros((w, max(1, len(hdr))), dtype=np.int64)
        offs = np.zeros(w + 1, dtype=np.uint64)
        h = C.c_void_p()
        self.check(self.lib.dampr_kv_all_to_all(self.h, self.comm, kv.h, _ptr(hdr) if len(hdr) else None, len(hdr),
                                                C.byref(h), _ptr(offs), _ptr(allh) if len(hdr) else None))
        return KV(self, None, handle=h), offs, (allh[:, :len(hdr)] if len(hdr) else None)

    def synth_kv(self, seed, n, n_keys):
        kv = KV(self, n)
        self.check(self.lib.dampr_synth_kv(self.h, kv.h, int(seed), int(n), int(n_keys)))
        return kv

    def kv_from_records(self, recs):
        """recs: numpy array of shape (n, 2) uint64 (or a structured 16-byte dtype)."""
        recs = np.ascontiguousarray(recs)
        assert recs.nbytes % 16 == 0
        n = recs.nbytes // 16
        kv = KV(self, n)
        self.check(self.lib.dampr_kv_upload(self.h, kv.h, 0, _ptr(recs), n))
        self.sync()
        return kv


class TextBuf(object):
    def __init__(self, ctx, capacity):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx.lib.dampr_textbuf_create(ctx.h, int(capacity), C.byref(h)))
        self.h = h
        self.capacity = int(capacity)
        self.n = 0

    def set_length(self, n):
        self.ctx.check(self.ctx.lib.dampr_textbuf_set_length(self.ctx.h, self.h, int(n)))
        self.n = int(n)

    def upload(self, off, host_u8, length=None):
        """Async copy of host bytes (numpy uint8 view; pinned for full speed) to text[off:]."""
        length = len(host_u8) if length is None else length
        self.ctx.check(self.ctx.lib.dampr_textbuf_upload(self.ctx.h, self.h, int(off), _ptr(host_u8), int(length)))

    def upload_file(self, off, path, file_off, length):
        """Async copy of bytes [file_off, file_off + length) of a file to text[off:]: the library's copy threads
        pread() the page cache into its page-locked ring, slot by slot, ahead of the DMA."""
        self.ctx.check(self.ctx.lib.dampr_textbuf_upload_file(self.ctx.h, self.h, int(off), os.fsencode(path),
                                                              int(file_off), int(length)))

    def upload_all(self, data):
        """Convenience: whole text from bytes / numpy (blocking)."""
        arr = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        self.set_length(len(arr))
        self.upload(0, arr)
        self.ctx.sync()

    def download(self, off, length):
        out = np.empty(int(length), dtype=np.uint8)
        self.ctx.check(self.ctx.lib.dampr_textbuf_download(self.ctx.h, self.h, int(off), _ptr(out), int(length)))
        return out

    def free(self):
        if self.h is not None:
            self.ctx.lib.dampr_textbuf_destroy(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h is not None:
                self.free()
        except Exception:
            pass


class Table(object):
    """Device combiner table: token key code -> count (ReducedWriter, dataset.py:84-117)."""

    def __init__(self, ctx, capacity_log2=22):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx.lib.dampr_table_create(ctx.h, int(capacity_log2), C.byref(h)))
        self.h = h
        self.capacity = 1 << capacity_log2

    def clear(self):
        self.ctx.check(self.ctx.lib.dampr_table_clear(self.ctx.h, self.h))

    def count(self, tb, lo, hi, mode, cr_is_data=False):
        """cr_is_data: '\\r' is an ordinary byte (the reference's binary-mode .gz reader) instead of a line end"""
        m = int(mode) | (TOK_FLAG_CR_DATA if cr_is_data else 0)
        self.ctx.check(self.ctx.lib.dampr_text_count(self.ctx.h, self.h, tb.h, int(lo), int(hi), m))

    def fallback_lines(self):
        """uint64[]: (byte offset << 16) | length of every line the [^\\w]+ tokenisers handed back to the host"""
        n = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_table_fallback_lines(self.ctx.h, self.h, None, 0, C.byref(n)))
        out = np.empty(n.value, dtype=np.uint64)
        if n.value:
            self.ctx.check(self.ctx.lib.dampr_table_fallback_lines(self.ctx.h, self.h, _ptr(out), len(out), C.byref(n)))
        return out

    def verify(self, tb, lo, hi, mode):
        self.ctx.check(self.ctx.lib.dampr_text_verify(self.ctx.h, self.h, tb.h, int(lo), int(hi), int(mode)))

    def stats(self):
        st = (C.c_uint64 * 8)()
        self.ctx.check(self.ctx.lib.dampr_table_stats(self.ctx.h, self.h, st))
        return {"entries": st[0], "lines": st[1], "empty": st[2], "folded": st[3], "flags": st[4],
                "hashed": st[5], "raw": st[6], "fallback": st[7]}

    def fetch(self):
        """(codes, counts, reps) numpy uint64 arrays (unordered)."""
        n = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_table_fetch(self.ctx.h, self.h, None, None, None, 0, C.byref(n)))
        m = n.value
        codes = np.empty(m, dtype=np.uint64)
        counts = np.empty(m, dtype=np.uint64)
        reps = np.empty(m, dtype=np.uint64)
        if m:
            self.ctx.check(self.ctx.lib.dampr_table_fetch(self.ctx.h, self.h, _ptr(codes), _ptr(counts), _ptr(reps),
                                                          m, C.byref(n)))
        return codes, counts, reps

    def fetch_words(self, tb, mode, width=32, with_codes=True):
        """(words 'S<width>' array decoded on the device, counts, codes, reps); codes and reps are None
        when with_codes is false (tables without hashed tokens need neither)."""
        n = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_table_fetch_words(self.ctx.h, self.h, None, int(mode), int(width), None,
                                                            None, None, None, 0, C.byref(n)))
        m = n.value
        words = np.empty((m, width), dtype=np.uint8)   # the kernel writes every byte (NUL padded)
        counts = np.empty(m, dtype=np.uint64)
        codes = np.empty(m, dtype=np.uint64) if with_codes else None
        reps = np.empty(m, dtype=np.uint64) if with_codes else None
        if m:
            self.ctx.check(self.ctx.lib.dampr_table_fetch_words(
                self.ctx.h, self.h, tb.h if tb is not None else None, int(mode), int(width), _ptr(words),
                _ptr(counts), _ptr(codes) if with_codes else None, _ptr(reps) if with_codes else None, m,
                C.byref(n)))
        return words.view("S%d" % width).ravel(), counts, codes, reps

    def to_kv(self):
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.dampr_table_to_kv(self.ctx.h, self.h, C.byref(h)))
        return KV(self.ctx, None, handle=h)

    def free(self):
        if self.h is not None:
            self.ctx.lib.dampr_table_destroy(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h is not None:
                self.free()
        except Exception:
            pass


class KV(object):
    """Device array of 16-byte (u64 key, u64 value) records."""

    def __init__(self, ctx, capacity, handle=None):
        self.ctx = ctx
        if handle is None:
            handle = C.c_void_p()
            ctx.check(ctx.lib.dampr_kv_create(ctx.h, int(capacity), C.byref(handle)))
        self.h = handle

    def __len__(self):
        n = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_kv_size(self.ctx.h, self.h, C.byref(n)))
        return n.value

    def set_size(self, n):
        self.ctx.check(self.ctx.lib.dampr_kv_set_size(self.ctx.h, self.h, int(n)))

    def devptr(self):
        p = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_kv_devptr(self.ctx.h, self.h, C.byref(p)))
        return p.value

    def upload_columns(self, off, keys, vals):
        """Column chunks -> records [off, off + len(keys)) (interleaved on the device)."""
        keys = np.ascontiguousarray(keys).view(np.uint64)
        vals = np.ascontiguousarray(vals)
        assert vals.dtype.itemsize == 8 and len(vals) == len(keys)
        self.ctx.check(self.ctx.lib.dampr_kv_upload_columns(self.ctx.h, self.h, int(off), _ptr(keys),
                                                            _ptr(vals.view(np.uint64)), len(keys)))

    def upload(self, off, recs, count=None):
        count = recs.nbytes // 16 if count is None else count
        self.ctx.check(self.ctx.lib.dampr_kv_upload(self.ctx.h, self.h, int(off), _ptr(recs), int(count)))

    def records(self):
        """Download as an (n, 2) uint64 array."""
        n = len(self)
        out = np.empty((n, 2), dtype=np.uint64)
        self.ctx.check(self.ctx.lib.dampr_kv_download(self.ctx.h, self.h, 0, _ptr(out), n))
        return out

    def records_into(self, out, off=0):
        """Download records [off, off + len(out)) into a caller-provided contiguous (m, 2) uint64 array."""
        m = len(out)
        assert out.dtype == np.uint64 and out.ndim == 2 and out.shape[1] == 2 and out.flags.c_contiguous
        assert off + m <= len(self)
        self.ctx.check(self.ctx.lib.dampr_kv_download(self.ctx.h, self.h, int(off), _ptr(out), m))
        return out

    def columns(self):
        n = len(self)
        keys = np.empty(n, dtype=np.uint64)
        vals = np.empty(n, dtype=np.uint64)
        self.ctx.check(self.ctx.lib.dampr_kv_download_columns(self.ctx.h, self.h, 0, _ptr(keys), _ptr(vals), n))
        return keys, vals

    def columns_into(self, keys, vals):
        """Download into caller-provided contiguous uint64 arrays of len(self) elements (no allocation)."""
        n = len(self)
        assert keys.dtype == np.uint64 and vals.dtype == np.uint64 and len(keys) == n and len(vals) == n
        assert keys.flags.c_contiguous and vals.flags.c_contiguous
        self.ctx.check(self.ctx.lib.dampr_kv_download_columns(self.ctx.h, self.h, 0, _ptr(keys), _ptr(vals), n))

    def decode_words(self, mode, width=32):
        """Keys are token codes: 'S<width>' array decoded on the device (hashed codes -> b'')."""
        n = len(self)
        words = np.empty((n, width), dtype=np.uint8)
        self.ctx.check(self.ctx.lib.dampr_kv_decode_words(self.ctx.h, self.h, int(mode), int(width), _ptr(words)))
        return words.view("S%d" % width).ravel()

    def sort(self, xform=KEY_MIX):
        self.ctx.check(self.ctx.lib.dampr_kv_sort(self.ctx.h, self.h, int(xform)))
        return self

    def sort_reduce(self, op, xform=KEY_MIX, sorted_run=False):
        """One record per key. The groups come out in key order under `xform`, except for the commutative
        integer folds under KEY_MIX (SUM / COUNT / MIN / MAX), which the leaves fold through a shared-memory
        hash table: there the order is by bucket of the mixed key only. sorted_run=True sorts those too, so
        the result can feed the k-way merge as a sorted run."""
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.dampr_kv_sort_reduce(self.ctx.h, self.h, int(xform), int(op), C.byref(h)))
        out = KV(self.ctx, None, handle=h)
        if sorted_run and xform == KEY_MIX and op in (OP_SUM_I64, OP_COUNT, OP_MIN_I64, OP_MAX_I64):
            out.sort(xform)
        return out

    def reduce_by_key(self, op):
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.dampr_kv_reduce_by_key(self.ctx.h, self.h, int(op), C.byref(h)))
        return KV(self.ctx, None, handle=h)

    def count_groups(self):
        """number of key groups of a key-sorted kv (nothing but the count leaves the device)"""
        g = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_kv_group_offsets(self.ctx.h, self.h, None, 0, C.byref(g)))
        return int(g.value)

    def group_offsets(self):
        g = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_kv_group_offsets(self.ctx.h, self.h, None, 0, C.byref(g)))
        offs = np.empty(g.value + 1, dtype=np.uint64)
        self.ctx.check(self.ctx.lib.dampr_kv_group_offsets(self.ctx.h, self.h, _ptr(offs), len(offs), C.byref(g)))
        return offs

    def join_ranges(self, right, xform):
        g = C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_kv_join_ranges(self.ctx.h, self.h, right.h, int(xform), None, 0, C.byref(g)))
        rows = np.empty((g.value, 4), dtype=np.uint64)
        if g.value:
            self.ctx.check(self.ctx.lib.dampr_kv_join_ranges(self.ctx.h, self.h, right.h, int(xform), _ptr(rows),
                                                             g.value, C.byref(g)))
        return rows

    def hash_probe(self, probe):
        """self = build side (unique keys). Returns (values KV aligned with probe, hit uint8 array)."""
        h = C.c_void_p()
        hit = np.empty(len(probe), dtype=np.uint8)
        self.ctx.check(self.ctx.lib.dampr_kv_hash_probe(self.ctx.h, self.h, probe.h, C.byref(h), _ptr(hit)))
        return KV(self.ctx, None, handle=h), hit

    def hash_join(self, probe):
        """self = build side (unique keys). Returns (matched probe records KV, (key, build value) KV), compacted on
        the device in probe order."""
        hp, hb = C.c_void_p(), C.c_void_p()
        self.ctx.check(self.ctx.lib.dampr_kv_hash_join(self.ctx.h, self.h, probe.h, C.byref(hp), C.byref(hb)))
        return KV(self.ctx, None, handle=hp), KV(self.ctx, None, handle=hb)

    def partition_by_owner(self, n_dest):
        h = C.c_void_p()
        counts = np.zeros(n_dest, dtype=np.uint64)
        self.ctx.check(self.ctx.lib.dampr_kv_partition_by_owner(self.ctx.h, self.h, int(n_dest), C.byref(h), _ptr(counts)))
        return KV(self.ctx, None, handle=h), counts

    def free(self):
        if self.h is not None:
            self.ctx.lib.dampr_kv_destroy(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            if self.ctx.h is not None:
                self.free()
        except Exception:
            pass


def host_join_tsv(columns, prefix=None, first=0, max_files=16, col_pre=None, row_end=None):
    """Rows of tab-separated text from columns (native host loop). Each column is either a numpy
    'S<w>' array (NUL-padded fixed-width strings), a pair (inv uint32 array, list of bytes) or a pair
    (inv uint32 array, int64 array of the distinct values). With `prefix` the rows are written to part files prefix<first>, prefix<first+1>, ... (row ranges, one
    writer thread per file; returns the file names) instead of returned."""
    lib = load_library()
    k = len(columns)
    n = None
    kinds = (C.c_int32 * k)()
    ptrs = (C.c_void_p * k)()
    widths = (C.c_uint32 * k)()
    aux = (C.c_void_p * k)()
    aux2 = (C.c_void_p * k)()
    keep = []
    for c, col in enumerate(columns):
        if isinstance(col, np.ndarray):
            assert col.dtype.kind == "S"
            arr = np.ascontiguousarray(col)
            kinds[c], widths[c] = 0, arr.dtype.itemsize
            ptrs[c] = arr.ctypes.data
            keep.append(arr)
            m = len(arr)
        elif isinstance(col[1], np.ndarray):   # (inv, int64 | float64 values): formatted natively
            inv, vals = col
            inv = np.ascontiguousarray(inv, dtype=np.uint32)
            if vals.dtype == np.float64:       # Python's repr(float) of every distinct value (kind 3)
                vals = np.ascontiguousarray(vals)
                kinds[c], widths[c] = 3, len(vals)
            else:
                vals = np.ascontiguousarray(vals, dtype=np.int64)
                kinds[c], widths[c] = 2, len(vals)
            ptrs[c], aux[c] = inv.ctypes.data, vals.ctypes.data
            keep.extend([inv, vals])
            m = len(inv)
        else:
            inv, strs = col
            inv = np.ascontiguousarray(inv, dtype=np.uint32)
            blob = b"".join(strs)
            off = np.zeros(len(strs) + 1, dtype=np.uint32)
            np.cumsum([len(s) for s in strs], out=off[1:])
            bl = np.frombuffer(blob, dtype=np.uint8) if blob else np.zeros(1, dtype=np.uint8)
            kinds[c], widths[c] = 1, 0
            ptrs[c], aux[c], aux2[c] = inv.ctypes.data, bl.ctypes.data, off.ctypes.data
            keep.extend([inv, bl, off])
            m = len(inv)
        assert n is None or n == m
        n = m
    out_len = C.c_uint64(0)
    if prefix is not None:
        nf = C.c_uint32(0)
        if col_pre is not None:
            # formatted rows (sink_json): a byte string in front of every column, row_end instead of the newline
            pre = (C.c_char_p * k)(*[bytes(x) for x in col_pre])
            rc = lib.dampr_host_sink_fmt(os.fsencode(prefix), int(first), int(max_files), n, k, kinds, ptrs, widths,
                                         aux, aux2, pre, bytes(row_end), C.byref(out_len), C.byref(nf))
        else:
            rc = lib.dampr_host_sink_tsv(os.fsencode(prefix), int(first), int(max_files), n, k, kinds, ptrs, widths,
                                         aux, aux2, C.byref(out_len), C.byref(nf))
        if rc:
            raise DeviceError("dampr_host_sink_tsv(%r) failed (%d)" % (prefix, rc))
        return ["%s%d" % (prefix, first + j) for j in range(nf.value)]
    rc = lib.dampr_host_join_tsv(n, k, kinds, ptrs, widths, aux, aux2, None, 0, C.byref(out_len))
    if rc:
        raise DeviceError("dampr_host_join_tsv failed (%d)" % rc)
    out = np.empty(out_len.value, dtype=np.uint8)
    rc = lib.dampr_host_join_tsv(n, k, kinds, ptrs, widths, aux, aux2, _ptr(out), len(out), C.byref(out_len))
    if rc:
        raise DeviceError("dampr_host_join_tsv failed (%d)" % rc)
    return out


def host_unique_small(col, table=1 << 20, with_rows=False):
    """(uniq ascending, inv uint32[, first row of every distinct value]) of an int64 column whose values
    are mostly in [0, table), or None when too many values fall outside (the caller then uses a sort)."""
    lib = load_library()
    col = np.ascontiguousarray(col, dtype=np.int64)
    n = len(col)
    # the presence table is cleared and scanned once: keep it proportional to the column
    table = int(min(table, max(4096, 1 << int(2 * n - 1).bit_length())))
    cap = n // 8 + 16
    uniq = np.empty(min(n, table), dtype=np.int64)
    inv = np.empty(n, dtype=np.uint32)
    bv = np.empty(cap, dtype=np.int64)
    br = np.empty(cap, dtype=np.uint64)
    m, nb = C.c_uint64(0), C.c_uint64(0)
    rows = np.empty(min(n, table), dtype=np.uint32) if with_rows else None
    rc = lib.dampr_host_unique_small(_ptr(col), n, table, _ptr(uniq), C.byref(m), _ptr(inv), _ptr(rows), _ptr(bv),
                                     _ptr(br), cap, C.byref(nb))
    if rc:
        return None
    m, nb = m.value, nb.value
    uniq = uniq[:m]
    rows = rows[:m].astype(np.int64) if with_rows else None
    if nb:
        bv, br = bv[:nb], br[:nb].astype(np.int64)
        if int(bv.min()) < table:   # negative values: the two ranges would interleave
            return None
        ul, il = np.unique(bv, return_inverse=True)
        inv[br] = il.astype(np.uint32) + np.uint32(m)
        uniq = np.concatenate((uniq, ul))
        if with_rows:
            rb = np.empty(len(ul), dtype=np.int64)
            rb[il] = br
            rows = np.concatenate((rows, rb))
    return (uniq, inv, rows) if with_rows else (uniq, inv)


def kv_merge_ranges(ctx, kv, offsets, xform, op=-1):
    return ctx.kv_merge_ranges(kv, offsets, xform, op)


def kv_merge(ctx, runs, xform, op=-1):
    return ctx.kv_merge(runs, xform, op)

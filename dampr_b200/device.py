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
TF_RECFULL, TF_NEGZERO = 64, 128   # field scans: record buffer full / a float() field parsed to -0.0
TF_JSON_KEY_KIND, TF_JSON_VAL_KIND = 256, 512   # JSON scans: a key / value member of the other JSON kind
TF_NAN = 1024   # expression scans: a computed float value is a NaN
TOK_FLAG_CR_DATA = 0x100
# delimited-field scans (dampr_text_fields)
FIELD_KEY_STR, FIELD_KEY_INT = 0, 1
FIELD_VAL_ONE = 0x7FFFFFFF
FIELD_SEP_WS = 256   # sep: split like str.split() (runs of ASCII whitespace, no '' fields)
FIELD_SEP_JSON = 257   # sep of the JSON-lines calls: fields are the members of json.loads(line)
JSON_MAX_MEMBERS, JSON_MAX_NAME, JSON_MAX_DEPTH = 8, 64, 64
JSON_PATH_SEP, JSON_MAX_PATH, JSON_MAX_NODES = 0x1F, 4, 16   # member paths: names joined by JSON_PATH_SEP
FIELDS_HALO = 65536
FIELD_KEYS_MAX = 4   # components of a tuple key (dampr_field_keys)
# computed keys and values of a field scan (dampr_field_expr): limits, program types, load slot kinds
EXPR_MAX_OPS, EXPR_MAX_LOADS, EXPR_MAX_DEPTH, EXPR_MAX_CONSTS = 32, 4, 8, 16
EXPR_NONE, EXPR_INT, EXPR_F64 = 0, 1, 2
LOAD_INT, LOAD_F64, LOAD_LEN = 0, 1, 2
# WHERE predicates of a field scan (dampr_field_pred): kinds, comparisons, limits per call
PRED_STR, PRED_INT, PRED_F64, PRED_NFIELDS, PRED_MEMBER, PRED_LEN, PRED_NONBLANK, PRED_AND, PRED_OR, PRED_NOT = range(10)
CMP_EQ, CMP_NE, CMP_LT, CMP_LE, CMP_GT, CMP_GE, CMP_IN, CMP_NOT_IN, CMP_CONTAINS, CMP_NOT_CONTAINS, CMP_STARTS, \
    CMP_ENDS = range(12)
PRED_MAX, PRED_MAX_CONSTS, PRED_MAX_BYTES, PRED_MAX_OPS = 8, 64, 1024, 8
FIELD_LINE = -(1 << 31)   # a predicate's field that is the whole line

KERNEL_NAMES = {
    1: "text_count", 2: "table_extract", 3: "text_verify", 4: "part_hist", 5: "part_scatter",
    6: "leaf_sort", 7: "seg_reduce", 8: "merge", 9: "join", 10: "probe", 11: "synth", 12: "misc",
    13: "text_fields", 14: "text_fields_count",
}


def decode_fold(acc, op):
    """int64 values of a field scan's accumulators (uint64): MAX keeps v ^ 2^63, MIN ~(v ^ 2^63), SUM v; float64
    values under MIN_F64 / MAX_F64, whose codes are bits ^ (sign ? ~0 : 2^63) (MIN: the complement)"""
    acc = np.asarray(acc, dtype=np.uint64)
    if op in (OP_MIN_F64, OP_MAX_F64):
        c = ~acc if op == OP_MIN_F64 else acc
        return np.where(c >> np.uint64(63) != 0, c ^ np.uint64(1 << 63), ~c).view(np.float64)
    if op == OP_MIN_I64:
        acc = ~acc
    if op in (OP_MIN_I64, OP_MAX_I64):
        acc = acc ^ np.uint64(1 << 63)
    return acc.view(np.int64)


class FieldPred(C.Structure):
    """dampr_field_pred"""
    _fields_ = [("kind", C.c_int32), ("field", C.c_int32), ("cmp", C.c_int32), ("n", C.c_int32),
                ("ints", C.POINTER(C.c_int64)), ("f64", C.c_double), ("bytes", C.POINTER(C.c_uint8)),
                ("lens", C.POINTER(C.c_uint32))]


class FieldsSpec(C.Structure):
    """dampr_fields_spec"""
    _fields_ = [("sep", C.c_int32), ("key_field", C.c_int32), ("key_kind", C.c_int32), ("val_field", C.c_int32),
                ("op", C.c_int32), ("cr_is_data", C.c_int32), ("preds", C.POINTER(FieldPred)), ("npreds", C.c_int32)]


def fields_spec(spec, cr_is_data, preds):
    """dampr_fields_spec of spec = (sep byte or FIELD_SEP_WS, key field, key kind, value field or FIELD_VAL_ONE, op)
    and the WHERE predicates preds = [(PRED_*, field, CMP_*, constants)]: constants a tuple of str (PRED_STR), int
    (PRED_INT, PRED_NFIELDS, PRED_LEN) or one float (PRED_F64), () for PRED_NONBLANK, PRED_MEMBER (or, over member
    paths, the member's last name, a str) and the connectives
    PRED_AND / PRED_OR / PRED_NOT of a postfix program. The returned structure keeps its constant arrays alive."""
    sep, kf, kind, vf, op = spec
    arr = (FieldPred * max(1, len(preds)))()
    keep = [arr]
    for p, (pk, field, cmp, consts) in zip(arr, preds):
        p.kind, p.field, p.cmp, p.n = int(pk), int(field), int(cmp), len(consts)
        if pk == PRED_F64:
            p.f64 = float(consts[0])
        elif pk == PRED_STR or pk == PRED_MEMBER:   # a member test's one constant: the substring of a str container
            raw = [c.encode("utf-8") for c in consts]
            b = (C.c_uint8 * max(1, sum(map(len, raw)))).from_buffer_copy(b"".join(raw).ljust(1, b"\0"))
            ln = (C.c_uint32 * len(raw))(*map(len, raw))
            p.bytes, p.lens = C.cast(b, C.POINTER(C.c_uint8)), C.cast(ln, C.POINTER(C.c_uint32))
            keep += [b, ln]
        elif consts:
            v = (C.c_int64 * len(consts))(*map(int, consts))
            p.ints = C.cast(v, C.POINTER(C.c_int64))
            keep.append(v)
    s = FieldsSpec(int(sep), int(kf), int(kind), int(vf), int(op), 1 if cr_is_data else 0,
                   C.cast(arr, C.POINTER(FieldPred)), len(preds))
    s._keep = keep
    return s


class FieldKeys(C.Structure):
    """dampr_field_keys"""
    _fields_ = [("n", C.c_int32), ("field", C.c_int32 * FIELD_KEYS_MAX), ("kind", C.c_int32 * FIELD_KEYS_MAX)]


def field_keys(keys):
    """dampr_field_keys of the tuple key components keys = [(field index, FIELD_KEY_STR | FIELD_KEY_INT)]"""
    k = FieldKeys()
    k.n = len(keys)
    for j, (i, kind) in enumerate(keys[:FIELD_KEYS_MAX]):
        k.field[j], k.kind[j] = int(i), int(kind)
    return k


class FieldExpr(C.Structure):
    """dampr_field_expr"""
    _fields_ = [("key_type", C.c_int32), ("key_len", C.c_int32), ("key_prog", C.c_int32 * EXPR_MAX_OPS),
                ("val_type", C.c_int32), ("val_len", C.c_int32), ("val_prog", C.c_int32 * EXPR_MAX_OPS),
                ("ci", C.c_int64 * EXPR_MAX_CONSTS), ("cf", C.c_double * EXPR_MAX_CONSTS), ("nloads", C.c_int32),
                ("load_field", C.c_int32 * EXPR_MAX_LOADS), ("load_kind", C.c_int32 * EXPR_MAX_LOADS)]


def field_expr(expr):
    """dampr_field_expr of expr = (key program or None, value program or None, int constants, float constants,
    loads): a program is (EXPR_INT | EXPR_F64, [opcode words]), loads [(field index, LOAD_*)]. Out-of-range lengths
    are passed on for the library to refuse."""
    key, val, ci, cf, loads = expr
    x = FieldExpr()
    for prog, t, n, words in ((key, "key_type", "key_len", x.key_prog), (val, "val_type", "val_len", x.val_prog)):
        if prog is not None:
            setattr(x, t, int(prog[0]))
            setattr(x, n, len(prog[1]))
            for i, w in enumerate(prog[1][:EXPR_MAX_OPS]):
                words[i] = int(w)
    for i, c in enumerate(ci[:EXPR_MAX_CONSTS]):
        x.ci[i] = int(c)
    for i, c in enumerate(cf[:EXPR_MAX_CONSTS]):
        x.cf[i] = float(c)
    x.nloads = len(loads)
    for j, (f, kind) in enumerate(loads[:EXPR_MAX_LOADS]):
        x.load_field[j], x.load_kind[j] = int(f), int(kind)
    return x


class JsonMembers(C.Structure):
    """dampr_json_members"""
    _fields_ = [("n", C.c_int32), ("bytes", C.c_char_p), ("len", C.POINTER(C.c_int32))]


def json_members(names):
    """dampr_json_members of the members: a name (str) or a path (a tuple of names, joined by JSON_PATH_SEP); the
    returned structure keeps its arrays alive"""
    raw = [bytes([JSON_PATH_SEP]).join(x.encode("ascii") for x in n) if isinstance(n, tuple) else n.encode("ascii")
           for n in names]
    ln = (C.c_int32 * max(1, len(raw)))(*map(len, raw))
    m = JsonMembers(len(raw), b"".join(raw), C.cast(ln, C.POINTER(C.c_int32)))
    m._keep = ln
    return m


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
    _sig(lib, "dampr_text_fields", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec))
    _sig(lib, "dampr_text_fields_records", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), vp)
    _sig(lib, "dampr_text_json_fields", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), C.POINTER(JsonMembers))
    _sig(lib, "dampr_text_json_fields_records", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), C.POINTER(JsonMembers),
         vp)
    _sig(lib, "dampr_text_fields_tuple", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), C.POINTER(FieldKeys))
    _sig(lib, "dampr_text_fields_tuple_records", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), C.POINTER(FieldKeys), vp)
    _sig(lib, "dampr_text_fields_expr", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), C.POINTER(FieldExpr))
    _sig(lib, "dampr_text_fields_expr_records", vp, vp, vp, u64, u64, C.POINTER(FieldsSpec), C.POINTER(FieldExpr), vp)
    _sig(lib, "dampr_table_fetch_field_keys", vp, vp, vp, i32, C.POINTER(FieldKeys), C.POINTER(u32), C.POINTER(vp),
         vp, vp, u64, pu64)
    _sig(lib, "dampr_table_stats", vp, vp, pu64)
    _sig(lib, "dampr_table_fallback_lines", vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_table_fetch", vp, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_table_to_kv", vp, vp, pvp)
    _sig(lib, "dampr_table_fetch_words", vp, vp, vp, i32, u32, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_table_fetch_words_leased", vp, vp, vp, i32, u32, i32, pvp, pu64, pu64)
    _sig(lib, "dampr_table_extracted_counts", vp, vp, pu64, pu64)
    _sig(lib, "dampr_count_dictionary", vp, vp, u64, u32, vp, u32, vp, vp, vp, pu64)
    _sig(lib, "dampr_count_dictionary_leased", vp, vp, u64, u32, vp, u32, pvp, pu64, pu64)
    _sig(lib, "dampr_result_lease", vp, u64, pvp, pu64)
    _sig(lib, "dampr_result_release", vp, u64)
    _sig(lib, "dampr_host_pool_threads", pu64)
    _sig(lib, "dampr_host_eval_f64", vp, u64, vp, u32, vp, vp, vp)
    _sig(lib, "dampr_kv_decode_words", vp, vp, i32, u32, vp)
    _sig(lib, "dampr_host_join_tsv", u64, i32, vp, vp, vp, vp, vp, vp, u64, pu64)
    _sig(lib, "dampr_host_sink_tsv", C.c_char_p, C.c_uint32, C.c_uint32, u64, i32, vp, vp, vp, vp, vp, pu64,
         C.POINTER(C.c_uint32))
    _sig(lib, "dampr_host_sink_fmt", C.c_char_p, C.c_uint32, C.c_uint32, u64, i32, vp, vp, vp, vp, vp, vp, C.c_char_p, pu64,
         C.POINTER(C.c_uint32))
    _sig(lib, "dampr_host_sink_timings", C.POINTER(C.c_double))
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


def _apply_result_cache():
    """settings.host_result_cache_bytes -> the library (read at every call that leases or keeps host memory)"""
    from . import settings
    set_option("host_result_cache_bytes", max(0, int(settings.host_result_cache_bytes or 0)))


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


class ResultLease(object):
    """A page-locked block of a context's result arena (dampr_result_lease) as the base object of numpy arrays:
    array() returns views whose memory is this block, every view and every slice of one keeps the lease alive, and
    the block goes back to the arena when the last of them is gone."""

    def __init__(self, ctx, handle, ptr, nbytes):
        self.ctx, self.handle, self.nbytes = ctx, int(handle), int(nbytes)
        self.__array_interface__ = {"shape": (self.nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 3}

    def array(self, offset, count, dtype):
        """`count` items of `dtype` at byte `offset` of the block"""
        dtype = np.dtype(dtype)
        raw = np.asarray(self)
        assert raw.base is self and offset + count * dtype.itemsize <= self.nbytes
        return raw[offset:offset + count * dtype.itemsize].view(dtype)

    def __del__(self):
        try:
            if self.handle and self.ctx.h is not None:
                self.ctx.lib.dampr_result_release(self.ctx.h, self.handle)
            self.handle = 0
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

    def count_dictionary(self, dev_ptr, n, stride=1, extra=()):
        """(sorted distinct values int64, inverse uint32, smallest row of every value int64) of a non-negative
        count column on the device (dampr_count_dictionary): rows 0..n-1 are the u64 values at dev_ptr (every
        `stride`-th), then the host values `extra`. None when a value is negative."""
        ex = np.ascontiguousarray(extra, dtype=np.int64)
        N = int(n) + len(ex)
        cptr = C.c_void_p(int(dev_ptr)) if n else None
        _apply_result_cache()
        # into one page-locked block of the result arena; without one (see dampr_result_lease), into pageable arrays
        m, p, lease = C.c_uint64(0), C.c_void_p(), C.c_uint64(0)
        rc = self.lib.dampr_count_dictionary_leased(self.h, cptr, int(n), int(stride), _ptr(ex) if len(ex) else None,
                                                    len(ex), C.byref(p), C.byref(lease), C.byref(m))
        if rc == -5:   # DAMPR_ERR_UNSUPPORTED
            return None
        self.check(rc)
        if lease.value:
            m = m.value
            blk = ResultLease(self, lease.value, p.value, 12 * m + 4 * N)
            return blk.array(0, m, np.int64), blk.array(8 * m, N, np.uint32), \
                blk.array(8 * m + 4 * N, m, np.uint32).astype(np.int64)
        uniq = np.empty(max(1, N), dtype=np.int64)
        inv = np.empty(N, dtype=np.uint32)
        rows = np.empty(max(1, N), dtype=np.uint32)
        m = C.c_uint64(0)
        rc = self.lib.dampr_count_dictionary(self.h, cptr, int(n), int(stride),
                                             _ptr(ex) if len(ex) else None, len(ex), _ptr(uniq), _ptr(inv),
                                             _ptr(rows), C.byref(m))
        if rc == -5:   # DAMPR_ERR_UNSUPPORTED
            return None
        self.check(rc)
        m = m.value
        return uniq[:m], inv, rows[:m].astype(np.int64)

    def count_dictionary_of(self, counts, extra=()):
        """count_dictionary of a host column (uploaded as the values of a kv's records)"""
        counts = np.ascontiguousarray(counts).view(np.uint64)
        kv = self.kv_from_columns(np.zeros(len(counts), dtype=np.uint64), counts)
        try:
            return self.count_dictionary(kv.devptr() + 8, len(counts), 2, extra)
        finally:
            kv.free()


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
        self.fetches = 0   # fetch_words / clear calls so far: tells whether extracted_counts() is still a given fetch's

    def clear(self):
        self.fetches += 1
        self.ctx.check(self.ctx.lib.dampr_table_clear(self.ctx.h, self.h))

    def extracted_counts(self):
        """(device pointer, length) of the count column the last fetch_words downloaded, in its row order"""
        p, n = C.c_uint64(0), C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_table_extracted_counts(self.ctx.h, self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def count(self, tb, lo, hi, mode, cr_is_data=False):
        """cr_is_data: '\\r' is an ordinary byte (the reference's binary-mode .gz reader) instead of a line end"""
        m = int(mode) | (TOK_FLAG_CR_DATA if cr_is_data else 0)
        self.ctx.check(self.ctx.lib.dampr_text_count(self.ctx.h, self.h, tb.h, int(lo), int(hi), m))

    def fields(self, tb, lo, hi, spec, cr_is_data=False, preds=()):
        """Fold the delimited fields of the lines starting in [lo, hi): spec = (sep byte or FIELD_SEP_WS, key field,
        key kind, value field or FIELD_VAL_ONE, op); bytes up to hi + FIELDS_HALO must be uploaded. preds: the WHERE
        predicates (see fields_spec), applied in order before the key and value are read."""
        s = fields_spec(spec, cr_is_data, preds)
        self.ctx.check(self.ctx.lib.dampr_text_fields(self.ctx.h, self.h, tb.h, int(lo), int(hi), C.byref(s)))

    def fields_records(self, tb, lo, hi, spec, kv, cr_is_data=False, preds=()):
        """Record mode of fields() (spec op OP_SUM_I64 or OP_SUM_F64): one {key code, value} record per line starting
        in [lo, hi) into kv's buffer, in line order, holes {0, 0} for the lines left to the host or dropped by preds;
        the table counts the lines per key. fields_stats()["records"] is the scan's record count (kv's size is the
        caller's)."""
        s = fields_spec(spec, cr_is_data, preds)
        self.ctx.check(self.ctx.lib.dampr_text_fields_records(self.ctx.h, self.h, tb.h, int(lo), int(hi), C.byref(s),
                                                              kv.h))

    def json_fields(self, tb, lo, hi, spec, members, cr_is_data=False, preds=()):
        """fields() over JSON lines: spec = (FIELD_SEP_JSON, key member, key kind, value member or FIELD_VAL_ONE, op),
        the member indices (and the predicates' fields) index `members`, a list of member names"""
        s, m = fields_spec(spec, cr_is_data, preds), json_members(members)
        self.ctx.check(self.ctx.lib.dampr_text_json_fields(self.ctx.h, self.h, tb.h, int(lo), int(hi), C.byref(s),
                                                           C.byref(m)))

    def json_fields_records(self, tb, lo, hi, spec, members, kv, cr_is_data=False, preds=()):
        """fields_records() over JSON lines, spec and members as json_fields()"""
        s, m = fields_spec(spec, cr_is_data, preds), json_members(members)
        self.ctx.check(self.ctx.lib.dampr_text_json_fields_records(self.ctx.h, self.h, tb.h, int(lo), int(hi),
                                                                   C.byref(s), C.byref(m), kv.h))

    def fields_tuple(self, tb, lo, hi, spec, keys, cr_is_data=False, preds=()):
        """fields() grouped by a tuple key: keys = [(field index, FIELD_KEY_STR | FIELD_KEY_INT)], 1 .. FIELD_KEYS_MAX
        components on spec's separator (spec's key field and kind are not read)"""
        s, k = fields_spec(spec, cr_is_data, preds), field_keys(keys)
        self.ctx.check(self.ctx.lib.dampr_text_fields_tuple(self.ctx.h, self.h, tb.h, int(lo), int(hi), C.byref(s),
                                                            C.byref(k)))

    def fields_tuple_records(self, tb, lo, hi, spec, keys, kv, cr_is_data=False, preds=()):
        """fields_records() grouped by a tuple key, keys as fields_tuple()"""
        s, k = fields_spec(spec, cr_is_data, preds), field_keys(keys)
        self.ctx.check(self.ctx.lib.dampr_text_fields_tuple_records(self.ctx.h, self.h, tb.h, int(lo), int(hi),
                                                                    C.byref(s), C.byref(k), kv.h))

    def fields_expr(self, tb, lo, hi, spec, expr, cr_is_data=False, preds=()):
        """fields() with a computed key and / or value: expr as field_expr() (lowering.text_fields_expr's programs);
        a key program's int keys are coded as FIELD_KEY_INT keys (fetch() decodes them), spec's key or value is read
        where expr has no program"""
        s, x = fields_spec(spec, cr_is_data, preds), field_expr(expr)
        self.ctx.check(self.ctx.lib.dampr_text_fields_expr(self.ctx.h, self.h, tb.h, int(lo), int(hi), C.byref(s),
                                                           C.byref(x)))

    def fields_expr_records(self, tb, lo, hi, spec, expr, kv, cr_is_data=False, preds=()):
        """fields_records() with a computed key and / or value, expr as fields_expr()"""
        s, x = fields_spec(spec, cr_is_data, preds), field_expr(expr)
        self.ctx.check(self.ctx.lib.dampr_text_fields_expr_records(self.ctx.h, self.h, tb.h, int(lo), int(hi),
                                                                   C.byref(s), C.byref(x), kv.h))

    def fetch_field_keys(self, tb, sep, keys):
        """(columns, counts, codes) of a tuple-key table, decoded on the device from each entry's representative line:
        one column per component of keys (as fields_tuple()), an 'S<width>' array for str components and an int64
        array for int() ones, all in one row order with the accumulators and key codes (uint64)"""
        k = field_keys(keys)
        widths, n = (C.c_uint32 * FIELD_KEYS_MAX)(), C.c_uint64(0)
        self.ctx.check(self.ctx.lib.dampr_table_fetch_field_keys(self.ctx.h, self.h, tb.h, int(sep), C.byref(k), widths,
                                                                 None, None, None, 0, C.byref(n)))
        m = n.value
        cols = [np.empty(m, dtype=np.int64) if kind == FIELD_KEY_INT else np.empty((m, max(1, widths[j])), np.uint8)
                for j, (_i, kind) in enumerate(keys)]
        counts, codes = np.empty(m, dtype=np.uint64), np.empty(m, dtype=np.uint64)
        if m:
            ptrs = (C.c_void_p * FIELD_KEYS_MAX)(*[_ptr(c) for c in cols])
            for j, c in enumerate(cols):
                widths[j] = c.shape[1] if c.ndim == 2 else 0
            self.ctx.check(self.ctx.lib.dampr_table_fetch_field_keys(self.ctx.h, self.h, tb.h, int(sep), C.byref(k),
                                                                     widths, ptrs, _ptr(counts), _ptr(codes), m,
                                                                     C.byref(n)))
        cols = [c.view("S%d" % c.shape[1]).ravel() if c.ndim == 2 else c for c in cols]
        return cols, counts, codes

    def fields_stats(self):
        """stats() of a field scan under the names of its counters. "records" is the record count in record mode;
        in table mode it counts the lines WHERE predicates dropped (record mode: records - lines - fallback)."""
        st = self.stats()
        return {"entries": st["entries"], "lines": st["lines"], "max_abs": st["empty"], "folded": st["folded"],
                "flags": st["flags"], "hashed": st["hashed"], "fallback": st["fallback"], "records": st["raw"]}

    def fields_fetch(self, op):
        """(codes, values int64) of a field scan: the accumulators decoded from their MIN / MAX codes"""
        codes, acc, _reps = self.fetch()
        return codes, decode_fold(acc, op)

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
        self.fetches += 1
        n = C.c_uint64(0)
        # one call into one page-locked block of the result arena: the arrays returned are views of it and keep it
        # leased for as long as any of them lives. Without a block (see dampr_result_lease): pageable arrays, below.
        p, lease = C.c_void_p(), C.c_uint64(0)
        _apply_result_cache()
        self.ctx.check(self.ctx.lib.dampr_table_fetch_words_leased(
            self.ctx.h, self.h, tb.h if tb is not None else None, int(mode), int(width), 1 if with_codes else 0,
            C.byref(p), C.byref(lease), C.byref(n)))
        if lease.value:
            m = n.value
            blk = ResultLease(self.ctx, lease.value, p.value, m * (width + (24 if with_codes else 8)))
            words = blk.array(0, m, "S%d" % width)
            counts = blk.array(m * width, m, np.uint64)
            if not with_codes:
                return words, counts, None, None
            return words, counts, blk.array(m * (width + 8), m, np.uint64), blk.array(m * (width + 16), m, np.uint64)
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
        _apply_result_cache()
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


def host_sink_timings():
    """Host-clock split of the last native sink call, milliseconds: the calling thread's dictionary preparation, then
    the largest value over the writer threads of the start delay, open(), row formatting, write() and close()."""
    out = (C.c_double * 6)()
    load_library().dampr_host_sink_timings(out)
    return dict(zip(("prep", "start", "open", "format", "write", "close"), out))


def host_pool_threads():
    """threads the library's host worker pool has started so far in this process"""
    n = C.c_uint64(0)
    load_library().dampr_host_pool_threads(C.byref(n))
    return n.value


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


def host_eval_f64(vals, prog, ci, cf):
    """float64 result of a lowered numeric expression (lowering.numeric_program) at every value of an int64 array,
    computed natively with CPython's rounding; None where CPython would raise or leave the IEEE path."""
    lib = load_library()
    vals = np.ascontiguousarray(vals, dtype=np.int64)
    p = np.ascontiguousarray(prog, dtype=np.int32)
    ci = np.ascontiguousarray(list(ci) or [0], dtype=np.int64)
    cf = np.ascontiguousarray(list(cf) or [0.0], dtype=np.float64)
    out = np.empty(len(vals), dtype=np.float64)
    rc = lib.dampr_host_eval_f64(_ptr(vals), len(vals), _ptr(p), len(p), _ptr(ci), _ptr(cf), _ptr(out))
    if rc == -5:   # DAMPR_ERR_UNSUPPORTED
        return None
    if rc:
        raise DeviceError("dampr_host_eval_f64: malformed program (%d)" % rc)
    return out


def kv_merge_ranges(ctx, kv, offsets, xform, op=-1):
    return ctx.kv_merge_ranges(kv, offsets, xform, op)


def kv_merge(ctx, runs, xform, op=-1):
    return ctx.kv_merge(runs, xform, op)

/*
 * dampr_b200.h — C-ABI of libdampr_b200.so: the H100-native (sm_90a) replacement for the
 * hot path of Refefer/Dampr: map -> partition-by-key -> spill -> external merge sort ->
 * combiner/reduce.
 *
 * The reference has NO native interface (it is pure Python); the boundary it exposes is the
 * Python DSL plus the runner slot `Dampr(graph, runner=MTRunner)` (reference dampr/dampr.py:835-843,
 * call site dampr/dampr.py:73).  This header is what a ctypes stub on the reference side binds
 * (see INTEGRATION.md).  Each entry point names the reference function(s) it replaces.
 *
 * Conventions
 *   - plain C, extern "C"; every function returns int32 status, 0 = ok, <0 = error
 *     (message: dampr_last_error(ctx), owned by the ctx, valid until the next call on it);
 *   - handles are opaque; the library owns device memory, the caller owns host memory;
 *   - variable-size outputs use a two-phase "count, then fetch into caller memory" protocol;
 *   - one host thread drives one ctx; a ctx owns one compute stream and one copy stream on
 *     one GPU; calls enqueue and return, dampr_ctx_sync / *_fetch / *_stats block;
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef DAMPR_B200_H
#define DAMPR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dampr_ctx dampr_ctx;         /* one GPU, streams, scratch arena            */
typedef struct dampr_textbuf dampr_textbuf; /* device-resident byte range of a text file  */
typedef struct dampr_table dampr_table;     /* map-side combiner table (key code -> acc)  */
typedef struct dampr_kv dampr_kv;           /* device array of 16-byte (u64 key, u64 val) */

/* ---- status codes ------------------------------------------------------------------- */
#define DAMPR_OK 0
#define DAMPR_ERR_CUDA (-1)     /* CUDA runtime error, see dampr_last_error            */
#define DAMPR_ERR_ARG (-2)      /* bad argument                                         */
#define DAMPR_ERR_NOMEM (-3)    /* device or pinned allocation failed                   */
#define DAMPR_ERR_OVERFLOW (-4) /* table full / 64-bit accumulator overflow (B12)       */
#define DAMPR_ERR_UNSUPPORTED (-5)

/* ---- library ------------------------------------------------------------------------- */
int32_t dampr_abi_version(void);
int32_t dampr_device_count(int32_t *out_n);
/* process-wide tuning switches; any other name, or a value out of range, returns DAMPR_ERR_ARG:
 *   "text_ctas"      2..4, default 4: resident CTAs per SM of the warp-autonomous tokenise kernel
 *   "text_kernel"    1 | 2, default 2: 2 = warp-autonomous tokenise kernel; 1 = first-generation kernel, also
 *                    the fallback for lines longer than 2 KB
 *   "host_threads"   1..256, default 16: upper bound on the copy threads of a staged host transfer
 *   "file_cufile"    0 | 1, default 0: 1 = file ingest through cuFile (GPUDirect Storage) instead of the
 *                    page-locked ring
 *   "cufile_threads" 1..64, default 8: reader threads of the cuFile ingest */
int32_t dampr_set_option(const char *name, int64_t value);

/* ---- context: replaces the process pool of StageRunner.run (stagerunner.py:15-43) ---- */
int32_t dampr_ctx_create(int32_t device, dampr_ctx **out);
int32_t dampr_ctx_destroy(dampr_ctx *ctx);
int32_t dampr_ctx_sync(dampr_ctx *ctx);
/* wait for the copy stream only (host staging buffers may be reused afterwards) */
int32_t dampr_ctx_sync_copy(dampr_ctx *ctx);
const char *dampr_last_error(dampr_ctx *ctx);
/* CUDA-event timings of the kernels launched since the last reset:
 * out[2*i] = kernel id (DAMPR_K_*), out[2*i+1] = milliseconds (as double bit pattern).
 * Returns the number of entries through *n (at most cap). Blocks until they completed. */
int32_t dampr_ctx_timings(dampr_ctx *ctx, double *out_ms, int32_t *out_ids, int32_t cap, int32_t *n);
int32_t dampr_ctx_timings_reset(dampr_ctx *ctx);
int32_t dampr_ctx_timing_enable(dampr_ctx *ctx, int32_t on);
/* Page-locked result memory. Every context keeps an arena of cudaHostAlloc blocks that results are downloaded
 * into. A lease is a block of at least `bytes` that stays the caller's until it is released, whatever else the
 * context is used for meanwhile; released blocks are reused and only returned to the system while the arena holds
 * more than dampr_set_option("host_result_cache_bytes") (default 64 MB). *lease == 0 and *host_ptr == NULL: no
 * block (bytes == 0, more than that option, or out of page-locked memory). */
int32_t dampr_result_lease(dampr_ctx *ctx, uint64_t bytes, void **host_ptr, uint64_t *lease);
int32_t dampr_result_release(dampr_ctx *ctx, uint64_t lease);
/* free / total device memory: the arena the spill trigger compares against (replaces the RSS
 * polling of InterpolativeMemoryChecker, memory.py:72-113) */
int32_t dampr_ctx_mem_info(dampr_ctx *ctx, uint64_t *free_bytes, uint64_t *total_bytes);
/* multiprocessor count of the context's device (grid sizing, roofline bookkeeping) */
int32_t dampr_ctx_num_sms(dampr_ctx *ctx, int32_t *out);
/* number of kernels this library launched on the ctx since creation */
int32_t dampr_ctx_launches(dampr_ctx *ctx, uint64_t *out);
/* raw handle of the compute stream (cudaStream_t) so torch.distributed collectives can be
 * ordered against it */
int32_t dampr_ctx_stream(dampr_ctx *ctx, uint64_t *out_stream);

#define DAMPR_K_TEXT_COUNT 1
#define DAMPR_K_TABLE_EXTRACT 2
#define DAMPR_K_TEXT_VERIFY 3
#define DAMPR_K_PART_HIST 4
#define DAMPR_K_PART_SCATTER 5
#define DAMPR_K_LEAF_SORT 6
#define DAMPR_K_SEG_REDUCE 7
#define DAMPR_K_MERGE 8
#define DAMPR_K_JOIN 9
#define DAMPR_K_PROBE 10
#define DAMPR_K_SYNTH 11
#define DAMPR_K_MISC 12
#define DAMPR_K_TEXT_FIELDS 13
#define DAMPR_K_TEXT_FIELDS_COUNT 14   /* dampr_text_fields_records' line-count pass and tile scan */

/* ---- pinned host memory (spill ring / ingest staging) -------------------------------- */
int32_t dampr_host_alloc(uint64_t nbytes, void **out);
int32_t dampr_host_free(void *p);
/* page-lock / release memory the caller allocated (the host buffer of spilled runs: MaxMemoryWriter's run files,
 * dataset.py:190-262, live in host memory here); copies from / to registered memory skip the staging ring */
int32_t dampr_host_register(void *p, uint64_t nbytes);
int32_t dampr_host_unregister(void *p);

/* ---- text ingest: replaces TextInput.chunks (inputs.py:48-56) + TextLineDataset.read
 *      (dataset.py:458-476): byte ranges of a file with the line-ownership rule ---------- */
/* capacity = number of text bytes the buffer can hold (the library adds lead-in and padding) */
int32_t dampr_textbuf_create(dampr_ctx *ctx, uint64_t capacity, dampr_textbuf **out);
int32_t dampr_textbuf_destroy(dampr_ctx *ctx, dampr_textbuf *tb);
/* declare the total length of the text that will be uploaded (pads the tail with '\n') */
int32_t dampr_textbuf_set_length(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t n);
/* async host->device copy of text bytes [off, off+len) on the copy stream */
int32_t dampr_textbuf_upload(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t off, const void *host,
                             uint64_t len);
/* the same from a FILE: bytes [file_off, file_off+len) of `path` -> text[off, off+len). The library's copy
 * threads pread() the page cache straight into its page-locked ring while the previous slot is in flight to
 * the device (replaces the open(...).readline loop of TextLineDataset.read, dataset.py:458-476, as the
 * ingest of the scan). */
int32_t dampr_textbuf_upload_file(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t off, const char *path,
                                  uint64_t file_off, uint64_t len);
/* blocking device->host copy of text bytes [off, off+len) */
int32_t dampr_textbuf_download(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t off, void *host,
                               uint64_t len);
/* device pointer of text byte 0 (for tests / zero-copy producers such as the synthetic generator) */
int32_t dampr_textbuf_devptr(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t *out_ptr);

/* ---- map-side combiner over text: replaces Map.stream of the tokenising lambdas
 *      (base.py:30-33; examples/wc.py:12; benchmarks/tf-idf-dampr.py:12-14) fused with
 *      ReducedWriter.add_record (dataset.py:100-105) --------------------------------------- */
#define DAMPR_TOK_WS 0                /* str.split(): maximal runs of non-whitespace         */
#define DAMPR_TOK_NONWORD_LOWER_SET 1 /* set(re.split(r'[^\w]+', line.lower())): per-line set */
#define DAMPR_TOK_NONWORD_LOWER 2     /* re.split(r'[^\w]+', line.lower()) without set():
                                         every token counts, '' tokens as re.split yields    */

/* OR-ed into `mode`: '\r' is an ordinary byte, as in the reference's binary-mode .gz reader
 * (GzipLineDataset, dataset.py:488-493). Without it '\r' ends lines (text mode, universal newlines). */
#define DAMPR_TOK_FLAG_CR_DATA 0x100

int32_t dampr_table_create(dampr_ctx *ctx, uint32_t capacity_log2, dampr_table **out);
int32_t dampr_table_destroy(dampr_ctx *ctx, dampr_table *t);
int32_t dampr_table_clear(dampr_ctx *ctx, dampr_table *t);

/* tokenise the lines whose first byte lies in [own_lo, own_hi) and fold (token -> +1) into the
 * table. Requires bytes [0, min(n, own_hi + halo)) to be uploaded. */
int32_t dampr_text_count(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                         uint64_t own_hi, int32_t mode);
/* second pass over the same range that byte-compares every hashed (long) token with the
 * representative of its table entry; sets DAMPR_TF_COLLISION if two different tokens share a code */
int32_t dampr_text_verify(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                          uint64_t own_hi, int32_t mode);

/* stats[0]=entries stats[1]=lines stats[2]=count of the '' token stats[3]=tokens folded
 * stats[4]=flags (DAMPR_TF_*) stats[5]=hashed(long) tokens stats[6]=raw tokens seen
 * stats[7]=lines handed back to the host (per-line fallback, see dampr_table_fallback_lines) */
#define DAMPR_TF_NONASCII 1u
#define DAMPR_TF_CR 2u
#define DAMPR_TF_LONGLINE 4u
#define DAMPR_TF_TABLEFULL 8u
#define DAMPR_TF_LONGTOKEN 16u
#define DAMPR_TF_COLLISION 32u
#define DAMPR_TF_RECFULL 64u   /* dampr_text_fields_records: more lines than the record buffer holds            */
#define DAMPR_TF_NEGZERO 128u  /* a float() field scan parsed a negative zero                                    */
#define DAMPR_TF_JSON_KEY_KIND 256u  /* a JSON scan read a key member of another JSON type than key_kind names       */
#define DAMPR_TF_JSON_VAL_KIND 512u  /* a JSON scan read a value member of another kind than its fold (see below)     */
int32_t dampr_table_stats(dampr_ctx *ctx, dampr_table *t, uint64_t stats[8]);
/* Per-line fallback of the [^\w]+ tokenisers: a line that holds a byte the device cannot tokenise the way
 * Python does (non-ASCII: Unicode \w / lower(); '\r' in text mode: universal newlines) contributes NOTHING to
 * the table, the line count or the '' token count; instead lines[i] = (byte offset of the line << 16) | length
 * (without its '\n') is reported here and the caller tokenises just those lines (TextLineDataset.read,
 * dataset.py:458-476 + the user's lambda) and adds the results. Order unspecified. Two-phase: lines == NULL
 * returns *n only. More than 65536 such lines, or one that cannot be isolated inside the kernel's window, set
 * DAMPR_TF_NONASCII instead (the whole scan is then the caller's). str.split mode keeps scan-wide flags. */
int32_t dampr_table_fallback_lines(dampr_ctx *ctx, dampr_table *t, uint64_t *lines, uint64_t cap, uint64_t *n);
/* ---- delimited-field fold over text: replaces Map.stream of `l.split(S)[i]` keys with `1` / `int()` / `float()` of `l.split(S)[j]`
 *      values (base.py:30-33) fused with ReducedWriter.add_record under +, min or max (dataset.py:100-105) -------- */
/* Below, line.split(sep) stands for the split that spec->sep selects: a separator byte, or str.split() under
 * DAMPR_FIELD_SEP_WS. */
#define DAMPR_FIELD_KEY_STR 0          /* key = line.split(sep)[key_field]                                   */
#define DAMPR_FIELD_KEY_INT 1          /* key = int(line.split(sep)[key_field])                              */
#define DAMPR_FIELD_VAL_ONE 0x7FFFFFFF /* val_field: the value is the constant 1                             */
/* sep: split like str.split() with no argument (line.split()): fields are the maximal runs of bytes other than ASCII
 * whitespace (0x09-0x0D, 0x1C-0x20; '\r' only under cr_is_data, otherwise the line is the caller's). Leading and
 * trailing whitespace make no field, no field is '', and a blank or all-whitespace line has 0 fields (every index is
 * missing). Field indices, negative ones and DAMPR_PRED_NFIELDS count these fields. Non-ASCII whitespace is never
 * seen: a line with a non-ASCII byte is the caller's, as under a separator byte. */
#define DAMPR_FIELD_SEP_WS 256
/* bytes past own_hi that must be uploaded before a dampr_text_fields call (a line longer than the kernel's window
 * is measured in global memory, up to 64 KB) */
#define DAMPR_FIELDS_HALO 65536
/* a WHERE predicate of a field scan: the stage's `filter(...)` calls in front of the fold, e.g. r[1] == 'GET',
 * int(r[2]) >= 500, float(r[3]) < 0.5, r[1] in ('GET', 'POST'), len(r) == 4 (r = line.split(sep)) */
#define DAMPR_PRED_STR 0      /* line.split(sep)[field], compared as bytes (UTF-8 byte order is code-point order)  */
#define DAMPR_PRED_INT 1      /* int(line.split(sep)[field]) against int64 constants                               */
#define DAMPR_PRED_F64 2      /* float(line.split(sep)[field]) against one double (IEEE: NaN is unequal to all)    */
#define DAMPR_PRED_NFIELDS 3  /* len(line.split(sep)) against one int64; `field` is unused                        */
#define DAMPR_PRED_MEMBER 4   /* JSON scans only: "m" in r (DAMPR_CMP_IN) / "m" not in r (DAMPR_CMP_NOT_IN), n = 0
                                 (a call over member paths: n = 0 or 1, see the JSON block)                       */
#define DAMPR_CMP_EQ 0
#define DAMPR_CMP_NE 1
#define DAMPR_CMP_LT 2
#define DAMPR_CMP_LE 3
#define DAMPR_CMP_GT 4
#define DAMPR_CMP_GE 5
#define DAMPR_CMP_IN 6        /* STR and INT only: equal to one of the n constants                                */
#define DAMPR_CMP_NOT_IN 7
/* string tests and boolean structure: `"ERROR" in l`, `r[6].startswith("/api/")`, `len(l) > 90`, `l.strip()`,
 * `r[1] == "GET" and (int(r[2]) >= 500 or not r[6].endswith(".js"))` */
#define DAMPR_PRED_LEN 5      /* len() of a STR field (or the line) against one int64 (EQ .. GE)                    */
#define DAMPR_PRED_NONBLANK 6 /* the STR field (or the line) holds a byte outside the str.split() whitespace class
                                 (`x.strip()` as a truth value); cmp EQ, n = 0                                      */
#define DAMPR_PRED_AND 7      /* connectives of a postfix program: pop b, pop a, push `a and b` / `a or b`; NOT    */
#define DAMPR_PRED_OR 8       /* pops a and pushes `not a`. field, cmp and n are unused (n = 0)                    */
#define DAMPR_PRED_NOT 9
#define DAMPR_CMP_CONTAINS 8      /* STR only: the one constant is a substring of the field (`S in X`)            */
#define DAMPR_CMP_NOT_CONTAINS 9  /* `S not in X`                                                                 */
#define DAMPR_CMP_STARTS 10       /* STR only: the field starts with one of the n constants (`X.startswith(S)`)   */
#define DAMPR_CMP_ENDS 11         /* `X.endswith(S)`                                                              */
/* `field` of a STR, LEN or NONBLANK predicate that reads the whole line (no '\n'), not one of its fields: separator
 * byte and DAMPR_FIELD_SEP_WS calls only */
#define DAMPR_FIELD_LINE (-0x7FFFFFFF - 1)
#define DAMPR_PRED_MAX_OPS 8          /* connectives per call                                                     */
#define DAMPR_PRED_MAX 8              /* predicates (leaves) per call                                             */
#define DAMPR_PRED_MAX_CONSTS 64      /* constants (set members included) over all predicates of a call           */
#define DAMPR_PRED_MAX_BYTES 1024     /* bytes of STR constants over all predicates of a call                     */
typedef struct dampr_field_pred {
    int32_t kind;           /* DAMPR_PRED_*                                                                       */
    int32_t field;          /* i of line.split(sep)[i]; negative counts from the end, as in Python                */
    int32_t cmp;            /* DAMPR_CMP_*                                                                        */
    int32_t n;              /* constants: 1 for EQ .. GE, 1 .. DAMPR_PRED_MAX_CONSTS members for IN / NOT_IN      */
    const int64_t *ints;    /* INT, NFIELDS: the n constants                                                      */
    double f64;             /* F64: the constant                                                                  */
    const uint8_t *bytes;   /* STR: the n constants back to back                                                  */
    const uint32_t *lens;   /* STR: their lengths in bytes                                                        */
} dampr_field_pred;
typedef struct dampr_fields_spec {
    int32_t sep;        /* separator byte: ASCII, not NUL, '\n' or '\r'; or DAMPR_FIELD_SEP_WS (line.split())  */
    int32_t key_field;  /* i of line.split(sep)[i]; negative counts from the end, as in Python              */
    int32_t key_kind;   /* DAMPR_FIELD_KEY_STR | DAMPR_FIELD_KEY_INT                                         */
    int32_t val_field;  /* j of int() / float() of line.split(sep)[j], negative from the end, or
                           DAMPR_FIELD_VAL_ONE (int ops of dampr_text_fields only)                            */
    int32_t op;         /* dampr_text_fields: DAMPR_OP_SUM_I64 | MIN_I64 | MAX_I64 (int() values) or
                           DAMPR_OP_MIN_F64 | MAX_F64 (float() values); dampr_text_fields_records:
                           DAMPR_OP_SUM_I64 (int() values) | DAMPR_OP_SUM_F64 (float() values)               */
    int32_t cr_is_data; /* 1: '\r' is an ordinary byte (binary-mode .gz); 0: it ends lines (text mode)        */
    const dampr_field_pred *preds; /* WHERE predicates, applied in order before the key and value are read       */
    int32_t npreds;     /* entries of preds: 0 .. DAMPR_PRED_MAX + DAMPR_PRED_MAX_OPS, at most DAMPR_PRED_MAX of
                           them leaves and DAMPR_PRED_MAX_OPS connectives; 0 (preds unused) is the plain scan        */
} dampr_fields_spec;
/* WHERE (npreds > 0): on each line the device can take (the byte and length rules below), the predicates are
 * evaluated in order as Python's filters would be. The first false one drops the line: no key or value is read,
 * nothing is inserted, record mode writes a hole {0, 0}, and the line goes nowhere else. A predicate the device
 * cannot decide (its field does not exist, an INT field that is not [+-]?[0-9]{1,18}, an F64 field outside the
 * float() rule below) hands the line to the caller as a fallback line, whose filters then decide or raise. Only a
 * line that passes every predicate has its key and value read, under the rules below. A -0.0 in a predicate's field
 * does not set DAMPR_TF_NEGZERO. Dropped lines are counted: dampr_text_fields puts their number in stats[6];
 * in record mode it is stats[6] - stats[1] - stats[7] (records - folded lines - fallback lines).
 * Programs: preds is a postfix program over leaves (every kind up to DAMPR_PRED_NONBLANK) and connectives. Each leaf
 * is T, F or U (undecided: the cases above, a missing field or member, a JSON member that is not a string without
 * escapes under CONTAINS .. ENDS, LEN or NONBLANK). Connectives combine left-sequentially, as Python's short circuit
 * does: `a and b` is F if a is F, U if a is U, else b; `a or b` is T if a is T, U if a is U, else b; `not a` keeps U.
 * The values left on the stack (one per filter call; a list without connectives leaves one per leaf, today's chain)
 * are combined the same way with `and`, bottom first. F drops the line, U hands it to the caller, T reads the key and
 * value. A program with a connective that finds fewer operands than it pops, more than DAMPR_PRED_MAX leaves or
 * DAMPR_PRED_MAX_OPS connectives, a new kind or comparison under another kind than the ones named above, or (in a
 * JSON call) DAMPR_FIELD_LINE returns DAMPR_ERR_ARG. */
/* fold (key code -> value) of the lines whose first byte lies in [own_lo, own_hi) into the table (cleared by the
 * caller before the first range; ranges of one scan accumulate). Needs bytes [0, min(n, own_hi + DAMPR_FIELDS_HALO))
 * uploaded. The device folds a line only when every byte is ASCII and not NUL, it holds no '\r' (unless
 * cr_is_data), every field it reads exists, every int() field is exactly [+-]?[0-9]{1,18}, every float() field is
 * one the device parses to Python's bits ([ \t]*[+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?[ \t]* with at most 19
 * significant digits, see csrc/fparse.cuh), and it ends within 4 KB of its start. Every other line goes onto the
 * fallback list (dampr_table_fallback_lines) for the caller to run its own functions on; more lines than the list
 * holds set DAMPR_TF_NONASCII, a line of 64 KB or more sets DAMPR_TF_LONGLINE (the whole scan is then the caller's).
 * Key codes: str keys of 1..9 bytes pack 7 bits per byte (dampr_table_fetch_words with DAMPR_TOK_WS decodes them);
 * '' and longer keys are hashed codes (bit 63) with a representative occurrence, byte-compared on every insert
 * (DAMPR_TF_COLLISION on a mismatch); int keys v are v ^ 2^63. No key code is 0.
 * Accumulators (the table's counts): SUM = the two's-complement sum; MAX = v ^ 2^63 of the maximum; MIN =
 * ~(v ^ 2^63) of the minimum (order-preserving codes whose identity is the cleared 0). MAX_F64 holds the code
 * c = bits ^ (sign ? ~0 : 2^63) of the largest double, MIN_F64 ~c of the smallest. A parsed -0.0 sets
 * DAMPR_TF_NEGZERO (Python's min / max of 0.0 and -0.0 depends on the order of the arguments).
 * dampr_table_stats after the scan: stats[0]=entries stats[1]=lines folded on the device stats[2]=max |value|
 * folded (int values) stats[3]=records folded (= stats[1]) stats[4]=flags stats[5]=hashed str keys
 * stats[7]=fallback lines. */
int32_t dampr_text_fields(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo, uint64_t own_hi,
                          const dampr_fields_spec *spec);
/* record mode of the same scan, for folds whose result depends on the order of the values (float sums) or that
 * need a count per key (mean()): one 16-byte record {key code, value} per line owned by [own_lo, own_hi) is written
 * to rec's buffer, value = the int64 of int() (DAMPR_OP_SUM_I64) or the bits of float() (DAMPR_OP_SUM_F64). Records
 * are in line order: the lines of one scan (the ranges since the table was cleared) take indices 0, 1, 2, ...
 * whatever the ranges and the grid schedule. A line the device does not take (the fallback list, the rules above)
 * is a hole record {0, 0}; key code 0 is never a real code. The table takes one insert per taken line and counts
 * lines per key (its counts), keeps the representatives of hashed keys and checks them, exactly as above.
 * stats[6] = records of the scan so far (taken lines + holes), the index the next range starts at. When the index
 * reaches rec's capacity the kernel writes nothing past it and sets DAMPR_TF_RECFULL (stats[6] still counts every
 * line: a buffer of that many records holds the scan). The caller sets rec's size (dampr_kv_set_size) from stats[6].
 * Three kernels per range: a line count per 16 KB tile, one CTA's scan of the counts, the fold. */
int32_t dampr_text_fields_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                  uint64_t own_hi, const dampr_fields_spec *spec, dampr_kv *rec);
/* ---- tuple keys: `(l.split(S)[i], int(l.split(S)[j]), ...)`, GROUP BY of 1 .. DAMPR_FIELD_KEYS_MAX fields ----------
 * The same folds, predicates, line rules and stats as dampr_text_fields / dampr_text_fields_records, with the key
 * made of the components of `keys` instead of spec->key_field / spec->key_kind (neither is read). spec->sep is a
 * separator byte or DAMPR_FIELD_SEP_WS (DAMPR_FIELD_SEP_JSON returns DAMPR_ERR_ARG, as does n outside 1 .. 4). A
 * line is taken only when every component exists and every INT component is [+-]?[0-9]{1,18}.
 * - Key code: the two running states of the field keys' seeded hash are fed, in order, the bytes of each STR
 *   component, the 8 little-endian bytes of v ^ 2^63 of each INT component v, and one 0xFF byte between two
 *   components (it never occurs in a taken line); the code is mix64(state ^ L * 0x9E3779B97F4A7C15) | 2^63 with L
 *   the number of bytes fed, as for a hashed field key. Component kinds are fixed per call, so the bytes fed name
 *   the tuple. No code is 0.
 * - Representative: the LINE, (offset << 20) | length, the lowest-offset taken line of each entry. Every later
 *   insert of another line re-splits the representative line (in global memory, same rules) and compares its
 *   components with its own: STR as bytes, INT as parsed values. A mismatch sets DAMPR_TF_COLLISION. stats[5]
 *   (hashed str keys) stays 0.
 * dampr_table_fetch_words does not decode these tables: dampr_table_fetch_field_keys does. */
#define DAMPR_FIELD_KEYS_MAX 4
typedef struct dampr_field_keys {
    int32_t n;                              /* components: 1 .. DAMPR_FIELD_KEYS_MAX                            */
    int32_t field[DAMPR_FIELD_KEYS_MAX];    /* i of line.split(sep)[i]; negative counts from the end            */
    int32_t kind[DAMPR_FIELD_KEYS_MAX];     /* DAMPR_FIELD_KEY_STR | DAMPR_FIELD_KEY_INT                        */
} dampr_field_keys;
int32_t dampr_text_fields_tuple(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo, uint64_t own_hi,
                                const dampr_fields_spec *spec, const dampr_field_keys *keys);
int32_t dampr_text_fields_tuple_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                        uint64_t own_hi, const dampr_fields_spec *spec, const dampr_field_keys *keys,
                                        dampr_kv *rec);
/* ---- computed keys and values: `int(r[2]) * int(r[3])`, `float(r[5]) / 1000`, `int(r[0]) // 3600`, `len(r)`,
 *      `len(r[1])`, constant keys (`lambda x: 1`) ------------------------------------------------------------------
 * The same folds, predicates, line rules and stats as dampr_text_fields / dampr_text_fields_records (sep a separator
 * byte or DAMPR_FIELD_SEP_WS), with the key and / or the value computed per line by a postfix program over the typed
 * stack of csrc/common.cuh's EvalOp opcodes (op | arg << 8; every opcode but EV_X and EV_LOG). Its leaves are int
 * and float constants (ci[arg], cf[arg]), the line's field count (EV_NF) and load slots (EV_LOAD arg): slot j is
 * int(), float() or len() of field load_field[j] of the line's split, the field rules of the scan above (a missing
 * field, or an int() / float() field the device does not parse, makes the line a fallback line). The key program
 * (key_type DAMPR_EXPR_INT) replaces spec->key_field / key_kind: the key is its int64 v, coded v ^ 2^63 as an int
 * key. The value program (val_type DAMPR_EXPR_INT or DAMPR_EXPR_F64, the type op folds) replaces spec->val_field.
 * DAMPR_EXPR_NONE keeps the spec's key or value.
 * - A line is taken only when every operation reaches CPython's result: a zero divisor of / // % (int or float),
 *   INT64_MIN // -1, an int + - * unary - or abs() leaving int64, int / int with an operand beyond +-2^53, int() of a
 *   NaN, an infinity or a float outside int64, and a key equal to INT64_MIN make it a fallback line. Float operations
 *   are single IEEE roundings (no contraction), int -> float rounds half-even, // and % floor towards -inf.
 * - A computed float value that is -0.0 sets DAMPR_TF_NEGZERO, a NaN sets DAMPR_TF_NAN (both matter under min / max).
 * - With a key program each CTA folds its lines' values of up to 32 key codes in shared memory and inserts each code
 *   once (a constant key or a few buckets would otherwise send every line to one table slot).
 * Malformed programs return DAMPR_ERR_ARG: a stack underflow, a depth above DAMPR_EXPR_MAX_DEPTH, a final depth other
 * than 1, an unknown opcode, an operand of the wrong type, a constant or load slot out of range, a result type that
 * does not match op, more than DAMPR_EXPR_MAX_OPS operations, or no program at all. */
#define DAMPR_EXPR_MAX_OPS 32
#define DAMPR_EXPR_MAX_LOADS 4
#define DAMPR_EXPR_MAX_DEPTH 8
#define DAMPR_EXPR_MAX_CONSTS 16
#define DAMPR_EXPR_NONE 0
#define DAMPR_EXPR_INT 1
#define DAMPR_EXPR_F64 2
#define DAMPR_LOAD_INT 0    /* int(line.split(sep)[field]): [+-]?[0-9]{1,18}                                      */
#define DAMPR_LOAD_F64 1    /* float(line.split(sep)[field]): the float() rule above                               */
#define DAMPR_LOAD_LEN 2    /* len(line.split(sep)[field]), an int                                                 */
#define DAMPR_TF_NAN 1024u  /* an expression scan computed a NaN value                                             */
typedef struct dampr_field_expr {
    int32_t key_type;                          /* DAMPR_EXPR_NONE | DAMPR_EXPR_INT                                */
    int32_t key_len;                           /* operations of the key program                                  */
    int32_t key_prog[DAMPR_EXPR_MAX_OPS];
    int32_t val_type;                          /* DAMPR_EXPR_NONE | DAMPR_EXPR_INT | DAMPR_EXPR_F64              */
    int32_t val_len;
    int32_t val_prog[DAMPR_EXPR_MAX_OPS];
    int64_t ci[DAMPR_EXPR_MAX_CONSTS];         /* int constants, shared by both programs                         */
    double cf[DAMPR_EXPR_MAX_CONSTS];          /* float constants                                                */
    int32_t nloads;                            /* 0 .. DAMPR_EXPR_MAX_LOADS                                      */
    int32_t load_field[DAMPR_EXPR_MAX_LOADS];  /* i of line.split(sep)[i]; negative counts from the end          */
    int32_t load_kind[DAMPR_EXPR_MAX_LOADS];   /* DAMPR_LOAD_*                                                   */
} dampr_field_expr;
int32_t dampr_text_fields_expr(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo, uint64_t own_hi,
                               const dampr_fields_spec *spec, const dampr_field_expr *expr);
int32_t dampr_text_fields_expr_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                       uint64_t own_hi, const dampr_fields_spec *spec, const dampr_field_expr *expr,
                                       dampr_kv *rec);
/* decode a tuple-key table ON THE DEVICE: each entry's representative line is split again (sep and keys as in the
 * scan) into one column per component. Two phases: cols == NULL sets *n (entries) and widths[j] (the longest STR
 * component j, 0 for INT components) only. Then cols[j] = uint8[*n * widths[j]] (STR: NUL-padded, widths[j] >= 1,
 * a longer component is cut at widths[j]) or int64[*n] (INT), counts[i] the accumulator and codes[i] the key code
 * of row i (either may be NULL). Rows are in one unspecified order shared by every column. */
int32_t dampr_table_fetch_field_keys(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t sep,
                                     const dampr_field_keys *keys, uint32_t widths[DAMPR_FIELD_KEYS_MAX],
                                     void *const cols[DAMPR_FIELD_KEYS_MAX], uint64_t *counts, uint64_t *codes,
                                     uint64_t cap, uint64_t *n);
/* ---- JSON-lines fold: `Dampr.json(path)` (map(json.loads)) with r["k"] keys and r["v"] / int(r["v"]) /
 *      float(r["v"]) values, and filters on r["m"] -------------------------------------------------------------------
 * The same folds as dampr_text_fields / dampr_text_fields_records with spec->sep = DAMPR_FIELD_SEP_JSON (the field
 * calls reject it, these calls take nothing else). key_field, val_field and every predicate's `field` index the
 * member list; no index is negative, and DAMPR_PRED_NFIELDS is not taken. Each line is json.loads'd:
 * - The device takes a line only when the whole line is one JSON text whose top-level value is an object (json.loads'
 *   grammar: escapes \" \\ \/ \b \f \n \r \t \uXXXX, no raw byte below 0x20 in a string, numbers
 *   -?(0|[1-9]\d*)(\.\d+)?([eE][+-]?\d+)?, the literals true / false / null, only JSON whitespace around tokens),
 *   nested at most DAMPR_JSON_MAX_DEPTH deep, every byte ASCII (no '\r' unless cr_is_data, where it is whitespace),
 *   no top-level member name holds a backslash, every member it reads exists, and it ends within 4 KB of its start.
 *   NaN, Infinity and -Infinity are not taken. Every other line is a fallback line, as above.
 * - Only top-level members count; a name that occurs twice takes its last occurrence (as dict does).
 * - key_kind STR: the member is a string without escapes, coded like a field key from the bytes between its quotes
 *   (the representative points at them). INT: a JSON integer of at most 18 digits, coded v ^ 2^63.
 * - Values: the int ops take a JSON integer of at most 18 digits; the float ops (and DAMPR_OP_SUM_F64 records) take
 *   any JSON number through the float() rule above.
 * - A key member of another JSON type than key_kind's (a number, literal, object or array under STR; a string,
 *   float-syntax number, literal, object or array under INT) sets DAMPR_TF_JSON_KEY_KIND; a value member that is not
 *   a JSON integer under the int ops, or not a float-syntax number (a '.' or an exponent) under the float ops, sets
 *   DAMPR_TF_JSON_VAL_KIND. Both only on lines the predicates keep, whatever else the line holds; the line is then a
 *   fallback line unless the scan takes that member anyway (any number under the float ops). A caller whose r["k"]
 *   or r["v"] is read bare learns from them that its column would hold another Python type.
 * - Predicates: STR takes a string member without escapes, INT a JSON integer of at most 18 digits, F64 any JSON
 *   number; a member of another type, or a missing one, makes the predicate undecided (a fallback line).
 *   DAMPR_PRED_MEMBER never is at the top level.
 * - Paths: a member may be a path r[n1][n2]..[nk] of 2 .. DAMPR_JSON_MAX_PATH names, its bytes the names joined by
 *   DAMPR_JSON_PATH_SEP (each name 1 .. DAMPR_JSON_MAX_NAME bytes). The names of all paths form at most
 *   DAMPR_JSON_MAX_NODES distinct (parent, name) nodes, and no two members name the same path; an empty name in a
 *   path, a longer path, more nodes or a repeated path return DAMPR_ERR_ARG. A call without a path runs exactly as
 *   above. In a call with one:
 *   - Every prefix r[n1]..[ni] (i < k) must be a present object for the member to be read. A missing or non-object
 *     prefix (Python's KeyError / TypeError) makes a key or value read a fallback line, and any predicate on the
 *     member undecided. "m" in r[n1]..[ni] is the member r[n1]..[ni][m] under DAMPR_PRED_MEMBER, decided when
 *     r[n1]..[ni] is an object. Such a predicate may carry one STR constant (n = 1, the bytes of m): where
 *     r[n1]..[ni] is itself a member of the call and a string without escapes, the predicate is the substring test
 *     of m in it, as Python's `in` on a str. Under any other parent it is undecided.
 *   - The last occurrence of a name wins at every level: a later duplicate of an interior name replaces its whole
 *     subtree (`{"a":{"b":1},"a":{"c":2}}` has no r["a"]["b"]; `{"a":{"b":1},"a":5}` makes it a TypeError).
 *   - Names are compared in the top-level object and in the objects of interior path names; a name with a backslash
 *     in one of them makes the line a fallback line. Names elsewhere are skipped, escaped or not.
 *   - The kinds, flags, number rules and limits above apply to a path's leaf as to a top-level member. */
#define DAMPR_FIELD_SEP_JSON 257
#define DAMPR_JSON_MAX_MEMBERS 8   /* members per call                                                                */
#define DAMPR_JSON_MAX_NAME 64     /* bytes per member name: ASCII, no '"', '\\' or byte below 0x20                   */
#define DAMPR_JSON_MAX_DEPTH 64    /* the top-level object is depth 1; a line nested deeper is a fallback line        */
#define DAMPR_JSON_PATH_SEP 0x1F   /* joins the names of a path member                                               */
#define DAMPR_JSON_MAX_PATH 4      /* names per path                                                                  */
#define DAMPR_JSON_MAX_NODES 16    /* distinct (parent, name) nodes over a call's paths                              */
typedef struct dampr_json_members {
    int32_t n;               /* 1 .. DAMPR_JSON_MAX_MEMBERS                                                       */
    const char *bytes;       /* the names (paths) back to back                                                     */
    const int32_t *len;      /* their lengths in bytes                                                             */
} dampr_json_members;
int32_t dampr_text_json_fields(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo, uint64_t own_hi,
                               const dampr_fields_spec *spec, const dampr_json_members *members);
int32_t dampr_text_json_fields_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                       uint64_t own_hi, const dampr_fields_spec *spec,
                                       const dampr_json_members *members, dampr_kv *rec);
/* compact the table into caller memory: codes[i], counts[i], reps[i] (rep = offset<<20 | len of the
 * lowest-offset occurrence, hashed tokens only, else 0). cap = array capacity; *n = entries written.
 * Pass all three arrays NULL to query *n only. Order is unspecified (dampr_table_to_kv +
 * dampr_kv_sort give a sorted run). Replaces ReducedWriter.flush (dataset.py:107-117). */
int32_t dampr_table_fetch(dampr_ctx *ctx, dampr_table *t, uint64_t *codes, uint64_t *counts,
                          uint64_t *reps, uint64_t cap, uint64_t *n);
/* key materialisation (K9): like dampr_table_fetch, plus every key decoded ON THE DEVICE into a
 * fixed-width NUL-padded ASCII string words[i*width .. +width) (hashed tokens are read back from
 * their representative occurrence in `tb`, truncated to `width`; their true length is in reps).
 * width: multiple of 8 in [16, 256]. words == NULL queries *n only; codes / reps may be NULL when the
 * caller does not need them (no hashed tokens in the table). */
int32_t dampr_table_fetch_words(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t mode,
                                uint32_t width, uint8_t *words, uint64_t *counts, uint64_t *codes,
                                uint64_t *reps, uint64_t cap, uint64_t *n);
/* dampr_table_fetch_words in one call, into a page-locked block leased from the context's result arena:
 * *host_ptr = words[*n * width] | counts[*n] and, with_codes != 0, | codes[*n] | reps[*n]. The block is the caller's
 * until dampr_result_release(ctx, *lease). *lease == 0 with *n > 0: the arena gave no block (the result is larger
 * than the "host_result_cache_bytes" option, or page-locked memory ran out) and nothing was fetched. */
int32_t dampr_table_fetch_words_leased(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t mode,
                                       uint32_t width, int32_t with_codes, void **host_ptr, uint64_t *lease,
                                       uint64_t *n);
/* device pointer and length of the count column the last dampr_table_fetch_words downloaded, in the same row
 * order; it stays valid until the table is cleared, fetched again or destroyed (*n = 0 after a clear) */
int32_t dampr_table_extracted_counts(dampr_ctx *ctx, dampr_table *t, uint64_t *dev_ptr, uint64_t *n);
/* dictionary encoding of a non-negative count column ON THE DEVICE: row i < n holds counts[i * stride] (a device
 * array; stride 2 reads the values of a kv's records at devptr + 8), rows n .. n + n_extra - 1 hold the host values
 * extra[]. Writes the sorted distinct values uniq[0 .. *n_uniq), inv[i] (their index, per row) and rows[j] (the
 * smallest row holding uniq[j]); every output array holds n + n_extra entries. Values below a bound are ranked
 * through a presence table, the few above it are folded by dampr_kv_sort_reduce. A negative value returns
 * DAMPR_ERR_UNSUPPORTED. n + n_extra < 2^32. */
int32_t dampr_count_dictionary(dampr_ctx *ctx, const uint64_t *counts, uint64_t n, uint32_t stride,
                               const int64_t *extra, uint32_t n_extra, int64_t *uniq, uint32_t *inv,
                               uint32_t *rows, uint64_t *n_uniq);
/* the same into a leased block: *host_ptr = uniq[*n_uniq] (int64) | inv[n + n_extra] (uint32) | rows[*n_uniq]
 * (uint32). *lease == 0 with *n_uniq > 0: the arena gave no block and nothing was downloaded. */
int32_t dampr_count_dictionary_leased(dampr_ctx *ctx, const uint64_t *counts, uint64_t n, uint32_t stride,
                                      const int64_t *extra, uint32_t n_extra, void **host_ptr, uint64_t *lease,
                                      uint64_t *n_uniq);
/* the same decoding for a kv whose keys are token codes (an exchanged / merged run): exact codes ->
 * words_host[i*width ..], hashed codes -> all-NUL (the caller patches them from their strings) */
int32_t dampr_kv_decode_words(dampr_ctx *ctx, dampr_kv *kv, int32_t mode, uint32_t width,
                              uint8_t *words_host);
/* host-side sink formatting (SinkWriter, dataset.py:264-282): joins ncols columns with '\t', rows end
 * with '\n'. kinds[c] == 0: ptrs[c] = u8[n][widths[c]] NUL-padded strings; kinds[c] == 1: ptrs[c] =
 * u32 inv[n] into a dictionary of strings aux[c] (bytes) / aux2[c] (u32 offsets[m+1]); kinds[c] == 2:
 * the same with a dictionary of int64 values aux[c][widths[c]], written in decimal.
 * out == NULL computes *out_len only. Pure host code, no device work. */
/* Python's repr(float) of n doubles into 24-byte slots (lens[i] bytes used): what print(value) writes for a float
 * (SinkWriter.add_record dataset.py:264-282; sink_tsv dampr.py:521-529). The join / sink entry points below take
 * float dictionaries directly (kind 3: ptrs = u32 inv[n], aux = double values[m], widths = m). */
int32_t dampr_host_format_f64(const double *vals, uint64_t n, uint8_t *slots, uint8_t *lens);
int32_t dampr_host_join_tsv(uint64_t n, int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                            const uint32_t *widths, const void *const *aux, const void *const *aux2,
                            uint8_t *out, uint64_t cap, uint64_t *out_len);
/* the same rows written straight to part files `<prefix><first_index + j>`, j < *n_files <= max_files:
 * large outputs are split by row range, every file is formatted and written by its own thread (buffered
 * writes to one file serialise on its inode lock). Replaces SinkStageRunner.sink (stagerunner.py:165-189)
 * + SinkWriter's print-per-record loop (dataset.py:264-282). */
int32_t dampr_host_sink_tsv(const char *prefix, uint32_t first_index, uint32_t max_files, uint64_t n,
                            int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                            const uint32_t *widths, const void *const *aux, const void *const *aux2,
                            uint64_t *out_len, uint32_t *n_files);
/* host-clock split of the last dampr_host_sink_tsv / dampr_host_sink_fmt call in this process, milliseconds:
 * out_ms[0] dictionary preparation on the calling thread, then the largest value over the writer threads of
 * [1] the delay before the thread started, [2] open(), [3] row formatting, [4] write(), [5] close() */
int32_t dampr_host_sink_timings(double *out_ms);
/* threads the library's host worker pool has started so far in this process (the sink, dampr_host_join_tsv and
 * dampr_host_unique_small share one pool of at most 16, parked between calls and joined at exit) */
int32_t dampr_host_pool_threads(uint64_t *started);
/* the same part files with col_pre[c] (NUL-terminated, may be empty) written in front of column c and row_end in
 * place of the newline, no separators of its own: the lines of sink_json (json.dumps(value) per record,
 * dampr.py:531-539) are col_pre = `["`, `", `, `, ` ... and row_end = `]\n` */
int32_t dampr_host_sink_fmt(const char *prefix, uint32_t first_index, uint32_t max_files, uint64_t n,
                            int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                            const uint32_t *widths, const void *const *aux, const void *const *aux2,
                            const char *const *col_pre, const char *row_end, uint64_t *out_len,
                            uint32_t *n_files);
/* dictionary encoding of an int64 column (host helper of the frame layer): values in [0, table) are
 * ranked through a presence table -> uniq[0..*n_uniq) ascending and inv[i]; other values are handed
 * back in big_vals / big_rows (at most big_cap, else the call fails) and their inv[] is untouched.
 * first_row (optional) receives the first row holding each distinct value. n < 2^32. */
int32_t dampr_host_unique_small(const int64_t *col, uint64_t n, uint64_t table, int64_t *uniq,
                                uint64_t *n_uniq, uint32_t *inv, uint32_t *first_row, int64_t *big_vals,
                                uint64_t *big_rows, uint64_t big_cap, uint64_t *n_big);
/* out[r] = a lowered numeric expression of vals[r] (host): prog is postfix, one int32 per operation, the opcode in
 * the low byte and the constant's index above it — 0 push vals[r], 1 push ci[idx], 2 push cf[idx], 3 float() of an
 * int, 4/5/6 int + - *, 7/8/9/10 float + - * /, 11 int / int (true division), 12 math.log, 13 int negation,
 * 14 float negation. CPython's results to the bit; DAMPR_ERR_UNSUPPORTED where CPython would raise or leave the
 * IEEE path (zero divisor, log of a value that is not finite and positive, int64 overflow, int / int beyond 2^53),
 * DAMPR_ERR_ARG for a malformed program. */
int32_t dampr_host_eval_f64(const int64_t *vals, uint64_t n, const int32_t *prog, uint32_t prog_len,
                            const int64_t *ci, const double *cf, double *out);
/* same, but leaves the run on the device as a kv (key = code, val = count) */
int32_t dampr_table_to_kv(dampr_ctx *ctx, dampr_table *t, dampr_kv **out);

/* ---- kv records: 16-byte (u64 key, u64 value) pairs --------------------------------- */
int32_t dampr_kv_create(dampr_ctx *ctx, uint64_t capacity, dampr_kv **out);
int32_t dampr_kv_destroy(dampr_ctx *ctx, dampr_kv *kv);
int32_t dampr_kv_size(dampr_ctx *ctx, dampr_kv *kv, uint64_t *n);
int32_t dampr_kv_set_size(dampr_ctx *ctx, dampr_kv *kv, uint64_t n);
int32_t dampr_kv_devptr(dampr_ctx *ctx, dampr_kv *kv, uint64_t *out_ptr);
/* async copies of interleaved records [off, off+count) */
int32_t dampr_kv_upload(dampr_ctx *ctx, dampr_kv *kv, uint64_t off, const void *host_records,
                        uint64_t count);
int32_t dampr_kv_download(dampr_ctx *ctx, dampr_kv *kv, uint64_t off, void *host_records,
                          uint64_t count);
/* columnar <-> interleaved: host keys[] and vals[] (8 bytes each) */
int32_t dampr_kv_upload_columns(dampr_ctx *ctx, dampr_kv *kv, uint64_t off, const uint64_t *keys,
                                const uint64_t *vals, uint64_t count);
int32_t dampr_kv_download_columns(dampr_ctx *ctx, dampr_kv *kv, uint64_t off, uint64_t *keys,
                                  uint64_t *vals, uint64_t count);

/* key transforms applied on the fly by sort/partition (the stored key is never modified) */
#define DAMPR_KEY_RAW 0   /* order by the unsigned 64-bit key                                   */
#define DAMPR_KEY_MIX 1   /* order by a bijective 64-bit mix of the key: balanced partitions,
                             grouping only (Splitter.partition, base.py:6-8)                      */
#define DAMPR_KEY_I64 2   /* order as signed 64-bit                                              */
#define DAMPR_KEY_F64 3   /* order as IEEE double                                                */

/* partition-by-key + in-partition sort: replaces CSDatasetWriter.flush (dataset.py:236-253) +
 * Splitter.partition (base.py:6-8) + SortedWriter sort (dataset.py:162-164). Stable.
 * Result replaces the contents of `kv` (ping-pong buffer inside the library). */
int32_t dampr_kv_sort(dampr_ctx *ctx, dampr_kv *kv, int32_t key_xform);

/* reduce ops for the combiner / reducer (ARReduce.reduce binops, dampr.py:661-708) */
#define DAMPR_OP_SUM_I64 0
#define DAMPR_OP_SUM_F64 1
#define DAMPR_OP_COUNT 2
#define DAMPR_OP_MIN_I64 3
#define DAMPR_OP_MAX_I64 4
#define DAMPR_OP_MIN_F64 5
#define DAMPR_OP_MAX_F64 6
#define DAMPR_OP_FIRST 7
#define DAMPR_OP_LAST 8

/* segmented reduce of a key-sorted kv: one output record per key. Replaces
 * Dataset.grouped_read + Reduce.reduce (dataset.py:429-433, base.py:204-207). out is created; `sorted`
 * is left untouched. ONE pass over the input: tiles of 4096 records, head flags, fold; a key that straddles
 * tiles is folded across them in order. */
int32_t dampr_kv_reduce_by_key(dampr_ctx *ctx, dampr_kv *sorted, int32_t op, dampr_kv **out);
/* group boundaries of a key-sorted kv: offsets[g] = first record of group g, offsets[G] = n.
 * two-phase: pass offsets=NULL to get *n_groups. */
int32_t dampr_kv_group_offsets(dampr_ctx *ctx, dampr_kv *sorted, uint64_t *offsets, uint64_t cap,
                               uint64_t *n_groups);

/* k-way merge of key-sorted runs + optional segmented reduce: replaces MergeDataset.read
 * (dataset.py:571-579) + PartialReduceCombiner._combine (base.py:397-399). op < 0 = merge only.
 * One read of the runs, one write of the result: sampled splitters -> merge-path style cut vectors ->
 * one CTA per <= 4096-record partition (csrc/merge.cu). Stable: equal keys come out in run order, then in
 * position order (heapq.merge's order); any number of runs (more than 64 are merged in two levels). */
int32_t dampr_kv_merge(dampr_ctx *ctx, dampr_kv **runs, int32_t n_runs, int32_t key_xform,
                       int32_t op, dampr_kv **out);

/* the same merge over runs given as consecutive slices of ONE kv: run i = records [offsets[i], offsets[i+1])
 * (offsets has n_runs + 1 entries). The shape sorted runs have after the all-to-all (one run per source
 * rank) and after a spill upload (one run per batch). */
int32_t dampr_kv_merge_ranges(dampr_ctx *ctx, dampr_kv *kv, const uint64_t *offsets, int32_t n_runs,
                              int32_t key_xform, int32_t op, dampr_kv **out);

/* fused sort + reduce for associative ops (a_group_by(...).sum()/count()/...). CONSUMES `kv`: the
 * partition levels and the leaves use both of its buffers as scratch, so its contents are undefined
 * afterwards and its size is reset to 0 (destroy it, or upload new records). out is created. */
int32_t dampr_kv_sort_reduce(dampr_ctx *ctx, dampr_kv *kv, int32_t key_xform, int32_t op,
                             dampr_kv **out);

/* merge join of two key-sorted kvs: replaces InnerJoin.reduce / LeftJoin.reduce
 * (base.py:264-283, 295-315). Both inputs must be sorted with `key_xform`. Emits one row per
 * LEFT key group: rows[4*i+0..3] = left_begin, left_end, right_begin, right_end (record index
 * ranges; right_begin == right_end when the key has no match, which is what the left join keeps
 * and the inner join drops). Two-phase: rows == NULL returns *n_rows only. */
int32_t dampr_kv_join_ranges(dampr_ctx *ctx, dampr_kv *left_sorted, dampr_kv *right_sorted,
                             int32_t key_xform, uint64_t *rows, uint64_t cap, uint64_t *n_rows);

/* broadcast hash-probe join: replaces MapAllJoin.map (base.py:165-178) for agg=dict/set with a
 * membership/lookup crosser. build keys must be unique. out_vals[i] = build value of probe key i,
 * out_hit[i] = 1/0. */
int32_t dampr_kv_hash_probe(dampr_ctx *ctx, dampr_kv *build, dampr_kv *probe, dampr_kv **out_vals,
                            uint8_t *out_hit_host);

/* the same join with the result compacted ON THE DEVICE: out_probe[i] / out_build[i] = the i-th probe record that
 * found a partner (probe order kept) and (its key, the partner's build value). Inner join of a fact table with a
 * dimension table (PJoin.reduce with many=True over unique right keys, dampr.py:780-802) without a row of the
 * misses ever leaving the device. Both outputs are created. */
int32_t dampr_kv_hash_join(dampr_ctx *ctx, dampr_kv *build, dampr_kv *probe, dampr_kv **out_probe,
                           dampr_kv **out_build);

/* split a kv by destination rank: owner = mix(key) % n_dest; produces destination-contiguous
 * records in `out` and counts[n_dest] on the host. The payload then moves with one all-to-all
 * (torch.distributed/NCCL over NVLink) — replaces DefaultShuffler.shuffle (base.py:416-433). */
int32_t dampr_kv_partition_by_owner(dampr_ctx *ctx, dampr_kv *kv, int32_t n_dest, dampr_kv **out,
                                    uint64_t *counts_host);

/* ---- S1 across GPUs: the shuffle exchange inside the C-ABI (SURVEY §8(b) kv_all_to_all) --------------------
 * One process per GPU. dampr_comm_unique_id on rank 0 -> the host runtime hands the bytes to every rank (any
 * bootstrap it has: torch.distributed, MPI, a file) -> dampr_comm_create on every rank (ncclCommInitRank).
 * dampr_kv_all_to_all replaces DefaultShuffler.shuffle (base.py:416-433) + the per-partition run files the
 * reducers read (stagerunner.py:269-282): every record goes to the rank that owns its key
 * (owner = mix(key) % world, the same function on every rank = one Splitter for all inputs, base.py:264-283).
 * *out = this rank's records, those of source rank s at [out_offsets[s], out_offsets[s+1]) in the order rank s
 * held them (a key-sorted input arrives as world sorted runs: the input of dampr_kv_merge_ranges).
 * header / headers_all: n_header (<= 64) int64 values per rank, all-gathered with the counts (row s of
 * headers_all = rank s's header) so that line counts / flags need no collective of their own.
 * NCCL is bound at run time (dlopen libnccl.so.2); without it these calls fail, nothing else does. */
typedef struct dampr_comm dampr_comm;
#define DAMPR_COMM_ID_BYTES 128
int32_t dampr_comm_unique_id(uint8_t *out_id, uint32_t cap);
int32_t dampr_comm_create(dampr_ctx *ctx, int32_t rank, int32_t world, const uint8_t *id, uint32_t id_bytes,
                          dampr_comm **out);
int32_t dampr_comm_destroy(dampr_comm *comm);
int32_t dampr_kv_all_to_all(dampr_ctx *ctx, dampr_comm *comm, dampr_kv *kv, const int64_t *header,
                            int32_t n_header, dampr_kv **out, uint64_t *out_offsets, int64_t *headers_all);

/* ---- synthetic inputs (bench/test tooling; deterministic, same algorithm as oracle/gen.py) */
int32_t dampr_synth_text(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t seed, uint64_t n_lines,
                         const uint8_t *vocab_bytes, const uint32_t *vocab_off, uint32_t vocab_n,
                         const uint64_t *cdf, uint64_t *out_nbytes);
int32_t dampr_synth_kv(dampr_ctx *ctx, dampr_kv *kv, uint64_t seed, uint64_t n, uint64_t n_keys);

#ifdef __cplusplus
}
#endif
#endif /* DAMPR_B200_H */

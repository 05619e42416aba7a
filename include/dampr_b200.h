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
/* process-wide tuning switches: "kv_scatter" (2 = atomic-rank scatter, up to 12 digit bits per level,
 * default; 1 = first-generation ballot scatter, 10 bits), "kv_cluster" (1 = thread-block-cluster leaf over
 * distributed shared memory, default), "kv_tile" (4096 | 8192 records per scatter tile), "kv_max_bits";
 * "scatter_tma" (first-generation scatter only: 1 = TMA bulk stores, 0 = coalesced 16-byte stores); "text_ctas" (3 = single-window 3 CTAs/SM variant of the v2
 * tokenise kernel, default; 2 = double-buffered 2 CTAs/SM); "text_kernel" (2 = warp-autonomous tokenise kernel, default;
 * 1 = first-generation kernel, also the fallback for lines longer than 2 KB) */
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
int32_t dampr_table_stats(dampr_ctx *ctx, dampr_table *t, uint64_t stats[8]);
/* Per-line fallback of the [^\w]+ tokenisers: a line that holds a byte the device cannot tokenise the way
 * Python does (non-ASCII: Unicode \w / lower(); '\r' in text mode: universal newlines) contributes NOTHING to
 * the table, the line count or the '' token count; instead lines[i] = (byte offset of the line << 16) | length
 * (without its '\n') is reported here and the caller tokenises just those lines (TextLineDataset.read,
 * dataset.py:458-476 + the user's lambda) and adds the results. Order unspecified. Two-phase: lines == NULL
 * returns *n only. More than 65536 such lines, or one that cannot be isolated inside the kernel's window, set
 * DAMPR_TF_NONASCII instead (the whole scan is then the caller's). str.split mode keeps scan-wide flags. */
int32_t dampr_table_fallback_lines(dampr_ctx *ctx, dampr_table *t, uint64_t *lines, uint64_t cap, uint64_t *n);
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

// merge.cu — K5: k-way merge of key-sorted runs + head-flag segmented reduce.
//
// Replaces
//   MergeDataset.read              dampr/dataset.py:567-579   heapq.merge of the sorted spill runs
//   PartialReduceCombiner._combine dampr/base.py:393-402      fold equal keys while merging
//   Dataset.grouped_read + Reduce  dampr/dataset.py:429-433, dampr/base.py:204-207 (sorted input -> groups)
//
// One read of the runs, one write of the result (merge) or of the groups (merge + reduce):
//   1. every S-th record of every run is a sample (key, run, position); the samples are sorted with the
//      partition/leaf machinery of kv.cu (they are ~1/128 of the input);
//   2. every m-th sorted sample is a boundary; a binary search per (boundary, run) turns it into a cut
//      vector.  Ties are broken by (run, position), so between two consecutive cut vectors lie at most
//      (m + k) * S <= 4096 records whatever the key distribution (heavy duplicates included) and the
//      merge is stable: equal keys come out in run order, then in position order — heapq.merge's order;
//   3. one CTA per partition loads its k sub-ranges into shared memory (run-major, so the shared-memory
//      index IS the stable tie-break), sorts them with the leaf's counting sort + rank-by-(key, index)
//      and writes the merged records — or folds equal keys first (segmented reduce) and writes one record
//      per key to a staging buffer;
//   4. reduce only: a key whose records straddle partitions is folded across them in partition order by
//      the partition where it starts (cont flags + scan + gather).
// A single sorted run (dampr_kv_reduce_by_key) skips 1-2 and the shared-memory sort: tiles of 4096
// consecutive records, head flags, fold, gather.
#include <algorithm>

#include "common.cuh"
#include "leaf.cuh"

namespace {

constexpr int M_MAX_RUNS = 64;
constexpr u64 M_POS_MASK = (1ULL << 40) - 1;

struct RunDesc {
    const ulonglong2 *rec;
    u64 n;
};

__global__ void merge_sample_kernel(const RunDesc *__restrict__ runs, const u64 *__restrict__ soff, u32 k, u32 S,
                                    int xf, ulonglong2 *__restrict__ samples) {
    const u64 ns = soff[k];
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < ns; i += (u64)gridDim.x * blockDim.x) {
        u32 r = 0;
        while (r + 1 < k && soff[r + 1] <= i) ++r;
        const u64 pos = (i - soff[r] + 1) * (u64)S - 1;
        samples[i] = make_ulonglong2(key_xform(runs[r].rec[pos].x, xf), ((u64)r << 40) | pos);
    }
}

// first index in run with xf(key) >= s (strict = false) or > s (strict = true)
__device__ __forceinline__ u64 run_bound(const RunDesc &run, u64 s, int xf, bool strict) {
    u64 lo = 0, hi = run.n;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        const u64 km = key_xform(run.rec[mid].x, xf);
        if (strict ? (km <= s) : (km < s)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// cuts[(j + 1) * k + r] for boundary j, plus rows 0 and nbnd + 1 and the partition key bounds
__global__ void merge_cut_kernel(const RunDesc *__restrict__ runs, u32 k, const ulonglong2 *__restrict__ sorted_samples,
                                 u32 m, u64 nbnd, int xf, u64 *__restrict__ cuts, u64 *__restrict__ bkeys) {
    const u64 total = (nbnd + 1) * k;
    for (u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
        const u64 j = t / k;
        const u32 r = (u32)(t % k);
        if (j == nbnd) {
            cuts[r] = 0;
            cuts[(nbnd + 1) * k + r] = runs[r].n;
            if (r == 0) {
                u64 mn = ~0ULL, mx = 0;
                for (u32 q = 0; q < k; ++q)
                    if (runs[q].n) {
                        mn = min(mn, key_xform(runs[q].rec[0].x, xf));
                        mx = max(mx, key_xform(runs[q].rec[runs[q].n - 1].x, xf));
                    }
                if (mn > mx) mn = mx = 0;
                bkeys[0] = mn;
                bkeys[nbnd + 1] = mx;
            }
            continue;
        }
        const ulonglong2 smp = sorted_samples[(j + 1) * (u64)m - 1];
        const u32 rs = (u32)(smp.y >> 40);
        const u64 ps = smp.y & M_POS_MASK;
        u64 c;
        if (r == rs) c = ps + 1;
        else c = run_bound(runs[r], smp.x, xf, r < rs);
        cuts[(j + 1) * k + r] = c;
        if (r == 0) bkeys[j + 1] = smp.x;
    }
}

struct TileExtra {
    u64 roff[M_MAX_RUNS + 1];  // smem offset of every run's sub-range
    u64 rlo[M_MAX_RUNS];       // first record of the sub-range in its run
    u64 out_off;
    u32 n;
};

// reduce_op < 0: merged records to out[out_off ...). Otherwise one record per key of the partition to
// out[out_off ...) (staging) and (start, groups) to part_start / part_groups.
__global__ void __launch_bounds__(L_THREADS, 2)
merge_tile_kernel(const RunDesc *__restrict__ runs, u32 k, const u64 *__restrict__ cuts,
                  const u64 *__restrict__ bkeys, u64 P, int xf, int reduce_op, ulonglong2 *__restrict__ out,
                  u64 *__restrict__ part_start, u32 *__restrict__ part_groups, u32 *__restrict__ err_flag) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    LeafSmem &s = *reinterpret_cast<LeafSmem *>(smem_raw);
    TileExtra &x = *reinterpret_cast<TileExtra *>(smem_raw + sizeof(LeafSmem));
    const u32 tid = threadIdx.x;
    for (u64 p = blockIdx.x; p < P; p += gridDim.x) {
        if (tid == 0) {
            u64 run = 0, oo = 0;
            for (u32 r = 0; r < k; ++r) {
                const u64 lo = cuts[p * k + r], hi = cuts[(p + 1) * k + r];
                x.roff[r] = run;
                x.rlo[r] = lo;
                run += hi - lo;
                oo += lo;
            }
            x.roff[k] = run;
            x.out_off = oo;
            x.n = (u32)min(run, (u64)0xFFFFFFFFu);
        }
        __syncthreads();
        const u32 n = x.n;
        const u64 out_off = x.out_off;
        if (n > (u32)L_CAP) {  // cannot happen (see the bound in the header); never write out of bounds
            if (tid == 0) {
                atomicExch(err_flag, 1u);
                if (reduce_op >= 0) {
                    part_start[p] = out_off;
                    part_groups[p] = 0;
                }
            }
            __syncthreads();
            continue;
        }
        const u64 klo = (k > 1) ? bkeys[p] : 0ULL;
        for (u32 i = tid; i < n; i += L_THREADS) {
            u32 lo = 0, hi = k;  // last r with roff[r] <= i
            while (hi - lo > 1) {
                const u32 mid = (lo + hi) >> 1;
                if (x.roff[mid] <= i) lo = mid;
                else hi = mid;
            }
            const ulonglong2 rc = runs[lo].rec[x.rlo[lo] + (i - x.roff[lo])];
            s.sk[i] = key_xform(rc.x, xf) - klo;
            s.val[i] = rc.y;
        }
        __syncthreads();
        if (k > 1) {
            const u64 span = bkeys[p + 1] - klo;
            int shift = 0;
            while (shift < 64 && (span >> shift) >= (u64)L_BINS) ++shift;
            leaf_sort_core(s, n, shift, 0);
        } else {
            for (u32 i = tid; i < n; i += L_THREADS) s.fin[i] = (u16)i;
            __syncthreads();
        }
        if (reduce_op < 0) {
            for (u32 i = tid; i < n; i += L_THREADS) {
                const u32 o = s.fin[i];
                out[out_off + i] = make_ulonglong2(key_unxform(s.sk[o] + klo, xf), s.val[o]);
            }
        } else {
            const u32 g = leaf_seg_reduce(s, n, reduce_op, xf, klo, out + out_off);
            if (tid == 0) {
                part_start[p] = out_off;
                part_groups[p] = g;
            }
        }
        __syncthreads();
    }
}

// cont[p] = the first group of partition p continues the last group of the previous non-empty partition
__global__ void merge_cont_kernel(const ulonglong2 *__restrict__ tmp, const u64 *__restrict__ pstart,
                                  const u32 *__restrict__ pg, u64 P, u32 *__restrict__ contrib,
                                  unsigned char *__restrict__ cont) {
    for (u64 p = blockIdx.x * (u64)blockDim.x + threadIdx.x; p < P; p += (u64)gridDim.x * blockDim.x) {
        const u32 g = pg[p];
        u32 c = 0;
        if (g) {
            u64 q = p;
            while (q > 0 && pg[q - 1] == 0) --q;
            if (q > 0) {
                --q;
                c = (tmp[pstart[q] + pg[q] - 1].x == tmp[pstart[p]].x) ? 1u : 0u;
            }
        }
        cont[p] = (unsigned char)c;
        contrib[p] = g - c;
    }
}

__global__ void merge_gather_kernel(const ulonglong2 *__restrict__ tmp, const u64 *__restrict__ pstart,
                                    const u32 *__restrict__ pg, const unsigned char *__restrict__ cont,
                                    const u64 *__restrict__ poff, u64 P, int op, ulonglong2 *__restrict__ out) {
    const int cop = (op == DAMPR_OP_COUNT) ? DAMPR_OP_SUM_I64 : op;
    for (u64 p = blockIdx.x; p < P; p += gridDim.x) {
        const u32 g = pg[p], c = cont[p];
        const u64 st = pstart[p], off = poff[p];
        for (u32 i = threadIdx.x + c; i < g; i += blockDim.x) {
            ulonglong2 rec = tmp[st + i];
            if (i == g - 1) {
                // the key may go on in the following partitions: fold their leading groups in order
                u64 q = p + 1;
                while (q < P) {
                    const u32 gq = pg[q];
                    if (gq == 0) {
                        ++q;
                        continue;
                    }
                    if (!cont[q]) break;
                    rec.y = apply_op(cop, rec.y, tmp[pstart[q]].y);
                    if (gq > 1) break;
                    ++q;
                }
            }
            out[off + i - c] = rec;
        }
    }
}

// merge (op < 0) or merge + reduce of k <= M_MAX_RUNS device runs into a new kv
static int merge_small_k(dampr_ctx *ctx, const std::vector<RunDesc> &runs, int xf, int op, dampr_kv **out) {
    const u32 k = (u32)runs.size();
    u64 N = 0;
    for (auto &r : runs) N += r.n;
    int rc;
    if (N == 0) return dampr_kv_create(ctx, 0, out);
    DevBuf d_runs, d_soff, d_samples, d_salt, d_cuts, d_bkeys, d_err;
    u64 P = 0, nbnd = 0;
    const size_t rbytes = k * sizeof(RunDesc);
    {
        char *hp = (char *)host_pin(ctx, 1, rbytes + (k + 1) * 8 + 64);
        if (!hp) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
        memcpy(hp, runs.data(), rbytes);
        CUDA_TRY(ctx, d_runs.alloc(rbytes));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_runs.p, hp, rbytes, cudaMemcpyHostToDevice, ctx->stream));
        if (k > 1) {
            const u32 S = std::max<u32>(1, (u32)L_CAP / (4 * k)), m = 3 * k;
            u64 *soff = (u64 *)(hp + ((rbytes + 15) & ~(size_t)15));
            u64 ns = 0;
            for (u32 r = 0; r < k; ++r) {
                soff[r] = ns;
                ns += runs[r].n / S;
            }
            soff[k] = ns;
            nbnd = ns / m;
            P = nbnd + 1;
            CUDA_TRY(ctx, d_soff.alloc((k + 1) * 8));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_soff.p, soff, (k + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
            host_pin_used(ctx, 1);
            CUDA_TRY(ctx, d_cuts.alloc((P + 1) * k * 8));
            CUDA_TRY(ctx, d_bkeys.alloc((P + 1) * 8));
            if (ns) {
                CUDA_TRY(ctx, d_samples.alloc(ns * 16));
                CUDA_TRY(ctx, d_salt.alloc(ns * 16));
                {
                    ScopedTimer tm(ctx, DAMPR_K_MERGE);
                    merge_sample_kernel<<<(unsigned)std::min<u64>((ns + 255) / 256, (u64)ctx->num_sms * 8), 256, 0, ctx->stream>>>(
                        (const RunDesc *)d_runs.p, (const u64 *)d_soff.p, k, S, xf, (ulonglong2 *)d_samples.p);
                }
                CUDA_TRY(ctx, cudaGetLastError());
                // stable sort by key: ties keep the (run, position) order the samples were written in
                rc = kv_sort_device_range(ctx, (ulonglong2 *)d_samples.p, (ulonglong2 *)d_salt.p, ns, DAMPR_KEY_RAW);
                if (rc) return rc;
            }
            {
                ScopedTimer tm(ctx, DAMPR_K_MERGE);
                const u64 total = (nbnd + 1) * k;
                merge_cut_kernel<<<(unsigned)std::min<u64>((total + 127) / 128, (u64)ctx->num_sms * 16), 128, 0, ctx->stream>>>(
                    (const RunDesc *)d_runs.p, k, (const ulonglong2 *)d_samples.p, m, nbnd, xf, (u64 *)d_cuts.p,
                    (u64 *)d_bkeys.p);
            }
            CUDA_TRY(ctx, cudaGetLastError());
        } else {
            host_pin_used(ctx, 1);
            // one sorted run: fixed tiles
            P = (N + L_CAP - 1) / L_CAP;
            std::vector<u64> cuts(P + 1);
            for (u64 p = 0; p <= P; ++p) cuts[p] = std::min(N, p * (u64)L_CAP);
            u64 *hc = (u64 *)host_pin(ctx, 0, (P + 1) * 8);
            if (!hc) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
            memcpy(hc, cuts.data(), (P + 1) * 8);
            CUDA_TRY(ctx, d_cuts.alloc((P + 1) * 8));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_cuts.p, hc, (P + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
            host_pin_used(ctx, 0);
        }
    }
    CUDA_TRY(ctx, d_err.alloc(8));
    CUDA_TRY(ctx, cudaMemsetAsync(d_err.p, 0, 8, ctx->stream));
    const size_t smem = sizeof(LeafSmem) + sizeof(TileExtra);
    CUDA_TRY(ctx, cudaFuncSetAttribute(merge_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const u32 grid = (u32)std::min<u64>(P, (u64)ctx->num_sms * 2);
    if (op < 0) {
        rc = dampr_kv_create(ctx, N, out);
        if (rc) return rc;
        (*out)->n = N;
        {
            ScopedTimer tm(ctx, DAMPR_K_MERGE);
            merge_tile_kernel<<<grid, L_THREADS, smem, ctx->stream>>>((const RunDesc *)d_runs.p, k, (const u64 *)d_cuts.p,
                                                                     (const u64 *)d_bkeys.p, P, xf, -1, (*out)->rec, nullptr,
                                                                     nullptr, (u32 *)d_err.p);
        }
        CUDA_TRY(ctx, cudaGetLastError());
        u32 *he = (u32 *)ctx->h_scratch;
        CUDA_TRY(ctx, cudaMemcpyAsync(he, d_err.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        if (he[0]) {
            dampr_kv_destroy(ctx, *out);
            *out = nullptr;
            return set_err(ctx, DAMPR_ERR_CUDA, "%s", "merge partition exceeded its tile (internal error)");
        }
        return DAMPR_OK;
    }
    DevBuf d_tmp, d_pstart, d_pg, d_contrib, d_cont, d_poff;
    CUDA_TRY(ctx, d_tmp.alloc(N * 16));
    CUDA_TRY(ctx, d_pstart.alloc(P * 8));
    CUDA_TRY(ctx, d_pg.alloc(P * 4));
    CUDA_TRY(ctx, d_contrib.alloc(P * 4));
    CUDA_TRY(ctx, d_cont.alloc(P));
    CUDA_TRY(ctx, d_poff.alloc((P + 1) * 8));
    {
        ScopedTimer tm(ctx, DAMPR_K_MERGE);
        merge_tile_kernel<<<grid, L_THREADS, smem, ctx->stream>>>((const RunDesc *)d_runs.p, k, (const u64 *)d_cuts.p,
                                                                 (const u64 *)d_bkeys.p, P, xf, op, (ulonglong2 *)d_tmp.p,
                                                                 (u64 *)d_pstart.p, (u32 *)d_pg.p, (u32 *)d_err.p);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_SEG_REDUCE);
        merge_cont_kernel<<<(unsigned)std::min<u64>((P + 255) / 256, (u64)ctx->num_sms * 8), 256, 0, ctx->stream>>>(
            (const ulonglong2 *)d_tmp.p, (const u64 *)d_pstart.p, (const u32 *)d_pg.p, P, (u32 *)d_contrib.p,
            (unsigned char *)d_cont.p);
        scan_u32_to_u64_kernel<<<1, 1024, 0, ctx->stream>>>((const u32 *)d_contrib.p, (u64 *)d_poff.p, (u32)P);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    u64 *hs = ctx->h_scratch;
    CUDA_TRY(ctx, cudaMemcpyAsync(hs, (u64 *)d_poff.p + P, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(hs + 1, d_err.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if ((u32)hs[1]) return set_err(ctx, DAMPR_ERR_CUDA, "%s", "merge partition exceeded its tile (internal error)");
    const u64 G = hs[0];
    rc = dampr_kv_create(ctx, G, out);
    if (rc) return rc;
    (*out)->n = G;
    {
        ScopedTimer tm(ctx, DAMPR_K_SEG_REDUCE);
        merge_gather_kernel<<<(unsigned)std::min<u64>(P, (u64)ctx->num_sms * 8), 256, 0, ctx->stream>>>(
            (const ulonglong2 *)d_tmp.p, (const u64 *)d_pstart.p, (const u32 *)d_pg.p, (const unsigned char *)d_cont.p,
            (const u64 *)d_poff.p, P, op, (*out)->rec);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

}  // namespace

extern "C" {

// k-way merge of key-sorted runs (+ optional segmented reduce); stable: ties come out in run order, then in
// position order, exactly what heapq.merge produces (dataset.py:571-579)
int32_t dampr_kv_merge(dampr_ctx *ctx, dampr_kv **runs, int32_t n_runs, int32_t key_xf, int32_t op,
                       dampr_kv **out) {
    ARG_CHECK(ctx, ctx && runs && out && n_runs >= 0, "null");
    ARG_CHECK(ctx, key_xf >= 0 && key_xf <= DAMPR_KEY_F64, "unknown key transform");
    ARG_CHECK(ctx, op <= DAMPR_OP_LAST, "unknown reduce op");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    std::vector<RunDesc> cur;
    for (int i = 0; i < n_runs; ++i) {
        ARG_CHECK(ctx, runs[i] != nullptr, "null run");
        ARG_CHECK(ctx, runs[i]->n <= M_POS_MASK, "run too long");
        if (runs[i]->n) cur.push_back(RunDesc{runs[i]->rec, runs[i]->n});  // dropping empty runs keeps the run order
    }
    if (cur.empty()) return dampr_kv_create(ctx, 0, out);
    // more runs than one pass takes: merge groups of M_MAX_RUNS consecutive runs first (order-preserving).
    // Partial folds of COUNT are counts, combined by addition from the second level on.
    std::vector<dampr_kv *> temps;
    int level_op = op;
    int rc = DAMPR_OK;
    while (cur.size() > (size_t)M_MAX_RUNS) {
        std::vector<RunDesc> next;
        std::vector<dampr_kv *> made;
        for (size_t i = 0; i < cur.size() && rc == DAMPR_OK; i += M_MAX_RUNS) {
            std::vector<RunDesc> grp(cur.begin() + i, cur.begin() + std::min(cur.size(), i + (size_t)M_MAX_RUNS));
            dampr_kv *t = nullptr;
            rc = merge_small_k(ctx, grp, key_xf, level_op, &t);
            if (rc == DAMPR_OK) {
                made.push_back(t);
                if (t->n) next.push_back(RunDesc{t->rec, t->n});
            }
        }
        for (auto *t : temps) dampr_kv_destroy(ctx, t);
        temps.swap(made);
        if (rc) break;
        cur.swap(next);
        if (level_op == DAMPR_OP_COUNT) level_op = DAMPR_OP_SUM_I64;
        if (cur.empty()) break;
    }
    if (rc == DAMPR_OK) {
        if (cur.empty()) rc = dampr_kv_create(ctx, 0, out);
        else rc = merge_small_k(ctx, cur, key_xf, level_op, out);
    }
    for (auto *t : temps) dampr_kv_destroy(ctx, t);
    return rc;
}

// the same merge over runs that are CONSECUTIVE SLICES of one kv: run i = records [offsets[i], offsets[i+1]).
// This is how sorted runs arrive from the all-to-all (one run per source rank, back to back in the receive
// buffer) and from the spill uploads (one run per batch).
int32_t dampr_kv_merge_ranges(dampr_ctx *ctx, dampr_kv *kv, const uint64_t *offsets, int32_t n_runs,
                              int32_t key_xf, int32_t op, dampr_kv **out) {
    ARG_CHECK(ctx, ctx && kv && out && n_runs >= 0 && (offsets || n_runs == 0), "null");
    std::vector<dampr_kv> views((size_t)n_runs);
    std::vector<dampr_kv *> ptrs((size_t)n_runs);
    for (int i = 0; i < n_runs; ++i) {
        ARG_CHECK(ctx, offsets[i] <= offsets[i + 1] && offsets[i + 1] <= kv->n, "run offsets out of range");
        views[i].rec = kv->rec + offsets[i];
        views[i].alt = nullptr;
        views[i].capacity = views[i].n = offsets[i + 1] - offsets[i];
        ptrs[i] = &views[i];
    }
    return dampr_kv_merge(ctx, ptrs.data(), n_runs, key_xf, op, out);
}

// segmented reduce of a key-sorted kv in ONE pass over it: tiles of 4096 records, head flags, fold, then the
// groups are compacted (a key that straddles tiles is folded across them in order). `sorted` is not modified.
int32_t dampr_kv_reduce_by_key(dampr_ctx *ctx, dampr_kv *sorted, int32_t op, dampr_kv **out) {
    ARG_CHECK(ctx, ctx && sorted && out, "null");
    ARG_CHECK(ctx, op >= 0 && op <= DAMPR_OP_LAST, "unknown reduce op");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    std::vector<RunDesc> one;
    if (sorted->n) one.push_back(RunDesc{sorted->rec, sorted->n});
    if (one.empty()) return dampr_kv_create(ctx, 0, out);
    return merge_small_k(ctx, one, DAMPR_KEY_RAW, op, out);
}

}  // extern "C"

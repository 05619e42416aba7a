// ops.cu — columnar transfers, merge join (K6), broadcast hash probe (K7), synthetic inputs.
//
//   InnerJoin.reduce / LeftJoin.reduce   dampr/base.py:264-283, 295-315  -> dampr_kv_join_ranges
//   MapAllJoin.map (agg=dict/set)        dampr/base.py:165-178           -> dampr_kv_hash_probe
#include "common.cuh"

namespace {

__global__ void interleave_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ vals,
                                  ulonglong2 *__restrict__ out, u64 n) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        out[i] = make_ulonglong2(keys[i], vals ? vals[i] : 0ULL);
}

__global__ void deinterleave_kernel(const ulonglong2 *__restrict__ in, u64 *__restrict__ keys,
                                    u64 *__restrict__ vals, u64 n) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        ulonglong2 r = in[i];
        if (keys) keys[i] = r.x;
        if (vals) vals[i] = r.y;
    }
}

// heads of a key-sorted array: flag + per-tile counts, then ranks (same scheme as kv.cu)
__global__ void heads_count_kernel(const ulonglong2 *__restrict__ in, u64 n, u32 *__restrict__ tile_cnt) {
    __shared__ u32 wsum[32];
    const u64 t0 = (u64)blockIdx.x * 4096ULL;
    u32 cnt = 0;
    for (int k = 0; k < 8; ++k) {
        u64 i = t0 + (u64)threadIdx.x * 8 + k;
        if (i < n && (i == 0 || in[i].x != in[i - 1].x)) ++cnt;
    }
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_down_sync(0xFFFFFFFFu, cnt, d);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 t = 0;
        for (u32 w = 0; w < blockDim.x / 32; ++w) t += wsum[w];
        tile_cnt[blockIdx.x] = t;
    }
}

__global__ void heads_write_kernel(const ulonglong2 *__restrict__ in, u64 n, const u64 *__restrict__ tile_base,
                                   u64 *__restrict__ offsets) {
    __shared__ u32 wsum[32];
    const u64 t0 = (u64)blockIdx.x * 4096ULL;
    u32 flags = 0;
    for (int k = 0; k < 8; ++k) {
        u64 i = t0 + (u64)threadIdx.x * 8 + k;
        if (i < n && (i == 0 || in[i].x != in[i - 1].x)) flags |= 1u << k;
    }
    u32 cnt = __popc(flags), v = cnt;
    for (int d = 1; d < 32; d <<= 1) {
        u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((int)(threadIdx.x & 31) >= d) v += o;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    u32 woff = 0;
    for (u32 w = 0; w < (threadIdx.x >> 5); ++w) woff += wsum[w];
    u64 g = tile_base[blockIdx.x] + woff + v - cnt;
    for (int k = 0; k < 8; ++k)
        if (flags & (1u << k)) offsets[g++] = t0 + (u64)threadIdx.x * 8 + k;
}

__global__ void scan_tiles_kernel(const u32 *__restrict__ in, u64 *__restrict__ out, u32 n) {
    __shared__ u64 wsum[32];
    __shared__ u64 carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (u32 base = 0; base < n + 1; base += blockDim.x) {
        u32 i = base + threadIdx.x;
        u64 x = (i < n) ? in[i] : 0;
        u64 v = x;
        for (int d = 1; d < 32; d <<= 1) {
            u64 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
            if ((int)(threadIdx.x & 31) >= d) v += o;
        }
        if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = v;
        __syncthreads();
        u64 woff = 0;
        for (u32 w = 0; w < (threadIdx.x >> 5); ++w) woff += wsum[w];
        u64 excl = carry + woff + v - x;
        if (i <= n) out[i] = excl;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = excl + x;
        __syncthreads();
    }
}

// one thread per left group: binary search the right groups (both ordered by xf(key))
__global__ void join_ranges_kernel(const ulonglong2 *__restrict__ L, const u64 *__restrict__ lo, u64 GL, u64 NL,
                                   const ulonglong2 *__restrict__ R, const u64 *__restrict__ ro, u64 GR, u64 NR,
                                   int xf, u64 *__restrict__ rows) {
    for (u64 g = blockIdx.x * (u64)blockDim.x + threadIdx.x; g < GL; g += (u64)gridDim.x * blockDim.x) {
        u64 lb = lo[g], le = (g + 1 < GL) ? lo[g + 1] : NL;
        u64 key = key_xform(L[lb].x, xf);
        u64 a = 0, b = GR;  // first right group with key >= key
        while (a < b) {
            u64 m = (a + b) >> 1;
            if (key_xform(R[ro[m]].x, xf) < key) a = m + 1;
            else b = m;
        }
        u64 rb = 0, re = 0;
        if (a < GR && key_xform(R[ro[a]].x, xf) == key) {
            rb = ro[a];
            re = (a + 1 < GR) ? ro[a + 1] : NR;
        }
        rows[4 * g + 0] = lb;
        rows[4 * g + 1] = le;
        rows[4 * g + 2] = rb;
        rows[4 * g + 3] = re;
    }
}

// open-addressing build / probe (keys unique on the build side); slot 0..cap-1, empty = flag array
__global__ void probe_build_kernel(const ulonglong2 *__restrict__ build, u64 n, u64 *__restrict__ tk,
                                   u64 *__restrict__ tv, u32 *__restrict__ used, u64 mask, u64 *__restrict__ dup) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        ulonglong2 r = build[i];
        u64 slot = mix64(r.x) & mask;
        for (;;) {
            u32 prev = atomicCAS(&used[slot], 0u, 1u);
            if (prev == 0u) {
                tk[slot] = r.x;
                tv[slot] = r.y;
                __threadfence();
                atomicExch(&used[slot], 2u);
                break;
            }
            // wait until the owner published its key
            while (atomicAdd(&used[slot], 0u) != 2u) {
            }
            if (((volatile u64 *)tk)[slot] == r.x) {
                atomicAdd(dup, 1ULL);  // duplicate build key: keep the first
                break;
            }
            slot = (slot + 1) & mask;
        }
    }
}

__global__ void probe_lookup_kernel(const ulonglong2 *__restrict__ probe, u64 n, const u64 *__restrict__ tk,
                                    const u64 *__restrict__ tv, const u32 *__restrict__ used, u64 mask,
                                    ulonglong2 *__restrict__ out, u8 *__restrict__ hit) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 key = probe[i].x;
        u64 slot = mix64(key) & mask;
        u64 val = 0;
        u8 h = 0;
        for (;;) {
            if (used[slot] == 0u) break;
            if (tk[slot] == key) {
                val = tv[slot];
                h = 1;
                break;
            }
            slot = (slot + 1) & mask;
        }
        out[i] = make_ulonglong2(key, val);
        hit[i] = h;
    }
}

// ---- compaction of the probe result: matched records only, probe order kept --------------------
constexpr int HC_THREADS = 512;
constexpr int HC_TILE = HC_THREADS * 8;
__global__ void __launch_bounds__(HC_THREADS)
hits_count_kernel(const u8 *__restrict__ hit, u64 n, u32 *__restrict__ tile_cnt) {
    __shared__ u32 wsum[HC_THREADS / 32];
    const u64 t0 = (u64)blockIdx.x * HC_TILE + (u64)threadIdx.x * 8;
    u32 c = 0;
    if (t0 + 8 <= n) {
        const u64 w = *reinterpret_cast<const u64 *>(hit + t0);  // 8 flags (0 / 1) per load
        c = (u32)__popcll(w & 0x0101010101010101ULL);
    } else {
        for (u64 i = t0; i < n && i < t0 + 8; ++i) c += hit[i] ? 1u : 0u;
    }
    for (int d = 16; d > 0; d >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, d);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 t = 0;
        for (int w = 0; w < HC_THREADS / 32; ++w) t += wsum[w];
        tile_cnt[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(HC_THREADS)
hits_compact_kernel(const ulonglong2 *__restrict__ probe, const ulonglong2 *__restrict__ vals,
                    const u8 *__restrict__ hit, u64 n, const u64 *__restrict__ tile_base,
                    ulonglong2 *__restrict__ out_probe, ulonglong2 *__restrict__ out_build) {
    __shared__ u32 wsum[HC_THREADS / 32];
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u64 t0 = (u64)blockIdx.x * HC_TILE + (u64)threadIdx.x * 8;
    u32 flags = 0;
    for (int k = 0; k < 8; ++k)
        if (t0 + k < n && hit[t0 + k]) flags |= 1u << k;
    const u32 c = (u32)__popc(flags);
    u32 v = c;
    for (int d = 1; d < 32; d <<= 1) {
        u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((int)lane >= d) v += o;
    }
    if (lane == 31) wsum[warp] = v;
    __syncthreads();
    u32 woff = 0;
    for (u32 w = 0; w < warp; ++w) woff += wsum[w];
    u64 pos = tile_base[blockIdx.x] + woff + v - c;
    for (int k = 0; k < 8; ++k)
        if (flags & (1u << k)) {
            out_probe[pos] = probe[t0 + k];
            out_build[pos] = vals[t0 + k];
            ++pos;
        }
}

// ---- synthetic inputs (same integer algorithm as oracle/gen.py) -------------------------------
__host__ __device__ __forceinline__ u64 splitmix64(u64 x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

__device__ __forceinline__ u32 cdf_lookup(const u64 *__restrict__ cdf, u32 n, u64 r) {
    // first index with cdf[idx] >= r  (numpy.searchsorted(cdf, r, side='left')), clamped to n-1
    u32 a = 0, b = n;
    while (a < b) {
        u32 m = (a + b) >> 1;
        if (cdf[m] < r) a = m + 1;
        else b = m;
    }
    return a < n ? a : n - 1;
}

__global__ void synth_len_kernel(u64 seed, u64 n_lines, const u32 *__restrict__ voff, u32 vn,
                                 const u64 *__restrict__ cdf, u32 *__restrict__ line_len) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n_lines; i += (u64)gridDim.x * blockDim.x) {
        u64 r0 = splitmix64(seed ^ (i * 0x9E3779B97F4A7C15ULL));
        u32 ntok = 5 + (u32)(r0 % 15ULL);
        u32 len = ntok;  // separators + newline
        for (u32 j = 0; j < ntok; ++j) {
            u64 r = splitmix64(r0 + (u64)(j + 1) * 0xD1B54A32D192ED03ULL);
            u32 w = cdf_lookup(cdf, vn, r);
            len += voff[w + 1] - voff[w];
        }
        line_len[i] = len;
    }
}

__global__ void synth_write_kernel(u64 seed, u64 n_lines, const u8 *__restrict__ vbytes, const u32 *__restrict__ voff,
                                   u32 vn, const u64 *__restrict__ cdf, const u64 *__restrict__ line_off,
                                   u8 *__restrict__ text) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n_lines; i += (u64)gridDim.x * blockDim.x) {
        u64 r0 = splitmix64(seed ^ (i * 0x9E3779B97F4A7C15ULL));
        u32 ntok = 5 + (u32)(r0 % 15ULL);
        u8 *p = text + line_off[i];
        for (u32 j = 0; j < ntok; ++j) {
            u64 r = splitmix64(r0 + (u64)(j + 1) * 0xD1B54A32D192ED03ULL);
            u32 w = cdf_lookup(cdf, vn, r);
            u32 a = voff[w], b = voff[w + 1];
            for (u32 k = a; k < b; ++k) *p++ = vbytes[k];
            *p++ = (j + 1 == ntok) ? '\n' : ' ';
        }
    }
}

__global__ void synth_kv_kernel(u64 seed, u64 n, u64 n_keys, ulonglong2 *__restrict__ out) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 r = splitmix64(seed + i);
        u64 key = (r % n_keys) * 0x9E3779B97F4A7C15ULL;
        u64 r2 = splitmix64(r ^ 0x5851F42D4C957F2DULL);
        long long val = (long long)(r2 % 2000ULL) - 1000LL;
        out[i] = make_ulonglong2(key, (u64)val);
    }
}

// group offsets of a key-sorted kv into a device array (G+1 entries, last = n)
static int device_group_offsets(dampr_ctx *ctx, dampr_kv *kv, DevBuf &offs, u64 *G) {
    const u64 n = kv->n;
    *G = 0;
    if (n == 0) {
        CUDA_TRY(ctx, offs.alloc(8));
        return DAMPR_OK;
    }
    const u64 ntiles = (n + 4095) / 4096;
    DevBuf d_cnt, d_base;
    CUDA_TRY(ctx, d_cnt.alloc(ntiles * 4));
    CUDA_TRY(ctx, d_base.alloc((ntiles + 1) * 8));
    {
        ScopedTimer tm(ctx, DAMPR_K_JOIN);
        heads_count_kernel<<<(unsigned)ntiles, 512, 0, ctx->stream>>>(kv->rec, n, (u32 *)d_cnt.p);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        scan_tiles_kernel<<<1, 1024, 0, ctx->stream>>>((const u32 *)d_cnt.p, (u64 *)d_base.p, (u32)ntiles);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    u64 total = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&total, (u64 *)d_base.p + ntiles, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(ctx, offs.alloc((total + 1) * 8));
    {
        ScopedTimer tm(ctx, DAMPR_K_JOIN);
        heads_write_kernel<<<(unsigned)ntiles, 512, 0, ctx->stream>>>(kv->rec, n, (const u64 *)d_base.p, (u64 *)offs.p);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *G = total;
    return DAMPR_OK;
}

}  // namespace

extern "C" {

int32_t dampr_kv_upload_columns(dampr_ctx *ctx, dampr_kv *kv, uint64_t off, const uint64_t *keys,
                                const uint64_t *vals, uint64_t count) {
    ARG_CHECK(ctx, ctx && kv && (keys || count == 0), "null");
    ARG_CHECK(ctx, off + count <= kv->capacity, "upload exceeds kv capacity");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    if (count && count * 8 >= (8u << 20) && !host_is_pinned(keys) && !(vals && host_is_pinned(vals))) {
        // pageable columns: the copy threads interleave them on their way into the page-locked ring
        int rc = staged_h2d_columns(ctx, kv->rec + off, (const u64 *)keys, (const u64 *)vals, count, ctx->copy);
        if (rc) return rc;
    } else if (count) {
        const int slot = ctx->up_tmp_next;
        ctx->up_tmp_next ^= 1;
        if (!ctx->up_tmp_ev[slot]) CUDA_TRY(ctx, cudaEventCreateWithFlags(&ctx->up_tmp_ev[slot], cudaEventDisableTiming));
        CUDA_TRY(ctx, cudaEventSynchronize(ctx->up_tmp_ev[slot]));  // the interleave kernel that last read this block
        if (ctx->up_tmp_bytes[slot] < count * 16) {
            if (ctx->up_tmp[slot]) cudaFree(ctx->up_tmp[slot]);
            ctx->up_tmp[slot] = nullptr;
            ctx->up_tmp_bytes[slot] = 0;
            CUDA_TRY(ctx, cudaMalloc(&ctx->up_tmp[slot], count * 16));
            ctx->up_tmp_bytes[slot] = count * 16;
        }
        u64 *tmp = (u64 *)ctx->up_tmp[slot];
        int rc = staged_h2d(ctx, tmp, keys, count * 8, ctx->copy);
        if (rc == DAMPR_OK && vals) rc = staged_h2d(ctx, tmp + count, vals, count * 8, ctx->copy);
        if (rc) return rc;
        ctx->launches++;
        interleave_kernel<<<ctx->num_sms * 4, 256, 0, ctx->copy>>>(tmp, vals ? tmp + count : nullptr, kv->rec + off, count);
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaEventRecord(ctx->up_tmp_ev[slot], ctx->copy));
    }
    if (off + count > kv->n) kv->n = off + count;
    CUDA_TRY(ctx, cudaEventRecord(ctx->upload_done, ctx->copy));
    ctx->upload_pending = true;
    return DAMPR_OK;
}

int32_t dampr_kv_download_columns(dampr_ctx *ctx, dampr_kv *kv, uint64_t off, uint64_t *keys,
                                  uint64_t *vals, uint64_t count) {
    ARG_CHECK(ctx, ctx && kv, "null");
    ARG_CHECK(ctx, off + count <= kv->n, "download exceeds kv size");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    if (count == 0) return DAMPR_OK;
    u64 *tmp = (u64 *)pool_alloc(ctx, count * 16);
    ARG_CHECK(ctx, tmp != nullptr, "device allocation failed");
    ctx->launches++;
    deinterleave_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(kv->rec + off, tmp, tmp + count, count);
    CUDA_TRY(ctx, cudaGetLastError());
    int rc = DAMPR_OK;
    if (keys) rc = staged_d2h(ctx, keys, tmp, count * 8, ctx->stream);
    if (rc == DAMPR_OK && vals) rc = staged_d2h(ctx, vals, tmp + count, count * 8, ctx->stream);
    if (rc == DAMPR_OK && !(keys || vals)) CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    pool_free(ctx, tmp);
    if (rc) return rc;
    return DAMPR_OK;
}

int32_t dampr_kv_join_ranges(dampr_ctx *ctx, dampr_kv *left_sorted, dampr_kv *right_sorted, int32_t key_xf,
                             uint64_t *rows, uint64_t cap, uint64_t *n_rows) {
    ARG_CHECK(ctx, ctx && left_sorted && right_sorted && n_rows, "null");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    DevBuf lo, ro;
    u64 GL = 0, GR = 0;
    int rc = device_group_offsets(ctx, left_sorted, lo, &GL);
    if (rc) return rc;
    *n_rows = GL;
    if (!rows) return DAMPR_OK;  // phase 1
    ARG_CHECK(ctx, cap >= GL, "rows array too small");
    if (GL == 0) return DAMPR_OK;
    rc = device_group_offsets(ctx, right_sorted, ro, &GR);
    if (rc) return rc;
    DevBuf d_rows;
    CUDA_TRY(ctx, d_rows.alloc(GL * 32));
    {
        ScopedTimer tm(ctx, DAMPR_K_JOIN);
        join_ranges_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(left_sorted->rec, (const u64 *)lo.p, GL,
                                                                     left_sorted->n, right_sorted->rec,
                                                                     (const u64 *)ro.p, GR, right_sorted->n, key_xf,
                                                                     (u64 *)d_rows.p);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(rows, d_rows.p, GL * 32, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return DAMPR_OK;
}

int32_t dampr_kv_hash_probe(dampr_ctx *ctx, dampr_kv *build, dampr_kv *probe, dampr_kv **out_vals,
                            uint8_t *out_hit_host) {
    ARG_CHECK(ctx, ctx && build && probe && out_vals && out_hit_host, "null");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    int rc = dampr_kv_create(ctx, probe->n, out_vals);
    if (rc) return rc;
    (*out_vals)->n = probe->n;
    if (probe->n == 0) return DAMPR_OK;
    u64 cap = 1024;
    while (cap < 2 * build->n) cap <<= 1;
    DevBuf tk, tv, used, hit;
    CUDA_TRY(ctx, tk.alloc(cap * 8));
    CUDA_TRY(ctx, tv.alloc(cap * 8));
    CUDA_TRY(ctx, used.alloc(cap * 4));
    CUDA_TRY(ctx, hit.alloc(probe->n));
    CUDA_TRY(ctx, cudaMemsetAsync(used.p, 0, cap * 4, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scratch, 0, 8, ctx->stream));
    {
        ScopedTimer tm(ctx, DAMPR_K_PROBE);
        if (build->n)
            probe_build_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(build->rec, build->n, (u64 *)tk.p, (u64 *)tv.p,
                                                                         (u32 *)used.p, cap - 1, ctx->d_scratch);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_PROBE);
        probe_lookup_kernel<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(probe->rec, probe->n, (const u64 *)tk.p,
                                                                      (const u64 *)tv.p, (const u32 *)used.p, cap - 1,
                                                                      (*out_vals)->rec, (u8 *)hit.p);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(out_hit_host, hit.p, probe->n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return DAMPR_OK;
}

int32_t dampr_kv_hash_join(dampr_ctx *ctx, dampr_kv *build, dampr_kv *probe, dampr_kv **out_probe,
                           dampr_kv **out_build) {
    ARG_CHECK(ctx, ctx && build && probe && out_probe && out_build, "null");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    *out_probe = *out_build = nullptr;
    const u64 n = probe->n;
    if (n == 0) {
        int rc = dampr_kv_create(ctx, 0, out_probe);
        if (rc) return rc;
        return dampr_kv_create(ctx, 0, out_build);
    }
    u64 cap = 1024;
    while (cap < 2 * build->n) cap <<= 1;
    const u64 ntiles = (n + HC_TILE - 1) / HC_TILE;
    DevBuf tk, tv, used, hit, vals, tcnt, tbase;
    CUDA_TRY(ctx, tk.alloc(cap * 8));
    CUDA_TRY(ctx, tv.alloc(cap * 8));
    CUDA_TRY(ctx, used.alloc(cap * 4));
    CUDA_TRY(ctx, hit.alloc(n + 8));
    CUDA_TRY(ctx, vals.alloc(n * 16));
    CUDA_TRY(ctx, tcnt.alloc(ntiles * 4));
    CUDA_TRY(ctx, tbase.alloc((ntiles + 1) * 8));
    CUDA_TRY(ctx, cudaMemsetAsync(used.p, 0, cap * 4, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scratch, 0, 8, ctx->stream));
    {
        ScopedTimer tm(ctx, DAMPR_K_PROBE);
        if (build->n)
            probe_build_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(build->rec, build->n, (u64 *)tk.p, (u64 *)tv.p,
                                                                         (u32 *)used.p, cap - 1, ctx->d_scratch);
        probe_lookup_kernel<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(probe->rec, n, (const u64 *)tk.p, (const u64 *)tv.p,
                                                                      (const u32 *)used.p, cap - 1, (ulonglong2 *)vals.p,
                                                                      (u8 *)hit.p);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_JOIN);
        hits_count_kernel<<<(unsigned)ntiles, HC_THREADS, 0, ctx->stream>>>((const u8 *)hit.p, n, (u32 *)tcnt.p);
        scan_tiles_kernel<<<1, 1024, 0, ctx->stream>>>((const u32 *)tcnt.p, (u64 *)tbase.p, (u32)ntiles);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scratch, (u64 *)tbase.p + ntiles, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    const u64 m = ctx->h_scratch[0];
    int rc = dampr_kv_create(ctx, m, out_probe);
    if (rc) return rc;
    rc = dampr_kv_create(ctx, m, out_build);
    if (rc) {
        dampr_kv_destroy(ctx, *out_probe);
        *out_probe = nullptr;
        return rc;
    }
    (*out_probe)->n = (*out_build)->n = m;
    if (m) {
        ScopedTimer tm(ctx, DAMPR_K_JOIN);
        hits_compact_kernel<<<(unsigned)ntiles, HC_THREADS, 0, ctx->stream>>>(probe->rec, (const ulonglong2 *)vals.p,
                                                                            (const u8 *)hit.p, n, (const u64 *)tbase.p,
                                                                            (*out_probe)->rec, (*out_build)->rec);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

int32_t dampr_synth_text(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t seed, uint64_t n_lines,
                         const uint8_t *vocab_bytes, const uint32_t *vocab_off, uint32_t vocab_n,
                         const uint64_t *cdf, uint64_t *out_nbytes) {
    ARG_CHECK(ctx, ctx && tb && vocab_bytes && vocab_off && cdf && out_nbytes && vocab_n > 0, "null");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    DevBuf d_vb, d_vo, d_cdf, d_len, d_off;
    const u64 vbytes = vocab_off[vocab_n];
    CUDA_TRY(ctx, d_vb.alloc(vbytes));
    CUDA_TRY(ctx, d_vo.alloc((vocab_n + 1) * 4));
    CUDA_TRY(ctx, d_cdf.alloc((u64)vocab_n * 8));
    CUDA_TRY(ctx, d_len.alloc(n_lines * 4));
    CUDA_TRY(ctx, d_off.alloc((n_lines + 1) * 8));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_vb.p, vocab_bytes, vbytes, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_vo.p, vocab_off, (vocab_n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_cdf.p, cdf, (u64)vocab_n * 8, cudaMemcpyHostToDevice, ctx->stream));
    {
        ScopedTimer tm(ctx, DAMPR_K_SYNTH);
        synth_len_kernel<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(seed, n_lines, (const u32 *)d_vo.p, vocab_n,
                                                                   (const u64 *)d_cdf.p, (u32 *)d_len.p);
    }
    // exclusive scan in blocks of 2^31 lines is not needed: n_lines fits u32 for every config here
    ARG_CHECK(ctx, n_lines < 0xFFFFFFFFULL, "too many lines");
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        scan_tiles_kernel<<<1, 1024, 0, ctx->stream>>>((const u32 *)d_len.p, (u64 *)d_off.p, (u32)n_lines);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    u64 total = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&total, (u64 *)d_off.p + n_lines, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    ARG_CHECK(ctx, total + 128 <= tb->capacity, "textbuf too small for the synthetic text");
    {
        ScopedTimer tm(ctx, DAMPR_K_SYNTH);
        synth_write_kernel<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(seed, n_lines, (const u8 *)d_vb.p, (const u32 *)d_vo.p,
                                                                     vocab_n, (const u64 *)d_cdf.p, (const u64 *)d_off.p,
                                                                     tb->text);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    // pad to a multiple of 64 bytes by extending the last line with the words "a" / "aa"
    u64 pad = (64 - (total % 64)) % 64;
    if (pad == 1) pad = 65;
    if (pad && total > 0) {
        std::string tail;
        u64 left = pad;
        while (left > 0) {
            if (left == 3) {
                tail += " aa";
                left -= 3;
            } else {
                tail += " a";
                left -= 2;
            }
        }
        tail += "\n";
        // overwrite the final '\n' and append
        CUDA_TRY(ctx, cudaMemcpyAsync(tb->text + total - 1, tail.data(), tail.size(), cudaMemcpyHostToDevice, ctx->stream));
        total += pad;
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *out_nbytes = total;
    int rc = dampr_textbuf_set_length(ctx, tb, total);
    if (rc) return rc;
    return dampr_ctx_sync(ctx);
}

int32_t dampr_synth_kv(dampr_ctx *ctx, dampr_kv *kv, uint64_t seed, uint64_t n, uint64_t n_keys) {
    ARG_CHECK(ctx, ctx && kv && n_keys > 0, "null");
    ARG_CHECK(ctx, n <= kv->capacity, "kv too small");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    {
        ScopedTimer tm(ctx, DAMPR_K_SYNTH);
        synth_kv_kernel<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(seed, n, n_keys, kv->rec);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    kv->n = n;
    return DAMPR_OK;
}

// download a byte range of a text buffer (synthetic text -> host for the e2e / CPU legs)
int32_t dampr_textbuf_download(dampr_ctx *ctx, dampr_textbuf *tb, uint64_t off, void *host, uint64_t len) {
    ARG_CHECK(ctx, ctx && tb && (host || len == 0), "null");
    ARG_CHECK(ctx, off + len <= tb->n, "download exceeds text length");
    wait_uploads(ctx);
    if (len) CUDA_TRY(ctx, cudaMemcpyAsync(host, tb->text + off, len, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return DAMPR_OK;
}

}  // extern "C"

// ---- a lowered numeric lambda over the distinct values of an int64 column (host) ----------------------------------
// The cross of a frame with a one-row broadcast evaluates the user's function once per distinct value of the field it
// reads (plan._lower_cross). For expressions of + - * / neg, float() and math.log over that field, int and float
// constants and the broadcast value, plan.py compiles the tree into this postfix program, typed the way CPython types
// it. Every operation is the IEEE double operation CPython performs (the library is built without contraction or
// fast-math, and log is the C library's, which math.log calls for a finite positive argument), so the results are
// CPython's to the bit. Wherever CPython would raise or take another road (a zero divisor, a log argument that is not
// finite and positive, an int leaving int64, an int true division beyond 2^53) the call returns
// DAMPR_ERR_UNSUPPORTED and the caller evaluates the function in Python instead.
#include <cmath>

namespace {
// (the opcodes, EvalOp, are common.cuh's: the field scans' programs share them)
union EvalSlot {
    long long i;
    double f;
};
}  // namespace

extern "C" int32_t dampr_host_eval_f64(const int64_t *vals, uint64_t n, const int32_t *prog, uint32_t prog_len,
                                       const int64_t *ci, const double *cf, double *out) {
    if ((!vals || !out) && n) return DAMPR_ERR_ARG;
    if (!prog || prog_len == 0 || prog_len > 256) return DAMPR_ERR_ARG;
    // the program is checked once: every operation finds its operands, one value is left
    int depth = 0;
    for (uint32_t pc = 0; pc < prog_len; ++pc) {
        const int32_t op = prog[pc] & 0xFF;
        const bool push = op <= EV_CF, unary = op == EV_I2F || op == EV_LOG || op == EV_INEG || op == EV_FNEG;
        if (op > EV_FNEG || depth < (push ? 0 : unary ? 1 : 2)) return DAMPR_ERR_ARG;
        depth += push ? 1 : unary ? 0 : -1;
        if (depth > 64) return DAMPR_ERR_ARG;
    }
    if (depth != 1) return DAMPR_ERR_ARG;
    const long long LIM53 = 1LL << 53;
    EvalSlot st[64];
    for (uint64_t r = 0; r < n; ++r) {
        int sp = 0;
        for (uint32_t pc = 0; pc < prog_len; ++pc) {
            const int32_t op = prog[pc] & 0xFF, arg = prog[pc] >> 8;
            EvalSlot &a = st[sp >= 2 ? sp - 2 : 0], &b = st[sp >= 1 ? sp - 1 : 0];
            switch (op) {
                case EV_X: st[sp++].i = vals[r]; break;
                case EV_CI: st[sp++].i = ci[arg]; break;
                case EV_CF: st[sp++].f = cf[arg]; break;
                case EV_I2F: b.f = (double)b.i; break;
                case EV_IADD: if (__builtin_add_overflow(a.i, b.i, &a.i)) return DAMPR_ERR_UNSUPPORTED; --sp; break;
                case EV_ISUB: if (__builtin_sub_overflow(a.i, b.i, &a.i)) return DAMPR_ERR_UNSUPPORTED; --sp; break;
                case EV_IMUL: if (__builtin_mul_overflow(a.i, b.i, &a.i)) return DAMPR_ERR_UNSUPPORTED; --sp; break;
                case EV_FADD: a.f = a.f + b.f; --sp; break;
                case EV_FSUB: a.f = a.f - b.f; --sp; break;
                case EV_FMUL: a.f = a.f * b.f; --sp; break;
                case EV_FDIV:
                    if (b.f == 0.0) return DAMPR_ERR_UNSUPPORTED;
                    a.f = a.f / b.f;
                    --sp;
                    break;
                case EV_IDIV:
                    if (b.i == 0 || a.i > LIM53 || a.i < -LIM53 || b.i > LIM53 || b.i < -LIM53) return DAMPR_ERR_UNSUPPORTED;
                    a.f = (double)a.i / (double)b.i;
                    --sp;
                    break;
                case EV_LOG:
                    if (!(b.f > 0.0) || !std::isfinite(b.f)) return DAMPR_ERR_UNSUPPORTED;
                    b.f = log(b.f);
                    break;
                case EV_INEG: if (b.i == INT64_MIN) return DAMPR_ERR_UNSUPPORTED; b.i = -b.i; break;
                case EV_FNEG: b.f = -b.f; break;
                default: return DAMPR_ERR_ARG;
            }
        }
        out[r] = st[0].f;
    }
    return DAMPR_OK;
}

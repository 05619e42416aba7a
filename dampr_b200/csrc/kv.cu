// kv.cu — K3/K4: radix partition, in-partition sort, segmented reduce over 16-byte records.
//
// Replaces the reference's shuffle/sort/reduce for (key, value) records:
//   Splitter.partition            dampr/base.py:6-8          hash(key) % n_partitions
//   CSDatasetWriter.flush         dampr/dataset.py:236-253   route every record to its partition
//   SortedWriter._write_to_gzip   dampr/dataset.py:162-164   list.sort(key=itemgetter(0)) (stable)
//   Dataset.grouped_read          dampr/dataset.py:429-433   group adjacent equal keys
//   ARReduce._reduce / Reduce     dampr/dampr.py:678-683, dampr/base.py:204-207  fold a group
// (the k-way merge of sorted runs, MergeDataset.read dataset.py:571-579, lives in merge.cu)
//
// Design, second generation:
//   * ONE partition level of up to 12 key bits (4096 buckets) for up to ~1.1e8 records, then one
//     leaf pass: two data passes instead of three.  A level is histogram -> scans -> scatter over
//     per-CTA contiguous record ranges ("pieces"), so a bucket receives its records in input order
//     (stable) and nothing but the per-piece histogram touches HBM with atomics.
//   * scatter: every record takes its rank inside (tile, bucket) from ONE shared-memory atomic; the
//     arbitrary order the atomics hand out is repaired by ranking each record among the (one or two)
//     tile mates of its bucket by tile index; long runs (skew) are sorted by a warp through a presence
//     bitmap.  No per-warp histograms, no ballots per digit bit: the per-tile cost no longer grows with
//     warps x buckets, which is what allows 12 bits.
//   * leaf: a thread-block CLUSTER of 8 CTAs sorts a whole ~24K-record bucket.  Each CTA loads 1/8 of
//     the bucket, the 8 CTAs agree on a 256-bin histogram through distributed shared memory, every
//     record is stored straight into the shared memory of the CTA that owns its bin
//     (st.shared::cluster), and each CTA finishes with a counting sort + rank-by-(key, original index)
//     of its ~3K records.  Segments of at most 4096 records use the single-CTA leaf.
//   * segmented reduce (SUM/COUNT/MIN/MAX/FIRST/LAST) is fused into both leaves.
#include <algorithm>
#include <cooperative_groups.h>

#include "common.cuh"
#include "leaf.cuh"

namespace cg = cooperative_groups;

int g_kv_scatter = 1;   // 1 = staged runs ranked by ballots, TMA bulk stores, 10 bits per level (default: fastest measured);
                        // 3 = staged runs ranked by one atomic + SWAR compares; 2 = 12-bit table scatter for the first level
int g_kv_hist = 2;      // 2 = unrolled histogram, several CTAs per piece (default); 1 = first generation
int g_kv_cluster = 0;   // 1 = cluster/DSMEM leaf for segments above one CTA's capacity (measured slower, see DESIGN.md)
int g_kv_hints = 1;     // L2 eviction-priority hints in the table scatter (evict-first loads, evict-last stores)
int g_kv_max_bits = 12; // digit bits of the table scatter's level (kv_scatter = 2)

namespace {

// ---- first-generation scatter (kept selectable for A/B measurements) ---------------------------
constexpr int P_THREADS = 512;
constexpr int P_WARPS = P_THREADS / 32;
constexpr int P_TILE = 4096;                 // records per tile
constexpr int P_PER_WARP = P_TILE / P_WARPS;  // 256
constexpr int P_ROUNDS = P_PER_WARP / 32;     // 8
constexpr int P1_MAX_BITS = 10;
constexpr int P1_MAX_NB = 1 << P1_MAX_BITS;

// ---- second generation ---------------------------------------------------------------------------
constexpr int P2_MAX_BITS = 12;
constexpr int P2_MAX_NB = 1 << P2_MAX_BITS;
constexpr int HOT_L = 32;  // (tile, bucket) runs longer than this are sorted by a warp


constexpr u64 C_NMAX = 27500;   // records per cluster chunk (8 x 4096 minus slack for bin granularity)
constexpr u64 C_TARGET = 25000; // planned average segment size when the cluster leaf is in use
constexpr u64 S_TARGET = 2600;  // planned average segment size for single-CTA leaves
int g_kv_leaf_target = (int)S_TARGET;   // (dampr_set_option "kv_leaf_target": experiments with more, smaller segments)

struct Piece {
    u64 start, end;
    u32 seg;
    u32 pad;
};

struct DigitSpec {
    int xf;     // key transform
    u64 base;   // subtracted after the transform
    int shift;  // digit = ((xf(key) - base) >> shift) & mask
    u32 mask;
    int owner_mod;  // if > 0: digit = mix64(key) % owner_mod (exchange partition)
};

__device__ __forceinline__ u32 digit_of(u64 key, const DigitSpec &d) {
    if (d.owner_mod > 0) return (u32)(mix64(key) % (u64)d.owner_mod);
    return (u32)(((key_xform(key, d.xf) - d.base) >> d.shift) & d.mask);
}

// piece p of a uniform decomposition (no descriptor array: used by the single-segment level)
__device__ __forceinline__ Piece uniform_piece(u32 p, u64 start, u64 n, u64 R) {
    Piece pc;
    pc.start = start + min(n, (u64)p * R);
    pc.end = start + min(n, (u64)(p + 1) * R);
    pc.seg = 0;
    pc.pad = 0;
    return pc;
}

// ---- level histogram (v1) -----------------------------------------------------------------------
__global__ void __launch_bounds__(P_THREADS)
part_hist_kernel(const ulonglong2 *__restrict__ in, const Piece *__restrict__ pieces,
                 const u32 *__restrict__ cta_piece_begin, DigitSpec ds, u32 nb,
                 u32 *__restrict__ piece_hist) {
    __shared__ u32 sh[P1_MAX_NB];
    const u32 pb = cta_piece_begin[blockIdx.x], pe = cta_piece_begin[blockIdx.x + 1];
    for (u32 p = pb; p < pe; ++p) {
        for (u32 b = threadIdx.x; b < nb; b += blockDim.x) sh[b] = 0;
        __syncthreads();
        const Piece pc = pieces[p];
        for (u64 i = pc.start + threadIdx.x; i < pc.end; i += blockDim.x) {
            u64 key = in[i].x;
            atomicAdd(&sh[digit_of(key, ds)], 1u);
        }
        __syncthreads();
        for (u32 b = threadIdx.x; b < nb; b += blockDim.x) piece_hist[(u64)p * nb + b] = sh[b];
        __syncthreads();
    }
}

// ---- level histogram (v2): HS CTAs per piece, 8 keys in flight per thread, folded into the piece
// histogram (and the bucket totals when `tot` is given) with global reductions ----------------------
constexpr int H2_THREADS = 1024;
constexpr int H2_UNROLL = 8;
__global__ void __launch_bounds__(H2_THREADS, 2)
part_hist2_kernel(const ulonglong2 *__restrict__ in, const Piece *__restrict__ pieces, u64 ustart, u64 un,
                  u64 uR, u32 hs, DigitSpec ds, u32 nb, u32 *__restrict__ piece_hist,
                  u32 *__restrict__ tot) {
    __shared__ u32 sh[P2_MAX_NB];
    const u32 p = blockIdx.x / hs, sub = blockIdx.x % hs;
    const Piece pc = pieces ? pieces[p] : uniform_piece(p, ustart, un, uR);
    const u64 len = pc.end - pc.start;
    const u64 per = ((len + hs - 1) / hs + 15) & ~15ULL;
    const u64 lo = pc.start + min(len, (u64)sub * per), hi = pc.start + min(len, (u64)(sub + 1) * per);
    for (u32 b = threadIdx.x; b < nb; b += H2_THREADS) sh[b] = 0;
    __syncthreads();
    u64 i = lo + threadIdx.x;
    for (; i + (u64)(H2_UNROLL - 1) * H2_THREADS < hi; i += (u64)H2_UNROLL * H2_THREADS) {
        u64 k[H2_UNROLL];
#pragma unroll
        for (int u = 0; u < H2_UNROLL; ++u) k[u] = in[i + (u64)u * H2_THREADS].x;
#pragma unroll
        for (int u = 0; u < H2_UNROLL; ++u) atomicAdd(&sh[digit_of(k[u], ds)], 1u);
    }
    for (; i < hi; i += H2_THREADS) atomicAdd(&sh[digit_of(in[i].x, ds)], 1u);
    __syncthreads();
    for (u32 b = threadIdx.x; b < nb; b += H2_THREADS) {
        const u32 c = sh[b];
        if (hs == 1) piece_hist[(u64)p * nb + b] = c;
        else if (c) atomicAdd(&piece_hist[(u64)p * nb + b], c);
        if (tot && c) atomicAdd(&tot[b], c);
    }
}

// ---- per-segment scan (general levels): bucket bases, per-piece offsets, next-level offsets ------
// one CTA of 1024 threads per segment, nb <= 4096 (up to 4 buckets per thread)
__global__ void __launch_bounds__(1024)
part_scan_kernel(const u32 *__restrict__ piece_hist, const u32 *__restrict__ seg_piece_begin,
                 const u64 *__restrict__ seg_off, u32 nb, u64 *__restrict__ piece_off,
                 u64 *__restrict__ next_seg_off) {
    __shared__ u64 wsum[32];
    const u32 s = blockIdx.x;
    const u32 bpt = (nb + 1023) / 1024;
    const u32 b0 = threadIdx.x * bpt;
    const u32 pb = seg_piece_begin[s], pe = seg_piece_begin[s + 1];
    u64 tot[4] = {0, 0, 0, 0};
    for (u32 p = pb; p < pe; ++p)
        for (u32 j = 0; j < bpt; ++j)
            if (b0 + j < nb) tot[j] += piece_hist[(u64)p * nb + b0 + j];
    u64 sum = tot[0] + tot[1] + tot[2] + tot[3];
    u64 v = sum;
    for (int d = 1; d < 32; d <<= 1) {
        u64 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((int)(threadIdx.x & 31) >= d) v += o;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    u64 woff = 0;
    for (u32 w = 0; w < (threadIdx.x >> 5); ++w) woff += wsum[w];
    u64 run = seg_off[s] + woff + v - sum;
    for (u32 j = 0; j < bpt; ++j) {
        if (b0 + j >= nb) break;
        next_seg_off[(u64)s * nb + b0 + j] = run;
        u64 r2 = run;
        for (u32 p = pb; p < pe; ++p) {
            u32 h = piece_hist[(u64)p * nb + b0 + j];
            piece_off[(u64)p * nb + b0 + j] = r2;
            r2 += h;
        }
        run += tot[j];
    }
}

// ---- single-segment level: exclusive scan of the bucket totals (one CTA) ... ----------------------
__global__ void __launch_bounds__(1024)
bucket_scan_kernel(const u32 *__restrict__ tot, u32 nb, u64 start, u64 n, u64 *__restrict__ seg_off) {
    __shared__ u64 wsum[32];
    const u32 bpt = (nb + 1023) / 1024;
    const u32 b0 = threadIdx.x * bpt;
    u64 t[4] = {0, 0, 0, 0};
    for (u32 j = 0; j < bpt; ++j)
        if (b0 + j < nb) t[j] = tot[b0 + j];
    u64 sum = t[0] + t[1] + t[2] + t[3];
    u64 v = sum;
    for (int d = 1; d < 32; d <<= 1) {
        u64 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((int)(threadIdx.x & 31) >= d) v += o;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    u64 woff = 0;
    for (u32 w = 0; w < (threadIdx.x >> 5); ++w) woff += wsum[w];
    u64 run = start + woff + v - sum;
    for (u32 j = 0; j < bpt; ++j) {
        if (b0 + j >= nb) break;
        seg_off[b0 + j] = run;
        run += t[j];
    }
    if (threadIdx.x == 0) seg_off[nb] = start + n;
}

// ---- ... and the per-piece offsets inside every bucket: 32 buckets (lanes) x 32 piece groups (warps)
// per CTA, so both passes over the piece histogram are coalesced --------------------------------------
__global__ void __launch_bounds__(1024)
column_offsets_kernel(const u32 *__restrict__ piece_hist, u32 np, u32 nb, const u64 *__restrict__ seg_off,
                      u64 *__restrict__ piece_off) {
    __shared__ u64 wtot[32][33];
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const u32 b = blockIdx.x * 32 + lane;
    const u32 pg = (np + 31) / 32;
    const u32 p0 = min(np, w * pg), p1 = min(np, (w + 1) * pg);
    u64 sum = 0;
    if (b < nb)
        for (u32 p = p0; p < p1; ++p) sum += piece_hist[(u64)p * nb + b];
    wtot[w][lane] = sum;
    __syncthreads();
    u64 run = 0;
    for (u32 k = 0; k < w; ++k) run += wtot[k][lane];
    if (b < nb) {
        run += seg_off[b];
        for (u32 p = p0; p < p1; ++p) {
            const u32 h = piece_hist[(u64)p * nb + b];
            piece_off[(u64)p * nb + b] = run;
            run += h;
        }
    }
}

// ---- level scatter (v1: ballots per digit bit, per-warp histograms, TMA bulk stores) --------------
struct ScatterSmem {
    alignas(16) ulonglong2 stage[P_TILE];
    u64 run_off[P1_MAX_NB];
    u16 warp_hist[P_WARPS][P1_MAX_NB];
    u32 local_base[P1_MAX_NB + 1];
    u32 tile_cnt[P1_MAX_NB];
    u32 wsum[32];
};

// clear the first 2^dbits counters of every warp's row, two 16-bit counters per store, shifts instead of the
// division by the (run-time) bucket count the first version paid eight times per thread and tile
__device__ __forceinline__ void zero_warp_hist(ScatterSmem &s, u32 dbits) {
    const u32 wpr = max(1u, (1u << dbits) >> 1);   // 32-bit words per row
    const u32 wshift = dbits ? dbits - 1 : 0;
    for (u32 i = threadIdx.x; i < P_WARPS * wpr; i += P_THREADS)
        reinterpret_cast<u32 *>(s.warp_hist[i >> wshift])[i & (wpr - 1)] = 0;
}

template <bool USE_TMA>
__global__ void __launch_bounds__(P_THREADS, 2)
part_scatter_kernel(const ulonglong2 *__restrict__ in, ulonglong2 *__restrict__ out,
                    const Piece *__restrict__ pieces, const u32 *__restrict__ cta_piece_begin, u64 ustart, u64 un,
                    u64 uR, DigitSpec ds, u32 nb, const u64 *__restrict__ piece_off) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ScatterSmem &s = *reinterpret_cast<ScatterSmem *>(smem_raw);
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 pb = pieces ? cta_piece_begin[blockIdx.x] : blockIdx.x;
    const u32 pe = pieces ? cta_piece_begin[blockIdx.x + 1] : blockIdx.x + 1;
    u32 dbits = 0;
    while ((1u << dbits) < nb) ++dbits;

    for (u32 p = pb; p < pe; ++p) {
        const Piece pc = pieces ? pieces[p] : uniform_piece(p, ustart, un, uR);
        for (u32 b = tid; b < nb; b += P_THREADS) s.run_off[b] = piece_off[(u64)p * nb + b];
        // the per-warp histograms are cleared here for the first tile and, for every later one, next to the
        // stores of the tile before it (they are dead once the records are staged): no barrier of their own
        zero_warp_hist(s, dbits);
        __syncthreads();
        for (u64 t0 = pc.start; t0 < pc.end; t0 += P_TILE) {
            const u32 tn = (u32)min((u64)P_TILE, pc.end - t0);
            ulonglong2 rec[P_ROUNDS];
            u32 dig[P_ROUNDS];
            u32 rnk[P_ROUNDS];
#pragma unroll
            for (int r = 0; r < P_ROUNDS; ++r) {
                u32 li = warp * P_PER_WARP + r * 32 + lane;
                if (li < tn) rec[r] = in[t0 + li];
            }
            if (t0 + P_TILE < pc.end) {
                const char *nxt = reinterpret_cast<const char *>(in + t0 + P_TILE);
                const u32 nbytes = (u32)min((u64)P_TILE, pc.end - t0 - P_TILE) * 16u;
                if (tid * 128u < nbytes) asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt + tid * 128u));
            }
            // Per round one packed word: digit (10 bits) | leader lane << 10 | rank among the set's lanes << 15
            // | (set size - 1) << 20 | valid << 25.
#pragma unroll
            for (int r = 0; r < P_ROUNDS; ++r) {
                const u32 li = warp * P_PER_WARP + r * 32 + lane;
                const bool valid = li < tn;
                const u32 vmask = __ballot_sync(0xFFFFFFFFu, valid);
                const u32 d = valid ? digit_of(rec[r].x, ds) : 0u;
                u32 peers = vmask;
                for (u32 bit = 0; bit < dbits; ++bit) {
                    const u32 mine = (d >> bit) & 1u;
                    const u32 bal = __ballot_sync(0xFFFFFFFFu, mine);
                    peers &= mine ? bal : ~bal;
                }
                dig[r] = valid ? (d | (((u32)__ffs(peers) - 1u) << 10) | ((u32)__popc(peers & ((1u << lane) - 1u)) << 15) |
                                  (((u32)__popc(peers) - 1u) << 20) | (1u << 25))
                               : 0u;
            }
            u32 *wh32 = reinterpret_cast<u32 *>(s.warp_hist[warp]);
#pragma unroll
            for (int r = 0; r < P_ROUNDS; ++r) {
                const u32 pk = dig[r];
                rnk[r] = 0;
                if ((pk >> 25) && ((pk >> 10) & 31u) == lane) {
                    const u32 d = pk & 1023u, c = ((pk >> 20) & 31u) + 1u;
                    const u32 w = atomicAdd(&wh32[d >> 1], (d & 1u) ? (c << 16) : c);
                    rnk[r] = (d & 1u) ? (w >> 16) : (w & 0xFFFFu);
                }
            }
#pragma unroll
            for (int r = 0; r < P_ROUNDS; ++r) {
                const u32 pk = dig[r];
                const u32 old = __shfl_sync(0xFFFFFFFFu, rnk[r], (pk >> 25) ? ((pk >> 10) & 31u) : lane);
                rnk[r] = old + ((pk >> 15) & 31u);
                dig[r] = (pk >> 25) ? (pk & 1023u) : 0xFFFFFFFFu;
            }
            __syncthreads();
            for (u32 b = tid; b < nb; b += P_THREADS) {
                u32 run = 0;
#pragma unroll
                for (int w = 0; w < P_WARPS; ++w) {
                    u32 c = s.warp_hist[w][b];
                    s.warp_hist[w][b] = (u16)run;
                    run += c;
                }
                s.tile_cnt[b] = run;
            }
            __syncthreads();
            {
                u32 c0 = (2 * tid < nb) ? s.tile_cnt[2 * tid] : 0;
                u32 c1 = (2 * tid + 1 < nb) ? s.tile_cnt[2 * tid + 1] : 0;
                u32 v = c0 + c1;
                u32 tsum = v;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                    if ((int)lane >= d) v += o;
                }
                if (lane == 31) s.wsum[warp] = v;
                __syncthreads();
                u32 woff = 0;
                for (u32 w = 0; w < warp; ++w) woff += s.wsum[w];
                u32 excl = woff + v - tsum;
                if (2 * tid < nb) s.local_base[2 * tid] = excl;
                if (2 * tid + 1 < nb) s.local_base[2 * tid + 1] = excl + c0;
            }
            __syncthreads();
#pragma unroll
            for (int r = 0; r < P_ROUNDS; ++r) {
                if (dig[r] != 0xFFFFFFFFu) {
                    u32 pos = s.local_base[dig[r]] + s.warp_hist[warp][dig[r]] + rnk[r];
                    s.stage[pos] = rec[r];
                }
            }
            if (USE_TMA) fence_proxy_async();
            __syncthreads();
            if (USE_TMA) {
                // the thread that sends a bucket's run also advances the bucket's cursor: no pass (and no
                // barrier) of its own for that
                for (u32 b = tid; b < nb; b += P_THREADS) {
                    const u32 c = s.tile_cnt[b];
                    if (c) {
                        const u64 ro = s.run_off[b];
                        tma_store_1d(out + ro, &s.stage[s.local_base[b]], c * 16u);
                        s.run_off[b] = ro + c;
                    }
                }
                tma_store_commit();
                zero_warp_hist(s, dbits);
                tma_store_wait_read();
                __syncthreads();
            } else {
                for (u32 j = tid; j < tn; j += P_THREADS) {
                    ulonglong2 rc = s.stage[j];
                    u32 d = digit_of(rc.x, ds);
                    out[s.run_off[d] + (j - s.local_base[d])] = rc;
                }
                zero_warp_hist(s, dbits);
                __syncthreads();
                for (u32 b = tid; b < nb; b += P_THREADS) s.run_off[b] += s.tile_cnt[b];
                __syncthreads();
            }
        }
    }
    if (USE_TMA) tma_store_wait_all();
}

// ---- level scatter (v2): one shared-memory atomic per record + an 8-slot index table per bucket ------
// Tile = 4096 records (512 threads x 8), up to 4096 buckets. Every record takes its (arbitrary) slot
// inside (tile, bucket) from ONE packed 16-bit shared-memory atomic and drops its tile index into the
// bucket's row of an 8-slot table; after one barrier it reads the row back with a single 16-byte load and
// ranks itself among its tile mates with SWAR halfword compares (stable: by tile index = input order),
// then stores its 16 bytes straight into the bucket's run. Two barriers per tile; the counters are
// double buffered so the bucket cursors are advanced while the next tile is already loading.
// A tile in which some bucket receives more than 8 records (fewer buckets than records per tile, skew,
// duplicates) takes the general path: exclusive scan of the tile's bucket counts, a compact index list
// per bucket, long runs sorted by a warp through a presence bitmap (O(T) per tile whatever the skew).
// Streaming loads carry an L2 evict-first policy and the scattered stores evict-last, so half-written
// sectors of the 296 x 4096 write fronts stay in L2 until their neighbours arrive (the first build,
// without hints, read 2.1x and wrote 1.5x the algorithmic bytes from DRAM: profiles/r02_kv_a_*).
constexpr int S3_NT = 512;
constexpr int S3_RPT = 8;
constexpr int S3_T = S3_NT * S3_RPT;  // 4096
constexpr int S3_W = 8;               // table slots per bucket

struct Scatter3Smem {
    u32 run_off[P2_MAX_NB];                     // cursor of every bucket, relative to the level's first record
    alignas(16) u32 cnt[2][P2_MAX_NB / 2];      // packed 16-bit counters, double buffered
    alignas(16) u16 tab[P2_MAX_NB][S3_W];       // tile indices by (bucket, slot); the general path overlays it
    u32 ovf[2];
    u32 wsum[32];
};
// overlay of the general path inside `tab` (64 KB)
struct Scatter3Slow {
    alignas(16) u32 base[P2_MAX_NB + 4];
    u32 bitmap[S3_NT / 32][S3_T / 32];
    u16 sidx[S3_T];
    u16 hot[S3_T / 32];
    u32 nhot;
};
static_assert(sizeof(Scatter3Slow) <= sizeof(u16) * P2_MAX_NB * S3_W, "slow-path overlay must fit the table");

__device__ __forceinline__ u64 l2_policy_evict_first() {
    u64 p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ u64 l2_policy_evict_last() {
    u64 p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ ulonglong2 ld_rec_hint(const ulonglong2 *p, u64 pol) {
    ulonglong2 r;
    asm volatile("ld.global.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(r.x), "=l"(r.y) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void st_rec_hint(ulonglong2 *p, const ulonglong2 &r, u64 pol) {
    asm volatile("st.global.L2::cache_hint.v2.u64 [%0], {%1, %2}, %3;" ::"l"(p), "l"(r.x), "l"(r.y), "l"(pol) : "memory");
}

template <bool HINTS>
__global__ void __launch_bounds__(S3_NT, 2)
part_scatter2_kernel(const ulonglong2 *__restrict__ in, ulonglong2 *__restrict__ out,
                     const Piece *__restrict__ pieces, const u32 *__restrict__ cta_piece_begin, u64 ustart,
                     u64 un, u64 uR, u64 out_base, DigitSpec ds, u32 nb, const u64 *__restrict__ piece_off) {
    constexpr int NT = S3_NT, RPT = S3_RPT, T = S3_T, NW = NT / 32, WPL = T / 32 / 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Scatter3Smem &s = *reinterpret_cast<Scatter3Smem *>(smem_raw);
    Scatter3Slow &sl_ = *reinterpret_cast<Scatter3Slow *>(&s.tab[0][0]);
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 pb = pieces ? cta_piece_begin[blockIdx.x] : blockIdx.x;
    const u32 pe = pieces ? cta_piece_begin[blockIdx.x + 1] : blockIdx.x + 1;
    u64 pol_in = 0, pol_out = 0;
    if (HINTS) {
        pol_in = l2_policy_evict_first();
        pol_out = l2_policy_evict_last();
    }
    ulonglong2 *const obase = out + out_base;
    u32 tile_no = 0;

    for (u32 p = pb; p < pe; ++p) {
        const Piece pc = pieces ? pieces[p] : uniform_piece(p, ustart, un, uR);
        __syncthreads();  // the previous piece's last tile is done with the cursors
        for (u32 b = tid; b < (u32)P2_MAX_NB; b += NT) s.run_off[b] = (b < nb) ? (u32)(piece_off[(u64)p * nb + b] - out_base) : 0u;
        for (u32 b = tid; b < (u32)P2_MAX_NB; b += NT) (&s.cnt[0][0])[b] = 0;  // both counter buffers
        if (tid < 2) s.ovf[tid] = 0;
        __syncthreads();
        for (u64 t0 = pc.start; t0 < pc.end; t0 += T, ++tile_no) {
            const u32 tn = (u32)min((u64)T, pc.end - t0);
            const u32 buf = tile_no & 1u;
            u32 *cnt32 = s.cnt[buf];
            ulonglong2 rec[RPT];
            u32 dsl[RPT];  // digit | slot << 16
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const u32 li = r * NT + tid;
                if (li < tn) rec[r] = HINTS ? ld_rec_hint(in + t0 + li, pol_in) : in[t0 + li];
            }
            if (t0 + T < pc.end) {  // the next tile: pull it into L2 while this one is ranked
                const char *nxt = reinterpret_cast<const char *>(in + t0 + T);
                const u32 nbytes = (u32)min((u64)T, pc.end - t0 - T) * 16u;
                for (u32 off = tid * 128u; off < nbytes; off += NT * 128u)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt + off));
            }
            bool over = false;
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const u32 li = r * NT + tid;
                dsl[r] = 0;
                if (li < tn) {
                    const u32 d = digit_of(rec[r].x, ds);
                    const u32 old = atomicAdd(&cnt32[d >> 1], (d & 1u) ? 0x10000u : 1u);
                    const u32 slot = (d & 1u) ? (old >> 16) : (old & 0xFFFFu);
                    dsl[r] = d | (slot << 16);
                    if (slot < (u32)S3_W) s.tab[d][slot] = (u16)li;
                    else over = true;
                }
            }
            if (over) s.ovf[buf] = 1;
            __syncthreads();
            if (!s.ovf[buf]) {
                // ---- fast path: rank among the <= 8 tile mates of the bucket, SWAR on halfwords -------------
                const u16 *cnt16 = reinterpret_cast<const u16 *>(cnt32);
#pragma unroll
                for (int r = 0; r < RPT; ++r) {
                    const u32 li = r * NT + tid;
                    if (li < tn) {
                        const u32 d = dsl[r] & 0xFFFFu;
                        const u32 L = cnt16[d];
                        u32 rk = 0;
                        if (L > 1) {
                            const uint4 row = *reinterpret_cast<const uint4 *>(&s.tab[d][0]);
                            const u64 lo = (u64)row.x | ((u64)row.y << 32), hi = (u64)row.z | ((u64)row.w << 32);
                            const u64 H = 0x8000800080008000ULL, lim = (u64)li * 0x0001000100010001ULL;
                            const u64 lt0 = ~((lo | H) - lim) & H, lt1 = ~((hi | H) - lim) & H;  // bit 15: entry < li
                            const u64 m0 = (L >= 4) ? ~0ULL : ((1ULL << (16 * L)) - 1ULL);
                            const u64 m1 = (L >= 8) ? ~0ULL : ((L > 4) ? ((1ULL << (16 * (L - 4))) - 1ULL) : 0ULL);
                            rk = (u32)__popcll(lt0 & m0) + (u32)__popcll(lt1 & m1);
                        }
                        ulonglong2 *dst = obase + s.run_off[d] + rk;
                        if (HINTS) st_rec_hint(dst, rec[r], pol_out);
                        else *dst = rec[r];
                    }
                }
                __syncthreads();
            } else {
                // ---- general path (the table is overlaid): scan, compact index lists, hot runs -----------------
                const u16 *cnt16 = reinterpret_cast<const u16 *>(cnt32);
                {
                    const u32 b0 = tid * 8u;
                    u32 c[8];
                    {
                        const uint4 a = *reinterpret_cast<const uint4 *>(&cnt32[b0 >> 1]);
                        c[0] = a.x & 0xFFFFu, c[1] = a.x >> 16, c[2] = a.y & 0xFFFFu, c[3] = a.y >> 16;
                        c[4] = a.z & 0xFFFFu, c[5] = a.z >> 16, c[6] = a.w & 0xFFFFu, c[7] = a.w >> 16;
                    }
                    __syncthreads();  // every thread has read its counters: the table may be overwritten
                    if (tid == 0) sl_.nhot = 0;
                    __syncthreads();
                    u32 sum = 0;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        sum += c[j];
                        if (c[j] > HOT_L) sl_.hot[atomicAdd(&sl_.nhot, 1u)] = (u16)(b0 + j);
                    }
                    u32 v = sum;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                        if ((int)lane >= d) v += o;
                    }
                    if (lane == 31) s.wsum[warp] = v;
                    __syncthreads();
                    u32 woff = 0;
                    for (u32 w = 0; w < warp; ++w) woff += s.wsum[w];
                    u32 run = woff + v - sum;
                    u32 e[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        e[j] = run;
                        run += c[j];
                    }
                    *reinterpret_cast<uint4 *>(&sl_.base[b0]) = make_uint4(e[0], e[1], e[2], e[3]);
                    *reinterpret_cast<uint4 *>(&sl_.base[b0 + 4]) = make_uint4(e[4], e[5], e[6], e[7]);
                    if (tid == NT - 1) sl_.base[P2_MAX_NB] = tn;
                }
                __syncthreads();
#pragma unroll
                for (int r = 0; r < RPT; ++r) {
                    const u32 li = r * NT + tid;
                    if (li < tn) sl_.sidx[sl_.base[dsl[r] & 0xFFFFu] + (dsl[r] >> 16)] = (u16)li;
                }
                __syncthreads();
                const u32 nh = sl_.nhot;
                if (nh) {
                    u32 *bm = sl_.bitmap[warp];
                    for (u32 hi = warp; hi < nh; hi += NW) {
                        const u32 h = sl_.hot[hi];
                        const u32 st = sl_.base[h], L = sl_.base[h + 1] - st;
                        for (u32 w = lane; w < T / 32; w += 32) bm[w] = 0;
                        __syncwarp();
                        for (u32 j = lane; j < L; j += 32) {
                            const u32 x = sl_.sidx[st + j];
                            atomicOr(&bm[x >> 5], 1u << (x & 31));
                        }
                        __syncwarp();
                        u32 words[WPL];
                        u32 cl = 0;
#pragma unroll
                        for (int k = 0; k < WPL; ++k) {
                            words[k] = bm[lane * WPL + k];
                            cl += __popc(words[k]);
                        }
                        u32 v = cl;
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                            u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                            if ((int)lane >= d) v += o;
                        }
                        u32 pos = st + v - cl;
#pragma unroll
                        for (int k = 0; k < WPL; ++k) {
                            u32 wd = words[k];
                            while (wd) {
                                const u32 bit = __ffs(wd) - 1;
                                wd &= wd - 1;
                                sl_.sidx[pos++] = (u16)((lane * WPL + k) * 32 + bit);
                            }
                        }
                        __syncwarp();
                    }
                    __syncthreads();
                }
#pragma unroll
                for (int r = 0; r < RPT; ++r) {
                    const u32 li = r * NT + tid;
                    if (li < tn) {
                        const u32 d = dsl[r] & 0xFFFFu;
                        const u32 st = sl_.base[d], L = sl_.base[d + 1] - st;
                        u32 rk = 0;
                        if (L > HOT_L) {  // sorted by a warp above: lower bound
                            u32 lo = 0, hi = L;
                            while (lo < hi) {
                                const u32 mid = (lo + hi) >> 1;
                                if (sl_.sidx[st + mid] < li) lo = mid + 1;
                                else hi = mid;
                            }
                            rk = lo;
                        } else if (L > 1) {
                            for (u32 j = 0; j < L; ++j) rk += (sl_.sidx[st + j] < li) ? 1u : 0u;
                        }
                        ulonglong2 *dst = obase + s.run_off[d] + rk;
                        if (HINTS) st_rec_hint(dst, rec[r], pol_out);
                        else *dst = rec[r];
                    }
                }
                (void)cnt16;
                __syncthreads();
            }
            // ---- advance the cursors, clear this tile's counters (8 consecutive buckets per thread). No barrier:
            // the next tile counts into the other buffer and its own barrier orders everything else.
            {
                const u32 b0 = tid * 8u;
                uint4 *cp = reinterpret_cast<uint4 *>(&cnt32[b0 >> 1]);
                const uint4 a = *cp;
                uint4 *rp = reinterpret_cast<uint4 *>(&s.run_off[b0]);
                uint4 r0 = rp[0], r1 = rp[1];
                r0.x += a.x & 0xFFFFu, r0.y += a.x >> 16, r0.z += a.y & 0xFFFFu, r0.w += a.y >> 16;
                r1.x += a.z & 0xFFFFu, r1.y += a.z >> 16, r1.z += a.w & 0xFFFFu, r1.w += a.w >> 16;
                rp[0] = r0;
                rp[1] = r1;
                *cp = make_uint4(0, 0, 0, 0);
                if (tid == 0) s.ovf[buf] = 0;
            }
        }
    }
}

// ---- level scatter (v3): staged bucket runs (like v1) ranked with ONE atomic per record (like v2) ---------
// What the measurements of this round say (profiles/r02_kv_*): the fan-out of a level is bounded by the L2,
// not by the SM — every (piece, bucket) pair is a write front that occupies a 128-byte line until its
// neighbours arrive, and 296 pieces x 4096 buckets do not fit (DRAM reads 2.1x, writes 1.5x the algorithmic
// bytes: ECC read-modify-write of half-written sectors); 296 x 1024 do, if every tile hands each bucket a
// contiguous run. So: 10 bits per level, the tile staged bucket-major in shared memory and every bucket's run
// written by one TMA bulk store (v1's data path), but the rank of a record inside (tile, bucket) comes from one
// packed 16-bit atomic plus a SWAR compare against the tile indices of its bucket mates (v1 spent ~120 of its
// 231 warp-instructions per 32 records on one ballot per digit bit and per-warp histograms).
constexpr int S4_NT = 512;
constexpr int S4_RPT = 8;
constexpr int S4_T = S4_NT * S4_RPT;           // 4096
constexpr int S4_NB = P1_MAX_NB;               // 1024
constexpr int S4_SIDX = S4_T + 7 * S4_NB + 8;  // bucket index lists, each padded to a multiple of 8 entries

struct Scatter4Smem {
    alignas(16) ulonglong2 stage[S4_T];
    u64 run_off[S4_NB];
    alignas(16) u16 sidx[S4_SIDX];
    alignas(16) u32 cnt[2][S4_NB / 2];   // packed 16-bit counters, double buffered
    u32 base[S4_NB + 2];                 // padded list start << 16 | staging start
    u32 bitmap[S4_NT / 32][S4_T / 32];   // hot runs only
    u16 hot[S4_T / 32];
    u32 nhot;
    u32 wsum[32];
};

__global__ void __launch_bounds__(S4_NT, 2)
part_scatter3_kernel(const ulonglong2 *__restrict__ in, ulonglong2 *__restrict__ out,
                     const Piece *__restrict__ pieces, const u32 *__restrict__ cta_piece_begin, u64 ustart,
                     u64 un, u64 uR, DigitSpec ds, u32 nb, const u64 *__restrict__ piece_off) {
    constexpr int NT = S4_NT, RPT = S4_RPT, T = S4_T, NW = NT / 32, WPL = T / 32 / 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Scatter4Smem &s = *reinterpret_cast<Scatter4Smem *>(smem_raw);
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 pb = pieces ? cta_piece_begin[blockIdx.x] : blockIdx.x;
    const u32 pe = pieces ? cta_piece_begin[blockIdx.x + 1] : blockIdx.x + 1;
    u32 tile_no = 0;

    for (u32 p = pb; p < pe; ++p) {
        const Piece pc = pieces ? pieces[p] : uniform_piece(p, ustart, un, uR);
        __syncthreads();
        for (u32 b = tid; b < (u32)S4_NB; b += NT) {
            s.run_off[b] = (b < nb) ? piece_off[(u64)p * nb + b] : 0ULL;
            (&s.cnt[0][0])[b] = 0;
        }
        __syncthreads();
        for (u64 t0 = pc.start; t0 < pc.end; t0 += T, ++tile_no) {
            const u32 tn = (u32)min((u64)T, pc.end - t0);
            const u32 buf = tile_no & 1u;
            u32 *cnt32 = s.cnt[buf];
            ulonglong2 rec[RPT];
            u32 dsl[RPT];  // digit | slot << 16
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const u32 li = r * NT + tid;
                if (li < tn) rec[r] = in[t0 + li];
            }
            if (t0 + T < pc.end) {  // the next tile: pull it into L2 while this one is ranked and staged
                const char *nxt = reinterpret_cast<const char *>(in + t0 + T);
                const u32 nbytes = (u32)min((u64)T, pc.end - t0 - T) * 16u;
                for (u32 off = tid * 128u; off < nbytes; off += NT * 128u)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt + off));
            }
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const u32 li = r * NT + tid;
                dsl[r] = 0;
                if (li < tn) {
                    const u32 d = digit_of(rec[r].x, ds);
                    const u32 old = atomicAdd(&cnt32[d >> 1], (d & 1u) ? 0x10000u : 1u);
                    dsl[r] = d | (((d & 1u) ? (old >> 16) : (old & 0xFFFFu)) << 16);
                }
            }
            if (tid == 0) s.nhot = 0;
            __syncthreads();
            // ---- scan of the bucket counts (2 buckets per thread): staging offsets and padded list offsets ----
            {
                const u32 w = cnt32[tid];  // buckets 2 tid, 2 tid + 1
                const u32 c0 = w & 0xFFFFu, c1 = w >> 16;
                if (c0 > HOT_L) s.hot[atomicAdd(&s.nhot, 1u)] = (u16)(2 * tid);
                if (c1 > HOT_L) s.hot[atomicAdd(&s.nhot, 1u)] = (u16)(2 * tid + 1);
                const u32 p0 = (c0 + 7u) & ~7u, p1 = (c1 + 7u) & ~7u;
                const u32 mine = (c0 + c1) | ((p0 + p1) << 16);  // both sums stay below 2^16
                u32 v = mine;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                    if ((int)lane >= d) v += o;
                }
                if (lane == 31) s.wsum[warp] = v;
                __syncthreads();
                u32 woff = 0;
                for (u32 ww = 0; ww < warp; ++ww) woff += s.wsum[ww];
                const u32 ex = woff + v - mine;
                s.base[2 * tid] = ex;
                s.base[2 * tid + 1] = ex + (c0 | (p0 << 16));
                if (tid == NT - 1) s.base[S4_NB] = ex + mine;
            }
            __syncthreads();
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const u32 li = r * NT + tid;
                if (li < tn) s.sidx[(s.base[dsl[r] & 0xFFFFu] >> 16) + (dsl[r] >> 16)] = (u16)li;
            }
            __syncthreads();
            const u32 nh = s.nhot;
            if (nh) {
                // skew: a warp sorts the tile indices of a long run through a presence bitmap
                u32 *bm = s.bitmap[warp];
                for (u32 hi = warp; hi < nh; hi += NW) {
                    const u32 h = s.hot[hi];
                    const u32 st = s.base[h] >> 16, L = (s.base[h + 1] & 0xFFFFu) - (s.base[h] & 0xFFFFu);
                    for (u32 w = lane; w < T / 32; w += 32) bm[w] = 0;
                    __syncwarp();
                    for (u32 j = lane; j < L; j += 32) {
                        const u32 x = s.sidx[st + j];
                        atomicOr(&bm[x >> 5], 1u << (x & 31));
                    }
                    __syncwarp();
                    u32 words[WPL];
                    u32 cl = 0;
#pragma unroll
                    for (int k = 0; k < WPL; ++k) {
                        words[k] = bm[lane * WPL + k];
                        cl += __popc(words[k]);
                    }
                    u32 v = cl;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                        if ((int)lane >= d) v += o;
                    }
                    u32 pos = st + v - cl;
#pragma unroll
                    for (int k = 0; k < WPL; ++k) {
                        u32 wd = words[k];
                        while (wd) {
                            const u32 bit = __ffs(wd) - 1;
                            wd &= wd - 1;
                            s.sidx[pos++] = (u16)((lane * WPL + k) * 32 + bit);
                        }
                    }
                    __syncwarp();
                }
                __syncthreads();
            }
            // ---- rank inside (tile, bucket) by tile index, stage bucket-major -----------------------------------
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const u32 li = r * NT + tid;
                if (li < tn) {
                    const u32 d = dsl[r] & 0xFFFFu;
                    const u32 b0 = s.base[d], b1 = s.base[d + 1];
                    const u32 lst = b0 >> 16, L = (b1 & 0xFFFFu) - (b0 & 0xFFFFu);
                    u32 rk = 0;
                    if (L > HOT_L) {  // sorted by a warp above: lower bound
                        u32 lo = 0, hi = L;
                        while (lo < hi) {
                            const u32 mid = (lo + hi) >> 1;
                            if (s.sidx[lst + mid] < li) lo = mid + 1;
                            else hi = mid;
                        }
                        rk = lo;
                    } else if (L > 1) {
                        // 8 tile indices per 16-byte row; halfword-wise "entry < li" by SWAR (entries < 2^15)
                        const u64 H = 0x8000800080008000ULL, lim = (u64)li * 0x0001000100010001ULL;
                        for (u32 j = 0; j < L; j += 8) {
                            const uint4 row = *reinterpret_cast<const uint4 *>(&s.sidx[lst + j]);
                            const u64 lo = (u64)row.x | ((u64)row.y << 32), hi = (u64)row.z | ((u64)row.w << 32);
                            const u32 left = L - j;
                            const u64 m0 = (left >= 4) ? ~0ULL : ((1ULL << (16 * left)) - 1ULL);
                            const u64 m1 = (left >= 8) ? ~0ULL : ((left > 4) ? ((1ULL << (16 * (left - 4))) - 1ULL) : 0ULL);
                            rk += (u32)__popcll(~((lo | H) - lim) & H & m0) + (u32)__popcll(~((hi | H) - lim) & H & m1);
                        }
                    }
                    s.stage[(b0 & 0xFFFFu) + rk] = rec[r];
                }
            }
            fence_proxy_async();
            __syncthreads();
            // ---- every bucket's run leaves with one TMA bulk store; cursors advance, counters clear -----------------
            {
                const u32 w = cnt32[tid];
                const u32 c0 = w & 0xFFFFu, c1 = w >> 16;
                const u32 s0 = s.base[2 * tid] & 0xFFFFu;
                u64 r0 = s.run_off[2 * tid], r1 = s.run_off[2 * tid + 1];
                if (c0) tma_store_1d(out + r0, &s.stage[s0], c0 * 16u);
                if (c1) tma_store_1d(out + r1, &s.stage[s0 + c0], c1 * 16u);
                tma_store_commit();
                s.run_off[2 * tid] = r0 + c0;
                s.run_off[2 * tid + 1] = r1 + c1;
                cnt32[tid] = 0;
                tma_store_wait_read();  // the staging area is reused by the next tile
            }
            __syncthreads();
        }
    }
    tma_store_wait_all();
}

// single-CTA leaf. reduce_op < 0: sort only, records written to out[ch.start ..). Otherwise one record
// per key group is written compacted at out[ch.start ..) and (start, groups) to the entry table.
__global__ void __launch_bounds__(L_THREADS, 2)
leaf_sort_kernel(const ulonglong2 *__restrict__ data, ulonglong2 *__restrict__ out,
                 const LeafChunk *__restrict__ chunks, u32 nchunks, int xf, u64 base, int reduce_op,
                 u64 *__restrict__ entry_start, u32 *__restrict__ entry_groups) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    LeafSmem &s = *reinterpret_cast<LeafSmem *>(smem_raw);
    const u32 tid = threadIdx.x;
    for (u32 c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const LeafChunk ch = chunks[c];
        const u32 n = ch.n;
        if (c + gridDim.x < nchunks) {
            // pull the chunk this CTA handles next into L2 (one 128-byte line per thread per pass)
            const LeafChunk nx = chunks[c + gridDim.x];
            const char *nb = reinterpret_cast<const char *>(data + nx.start);
            for (u32 off = tid * 128u; off < nx.n * 16u; off += L_THREADS * 128u)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(nb + off));
        }
        ulonglong2 rr[L_IPT];
#pragma unroll
        for (int k = 0; k < L_IPT; ++k) {
            const u32 i = tid + k * L_THREADS;
            if (i < n) rr[k] = data[ch.start + i];
        }
#pragma unroll
        for (int k = 0; k < L_IPT; ++k) {
            const u32 i = tid + k * L_THREADS;
            if (i < n) {
                if (reduce_op >= 0) s.val[i] = rr[k].y;
                s.sk[i] = key_xform(rr[k].x, xf) - base;
            }
        }
        __syncthreads();
        if (reduce_op < 0) {
            // sort only: the records stay in registers; each one computes its final position and leaves
            // directly (no gather pass over shared memory, no inverse key transform)
            u32 slot[L_IPT];
            const bool heavy = leaf_bin_records(s, n, ch.bin_shift, ch.bin_base, slot);
            if (heavy) leaf_sort_heavy_bins(s, n);
#pragma unroll
            for (int k = 0; k < L_IPT; ++k) {
                const u32 i = tid + k * L_THREADS;
                if (i < n) out[ch.start + leaf_final_pos<false>(s, n, i, slot[k], heavy)] = rr[k];
            }
            __syncthreads();
            continue;
        }
        if (reduce_op >= 0 && hash_fold_op(xf, reduce_op)) {
            const u32 g = leaf_hash_fold(s, n, reduce_op, xf, base, out + ch.start);
            if (tid == 0) {
                entry_start[ch.entry] = ch.start;
                entry_groups[ch.entry] = g;
            }
            __syncthreads();
            continue;
        }
        leaf_sort_core<false>(s, n, ch.bin_shift, ch.bin_base);
        {
            const u32 g = leaf_seg_reduce(s, n, reduce_op, xf, base, out + ch.start);
            if (tid == 0) {
                entry_start[ch.entry] = ch.start;
                entry_groups[ch.entry] = g;
            }
        }
        __syncthreads();
    }
}

// cluster leaf: 8 CTAs sort one chunk of up to C_NMAX records (see the file header).
// An exchange that would overflow a CTA (a fine bin larger than its capacity: heavy duplicates / skew
// inside the chunk) writes nothing and reports the chunk in ovf_list; the host re-sorts those chunks with
// further partition levels.
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(L_THREADS, 2)
cluster_leaf_kernel(const ulonglong2 *__restrict__ data, ulonglong2 *__restrict__ out,
                    const LeafChunk *__restrict__ chunks, u32 nchunks, int xf, u64 base, int reduce_op,
                    u64 *__restrict__ entry_start, u32 *__restrict__ entry_groups, u32 *__restrict__ ovf_count,
                    u32 *__restrict__ ovf_list) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    LeafSmem &s = *reinterpret_cast<LeafSmem *>(smem_raw);
    cg::cluster_group cluster = cg::this_cluster();
    const u32 tid = threadIdx.x;
    const u32 rank = cluster.block_rank();
    const u32 ncl = gridDim.x / CL, cid = blockIdx.x / CL;
    for (u32 c = cid; c < nchunks; c += ncl) {
        const LeafChunk ch = chunks[c];
        const u32 n = ch.n;
        const u32 S = (n + CL - 1) / CL;  // slice per CTA, <= L_CAP
        const u32 lo = min(n, rank * S), hi = min(n, lo + S);
        if (c + ncl < nchunks) {
            const LeafChunk nx = chunks[c + ncl];
            const u32 S2 = (nx.n + CL - 1) / CL;
            const u32 lo2 = min(nx.n, rank * S2), hi2 = min(nx.n, lo2 + S2);
            const char *nb = reinterpret_cast<const char *>(data + nx.start + lo2);
            for (u32 off = tid * 128u; off < (hi2 - lo2) * 16u; off += L_THREADS * 128u)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(nb + off));
        }
        if (tid < CF) s.fh[tid] = 0;
        if (tid == 0) s.ovf = 0;
        __syncthreads();
        // ---- my slice: fine-bin histogram, the atomic's return value is the record's slot --------------
        ulonglong2 rec[L_IPT];
        u32 pk[L_IPT];
#pragma unroll
        for (int k = 0; k < L_IPT; ++k) {
            const u32 i = tid + k * L_THREADS;
            if (lo + i < hi) rec[k] = data[ch.start + lo + i];
        }
#pragma unroll
        for (int k = 0; k < L_IPT; ++k) {
            const u32 i = tid + k * L_THREADS;
            pk[k] = 0;
            if (lo + i < hi) {
                const u64 skv = key_xform(rec[k].x, xf) - base;
                rec[k].x = skv;
                const u32 f = (u32)min((skv >> ch.bin_shift) - ch.bin_base, (u64)(CF - 1));
                pk[k] = f | (atomicAdd(&s.fh[f], 1u) << 8);
            }
        }
        cluster.sync();
        // ---- all CTAs derive the same bin -> CTA assignment from the 8 histograms ---------------------
        u32 tot = 0, before = 0;
        if (tid < CF) {
#pragma unroll
            for (u32 r = 0; r < CL; ++r) {
                const u32 *rfh = cluster.map_shared_rank(s.fh, r);
                const u32 cnt = rfh[tid];
                before += (r < rank) ? cnt : 0u;
                tot += cnt;
            }
        }
        u32 total;
        const u32 g0 = block_excl_scan(s, tot, &total);
        // CTA o owns the fine bins [32 o, 32 o + 32): with hashed (or locally uniform) keys every CTA receives
        // n/8 +- a few dozen records, and exactly 32 bins per CTA give the local sort 8192 bins
        if (tid < CF) s.gpos[tid] = g0;
        if (tid == CF - 1) s.gpos[CF] = g0 + tot;
        __syncthreads();
        if (tid < CF) s.dpos[tid] = (u16)(g0 - s.gpos[tid & ~(CF / CL - 1)] + before);
        if (tid < CL) {
            s.firstg[tid] = s.gpos[tid * (CF / CL)];
            s.endg[tid] = s.gpos[(tid + 1) * (CF / CL)];
            if (s.gpos[(tid + 1) * (CF / CL)] - s.gpos[tid * (CF / CL)] > (u32)L_CAP) s.ovf = 1;
        }
        __syncthreads();
        const bool ovf = s.ovf != 0;
        // ---- exchange: every record goes straight into the owner's shared memory ------------------------
        if (!ovf) {
#pragma unroll
            for (int k = 0; k < L_IPT; ++k) {
                const u32 i = tid + k * L_THREADS;
                if (lo + i < hi) {
                    const u32 f = pk[k] & 255u;
                    const u32 o = f / (u32)(CF / CL);
                    const u32 p = (u32)s.dpos[f] + (pk[k] >> 8);
                    u64 *rsk = cluster.map_shared_rank(s.sk, o);
                    u64 *rval = cluster.map_shared_rank(s.val, o);
                    u16 *raux = cluster.map_shared_rank(s.aux, o);
                    rsk[p] = rec[k].x;
                    rval[p] = rec[k].y;
                    raux[p] = (u16)(lo + i);
                }
            }
        }
        cluster.sync();
        if (ovf) {
            if (rank == 0 && tid == 0) ovf_list[atomicAdd(ovf_count, 1u)] = c;
            if (reduce_op >= 0 && tid == 0) {
                entry_start[ch.entry + rank] = ch.start;
                entry_groups[ch.entry + rank] = 0;
            }
            continue;
        }
        // ---- local finish ------------------------------------------------------------------------------------
        const u32 m = s.endg[rank] - s.firstg[rank];
        const u64 ostart = ch.start + s.firstg[rank];
        if (reduce_op >= 0 && hash_fold_op(xf, reduce_op)) {
            const u32 g = leaf_hash_fold(s, m, reduce_op, xf, base, out + ostart);
            if (tid == 0) {
                entry_start[ch.entry + rank] = ostart;
                entry_groups[ch.entry + rank] = g;
            }
            __syncthreads();
            continue;
        }
        const u32 nbo = CF / CL;
        int k = 0;
        while (((nbo << (k + 1)) <= (u32)L_BINS) && (k + 1) <= ch.bin_shift) ++k;
        leaf_sort_core<true>(s, m, ch.bin_shift - k, (ch.bin_base + (u64)rank * nbo) << k);
        if (reduce_op < 0) {
            for (u32 i = tid; i < m; i += L_THREADS) {
                const u32 o = s.fin[i];
                out[ostart + i] = make_ulonglong2(key_unxform(s.sk[o] + base, xf), s.val[o]);
            }
        } else {
            const u32 g = leaf_seg_reduce(s, m, reduce_op, xf, base, out + ostart);
            if (tid == 0) {
                entry_start[ch.entry + rank] = ostart;
                entry_groups[ch.entry + rank] = g;
            }
        }
        __syncthreads();
    }
}

// reduce a whole range that holds a single key (all keys equal): one CTA
__global__ void single_group_reduce_kernel(const ulonglong2 *__restrict__ data, u64 start, u64 n, int op,
                                           ulonglong2 *__restrict__ out_rec) {
    __shared__ u64 part[32];
    u64 acc = 0;
    bool have = false;
    // FIRST/LAST depend on order: handled by thread 0 directly
    if (op == DAMPR_OP_FIRST || op == DAMPR_OP_LAST) {
        if (threadIdx.x == 0) {
            ulonglong2 r = data[start + (op == DAMPR_OP_FIRST ? 0 : n - 1)];
            *out_rec = r;
        }
        return;
    }
    if (op == DAMPR_OP_SUM_F64) {
        // deterministic: fixed strided partition + tree
        double a = 0.0;
        for (u64 i = threadIdx.x; i < n; i += blockDim.x) a += __longlong_as_double((long long)data[start + i].y);
        for (int d = 16; d > 0; d >>= 1) a += __shfl_down_sync(0xFFFFFFFFu, a, d);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = (u64)__double_as_longlong(a);
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (u32 w = 0; w < blockDim.x / 32; ++w) t += __longlong_as_double((long long)part[w]);
            *out_rec = make_ulonglong2(data[start].x, (u64)__double_as_longlong(t));
        }
        return;
    }
    for (u64 i = threadIdx.x; i < n; i += blockDim.x) {
        u64 v = (op == DAMPR_OP_COUNT) ? 1ULL : data[start + i].y;
        acc = have ? apply_op(op, acc, v) : v;
        have = true;
    }
    // combine across lanes / warps (ops here are commutative)
    for (int d = 16; d > 0; d >>= 1) {
        u64 o = __shfl_down_sync(0xFFFFFFFFu, acc, d);
        u32 oh = __shfl_down_sync(0xFFFFFFFFu, (u32)have, d);
        if (oh) {
            acc = have ? apply_op(op, acc, o) : o;
            have = true;
        }
    }
    __shared__ u32 parth[32];
    if ((threadIdx.x & 31) == 0) {
        part[threadIdx.x >> 5] = acc;
        parth[threadIdx.x >> 5] = have;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        u64 t = 0;
        bool th = false;
        for (u32 w = 0; w < blockDim.x / 32; ++w)
            if (parth[w]) {
                t = th ? apply_op(op, t, part[w]) : part[w];
                th = true;
            }
        *out_rec = make_ulonglong2(data[start].x, t);
    }
}

// ---- misc kernels -------------------------------------------------------------------------------
__global__ void minmax_kernel(const ulonglong2 *__restrict__ in, u64 n, int xf, u64 *out /*[2]: min,max*/) {
    u64 mn = ~0ULL, mx = 0;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 k = key_xform(in[i].x, xf);
        mn = min(mn, k);
        mx = max(mx, k);
    }
    for (int d = 16; d > 0; d >>= 1) {
        mn = min(mn, __shfl_down_sync(0xFFFFFFFFu, mn, d));
        mx = max(mx, __shfl_down_sync(0xFFFFFFFFu, mx, d));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&out[0], mn);
        atomicMax(&out[1], mx);
    }
}

__global__ void copy_records_kernel(const ulonglong2 *__restrict__ in, ulonglong2 *__restrict__ out, u64 n) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) out[i] = in[i];
}

// copies the groups of every entry (start, count) of the table to its offset in the output
__global__ void gather_groups_kernel(const ulonglong2 *__restrict__ tmp, const u64 *__restrict__ entry_start,
                                     const u32 *__restrict__ entry_groups, const u64 *__restrict__ entry_out_off,
                                     u32 nentries, ulonglong2 *__restrict__ out) {
    for (u32 c = blockIdx.x; c < nentries; c += gridDim.x) {
        const u32 g = entry_groups[c];
        const u64 src = entry_start[c], dst = entry_out_off[c];
        for (u32 i = threadIdx.x; i < g; i += blockDim.x) out[dst + i] = tmp[src + i];
    }
}

__global__ void group_heads_kernel(const ulonglong2 *__restrict__ in, u64 n, u64 *__restrict__ offsets, u64 cap,
                                   u64 *__restrict__ cursor_unused, u64 *__restrict__ count) {
    // two uses: offsets == nullptr -> count heads; otherwise heads are written at their rank,
    // which requires a scan: this kernel is launched with one CTA per 4096-record tile after
    // tile head counts were scanned into cursor_unused (tile base).
    __shared__ u32 wsum[32];
    const u64 t0 = (u64)blockIdx.x * 4096ULL;
    u32 flags = 0, cnt = 0;
    for (int k = 0; k < 8; ++k) {
        u64 i = t0 + (u64)threadIdx.x * 8 + k;
        if (i < n) {
            bool head = (i == 0) || (in[i].x != in[i - 1].x);
            flags |= head ? (1u << k) : 0u;
        }
    }
    cnt = __popc(flags);
    u32 v = cnt;
    for (int d = 1; d < 32; d <<= 1) {
        u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((int)(threadIdx.x & 31) >= d) v += o;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = v;
    __syncthreads();
    u32 woff = 0;
    for (u32 w = 0; w < (threadIdx.x >> 5); ++w) woff += wsum[w];
    if (!offsets) {
        if (threadIdx.x == blockDim.x - 1) ((u32 *)count)[blockIdx.x] = woff + v;
        return;
    }
    u64 g = cursor_unused[blockIdx.x] + woff + v - cnt;
    for (int k = 0; k < 8; ++k)
        if (flags & (1u << k)) {
            if (g < cap) offsets[g] = t0 + (u64)threadIdx.x * 8 + k;
            ++g;
        }
}

// ---- host-side orchestration ------------------------------------------------------------------
static int bits_for(u64 n, u64 leaf_avg) {
    int b = 0;
    while (((n + leaf_avg - 1) / leaf_avg) > (1ULL << b)) ++b;
    return b;
}

static int g_use_tma = 1;

static int scatter_ctas(dampr_ctx *ctx) { return ctx->num_sms * 2; }
static u64 scatter_tile() { return (u64)P_TILE; }  // both scatter generations use 4096-record tiles
static_assert(P_TILE == S3_T, "tile sizes");

static int run_scatter(dampr_ctx *ctx, int G, const ulonglong2 *src, ulonglong2 *dst, const Piece *pieces,
                       const u32 *cta_pb, u64 ustart, u64 un, u64 uR, u64 out_base, DigitSpec ds, u32 nb,
                       const u64 *poff, bool v2) {
    ScopedTimer tm(ctx, DAMPR_K_PART_SCATTER);
    if (!v2 && g_kv_scatter == 3 && nb <= (u32)S4_NB) {
        const size_t smem = sizeof(Scatter4Smem);
        CUDA_TRY(ctx, cudaFuncSetAttribute(part_scatter3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        part_scatter3_kernel<<<G, S4_NT, smem, ctx->stream>>>(src, dst, pieces, cta_pb, ustart, un, uR, ds, nb, poff);
        CUDA_TRY(ctx, cudaGetLastError());
        return DAMPR_OK;
    }
    if (v2) {
        const size_t smem = sizeof(Scatter3Smem);
        if (g_kv_hints) {
            CUDA_TRY(ctx, cudaFuncSetAttribute(part_scatter2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            part_scatter2_kernel<true><<<G, S3_NT, smem, ctx->stream>>>(src, dst, pieces, cta_pb, ustart, un, uR, out_base, ds,
                                                                       nb, poff);
        } else {
            CUDA_TRY(ctx, cudaFuncSetAttribute(part_scatter2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            part_scatter2_kernel<false><<<G, S3_NT, smem, ctx->stream>>>(src, dst, pieces, cta_pb, ustart, un, uR, out_base, ds,
                                                                        nb, poff);
        }
        CUDA_TRY(ctx, cudaGetLastError());
        return DAMPR_OK;
    }
    const size_t smem = sizeof(ScatterSmem);
    if (g_use_tma) {
        cudaFuncSetAttribute(part_scatter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        part_scatter_kernel<true><<<G, P_THREADS, smem, ctx->stream>>>(src, dst, pieces, cta_pb, ustart, un, uR, ds, nb, poff);
    } else {
        cudaFuncSetAttribute(part_scatter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        part_scatter_kernel<false><<<G, P_THREADS, smem, ctx->stream>>>(src, dst, pieces, cta_pb, ustart, un, uR, ds, nb, poff);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

// which scatter a level of nb buckets over n records uses: the table scatter wants at least as many buckets as
// a tile has records... it is still correct below that (every tile takes its general path), the ballot scatter
// is faster there and handles at most 1024 buckets; cursors of the table scatter are 32-bit
static bool use_v2_scatter(u32 nb, u64 n) {
    if (g_kv_scatter < 2 || n >= (1ULL << 32)) return false;
    return nb > (u32)P1_MAX_NB;
}

// One partition level over records [start, start+n) of `src` into `dst`: every segment of
// seg_off is split by the digit `ds` into nb sub-segments (stable). seg_off is replaced by the
// (S*nb + 1) offsets of the next level. The offsets travel to the host while the scatter runs.
static int partition_level(dampr_ctx *ctx, const ulonglong2 *src, ulonglong2 *dst, u64 start, u64 n,
                           std::vector<u64> &seg_off, DigitSpec ds, u32 nb) {
    const int G = scatter_ctas(ctx);
    const u64 S = seg_off.size() - 1;
    const u64 T = scatter_tile();
    u64 R = (n + G - 1) / G;
    R = ((R + T - 1) / T) * T;
    cudaEvent_t ev;
    CUDA_TRY(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    struct EvGuard {
        cudaEvent_t e;
        ~EvGuard() { cudaEventDestroy(e); }
    } evg{ev};

    const bool v2 = use_v2_scatter(nb, n);
    if (S == 1 && g_kv_hist == 2) {
        // ---- single segment: uniform pieces computed on the device, nothing uploaded ----------------------
        const u32 NP = (u32)G;
        DevBuf d_hist, d_tot, d_seg, d_poff;
        CUDA_TRY(ctx, d_hist.alloc((u64)NP * nb * 4));
        CUDA_TRY(ctx, d_tot.alloc((u64)nb * 4));
        CUDA_TRY(ctx, d_seg.alloc((u64)(nb + 1) * 8));
        CUDA_TRY(ctx, d_poff.alloc((u64)NP * nb * 8));
        const u32 hs = (u32)std::max(1, (2 * ctx->num_sms + (int)NP - 1) / (int)NP);
        CUDA_TRY(ctx, cudaMemsetAsync(d_tot.p, 0, (u64)nb * 4, ctx->stream));
        if (hs > 1) CUDA_TRY(ctx, cudaMemsetAsync(d_hist.p, 0, (u64)NP * nb * 4, ctx->stream));
        {
            ScopedTimer tm(ctx, DAMPR_K_PART_HIST);
            part_hist2_kernel<<<NP * hs, H2_THREADS, 0, ctx->stream>>>(src, nullptr, start, n, R, hs, ds, nb,
                                                                     (u32 *)d_hist.p, (u32 *)d_tot.p);
        }
        {
            ScopedTimer tm(ctx, DAMPR_K_MISC);
            bucket_scan_kernel<<<1, 1024, 0, ctx->stream>>>((const u32 *)d_tot.p, nb, start, n, (u64 *)d_seg.p);
            column_offsets_kernel<<<(nb + 31) / 32, 1024, 0, ctx->stream>>>((const u32 *)d_hist.p, NP, nb,
                                                                           (const u64 *)d_seg.p, (u64 *)d_poff.p);
        }
        CUDA_TRY(ctx, cudaGetLastError());
        u64 *h_next = (u64 *)host_pin(ctx, 0, (u64)(nb + 1) * 8);
        if (!h_next) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
        CUDA_TRY(ctx, cudaMemcpyAsync(h_next, d_seg.p, (u64)(nb + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaEventRecord(ev, ctx->stream));
        int rc = run_scatter(ctx, G, src, dst, nullptr, nullptr, start, n, R, start, ds, nb, (const u64 *)d_poff.p, v2);
        if (rc) return rc;
        CUDA_TRY(ctx, cudaEventSynchronize(ev));  // the scatter is still running
        seg_off.assign(h_next, h_next + nb + 1);
        return DAMPR_OK;
    }

    // ---- general level: pieces split at CTA-range boundaries and at segment boundaries ---------------
    std::vector<Piece> pieces;
    std::vector<u32> cta_pb(G + 1, 0), seg_pb(S + 1, 0);
    {
        u64 s_idx = 0;
        for (int c = 0; c < G; ++c) {
            u64 lo = start + std::min(n, (u64)c * R), hi = start + std::min(n, (u64)(c + 1) * R);
            cta_pb[c] = (u32)pieces.size();
            u64 pos = lo;
            while (pos < hi) {
                while (seg_off[s_idx + 1] <= pos) ++s_idx;
                u64 e = std::min(hi, seg_off[s_idx + 1]);
                pieces.push_back(Piece{pos, e, (u32)s_idx, 0});
                pos = e;
            }
        }
        cta_pb[G] = (u32)pieces.size();
        // seg_piece_begin: pieces are ordered by start, hence by segment
        u32 pi = 0;
        for (u64 s2 = 0; s2 < S; ++s2) {
            while (pi < pieces.size() && pieces[pi].seg < s2) ++pi;
            seg_pb[s2] = pi;
        }
        seg_pb[S] = (u32)pieces.size();
        // empty segments: seg_pb must be monotone; fix holes
        for (u64 s2 = S; s2-- > 0;)
            if (seg_pb[s2] > seg_pb[s2 + 1]) seg_pb[s2] = seg_pb[s2 + 1];
    }
    const u64 NP = pieces.size();
    DevBuf d_pieces, d_cta_pb, d_seg_pb, d_seg_off, d_hist, d_poff, d_next;
    CUDA_TRY(ctx, d_pieces.alloc(NP * sizeof(Piece)));
    CUDA_TRY(ctx, d_cta_pb.alloc((G + 1) * 4));
    CUDA_TRY(ctx, d_seg_pb.alloc((S + 1) * 4));
    CUDA_TRY(ctx, d_seg_off.alloc((S + 1) * 8));
    CUDA_TRY(ctx, d_hist.alloc(NP * nb * 4));
    CUDA_TRY(ctx, d_poff.alloc(NP * nb * 8));
    CUDA_TRY(ctx, d_next.alloc((S * nb + 1) * 8));
    {
        // descriptors go up through page-locked scratch (a pageable source synchronises the stream)
        const size_t b0 = NP * sizeof(Piece), b1 = (G + 1) * 4, b2 = (S + 1) * 4, b3 = (S + 1) * 8;
        const size_t o1 = (b0 + 15) & ~(size_t)15, o2 = o1 + ((b1 + 15) & ~(size_t)15), o3 = o2 + ((b2 + 15) & ~(size_t)15);
        char *hp = (char *)host_pin(ctx, 1, o3 + b3);
        if (!hp) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
        memcpy(hp, pieces.data(), b0);
        memcpy(hp + o1, cta_pb.data(), b1);
        memcpy(hp + o2, seg_pb.data(), b2);
        memcpy(hp + o3, seg_off.data(), b3);
        CUDA_TRY(ctx, cudaMemcpyAsync(d_pieces.p, hp, b0, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_cta_pb.p, hp + o1, b1, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_seg_pb.p, hp + o2, b2, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_seg_off.p, hp + o3, b3, cudaMemcpyHostToDevice, ctx->stream));
        host_pin_used(ctx, 1);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_PART_HIST);
        if (g_kv_hist == 2)
            part_hist2_kernel<<<(unsigned)NP, H2_THREADS, 0, ctx->stream>>>(src, (const Piece *)d_pieces.p, 0, 0, 0, 1, ds, nb,
                                                                           (u32 *)d_hist.p, nullptr);
        else
            part_hist_kernel<<<G, P_THREADS, 0, ctx->stream>>>(src, (const Piece *)d_pieces.p, (const u32 *)d_cta_pb.p, ds,
                                                              nb, (u32 *)d_hist.p);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        part_scan_kernel<<<(unsigned)S, 1024, 0, ctx->stream>>>((const u32 *)d_hist.p, (const u32 *)d_seg_pb.p,
                                                               (const u64 *)d_seg_off.p, nb, (u64 *)d_poff.p,
                                                               (u64 *)d_next.p);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    u64 *h_next = (u64 *)host_pin(ctx, 0, (S * nb + 1) * 8);
    if (!h_next) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
    CUDA_TRY(ctx, cudaMemcpyAsync(h_next, d_next.p, S * nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaEventRecord(ev, ctx->stream));
    int rc = run_scatter(ctx, G, src, dst, (const Piece *)d_pieces.p, (const u32 *)d_cta_pb.p, 0, 0, 0, start, ds, nb,
                         (const u64 *)d_poff.p, v2);
    if (rc) return rc;
    CUDA_TRY(ctx, cudaEventSynchronize(ev));
    h_next[S * nb] = start + n;
    seg_off.assign(h_next, h_next + S * nb + 1);
    // the device buffers of this level are released to the pool with the stream's position recorded,
    // so nothing reuses them before the scatter has finished
    return DAMPR_OK;
}

// clusters of the leaf kernel the device keeps resident at once (the kernel is persistent: a cluster that does
// not fit the first wave would start only after another one has finished ALL its chunks)
static int cluster_leaf_max_active(dampr_ctx *ctx, size_t smem) {
    static int cached[64] = {0};
    int &c = cached[ctx->device & 63];
    if (c > 0) return c;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(ctx->num_sms * 2 / CL * CL), 1, 1);
    cfg.blockDim = dim3(L_THREADS, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, cluster_leaf_kernel, &cfg) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        n = std::max(1, ctx->num_sms * 2 / CL * 3 / 4);
    }
    c = n;
    return c;
}

static int copy_range(dampr_ctx *ctx, const ulonglong2 *from, ulonglong2 *to, u64 start, u64 n) {
    if (from == to || n == 0) return DAMPR_OK;
    ScopedTimer tm(ctx, DAMPR_K_MISC);
    copy_records_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(from + start, to + start, n);
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

static int key_range(dampr_ctx *ctx, const ulonglong2 *rec, u64 n, int xf, u64 *base, int *top, bool scan_mix);

// Sort records [start, start+n) that currently live in `cur` (scratch = `alt`, same indexing).
// Digits are taken from bit `top` downwards of (xf(key) - base). reduce_op < 0: on return the sorted
// range is in `target` (either buffer; the last pass writes there, nothing is copied). reduce_op >= 0:
// the key groups of the range are appended, in order, to gout[*gcount...] and both buffers are scratch.
static int sort_range(dampr_ctx *ctx, ulonglong2 *cur, ulonglong2 *alt, u64 start, u64 n, int xf, u64 base,
                      int top, int reduce_op, ulonglong2 *gout, u64 *gcount, int depth, ulonglong2 *target,
                      bool allow_cluster) {
    if (n == 0) return DAMPR_OK;
    if (depth > 0 && top > 0) {
        // a segment that is still too large after a level (skew / heavy hitters): its keys usually occupy a
        // small part of the remaining key range. Re-basing on the segment's own minimum and maximum makes the
        // next digits split it (the top bit of the new span is set), so every recursion makes progress and a
        // segment whose keys are all equal is recognised at once.
        u64 b2;
        int t2;
        int rc = key_range(ctx, cur + start, n, xf, &b2, &t2, true);
        if (rc) return rc;
        base = b2;
        top = t2;
    }
    if (top <= 0 || depth > 70) {
        // all keys equal: already "sorted" (stable); a single group when reducing
        if (reduce_op >= 0) {
            ScopedTimer tm(ctx, DAMPR_K_SEG_REDUCE);
            single_group_reduce_kernel<<<1, 1024, 0, ctx->stream>>>(cur, start, n, reduce_op, gout + *gcount);
            *gcount += 1;
            CUDA_TRY(ctx, cudaGetLastError());
            return DAMPR_OK;
        }
        return copy_range(ctx, cur, target, start, n);
    }
    const bool use_cluster = allow_cluster && g_kv_cluster && n > (u64)L_CAP;
    // ---- plan the levels ---------------------------------------------------------------------
    // at least 8 bits per call when a level is needed at all: surplus buckets cost nothing (small segments
    // are packed into shared leaf chunks) and skewed inputs need the resolution. With the table scatter the
    // first level takes 12 bits whenever the key has them (its fast path wants buckets >= records per tile);
    // further levels (more than ~1.1e8 records) use the ballot scatter with at most 10 bits each.
    int total_bits = bits_for(n, use_cluster ? C_TARGET : (u64)g_kv_leaf_target);
    if (total_bits > 0) total_bits = std::max(total_bits, 8);
    total_bits = std::min(top, total_bits);
    std::vector<int> lev_bits;
    {
        int left = total_bits;
        const bool table = g_kv_scatter == 2 && n < (1ULL << 32) && n >= 65536 && top >= g_kv_max_bits &&
                           g_kv_max_bits > P1_MAX_BITS;
        if (table && left > 0) {
            lev_bits.push_back(g_kv_max_bits);
            left = std::max(0, left - g_kv_max_bits);
        }
        if (left > 0) {
            const int nl = (left + P1_MAX_BITS - 1) / P1_MAX_BITS;
            for (int l = 0; l < nl; ++l) {
                int bq = (left + (nl - l) - 1) / (nl - l);
                lev_bits.push_back(bq);
                left -= bq;
            }
        }
    }
    const int nlev = (int)lev_bits.size();
    std::vector<u64> seg_off{start, start + n};
    ulonglong2 *src = cur, *dst = alt;
    int consumed = 0;
    for (int l = 0; l < nlev; ++l) {
        const int bits = lev_bits[l];
        const u32 nb = 1u << bits;
        DigitSpec ds{xf, base, top - consumed - bits, nb - 1, 0};
        int rc = partition_level(ctx, src, dst, start, n, seg_off, ds, nb);
        if (rc) return rc;
        std::swap(src, dst);
        consumed += bits;
    }
    // data now in `src`; `dst` is free
    // ---- leaves --------------------------------------------------------------------------------
    const int rem_top = top - consumed;  // bits left below the partition digits
    const u64 S = seg_off.size() - 1;
    // sort only: leaves read src and write the target (in place when they are the same buffer).
    // reduce: leaves write their compacted groups into the free buffer, src stays intact.
    ulonglong2 *leaf_out = (reduce_op >= 0) ? dst : target;
    std::vector<LeafChunk> small, clus;
    struct Big {
        u64 start, n;
        u32 after_entry;  // entries emitted before it (ordering of the reduce output)
        u64 seg;          // flattened digit value of the segment
    };
    std::vector<Big> bigs;
    u32 nentries = 0;
    {
        u64 s0 = 0;
        while (s0 < S) {
            const u64 sz = seg_off[s0 + 1] - seg_off[s0];
            if (sz == 0) {
                ++s0;
                continue;
            }
            const u64 cap = use_cluster ? C_NMAX : (u64)L_CAP;
            if (sz > cap) {
                bigs.push_back(Big{seg_off[s0], sz, nentries, s0});
                ++s0;
                continue;
            }
            u64 s1 = s0 + 1;
            u64 tot = sz;
            // a chunk stays "small" (single CTA, up to L_BINS segments) while it fits one CTA; beyond that it
            // becomes a cluster chunk of at most CF segments
            while (s1 < S) {
                const u64 nx = seg_off[s1 + 1] - seg_off[s1];
                const u64 nseg = s1 - s0 + 1;
                if (tot + nx <= (u64)L_CAP && nseg <= (u64)L_BINS) {
                } else if (use_cluster && tot + nx <= C_NMAX && nseg <= (u64)CF && tot + nx > (u64)L_CAP) {
                } else
                    break;
                tot += nx;
                ++s1;
            }
            const u64 nseg = s1 - s0;
            LeafChunk lc;
            lc.start = seg_off[s0];
            lc.n = (u32)tot;
            lc.pad = 0;
            lc.entry = nentries;
            const bool is_cluster = tot > (u64)L_CAP;
            const u64 nbins = is_cluster ? (u64)CF : (u64)L_BINS;
            // bins: (segment index relative to s0) << k | next k key bits.  The segment index of a record is
            // ((sk - base) >> rem_top); recursive calls pass a base that clears the bits above `top`.
            int k = 0;
            while (((nseg << (k + 1)) <= nbins) && (k + 1) <= rem_top) ++k;
            lc.bin_shift = rem_top - k;
            lc.bin_base = ((u64)s0) << k;
            if (is_cluster) {
                clus.push_back(lc);
                nentries += CL;
            } else {
                small.push_back(lc);
                nentries += 1;
            }
            s0 = s1;
        }
    }
    DevBuf d_small, d_clus, d_estart, d_egroups, d_ovf;
    const size_t nsmall = small.size(), nclus = clus.size();
    if (reduce_op >= 0 && nentries) {
        CUDA_TRY(ctx, d_estart.alloc((u64)nentries * 8));
        CUDA_TRY(ctx, d_egroups.alloc((u64)nentries * 4));
    }
    u32 *h_ovf = nullptr;
    if (nsmall || nclus) {
        const size_t bs = nsmall * sizeof(LeafChunk), bc = nclus * sizeof(LeafChunk);
        char *hp = (char *)host_pin(ctx, 1, bs + bc + 16);
        if (!hp) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
        if (bs) memcpy(hp, small.data(), bs);
        if (bc) memcpy(hp + bs, clus.data(), bc);
        const size_t smem = sizeof(LeafSmem);
        if (nsmall) {
            CUDA_TRY(ctx, d_small.alloc(bs));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_small.p, hp, bs, cudaMemcpyHostToDevice, ctx->stream));
            CUDA_TRY(ctx, cudaFuncSetAttribute(leaf_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const u32 grid = (u32)std::min<size_t>(nsmall, (size_t)ctx->num_sms * 2);
            ScopedTimer tm(ctx, DAMPR_K_LEAF_SORT);
            leaf_sort_kernel<<<grid, L_THREADS, smem, ctx->stream>>>(src, leaf_out, (const LeafChunk *)d_small.p, (u32)nsmall,
                                                                    xf, base, reduce_op, (u64 *)d_estart.p,
                                                                    (u32 *)d_egroups.p);
        }
        if (nclus) {
            CUDA_TRY(ctx, d_clus.alloc(bc));
            CUDA_TRY(ctx, d_ovf.alloc((nclus + 1) * 4));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_clus.p, hp + bs, bc, cudaMemcpyHostToDevice, ctx->stream));
            CUDA_TRY(ctx, cudaMemsetAsync(d_ovf.p, 0, 4, ctx->stream));
            CUDA_TRY(ctx, cudaFuncSetAttribute(cluster_leaf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const u32 maxcl = (u32)cluster_leaf_max_active(ctx, smem);
            const u32 grid = (u32)std::min<size_t>(nclus, (size_t)maxcl) * CL;
            ScopedTimer tm(ctx, DAMPR_K_LEAF_SORT);
            cluster_leaf_kernel<<<grid, L_THREADS, smem, ctx->stream>>>(src, leaf_out, (const LeafChunk *)d_clus.p, (u32)nclus,
                                                                       xf, base, reduce_op, (u64 *)d_estart.p,
                                                                       (u32 *)d_egroups.p, (u32 *)d_ovf.p,
                                                                       (u32 *)d_ovf.p + 1);
        }
        CUDA_TRY(ctx, cudaGetLastError());
        host_pin_used(ctx, 1);
        if (nclus) {
            h_ovf = (u32 *)host_pin(ctx, 0, (nclus + 1) * 4);
            if (!h_ovf) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
            CUDA_TRY(ctx, cudaMemcpyAsync(h_ovf, d_ovf.p, (nclus + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
        }
    }
    // chunks the cluster leaf could not balance (read before anything else reuses the pinned slot)
    std::vector<u32> ov;
    if (nclus) {
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        ov.assign(h_ovf + 1, h_ovf + 1 + std::min<u32>(h_ovf[0], (u32)nclus));
    }
    if (reduce_op < 0) {
        // big segments: recurse (their data is in `src`; scratch is `dst`)
        for (auto &b : bigs) {
            // keys in the segment share all bits >= rem_top: new base clears them
            int rc = sort_range(ctx, src, dst, b.start, b.n, xf, base + (b.seg << rem_top), rem_top, -1, nullptr, nullptr,
                                depth + 1, target, allow_cluster);
            if (rc) return rc;
        }
        {
            for (u32 ci : ov) {
                // a chunk the cluster could not balance (skew inside it): its records are untouched in `src`.
                // They share every bit above bin_shift + 8 of (sk - base): sort them on the bits below.
                const LeafChunk &lc = clus[ci];
                const int sub_top = std::min(top, lc.bin_shift + 8);
                const u64 sub_base = base + ((lc.bin_base << lc.bin_shift));
                int rc = sort_range(ctx, src, dst, lc.start, lc.n, xf, sub_base, sub_top, -1, nullptr, nullptr, depth + 1,
                                    target, false);
                if (rc) return rc;
            }
        }
        return DAMPR_OK;
    }
    // ---- reduce: gather entry groups in order, interleaving the big segments ---------------------------
    std::vector<u32> eg(nentries);
    if (nentries) {
        CUDA_TRY(ctx, cudaMemcpyAsync(eg.data(), d_egroups.p, (u64)nentries * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (!ov.empty()) {
        // rare: redo the leaf stage of this range without the cluster leaf (src is intact)
        for (u64 s0 = 0; s0 < S; ++s0) {
            const u64 sz = seg_off[s0 + 1] - seg_off[s0];
            if (sz == 0) continue;
            int rc = sort_range(ctx, src, dst, seg_off[s0], sz, xf, base + (s0 << rem_top), rem_top, reduce_op, gout, gcount,
                                depth + 1, nullptr, false);
            if (rc) return rc;
        }
        return DAMPR_OK;
    }
    u32 ei = 0;
    size_t bi = 0;
    while (ei < nentries || bi < bigs.size()) {
        const u32 run_end = (bi < bigs.size()) ? bigs[bi].after_entry : nentries;
        if (ei < run_end) {
            const u32 cntE = run_end - ei;
            u64 *off = (u64 *)host_pin(ctx, 1, (u64)cntE * 8);
            if (!off) return set_err(ctx, DAMPR_ERR_NOMEM, "%s", "pinned scratch allocation failed");
            u64 run = *gcount;
            for (u32 e = ei; e < run_end; ++e) {
                off[e - ei] = run;
                run += eg[e];
            }
            DevBuf d_off;
            CUDA_TRY(ctx, d_off.alloc((u64)cntE * 8));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_off.p, off, (u64)cntE * 8, cudaMemcpyHostToDevice, ctx->stream));
            {
                ScopedTimer tm(ctx, DAMPR_K_SEG_REDUCE);
                gather_groups_kernel<<<(unsigned)std::min<size_t>(cntE, (size_t)ctx->num_sms * 8), 256, 0, ctx->stream>>>(
                    leaf_out, (const u64 *)d_estart.p + ei, (const u32 *)d_egroups.p + ei, (const u64 *)d_off.p, cntE, gout);
            }
            CUDA_TRY(ctx, cudaGetLastError());
            CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // pinned `off` is reused by the next run
            *gcount = run;
            ei = run_end;
        }
        if (bi < bigs.size() && bigs[bi].after_entry == ei) {
            int rc = sort_range(ctx, src, dst, bigs[bi].start, bigs[bi].n, xf, base + (bigs[bi].seg << rem_top), rem_top,
                                reduce_op, gout, gcount, depth + 1, nullptr, allow_cluster);
            if (rc) return rc;
            ++bi;
        }
    }
    return DAMPR_OK;
}

static int ensure_alt(dampr_ctx *ctx, dampr_kv *kv) {
    if (!kv->alt) {
        kv->alt = (ulonglong2 *)pool_alloc(ctx, (kv->capacity ? kv->capacity : 1) * sizeof(ulonglong2));
        if (!kv->alt) {
            ctx->err = "device allocation (kv scratch) failed";
            return DAMPR_ERR_NOMEM;
        }
    }
    return DAMPR_OK;
}

// key range -> (base, top)
static int key_range(dampr_ctx *ctx, const ulonglong2 *rec, u64 n, int xf, u64 *base, int *top, bool scan_mix) {
    if (xf == DAMPR_KEY_MIX && !scan_mix) {
        *base = 0;
        *top = 64;
        return DAMPR_OK;
    }
    u64 init[2] = {~0ULL, 0ULL};
    ctx->h_scratch[0] = init[0];
    ctx->h_scratch[1] = init[1];
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_scratch, ctx->h_scratch, 16, cudaMemcpyHostToDevice, ctx->stream));
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        minmax_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(rec, n, xf, ctx->d_scratch);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scratch + 2, ctx->d_scratch, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    u64 mn = ctx->h_scratch[2], mx = ctx->h_scratch[3];
    *base = mn;
    u64 span = mx - mn;
    int t = 0;
    while (t < 64 && (span >> t) != 0) ++t;
    *top = t;
    return DAMPR_OK;
}

}  // namespace

// shared with merge.cu: sort-only entry over a raw device range (data in `cur`, result in `cur`)
int kv_sort_device_range(dampr_ctx *ctx, ulonglong2 *cur, ulonglong2 *alt, u64 n, int xf) {
    if (n < 2) return DAMPR_OK;
    u64 base;
    int top;
    int rc = key_range(ctx, cur, n, xf, &base, &top, false);
    if (rc) return rc;
    return sort_range(ctx, cur, alt, 0, n, xf, base, top, -1, nullptr, nullptr, 0, cur, true);
}

extern "C" {

int32_t dampr_set_option(const char *name, int64_t value) {
    if (!name) return DAMPR_ERR_ARG;
    if (!strcmp(name, "scatter_tma")) {
        g_use_tma = value != 0;
        return DAMPR_OK;
    }
    if (!strcmp(name, "kv_scatter")) {
        if (value < 1 || value > 3) return DAMPR_ERR_ARG;
        g_kv_scatter = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "kv_hist")) {
        if (value != 1 && value != 2) return DAMPR_ERR_ARG;
        g_kv_hist = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "kv_cluster")) {
        g_kv_cluster = value != 0;
        return DAMPR_OK;
    }
    if (!strcmp(name, "kv_hints")) {
        g_kv_hints = value != 0;
        return DAMPR_OK;
    }
    if (!strcmp(name, "kv_max_bits")) {
        if (value < 4 || value > P2_MAX_BITS) return DAMPR_ERR_ARG;
        g_kv_max_bits = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "text_ctas")) {
        if (value < 2 || value > 4) return DAMPR_ERR_ARG;
        g_text_ctas = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "kv_leaf_target")) {
        if (value < 64 || value > (int64_t)L_CAP) return DAMPR_ERR_ARG;
        g_kv_leaf_target = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "file_cufile")) {
        if (value != 0 && value != 1) return DAMPR_ERR_ARG;
        g_file_cufile = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "cufile_threads")) {
        if (value < 1 || value > 64) return DAMPR_ERR_ARG;
        g_cufile_threads = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "host_threads")) {
        if (value < 1 || value > 256) return DAMPR_ERR_ARG;
        g_host_threads_cap = (int)value;
        return DAMPR_OK;
    }
    if (!strcmp(name, "text_kernel")) {
        if (value != 1 && value != 2) return DAMPR_ERR_ARG;
        g_text_kernel = (int)value;
        return DAMPR_OK;
    }
    return DAMPR_ERR_ARG;
}

int32_t dampr_kv_sort(dampr_ctx *ctx, dampr_kv *kv, int32_t key_xf) {
    ARG_CHECK(ctx, ctx && kv, "null");
    CtxScope scope_(ctx);
    ARG_CHECK(ctx, key_xf >= 0 && key_xf <= DAMPR_KEY_F64, "unknown key transform");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    if (kv->n < 2) return DAMPR_OK;
    int rc = ensure_alt(ctx, kv);
    if (rc) return rc;
    u64 base;
    int top;
    rc = key_range(ctx, kv->rec, kv->n, key_xf, &base, &top, false);
    if (rc) return rc;
    return sort_range(ctx, kv->rec, kv->alt, 0, kv->n, key_xf, base, top, -1, nullptr, nullptr, 0, kv->rec, true);
}

int32_t dampr_kv_sort_reduce(dampr_ctx *ctx, dampr_kv *kv, int32_t key_xf, int32_t op, dampr_kv **out) {
    ARG_CHECK(ctx, ctx && kv && out, "null");
    CtxScope scope_(ctx);
    ARG_CHECK(ctx, key_xf >= 0 && key_xf <= DAMPR_KEY_F64, "unknown key transform");
    ARG_CHECK(ctx, op >= 0 && op <= DAMPR_OP_LAST, "unknown reduce op");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    int rc = dampr_kv_create(ctx, kv->n, out);  // at most n groups
    if (rc) return rc;
    if (kv->n == 0) return DAMPR_OK;
    rc = ensure_alt(ctx, kv);
    if (rc) return rc;
    u64 base;
    int top;
    rc = key_range(ctx, kv->rec, kv->n, key_xf, &base, &top, false);
    if (rc) return rc;
    u64 g = 0;
    rc = sort_range(ctx, kv->rec, kv->alt, 0, kv->n, key_xf, base, top, op, (*out)->rec, &g, 0, nullptr, true);
    if (rc) return rc;
    (*out)->n = g;
    // the partition levels ping-pong between the two buffers of `kv` and the leaves stage their group
    // records in whichever is free: the input is consumed
    kv->n = 0;
    return DAMPR_OK;
}

int32_t dampr_kv_group_offsets(dampr_ctx *ctx, dampr_kv *sorted, uint64_t *offsets, uint64_t cap,
                               uint64_t *n_groups) {
    ARG_CHECK(ctx, ctx && sorted && n_groups, "null");
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    const u64 n = sorted->n;
    if (n == 0) {
        *n_groups = 0;
        if (offsets && cap >= 1) offsets[0] = 0;
        return DAMPR_OK;
    }
    const u64 ntiles = (n + 4095) / 4096;
    DevBuf d_cnt, d_base, d_offs;
    CUDA_TRY(ctx, d_cnt.alloc(ntiles * 4));
    CUDA_TRY(ctx, d_base.alloc((ntiles + 1) * 8));
    {
        ScopedTimer tm(ctx, DAMPR_K_SEG_REDUCE);
        group_heads_kernel<<<(unsigned)ntiles, 512, 0, ctx->stream>>>(sorted->rec, n, nullptr, 0, nullptr, (u64 *)d_cnt.p);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        scan_u32_to_u64_kernel<<<1, 1024, 0, ctx->stream>>>((const u32 *)d_cnt.p, (u64 *)d_base.p, (u32)ntiles);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    u64 total = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(&total, (u64 *)d_base.p + ntiles, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    *n_groups = total;
    if (!offsets) return DAMPR_OK;
    ARG_CHECK(ctx, cap >= total + 1, "offsets array too small (need n_groups + 1)");
    CUDA_TRY(ctx, d_offs.alloc((total + 1) * 8));
    {
        ScopedTimer tm(ctx, DAMPR_K_SEG_REDUCE);
        group_heads_kernel<<<(unsigned)ntiles, 512, 0, ctx->stream>>>(sorted->rec, n, (u64 *)d_offs.p, total,
                                                                     (u64 *)d_base.p, nullptr);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(offsets, d_offs.p, total * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    offsets[total] = n;
    return DAMPR_OK;
}

// destination-contiguous split for the exchange: owner = mix64(key) % n_dest
int32_t dampr_kv_partition_by_owner(dampr_ctx *ctx, dampr_kv *kv, int32_t n_dest, dampr_kv **out,
                                    uint64_t *counts_host) {
    ARG_CHECK(ctx, ctx && kv && out && counts_host, "null");
    CtxScope scope_(ctx);
    ARG_CHECK(ctx, n_dest >= 1 && n_dest <= P1_MAX_NB, "n_dest out of range");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    int rc = dampr_kv_create(ctx, kv->n, out);
    if (rc) return rc;
    (*out)->n = kv->n;
    if (kv->n == 0) {
        for (int i = 0; i < n_dest; ++i) counts_host[i] = 0;
        return DAMPR_OK;
    }
    std::vector<u64> seg_off{0, kv->n};
    DigitSpec ds{DAMPR_KEY_RAW, 0, 0, 0, n_dest};
    rc = partition_level(ctx, kv->rec, (*out)->rec, 0, kv->n, seg_off, ds, (u32)n_dest);
    if (rc) return rc;
    for (int i = 0; i < n_dest; ++i) counts_host[i] = seg_off[i + 1] - seg_off[i];
    return DAMPR_OK;
}

}  // extern "C"

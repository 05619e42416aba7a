// leaf.cuh — shared-memory sort / fold of up to 4096 records by one CTA: the building block of the leaf
// kernels (kv.cu) and of the k-way merge tiles (merge.cu).
#pragma once
#include "common.cuh"

namespace {

constexpr int L_THREADS = 512;
constexpr int L_CAP = 4096;    // records per leaf CTA
constexpr int L_BINS = 8192;   // counting-sort bins
constexpr int L_IPT = L_CAP / L_THREADS;  // 8
constexpr int L_HEAVY = 32;    // bins above this population are sorted by a warp when they hold one key

// ---- leaves ------------------------------------------------------------------------------------------
struct LeafChunk {
    u64 start;      // first record
    u32 n;          // records, <= L_CAP
    int bin_shift;  // bin = ((xf(key) - base) >> bin_shift) - bin_base
    u64 bin_base;
    u32 entry;      // first entry of the chunk in the (start, groups) table of the reduce path
    u32 pad;
};

struct LeafSmem {
    alignas(16) u64 sk[L_CAP];  // key_xform(key) - base
    u64 val[L_CAP];
    u16 cnt[L_BINS];  // counts, then bin starts (hash path: slot -> record index + 1)
    u16 ord[L_CAP];   // bin order -> record index (hash path: representative flags)
    u16 fin[L_CAP];   // final order -> record index
    u32 heavy_bm[(L_THREADS / 32) * (L_CAP / 32)];  // leaf_sort_heavy_bins: per warp, a presence bitmap of record indices
    u32 heavy_flag[L_BINS / 32];                    // leaf_sort_heavy_bins: a bit per heavy bin that holds one key
    // Unused bytes that keep `wsum` at its offset. Moving it makes ptxas schedule leaf_sort_kernel and
    // merge_tile_kernel differently: on an H100 80GB HBM3 at 700 W, the leaves of a 1e8-record sort took 8 %
    // less time and an 8-run merge of 1e8 records 0.4 % more. That trade is for a change of its own.
    u32 unused[401];
    u32 wsum[32];
};

__device__ __forceinline__ u64 apply_op(int op, u64 acc, u64 v) {
    switch (op) {
        case DAMPR_OP_SUM_I64: return acc + v;
        case DAMPR_OP_COUNT: return acc + v;
        case DAMPR_OP_SUM_F64: return (u64)__double_as_longlong(__longlong_as_double((long long)acc) + __longlong_as_double((long long)v));
        case DAMPR_OP_MIN_I64: return ((long long)v < (long long)acc) ? v : acc;
        case DAMPR_OP_MAX_I64: return ((long long)v > (long long)acc) ? v : acc;
        case DAMPR_OP_MIN_F64: return (__longlong_as_double((long long)v) < __longlong_as_double((long long)acc)) ? v : acc;
        case DAMPR_OP_MAX_F64: return (__longlong_as_double((long long)v) > __longlong_as_double((long long)acc)) ? v : acc;
        case DAMPR_OP_FIRST: return acc;
        case DAMPR_OP_LAST: return v;
    }
    return acc;
}

__device__ __forceinline__ bool hash_fold_op(int xf, int op) {
    return xf == DAMPR_KEY_MIX &&
           (op == DAMPR_OP_SUM_I64 || op == DAMPR_OP_COUNT || op == DAMPR_OP_MIN_I64 || op == DAMPR_OP_MAX_I64);
}

// block-wide exclusive scan of one u32 per thread (L_THREADS threads); returns the exclusive prefix,
// *total receives the block total. Contains two __syncthreads.
__device__ __forceinline__ u32 block_excl_scan(LeafSmem &s, u32 x, u32 *total) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 v = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if ((int)lane >= d) v += o;
    }
    __syncthreads();  // wsum may still be read by a previous scan
    if (lane == 31) s.wsum[warp] = v;
    __syncthreads();
    u32 woff = 0, tot = 0;
    for (u32 w = 0; w < L_THREADS / 32; ++w) {
        const u32 ws = s.wsum[w];
        if (w < warp) woff += ws;
        tot += ws;
    }
    *total = tot;
    return woff + v - x;
}

// Counting sort of the n records held in s.sk (+ s.val): the first half — one atomic per record whose return
// value is the record's (arbitrary) slot inside its bin, exclusive scan of the bin counts (s.cnt then holds the
// bin starts), every record's index dropped into its bin's range of s.ord. slot[k] = bin << 16 | slot for the
// thread's records i = tid + k * L_THREADS. Ends with a barrier.
__device__ __forceinline__ bool leaf_bin_records(LeafSmem &s, u32 n, int bin_shift, u64 bin_base, u32 (&slot)[L_IPT]) {
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {
        uint4 *z = reinterpret_cast<uint4 *>(s.cnt);  // 8 counters per 16-byte store
        for (u32 i = tid; i < L_BINS / 8; i += L_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    // u16 counters packed two per u32 word, updated through the word
    u32 *cnt32 = reinterpret_cast<u32 *>(s.cnt);
#pragma unroll
    for (int k = 0; k < L_IPT; ++k) {
        const u32 i = tid + k * L_THREADS;
        slot[k] = 0;
        if (i < n) {
            const u64 bin64 = (s.sk[i] >> bin_shift) - bin_base;
            const u32 bin = (u32)min(bin64, (u64)(L_BINS - 1));
            const u32 old = atomicAdd(&cnt32[bin >> 1], (bin & 1) ? 0x10000u : 1u);
            slot[k] = ((bin & 1) ? (old >> 16) : (old & 0xFFFFu)) | (bin << 16);
        }
    }
    __syncthreads();
    // exclusive scan of cnt[0..L_BINS): 16 bins per thread
    bool heavy = false;
    {
        u32 loc[16];
        u32 sum = 0;
        {
            const uint4 *c4 = reinterpret_cast<const uint4 *>(s.cnt) + tid * 2;
            const uint4 a = c4[0], b = c4[1];
            const u32 w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                loc[2 * k] = w[k] & 0xFFFFu;
                loc[2 * k + 1] = w[k] >> 16;
                sum += loc[2 * k] + loc[2 * k + 1];
                heavy |= (loc[2 * k] > (u32)L_HEAVY) | (loc[2 * k + 1] > (u32)L_HEAVY);
            }
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
        u32 w[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const u32 lo = run;
            run += loc[2 * k];
            w[k] = lo | (run << 16);
            run += loc[2 * k + 1];
        }
        uint4 *c4 = reinterpret_cast<uint4 *>(s.cnt) + tid * 2;  // bin starts
        c4[0] = make_uint4(w[0], w[1], w[2], w[3]);
        c4[1] = make_uint4(w[4], w[5], w[6], w[7]);
    }
    heavy = __syncthreads_or(heavy ? 1 : 0) != 0;
#pragma unroll
    for (int k = 0; k < L_IPT; ++k) {
        const u32 i = tid + k * L_THREADS;
        if (i < n) s.ord[s.cnt[slot[k] >> 16] + (slot[k] & 0xFFFFu)] = (u16)i;
    }
    __syncthreads();
    return heavy;
}

// Heavy bins (many records of ONE key: duplicate-heavy inputs) would cost every member a walk over the whole
// bin. A warp checks that the bin holds a single key and, if so, sorts the bin's record indices through a
// presence bitmap (O(members + 128)); the bin is flagged and its members take their rank by binary search.
__device__ __forceinline__ void leaf_sort_heavy_bins(LeafSmem &s, u32 n) {
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    u32 *flags = s.heavy_flag;
    u32 *bm = s.heavy_bm + warp * (L_CAP / 32);
    if (tid < L_BINS / 32) flags[tid] = 0;
    __syncthreads();
    constexpr u32 BPW = L_BINS / (L_THREADS / 32);  // bins per warp
    for (u32 b = warp * BPW; b < (warp + 1) * BPW; b += 32) {
        const u32 st = s.cnt[b + lane];
        const u32 en = (b + lane + 1 < (u32)L_BINS) ? s.cnt[b + lane + 1] : n;
        u32 hm = __ballot_sync(0xFFFFFFFFu, en - st > (u32)L_HEAVY);
        while (hm) {
            const u32 l = (u32)__ffs(hm) - 1u;
            hm &= hm - 1;
            const u32 hst = __shfl_sync(0xFFFFFFFFu, st, l), hen = __shfl_sync(0xFFFFFFFFu, en, l);
            const u64 k0 = s.sk[s.ord[hst]];
            bool eq = true;
            for (u32 j = hst + lane; j < hen; j += 32) eq &= s.sk[s.ord[j]] == k0;
            if (!__all_sync(0xFFFFFFFFu, eq)) continue;  // several keys share the bin: the member walk handles it
            for (u32 w = lane; w < (u32)(L_CAP / 32); w += 32) bm[w] = 0;
            __syncwarp();
            for (u32 j = hst + lane; j < hen; j += 32) {
                const u32 x = s.ord[j];
                atomicOr(&bm[x >> 5], 1u << (x & 31));
            }
            __syncwarp();
            constexpr int WPL = L_CAP / 32 / 32;
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
            u32 pos = hst + v - cl;
#pragma unroll
            for (int k = 0; k < WPL; ++k) {
                u32 wd = words[k];
                while (wd) {
                    const u32 bit = __ffs(wd) - 1;
                    wd &= wd - 1;
                    s.ord[pos++] = (u16)((lane * WPL + k) * 32 + bit);
                }
            }
            __syncwarp();
            if (lane == 0) atomicOr(&flags[(b + l) >> 5], 1u << ((b + l) & 31));
        }
    }
    __syncthreads();
}

// second half: the final position of record i — its bin's start plus its rank inside the bin by (key, smem index),
// the smem index being the record's input position
__device__ __forceinline__ u32 leaf_final_pos(const LeafSmem &s, u32 n, u32 i, u32 slotinfo, bool heavy = false) {
    const u32 bin = slotinfo >> 16;
    const u32 st = s.cnt[bin];
    const u32 en = (bin + 1 < L_BINS) ? s.cnt[bin + 1] : n;
    u32 r = 0;
    if (heavy && en - st > (u32)L_HEAVY && ((s.heavy_flag[bin >> 5] >> (bin & 31)) & 1u)) {
        // single-key bin whose indices a warp sorted (leaf_sort_heavy_bins): rank = lower bound of my index
        u32 lo = st, hi = en;
        while (lo < hi) {
            const u32 mid = (lo + hi) >> 1;
            if (s.ord[mid] < i) lo = mid + 1;
            else hi = mid;
        }
        return lo;
    }
    if (en - st > 1) {
        const u64 ki = s.sk[i];
        for (u32 j = st; j < en; ++j) {
            const u32 o = s.ord[j];
            const u64 ko = s.sk[o];
            r += (ko < ki || (ko == ki && o < i)) ? 1u : 0u;
        }
    }
    return st + r;
}

// Sort the n records held in s.sk / s.val. Result: s.fin[position] = record index.
__device__ __forceinline__ void leaf_sort_core(LeafSmem &s, u32 n, int bin_shift, u64 bin_base) {
    const u32 tid = threadIdx.x;
    u32 slot[L_IPT];
    const bool heavy = leaf_bin_records(s, n, bin_shift, bin_base, slot);
    if (heavy) leaf_sort_heavy_bins(s, n);
#pragma unroll
    for (int k = 0; k < L_IPT; ++k) {
        const u32 i = tid + k * L_THREADS;
        if (i < n) s.fin[leaf_final_pos(s, n, i, slot[k], heavy)] = (u16)i;
    }
    __syncthreads();
}

// commutative integer folds under the MIX order (a_group_by(...).sum()/count()/min()/max()): no sort.
// Every record looks its key up in a shared-memory index (slot -> first record holding the key) and folds
// its value into that record with a shared-memory atomic. Writes one record per key (in record order) to
// out[0..groups) and returns the group count.
__device__ __forceinline__ u32 leaf_hash_fold(LeafSmem &s, u32 n, int reduce_op, int xf, u64 base,
                                              ulonglong2 *__restrict__ out) {
    const u32 tid = threadIdx.x;
    {
        uint4 *z = reinterpret_cast<uint4 *>(s.cnt);
        for (u32 i = tid; i < L_BINS / 8; i += L_THREADS) z[i] = make_uint4(0, 0, 0, 0);
        uint4 *z2 = reinterpret_cast<uint4 *>(s.ord);
        for (u32 i = tid; i < L_CAP / 8; i += L_THREADS) z2[i] = make_uint4(0, 0, 0, 0);
    }
    if (reduce_op == DAMPR_OP_COUNT)
        for (u32 i = tid; i < n; i += L_THREADS) s.val[i] = 1ULL;
    __syncthreads();
    for (u32 i = tid; i < n; i += L_THREADS) {
        const u64 ki = s.sk[i];
        u32 slot = (u32)(ki >> 13) & (L_BINS - 1);  // the partition consumed the top bits
        slot = (slot ^ (u32)(ki >> 37)) & (L_BINS - 1);
        for (;;) {
            u32 cur = s.cnt[slot];
            if (cur == 0) {
                cur = atomicCAS(&s.cnt[slot], (unsigned short)0, (unsigned short)(i + 1));
                if (cur == 0) {
                    s.ord[i] = 1;  // this record represents its key
                    break;
                }
            }
            if (s.sk[cur - 1] == ki) {
                unsigned long long *acc = &s.val[cur - 1];
                const u64 v = s.val[i];
                if (reduce_op == DAMPR_OP_MIN_I64) atomicMin((long long *)acc, (long long)v);
                else if (reduce_op == DAMPR_OP_MAX_I64) atomicMax((long long *)acc, (long long)v);
                else atomicAdd(acc, v);
                break;
            }
            slot = (slot + 1) & (L_BINS - 1);
        }
    }
    __syncthreads();
    u32 flags = 0;
#pragma unroll
    for (int k = 0; k < L_IPT; ++k) {
        const u32 p = tid * L_IPT + k;
        if (p < n && s.ord[p]) flags |= 1u << k;
    }
    u32 total;
    u32 gidx = block_excl_scan(s, __popc(flags), &total);
#pragma unroll
    for (int k = 0; k < L_IPT; ++k)
        if (flags & (1u << k)) {
            const u32 p = tid * L_IPT + k;
            out[gidx++] = make_ulonglong2(key_unxform(s.sk[p] + base, xf), s.val[p]);
        }
    return total;
}

// segmented reduce over the sorted order s.fin: one thread per group head walks its group. Positions are dealt
// to the threads warp by warp, 32 consecutive positions per round (conflict-free shared-memory reads; the
// blocked layout of the first build cost 16-way bank conflicts), head ranks come from ballots.
__device__ __forceinline__ u32 leaf_seg_reduce(LeafSmem &s, u32 n, int reduce_op, int xf, u64 base,
                                               ulonglong2 *__restrict__ out) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32 lt = (1u << lane) - 1u;
    const u16 *fin = s.fin;
    u32 headbits = 0, run = 0;
    u32 rank[L_IPT];
#pragma unroll
    for (int k = 0; k < L_IPT; ++k) {
        const u32 p = warp * (32u * L_IPT) + k * 32u + lane;
        bool head = false;
        if (p < n) head = (p == 0) || (s.sk[fin[p]] != s.sk[fin[p - 1]]);
        const u32 b = __ballot_sync(0xFFFFFFFFu, head);
        rank[k] = run + (u32)__popc(b & lt);
        run += (u32)__popc(b);
        headbits |= head ? (1u << k) : 0u;
    }
    __syncthreads();  // wsum may still be read by an earlier scan
    if (lane == 0) s.wsum[warp] = run;
    __syncthreads();
    u32 woff = 0, total = 0;
    for (u32 w = 0; w < L_THREADS / 32; ++w) {
        const u32 ws = s.wsum[w];
        if (w < warp) woff += ws;
        total += ws;
    }
#pragma unroll
    for (int k = 0; k < L_IPT; ++k) {
        if (headbits & (1u << k)) {
            const u32 p = warp * (32u * L_IPT) + k * 32u + lane;
            const u64 ksk = s.sk[fin[p]];
            u64 acc = (reduce_op == DAMPR_OP_COUNT) ? 1ULL : s.val[fin[p]];
            for (u32 q = p + 1; q < n && s.sk[fin[q]] == ksk; ++q) {
                const u64 val = (reduce_op == DAMPR_OP_COUNT) ? 1ULL : s.val[fin[q]];
                acc = apply_op(reduce_op, acc, val);
            }
            out[woff + rank[k]] = make_ulonglong2(key_unxform(ksk + base, xf), acc);
        }
    }
    return total;
}

// exclusive scan of u32 counts into u64 offsets (single CTA, sequential over blocks of 1024)
__global__ void scan_u32_to_u64_kernel(const u32 *__restrict__ in, u64 *__restrict__ out, u32 n) {
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


}  // namespace

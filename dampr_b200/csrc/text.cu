// text.cu — K0/K1/K2: line ownership + tokenise + normalise + key code + map-side combine.
//
// Replaces, for the lowered text idioms, the reference's per-record Python in the map stage:
//   TextLineDataset.read      dampr/dataset.py:458-476  (line ownership, '\n' stripping)
//   Map.stream(user lambdas)  dampr/base.py:30-33 with examples/wc.py:12 (`x.split()`) and
//                             benchmarks/tf-idf-dampr.py:12-14 (`set(RX.split(x.lower()))`)
//   ReducedWriter.add_record  dampr/dataset.py:100-105  (dict combiner, binop = +1)
//
// Design: persistent CTAs, 2 per SM. Each CTA owns 6 KB tiles of the text; a tile is
// pulled into shared memory with one TMA 1-D bulk copy (cp.async.bulk + mbarrier), classified
// 4 bytes at a time with SWAR arithmetic into bit masks (word chars, newlines), token starts are
// ranked with a block scan, every token start is walked once to produce a 64-bit key code
// (exact base-38 / 7-bit packing for short tokens, seeded hash with bit 63 set for long ones),
// per-line de-duplication (set() semantics) is a backward scan over the token array, and the
// survivors are folded into a per-CTA shared-memory hash table that is flushed to the global
// (L2-resident) table once per CTA. HBM traffic = the text, read once.
#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <thread>

#include <charconv>
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <cmath>
#include <limits>

#include "common.cuh"

namespace {

constexpr int T_THREADS = 256;
constexpr int T_LEAD = 32;
constexpr int T_OWN = 6144;
constexpr int T_HALO = 4096;
constexpr int T_WIN = T_LEAD + T_OWN + T_HALO;  // 10272
constexpr int T_WORDS = T_WIN / 32;             // 321
constexpr int T_TOKCAP = (T_WIN - T_LEAD) / 2 + 16;
constexpr int T_STAB = 2048;  // shared-memory combiner entries
constexpr int T_STAB_PROBES = 12;
constexpr u32 G_MAX_PROBES = 1u << 14;

static_assert(T_WIN % 32 == 0, "window must be a whole number of mask words");
static_assert(TEXT_LEAD >= T_LEAD, "textbuf lead-in too small");
static_assert(TEXT_TAIL_PAD >= T_WIN + 64, "textbuf tail pad too small");

struct TableView {
    u64 *keys;
    u64 *counts;
    u64 *reps;
    u64 *stats;
    u64 mask;
    u64 seed;
};

// stats slots
enum { ST_ENTRIES = 0, ST_LINES = 1, ST_EMPTY = 2, ST_FOLDED = 3, ST_FLAGS = 4, ST_LONG = 5, ST_RAW = 6 };

struct Smem {
    alignas(16) u8 text[T_WIN];
    u32 w[T_WORDS + 3];
    u32 nl[T_WORDS + 3];
    u32 pre[T_WORDS + 3];  // exclusive prefix: (newlines << 16) | token starts
    alignas(8) u64 tkey[T_TOKCAP];
    u16 tline[T_TOKCAP];
    u16 tpos[T_TOKCAP];
    alignas(8) u64 tabk[T_STAB];
    u32 tabc[T_STAB];
    alignas(8) u64 bar;
    u32 q0;
    u32 tl;
    u32 warp_sum[T_THREADS / 32];
    u32 ntok;
    u32 flags;
    u8 lut[128];
};

// ---- SWAR classification of 4 ASCII bytes -------------------------------------------------
__device__ __forceinline__ u32 ge7(u32 x7, u32 k) {  // bit7 of each byte set iff byte >= k (bytes < 0x80)
    return (x7 + (0x80u - k) * 0x01010101u) & 0x80808080u;
}
__device__ __forceinline__ u32 eq7(u32 x7, u32 k) {  // bit7 set iff byte == k
    u32 z = x7 ^ (k * 0x01010101u);
    return ~(z + 0x7F7F7F7Fu) & 0x80808080u;
}
__device__ __forceinline__ u32 movemask4(u32 hi) {  // bits 7,15,23,31 -> bits 0..3
    return (((hi >> 7) & 0x01010101u) * 0x01020408u) >> 24;
}

template <int MODE>
__device__ __forceinline__ void classify4(u32 x, u32 &wbits, u32 &nlbits, u32 &bad) {
    u32 x7 = x & 0x7F7F7F7Fu;
    u32 hi = x & 0x80808080u;
    bad |= hi;
    u32 nl = eq7(x7, 0x0A) & ~hi;
    u32 word;
    if (MODE == DAMPR_TOK_WS) {
        // str.split() whitespace: 0x09-0x0D, 0x1C-0x1F, 0x20
        u32 ws = (ge7(x7, 0x09) & ~ge7(x7, 0x0E)) | (ge7(x7, 0x1C) & ~ge7(x7, 0x21));
        word = ~ws & 0x80808080u;
    } else {
        // \w for ASCII: [0-9A-Za-z_]; a '\r' makes universal-newline semantics differ -> flag
        u32 y = x7 | 0x20202020u;
        u32 alpha = ge7(y, 0x61) & ~ge7(y, 0x7B);
        u32 digit = ge7(x7, 0x30) & ~ge7(x7, 0x3A);
        u32 us = eq7(x7, 0x5F);
        word = (alpha | digit | us);
    }
    // a '\r' ends a line under universal newlines: tokens of the \w modes and the LINE COUNT of every mode then
    // differ from what this kernel computes -> flag (bit6, kept apart from the non-ASCII bit7); str.split token
    // counts are unaffected ('\r' is whitespace) and the host ignores the flag for them
    bad |= (eq7(x7, 0x0D) >> 1);
    word &= ~hi;
    wbits = movemask4(word);
    nlbits = movemask4(nl);
}

__device__ __forceinline__ bool wbit(const Smem &s, u32 pos) { return (s.w[pos >> 5] >> (pos & 31)) & 1u; }

// insert into the global table
__device__ __forceinline__ void gtab_add(const TableView &t, u64 key, u64 cnt, u64 rep) {
    u64 slot = mix64(key) & t.mask;
    for (u32 probe = 0; probe < G_MAX_PROBES; ++probe) {
        u64 k = *((volatile u64 *)&t.keys[slot]);
        if (k == 0) {
            k = atomicCAS(&t.keys[slot], 0ULL, key);
            if (k == 0) {
                atomicAdd(&t.stats[ST_ENTRIES], 1ULL);
                k = key;
            }
        }
        if (k == key) {
            atomicAdd(&t.counts[slot], cnt);
            if (rep != ~0ULL) atomicMin(&t.reps[slot], rep);
            return;
        }
        slot = (slot + 1) & t.mask;
    }
    atomicOr(&t.stats[ST_FLAGS], (u64)DAMPR_TF_TABLEFULL);
}

__device__ __forceinline__ long long gtab_find(const TableView &t, u64 key) {
    u64 slot = mix64(key) & t.mask;
    for (u32 probe = 0; probe < G_MAX_PROBES; ++probe) {
        u64 k = t.keys[slot];
        if (k == key) return (long long)slot;
        if (k == 0) return -1;
        slot = (slot + 1) & t.mask;
    }
    return -1;
}

template <int MODE>
__device__ __forceinline__ u32 norm_byte(const Smem &s, u32 c) {
    if (MODE == DAMPR_TOK_WS) return c;
    return s.lut[c & 127];
}

// key code of the token starting at window position pos (len bytes; may run past the window,
// in which case the remainder is read from global memory at gtext + gpos)
template <int MODE>
__device__ u64 token_code(const Smem &s, u32 pos, u32 len, const u8 *gtok, u64 seed, bool &hashed) {
    constexpr u32 MAXEXACT = (MODE == DAMPR_TOK_WS) ? 9u : 12u;
    bool exact = len <= MAXEXACT;
    if (exact) {
        u64 code = 0;
        bool nul = false;
        for (int i = (int)len - 1; i >= 0; --i) {
            u32 c = s.text[pos + i];
            if (MODE == DAMPR_TOK_WS) {
                nul |= (c == 0);
                code = (code << 7) | (c & 127);
            } else {
                code = code * 38ULL + s.lut[c & 127];
            }
        }
        if (!nul) {
            hashed = false;
            return code;
        }
    }
    hashed = true;
    u32 h1 = (u32)seed ^ 0x811C9DC5u, h2 = (u32)(seed >> 32) ^ 0x9747B28Cu;
    for (u32 i = 0; i < len; ++i) {
        u32 c = (pos + i < (u32)T_WIN) ? (u32)s.text[pos + i] : (u32)gtok[i];
        u32 v = norm_byte<MODE>(s, c);
        h1 = (h1 ^ v) * 16777619u;
        h2 = (h2 ^ v) * 0x85EBCA6Bu + 0x9E3779B9u;
        h2 = (h2 << 13) | (h2 >> 19);
    }
    u64 h = mix64((((u64)h1) << 32 | h2) ^ ((u64)len * 0x9E3779B97F4A7C15ULL));
    return h | 0x8000000000000000ULL;
}

// length of the token starting at window position pos
template <int MODE>
__device__ u32 token_len(const Smem &s, u32 pos, const u8 *gtok) {
    u32 wi = pos >> 5, bi = pos & 31;
    u32 m = (~s.w[wi]) >> bi;
    if (m) return (u32)__ffs(m) - 1u;
    u32 len = 32 - bi;
    for (++wi; wi < (u32)T_WORDS; ++wi) {
        m = ~s.w[wi];
        if (m) return len + (u32)__ffs(m) - 1u;
        len += 32;
    }
    // token runs past the window: continue in global memory (tail pad guarantees a terminator)
    for (;; ++len) {
        u32 c = gtok[len];
        bool word;
        if (MODE == DAMPR_TOK_WS)
            word = !((c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x20)) && c < 0x80;
        else
            word = ((c | 0x20) >= 0x61 && (c | 0x20) <= 0x7A) || (c >= 0x30 && c <= 0x39) || c == 0x5F;
        if (!word) return len;
        if (len > (1u << 30)) return len;
    }
}

template <int MODE, bool VERIFY>
__global__ void __launch_bounds__(T_THREADS, 2)
text_count_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, u64 base_offset,
                  TableView tab) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x;
    const u64 ntiles = (own_hi - own_lo + T_OWN - 1) / T_OWN;

    if (tid == 0) {
        mbar_init(&s.bar, 1);
        fence_mbar_init();
        s.flags = 0;
    }
    for (int i = tid; i < T_STAB; i += T_THREADS) {
        s.tabk[i] = 0;
        s.tabc[i] = 0;
    }
    if (tid < 128) {
        u32 c = tid, v = 0;
        if (c >= '0' && c <= '9') v = c - '0' + 1;
        else if (c == '_') v = 11;
        else if (c >= 'a' && c <= 'z') v = c - 'a' + 12;
        else if (c >= 'A' && c <= 'Z') v = c - 'A' + 12;
        s.lut[tid] = (u8)v;
    }
    __syncthreads();

    u64 acc_lines = 0, acc_empty = 0, acc_folded = 0, acc_long = 0, acc_raw = 0;
    u32 parity = 0;

    for (u64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const u64 sgl = own_lo + tile * (u64)T_OWN;                       // global start of tile
        const u32 own_len = (u32)min((u64)T_OWN, own_hi - sgl);           // owned bytes
        // ---- TMA bulk load of the window [sgl - LEAD, sgl - LEAD + WIN) ----------------------
        if (tid == 0) {
            fence_proxy_async();
            mbar_expect_tx(&s.bar, T_WIN);
            tma_load_1d(s.text, text + sgl - T_LEAD, T_WIN, &s.bar);
            s.q0 = 0xFFFFFFFFu;
            s.tl = 0xFFFFFFFFu;
        }
        __syncthreads();
        mbar_wait(&s.bar, parity);
        parity ^= 1;

        // ---- phase A: classify, build masks, find first owned line start / last terminator ---
        const u32 own_end_w = T_LEAD + own_len;  // window coord one past the owned bytes
        u32 bad = 0;
        for (int i = tid; i < T_WORDS; i += T_THREADS) {
            const uint4 *p = reinterpret_cast<const uint4 *>(s.text + 32 * i);
            uint4 a = p[0], b = p[1];
            u32 wm = 0, nm = 0, wb, nb;
            classify4<MODE>(a.x, wb, nb, bad); wm |= wb;        nm |= nb;
            classify4<MODE>(a.y, wb, nb, bad); wm |= wb << 4;   nm |= nb << 4;
            classify4<MODE>(a.z, wb, nb, bad); wm |= wb << 8;   nm |= nb << 8;
            classify4<MODE>(a.w, wb, nb, bad); wm |= wb << 12;  nm |= nb << 12;
            classify4<MODE>(b.x, wb, nb, bad); wm |= wb << 16;  nm |= nb << 16;
            classify4<MODE>(b.y, wb, nb, bad); wm |= wb << 20;  nm |= nb << 20;
            classify4<MODE>(b.z, wb, nb, bad); wm |= wb << 24;  nm |= nb << 24;
            classify4<MODE>(b.w, wb, nb, bad); wm |= wb << 28;  nm |= nb << 28;
            s.w[i] = wm;
            s.nl[i] = nm;
            if (nm) {
                // first newline at window pos >= LEAD-1  -> q0 = pos+1
                u32 base = 32u * i;
                u32 m0 = nm;
                if (base + 31 < (u32)(T_LEAD - 1)) m0 = 0;
                else if (base < (u32)(T_LEAD - 1)) m0 &= ~((1u << ((T_LEAD - 1) - base)) - 1u);
                if (m0) atomicMin(&s.q0, base + __ffs(m0));  // +1 folded in (ffs is 1-based)
                // first newline at window pos >= own_end_w - 1 -> terminator of last owned line
                u32 lo = own_end_w - 1;
                u32 m1 = nm;
                if (base + 31 < lo) m1 = 0;
                else if (base < lo) m1 &= ~((1u << (lo - base)) - 1u);
                if (m1) atomicMin(&s.tl, base + __ffs(m1) - 1);
            }
        }
        if (bad) atomicOr(&s.flags, ((bad & 0x80808080u) ? DAMPR_TF_NONASCII : 0u) |
                                    ((bad & 0x40404040u) ? DAMPR_TF_CR : 0u));
        __syncthreads();

        // ---- region of token starts handled by this tile -------------------------------------
        u32 rlo, rhi;  // [rlo, rhi) window coords
        if (MODE == DAMPR_TOK_WS) {
            rlo = T_LEAD;
            rhi = own_end_w;
        } else {
            u32 q0 = s.q0, tl = s.tl;
            if (q0 >= own_end_w) {  // no line starts inside this tile
                rlo = rhi = 0;
            } else if (tl == 0xFFFFFFFFu) {  // last owned line does not end inside the window
                rlo = rhi = 0;
                if (tid == 0) atomicOr(&s.flags, DAMPR_TF_LONGLINE);
            } else {
                rlo = q0;
                rhi = tl + 1;
            }
        }

        // ---- phase B: token starts, ranks (block exclusive scan over mask words) -------------
        {
            // each thread owns words 2t and 2t+1
            u32 cnt[2];
            u32 smask[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                int i = 2 * tid + k;
                u32 st = 0, nlm = 0;
                if (i < T_WORDS) {
                    u32 wm = s.w[i];
                    u32 prev = (i > 0) ? (s.w[i - 1] >> 31) : 0u;
                    st = wm & ~((wm << 1) | prev);
                    nlm = s.nl[i];
                    u32 base = 32u * i;
                    // restrict to [rlo, rhi)
                    u32 keep = 0xFFFFFFFFu;
                    if (base + 32 <= rlo || base >= rhi) keep = 0;
                    else {
                        if (base < rlo) keep &= ~((1u << (rlo - base)) - 1u);
                        if (base + 32 > rhi) keep &= (1u << (rhi - base)) - 1u;
                    }
                    st &= keep;
                    nlm &= keep;
                }
                smask[k] = st;
                cnt[k] = (u32)__popc(st) | ((u32)__popc(nlm) << 16);
            }
            u32 tsum = cnt[0] + cnt[1];
            // warp inclusive scan
            u32 v = tsum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                if ((tid & 31) >= d) v += o;
            }
            if ((tid & 31) == 31) s.warp_sum[tid >> 5] = v;
            __syncthreads();
            u32 woff = 0;
#pragma unroll
            for (int wj = 0; wj < T_THREADS / 32; ++wj)
                if (wj < (tid >> 5)) woff += s.warp_sum[wj];
            u32 excl = woff + v - tsum;
            if (2 * tid < T_WORDS) s.pre[2 * tid] = excl;
            if (2 * tid + 1 < T_WORDS) s.pre[2 * tid + 1] = excl + cnt[0];
            if (tid == T_THREADS - 1) s.ntok = (woff + v) & 0xFFFFu;
            // stash start masks in place of nothing: recomputed in phase C (cheap)
            (void)smask;
        }
        __syncthreads();

        // ---- phase C: walk every token start once -> key code, line id ----------------------
        const u8 *gwin = text + sgl - T_LEAD;  // global address of window byte 0
        for (int i = tid; i < T_WORDS; i += T_THREADS) {
            u32 wm = s.w[i];
            u32 prev = (i > 0) ? (s.w[i - 1] >> 31) : 0u;
            u32 st = wm & ~((wm << 1) | prev);
            u32 base = 32u * i;
            u32 keep = 0xFFFFFFFFu;
            if (base + 32 <= rlo || base >= rhi) keep = 0;
            else {
                if (base < rlo) keep &= ~((1u << (rlo - base)) - 1u);
                if (base + 32 > rhi) keep &= (1u << (rhi - base)) - 1u;
            }
            st &= keep;
            u32 nlm = s.nl[i] & keep;
            u32 pre = s.pre[i];
            u32 tix = pre & 0xFFFFu;
            u32 lbase = pre >> 16;
            while (st) {
                u32 b = (u32)__ffs(st) - 1u;
                st &= st - 1;
                u32 pos = base + b;
                u32 len = token_len<MODE>(s, pos, gwin + pos);
                bool hashed;
                u64 code = token_code<MODE>(s, pos, len, gwin + pos, tab.seed, hashed);
                s.tkey[tix] = code;
                s.tline[tix] = (u16)(lbase + __popc(nlm & ((1u << b) - 1u)));
                s.tpos[tix] = (u16)pos;
                ++tix;
            }
        }
        __syncthreads();

        // ---- phase D: per-line de-dup (set semantics) + fold into the combiner ---------------
        const u32 ntok = s.ntok;
        acc_raw += (tid == 0) ? ntok : 0;
        for (u32 t = tid; t < ntok; t += T_THREADS) {
            u64 key = s.tkey[t];
            bool dup = false;
            if (MODE == DAMPR_TOK_NONWORD_LOWER_SET) {
                u16 ln = s.tline[t];
                for (int j = (int)t - 1; j >= 0 && s.tline[j] == ln; --j)
                    if (s.tkey[j] == key) {
                        dup = true;
                        break;
                    }
            }
            bool hashed = (key >> 63) != 0;
            // the de-dup compares codes only: the verify pass still byte-compares a hashed duplicate with the
            // entry's representative, so a different word of the same code on the line sets TF_COLLISION
            if (dup && !(VERIFY && hashed)) continue;
            if (VERIFY) {
                if (hashed) {
                    u32 pos = s.tpos[t];
                    u32 len = token_len<MODE>(s, pos, gwin + pos);
                    long long slot = gtab_find(tab, key);
                    bool ok = slot >= 0;
                    if (ok) {
                        u64 rep = tab.reps[slot];
                        u64 roff = rep >> 20;
                        u32 rlen = (u32)(rep & 0xFFFFFu);
                        ok = (rlen == min(len, 0xFFFFFu)) && roff >= base_offset;
                        if (ok) {
                            const u8 *a = gwin + pos;
                            const u8 *bptr = text + (roff - base_offset);
                            for (u32 i2 = 0; i2 < len; ++i2) {
                                u32 ca = a[i2], cb = bptr[i2];
                                if (MODE != DAMPR_TOK_WS) {
                                    if (ca >= 'A' && ca <= 'Z') ca |= 0x20;
                                    if (cb >= 'A' && cb <= 'Z') cb |= 0x20;
                                }
                                if (ca != cb) {
                                    ok = false;
                                    break;
                                }
                            }
                        }
                    }
                    if (!ok) atomicOr(&s.flags, DAMPR_TF_COLLISION);
                }
                continue;
            }
            acc_folded++;
            if (hashed) {
                u32 pos = s.tpos[t];
                u32 len = token_len<MODE>(s, pos, gwin + pos);
                if (len >= (1u << 20)) {
                    atomicOr(&s.flags, DAMPR_TF_LONGTOKEN);
                    len = (1u << 20) - 1;
                }
                u64 goff = base_offset + (sgl - T_LEAD) + pos;
                gtab_add(tab, key, 1ULL, (goff << 20) | len);
                acc_long++;
                continue;
            }
            u32 slot = (u32)(mix64(key) >> 20) & (T_STAB - 1);
            bool placed = false;
#pragma unroll 1
            for (int pr = 0; pr < T_STAB_PROBES; ++pr) {
                u64 k = s.tabk[slot];
                if (k == 0) {
                    k = atomicCAS(&s.tabk[slot], 0ULL, key);
                    if (k == 0) k = key;
                }
                if (k == key) {
                    atomicAdd(&s.tabc[slot], 1u);
                    placed = true;
                    break;
                }
                slot = (slot + 1) & (T_STAB - 1);
            }
            if (!placed) gtab_add(tab, key, 1ULL, ~0ULL);
        }

        // ---- phase E: owned lines and the '' token -------------------------------------------
        if (!VERIFY) {
            // lines whose first byte lies in [sgl, sgl+own_len): newline at window pos in
            // [LEAD-1, own_end_w-1)
            for (int i = tid; i < T_WORDS; i += T_THREADS) {
                u32 base = 32u * i;
                u32 nm = s.nl[i];
                if (!nm) continue;
                u32 lo = T_LEAD - 1, hi = own_end_w - 1;  // [lo, hi)
                u32 keep = 0xFFFFFFFFu;
                if (base + 32 <= lo || base >= hi) keep = 0;
                else {
                    if (base < lo) keep &= ~((1u << (lo - base)) - 1u);
                    if (base + 32 > hi) keep &= (1u << (hi - base)) - 1u;
                }
                u32 starts = nm & keep;
                // a line start at global position >= n does not exist
                while (starts) {
                    u32 b = (u32)__ffs(starts) - 1u;
                    starts &= starts - 1;
                    u64 gp = sgl - T_LEAD + base + b + 1;  // global position of the line start
                    if (gp < n) acc_lines++;
                }
                if (MODE != DAMPR_TOK_WS && rhi > rlo) {
                    // terminators of owned lines: newline bits inside [rlo, rhi)
                    u32 keep2 = 0xFFFFFFFFu;
                    if (base + 32 <= rlo || base >= rhi) keep2 = 0;
                    else {
                        if (base < rlo) keep2 &= ~((1u << (rlo - base)) - 1u);
                        if (base + 32 > rhi) keep2 &= (1u << (rhi - base)) - 1u;
                    }
                    u32 terms = nm & keep2;
                    while (terms) {
                        u32 b = (u32)__ffs(terms) - 1u;
                        terms &= terms - 1;
                        u32 p = base + b;
                        // the terminator at global n belongs to an unterminated last line only if
                        // that line is non-empty (start < n); a start == n is not a line
                        // find the line start q: previous newline + 1 (>= rlo)
                        u32 q;
                        {
                            int wi = (int)(p >> 5);
                            u32 bi = p & 31;
                            u32 m = s.nl[wi] & ((bi == 0) ? 0u : ((1u << bi) - 1u));
                            for (;;) {
                                if (m) {
                                    q = 32u * wi + (31u - (u32)__clz(m)) + 1u;
                                    break;
                                }
                                --wi;
                                if (wi < 0) {
                                    q = rlo;
                                    break;
                                }
                                m = s.nl[wi];
                            }
                            if (q < rlo) q = rlo;
                        }
                        u64 gq = sgl - T_LEAD + q;
                        if (gq >= n) continue;  // virtual newline after a terminated file
                        bool A = !wbit(s, q);
                        bool B = (p > q) && !wbit(s, p - 1);
                        if (MODE == DAMPR_TOK_NONWORD_LOWER_SET) acc_empty += (A || B) ? 1 : 0;
                        else acc_empty += (A ? 1 : 0) + (B ? 1 : 0);
                    }
                }
            }
        }
        __syncthreads();  // window and token arrays are reused by the next tile
    }

    // ---- flush the shared-memory combiner (ReducedWriter.flush, dataset.py:107-113) -----------
    if (!VERIFY) {
        for (int i = tid; i < T_STAB; i += T_THREADS) {
            u64 k = s.tabk[i];
            if (k) gtab_add(tab, k, (u64)s.tabc[i], ~0ULL);
        }
    }
    // block-reduce the counters
    u64 vals[5] = {acc_lines, acc_empty, acc_folded, acc_long, acc_raw};
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        u64 v = vals[k];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, d);
        vals[k] = v;
    }
    if (!VERIFY && (tid & 31) == 0) {
        if (vals[0]) atomicAdd(&tab.stats[ST_LINES], vals[0]);
        if (vals[1]) atomicAdd(&tab.stats[ST_EMPTY], vals[1]);
        if (vals[2]) atomicAdd(&tab.stats[ST_FOLDED], vals[2]);
        if (vals[3]) atomicAdd(&tab.stats[ST_LONG], vals[3]);
        if (vals[4]) atomicAdd(&tab.stats[ST_RAW], vals[4]);
    }
    __syncthreads();
    if (tid == 0 && s.flags) atomicOr(&tab.stats[ST_FLAGS], (u64)s.flags);
}

__global__ void table_init_kernel(u64 *keys, u64 *counts, u64 *reps, u64 cap, u64 *stats) {
    u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < cap; i += stride) {
        keys[i] = 0;
        counts[i] = 0;
        reps[i] = ~0ULL;
    }
    if (blockIdx.x == 0 && threadIdx.x < 8) stats[threadIdx.x] = 0;
}

__global__ void table_extract_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ counts,
                                     const u64 *__restrict__ reps, u64 cap, u64 *out_codes,
                                     u64 *out_counts, u64 *out_reps, ulonglong2 *out_kv, u64 out_cap,
                                     u64 *cursor) {
    u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < cap; i += stride) {
        u64 k = keys[i];
        bool have = k != 0;
        // warp-aggregated cursor bump
        u32 m = __ballot_sync(0xFFFFFFFFu, have);
        u64 base = 0;
        if (m) {
            int leader = __ffs(m) - 1;
            if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(cursor, (u64)__popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
        }
        if (have) {
            u64 idx = base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
            if (idx < out_cap) {
                if (out_kv) out_kv[idx] = make_ulonglong2(k, counts[i]);
                if (out_codes) out_codes[idx] = k;
                if (out_counts) out_counts[idx] = counts[i];
                if (out_reps) {
                    u64 r = reps[i];
                    out_reps[idx] = (r == ~0ULL) ? 0ULL : r;
                }
            }
        }
    }
}

template <int MODE, bool VERIFY>
int launch_text(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 lo, u64 hi) {
    if (hi <= lo) return DAMPR_OK;
    size_t smem = sizeof(Smem);
    auto kern = text_count_kernel<MODE, VERIFY>;
    CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    u64 ntiles = (hi - lo + T_OWN - 1) / T_OWN;
    u64 grid = (u64)ctx->num_sms * 2;
    if (grid > ntiles) grid = ntiles;
    TableView tv{t->keys, t->counts, t->reps, t->stats, t->cap - 1, 0x243F6A8885A308D3ULL};
    wait_uploads(ctx);
    {
        ScopedTimer tm(ctx, VERIFY ? DAMPR_K_TEXT_VERIFY : DAMPR_K_TEXT_COUNT);
        kern<<<(unsigned)grid, T_THREADS, smem, ctx->stream>>>(tb->text, tb->n, lo, hi, 0, tv);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

}  // namespace

extern "C" {

int32_t dampr_table_create(dampr_ctx *ctx, uint32_t capacity_log2, dampr_table **out) {
    ARG_CHECK(ctx, ctx && out, "null");
    ARG_CHECK(ctx, capacity_log2 >= 10 && capacity_log2 <= 32, "table capacity_log2 out of range");
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    dampr_table *t = new dampr_table();
    t->cap_log2 = capacity_log2;
    t->cap = 1ULL << capacity_log2;
    t->keys = t->counts = t->reps = t->stats = t->fb = t->tiles = t->ext = nullptr;
    t->ext_cap = t->ext_n = 0;
    t->fb_cap = 1u << 16;
    if (cudaMalloc(&t->keys, t->cap * 8) != cudaSuccess || cudaMalloc(&t->counts, t->cap * 8) != cudaSuccess ||
        cudaMalloc(&t->reps, t->cap * 8) != cudaSuccess || cudaMalloc(&t->stats, 8 * 8) != cudaSuccess ||
        cudaMalloc(&t->fb, (size_t)t->fb_cap * 8) != cudaSuccess) {
        cudaFree(t->keys);
        cudaFree(t->counts);
        cudaFree(t->reps);
        cudaFree(t->stats);
        cudaFree(t->fb);
        delete t;
        ctx->err = "cudaMalloc(table) failed";
        cudaGetLastError();
        return DAMPR_ERR_NOMEM;
    }
    *out = t;
    return dampr_table_clear(ctx, t);
}

int32_t dampr_table_destroy(dampr_ctx *ctx, dampr_table *t) {
    if (!t) return DAMPR_OK;
    if (ctx) {
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);
    }
    cudaFree(t->keys);
    cudaFree(t->counts);
    cudaFree(t->reps);
    cudaFree(t->stats);
    cudaFree(t->fb);
    cudaFree(t->tiles);
    cudaFree(t->ext);
    delete t;
    return DAMPR_OK;
}

int32_t dampr_table_clear(dampr_ctx *ctx, dampr_table *t) {
    ARG_CHECK(ctx, ctx && t, "null");
    t->ext_n = 0;
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        table_init_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(t->keys, t->counts, t->reps, t->cap,
                                                                    t->stats);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

int32_t dampr_text_count(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                         uint64_t own_hi, int32_t mode) {
    ARG_CHECK(ctx, ctx && t && tb, "null");
    ARG_CHECK(ctx, own_lo <= own_hi && own_hi <= tb->n, "ownership range outside the text");
    ARG_CHECK(ctx, (own_lo % 16) == 0, "own_lo must be a multiple of 16");
    if (g_text_kernel == 2) return launch_text_count_v2(ctx, t, tb, own_lo, own_hi, mode);
    mode &= ~DAMPR_TOK_FLAG_CR_DATA;  // the first-generation kernel flags every '\r' scan-wide; the host decides
    switch (mode) {
        case DAMPR_TOK_WS: return launch_text<DAMPR_TOK_WS, false>(ctx, t, tb, own_lo, own_hi);
        case DAMPR_TOK_NONWORD_LOWER_SET:
            return launch_text<DAMPR_TOK_NONWORD_LOWER_SET, false>(ctx, t, tb, own_lo, own_hi);
        case DAMPR_TOK_NONWORD_LOWER:
            return launch_text<DAMPR_TOK_NONWORD_LOWER, false>(ctx, t, tb, own_lo, own_hi);
    }
    ctx->err = "unknown tokeniser mode";
    return DAMPR_ERR_ARG;
}

int32_t dampr_text_verify(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                          uint64_t own_hi, int32_t mode) {
    ARG_CHECK(ctx, ctx && t && tb, "null");
    ARG_CHECK(ctx, own_lo <= own_hi && own_hi <= tb->n, "ownership range outside the text");
    ARG_CHECK(ctx, (own_lo % 16) == 0, "own_lo must be a multiple of 16");
    switch (mode) {
        case DAMPR_TOK_WS: return launch_text<DAMPR_TOK_WS, true>(ctx, t, tb, own_lo, own_hi);
        case DAMPR_TOK_NONWORD_LOWER_SET:
            return launch_text<DAMPR_TOK_NONWORD_LOWER_SET, true>(ctx, t, tb, own_lo, own_hi);
        case DAMPR_TOK_NONWORD_LOWER:
            return launch_text<DAMPR_TOK_NONWORD_LOWER, true>(ctx, t, tb, own_lo, own_hi);
    }
    ctx->err = "unknown tokeniser mode";
    return DAMPR_ERR_ARG;
}

int32_t dampr_table_stats(dampr_ctx *ctx, dampr_table *t, uint64_t stats[8]) {
    ARG_CHECK(ctx, ctx && t && stats, "null");
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scratch, t->stats, 64, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(stats, ctx->h_scratch, 64);
    return DAMPR_OK;
}

int32_t dampr_table_fallback_lines(dampr_ctx *ctx, dampr_table *t, uint64_t *lines, uint64_t cap, uint64_t *n) {
    ARG_CHECK(ctx, ctx && t && n, "null");
    uint64_t st[8];
    int rc = dampr_table_stats(ctx, t, st);
    if (rc) return rc;
    *n = st[7];
    if (!lines) return DAMPR_OK;
    ARG_CHECK(ctx, st[7] <= (uint64_t)t->fb_cap, "fallback list overflowed (DAMPR_TF_NONASCII is set)");
    ARG_CHECK(ctx, cap >= st[7], "lines array too small");
    if (st[7]) {
        CUDA_TRY(ctx, cudaMemcpyAsync(lines, t->fb, st[7] * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return DAMPR_OK;
}

int32_t dampr_table_fetch(dampr_ctx *ctx, dampr_table *t, uint64_t *codes, uint64_t *counts,
                          uint64_t *reps, uint64_t cap, uint64_t *n) {
    ARG_CHECK(ctx, ctx && t && n, "null");
    uint64_t st[8];
    int rc = dampr_table_stats(ctx, t, st);
    if (rc) return rc;
    *n = st[0];
    if (!codes && !counts && !reps) return DAMPR_OK;  // phase 1: count only
    ARG_CHECK(ctx, cap >= st[0], "fetch arrays too small");
    u64 m = st[0];
    if (m == 0) return DAMPR_OK;
    u64 *d = (u64 *)pool_alloc(ctx, (3 * m + 1) * 8);
    ARG_CHECK(ctx, d != nullptr, "device allocation failed");
    CUDA_TRY(ctx, cudaMemsetAsync(d + 3 * m, 0, 8, ctx->stream));
    {
        ScopedTimer tm(ctx, DAMPR_K_TABLE_EXTRACT);
        table_extract_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
            t->keys, t->counts, t->reps, t->cap, d, d + m, d + 2 * m, nullptr, m, d + 3 * m);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && codes) e = cudaMemcpyAsync(codes, d, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && counts) e = cudaMemcpyAsync(counts, d + m, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && reps) e = cudaMemcpyAsync(reps, d + 2 * m, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    pool_free(ctx, d);
    if (e != cudaSuccess) {
        ctx->err = std::string("table fetch failed: ") + cudaGetErrorString(e);
        return DAMPR_ERR_CUDA;
    }
    return DAMPR_OK;
}

int32_t dampr_table_to_kv(dampr_ctx *ctx, dampr_table *t, dampr_kv **out) {
    ARG_CHECK(ctx, ctx && t && out, "null");
    uint64_t st[8];
    int rc = dampr_table_stats(ctx, t, st);
    if (rc) return rc;
    u64 m = st[0];
    rc = dampr_kv_create(ctx, m, out);
    if (rc) return rc;
    if (m) {
        CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_scratch, 0, 8, ctx->stream));
        {
            ScopedTimer tm(ctx, DAMPR_K_TABLE_EXTRACT);
            table_extract_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
                t->keys, t->counts, t->reps, t->cap, nullptr, nullptr, nullptr, (*out)->rec, m,
                ctx->d_scratch);
        }
        CUDA_TRY(ctx, cudaGetLastError());
    }
    (*out)->n = m;
    return DAMPR_OK;
}

}  // extern "C"

// ---- K9: key materialisation -------------------------------------------------------------------
// Decodes every table entry into a fixed-width, NUL-padded ASCII string on the device so the host
// never loops over keys in Python (strings travel inside pickles in the reference, dataset.py:129-137).
namespace {

__global__ void table_words_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ counts,
                                   const u64 *__restrict__ reps, u64 cap, const u8 *__restrict__ text, int mode,
                                   u32 width, u8 *__restrict__ out_words, u64 *__restrict__ out_counts,
                                   u64 *__restrict__ out_codes, u64 *__restrict__ out_reps, u64 out_cap,
                                   u64 *cursor) {
    u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < cap; i += stride) {
        u64 k = keys[i];
        bool have = k != 0;
        u32 m = __ballot_sync(0xFFFFFFFFu, have);
        u64 base = 0;
        if (m) {
            int leader = __ffs(m) - 1;
            if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(cursor, (u64)__popc(m));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
        }
        if (!have) continue;
        u64 idx = base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
        if (idx >= out_cap) continue;
        u8 *w = out_words + idx * width;
        u64 rep = reps[i];
        u32 n = 0;
        if (k >> 63) {
            // hashed (long) token: bytes of its representative occurrence
            u64 off = rep >> 20;
            u32 len = (u32)(rep & 0xFFFFFu);
            if (text && rep != ~0ULL) {
                for (; n < len && n < width; ++n) {
                    u32 c = text[off + n];
                    if (mode != DAMPR_TOK_WS && c >= 'A' && c <= 'Z') c |= 0x20;
                    w[n] = (u8)c;
                }
            }
        } else if (mode == DAMPR_TOK_WS) {
            u64 c = k;
            for (; c && n < width; ++n) {
                w[n] = (u8)(c & 127);
                c >>= 7;
            }
        } else {
            u64 c = k;
            const char *sym = "\0" "0123456789_abcdefghijklmnopqrstuvwxyz";
            for (; c && n < width; ++n) {
                w[n] = (u8)sym[c % 38];
                c /= 38;
            }
        }
        for (; n < width; ++n) w[n] = 0;
        out_counts[idx] = counts[i];
        out_codes[idx] = k;
        out_reps[idx] = (rep == ~0ULL) ? 0ULL : rep;
    }
}

}  // namespace

// the m entries of the table, decoded, into host arrays (page-locked ones are copied into directly)
static int fetch_words_into(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t mode, uint32_t width, u64 m,
                            uint8_t *words, uint64_t *counts, uint64_t *codes, uint64_t *reps) {
    t->ext_n = 0;
    if (m == 0) return DAMPR_OK;
    // the count column stays on the device (t->ext) for dampr_count_dictionary
    if (t->ext_cap < m) {
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        cudaFree(t->ext);
        t->ext = nullptr;
        t->ext_cap = 0;
        CUDA_TRY(ctx, cudaMalloc(&t->ext, m * 8));
        t->ext_cap = m;
    }
    u64 per = width + 16;
    u8 *d = (u8 *)pool_alloc(ctx, m * per + 8);
    ARG_CHECK(ctx, d != nullptr, "device allocation failed");
    u8 *d_words = d;
    u64 *d_counts = t->ext;
    u64 *d_codes = (u64 *)(d + m * width);
    u64 *d_reps = d_codes + m;
    u64 *d_cur = d_reps + m;
    CUDA_TRY(ctx, cudaMemsetAsync(d_cur, 0, 8, ctx->stream));
    {
        ScopedTimer tm(ctx, DAMPR_K_TABLE_EXTRACT);
        table_words_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(t->keys, t->counts, t->reps, t->cap,
                                                                     tb ? tb->text : nullptr, mode, width, d_words,
                                                                     d_counts, d_codes, d_reps, m, d_cur);
    }
    cudaError_t e = cudaGetLastError();
    // the small columns first (asynchronous, pageable), then the words through the pinned staging ring,
    // whose final synchronisation covers everything queued on the stream
    if (e == cudaSuccess) e = cudaMemcpyAsync(counts, d_counts, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && codes) e = cudaMemcpyAsync(codes, d_codes, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && reps) e = cudaMemcpyAsync(reps, d_reps, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    int rc2 = DAMPR_OK;
    if (e == cudaSuccess) rc2 = staged_d2h(ctx, words, d_words, m * width, ctx->stream);
    if (e == cudaSuccess && rc2 == DAMPR_OK) e = cudaStreamSynchronize(ctx->stream);
    pool_free(ctx, d);
    if (e != cudaSuccess) {
        ctx->err = std::string("table fetch_words failed: ") + cudaGetErrorString(e);
        return DAMPR_ERR_CUDA;
    }
    if (rc2 == DAMPR_OK) t->ext_n = m;
    return rc2;
}

extern "C" int32_t dampr_table_fetch_words(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t mode,
                                           uint32_t width, uint8_t *words, uint64_t *counts, uint64_t *codes,
                                           uint64_t *reps, uint64_t cap, uint64_t *n) {
    ARG_CHECK(ctx, ctx && t && n, "null");
    ARG_CHECK(ctx, width >= 16 && width <= 256 && (width % 8) == 0, "width must be a multiple of 8 in [16, 256]");
    uint64_t st[8];
    int rc = dampr_table_stats(ctx, t, st);
    if (rc) return rc;
    *n = st[0];
    if (!words) return DAMPR_OK;
    ARG_CHECK(ctx, cap >= st[0] && counts, "fetch arrays too small");   // codes / reps are optional
    return fetch_words_into(ctx, t, tb, mode, width, st[0], words, counts, codes, reps);
}

extern "C" int32_t dampr_table_fetch_words_leased(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t mode,
                                                  uint32_t width, int32_t with_codes, void **host_ptr,
                                                  uint64_t *lease, uint64_t *n) {
    ARG_CHECK(ctx, ctx && t && n && host_ptr && lease, "null");
    ARG_CHECK(ctx, width >= 16 && width <= 256 && (width % 8) == 0, "width must be a multiple of 8 in [16, 256]");
    *host_ptr = nullptr;
    *lease = 0;
    uint64_t st[8];
    int rc = dampr_table_stats(ctx, t, st);
    if (rc) return rc;
    const u64 m = *n = st[0];
    if (m == 0) return DAMPR_OK;
    u64 id = 0;
    result_lease(ctx, m * (width + (with_codes ? 24 : 8)), host_ptr, &id);
    if (!id) return DAMPR_OK;
    u8 *words = (u8 *)*host_ptr;
    uint64_t *counts = (uint64_t *)(words + m * width);
    rc = fetch_words_into(ctx, t, tb, mode, width, m, words, counts, with_codes ? counts + m : nullptr,
                          with_codes ? counts + 2 * m : nullptr);
    if (rc) {
        result_release(ctx, id);
        *host_ptr = nullptr;
        return rc;
    }
    *lease = id;
    return DAMPR_OK;
}

extern "C" int32_t dampr_table_extracted_counts(dampr_ctx *ctx, dampr_table *t, uint64_t *dev_ptr, uint64_t *n) {
    ARG_CHECK(ctx, ctx && t && dev_ptr && n, "null");
    *dev_ptr = (uint64_t)(uintptr_t)t->ext;
    *n = t->ext_n;
    return DAMPR_OK;
}

// ---- dictionary of a count column on the device ----------------------------------------------------------
// Sorted distinct values, the inverse (uint32, row order) and the smallest row holding each value. Values below a
// bound B go through a presence table: mark, count per 1024-entry block, scan the block counts, rank every present
// value. The few values at or above B (the head of a Zipf count distribution) are sorted and folded by
// dampr_kv_sort_reduce and found again by binary search. Row i < n reads counts[i * stride]; rows n.. are `extra`.
namespace {

constexpr u32 DICT_BLOCK = 1024;

__device__ __forceinline__ u64 dict_value(const u64 *counts, u64 n, u32 stride, const u64 *extra, u64 i) {
    return i < n ? counts[i * stride] : extra[i - n];
}

__global__ void dict_mark_kernel(const u64 *__restrict__ counts, u64 n, u32 stride, const u64 *__restrict__ extra,
                                 u64 rows, u64 bound, u32 *__restrict__ flag, u32 *__restrict__ first,
                                 ulonglong2 *__restrict__ big, u64 *__restrict__ ctr) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < rows; i += (u64)gridDim.x * blockDim.x) {
        const u64 v = dict_value(counts, n, stride, extra, i);
        if (v < bound) {
            if (!flag[v]) flag[v] = 1;
            if (first[v] > (u32)i) atomicMin(&first[v], (u32)i);
        } else {
            if ((long long)v < 0) ctr[1] = 1;   // negative: the two ranges would interleave
            const u64 s = atomicAdd((unsigned long long *)&ctr[0], 1ULL);
            big[s] = make_ulonglong2(v, i);
        }
    }
}

__global__ void dict_block_count_kernel(const u32 *__restrict__ flag, u32 *__restrict__ bsum) {
    const u32 present = __syncthreads_count(flag[blockIdx.x * (u64)DICT_BLOCK + threadIdx.x] != 0);
    if (threadIdx.x == 0) bsum[blockIdx.x] = present;
}

// exclusive scan of nb <= 4 * DICT_BLOCK block counts in one block; bsum[nb] = total
__global__ void dict_scan_kernel(u32 *__restrict__ bsum, u32 nb) {
    __shared__ u32 s[DICT_BLOCK];
    const u32 per = (nb + DICT_BLOCK - 1) / DICT_BLOCK;
    const u32 lo = threadIdx.x * per, hi = min(nb, lo + per);
    u32 acc = 0;
    for (u32 j = lo; j < hi; ++j) acc += bsum[j];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (u32 d = 1; d < DICT_BLOCK; d <<= 1) {
        const u32 x = threadIdx.x >= d ? s[threadIdx.x - d] : 0;
        __syncthreads();
        s[threadIdx.x] += x;
        __syncthreads();
    }
    u32 run = s[threadIdx.x] - acc;
    for (u32 j = lo; j < hi; ++j) {
        const u32 c = bsum[j];
        bsum[j] = run;
        run += c;
    }
    if (threadIdx.x == DICT_BLOCK - 1) bsum[nb] = s[DICT_BLOCK - 1];
}

// flag[v] becomes the rank of v among the present values; uniq / rows receive v and its first row
__global__ void dict_rank_kernel(u32 *__restrict__ flag, const u32 *__restrict__ first, const u32 *__restrict__ boff,
                                 long long *__restrict__ uniq, u32 *__restrict__ rows) {
    __shared__ u32 warp_tot[DICT_BLOCK / 32];
    const u64 v = blockIdx.x * (u64)DICT_BLOCK + threadIdx.x;
    const bool have = flag[v] != 0;
    const u32 m = __ballot_sync(0xFFFFFFFFu, have);
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_tot[w] = __popc(m);
    __syncthreads();
    if (w == 0) {
        const u32 x = warp_tot[lane];
        u32 incl = x;
        for (u32 d = 1; d < 32; d <<= 1) {
            const u32 y = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl += y;
        }
        warp_tot[lane] = incl - x;
    }
    __syncthreads();
    if (have) {
        const u32 r = boff[blockIdx.x] + warp_tot[w] + __popc(m & ((1u << lane) - 1u));
        flag[v] = r;
        uniq[r] = (long long)v;
        rows[r] = first[v];
    }
}

__global__ void dict_inv_kernel(const u64 *__restrict__ counts, u64 n, u32 stride, const u64 *__restrict__ extra,
                                u64 rows, u64 bound, const u32 *__restrict__ rank, u32 *__restrict__ inv) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < rows; i += (u64)gridDim.x * blockDim.x) {
        const u64 v = dict_value(counts, n, stride, extra, i);
        if (v < bound) inv[i] = rank[v];
    }
}

// the folded large values (key order) appended after the m_small ranked ones; the large rows' inverse by search
__global__ void dict_big_kernel(const ulonglong2 *__restrict__ big, u64 nbig, const ulonglong2 *__restrict__ red,
                                u64 nred, u32 m_small, long long *__restrict__ uniq, u32 *__restrict__ rows,
                                u32 *__restrict__ inv) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < nbig; i += (u64)gridDim.x * blockDim.x) {
        if (i < nred) {
            uniq[m_small + i] = (long long)red[i].x;
            rows[m_small + i] = (u32)red[i].y;
        }
        const u64 v = big[i].x;
        u64 lo = 0, hi = nred;
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (red[mid].x <= v) lo = mid;
            else hi = mid;
        }
        inv[big[i].y] = m_small + (u32)lo;
    }
}

}  // namespace

// host_ptr != nullptr: the outputs go into one lease of the context's result arena, taken once the number of distinct
// values is known (uniq, inv and rows are then ignored); *lease stays 0 when the arena gives none
static int count_dictionary(dampr_ctx *ctx, const uint64_t *counts, uint64_t n, uint32_t stride, const int64_t *extra,
                            uint32_t n_extra, int64_t *uniq, uint32_t *inv, uint32_t *rows, uint64_t *n_uniq,
                            void **host_ptr, uint64_t *lease) {
    ARG_CHECK(ctx, (counts || n == 0) && (extra || n_extra == 0), "null column");
    const u64 N = n + n_extra;
    ARG_CHECK(ctx, N < (1ULL << 32), "more than 2^32 rows");
    const u64 *col = (const u64 *)counts;
    *n_uniq = 0;
    if (N == 0) return DAMPR_OK;
    CtxScope scope_(ctx);
    CUDA_TRY(ctx, cudaSetDevice(ctx->device));
    wait_uploads(ctx);
    // the presence table is cleared and scanned once: proportional to the column, at most 2^22 entries
    u64 B = 4096;
    while (B < 2 * N && B < (1ULL << 22)) B <<= 1;
    const u32 nb = (u32)(B / DICT_BLOCK);
    // flag[B] first[B] bsum[nb + 1] | ctr[2] extra[n_extra] | uniq[N] | rows[N] inv[N] | big[N]
    const u64 o_ctr = ((2 * B + nb + 1) * 4 + 15) & ~15ULL;
    const u64 o_uniq = (o_ctr + 16 + n_extra * 8 + 15) & ~15ULL;
    const u64 o_rows = o_uniq + N * 8;
    const u64 o_inv = o_rows + N * 4;
    const u64 o_big = (o_inv + N * 4 + 15) & ~15ULL;
    DevBuf buf;
    CUDA_TRY(ctx, buf.alloc(o_big + N * 16));
    u8 *base = (u8 *)buf.p;
    u32 *flag = (u32 *)base, *first = flag + B, *bsum = first + B;
    u64 *ctr = (u64 *)(base + o_ctr);
    u64 *d_extra = ctr + 2;
    long long *d_uniq = (long long *)(base + o_uniq);
    u32 *d_rows = (u32 *)(base + o_rows), *d_inv = (u32 *)(base + o_inv);
    ulonglong2 *big = (ulonglong2 *)(base + o_big);
    CUDA_TRY(ctx, cudaMemsetAsync(flag, 0, B * 4, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(first, 0xFF, B * 4, ctx->stream));
    CUDA_TRY(ctx, cudaMemsetAsync(ctr, 0, 16, ctx->stream));
    if (n_extra) CUDA_TRY(ctx, cudaMemcpyAsync(d_extra, extra, n_extra * 8, cudaMemcpyHostToDevice, ctx->stream));
    const int grid = ctx->num_sms * 4;
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        dict_mark_kernel<<<grid, 256, 0, ctx->stream>>>(col, n, stride, d_extra, N, B, flag, first, big, ctr);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        dict_block_count_kernel<<<nb, DICT_BLOCK, 0, ctx->stream>>>(flag, bsum);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        dict_scan_kernel<<<1, DICT_BLOCK, 0, ctx->stream>>>(bsum, nb);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        dict_rank_kernel<<<nb, DICT_BLOCK, 0, ctx->stream>>>(flag, first, bsum, d_uniq, d_rows);
    }
    {
        ScopedTimer tm(ctx, DAMPR_K_MISC);
        dict_inv_kernel<<<grid, 256, 0, ctx->stream>>>(col, n, stride, d_extra, N, B, flag, d_inv);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    // how many values are large, whether one is negative, how many are small
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scratch, ctr, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->h_scratch + 2, bsum + nb, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    const u64 nbig = ctx->h_scratch[0];
    const bool negative = ctx->h_scratch[1] != 0;
    const u32 m_small = (u32)(ctx->h_scratch[2] & 0xFFFFFFFFu);
    if (negative) return set_err(ctx, DAMPR_ERR_UNSUPPORTED, "%s", "negative values in a count column");
    u64 m = m_small;
    if (nbig) {
        dampr_kv *kv = nullptr, *red = nullptr;
        int rc = dampr_kv_create(ctx, nbig, &kv);
        if (rc) return rc;
        cudaError_t e = cudaMemcpyAsync(kv->rec, big, nbig * 16, cudaMemcpyDeviceToDevice, ctx->stream);
        kv->n = nbig;
        rc = e == cudaSuccess ? dampr_kv_sort_reduce(ctx, kv, DAMPR_KEY_I64, DAMPR_OP_MIN_I64, &red)
                              : set_err(ctx, DAMPR_ERR_CUDA, "%s", cudaGetErrorString(e));
        if (rc == DAMPR_OK) {
            {
                ScopedTimer tm(ctx, DAMPR_K_MISC);
                dict_big_kernel<<<(unsigned)((nbig + 255) / 256), 256, 0, ctx->stream>>>(big, nbig, red->rec, red->n, m_small,
                                                                                       d_uniq, d_rows, d_inv);
            }
            m += red->n;
            e = cudaGetLastError();
            if (e != cudaSuccess) rc = set_err(ctx, DAMPR_ERR_CUDA, "%s", cudaGetErrorString(e));
        }
        dampr_kv_destroy(ctx, kv);
        if (red) dampr_kv_destroy(ctx, red);
        if (rc) return rc;
    }
    *n_uniq = m;
    u64 id = 0;
    if (host_ptr) {
        // uniq[m] | inv[N] | rows[m]
        result_lease(ctx, m * 8 + N * 4 + m * 4, host_ptr, &id);
        if (!id) return DAMPR_OK;
        uniq = (int64_t *)*host_ptr;
        inv = (uint32_t *)(uniq + m);
        rows = inv + N;
    }
    cudaError_t e = cudaMemcpyAsync(inv, d_inv, N * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(uniq, d_uniq, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(rows, d_rows, m * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        if (id) result_release(ctx, id);
        return set_err(ctx, DAMPR_ERR_CUDA, "count dictionary download failed: %s", cudaGetErrorString(e));
    }
    if (host_ptr) *lease = id;
    return DAMPR_OK;
}

extern "C" int32_t dampr_count_dictionary(dampr_ctx *ctx, const uint64_t *counts, uint64_t n, uint32_t stride,
                                          const int64_t *extra, uint32_t n_extra, int64_t *uniq, uint32_t *inv,
                                          uint32_t *rows, uint64_t *n_uniq) {
    ARG_CHECK(ctx, ctx && uniq && inv && rows && n_uniq && stride >= 1, "null");
    return count_dictionary(ctx, counts, n, stride, extra, n_extra, uniq, inv, rows, n_uniq, nullptr, nullptr);
}

extern "C" int32_t dampr_count_dictionary_leased(dampr_ctx *ctx, const uint64_t *counts, uint64_t n, uint32_t stride,
                                                 const int64_t *extra, uint32_t n_extra, void **host_ptr,
                                                 uint64_t *lease, uint64_t *n_uniq) {
    ARG_CHECK(ctx, ctx && host_ptr && lease && n_uniq && stride >= 1, "null");
    *host_ptr = nullptr;
    *lease = 0;
    return count_dictionary(ctx, counts, n, stride, extra, n_extra, nullptr, nullptr, nullptr, n_uniq, host_ptr, lease);
}

// ---- host-side sink formatting (SinkWriter, dataset.py:264-282: one print(value) per record) --------
// Joins k columns with '\t' and terminates rows with '\n'. Column kinds:
//   0  fixed-width NUL-padded bytes  ptr = u8[n][width]
//   1  dictionary                    ptr = u32 inv[n], aux = blob bytes, aux2 = u32 offsets[m+1]
//   2  dictionary of int64 values    ptr = u32 inv[n], aux = int64 values[m], widths = m (decimal text)
// out == NULL: only *out_len is computed.
namespace {
// Process-wide pool of host workers for the sink, the row joiner and dampr_host_unique_small: created on first use,
// parked on a condition variable between calls and joined when the library is unloaded or the process exits. A call
// holds lock() for as long as it uses the pool or its buffers; run(T, fn) calls fn(0) .. fn(T - 1), the caller taking
// its share, and returns when all have finished. A job is its own heap object, so a worker that wakes late sees a
// finished job and nothing of the caller's frame.
class HostPool {
    struct Job {
        const std::function<void(int)> *fn;
        int T;
        std::atomic<int> next{0}, left{0};
    };

  public:
    static constexpr int MAX_TASKS = 16;
    static HostPool &get() {
        static HostPool p;
        return p;
    }
    static int width() { return (int)std::max(1u, std::min(std::thread::hardware_concurrency(), (unsigned)MAX_TASKS)); }
    std::unique_lock<std::mutex> lock() { return std::unique_lock<std::mutex>(job_mu_); }
    void run(int T, const std::function<void(int)> &fn) {
        if (T <= 1) {
            if (T == 1) fn(0);
            return;
        }
        auto job = std::make_shared<Job>();
        job->fn = &fn;
        job->T = T;
        job->left.store(T);
        {
            std::lock_guard<std::mutex> lk(mu_);
            if (pid_ != getpid()) {
                // a forked child has none of its parent's threads: their handles are abandoned, not joined
                workers_ = new std::vector<std::thread>();
                pid_ = getpid();
            }
            while ((int)workers_->size() < std::min(T, width()) - 1) {
                workers_->emplace_back([this] { loop(); });
                ++started_;
            }
            cur_ = job;
            ++gen_;
        }
        cv_.notify_all();
        work(*job);
        std::unique_lock<std::mutex> lk(mu_);
        done_cv_.wait(lk, [&] { return job->left.load() == 0; });
    }
    // task t's output buffer of at least `bytes`, kept between calls so that its pages stay mapped; nullptr when
    // `bytes` is more than a task's share of the "host_result_cache_bytes" option (the caller then uses malloc)
    u8 *buffer(int t, size_t bytes) {
        if (t >= MAX_TASKS || bytes > (size_t)g_result_cache_bytes / MAX_TASKS) return nullptr;
        if (cap_[t] < bytes) {
            free(buf_[t]);
            buf_[t] = (u8 *)malloc(bytes);
            cap_[t] = buf_[t] ? bytes : 0;
        }
        return buf_[t];
    }
    u64 threads_started() {
        std::lock_guard<std::mutex> lk(mu_);
        return started_;
    }

  private:
    HostPool() : workers_(new std::vector<std::thread>()), pid_(getpid()) {}
    ~HostPool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        if (pid_ == getpid()) {
            for (auto &t : *workers_) t.join();
            delete workers_;
        }
        for (u8 *b : buf_) free(b);
    }
    void work(Job &j) {
        for (;;) {
            const int t = j.next.fetch_add(1);
            if (t >= j.T) break;
            (*j.fn)(t);
            if (j.left.fetch_sub(1) == 1) {
                std::lock_guard<std::mutex> lk(mu_);
                done_cv_.notify_all();
            }
        }
    }
    void loop() {
        u64 seen = 0;
        for (;;) {
            std::shared_ptr<Job> job;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return stop_ || gen_ != seen; });
                if (stop_) return;
                seen = gen_;
                job = cur_;
            }
            work(*job);
        }
    }
    std::mutex job_mu_, mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> *workers_;
    pid_t pid_;
    std::shared_ptr<Job> cur_;
    u64 gen_ = 0, started_ = 0;
    bool stop_ = false;
    u8 *buf_[MAX_TASKS] = {};
    size_t cap_[MAX_TASKS] = {};
};

struct JoinArgs {
    u64 n;
    int ncols;
    const int32_t *kinds;
    const void *const *ptrs;
    const uint32_t *widths;
    const void *const *aux;
    const void *const *aux2;
};

// kind 2 (dictionary of int64 values: ptr = u32 inv[n], aux = int64 values[m], widths = m) is turned into
// kind 1 once per call: the m distinct values are formatted in decimal here instead of in Python
struct IntDicts {
    std::vector<std::vector<u8>> blobs;
    std::vector<std::vector<u32>> offs;
    std::vector<int32_t> kinds;
    std::vector<const void *> aux, aux2;
    std::vector<u32> longest;   // per column: the longest string of a dictionary built here (0 otherwise)
};
// repr(float) of CPython (float_repr_style 'short': PyOS_double_to_string(x, 'r', 0, Py_DTSF_ADD_DOT_0), i.e. the
// shortest digit string that round-trips, laid out in fixed notation when -4 < decpt <= 16 and with an exponent of
// at least two digits otherwise) — what print(value) / sink_tsv write for a float (dampr.py:521-529). The digits
// come from std::to_chars (shortest round-trip, like David Gay's dtoa mode 0 that CPython uses). Returns the length
// (<= 24).
static int format_py_float(double v, char *out) {
    if (v != v) {
        memcpy(out, "nan", 3);
        return 3;
    }
    int n = 0;
    if (std::signbit(v)) {
        out[n++] = '-';
        v = -v;
    }
    if (v == std::numeric_limits<double>::infinity()) {
        memcpy(out + n, "inf", 3);
        return n + 3;
    }
    if (v == 0.0) {
        memcpy(out + n, "0.0", 3);
        return n + 3;
    }
    char tmp[40];
    const auto r = std::to_chars(tmp, tmp + sizeof tmp, v, std::chars_format::scientific);
    // tmp = d[.ddd]e(+|-)XX[X]
    char digits[24];
    int k = 0;
    const char *p = tmp;
    while (p < r.ptr && *p != 'e') {
        if (*p != '.') digits[k++] = *p;
        ++p;
    }
    ++p;  // 'e'
    const bool eneg = (*p == '-');
    ++p;
    int e10 = 0;
    while (p < r.ptr) e10 = e10 * 10 + (*p++ - '0');
    if (eneg) e10 = -e10;
    const int decpt = e10 + 1;
    if (decpt > -4 && decpt <= 16) {
        if (decpt <= 0) {
            out[n++] = '0';
            out[n++] = '.';
            for (int i = 0; i < -decpt; ++i) out[n++] = '0';
            memcpy(out + n, digits, k);
            n += k;
        } else if (decpt < k) {
            memcpy(out + n, digits, decpt);
            n += decpt;
            out[n++] = '.';
            memcpy(out + n, digits + decpt, k - decpt);
            n += k - decpt;
        } else {
            memcpy(out + n, digits, k);
            n += k;
            for (int i = 0; i < decpt - k; ++i) out[n++] = '0';
            out[n++] = '.';
            out[n++] = '0';
        }
    } else {
        out[n++] = digits[0];
        if (k > 1) {
            out[n++] = '.';
            memcpy(out + n, digits + 1, k - 1);
            n += k - 1;
        }
        out[n++] = 'e';
        int ex = decpt - 1;
        out[n++] = ex < 0 ? '-' : '+';
        if (ex < 0) ex = -ex;
        if (ex >= 100) {
            out[n++] = (char)('0' + ex / 100);
            ex %= 100;
            out[n++] = (char)('0' + ex / 10);
            out[n++] = (char)('0' + ex % 10);
        } else {
            out[n++] = (char)('0' + ex / 10);
            out[n++] = (char)('0' + ex % 10);
        }
    }
    return n;
}

// (the caller holds the pool's lock)
static void lower_int_dicts(HostPool &pool, int ncols, const int32_t *kinds, const uint32_t *widths,
                            const void *const *aux, const void *const *aux2, IntDicts &d) {
    d.longest.assign(ncols, 0);
    d.kinds.assign(kinds, kinds + ncols);
    d.aux.assign(aux, aux + ncols);
    d.aux2.assign(aux2, aux2 + ncols);
    d.blobs.resize(ncols);
    d.offs.resize(ncols);
    for (int c = 0; c < ncols; ++c) {
        if (kinds[c] == 3) {
            // dictionary of float64 values: ptr = u32 inv[n], aux = double values[m], widths = m -> kind 1 with
            // Python's repr of every distinct value, formatted here (on the pool for large dictionaries)
            const double *vals = (const double *)aux[c];
            const u32 m = widths[c];
            auto &blob = d.blobs[c];
            auto &off = d.offs[c];
            std::vector<char> slots((size_t)m * 24 + 24);
            std::vector<u8> lens((size_t)m + 1);
            const int T = (int)std::max<u32>(1, std::min<u32>(HostPool::width(), m / 1024));
            pool.run(T, [&](int t) {
                const u32 lo = (u32)((u64)m * t / T), hi = (u32)((u64)m * (t + 1) / T);
                for (u32 j = lo; j < hi; ++j) lens[j] = (u8)format_py_float(vals[j], slots.data() + (size_t)j * 24);
            });
            off.resize((size_t)m + 1);
            off[0] = 0;
            for (u32 j = 0; j < m; ++j) {
                off[j + 1] = off[j] + lens[j];
                d.longest[c] = std::max<u32>(d.longest[c], lens[j]);
            }
            blob.resize((size_t)off[m] + 1);
            for (u32 j = 0; j < m; ++j) memcpy(blob.data() + off[j], slots.data() + (size_t)j * 24, lens[j]);
            d.kinds[c] = 1;
            d.aux[c] = blob.data();
            d.aux2[c] = off.data();
            continue;
        }
        if (kinds[c] != 2) continue;
        const int64_t *vals = (const int64_t *)aux[c];
        const u32 m = widths[c];
        auto &blob = d.blobs[c];
        auto &off = d.offs[c];
        blob.reserve((size_t)m * 8);
        off.resize((size_t)m + 1);
        off[0] = 0;
        for (u32 j = 0; j < m; ++j) {
            char tmp[24];
            int64_t v = vals[j];
            u64 u = v < 0 ? (u64)0 - (u64)v : (u64)v;
            int k = 24;
            do {
                tmp[--k] = (char)('0' + u % 10);
                u /= 10;
            } while (u);
            if (v < 0) tmp[--k] = '-';
            blob.insert(blob.end(), tmp + k, tmp + 24);
            off[j + 1] = (u32)blob.size();
            d.longest[c] = std::max<u32>(d.longest[c], (u32)(24 - k));
        }
        if (blob.empty()) blob.push_back(0);
        d.kinds[c] = 1;
        d.aux[c] = blob.data();
        d.aux2[c] = off.data();
    }
}

// rows [lo, hi): returns the byte count; writes when out != nullptr
static u64 join_rows(const JoinArgs &a, u64 lo, u64 hi, u8 *out) {
    u64 pos = 0;
    for (u64 i = lo; i < hi; ++i) {
        for (int c = 0; c < a.ncols; ++c) {
            const u8 *src;
            u32 len;
            if (a.kinds[c] == 0) {
                const u8 *w = (const u8 *)a.ptrs[c] + i * a.widths[c];
                len = 0;
                while (len < a.widths[c] && w[len]) ++len;
                src = w;
            } else {
                u32 j = ((const u32 *)a.ptrs[c])[i];
                const u32 *off = (const u32 *)a.aux2[c];
                src = (const u8 *)a.aux[c] + off[j];
                len = off[j + 1] - off[j];
            }
            if (out) {
                memcpy(out + pos, src, len);
                out[pos + len] = (c + 1 == a.ncols) ? '\n' : '\t';
            }
            pos += len + 1;
        }
    }
    return pos;
}
// the same for a destination with >= 32 bytes of slack after the last row: fixed-width cells are copied
// whole (two or four 8-byte moves) and their length comes from a word-at-a-time NUL search
static u64 join_rows_fast(const JoinArgs &a, u64 lo, u64 hi, u8 *out) {
    u8 *p = out;
    for (u64 i = lo; i < hi; ++i) {
        for (int c = 0; c < a.ncols; ++c) {
            if (a.kinds[c] == 0) {
                const u32 width = a.widths[c];
                const u8 *w = (const u8 *)a.ptrs[c] + i * width;
                u32 len = 0;
                if ((width & 7u) == 0) {
                    while (len < width) {
                        u64 x;
                        memcpy(&x, w + len, 8);
                        memcpy(p + len, &x, 8);
                        const u64 z = (x - 0x0101010101010101ULL) & ~x & 0x8080808080808080ULL;
                        if (z) {
                            len += (u32)(__builtin_ctzll(z) >> 3);
                            break;
                        }
                        len += 8;
                    }
                } else {
                    while (len < width && w[len]) ++len;
                    memcpy(p, w, len);
                }
                p += len;
            } else {
                const u32 j = ((const u32 *)a.ptrs[c])[i];
                const u32 *off = (const u32 *)a.aux2[c];
                const u32 len = off[j + 1] - off[j];
                memcpy(p, (const u8 *)a.aux[c] + off[j], len);
                p += len;
            }
            *p++ = (c + 1 == a.ncols) ? '\n' : '\t';
        }
    }
    return (u64)(p - out);
}
// rows with a byte string in front of every column and a row ending instead of the TSV tabs / newline (JSON lines:
// pre = {"[\"", "\", ", ", "}, row_end = "]\n"): same cells, same dictionaries
struct RowFmt {
    std::vector<std::string> pre;
    std::string row_end;
};
static u64 join_rows_fmt(const JoinArgs &a, const RowFmt &f, u64 lo, u64 hi, u8 *out) {
    u8 *p = out;
    for (u64 i = lo; i < hi; ++i) {
        for (int c = 0; c < a.ncols; ++c) {
            const std::string &pre = f.pre[(size_t)c];
            memcpy(p, pre.data(), pre.size());
            p += pre.size();
            if (a.kinds[c] == 0) {
                const u32 width = a.widths[c];
                const u8 *w = (const u8 *)a.ptrs[c] + i * width;
                u32 len = 0;
                while (len < width && w[len]) ++len;
                memcpy(p, w, len);
                p += len;
            } else {
                const u32 j = ((const u32 *)a.ptrs[c])[i];
                const u32 *off = (const u32 *)a.aux2[c];
                const u32 len = off[j + 1] - off[j];
                memcpy(p, (const u8 *)a.aux[c] + off[j], len);
                p += len;
            }
        }
        memcpy(p, f.row_end.data(), f.row_end.size());
        p += f.row_end.size();
    }
    return (u64)(p - out);
}
}  // namespace

// repr(float) of n values into 24-byte slots (lens[i] bytes used each): the formatter of the float dictionaries
extern "C" int32_t dampr_host_format_f64(const double *vals, uint64_t n, uint8_t *slots, uint8_t *lens) {
    if ((!vals || !slots || !lens) && n) return DAMPR_ERR_ARG;
    for (uint64_t i = 0; i < n; ++i) lens[i] = (uint8_t)format_py_float(vals[i], (char *)slots + i * 24);
    return DAMPR_OK;
}

extern "C" int32_t dampr_host_join_tsv(uint64_t n, int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                                       const uint32_t *widths, const void *const *aux, const void *const *aux2,
                                       uint8_t *out, uint64_t cap, uint64_t *out_len) {
    if (!kinds || !ptrs || !out_len || ncols < 1 || ncols > 16) return DAMPR_ERR_ARG;
    HostPool &pool = HostPool::get();
    auto pool_lock = pool.lock();
    IntDicts idc;
    lower_int_dicts(pool, ncols, kinds, widths, aux, aux2, idc);
    JoinArgs a{n, ncols, idc.kinds.data(), ptrs, widths, idc.aux.data(), idc.aux2.data()};
    const int T = (int)std::min<u64>(HostPool::width(), std::max<u64>(1, n / 16384));
    std::vector<u64> lens(T, 0), offs(T + 1, 0);
    pool.run(T, [&](int t) { lens[t] = join_rows(a, n * t / T, n * (t + 1) / T, nullptr); });
    for (int t = 0; t < T; ++t) offs[t + 1] = offs[t] + lens[t];
    *out_len = offs[T];
    if (!out) return DAMPR_OK;
    if (offs[T] > cap) return DAMPR_ERR_ARG;
    pool.run(T, [&](int t) { join_rows(a, n * t / T, n * (t + 1) / T, out + offs[t]); });
    return DAMPR_OK;
}

// Host-clock split of the last sink_rows call, in milliseconds: the calling thread's dictionary preparation, then the
// largest value any worker saw for the delay before it started, open(), row formatting, write() and close().
namespace {
struct SinkTimes {
    double prep = 0, start = 0, open = 0, format = 0, write = 0, close = 0;
};
std::mutex g_sink_times_mu;
SinkTimes g_sink_times;
using SinkClock = std::chrono::steady_clock;
inline double ms_since(SinkClock::time_point t0) {
    return std::chrono::duration<double, std::milli>(SinkClock::now() - t0).count();
}
}  // namespace

extern "C" int32_t dampr_host_sink_timings(double *out_ms) {
    if (!out_ms) return DAMPR_ERR_ARG;
    std::lock_guard<std::mutex> lk(g_sink_times_mu);
    const SinkTimes &s = g_sink_times;
    const double v[6] = {s.prep, s.start, s.open, s.format, s.write, s.close};
    memcpy(out_ms, v, sizeof v);
    return DAMPR_OK;
}

extern "C" int32_t dampr_host_pool_threads(uint64_t *started) {
    if (!started) return DAMPR_ERR_ARG;
    *started = HostPool::get().threads_started();
    return DAMPR_OK;
}

// The same rows straight into part files.  Buffered writes to ONE file serialise on its inode lock, so
// large outputs are split by row range into up to max_files files `<prefix><first_index + j>`, each
// formatted and written by its own thread (the reference writes one part file per sink job as well:
// SinkStageRunner.sink stagerunner.py:165-189, SinkWriter dataset.py:264-282).
static int32_t sink_rows(const char *prefix, uint32_t first_index, uint32_t max_files, uint64_t n,
                         int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                         const uint32_t *widths, const void *const *aux, const void *const *aux2,
                         uint64_t *out_len, uint32_t *n_files, const RowFmt *fmt) {
    if (!prefix || !kinds || !ptrs || !out_len || !n_files || ncols < 1 || ncols > 16 || max_files < 1)
        return DAMPR_ERR_ARG;
    const auto t_call = SinkClock::now();
    HostPool &pool = HostPool::get();
    auto pool_lock = pool.lock();
    IntDicts idc;
    lower_int_dicts(pool, ncols, kinds, widths, aux, aux2, idc);
    kinds = idc.kinds.data();
    aux = idc.aux.data();
    aux2 = idc.aux2.data();
    JoinArgs a{n, ncols, kinds, ptrs, widths, aux, aux2};
    // the fixed part of the longest possible row: fixed widths, the longest string of every dictionary formatted
    // above, separators. A caller's own dictionary gives no length: each writer bounds it over its own rows.
    u64 row_fixed = (u64)ncols;
    if (fmt) {
        row_fixed = fmt->row_end.size();
        for (auto &x : fmt->pre) row_fixed += x.size();
    }
    for (int c = 0; c < ncols; ++c) row_fixed += kinds[c] == 0 ? widths[c] : idc.longest[c];
    const int T = (int)std::min<u64>(std::min<u64>(HostPool::width(), max_files), std::max<u64>(1, n / 32768));
    std::vector<u64> lens(T, 0);
    std::vector<SinkTimes> tms(T);
    tms[0].prep = ms_since(t_call);
    const auto t_go = SinkClock::now();
    std::atomic<int> bad{0};
    pool.run(T, [&](int t) {
        SinkTimes &tm = tms[t];
        tm.start = ms_since(t_go);
        auto t0 = SinkClock::now();
        const u64 lo = n * t / T, hi = n * (t + 1) / T;
        u64 max_row = row_fixed;
        for (int c = 0; c < ncols; ++c) {
            if (kinds[c] == 0 || idc.blobs[c].size()) continue;
            const u32 *off = (const u32 *)aux2[c];
            const u32 *inv = (const u32 *)ptrs[c];
            u32 m = 0;
            for (u64 i = lo; i < hi; ++i) m = std::max(m, inv[i]);
            u32 longest = 0;
            for (u32 j = 0; j <= m; ++j) longest = std::max(longest, off[j + 1] - off[j]);
            max_row += longest;
        }
        // the upper bound of the range: pages that are never written cost nothing, one pass over the rows
        const size_t need = (hi - lo) * max_row + 64;
        u8 *buf = hi > lo ? pool.buffer(t, need) : nullptr;
        const bool own = hi > lo && !buf;
        if (own) buf = (u8 *)malloc(need);
        if (hi > lo && !buf) {
            bad.store(1);
            return;
        }
        // Creating files in one directory serialises on the directory's lock: 16 writers that open at the same
        // moment queue for about 2 ms. Writer t opens its file after the first t/T of its rows, so the creations are
        // spread over the formatting and none waits for another.
        auto rows = [&](u64 from, u64 to, u8 *out) {
            return to > from ? (fmt ? join_rows_fmt(a, *fmt, from, to, out) : join_rows_fast(a, from, to, out)) : 0;
        };
        const u64 mid = lo + (hi - lo) * (u64)t / (u64)T;
        u64 len = rows(lo, mid, buf);
        tm.format = ms_since(t0);
        t0 = SinkClock::now();
        std::string path = std::string(prefix) + std::to_string(first_index + (u32)t);
        int fd = open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
        tm.open = ms_since(t0);
        if (fd < 0) {
            bad.store(1);
            if (own) free(buf);
            return;
        }
        t0 = SinkClock::now();
        len += rows(mid, hi, buf + len);
        tm.format += ms_since(t0);
        t0 = SinkClock::now();
        u64 done = 0;
        while (done < len) {
            ssize_t w = write(fd, buf + done, len - done);
            if (w <= 0) {
                bad.store(1);
                break;
            }
            done += (u64)w;
        }
        tm.write = ms_since(t0);
        t0 = SinkClock::now();
        if (own) free(buf);
        if (close(fd) != 0) bad.store(1);
        tm.close = ms_since(t0);
        lens[t] = len;
    });
    {
        SinkTimes mx;
        mx.prep = tms[0].prep;
        for (const SinkTimes &x : tms) {
            mx.start = std::max(mx.start, x.start);
            mx.open = std::max(mx.open, x.open);
            mx.format = std::max(mx.format, x.format);
            mx.write = std::max(mx.write, x.write);
            mx.close = std::max(mx.close, x.close);
        }
        std::lock_guard<std::mutex> lk(g_sink_times_mu);
        g_sink_times = mx;
    }
    u64 total = 0;
    for (int t = 0; t < T; ++t) total += lens[t];
    *out_len = total;
    *n_files = (u32)T;
    return bad.load() ? DAMPR_ERR_ARG : DAMPR_OK;
}

extern "C" int32_t dampr_host_sink_tsv(const char *prefix, uint32_t first_index, uint32_t max_files, uint64_t n,
                                       int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                                       const uint32_t *widths, const void *const *aux, const void *const *aux2,
                                       uint64_t *out_len, uint32_t *n_files) {
    return sink_rows(prefix, first_index, max_files, n, ncols, kinds, ptrs, widths, aux, aux2, out_len, n_files, nullptr);
}

// The same part files with a byte string in front of every column (col_pre[c], NUL-terminated, may be empty) and
// row_end instead of the newline: no separators of its own. sink_json's lines (SinkWriter.add_record over
// json.dumps(value), dampr.py:531-539) are this with pre = `["`, `", `, `, ` ... and row_end = `]\n`.
extern "C" int32_t dampr_host_sink_fmt(const char *prefix, uint32_t first_index, uint32_t max_files, uint64_t n,
                                       int32_t ncols, const int32_t *kinds, const void *const *ptrs,
                                       const uint32_t *widths, const void *const *aux, const void *const *aux2,
                                       const char *const *col_pre, const char *row_end, uint64_t *out_len,
                                       uint32_t *n_files) {
    if (!col_pre || !row_end || ncols < 1 || ncols > 16) return DAMPR_ERR_ARG;
    RowFmt f;
    for (int c = 0; c < ncols; ++c) f.pre.emplace_back(col_pre[c] ? col_pre[c] : "");
    f.row_end = row_end;
    return sink_rows(prefix, first_index, max_files, n, ncols, kinds, ptrs, widths, aux, aux2, out_len, n_files, &f);
}

// Sorted distinct values + inverse index of a non-negative int64 column (the dictionary encoding of a
// count column, plan.DictCol).  Values below `table` go through a presence table (two linear passes,
// no sort); the others are returned as-is in big_vals/big_rows for the caller to sort (rare: the tail
// of a Zipf count distribution).  uniq must hold min(n, table) values; *n_big <= big_cap or the call
// fails.  inv[i] for big rows is left untouched.  first_row (optional, min(n, table) entries) receives the
// first row holding each distinct value.
extern "C" int32_t dampr_host_unique_small(const int64_t *col, uint64_t n, uint64_t table, int64_t *uniq,
                                           uint64_t *n_uniq, uint32_t *inv, uint32_t *first_row,
                                           int64_t *big_vals, uint64_t *big_rows, uint64_t big_cap,
                                           uint64_t *n_big) {
    if (!col || !uniq || !n_uniq || !inv || !n_big || table == 0 || table > (1ULL << 26) || n >= (1ULL << 32))
        return DAMPR_ERR_ARG;
    // three passes, the two over the rows split over a few threads: (1) mark the values present (and the smallest
    // row holding each), collect the rows outside the table; (2) rank the marked values in ascending order;
    // (3) look every row's rank up
    std::vector<u32> rank(table, 0);
    std::vector<u32> first(first_row ? table : 0, 0xFFFFFFFFu);
    HostPool &pool = HostPool::get();
    auto pool_lock = pool.lock();
    const int T = (int)std::max<u64>(1, std::min<u64>(std::min(HostPool::width(), 8), n / 65536));
    std::vector<std::vector<std::pair<int64_t, u64>>> bigs((size_t)T);
    auto mark = [&](int t) {
        const u64 lo = n * t / T, hi = n * (t + 1) / T;
        auto &big = bigs[(size_t)t];
        for (u64 i = lo; i < hi; ++i) {
            const int64_t v = col[i];
            if (v >= 0 && (u64)v < table) {
                if (!rank[(u64)v]) rank[(u64)v] = 1;   // (every writer stores the same value)
                if (first_row) {
                    u32 *f = &first[(u64)v];
                    u32 cur = __atomic_load_n(f, __ATOMIC_RELAXED);
                    while ((u32)i < cur && !__atomic_compare_exchange_n(f, &cur, (u32)i, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {
                    }
                }
            } else {
                big.emplace_back(v, i);
            }
        }
    };
    pool.run(T, mark);
    u64 nb = 0;
    for (auto &big : bigs) {
        if (nb + big.size() > big_cap) return DAMPR_ERR_ARG;
        for (auto &pr : big) {
            big_vals[nb] = pr.first;
            big_rows[nb] = pr.second;
            ++nb;
        }
    }
    u64 m = 0;
    for (u64 v = 0; v < table; ++v) {
        if (rank[v]) {
            uniq[m] = (int64_t)v;
            if (first_row) first_row[m] = first[v];
            rank[v] = (u32)m++;
        }
    }
    auto look = [&](int t) {
        const u64 lo = n * t / T, hi = n * (t + 1) / T;
        for (u64 i = lo; i < hi; ++i) {
            const int64_t v = col[i];
            if (v >= 0 && (u64)v < table) inv[i] = rank[(u64)v];
        }
    };
    pool.run(T, look);
    *n_uniq = m;
    *n_big = nb;
    return DAMPR_OK;
}

// ---- K9 for exchanged runs: decode the key codes of a kv (key = token code) into fixed-width ASCII ----
namespace {
__global__ void kv_words_kernel(const ulonglong2 *__restrict__ rec, u64 n, int mode, u32 width,
                                u8 *__restrict__ out_words) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 k = rec[i].x;
        u8 *w = out_words + i * width;
        u32 m = 0;
        if (!(k >> 63)) {
            if (mode == DAMPR_TOK_WS) {
                for (; k && m < width; ++m) {
                    w[m] = (u8)(k & 127);
                    k >>= 7;
                }
            } else {
                const char *sym = "\0" "0123456789_abcdefghijklmnopqrstuvwxyz";
                for (; k && m < width; ++m) {
                    w[m] = (u8)sym[k % 38];
                    k /= 38;
                }
            }
        }
        for (; m < width; ++m) w[m] = 0;  // hashed codes stay empty: the caller patches them
    }
}
}  // namespace

extern "C" int32_t dampr_kv_decode_words(dampr_ctx *ctx, dampr_kv *kv, int32_t mode, uint32_t width,
                                         uint8_t *words_host) {
    ARG_CHECK(ctx, ctx && kv && (words_host || kv->n == 0), "null");
    ARG_CHECK(ctx, width >= 16 && width <= 256 && (width % 8) == 0, "width must be a multiple of 8 in [16, 256]");
    if (kv->n == 0) return DAMPR_OK;
    wait_uploads(ctx);
    u8 *d = (u8 *)pool_alloc(ctx, kv->n * width);
    ARG_CHECK(ctx, d != nullptr, "device allocation failed");
    {
        ScopedTimer tm(ctx, DAMPR_K_TABLE_EXTRACT);
        kv_words_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(kv->rec, kv->n, mode, width, d);
    }
    cudaError_t e = cudaGetLastError();
    int rc2 = DAMPR_OK;
    if (e == cudaSuccess) rc2 = staged_d2h(ctx, words_host, d, kv->n * width, ctx->stream);
    pool_free(ctx, d);
    if (e != cudaSuccess) {
        ctx->err = std::string("kv decode_words failed: ") + cudaGetErrorString(e);
        return DAMPR_ERR_CUDA;
    }
    return rc2;
}

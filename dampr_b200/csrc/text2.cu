// text2.cu — second-generation tokenise + normalise + key code + combine kernel (K0/K1/K2).
//
// Same semantics as text.cu (which stays as the byte-compare verifier and as the fallback for lines
// longer than this kernel's window); replaces the same reference code:
//   TextLineDataset.read dampr/dataset.py:458-476, Map.stream(user lambdas) dampr/base.py:30-33
//   (examples/wc.py:12, benchmarks/tf-idf-dampr.py:12-14), ReducedWriter.add_record dampr/dataset.py:100-105.
//
// What changed, driven by the ncu profile of v1 (profiles/r01_text_v1_*.txt: 7.2 warp-instructions per
// byte, 9 of 32 lanes active, 34 % of samples at block barriers):
//   * one block barrier per 16 KB tile: the tile arrives by TMA (cp.async.bulk + mbarrier; single window
//     at 3-4 CTAs/SM, double buffered at 2), all threads classify it 4 bytes per SWAR step into bit masks,
//     then every warp owns one 2 KB strip and needs no further block sync;
//   * one token per lane: token starts of 32 mask words are ranked with a warp scan and scattered to a
//     per-warp position buffer, so all lanes do the same work on different tokens;
//   * key codes without a per-character loop: the token's 12 bytes are fetched with three funnel
//     shifts, mapped to symbols with SWAR arithmetic and packed base-38 (or 7 bits per char for
//     str.split) in a fixed number of instructions;
//   * set() de-duplication by shuffle compares with the earlier lanes of the same line (the MATCH.ANY
//     variant, kept behind DAMPR_TEXT_USE_MATCH, measured slower) plus a short per-warp history of the
//     line that straddles a round;
//   * a 2-way bucketed shared-memory combiner absorbs the Zipf head; misses are queued per warp and
//     flushed 32 at a time to the L2-resident global table.
#include "common.cuh"

#ifndef DAMPR_TEXT_USE_MATCH
#define DAMPR_TEXT_USE_MATCH 0
#endif

static bool g_text_cr_is_data = false;  // set per launch from the mode flags (one host thread drives a ctx)

namespace {

constexpr int V_THREADS = 256;
constexpr int V_WARPS = V_THREADS / 32;
constexpr int V_LEAD = 32;
constexpr int V_STRIP = 2048;
constexpr int V_OWN = V_STRIP * V_WARPS;  // 16384
constexpr int V_HALO = 2048;
constexpr int V_WIN = V_LEAD + V_OWN + V_HALO;  // 18464
constexpr int V_WORDS = V_WIN / 32;             // 577
constexpr int V_STAB = 2048;
constexpr int V_STAB_LOG = 11;
constexpr int V_HCAP = 256;   // distinct tokens remembered for the line that straddles a round
constexpr int V_TPOS = 544;   // token starts of one 32-word batch (at most 512)
constexpr u32 V_G_MAX_PROBES = 1u << 14;

static_assert(V_WIN % 32 == 0, "window must be whole mask words");
static_assert(TEXT_LEAD >= V_LEAD, "lead-in");
static_assert(TEXT_TAIL_PAD >= V_WIN + 64, "tail pad");

struct TableView2 {
    u64 *keys;
    u64 *counts;
    u64 *reps;
    u64 *stats;
    u64 mask;
    u64 seed;
    u64 *fb;      // fallback list: (global offset of the line << 16) | length, lines the host must tokenise
    u32 fb_cap;
    u32 cr_is_data;  // 1: '\r' is an ordinary byte (binary-mode .gz sources); 0: it ends lines (text mode)
};
enum { S_ENTRIES = 0, S_LINES = 1, S_EMPTY = 2, S_FOLDED = 3, S_FLAGS = 4, S_LONG = 5, S_RAW = 6, S_FALLBACK = 7 };
constexpr int V_MAXBAD = 8;  // lines per warp region that may go to the host before the whole scan gives up

// WS (str.split mode): no per-line history; the miss queue also carries the representative of a long token
template <int HCAP, bool WS>
struct WarpScratchT {
    alignas(8) u64 hist[WS ? 1 : HCAP];
    alignas(8) u64 missq[64];  // keys that missed the shared-memory combiner, flushed 32 at a time
    alignas(8) u64 missr[WS ? 64 : 1];
    u32 dtab[WS ? 1 : 64];  // set() de-duplication of a round: lanes per hash slot
    u16 tpos[V_TPOS];
    u16 badterm[V_MAXBAD];  // terminators of the lines of this region that were handed to the host
};
constexpr u32 V_REP_UNPUB = 0xFFFFFFFFu;

// Three builds of the kernel, named by the CTAs per SM they are sized for (VAR):
//   2  double-buffered window (the next tile is in flight while this one is processed), 2048-entry combiner
//   3  single window, 2048-entry combiner: more warps to hide the smem / dependency latencies the ncu
//      profile shows; the other CTAs cover the TMA wait
//   4  single window, 1024-entry combiner, shorter per-line history (<= 64 registers per thread)
template <int VAR, bool WS>
struct Smem2T {
    static constexpr int NBUF = (VAR == 2) ? 2 : 1;
    static constexpr int HCAP = (VAR == 2) ? V_HCAP : (VAR == 3 ? V_HCAP / 2 : V_HCAP / 4);
    static constexpr int STAB_LOG = (VAR == 4) ? V_STAB_LOG - 1 : V_STAB_LOG;
    static constexpr int STAB = 1 << STAB_LOG;
    alignas(16) u8 text[NBUF][V_WIN];
    u32 w[NBUF][V_WORDS + 3];
    u32 nl[NBUF][V_WORDS + 3];
    u32 badw[NBUF][((V_WORDS + V_THREADS - 1) / V_THREADS) * V_WARPS];  // bit per 32-byte window word: holds a byte the device cannot tokenise
    alignas(8) u64 tabk[STAB];
    u32 tabc[STAB];
    // str.split mode: last occurrence (byte offset from own_lo - V_LEAD) of the long token an entry holds
    u32 tabr[WS ? STAB : 1];
    WarpScratchT<HCAP, WS> ws[V_WARPS];
    alignas(8) u64 bar[2];
    u32 flags;
};

__device__ __forceinline__ u32 ge7(u32 x7, u32 k) { return (x7 + (0x80u - k) * 0x01010101u) & 0x80808080u; }
__device__ __forceinline__ u32 eq7(u32 x7, u32 k) {
    u32 z = x7 ^ (k * 0x01010101u);
    return ~(z + 0x7F7F7F7Fu) & 0x80808080u;
}
__device__ __forceinline__ u32 movemask4(u32 hi) { return (((hi >> 7) & 0x01010101u) * 0x01020408u) >> 24; }

template <int MODE>
__device__ __forceinline__ void classify4(u32 x, u32 &wbits, u32 &nlbits, u32 &bad) {
    u32 x7 = x & 0x7F7F7F7Fu;
    u32 hi = x & 0x80808080u;
    bad |= hi;
    u32 nl = eq7(x7, 0x0A) & ~hi;
    u32 word;
    if (MODE == DAMPR_TOK_WS) {
        u32 ws = (ge7(x7, 0x09) & ~ge7(x7, 0x0E)) | (ge7(x7, 0x1C) & ~ge7(x7, 0x21));
        word = ~ws & 0x80808080u;
    } else {
        u32 y = x7 | 0x20202020u;
        u32 alpha = ge7(y, 0x61) & ~ge7(y, 0x7B);
        u32 digit = ge7(x7, 0x30) & ~ge7(x7, 0x3A);
        word = alpha | digit | eq7(x7, 0x5F);
    }
    // '\r' (universal newlines): flagged in every mode -- the \w tokenisers and the line count depend on it, the
    // str.split token counts do not and the host ignores the flag for them
    bad |= (eq7(x7, 0x0D) >> 1);
    word &= ~hi;
    wbits = movemask4(word);
    nlbits = movemask4(nl);
}

// returns the representative the entry held before this call (~0 if none / not a hashed token)
__device__ __forceinline__ u64 gtab_add2(const TableView2 &t, u64 key, u64 cnt, u64 rep) {
    u64 slot = mix64(key) & t.mask;
    for (u32 probe = 0; probe < V_G_MAX_PROBES; ++probe) {
        u64 k = *((volatile u64 *)&t.keys[slot]);
        if (k == 0) {
            k = atomicCAS(&t.keys[slot], 0ULL, key);
            if (k == 0) {
                atomicAdd(&t.stats[S_ENTRIES], 1ULL);
                k = key;
            }
        }
        if (k == key) {
            atomicAdd(&t.counts[slot], cnt);
            return (rep != ~0ULL) ? atomicMin(&t.reps[slot], rep) : ~0ULL;
        }
        slot = (slot + 1) & t.mask;
    }
    atomicOr(&t.stats[S_FLAGS], (u64)DAMPR_TF_TABLEFULL);
    return ~0ULL;
}

// keep [lo, hi) of the 32 positions starting at base
__device__ __forceinline__ u32 range_mask(u32 base, u32 lo, u32 hi) {
    if (base + 32 <= lo || base >= hi) return 0;
    u32 keep = 0xFFFFFFFFu;
    if (base < lo) keep &= ~((1u << (lo - base)) - 1u);
    if (base + 32 > hi) keep &= (1u << (hi - base)) - 1u;
    return keep;
}

// first set bit at position >= from in mask words [0, nwords): warp-cooperative, returns 0xFFFFFFFF if none
__device__ __forceinline__ u32 warp_find_first(const u32 *m, u32 from, u32 limit_words, u32 lane) {
    u32 w0 = from >> 5;
    for (u32 wb = w0; wb < limit_words; wb += 32) {
        u32 wi = wb + lane;
        u32 v = (wi < limit_words) ? m[wi] : 0u;
        if (wi == w0) v &= ~((1u << (from & 31)) - 1u);
        u32 b = __ballot_sync(0xFFFFFFFFu, v != 0);
        if (b) {
            u32 l = (u32)__ffs(b) - 1u;
            u32 vv = __shfl_sync(0xFFFFFFFFu, v, l);
            return (wb + l) * 32u + (u32)__ffs(vv) - 1u;
        }
    }
    return 0xFFFFFFFFu;
}

// symbols (1..37) of 4 word characters packed in a u32; bytes that are not word characters give garbage
__device__ __forceinline__ u32 sym4(u32 x) {
    u32 y = (x & 0x7F7F7F7Fu) | 0x20202020u;
    u32 letter = ((y + 0x1F1F1F1Fu) & 0x80808080u) >> 7;  // y >= 0x61: letters and '_' (0x7F)
    u32 us = eq7(y, 0x7F) >> 7;
    return y - 0x2F2F2F2Fu - letter * 0x26u - us * 31u;
}
__device__ __forceinline__ u32 pack38(u32 s) {  // s0 + 38 s1 + 38^2 s2 + 38^3 s3
    return (s & 0xFFu) + 38u * ((s >> 8) & 0xFFu) + 1444u * ((s >> 16) & 0xFFu) + 54872u * (s >> 24);
}

template <int MODE>
__device__ __forceinline__ bool is_word_byte(u32 c) {
    if (MODE == DAMPR_TOK_WS) return !((c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x20)) && c < 0x80;
    return ((c | 0x20) >= 0x61 && (c | 0x20) <= 0x7A) || (c >= 0x30 && c <= 0x39) || c == 0x5F;
}

// length of the token starting at window position pos (continues in global memory past the window)
template <int MODE>
__device__ __forceinline__ u32 token_len2(const u32 *wm, u32 pos, const u8 *gtok) {
    u32 wi = pos >> 5, bi = pos & 31;
    u32 m = (~wm[wi]) >> bi;
    if (m) return (u32)__ffs(m) - 1u;
    u32 len = 32 - bi;
    for (++wi; wi < (u32)V_WORDS; ++wi) {
        m = ~wm[wi];
        if (m) return len + (u32)__ffs(m) - 1u;
        len += 32;
    }
    for (;; ++len) {
        if (!is_word_byte<MODE>(gtok[len]) || len > (1u << 30)) return len;
    }
}

// 64-bit key code: exact packing for short tokens, seeded hash | 1<<63 for long ones (same codes as v1)
template <int MODE>
__device__ __forceinline__ u64 token_code2(const u8 *text, u32 pos, u32 len, const u8 *gtok, u64 seed, bool &hashed) {
    constexpr u32 MAXEXACT = (MODE == DAMPR_TOK_WS) ? 9u : 12u;
    if (len <= MAXEXACT) {
        const u32 *tw = reinterpret_cast<const u32 *>(text + (pos & ~3u));
        u32 w0 = tw[0], w1 = tw[1], w2 = tw[2], w3 = tw[3];
        u32 sh = (pos & 3u) * 8u;
        u32 b0 = __funnelshift_r(w0, w1, sh), b1 = __funnelshift_r(w1, w2, sh), b2 = __funnelshift_r(w2, w3, sh);
        // zero the bytes past the token
        u32 k0 = len >= 4 ? 0xFFFFFFFFu : ((1u << (8 * len)) - 1u);
        u32 k1 = len >= 8 ? 0xFFFFFFFFu : (len > 4 ? ((1u << (8 * (len - 4))) - 1u) : 0u);
        u32 k2 = len >= 12 ? 0xFFFFFFFFu : (len > 8 ? ((1u << (8 * (len - 8))) - 1u) : 0u);
        if (MODE == DAMPR_TOK_WS) {
            b0 &= k0; b1 &= k1; b2 &= k2;
            // a NUL inside the token cannot be packed: hashed path
            u32 z0 = (~(((b0 & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | b0) & 0x80808080u) & (k0 & 0x80808080u);
            u32 z1 = (~(((b1 & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | b1) & 0x80808080u) & (k1 & 0x80808080u);
            u32 z2 = (~(((b2 & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | b2) & 0x80808080u) & (k2 & 0x80808080u);
            if (!(z0 | z1 | z2)) {
                u64 x = ((u64)b1 << 32) | b0;
                x = (x & 0x007F007F007F007FULL) | ((x & 0x7F007F007F007F00ULL) >> 1);
                x = (x & 0x00003FFF00003FFFULL) | ((x & 0x3FFF00003FFF0000ULL) >> 2);
                x = (x & 0x000000000FFFFFFFULL) | ((x & 0x0FFFFFFF00000000ULL) >> 4);
                hashed = false;
                return x | ((u64)(b2 & 0x7Fu) << 56);
            }
        } else {
            u32 s0 = sym4(b0) & k0, s1 = sym4(b1) & k1, s2 = sym4(b2) & k2;
            u64 g0 = pack38(s0), g1 = pack38(s1), g2 = pack38(s2);
            hashed = false;
            return g0 + 2085136ULL * g1 + 4347792138496ULL * g2;  // 38^4, 38^8
        }
    }
    hashed = true;
    u32 h1 = (u32)seed ^ 0x811C9DC5u, h2 = (u32)(seed >> 32) ^ 0x9747B28Cu;
    for (u32 i = 0; i < len; ++i) {
        u32 c = (pos + i < (u32)V_WIN) ? (u32)text[pos + i] : (u32)gtok[i];
        u32 v = c;
        if (MODE != DAMPR_TOK_WS) {
            // same symbol alphabet as the exact path (1..37)
            u32 y = (c & 0x7F) | 0x20;
            v = (c >= '0' && c <= '9') ? c - 0x2F : (c == '_' ? 11u : y - 0x55u);
        }
        h1 = (h1 ^ v) * 16777619u;
        h2 = (h2 ^ v) * 0x85EBCA6Bu + 0x9E3779B9u;
        h2 = (h2 << 13) | (h2 >> 19);
    }
    u64 h = mix64((((u64)h1) << 32 | h2) ^ ((u64)len * 0x9E3779B97F4A7C15ULL));
    return h | 0x8000000000000000ULL;
}

// str.split mode: is the token of `len` bytes at a equal to the token that STARTS at b? (b's token must
// also end after len bytes.)  Aligned 4-byte loads + funnel shifts; reads up to 7 bytes past the tokens,
// which the window halo / the text buffer's tail pad cover.
__device__ __forceinline__ bool tok_equal_ws(const u8 *a, const u8 *b, u32 len) {
    const u32 *aw = reinterpret_cast<const u32 *>(reinterpret_cast<uintptr_t>(a) & ~(uintptr_t)3);
    const u32 *bw = reinterpret_cast<const u32 *>(reinterpret_cast<uintptr_t>(b) & ~(uintptr_t)3);
    const u32 sa = (u32)(reinterpret_cast<uintptr_t>(a) & 3) * 8u, sb = (u32)(reinterpret_cast<uintptr_t>(b) & 3) * 8u;
    u32 a0 = aw[0], b0 = bw[0], diff = 0, i = 0;
    for (; i + 4 <= len; i += 4) {
        const u32 a1 = aw[(i >> 2) + 1], b1 = bw[(i >> 2) + 1];
        diff |= __funnelshift_r(a0, a1, sa) ^ __funnelshift_r(b0, b1, sb);
        a0 = a1;
        b0 = b1;
    }
    const u32 a1 = aw[(i >> 2) + 1], b1 = bw[(i >> 2) + 1];
    const u32 xa = __funnelshift_r(a0, a1, sa), xb = __funnelshift_r(b0, b1, sb);
    const u32 rem = len - i;  // 0..3
    diff |= (xa ^ xb) & ((1u << (8u * rem)) - 1u);
    const u32 term = (xb >> (8u * rem)) & 0xFFu;
    return diff == 0 && !is_word_byte<DAMPR_TOK_WS>(term);
}

template <int MODE, int VAR>
__global__ void __launch_bounds__(V_THREADS, VAR)
text_count2_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, u64 base_offset, TableView2 tab) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr bool WS = (MODE == DAMPR_TOK_WS);
    typedef Smem2T<VAR, WS> Smem2;
    constexpr int NBUF = Smem2::NBUF;
    constexpr int HCAP = Smem2::HCAP;
    constexpr int V_STAB = Smem2::STAB;          // shadows the namespace-level defaults inside the kernel
    constexpr int V_STAB_LOG = Smem2::STAB_LOG;
    Smem2 &s = *reinterpret_cast<Smem2 *>(smem_raw);
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 lt_mask = (1u << lane) - 1u;
    const u64 ntiles = (own_hi - own_lo + V_OWN - 1) / V_OWN;
    WarpScratchT<HCAP, WS> &ws = s.ws[warp];

    if (tid == 0) {
        mbar_init(&s.bar[0], 1);
        mbar_init(&s.bar[1], 1);
        fence_mbar_init();
        s.flags = 0;
    }
    for (int i = tid; i < V_STAB; i += V_THREADS) {
        s.tabk[i] = 0;
        s.tabc[i] = 0;
        if (WS) s.tabr[i] = V_REP_UNPUB;
    }
    __syncthreads();

    u64 acc_lines = 0, acc_empty = 0, acc_folded = 0, acc_long = 0, acc_raw = 0;
    u32 my_flags = 0;
    u32 phase[2] = {0, 0};

    // add cnt occurrences of a long token to the global table; false if the representative the entry
    // already holds is a different string (a 64-bit code collision).  atomicMin hands back the
    // representative an earlier token of this code published; comparing every later one with it proves by
    // induction that the entry holds ONE token, so a collision cannot merge two words silently.
    auto hashed_insert = [&](u64 k, u64 rep, u64 cnt) -> bool {
        const u64 old = gtab_add2(tab, k, cnt, rep);
        if (old == ~0ULL || old == rep) return true;
        const u32 l2 = (u32)(rep & 0xFFFFFu);
        if ((u32)(old & 0xFFFFFu) != l2) return false;
        const u8 *pa = text + ((rep >> 20) - base_offset);
        const u8 *pb = text + ((old >> 20) - base_offset);
        if (WS) return tok_equal_ws(pa, pb, l2);
        bool same = true;
        for (u32 i = 0; same && i < l2; ++i) {
            u32 ca = pa[i], cb = pb[i];
            if (ca >= 'A' && ca <= 'Z') ca |= 0x20;
            if (cb >= 'A' && cb <= 'Z') cb |= 0x20;
            same = ca == cb;
        }
        return same;
    };

    u64 tile = blockIdx.x;
    if (tile < ntiles && tid == 0) {
        mbar_expect_tx(&s.bar[0], V_WIN);
        tma_load_1d(s.text[0], text + (own_lo + tile * (u64)V_OWN) - V_LEAD, V_WIN, &s.bar[0]);
    }
    u32 buf = 0;
    for (; tile < ntiles; tile += gridDim.x, buf ^= (NBUF - 1)) {
        const u64 sgl = own_lo + tile * (u64)V_OWN;
        const u32 own_len = (u32)min((u64)V_OWN, own_hi - sgl);
        const u8 *tx = s.text[buf];
        u32 *wm = s.w[buf];
        u32 *nm = s.nl[buf];
        mbar_wait(&s.bar[buf], phase[buf]);
        phase[buf] ^= 1;

        // ---- classify the whole window (all threads) ------------------------------------------------
        // A byte the device cannot tokenise like Python does (non-ASCII; '\r' where it ends lines) marks its
        // 32-byte word in badw. [^\w]+ modes hand just the LINES holding such bytes to the host (per-line
        // fallback, below); str.split mode keeps the scan-wide flags.
        u32 bad = 0;
        u32 *bw = s.badw[buf];
#pragma unroll 1
        for (int kk = 0; kk < (V_WORDS + V_THREADS - 1) / V_THREADS; ++kk) {
            const int i = tid + kk * V_THREADS;
            u32 wbad = 0;
            if (i < V_WORDS) {
                const uint4 *p = reinterpret_cast<const uint4 *>(tx + 32 * i);
                uint4 a = p[0], b = p[1];
                u32 wmk = 0, nmk = 0, wb, nb;
                classify4<MODE>(a.x, wb, nb, wbad); wmk |= wb;        nmk |= nb;
                classify4<MODE>(a.y, wb, nb, wbad); wmk |= wb << 4;   nmk |= nb << 4;
                classify4<MODE>(a.z, wb, nb, wbad); wmk |= wb << 8;   nmk |= nb << 8;
                classify4<MODE>(a.w, wb, nb, wbad); wmk |= wb << 12;  nmk |= nb << 12;
                classify4<MODE>(b.x, wb, nb, wbad); wmk |= wb << 16;  nmk |= nb << 16;
                classify4<MODE>(b.y, wb, nb, wbad); wmk |= wb << 20;  nmk |= nb << 20;
                classify4<MODE>(b.z, wb, nb, wbad); wmk |= wb << 24;  nmk |= nb << 24;
                classify4<MODE>(b.w, wb, nb, wbad); wmk |= wb << 28;  nmk |= nb << 28;
                wm[i] = wmk;
                nm[i] = nmk;
                if (tab.cr_is_data) wbad &= 0x80808080u;
            }
            bad |= wbad;
            if (!WS) {
                // the 32 words a warp classifies in one pass are consecutive: one ballot is their flag word
                const u32 bb = __ballot_sync(0xFFFFFFFFu, wbad != 0);
                if (lane == 0) bw[kk * V_WARPS + warp] = bb;
            }
        }
        if (WS && bad) my_flags |= ((bad & 0x80808080u) ? DAMPR_TF_NONASCII : 0u) | ((bad & 0x40404040u) ? DAMPR_TF_CR : 0u);
        __syncthreads();
        // every warp is past tile-1: its buffer may be refilled while this tile is processed
        if (NBUF == 2 && tid == 0) {
            u64 nxt = tile + gridDim.x;
            if (nxt < ntiles) {
                fence_proxy_async();
                mbar_expect_tx(&s.bar[buf ^ 1], V_WIN);
                tma_load_1d(s.text[buf ^ 1], text + (own_lo + nxt * (u64)V_OWN) - V_LEAD, V_WIN, &s.bar[buf ^ 1]);
            }
        }

        auto strip = [&]() {
        // ---- this warp's strip ----------------------------------------------------------------------
        const u32 st_lo = V_LEAD + warp * V_STRIP;  // window coords of the strip
        if (st_lo >= V_LEAD + own_len) return;      // (warp-uniform) strip beyond the owned bytes
        const u32 st_hi = min(st_lo + (u32)V_STRIP, (u32)V_LEAD + own_len);
        const u8 *gwin = text + sgl - V_LEAD;

        // lines whose first byte lies in the strip: newline at [st_lo-1, st_hi-1)
        {
            u32 lo = st_lo - 1, hi = st_hi - 1;
            for (u32 wb = lo >> 5; wb * 32 < hi; wb += 32) {
                u32 wi = wb + lane;
                if (wi * 32 < hi && wi < (u32)V_WORDS) {
                    u32 starts = nm[wi] & range_mask(wi * 32, lo, hi);
                    // a start at global position >= n is not a line (virtual newline padding)
                    while (starts) {
                        u32 b = (u32)__ffs(starts) - 1u;
                        starts &= starts - 1;
                        if (sgl - V_LEAD + wi * 32 + b + 1 < n) acc_lines++;
                    }
                }
            }
        }

        u32 rlo, rhi;  // token starts handled by this warp: [rlo, rhi)
        if (MODE == DAMPR_TOK_WS) {
            rlo = st_lo;
            rhi = st_hi;
        } else {
            u32 q = warp_find_first(nm, st_lo - 1, (st_hi + 31) >> 5, lane);
            if (q == 0xFFFFFFFFu || q + 1 >= st_hi) return;    // no line starts inside the strip
            u32 tl = warp_find_first(nm, st_hi - 1, V_WORDS, lane);
            if (tl == 0xFFFFFFFFu) {
                my_flags |= DAMPR_TF_LONGLINE;
                return;
            }
            rlo = q + 1;
            rhi = tl + 1;
        }

        // ---- per-line fallback ([^\w]+ modes): lines of this region that hold a byte the device cannot tokenise
        // produce no tokens here; their (offset, length) goes to the fallback list and the host tokenises them
        // with Python's own rules (universal newlines, Unicode \w, str.lower) and merges the counts.
        u32 nbad = 0;  // warp-uniform
        if (!WS) {
            const u32 fw0 = rlo >> 5, fw1 = (rhi - 1) >> 5;
            bool anyb = false;
            for (u32 g = fw0 >> 5; g <= (fw1 >> 5); ++g) {
                u32 fl = s.badw[buf][g];
                if (g == (fw0 >> 5)) fl &= ~((1u << (fw0 & 31)) - 1u);
                if (g == (fw1 >> 5) && (fw1 & 31) != 31) fl &= (1u << ((fw1 & 31) + 1)) - 1u;
                anyb |= fl != 0;
            }
            if (anyb) {
                u32 pos = rlo;
                while (pos < rhi) {
                    // next bad byte at or after pos (32 bytes per step, one per lane)
                    u32 bpos = 0xFFFFFFFFu;
                    for (u32 wq = pos >> 5; wq * 32 < rhi && bpos == 0xFFFFFFFFu; ++wq) {
                        if (!((s.badw[buf][wq >> 5] >> (wq & 31)) & 1u)) continue;
                        const u32 bp = wq * 32 + lane;
                        const u32 c = tx[bp];
                        const bool isb = bp >= pos && bp < rhi && (c >= 0x80u || (c == 0x0Du && !tab.cr_is_data));
                        const u32 bm = __ballot_sync(0xFFFFFFFFu, isb);
                        if (bm) bpos = wq * 32 + (u32)__ffs(bm) - 1u;
                    }
                    if (bpos == 0xFFFFFFFFu) break;
                    // its line: q = first byte (after the previous newline), p = terminator
                    u32 q;
                    {
                        int w2 = (int)(bpos >> 5);
                        u32 m = nm[w2] & (((bpos & 31) == 0) ? 0u : ((1u << (bpos & 31)) - 1u));
                        while (!m && w2 > (int)(rlo >> 5)) {
                            --w2;
                            m = nm[w2];
                        }
                        q = m ? (32u * w2 + (31u - (u32)__clz(m)) + 1u) : rlo;
                        if (q < rlo) q = rlo;
                    }
                    const u32 pterm = warp_find_first(nm, bpos, V_WORDS, lane);
                    if (pterm == 0xFFFFFFFFu || pterm >= rhi || nbad >= (u32)V_MAXBAD) {
                        // cannot be isolated here (line leaves the window / too many of them): scan-wide fallback
                        my_flags |= DAMPR_TF_NONASCII;
                        break;
                    }
                    if (lane == 0) {
                        ws.badterm[nbad] = (u16)pterm;
                        const u64 goff = base_offset + (sgl - V_LEAD) + q;
                        if (goff < n) {  // a start at or past n is the virtual terminator padding, not a line
                            const u64 ix = atomicAdd(&tab.stats[S_FALLBACK], 1ULL);
                            if (ix < (u64)tab.fb_cap) tab.fb[ix] = (goff << 16) | (u64)(pterm - q);
                            else my_flags |= DAMPR_TF_NONASCII;
                            acc_lines--;  // the host counts the lines of this range (universal newlines)
                        }
                    }
                    for (u32 w = (q >> 5) + lane; w * 32 < pterm; w += 32) {
                        const u32 km = range_mask(w * 32, q, pterm);
                        if (km) atomicAnd(&wm[w], ~km);
                    }
                    ++nbad;
                    pos = pterm + 1;
                }
                __syncwarp();
            }
        }

        // ---- batches of 32 mask words -----------------------------------------------------------------
        u32 hist_n = 0;
        u32 hist_line = 0xFFFFFFFFu;
        u32 line_base = 0;
        u32 nq = 0;   // queued combiner misses (warp-uniform)
        for (u32 wb = rlo >> 5; wb * 32 < rhi; wb += 32) {
            const u32 wi = wb + lane;
            u32 stm = 0, nlm = 0, wmk = 0;
            if (wi < (u32)V_WORDS && wi * 32 < rhi) {
                wmk = wm[wi];
                u32 prev = wi ? (wm[wi - 1] >> 31) : 0u;
                u32 keep = range_mask(wi * 32, rlo, rhi);
                stm = wmk & ~((wmk << 1) | prev) & keep;
                nlm = nm[wi] & keep;
            }
            // warp exclusive scans of token starts and newlines
            u32 c = (u32)__popc(stm) | ((u32)__popc(nlm) << 16);
            u32 v = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                if ((int)lane >= d) v += o;
            }
            const u32 tot = __shfl_sync(0xFFFFFFFFu, v, 31);
            const u32 excl = v - c;
            const u32 T = tot & 0xFFFFu;
            {
                u32 ix = excl & 0xFFFFu;
                u32 m = stm;
                while (m) {
                    u32 b = (u32)__ffs(m) - 1u;
                    m &= m - 1;
                    ws.tpos[ix++] = (u16)(wi * 32 + b);
                }
            }
            const u32 my_nl_base = line_base + (excl >> 16);
            __syncwarp();
            acc_raw += (lane == 0) ? T : 0;

            // ---- rounds: one token per lane ---------------------------------------------------------
            for (u32 r = 0; r < T; r += 32) {
                const u32 t = r + lane;
                const bool valid = t < T;
                const u32 vmask = __ballot_sync(0xFFFFFFFFu, valid);
                u64 key = 0;
                u32 line = 0, pos = 0, len = 0;
                bool hashed = false;
                if (valid) {
                    pos = ws.tpos[t];
                    len = token_len2<MODE>(wm, pos, gwin + pos);
                    key = token_code2<MODE>(tx, pos, len, gwin + pos, tab.seed, hashed);
                }
                if (MODE != DAMPR_TOK_WS) {
                    // line id = newlines of the region before the token
                    u32 src = valid ? ((pos >> 5) - wb) : 0u;
                    u32 nb_ = __shfl_sync(0xFFFFFFFFu, my_nl_base, src);
                    u32 nlw = __shfl_sync(0xFFFFFFFFu, nlm, src);
                    line = nb_ + (u32)__popc(nlw & ((1u << (pos & 31)) - 1u));
                }
                bool dup = !valid;
                if (MODE == DAMPR_TOK_NONWORD_LOWER_SET) {
#if DAMPR_TEXT_USE_MATCH
                    // (not built) merges equal codes here and in the combiner below without a byte compare: a
                    // build of it must pass the code-collision tests before it is selected
                    u32 m1 = 0, m2 = 0;
                    if (valid) {
                        m1 = __match_any_sync(vmask, key);
                        m2 = __match_any_sync(vmask, line);
                    }
                    if (valid && (m1 & m2 & lt_mask)) dup = true;
#else
                    // tokens of one line sit in consecutive lanes. Every lane drops its bit into the slot its
                    // key hashes to; the earlier lanes of the same line found in that slot are the only ones
                    // that can hold the same token, and they are compared exactly (64-bit key via shuffle).
                    // No false negatives: an equal key always lands in the same slot. (A compare with every
                    // earlier lane of the line by shuffles costs ~5 instructions per lane distance; MATCH.ANY
                    // iterates over the distinct values and is slower still.)
                    {
                        const u32 lkey = valid ? line : (0xFFFFFF00u | lane);
                        const u32 prev_line = __shfl_up_sync(0xFFFFFFFFu, lkey, 1);
                        const u32 seg_start = __ballot_sync(0xFFFFFFFFu, lane == 0 || prev_line != lkey);
                        const u32 first = 31u - (u32)__clz(seg_start & (lt_mask | (1u << lane)));  // first lane of my line
                        const u32 slot = (((u32)key ^ (u32)(key >> 32)) * 0x9E3779B1u) >> 26;
                        ws.dtab[lane] = 0;
                        ws.dtab[lane + 32] = 0;
                        __syncwarp();
                        if (valid) atomicOr(&ws.dtab[slot], 1u << lane);
                        __syncwarp();
                        u32 cand = valid ? (ws.dtab[slot] & lt_mask & ~((1u << first) - 1u)) : 0u;
                        while (__any_sync(0xFFFFFFFFu, cand != 0)) {
                            const u32 src = cand ? (31u - (u32)__clz(cand)) : lane;
                            const u64 ok = __shfl_sync(0xFFFFFFFFu, key, src);
                            if (cand) {
                                if (ok == key) dup = true;
                                cand &= ~(1u << src);
                            }
                        }
                    }
#endif
                    // tokens of the line that started in an earlier round: compare with its history
                    const bool in_hist_line = valid && line == hist_line;
                    if (__ballot_sync(0xFFFFFFFFu, in_hist_line) && hist_n) {
                        // the same slot scheme: lane j holds history entry j (the first 32 of them), tokens of
                        // the line look their slot up and compare with the entries found there
                        const u32 hslot = (((u32)key ^ (u32)(key >> 32)) * 0x9E3779B1u) >> 26;
                        const u64 hk = (lane < hist_n) ? ws.hist[lane] : 0ULL;
                        ws.dtab[lane] = 0;
                        ws.dtab[lane + 32] = 0;
                        __syncwarp();
                        if (lane < hist_n) atomicOr(&ws.dtab[(((u32)hk ^ (u32)(hk >> 32)) * 0x9E3779B1u) >> 26], 1u << lane);
                        __syncwarp();
                        u32 cand = in_hist_line ? ws.dtab[hslot] : 0u;
                        while (__any_sync(0xFFFFFFFFu, cand != 0)) {
                            const u32 src = cand ? (31u - (u32)__clz(cand)) : lane;
                            const u64 ok = __shfl_sync(0xFFFFFFFFu, hk, src);
                            if (cand) {
                                if (ok == key) dup = true;
                                cand &= ~(1u << src);
                            }
                        }
                        __syncwarp();
                        for (u32 j = 32; j < hist_n; ++j) {  // long lines: the rest of the history, entry by entry
                            const u64 hj = ws.hist[j];
                            if (in_hist_line && hj == key) dup = true;
                        }
                    }
                    // new history = distinct tokens of the line the last token of this round belongs to
                    const u32 last_lane = 31u - (u32)__clz(vmask);
                    const u32 last_line = __shfl_sync(0xFFFFFFFFu, line, last_lane);
                    if (last_line != hist_line) {
                        hist_line = last_line;
                        hist_n = 0;
                    }
                    const bool add = valid && !dup && line == last_line;
                    const u32 am = __ballot_sync(0xFFFFFFFFu, add);
                    const u32 na = (u32)__popc(am);
                    if (hist_n + na > (u32)HCAP) {
                        my_flags |= DAMPR_TF_LONGLINE;
                    } else {
                        if (add) ws.hist[hist_n + __popc(am & lt_mask)] = key;
                        hist_n += na;
                    }
                    __syncwarp();
                }
                // ---- fold: merge equal keys of the round, then one combiner update per distinct key --
                const bool live = valid && !dup;
                const u32 lmask = __ballot_sync(0xFFFFFFFFu, live);
                acc_folded += live ? 1 : 0;
                // long (hashed) tokens.  [^\\w]+ modes: rare, straight to the global table with inline K9
                // verification.  str.split mode: 10+ byte tokens are common and Zipf-hot, so they go through
                // the shared-memory combiner like the exact codes; an entry remembers the latest occurrence
                // of its token and every hit is compared with it (bytes) before it is counted.
                // set() de-duplication above compares codes only: a hashed token it dropped still goes to the
                // table with count 0, so its bytes are compared with the entry's representative like any other
                // and a different word of the same code sets TF_COLLISION instead of vanishing
                u64 myrep = ~0ULL;
                if (valid && hashed && (live || MODE == DAMPR_TOK_NONWORD_LOWER_SET)) {
                    u32 l2 = len;
                    if (l2 >= (1u << 20)) {
                        my_flags |= DAMPR_TF_LONGTOKEN;
                        l2 = (1u << 20) - 1;
                    }
                    myrep = ((base_offset + (sgl - V_LEAD) + pos) << 20) | l2;
                    acc_long += live ? 1 : 0;
                    if (!WS && !hashed_insert(key, myrep, live ? 1ULL : 0ULL)) my_flags |= DAMPR_TF_COLLISION;
                }
                const bool ins = live && (WS || !hashed);
                const u32 imask = __ballot_sync(0xFFFFFFFFu, ins);
                bool miss = false;
                // every inserting lane looks its slot pair up (convergent loads); one lane per distinct
                // key then updates the combiner
                u32 h = (u32)key * 0x9E3779B1u ^ (u32)(key >> 32) * 0x85EBCA6Bu;
                u32 slot = (h >> (32 - V_STAB_LOG)) & ~1u;
                u64 k0 = 0, k1 = 0;
                if (ins) {
                    const ulonglong2 kk = *reinterpret_cast<const ulonglong2 *>(&s.tabk[slot]);
                    k0 = kk.x;
                    k1 = kk.y;
                }
                if (ins) {
#if DAMPR_TEXT_USE_MATCH
                    u32 peers = __match_any_sync(imask, key);
#else
                    u32 peers = 1u << lane;  // no in-warp merge: equal keys serialise in the smem atomic
#endif
                    if (((u32)__ffs(peers) - 1u) == lane) {
                        const u32 cnt = (u32)__popc(peers);
                        int hs = -1;       // combiner entry of this key
                        bool fresh = false;  // this lane created it
                        if (k0 == key) {
                            hs = (int)slot;
                        } else if (k1 == key) {
                            hs = (int)slot + 1;
                        } else {
#pragma unroll 1
                            for (int pr = 0; pr < 2; ++pr) {  // 2-way bucket: a miss goes straight to the L2-resident global table
                                u64 k = s.tabk[slot];
                                if (k == 0) {
                                    k = atomicCAS(&s.tabk[slot], 0ULL, key);
                                    if (k == 0) {
                                        k = key;
                                        fresh = true;
                                    }
                                }
                                if (k == key) {
                                    hs = (int)slot;
                                    break;
                                }
                                slot = (slot + 1) & (V_STAB - 1);
                            }
                        }
                        if (WS && hashed && hs >= 0) {
                            const u32 r32 = (u32)(sgl - own_lo) + pos;
                            if (!fresh) {
                                const u32 prev = *reinterpret_cast<volatile u32 *>(&s.tabr[hs]);
                                if (prev == V_REP_UNPUB) {
                                    hs = -1;  // creator has not published yet: count this one in the global table
                                } else {
                                    const u8 *mine = (pos + len + 8u <= (u32)V_WIN) ? tx + pos : gwin + pos;
                                    if (!tok_equal_ws(mine, text + (own_lo + prev - V_LEAD), len)) my_flags |= DAMPR_TF_COLLISION;
                                }
                            }
                            if (hs >= 0) *reinterpret_cast<volatile u32 *>(&s.tabr[hs]) = r32;
                        }
                        if (hs >= 0) {
                            atomicAdd(&s.tabc[hs], cnt);
                        } else {
#if DAMPR_TEXT_USE_MATCH
                            if (!hashed_insert(key, myrep, (u64)cnt)) my_flags |= DAMPR_TF_COLLISION;
#else
                            miss = true;
#endif
                        }
                    }
                }
                (void)lmask;
                // misses go to the L2-resident global table in convergent batches of 32 (all lanes issue
                // their load + atomic together) instead of a few lanes at a time inside every round
                {
                    const u32 mm = __ballot_sync(0xFFFFFFFFu, miss);
                    if (mm) {
                        if (miss) {
                            const u32 qi = nq + __popc(mm & lt_mask);
                            ws.missq[qi] = key;
                            if (WS) ws.missr[qi] = myrep;
                        }
                        nq += (u32)__popc(mm);
                        __syncwarp();
                        if (nq >= 32) {
                            const u32 qi = nq - 32 + lane;
                            if (!hashed_insert(ws.missq[qi], WS ? ws.missr[qi] : ~0ULL, 1ULL)) my_flags |= DAMPR_TF_COLLISION;
                            nq -= 32;
                        }
                    }
                }
                __syncwarp();
            }
            line_base += tot >> 16;

            // ---- the '' token: terminators of owned lines in this batch ----------------------------
            if (MODE != DAMPR_TOK_WS) {
                u32 terms = nlm;
                while (terms) {
                    u32 b = (u32)__ffs(terms) - 1u;
                    terms &= terms - 1;
                    u32 p = wi * 32 + b;
                    if (nbad) {
                        bool gone = false;
                        for (u32 j = 0; j < nbad; ++j) gone |= ws.badterm[j] == (u16)p;
                        if (gone) continue;
                    }
                    u32 q;
                    {
                        int w2 = (int)(p >> 5);
                        u32 bi = p & 31;
                        u32 m = nm[w2] & ((bi == 0) ? 0u : ((1u << bi) - 1u));
                        for (;;) {
                            if (m) {
                                q = 32u * w2 + (31u - (u32)__clz(m)) + 1u;
                                break;
                            }
                            --w2;
                            if (w2 < 0) {
                                q = rlo;
                                break;
                            }
                            m = nm[w2];
                        }
                        if (q < rlo) q = rlo;
                    }
                    if (sgl - V_LEAD + q >= n) continue;  // virtual newline after a terminated file
                    bool A = !((wm[q >> 5] >> (q & 31)) & 1u);
                    bool B = (p > q) && !((wm[(p - 1) >> 5] >> ((p - 1) & 31)) & 1u);
                    if (MODE == DAMPR_TOK_NONWORD_LOWER_SET) acc_empty += (A || B) ? 1 : 0;
                    else acc_empty += (A ? 1 : 0) + (B ? 1 : 0);
                }
            }
            __syncwarp();
        }
        if (nq) {  // leftover misses of this strip
            if (lane < nq && !hashed_insert(ws.missq[lane], WS ? ws.missr[lane] : ~0ULL, 1ULL)) my_flags |= DAMPR_TF_COLLISION;
            __syncwarp();
        }
        };
        strip();
        if (NBUF == 1) {
            // single buffer: every warp must be done with the window before the next tile lands in it
            __syncthreads();
            if (tid == 0) {
                u64 nxt = tile + gridDim.x;
                if (nxt < ntiles) {
                    fence_proxy_async();
                    mbar_expect_tx(&s.bar[0], V_WIN);
                    tma_load_1d(s.text[0], text + (own_lo + nxt * (u64)V_OWN) - V_LEAD, V_WIN, &s.bar[0]);
                }
            }
        }
    }

    // ---- flush the shared-memory combiner, publish counters ----------------------------------------
    __syncthreads();
    for (int i = tid; i < V_STAB; i += V_THREADS) {
        const u64 k = s.tabk[i];
        if (!k) continue;
        u64 rep = ~0ULL;
        if (WS && (k >> 63)) {
            // representative of a long token = its latest occurrence in this CTA; its length is re-read
            const u64 goff = own_lo + s.tabr[i] - V_LEAD;
            u32 len = 0;
            while (len < (1u << 20) - 1u && is_word_byte<DAMPR_TOK_WS>(text[goff + len])) ++len;
            rep = ((base_offset + goff) << 20) | len;
        }
        if (!hashed_insert(k, rep, (u64)s.tabc[i])) my_flags |= DAMPR_TF_COLLISION;
    }
    u64 vals[5] = {acc_lines, acc_empty, acc_folded, acc_long, acc_raw};
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        u64 v = vals[k];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, d);
        vals[k] = v;
    }
    if (lane == 0) {
        if (vals[0]) atomicAdd(&tab.stats[S_LINES], vals[0]);
        if (vals[1]) atomicAdd(&tab.stats[S_EMPTY], vals[1]);
        if (vals[2]) atomicAdd(&tab.stats[S_FOLDED], vals[2]);
        if (vals[3]) atomicAdd(&tab.stats[S_LONG], vals[3]);
        if (vals[4]) atomicAdd(&tab.stats[S_RAW], vals[4]);
    }
    if (my_flags) atomicOr(&s.flags, my_flags);
    __syncthreads();
    if (tid == 0 && s.flags) atomicOr(&tab.stats[S_FLAGS], (u64)s.flags);
}

template <int MODE, int VAR>
int launch2n(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 lo, u64 hi) {
    if (hi <= lo) return DAMPR_OK;
    size_t smem = sizeof(Smem2T<VAR, MODE == DAMPR_TOK_WS>);
    auto kern = text_count2_kernel<MODE, VAR>;
    CUDA_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    u64 ntiles = (hi - lo + V_OWN - 1) / V_OWN;
    u64 grid = (u64)ctx->num_sms * VAR;
    if (grid > ntiles) grid = ntiles;
    TableView2 tv{t->keys, t->counts, t->reps, t->stats, t->cap - 1, 0x243F6A8885A308D3ULL, t->fb, t->fb_cap,
                  (u32)(g_text_cr_is_data ? 1 : 0)};
    wait_uploads(ctx);
    {
        ScopedTimer tm(ctx, DAMPR_K_TEXT_COUNT);
        kern<<<(unsigned)grid, V_THREADS, smem, ctx->stream>>>(tb->text, tb->n, lo, hi, 0, tv);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

template <int MODE>
int launch2(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 lo, u64 hi) {
    // str.split mode keeps 32-bit offsets (from the launch's own_lo) in the shared-memory combiner
    const u64 span = (MODE == DAMPR_TOK_WS) ? (1ULL << 31) : ~0ULL;
    for (u64 a = lo; a < hi;) {
        const u64 b = (hi - a > span) ? a + span : hi;
        const int rc = g_text_ctas == 4   ? launch2n<MODE, 4>(ctx, t, tb, a, b)
                       : g_text_ctas == 3 ? launch2n<MODE, 3>(ctx, t, tb, a, b)
                                          : launch2n<MODE, 2>(ctx, t, tb, a, b);
        if (rc != DAMPR_OK) return rc;
        a = b;
    }
    return DAMPR_OK;
}

}  // namespace

int launch_text_count_v2(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 lo, u64 hi, int mode) {
    g_text_cr_is_data = (mode & DAMPR_TOK_FLAG_CR_DATA) != 0;
    mode &= ~DAMPR_TOK_FLAG_CR_DATA;
    switch (mode) {
        case DAMPR_TOK_WS: return launch2<DAMPR_TOK_WS>(ctx, t, tb, lo, hi);
        case DAMPR_TOK_NONWORD_LOWER_SET: return launch2<DAMPR_TOK_NONWORD_LOWER_SET>(ctx, t, tb, lo, hi);
        case DAMPR_TOK_NONWORD_LOWER: return launch2<DAMPR_TOK_NONWORD_LOWER>(ctx, t, tb, lo, hi);
    }
    ctx->err = "unknown tokeniser mode";
    return DAMPR_ERR_ARG;
}

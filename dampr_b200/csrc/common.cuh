// common.cuh — shared declarations for libdampr_b200.so (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/dampr_b200.h"

typedef unsigned long long u64;
typedef uint32_t u32;
typedef uint16_t u16;
typedef uint8_t u8;

#define DAMPR_NUM_SMS_DEFAULT 132

struct TimedKernel {
    int id;
    cudaEvent_t beg, end;
};

struct PoolBlock {
    void *p;
    size_t bytes;
    cudaEvent_t ev_compute, ev_copy;  // work that may still touch the block when it was released
};

struct dampr_ctx {
    // device-memory pool: cudaMalloc / cudaFree take the driver's global lock (and cudaFree
    // synchronises the device); steady-state calls recycle blocks instead
    std::vector<PoolBlock> pool_free_list;
    std::unordered_map<void *, size_t> pool_live;
    size_t pool_cached_bytes = 0;
    int device;
    int num_sms;
    cudaStream_t stream;  // compute
    cudaStream_t copy;    // H2D / D2H
    std::string err;
    std::vector<TimedKernel> timings;
    std::vector<cudaEvent_t> event_pool;
    u64 launches;
    bool timing_enabled;
    // small device scratch for scalar results
    u64 *d_scratch;       // 4096 u64
    u64 *h_scratch;       // pinned mirror
    // last upload events (textbuf/kv uploads on `copy` that `stream` must wait for)
    cudaEvent_t upload_done;
    bool upload_pending;
    // pinned staging ring for transfers from / to pageable host memory (see staged_h2d in ctx.cu)
    static constexpr int STAGE_SLOTS = 4;
    static constexpr size_t STAGE_BYTES = 32u << 20;
    void *stage_slot[STAGE_SLOTS] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t stage_ev[STAGE_SLOTS] = {nullptr, nullptr, nullptr, nullptr};
    unsigned stage_next = 0;   // ring position of the uploads, carried over from call to call
    std::mutex stage_mu, dstage_mu;   // one staged transfer per ring at a time (the spill path uploads from a second host thread)
    void *dstage_slot[STAGE_SLOTS] = {nullptr, nullptr, nullptr, nullptr};   // the downloads' own ring
    cudaEvent_t dstage_ev[STAGE_SLOTS] = {nullptr, nullptr, nullptr, nullptr};

    // page-locked scratch (descriptor uploads / small downloads that must not synchronise the stream)
    void *h_pin[2] = {nullptr, nullptr};
    size_t h_pin_bytes[2] = {0, 0};
    cudaEvent_t h_pin_ev[2] = {nullptr, nullptr};  // last transfer that used the slot
    bool h_pin_busy[2] = {false, false};
    // two alternating device staging blocks of dampr_kv_upload_columns (a block taken from the pool would make
    // every call wait for the previous call's interleave kernel: no overlap of host copies and DMA)
    void *up_tmp[2] = {nullptr, nullptr};
    size_t up_tmp_bytes[2] = {0, 0};
    cudaEvent_t up_tmp_ev[2] = {nullptr, nullptr};
    int up_tmp_next = 0;
};

// Host <-> device copies that stay at PCIe speed for pageable host memory: the bytes go through the
// context's page-locked ring, moved on the host side by several threads, instead of through the driver's
// single-threaded staging copy.  Page-locked (cudaHostAlloc / dampr_host_alloc) memory is copied directly.
// staged_h2d returns when `src` may be reused (pageable) or like cudaMemcpyAsync (page-locked);
// staged_d2h returns when `dst` holds the data.
int staged_h2d(dampr_ctx *ctx, void *dst, const void *src, size_t bytes, cudaStream_t st);
int staged_d2h(dampr_ctx *ctx, void *dst, const void *src, size_t bytes, cudaStream_t st);
int staged_h2d_columns(dampr_ctx *ctx, void *dst_records, const u64 *keys, const u64 *vals, size_t count, cudaStream_t st);
bool host_is_pinned(const void *p);
extern int g_host_threads_cap;
extern int g_file_cufile, g_cufile_threads;

struct dampr_textbuf {
    u8 *alloc;      // device allocation
    u8 *text;       // alloc + TEXT_LEAD
    u64 capacity;   // bytes of text
    u64 alloc_bytes;
    u64 n;          // declared length
    u64 uploaded_hi;  // highest uploaded byte (informational)
};

struct dampr_table {
    u64 *keys;    // 0 = empty
    u64 *counts;
    u64 *reps;    // offset<<20 | len, min over occurrences (hashed tokens only); ~0 = none
    u64 *stats;   // device, 8 x u64
    u64 *fb;      // device: lines handed back to the host, (offset << 16) | length (count in stats[7])
    u32 fb_cap;
    u32 cap_log2;
    u64 cap;
};

struct dampr_kv {
    ulonglong2 *rec;   // current contents
    ulonglong2 *alt;   // ping-pong buffer (lazily allocated)
    u64 capacity;
    u64 n;
};

// page-locked scratch slot `which` of at least `bytes` (waits for the last transfer that used it);
// host_pin_used marks the transfers enqueued so far as users of the slot
void *host_pin(dampr_ctx *ctx, int which, size_t bytes);
void host_pin_used(dampr_ctx *ctx, int which);
// kv.cu internals shared with merge.cu
int kv_sort_device_range(dampr_ctx *ctx, ulonglong2 *cur, ulonglong2 *alt, u64 n, int xf);

// tuning switches (dampr_set_option)
extern int g_text_ctas;     // resident CTAs per SM of the v2 tokenise kernel: 2 (double-buffered) or 3
extern int g_text_kernel;   // 2 = warp-autonomous kernel (text2.cu), 1 = first-generation kernel (text.cu)
int launch_text_count_v2(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 lo, u64 hi, int mode);

#define TEXT_LEAD 64
#define TEXT_TAIL_PAD (64 * 1024)

static inline int set_err(dampr_ctx *ctx, int code, const char *fmt, const char *detail) {
    if (ctx) {
        char buf[512];
        snprintf(buf, sizeof buf, fmt, detail);
        ctx->err = buf;
    }
    return code;
}

#define CUDA_TRY(ctx, expr)                                                            \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess) {                                                       \
            char _b[512];                                                              \
            snprintf(_b, sizeof _b, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                     __FILE__, __LINE__);                                              \
            if (ctx) (ctx)->err = _b;                                                  \
            return (_e == cudaErrorMemoryAllocation) ? DAMPR_ERR_NOMEM : DAMPR_ERR_CUDA; \
        }                                                                              \
    } while (0)

#define ARG_CHECK(ctx, cond, msg)                               \
    do {                                                        \
        if (!(cond)) {                                          \
            if (ctx) (ctx)->err = std::string("bad argument: ") + msg; \
            return DAMPR_ERR_ARG;                               \
        }                                                       \
    } while (0)

void *pool_alloc(dampr_ctx *ctx, size_t bytes);  // nullptr on failure
void pool_free(dampr_ctx *ctx, void *p);
void pool_trim(dampr_ctx *ctx, size_t keep_bytes);

// scratch device buffer from the pool of the context the current API call runs on
extern thread_local dampr_ctx *tl_ctx;
struct CtxScope {
    dampr_ctx *prev;
    explicit CtxScope(dampr_ctx *c) : prev(tl_ctx) { tl_ctx = c; }
    ~CtxScope() { tl_ctx = prev; }
};
struct DevBuf {
    void *p = nullptr;
    dampr_ctx *owner = nullptr;
    ~DevBuf() {
        if (p) {
            if (owner) pool_free(owner, p);
            else cudaFree(p);
        }
    }
    cudaError_t alloc(size_t bytes) {
        owner = tl_ctx;
        if (owner) {
            p = pool_alloc(owner, bytes ? bytes : 16);
            return p ? cudaSuccess : cudaErrorMemoryAllocation;
        }
        return cudaMalloc(&p, bytes ? bytes : 16);
    }
};

// ---- kernel timing helpers (CUDA events on the launching stream) ----------------------
struct ScopedTimer {
    dampr_ctx *ctx;
    int idx;
    ScopedTimer(dampr_ctx *c, int id) : ctx(c), idx(-1) {
        c->launches++;
        if (!c->timing_enabled) return;
        TimedKernel tk;
        tk.id = id;
        if (cudaEventCreate(&tk.beg) != cudaSuccess) return;
        if (cudaEventCreate(&tk.end) != cudaSuccess) {
            cudaEventDestroy(tk.beg);
            return;
        }
        cudaEventRecord(tk.beg, c->stream);
        c->timings.push_back(tk);
        idx = (int)c->timings.size() - 1;
    }
    ~ScopedTimer() {
        if (idx >= 0) cudaEventRecord(ctx->timings[idx].end, ctx->stream);
    }
};

// make the compute stream wait for pending uploads issued on the copy stream
static inline void wait_uploads(dampr_ctx *ctx) {
    if (ctx->upload_pending) {
        cudaStreamWaitEvent(ctx->stream, ctx->upload_done, 0);
        ctx->upload_pending = false;
    }
}

// ---- device helpers ----------------------------------------------------------------------
__host__ __device__ __forceinline__ u64 mix64(u64 x) {
    // bijective finaliser (splitmix64 / murmur3 fmix style)
    x ^= x >> 30;
    x *= 0xBF58476D1CE4E5B9ULL;
    x ^= x >> 27;
    x *= 0x94D049BB133111EBULL;
    x ^= x >> 31;
    return x;
}

__host__ __device__ __forceinline__ u64 key_xform(u64 k, int xf) {
    switch (xf) {
        case DAMPR_KEY_MIX: return mix64(k);
        case DAMPR_KEY_I64: return k ^ 0x8000000000000000ULL;
        case DAMPR_KEY_F64: {
            u64 m = (u64)(-(long long)(k >> 63)) | 0x8000000000000000ULL;
            return k ^ m;
        }
        default: return k;
    }
}

// inverse of key_xform (every transform is a bijection on u64)
__host__ __device__ __forceinline__ u64 key_unxform(u64 t, int xf) {
    switch (xf) {
        case DAMPR_KEY_MIX: {
            t ^= (t >> 31) ^ (t >> 62);
            t *= 0x319642B2D24D8EC3ULL;  // inverse of 0x94D049BB133111EB mod 2^64
            t ^= (t >> 27) ^ (t >> 54);
            t *= 0x96DE1B173F119089ULL;  // inverse of 0xBF58476D1CE4E5B9 mod 2^64
            t ^= (t >> 30) ^ (t >> 60);
            return t;
        }
        case DAMPR_KEY_I64: return t ^ 0x8000000000000000ULL;
        case DAMPR_KEY_F64: return t ^ ((t >> 63) ? 0x8000000000000000ULL : ~0ULL);
        default: return t;
    }
}

#ifdef __CUDACC__
__device__ __forceinline__ u32 smem_u32(const void *p) {
    return (u32)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(u64 *bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64 *bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity) {
    u32 done = 0;
    u32 addr = smem_u32(bar);
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    }
}
// TMA 1-D bulk copy global -> shared (UBLKCP); bytes and both addresses multiples of 16
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, u32 bytes, u64 *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// TMA 1-D bulk copy shared -> global
__device__ __forceinline__ void tma_store_1d(void *gdst, const void *smem_src, u32 bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
                 "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_all() {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }
#endif

// Shared device/host helpers for libalq (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/alq.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libalq is written for sm_90a (H100) only"
#endif

constexpr int ALQ_MAX_WORLD = 8;

struct AlqComm {            // peer-memory group (alq_comm.cu)
    int world = 1, rank = 0;
    char* window = nullptr;           // this rank's window (peers write into it)
    char* peer[ALQ_MAX_WORLD] = {};   // mapped windows, peer[rank] == window
    size_t bytes = 0;
    unsigned long long epoch = 0;     // bumped per collective call: flags are epoch-tagged, never reset
    bool connected = false;
    // tail of the window reserved for the top-B exchange (alq_topb_exchange): 2 parities x world lists + flags
    static constexpr size_t kTopbWords = 16384;
    size_t topb_region_bytes() const { return 2 * (static_cast<size_t>(world) * kTopbWords * 8 + 1024); }
    // ... and, in front of it, the regions of the fused multi-GPU tail (alq_uncertainty_tail_sharded): 2 parities x
    // {histogram words, per-CTA counts, candidate words}
    static constexpr size_t kTailRegionBytes = 6u << 20;
    size_t tail_region_off() const { return bytes - topb_region_bytes() - kTailRegionBytes; }
    size_t greedy_bytes() const { return bytes > topb_region_bytes() + kTailRegionBytes ? bytes - topb_region_bytes() - kTailRegionBytes : 0; }
};

// system-scope flag helpers shared by the multi-GPU kernels
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// bounded spin: a dead peer must not hang the GPU (sets a sticky status instead); callers must stop consuming
// the window when it returns false.  timeout_cycles comes from the context option "spin_timeout_ms".
__device__ __forceinline__ bool wait_flag(const unsigned long long* p, unsigned long long want, int* status,
                                          long long timeout_cycles) {
    const long long t0 = clock64();
    while (ld_acquire_sys(p) != want) {
        if (clock64() - t0 > timeout_cycles) {
            if (status) { *reinterpret_cast<volatile int*>(status) = ALQ_ERR_STATE; __threadfence_system(); }   // may be a mapped host word
            return false;
        }
        __nanosleep(64);
    }
    return true;
}

struct alq_ctx {
    int device = 0;
    int sm_count = 132;
    int clock_khz = 1900000;              // SM clock (cached: the attribute query costs about a millisecond)
    size_t smem_optin = 0;
    cudaStream_t side_stream = nullptr;   // H2D pipelining for the *_host entry points
    cudaStream_t side_stream2 = nullptr;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    int* xchg_status_host = nullptr;      // pinned + mapped: sticky status of the asynchronous peer-window exchanges
    int* xchg_status_dev = nullptr;       // its device alias
    // grow-only scratch arenas (device) and pinned host staging
    void* scratch = nullptr;
    size_t scratch_bytes = 0;
    void* arena2 = nullptr;               // buffers of the *_host entry points
    size_t arena2_bytes = 0;
    void* pinned = nullptr;
    size_t pinned_bytes = 0;
    int64_t launches = 0;
    unsigned int* tile_counters = nullptr;   // ring of per-launch tile counters (dynamic scheduling of K1/K2)
    int tile_counter_next = 0;
    unsigned int* sel_ring = nullptr;        // ring of zeroed per-launch scratch of the fused score+select kernel
    int sel_ring_next = 0;
    unsigned int* sel_last_ctr = nullptr;    // counters / stamps of the last fused launch (alq_uncertainty_tail_timing)
    AlqComm comm;
    int k3_impl = 0;          // 0 auto, 1 fp32 SIMT, 2 wgmma 3xTF32
    int select_impl = 0;      // 0 auto, 1 multi-kernel radix select, 2 cluster-resident single launch
    int greedy_variant = 0;   // 0 auto, 1 direct loads, 2 bulk-copy pipeline, 3 persistent cooperative loop
    int l2_resident_mb = 24;  // persistent selection loop: MB of streamed rows kept in L2 across steps (evict_last hints); 0 = off.
                              // About half of the 50 MB L2: the rest serves the streamed rows and the agreement words
    int d2_fast_path = 1;     // D^2 draw of the persistent loop: certified per-CTA-mass path first (0: exact tree machinery only)
    int tail_buckets = 1;     // fused uncertainty tail on one GPU: route candidates to per-CTA score buckets (0: every CTA ranks
                              // its candidates against the whole list -- the general route, also the fallback for tie groups)
    int spin_timeout_ms = 20000;   // bounded spins on peer flags (a dead peer must not hang the GPU)
    int base_impl = 0;        // 0 auto, 1 sequential class loop, 2 parallel candidate lists + in-order resolve
    int balancing_loop = 0;   // 0 auto, 1 per-step path (K11 and K12 decline), 2 K11 (error beyond its limits), 3 K12 (the same)
    std::string err;
    // the bound of every spin on a peer or a CTA of the grid, in SM clock cycles
    long long spin_timeout_cycles() const { return static_cast<long long>(spin_timeout_ms) * clock_khz; }
};

#define ALQ_FAIL(ctx, code, ...)                                   \
    do {                                                           \
        char _b[512];                                              \
        snprintf(_b, sizeof(_b), __VA_ARGS__);                     \
        (ctx)->err = _b;                                           \
        return (code);                                             \
    } while (0)

#define ALQ_CUDA(ctx, call)                                                              \
    do {                                                                                 \
        cudaError_t _e = (call);                                                         \
        if (_e != cudaSuccess) {                                                         \
            ALQ_FAIL(ctx, ALQ_ERR_CUDA, "%s failed: %s (%s:%d)", #call,                  \
                     cudaGetErrorString(_e), __FILE__, __LINE__);                        \
        }                                                                                \
    } while (0)

#define ALQ_LAUNCH_CHECK(ctx)                                                            \
    do {                                                                                 \
        (ctx)->launches++;                                                               \
        cudaError_t _e = cudaGetLastError();                                             \
        if (_e != cudaSuccess) {                                                         \
            ALQ_FAIL(ctx, ALQ_ERR_CUDA, "kernel launch failed: %s (%s:%d)",              \
                     cudaGetErrorString(_e), __FILE__, __LINE__);                        \
        }                                                                                \
    } while (0)

// Grid-synchronising kernels (see alq_score.cu) must never share the device with another one of this process: every
// such launch is bracketed by these two (one event per device, process-wide).  Call them through alq_gridsync_launch.
void alq_gridsync_begin(alq_ctx* ctx, cudaStream_t st);
void alq_gridsync_end(alq_ctx* ctx, cudaStream_t st);
// Runs `launch` (enqueues one grid-synchronising kernel on `st` and returns its launch error) between
// alq_gridsync_begin and alq_gridsync_end, counts the launch and returns the launch error.
template <typename Launch>
cudaError_t alq_gridsync_launch(alq_ctx* ctx, cudaStream_t st, Launch&& launch) {
    alq_gridsync_begin(ctx, st);
    const cudaError_t e = launch();
    alq_gridsync_end(ctx, st);
    ctx->launches++;
    return e;
}

// The start-of-call handshake of a collective call over the group's windows (alq_comm.cu): once this rank has cleared
// its window for the call (earlier on `st`), store `tag` into ready[rank] of every rank's window, the u64
// ready[ALQ_MAX_WORLD] at its head.  Peers write into this window only after they have seen it.
int alq_comm_ready(alq_ctx* ctx, unsigned long long tag, cudaStream_t st);
// K10's tile histogram + per-class scan (alq_classes.cu): counts[k] = rows with avail != 0 and labels == k; an available
// row with a label outside [0, c) is not counted and, with `bad` given, the smallest such row is atomicMin'ed there.
// `tab` holds alq_class_table_entries(n, c) int32 entries of scratch.
int alq_class_table_pass(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int n, int c, int32_t* tab,
                         unsigned int* bad, int32_t* counts, cudaStream_t st);
size_t alq_class_table_entries(int64_t n, int c);
int alq_pinned_reserve(alq_ctx* ctx, size_t bytes);

// Device arenas, grow-only: each holds at least `bytes` afterwards.  Called through alq_scratch_carve alone.
int alq_scratch_reserve(alq_ctx* ctx, size_t bytes);
int alq_arena2_reserve(alq_ctx* ctx, size_t bytes);
// The bytes alq_scratch_reserve allocates when a call needs `bytes` and the arena has to grow.
size_t alq_scratch_alloc_bytes(size_t bytes);

// Hands out an arena's buffers in order, each on a 256-byte boundary.  With a null base it only measures: take()
// advances the offset alone and returns nullptr.
struct ScratchCursor {
    char* base;
    size_t off = 0;
    explicit ScratchCursor(void* b) : base(static_cast<char*>(b)) {}
    template <typename T>
    T* take(size_t count) {
        off = (off + 255) & ~size_t(255);
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * sizeof(T);
        return p;
    }
};

// The bytes that `layout(ScratchCursor&)`, a call's takes, spans.
template <typename Layout>
size_t alq_layout_bytes(Layout&& layout) {
    ScratchCursor m(nullptr);
    layout(m);
    return m.off;
}

// One call's device scratch, sized and carved by the same takes: runs `layout` once measuring, reserves exactly what it
// spans and runs it again on the arena, where its takes store the call's pointers.  A reservation may move the arena, so
// pointers from an earlier carve die with it.  ctx->scratch serves every entry point; an entry point that holds
// ctx->scratch buffers calls no other entry point that takes scratch.  ctx->arena2 is for the two that must hold buffers
// across such calls: alq_uncertainty_query_host and BASE's select (alq_mase.cu).
template <typename Layout>
int alq_scratch_carve(alq_ctx* ctx, Layout&& layout, bool arena2 = false) {
    const size_t bytes = alq_layout_bytes(layout);
    const int rc = arena2 ? alq_arena2_reserve(ctx, bytes) : alq_scratch_reserve(ctx, bytes);
    if (rc != ALQ_OK) return rc;
    ScratchCursor cur(arena2 ? ctx->arena2 : ctx->scratch);
    layout(cur);
    return ALQ_OK;
}

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
#define ALQ_NEG_INF (__int_as_float(0xff800000))
#define ALQ_POS_INF (__int_as_float(0x7f800000))

// Monotone float -> uint32 map: a < b  <=>  ord(a) < ord(b)   (-0.0 sorts just below +0.0).
__host__ __device__ __forceinline__ uint32_t alq_ord(float f) {
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float alq_unord(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

// arg-max key: larger value wins, equal values -> lower row wins.
__device__ __forceinline__ unsigned long long alq_maxkey(float v, uint32_t row) {
    return (static_cast<unsigned long long>(alq_ord(v)) << 32) | (0xffffffffu - row);
}
__host__ __device__ __forceinline__ uint32_t alq_maxkey_row(unsigned long long k) {
    return 0xffffffffu - static_cast<uint32_t>(k & 0xffffffffu);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

// streaming 128-bit load that does not pollute L1 (data is read exactly once per launch)
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

// float atomic min/max that is correct across signs (IEEE ordering trick).
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
    if (v >= 0.f) atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// ---- mbarrier + bulk-copy (TMA) primitives shared by the streaming pipelines -------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// before the barrier's words are reused as plain shared memory (PTX leaves any other access undefined)
__device__ __forceinline__ void mbar_inval(uint64_t* bar) {
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}


// bulk copy with an L2 eviction policy (createpolicy): rows that should stay resident in the 50 MB L2 across the steps of
// a selection loop are fetched evict_last, the rest evict_first so that the stream does not push them out
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void bulk_g2s_hint(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}

// ---- thread-block cluster helpers -------------------------------------------------------------------------
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// ---- block-wide bitonic sort of `n` (power of two, >= 64, n/2 <= blockDim.x threads used... see below) -------
// 64-bit keys ascending, data in shared memory `sk` on entry and exit.  Thread t owns elements (2t, 2t+1):
// every compare-exchange at distance j <= 32 happens in registers / warp shuffles (partner element i ^ j lives in
// lane (t ^ j/2) of the same warp), so only the distances >= 64 touch shared memory and need a block barrier:
// for n = 2048 that is 15 of the 66 steps.  All threads of the block must call it; threads with 2t >= n idle.
__device__ __forceinline__ void alq_cx_keep(unsigned long long& mine, unsigned long long other, bool keep_min) {
    const bool take = keep_min ? (other < mine) : (other > mine);
    if (take) mine = other;
}
__device__ __forceinline__ void alq_bitonic_reg_phase(unsigned long long& e0, unsigned long long& e1, int t, int k, int j_start) {
    // distances j_start, j_start/2, ..., 2 through shuffles, then distance 1 inside the thread
    const bool up = ((2 * t) & k) == 0;
    for (int j = j_start; j >= 2; j >>= 1) {
        const bool lower = ((2 * t) & j) == 0;
        const unsigned long long o0 = __shfl_xor_sync(0xffffffffu, e0, j >> 1);
        const unsigned long long o1 = __shfl_xor_sync(0xffffffffu, e1, j >> 1);
        alq_cx_keep(e0, o0, lower == up);
        alq_cx_keep(e1, o1, lower == up);
    }
    if ((e0 > e1) == up) { const unsigned long long x = e0; e0 = e1; e1 = x; }
}
__device__ __forceinline__ void alq_bitonic_sort_smem(unsigned long long* sk, int n) {
    const int t = threadIdx.x;
    const bool mine = 2 * t < n;                 // warps are either fully in or fully out (n >= 64)
    unsigned long long e0 = 0, e1 = 0;
    if (mine) { e0 = sk[2 * t]; e1 = sk[2 * t + 1]; }
    // stages k = 2 .. 64: every distance stays inside a warp
    if (mine) {
        for (int k = 2; k <= 64 && k <= n; k <<= 1) alq_bitonic_reg_phase(e0, e1, t, k, k >> 1);
        sk[2 * t] = e0; sk[2 * t + 1] = e1;
    }
    __syncthreads();
    for (int k = 128; k <= n; k <<= 1) {
        for (int j = k >> 1; j >= 64; j >>= 1) {        // block-wide distances: pair (l, l | j) per thread
            if (mine) {
                const int l = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                const unsigned long long x = sk[l], y = sk[l | j];
                if ((x > y) == ((l & k) == 0)) { sk[l] = y; sk[l | j] = x; }
            }
            __syncthreads();
        }
        if (mine) {
            e0 = sk[2 * t]; e1 = sk[2 * t + 1];
            alq_bitonic_reg_phase(e0, e1, t, k, 32);
            sk[2 * t] = e0; sk[2 * t + 1] = e1;
        }
        __syncthreads();
    }
}

// ---- K7's pair arithmetic: scipy's euclidean on fp32 rows, the exact d2 of every kernel that certifies distances ----
// (K7, K13's recheck, K15's recheck, K17, K18's recheck and fallback; the NumPy statement is probcover_oracle.exact_d2)
// one step: the fp32 entries widened to fp64 (exact), d = a - b, s + d * d, each operation rounded on its own (no FMA)
__device__ __forceinline__ double d2_step(double s, double a, double b) {
    const double df = __dsub_rn(a, b);
    return __dadd_rn(s, __dmul_rn(df, df));
}
// the whole chain over rows a and b, k ascending (16-byte aligned, d % 4 == 0)
__device__ __forceinline__ double exact_d2(const float* __restrict__ a, const float* __restrict__ b, int d) {
    const float4* a4 = reinterpret_cast<const float4*>(a);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    double s = 0.0;
    for (int k = 0; k < d / 4; ++k) {
        const float4 u = __ldg(a4 + k), v = __ldg(b4 + k);
        s = d2_step(s, u.x, v.x);
        s = d2_step(s, u.y, v.y);
        s = d2_step(s, u.z, v.z);
        s = d2_step(s, u.w, v.w);
    }
    return s;
}
// the ascending (d2, index) order: ties to the lower index
__device__ __forceinline__ bool pair_less(double a, int ca, double b, int cb) {
    return a < b || (a == b && ca < cb);
}

// ---- a row's log-sum-exp in fp64 (K19, K20; the NumPy statement is cal_oracle.log_softmax) ----
// m + log(sum_c exp(z_c - m)), m = max_c z_c, c ascending; NaN when a logit is NaN
__device__ __forceinline__ double row_lse(const float* __restrict__ zr, int C) {
    float mx = -INFINITY;
    bool nan = false;
    for (int c = 0; c < C; ++c) {
        const float v = __ldg(zr + c);
        nan |= v != v;
        mx = v > mx ? v : mx;
    }
    const double m = nan ? static_cast<double>(NAN) : static_cast<double>(mx);
    double s = 0.0;
    for (int c = 0; c < C; ++c) s = __dadd_rn(s, exp(__dsub_rn(static_cast<double>(__ldg(zr + c)), m)));
    return __dadd_rn(m, log(s));
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

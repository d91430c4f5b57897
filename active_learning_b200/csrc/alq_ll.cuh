// The LL-word protocol of the persistent grid-synchronising kernels (the selection loop in alq_greedy_persist.cu, K11 and
// K12 in alq_balancing*.cu, K14 in alq_probcover.cu, the fused tail in alq_score.cu): the word store / load / wait /
// gather, the CTA row segments, the min-agreement over one key word per CTA and the start-of-call ready wait.
#pragma once

#include "alq_common.cuh"

// The rows of a call and who streams them.  Rank r owns rows [off[r], off[r + 1]) and runs `grid` CTAs on them; global
// segment g = r * grid + b, CTA b of rank r, starts at off[r] + seg_lo(off[r + 1] - off[r], grid, b).  A single GPU is
// world 1, rank 0, off = {0, n}: segment b starts at seg_lo(n, grid, b).  Every array stays global and replicated, so
// every rank derives the same world * grid segments.
struct SegShard {
    int world, rank, grid;
    int off[ALQ_MAX_WORLD + 1];
};

// Where the LL words of a call live.  peer[r] is rank r's window (a single GPU: peer[0] is scratch of this call); every
// window has the same layout: u64 ready[ALQ_MAX_WORLD] (sharded calls), the key words [2 parities][world * grid] at
// `keyw` and the loop's own words at `pickw` (K11 / K12: one pick word per step).  Tags carry the call's epoch (0 on a
// single GPU).
struct LLWords {
    char* peer[ALQ_MAX_WORLD];
    unsigned int keyw, pickw;
    unsigned int tag_base;               // 0x80000000 | (epoch & 0x7f) << 24: never 0, a zeroed word is invalid
    unsigned long long ready_tag;        // sharded: epoch << 32, stored into every peer's ready[rank]; 0: no handshake
};

namespace {

constexpr int kSegRowsMax = 65535;               // the key word carries a 16-bit row offset (0xffff: empty segment)
constexpr unsigned int kEmptyOff = 0xffffu;

__host__ __device__ __forceinline__ int seg_lo(int n, int grid, int b) {
    return static_cast<int>(static_cast<long long>(n) * b / grid);
}

__host__ __device__ __forceinline__ int gseg_lo(const SegShard& S, int g) {
    const int r = g / S.grid;
    if (r >= S.world) return S.off[S.world];
    return S.off[r] + seg_lo(S.off[r + 1] - S.off[r], S.grid, g - r * S.grid);
}

__device__ __forceinline__ unsigned int ll_key_tag(const LLWords& W, unsigned int round) {
    return 0x8000u | ((W.tag_base >> 12) & 0x7000u) | (round & 0xfffu);
}

// 8 bytes = {32-bit tag, 32-bit payload} written with one plain store (single-copy atomic, so no fence and no separate
// flag) and polled at the destination until the tag matches.  `Args` is the kernel's argument block: it provides
// `int* status` (sticky failure word) and `long long timeout_cycles`.
__device__ __forceinline__ void ll_store(void* p, unsigned int tag, unsigned int payload) {
    const unsigned long long v = (static_cast<unsigned long long>(tag) << 32) | payload;
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void ll_store_raw(void* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ll_load(const void* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// Bounded spin; after a failure anywhere (sticky status) every wait returns at once, so the loop drains
// to its end in bounded time instead of hanging the GPU on a dead peer.
template <typename Args>
__device__ __forceinline__ bool ll_give_up(int spin, long long t0, const Args& A) {
    if ((spin & 63) != 63) return false;
    if (*reinterpret_cast<volatile int*>(A.status) != 0) return true;
    if (clock64() - t0 > A.timeout_cycles) { atomicCAS(A.status, 0, ALQ_ERR_STATE); return true; }
    return false;
}
template <typename Args>
__device__ __forceinline__ unsigned int ll_wait(const void* p, unsigned int tag, const Args& A) {
    unsigned long long v = ll_load(p);
    if (static_cast<unsigned int>(v >> 32) == tag) return static_cast<unsigned int>(v);
    const long long t0 = clock64();
    for (int spin = 0;; ++spin) {
        v = ll_load(p);
        if (static_cast<unsigned int>(v >> 32) == tag || ll_give_up(spin, t0, A)) break;
    }
    return static_cast<unsigned int>(v);
}
// Collect `nwords` LL words at `base` (stride `stride` bytes) whose top (64 - shift) bits equal `tag`.
// Polling is what floods L2 when 75 000 threads spin on words that are not there yet (measured: it slows the CTAs
// that still stream and every store behind it), so it is rationed: only the first kPollers threads (`ct`) poll;
// (1) one warp spins on 32 sentinel words spread over the range -- one load per lane per round -- and only when
// those have arrived (2) every poller loads its up-to-kBatch words as one batch (one L2 round trip), re-loading just
// the few still missing.  Called by every thread with ct < kPollers (named barrier 2); the caller follows it with a
// barrier of its own.
constexpr int kPollers = 320;
constexpr int kBatch = 8;
template <typename Args, typename Sink>
__device__ __forceinline__ void ll_gather(const char* base, int nwords, int stride, unsigned long long tag, int shift,
                                          const Args& A, int ct, Sink&& sink) {
    if (ct >= kPollers) return;
    if (ct < 32 && nwords > 0) {
        const char* sp = base + static_cast<size_t>(static_cast<long long>(ct) * nwords / 32) * stride;
        const long long t0 = clock64();
        for (int spin = 0; (ll_load(sp) >> shift) != tag; ++spin) {
            if (ll_give_up(spin, t0, A)) break;
            __nanosleep(40);
        }
    }
    asm volatile("bar.sync 2, %0;" ::"n"(kPollers) : "memory");
    for (int chunk = 0; chunk < nwords; chunk += kPollers * kBatch) {
        unsigned int pend = 0;
#pragma unroll
        for (int q = 0; q < kBatch; ++q)
            if (chunk + ct + q * kPollers < nwords) pend |= 1u << q;
        const long long t0 = clock64();
        for (int spin = 0; pend; ++spin) {
            unsigned long long w[kBatch];
#pragma unroll
            for (int q = 0; q < kBatch; ++q)
                if (pend & (1u << q)) w[q] = ll_load(base + static_cast<size_t>(chunk + ct + q * kPollers) * stride);
#pragma unroll
            for (int q = 0; q < kBatch; ++q)
                if ((pend & (1u << q)) && (w[q] >> shift) == tag) {
                    sink(chunk + ct + q * kPollers, w[q]);
                    pend &= ~(1u << q);
                }
            if (pend && ll_give_up(spin, t0, A)) break;
        }
    }
}

// The start-of-call handshake of a sharded call, the other half of alq_comm_ready: thread i < world of this rank waits
// until ready[i] (u64 ready[ALQ_MAX_WORLD] at the head of this rank's window) holds the call's tag, i.e. until rank i has
// cleared its window for this call.  No CTA stores into a peer's window before that; the caller follows with a barrier.
template <typename Args>
__device__ __forceinline__ void ll_ready_wait(const char* window, int i, const unsigned long long& tag, const Args& A) {
    const unsigned long long* rw = reinterpret_cast<const unsigned long long*>(window) + i;
    for (const long long t0 = clock64(); ld_acquire_sys(rw) != tag;) {
        if (clock64() - t0 > A.timeout_cycles) { atomicCAS(A.status, 0, ALQ_ERR_STATE); break; }
        __nanosleep(200);
    }
}

// One agreement on the grid's smallest key (hi32 << 32 | row, ~0: none).  s_key[0 .. kWarps) holds each warp's smallest
// key and a barrier has passed; `A` provides the segments S (SegShard) and the words W (LLWords).  The CTA's minimum goes
// as one word {tag16, row offset16, hi32} into slot rank * grid + b of every rank's window; every CTA gathers all
// world * grid words and returns the smallest key's row (-1: none, or a failed wait) to every thread.
template <int kWarps, typename Args>
__device__ __forceinline__ int ll_agree_min(const Args& A, unsigned long long* s_key, int* s_pick, unsigned int round,
                                         int row_lo, int tid) {
    const SegShard& S = A.S;
    const int nseg = S.world * S.grid, lane = tid & 31, warp = tid >> 5;
    const unsigned int tag16 = ll_key_tag(A.W, round);
    const size_t keyw = A.W.keyw + static_cast<size_t>(round & 1u) * nseg * 8;
    if (tid < S.world) {
        unsigned long long m = s_key[0];
        for (int w = 1; w < kWarps; ++w) m = s_key[w] < m ? s_key[w] : m;
        const unsigned long long off = m == ~0ull ? kEmptyOff : static_cast<unsigned long long>(static_cast<uint32_t>(m) - row_lo);
        ll_store_raw(A.W.peer[tid] + keyw + static_cast<size_t>(S.rank * S.grid + blockIdx.x) * 8,
                     (static_cast<unsigned long long>(tag16) << 48) | (off << 32) | (m >> 32));
    }
    unsigned long long mine = ~0ull;
    ll_gather(A.W.peer[S.rank] + keyw, nseg, 8, tag16, 48, A, tid, [&](int i, unsigned long long w) {
        const unsigned int off = static_cast<unsigned int>(w >> 32) & 0xffffu;
        if (off == kEmptyOff) return;
        const unsigned long long key = ((w & 0xffffffffull) << 32) | static_cast<uint32_t>(gseg_lo(S, i) + static_cast<int>(off));
        mine = key < mine ? key : mine;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, mine, o);
        mine = w < mine ? w : mine;
    }
    __syncthreads();                                              // s_key is reused
    if (lane == 0) s_key[warp] = mine;
    __syncthreads();
    if (tid == 0) {
        unsigned long long m = s_key[0];
        for (int w = 1; w < kWarps; ++w) m = s_key[w] < m ? s_key[w] : m;
        *s_pick = m == ~0ull ? -1 : static_cast<int>(static_cast<uint32_t>(m));
    }
    __syncthreads();
    return *s_pick;
}
// The same, not inlined: K12's loop sits at the 128-register cap of its launch bounds, and the exchange inlined into it
// spills.  K14 inlines it: out of line, its 10 000 steps took about 1.5 ms (2 %) longer on an H100 80GB HBM3 at 700 W.
template <int kWarps, typename Args>
__device__ __noinline__ int ll_agree_min_call(const Args& A, unsigned long long* s_key, int* s_pick, unsigned int round,
                                              int row_lo, int tid) {
    return ll_agree_min<kWarps>(A, s_key, s_pick, round, row_lo, tid);
}

}  // namespace

// Pieces shared by the selection-loop kernels (alq_greedy.cu: one launch per step; alq_greedy_persist.cu: one
// persistent cooperative launch for the whole loop).
#pragma once
#include <math.h>
#include <stdlib.h>

#include "alq_common.cuh"

namespace {

struct BlockSeg {        // one CTA's share of the rows
    int row_lo, row_hi, part, pad;
};

__device__ __forceinline__ float dist_dense(float n_i, float n_q, float dot) {
    return (n_i + n_q) - 2.0f * dot;
}


struct PipeCfg {
    int rows_per_tile;   // R
    int stages;
    int tile_floats;     // R * (d + c)
    int consumers;       // consumer warps
};

// NumPy pairwise_sum leaf (n <= 128) evaluated by an 8-lane group, bit-exact:
//   r[j] = a[j]; r[j] += a[i+j] for i = 8,16,..; ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7)); then the
//   n % 8 tail added one by one.
__device__ __forceinline__ float leaf_sum_group(const float* a, int len, int g_lane, unsigned gmask) {
    float res;
    if (len < 8) {
        res = 0.f;
        if (g_lane == 0)
            for (int i = 0; i < len; ++i) res += fmaxf(__ldcg(a + i), 0.f);
        return res;
    }
    const int stop = len - (len & 7);
    // issue every load of this lane first (<= 16: a leaf has <= 128 entries), then add in NumPy's order
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = (8 * j + g_lane < stop) ? __ldcg(a + 8 * j + g_lane) : 0.f;
    float tail[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) tail[j] = (g_lane == 0 && stop + j < len) ? __ldcg(a + stop + j) : 0.f;
    float r = fmaxf(v[0], 0.f);                      // prob = clip(min_dist, 0) (coreset_sampler.py:84)
#pragma unroll
    for (int j = 1; j < 16; ++j)
        if (8 * j < stop) r += fmaxf(v[j], 0.f);
    r = r + __shfl_down_sync(gmask, r, 1, 8);   // lanes 0,2,4,6: r0+r1, r2+r3, ...
    r = r + __shfl_down_sync(gmask, r, 2, 8);   // lanes 0,4
    r = r + __shfl_down_sync(gmask, r, 4, 8);   // lane 0
    res = r;
    if (g_lane == 0) {
#pragma unroll
        for (int j = 0; j < 7; ++j)
            if (stop + j < len) res += fmaxf(tail[j], 0.f);
    }
    return res;
}

// prob = c / S in IEEE fp32 (what NumPy computes).  Zero numerators (every labeled / picked slot) would take
// the division's special-operand slow path: 0 / S == +0 for S > 0, so answer those without dividing.
__device__ __forceinline__ double prob64(float raw, float total32) {
    const float c = fmaxf(raw, 0.f);
    return c > 0.f ? static_cast<double>(__fdiv_rn(c, total32)) : 0.0;
}

static void build_segments(int P, const int32_t* part_off, const int32_t* budget, int target_blocks,
                    std::vector<BlockSeg>& segs) {
    int64_t total = 0;
    for (int p = 0; p < P; ++p)
        if (budget[p] > 0) total += part_off[p + 1] - part_off[p];
    for (int p = 0; p < P; ++p) {
        const int rows = part_off[p + 1] - part_off[p];
        if (rows <= 0 || budget[p] <= 0) continue;
        int nb = static_cast<int>((static_cast<int64_t>(target_blocks) * rows + total / 2) / std::max<int64_t>(total, 1));
        nb = std::max(1, std::min(nb, rows));
        for (int b = 0; b < nb; ++b) {
            BlockSeg s;
            s.row_lo = part_off[p] + static_cast<int>(static_cast<int64_t>(rows) * b / nb);
            s.row_hi = part_off[p] + static_cast<int>(static_cast<int64_t>(rows) * (b + 1) / nb);
            s.part = p;
            s.pad = 0;
            if (s.row_hi > s.row_lo) segs.push_back(s);
        }
    }
}

// NumPy's pairwise-summation tree over n entries: a run of at most 128 entries is a leaf, a longer run of m entries
// splits at m / 2 rounded down to a multiple of 8.  Every D^2 pick rests on this rule being bit-exact.  Both D^2 loops
// (and alq_pairwise_leaf_bounds) read their trees from here.
struct PairTree {
    std::vector<int> leaf_off;                       // n_leaves + 1 entries, the last one is n
    struct Node { int height, l, r; };               // children: >= 0 leaf id, < 0 internal #(-v - 1)
    std::vector<Node> internal;                      // creation (post-) order: the root is the last one
    std::vector<int> order;                          // internal nodes by height 1, 2, .., creation order within a height
    std::vector<int> level_off;                      // n_levels + 1 offsets into `order`

    explicit PairTree(int n) {
        rec(0, n);
        leaf_off.push_back(n);
        int hmax = 0;
        for (const Node& nd : internal) hmax = std::max(hmax, nd.height);
        level_off.assign(hmax + 1, 0);
        for (const Node& nd : internal) ++level_off[nd.height];          // count per height, then exclusive prefix
        for (int h = 1; h <= hmax; ++h) level_off[h] += level_off[h - 1];
        std::vector<int> at(level_off.begin(), level_off.end() - 1);
        order.resize(internal.size());
        for (size_t k = 0; k < internal.size(); ++k) order[at[internal[k].height - 1]++] = static_cast<int>(k);
    }
    int n_leaves() const { return static_cast<int>(leaf_off.size()) - 1; }
    int n_levels() const { return static_cast<int>(level_off.size()) - 1; }

private:
    std::pair<int, int> rec(int lo, int m) {         // -> (ref, height)
        if (m <= 128) {
            leaf_off.push_back(lo);
            return {static_cast<int>(leaf_off.size()) - 1, 0};
        }
        int half = m / 2;
        half -= half % 8;
        const auto L = rec(lo, half);
        const auto R = rec(lo + half, m - half);
        const int h = std::max(L.second, R.second) + 1;
        internal.push_back({h, L.first, R.first});
        return {-static_cast<int>(internal.size()), h};
    }
};


// ---- LL words (alq_greedy_persist.cu, alq_balancing.cu) -------------------------------------------------------
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

}  // namespace

// alq_greedy_persist.cu: the whole B-step loop as ONE cooperative launch (variant 3).  Returns ALQ_OK, an error, or
// kPersistNotApplicable when the problem does not fit it (the caller falls back to the per-step variants).
constexpr int kPersistNotApplicable = -1;
int alq_greedy_persist(alq_ctx* ctx, const alq_greedy_desc* D, void* stream);

// Pieces shared by the selection-loop kernels (alq_greedy.cu: one launch per step; alq_greedy_persist.cu: one
// persistent cooperative launch for the whole loop).  The LL words of the persistent loop: alq_ll.cuh.
#pragma once
#include <math.h>
#include <stdlib.h>

#include "alq_ll.cuh"

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

}  // namespace

// alq_greedy_persist.cu: the whole B-step loop as ONE cooperative launch (variant 3).  Returns ALQ_OK, an error, or
// kPersistNotApplicable when the problem does not fit it (the caller falls back to the per-step variants).
constexpr int kPersistNotApplicable = -1;
int alq_greedy_persist(alq_ctx* ctx, const alq_greedy_desc* D, void* stream);

// K15 / K16 / K17: TypiClustSampler (Hacohen, Dekel & Weinshall, "Active Learning on a Budget", ICML 2022) on the device.
//
// alq_kmeans_rows       the pool rows L2-normalised (K13's normalise, alq_rows_split.cuh) and split into TF32 hi / lo
//                       with their fp64 squared norms, once per k-means.
// K15 alq_kmeans_assign label_i = the exact fp64 argmin over the centres c of d2(xhat_i, c) = exact_d2 (K7's pair
//                       arithmetic, alq_common.cuh), ties to the lowest centre.
//   split      the centres [K, d] through the same kernel (no normalisation): hi / lo and cn = |c|^2 in fp64.
//   domain     km_domain_kernel counts the rows and centres whose squared norm is not in [0, 2] (the band's slack is
//              absolute, DESIGN section 4) and the call refuses them by name before the screen (one 4-byte copy).
//   screen     one CTA per SM, persistent over 128-row blocks; for each, every 128-centre tile on the ring of
//              alq_wgmma.cuh (warpgroup 0 runs tc::ring_produce_rows, warpgroups 1-2 tc::ring_tile).  The epilogue
//              forms d2~ = nrm2_i + cn_c - 2 g in fp64 and the band b = band_coef(d) sqrt(nrm2_i) sqrt(cn_c) + slack of
//              DESIGN section 4, and keeps per row U = min_c (d2~ + b) and the two smallest lower bounds L1 (at c1) <= L2
//              of d2~ - b.  The four lanes holding a row's columns merge their states; if L2 > U every other centre is
//              strictly farther than c1 and the label is c1, otherwise the row goes on the recheck list.  n x K is never
//              formed.
//   recheck    a warp per listed row: exact_d2 to ALL K centres, lane-strided over the centres, the (d2, centre)
//              minimum (pair_less) over the warp.
//   Returns the rows whose label changed and the rows rechecked, in one 8-byte copy.
// K16 alq_kmeans_update centre_c = fl32(S_c / m_c), S_c the fp64 sum of the member rows in ascending row order, one
//              sequential chain per column.  A stable counting sort of the rows by label (per-chunk histograms, a scan,
//              then one warp per chunk places its rows in order with __match_any_sync), then one thread per (cluster,
//              column) runs the chain.  An empty cluster keeps its centre.
// K17 alq_typicality    for groups of rows (the available, unpicked rows of the clusters one cycle of the walk visits):
//              per row the k = min(k_max, m / 2) smallest exact fp64 d2 to the OTHER rows of its group (excluded by
//              position, so a duplicate row counts with d2 = 0), their ascending fp64 sum / k = mean, typicality =
//              1 / (mean + 1e-5), and per group the argmax (lowest position on ties).  64 x 64 block-diagonal tiles of
//              d2_step; each warp keeps the sorted 32 smallest of its rows across the lanes.  m x m is never formed.
// K21 alq_kmeans_nearest per cluster c < K the row labeled c with the smallest exact fp64 d2(xhat_i, centre_c), the lowest
//              row on ties, -1 for an empty cluster.  A thread per row computes its d2 to its own centre; an fp64 d2 >= 0
//              orders as its 64-bit pattern, so one atomicMin per row finds each cluster's smallest d2 and a second one,
//              over the rows that reach it, the lowest such row (the d2 leaves no bits of a 64-bit key for the row).
#include <math.h>

#include <algorithm>
#include <vector>

#include "alq_rows_split.cuh"
#include "alq_wgmma.cuh"

namespace tk {

using tc::BK;
using tc::BM;
constexpr int K_MAX = 32768;                    // K16's histogram lives in shared memory: 128 KB at K_MAX
constexpr double NRM2_MAX = 2.0;                // the band's absolute slack is derived for squared norms in [0, 2]

// ---- K15 ---------------------------------------------------------------------------------------------------------------
struct AssignParams {
    const double* nrm2;                // [n] |xhat_i|^2
    const double* cn;                  // [K] |c|^2
    int n, K, ctiles, kblocks, rblocks;
    double coef;                       // d2 error per unit of sqrt(nrm2_i) sqrt(cn_c) (DESIGN section 4)
    double slack;                      // absolute slack of the fp64 epilogue and of the exact value's own rounding
    int* labels;
    int* list;                         // [n] the rows left to the exact recheck
    unsigned int* counts;              // [0] labels changed, [1] rows listed
};

// rows (nrm2) and centres (cn) whose squared norm lies outside [0, NRM2_MAX], NaN and infinity included, are counted in
// *bad
__global__ void __launch_bounds__(256) km_domain_kernel(const double* __restrict__ nrm2, int n, const double* __restrict__ cn,
                                                        int k, unsigned int* bad) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<long long>(n) + k) return;
    const double v = i < n ? nrm2[i] : cn[i - n];
    if (!(v >= 0.0 && v <= NRM2_MAX)) atomicAdd(bad, 1u);
}

// the two smallest lower bounds (l1 at c1, then l2) and the smallest upper bound u of a row
struct Near {
    double u, l1, l2;
    int c1;
};
__device__ __forceinline__ void near_add(Near& s, double hi, double lo, int c) {
    s.u = fmin(s.u, hi);
    if (lo < s.l1) { s.l2 = s.l1; s.l1 = lo; s.c1 = c; }
    else if (lo < s.l2) s.l2 = lo;
}
__device__ __forceinline__ void near_merge(Near& s, int o) {
    const double u = __shfl_xor_sync(0xffffffffu, s.u, o), l1 = __shfl_xor_sync(0xffffffffu, s.l1, o);
    const double l2 = __shfl_xor_sync(0xffffffffu, s.l2, o);
    const int c1 = __shfl_xor_sync(0xffffffffu, s.c1, o);
    s.u = fmin(s.u, u);
    if (l1 < s.l1 || (l1 == s.l1 && c1 < s.c1)) { s.l2 = fmin(s.l1, l2); s.l1 = l1; s.c1 = c1; }
    else s.l2 = fmin(s.l2, l1);
}

__global__ void __launch_bounds__(tc::THREADS, 1)
km_assign_kernel(const __grid_constant__ CUtensorMap map_xhi, const __grid_constant__ CUtensorMap map_xlo,
                 const __grid_constant__ CUtensorMap map_chi, const __grid_constant__ CUtensorMap map_clo,
                 const AssignParams P) {
    extern __shared__ unsigned char smem_dyn[];
    const tc::Role me = tc::ring_role();
    const tc::Ring ring = tc::ring_init(smem_dyn);

    if (me.wg == 0) {
        tc::producer_regs();
        if (threadIdx.x == 0) tc::ring_produce_rows(ring, &map_xhi, &map_xlo, &map_chi, &map_clo, P.rblocks, P.ctiles, P.kblocks);
        return;
    }
    tc::consumer_regs();
    unsigned int changed = 0;
    uint32_t it = 0;
    for (int rb = blockIdx.x; rb < P.rblocks; rb += gridDim.x) {
        const int row0 = rb * BM + me.r_in_tile, row1 = row0 + 8;
        const double n0 = row0 < P.n ? __ldg(P.nrm2 + row0) : 0.0, n1 = row1 < P.n ? __ldg(P.nrm2 + row1) : 0.0;
        const double s0 = __dsqrt_rn(n0), s1 = __dsqrt_rn(n1);
        Near a{INFINITY, INFINITY, INFINITY, 0x7fffffff}, b{INFINITY, INFINITY, INFINITY, 0x7fffffff};
        for (int ct = 0; ct < P.ctiles; ++ct) {
            float acc[64];
            tc::ring_tile(ring, it, me, acc, P.kblocks);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = ct * BM + 8 * j + me.c_in_tile + e;
                    if (c >= P.K) continue;
                    const double nc = __ldg(P.cn + c), sc = __dsqrt_rn(nc);
                    const double d0 = __dsub_rn(__dadd_rn(n0, nc), 2.0 * static_cast<double>(acc[4 * j + e]));
                    const double d1 = __dsub_rn(__dadd_rn(n1, nc), 2.0 * static_cast<double>(acc[4 * j + 2 + e]));
                    const double b0 = __dadd_rn(__dmul_rn(P.coef, __dmul_rn(s0, sc)), P.slack);
                    const double b1 = __dadd_rn(__dmul_rn(P.coef, __dmul_rn(s1, sc)), P.slack);
                    near_add(a, __dadd_rn(d0, b0), __dsub_rn(d0, b0), c);
                    near_add(b, __dadd_rn(d1, b1), __dsub_rn(d1, b1), c);
                }
            }
        }
        // the four lanes of a row hold its columns 2 (lane % 4) + {0, 1} of every 8
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            near_merge(a, o);
            near_merge(b, o);
        }
        if ((me.lane & 3) == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = h ? row1 : row0;
                const Near& s = h ? b : a;
                if (row >= P.n) continue;
                if (s.l2 > s.u) {
                    if (P.labels[row] != s.c1) { P.labels[row] = s.c1; ++changed; }
                } else {
                    P.list[atomicAdd(P.counts + 1, 1u)] = row;
                }
            }
        }
    }
    if (changed) atomicAdd(P.counts, changed);
}

// the exact argmin of every listed row over all K centres (a warp per row)
constexpr int RECHECK_WARPS = 8;
__global__ void __launch_bounds__(RECHECK_WARPS * 32)
km_recheck_kernel(const float* __restrict__ xhat, const float* __restrict__ cen, int d, int K, const int* __restrict__ list,
                  const unsigned int* counts, int* __restrict__ labels, unsigned int* changed) {
    const int lane = threadIdx.x & 31;
    const unsigned int listed = counts[1];
    for (unsigned int w = blockIdx.x * RECHECK_WARPS + (threadIdx.x >> 5); w < listed; w += gridDim.x * RECHECK_WARPS) {
        const int row = list[w];
        const float* a = xhat + static_cast<size_t>(row) * d;
        double best = INFINITY;
        int bc = 0x7fffffff;
        for (int c = lane; c < K; c += 32) {            // ascending per lane: a strict < keeps the lowest centre
            const double s = exact_d2(a, cen + static_cast<size_t>(c) * d, d);
            if (s < best) { best = s; bc = c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
            if (pair_less(ob, oc, best, bc)) { best = ob; bc = oc; }
        }
        if (lane == 0 && labels[row] != bc) {
            labels[row] = bc;
            atomicAdd(changed, 1u);
        }
    }
}

// ---- K16 ---------------------------------------------------------------------------------------------------------------
constexpr int CHUNK = 1024;                     // rows per chunk of the counting sort

// hist[chunk][c] = rows of the chunk with label c (labels outside [0, K) belong to no cluster)
__global__ void __launch_bounds__(256) km_hist_kernel(const int* __restrict__ labels, int n, int K, int* __restrict__ hist) {
    extern __shared__ int h[];
    for (int c = threadIdx.x; c < K; c += blockDim.x) h[c] = 0;
    __syncthreads();
    const int lo = blockIdx.x * CHUNK, hi = min(n, lo + CHUNK);
    for (int r = lo + threadIdx.x; r < hi; r += blockDim.x) {
        const int c = labels[r];
        if (c >= 0 && c < K) atomicAdd(h + c, 1);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < K; c += blockDim.x) hist[static_cast<size_t>(blockIdx.x) * K + c] = h[c];
}

// hist[chunk][c] -> the chunk's first slot of cluster c inside the sorted order; count[c], start[c] (one block)
__global__ void __launch_bounds__(1024) km_scan_kernel(int* __restrict__ hist, int chunks, int K, int* __restrict__ count,
                                                      int* __restrict__ start) {
    for (int c = threadIdx.x; c < K; c += blockDim.x) {
        int run = 0;
        for (int b = 0; b < chunks; ++b) {
            const int v = hist[static_cast<size_t>(b) * K + c];
            hist[static_cast<size_t>(b) * K + c] = run;
            run += v;
        }
        count[c] = run;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int c = 0; c < K; ++c) { start[c] = run; run += count[c]; }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < K; c += blockDim.x) {
        const int s = start[c];
        for (int b = 0; b < chunks; ++b) hist[static_cast<size_t>(b) * K + c] += s;
    }
}

// one warp per chunk places its rows, 32 at a time in row order: a stable sort
__global__ void __launch_bounds__(32) km_place_kernel(const int* __restrict__ labels, int n, int K,
                                                     const int* __restrict__ hist, int* __restrict__ order) {
    extern __shared__ int slot[];
    const int lane = threadIdx.x;
    for (int c = lane; c < K; c += 32) slot[c] = hist[static_cast<size_t>(blockIdx.x) * K + c];
    __syncwarp();
    const int lo = blockIdx.x * CHUNK, hi = min(n, lo + CHUNK);
    for (int r0 = lo; r0 < hi; r0 += 32) {
        const int r = r0 + lane;
        int c = r < hi ? labels[r] : -1;
        if (c >= K) c = -1;
        const unsigned int same = __match_any_sync(0xffffffffu, c);
        const int rank = __popc(same & ((1u << lane) - 1u));
        const int at = c >= 0 ? slot[c] : 0;
        __syncwarp();
        if (c >= 0) {
            order[at + rank] = r;
            if (rank == 0) slot[c] = at + __popc(same);
        }
        __syncwarp();
    }
}

// centre[c][col] = fl32(S / m): one thread per (cluster, column), the members in ascending row order
constexpr int SUM_THREADS = 128;
__global__ void __launch_bounds__(SUM_THREADS) km_sum_kernel(const float* __restrict__ xhat, int d, const int* __restrict__ order,
                                                            const int* __restrict__ count, const int* __restrict__ start,
                                                            float* __restrict__ cen) {
    const int c = blockIdx.y, col = blockIdx.x * SUM_THREADS + threadIdx.x;
    const int m = count[c];
    if (col >= d || m == 0) return;
    const int* mem = order + start[c];
    double s = 0.0;
    int q = 0;
    for (; q + 8 <= m; q += 8) {                        // the loads run ahead; the adds stay one chain
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldg(xhat + static_cast<size_t>(__ldg(mem + q + u)) * d + col);
#pragma unroll
        for (int u = 0; u < 8; ++u) s = __dadd_rn(s, static_cast<double>(v[u]));
    }
    for (; q < m; ++q) s = __dadd_rn(s, static_cast<double>(__ldg(xhat + static_cast<size_t>(__ldg(mem + q)) * d + col)));
    cen[static_cast<size_t>(c) * d + col] = __double2float_rn(__ddiv_rn(s, static_cast<double>(m)));
}

// ---- K17 ---------------------------------------------------------------------------------------------------------------
constexpr int TT = 64;                          // rows and columns of a tile
constexpr int KC = 16;                          // columns of d staged per step
constexpr int TYP_THREADS = 256;
constexpr int TYP_WARPS = TYP_THREADS / 32;
constexpr int ROWS_PER_WARP = TT / TYP_WARPS;

struct TypArgs {
    const float* xhat;
    int d, groups, k_max;
    const int* rows;                   // [m_total] row ids, grouped
    const int* goff;                   // [groups + 1] group offsets into rows
    const int* toff;                   // [groups + 1] first row tile of each group
    double* typ;                       // [m_total]
};

// v into the warp's ascending list (lane l holds the l-th smallest)
__device__ __forceinline__ void list_insert(double& L, double v, int lane) {
    const int pos = __popc(__ballot_sync(0xffffffffu, L <= v));
    const double up = __shfl_up_sync(0xffffffffu, L, 1);
    if (lane == pos) L = v;
    else if (lane > pos) L = up;
}

__global__ void __launch_bounds__(TYP_THREADS) km_typ_kernel(const TypArgs A) {
    __shared__ float sI[TT][KC + 1], sJ[TT][KC + 1];
    __shared__ double sD[TT][TT + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tx = tid & 15, ty = tid >> 4;
    int g = 0, hi = A.groups;                           // the group of this row tile: toff[g] <= blockIdx.x < toff[g + 1]
    while (hi - g > 1) {
        const int mid = (g + hi) >> 1;
        if (A.toff[mid] <= static_cast<int>(blockIdx.x)) g = mid; else hi = mid;
    }
    const int base = A.goff[g], m = A.goff[g + 1] - base;
    const int i0 = (blockIdx.x - A.toff[g]) * TT;
    const int k = min(A.k_max, m / 2);
    if (k == 0) {                                       // a group of one row: no neighbours, typicality 0
        if (tid == 0) A.typ[base] = 0.0;
        return;
    }
    double L[ROWS_PER_WARP];
#pragma unroll
    for (int q = 0; q < ROWS_PER_WARP; ++q) L[q] = INFINITY;

    for (int j0 = 0; j0 < m; j0 += TT) {
        double acc[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[q][r] = 0.0;
        for (int k0 = 0; k0 < A.d; k0 += KC) {
            for (int e = tid; e < TT * KC; e += TYP_THREADS) {
                const int rr = e / KC, kk = e % KC, col = k0 + kk;
                const int pi = i0 + rr, pj = j0 + rr;
                sI[rr][kk] = (pi < m && col < A.d) ? __ldg(A.xhat + static_cast<size_t>(__ldg(A.rows + base + pi)) * A.d + col) : 0.f;
                sJ[rr][kk] = (pj < m && col < A.d) ? __ldg(A.xhat + static_cast<size_t>(__ldg(A.rows + base + pj)) * A.d + col) : 0.f;
            }
            __syncthreads();
#pragma unroll 4
            for (int kk = 0; kk < KC; ++kk) {             // zero columns past d add (0 - 0)^2 = 0: the sum is unchanged
                double a[4], b[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    a[q] = static_cast<double>(sI[ty + 16 * q][kk]);
                    b[q] = static_cast<double>(sJ[tx + 16 * q][kk]);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int r = 0; r < 4; ++r) acc[q][r] = d2_step(acc[q][r], a[q], b[r]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int pi = i0 + ty + 16 * q, pj = j0 + tx + 16 * r;
                sD[ty + 16 * q][tx + 16 * r] = (pj < m && pj != pi) ? acc[q][r] : INFINITY;   // the row itself by position
            }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < ROWS_PER_WARP; ++q) {
            const int ri = warp * ROWS_PER_WARP + q;
            for (int h = 0; h < TT / 32; ++h) {
                const double c = sD[ri][32 * h + lane];
                double thr = __shfl_sync(0xffffffffu, L[q], k - 1);
                unsigned int want = __ballot_sync(0xffffffffu, c < thr);
                while (want) {
                    const int src = __ffs(want) - 1;
                    list_insert(L[q], __shfl_sync(0xffffffffu, c, src), lane);
                    thr = __shfl_sync(0xffffffffu, L[q], k - 1);
                    want &= ~(1u << src);
                    want &= __ballot_sync(0xffffffffu, c < thr);
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < ROWS_PER_WARP; ++q) {
        const int pi = i0 + warp * ROWS_PER_WARP + q;
        double s = 0.0;
        for (int l = 0; l < k; ++l) s = __dadd_rn(s, __shfl_sync(0xffffffffu, L[q], l));   // ascending
        if (lane == 0 && pi < m)
            A.typ[base + pi] = __drcp_rn(__dadd_rn(__ddiv_rn(s, static_cast<double>(k)), 1e-5));
    }
}

// best[g] = the position (into rows) of the group's largest typicality, the lowest on ties (a block per group)
__global__ void __launch_bounds__(256) km_typ_argmax_kernel(const double* __restrict__ typ, const int* __restrict__ goff,
                                                           int* __restrict__ best) {
    __shared__ double sv[8];
    __shared__ int sp[8];
    const int g = blockIdx.x, lo = goff[g], hi = goff[g + 1];
    double v = -INFINITY;
    int p = 0x7fffffff;
    for (int q = lo + threadIdx.x; q < hi; q += blockDim.x) {
        const double t = typ[q];
        if (t > v) { v = t; p = q; }                    // ascending per thread: a strict > keeps the lowest
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int op = __shfl_xor_sync(0xffffffffu, p, o);
        if (ov > v || (ov == v && op < p)) { v = ov; p = op; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = v; sp[threadIdx.x >> 5] = p; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w)
            if (sv[w] > v || (sv[w] == v && sp[w] < p)) { v = sv[w]; p = sp[w]; }
        best[g] = p;
    }
}

// ---- K21 ---------------------------------------------------------------------------------------------------------------
// d2[i] = exact_d2(xhat_i, centre_{labels[i]}); best_d2[c] = the smallest over the rows labeled c (as 64-bit patterns)
__global__ void __launch_bounds__(256) km_near_d2_kernel(const float* __restrict__ xhat, int n, int d, const int* __restrict__ labels,
                                                         const float* __restrict__ cen, int K, double* __restrict__ d2,
                                                         unsigned long long* __restrict__ best_d2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = labels[i];
    if (c < 0 || c >= K) return;
    const double v = exact_d2(xhat + static_cast<size_t>(i) * d, cen + static_cast<size_t>(c) * d, d);
    d2[i] = v;
    atomicMin(best_d2 + c, static_cast<unsigned long long>(__double_as_longlong(v)));
}

// best_row[c] = the lowest row labeled c whose d2 equals best_d2[c]; best_row starts at 0xffffffff, which stays (-1 as
// int32) for an empty cluster
__global__ void __launch_bounds__(256) km_near_row_kernel(int n, const int* __restrict__ labels, int K, const double* __restrict__ d2,
                                                          const unsigned long long* __restrict__ best_d2,
                                                          unsigned int* __restrict__ best_row) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = labels[i];
    if (c < 0 || c >= K) return;
    if (static_cast<unsigned long long>(__double_as_longlong(d2[i])) == best_d2[c]) atomicMin(best_row + c, static_cast<unsigned int>(i));
}

}  // namespace tk

extern "C" int alq_kmeans_rows(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, int32_t normalise,
                               float* xhat, float* hi, float* lo, double* nrm2, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_rows: n=%lld outside [1, 2^31)", (long long)n);
    if (d < 4 || d % 4) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_rows: d=%d must be a positive multiple of 4", d);
    if ((normalise && (!x || ldx < d)) || !xhat || !hi || !lo || !nrm2)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_rows: null pointer or ldx < d");
    const int ni = static_cast<int>(n);
    rs::normalize_split_kernel<<<(ni + rs::NORM_WARPS - 1) / rs::NORM_WARPS, rs::NORM_WARPS * 32, 0,
                                 static_cast<cudaStream_t>(stream)>>>(x, ni, d, ldx, xhat, hi, lo, nrm2, normalise ? 1 : 0);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_kmeans_assign(alq_ctx* ctx, const float* xhat, const float* hi, const float* lo, const double* nrm2,
                                 int64_t n, int32_t d, const float* centres, int32_t k, int32_t* labels,
                                 int64_t* counts_host, void* stream) {
    using namespace tk;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_assign: n=%lld outside [1, 2^31)", (long long)n);
    if (d < 4 || d % 4) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_assign: d=%d must be a positive multiple of 4", d);
    if (k < 1 || k > K_MAX) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_assign: K=%d outside [1, %d]", k, K_MAX);
    if (!xhat || !hi || !lo || !nrm2 || !centres || !labels || !counts_host || !aligned16(xhat) || !aligned16(hi) ||
        !aligned16(lo))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_assign: null pointer or xhat / hi / lo not 16-byte aligned");
    if (!tc::get_encode()) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_kmeans_assign: cuTensorMapEncodeTiled is unavailable");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    const size_t ce = static_cast<size_t>(k) * d;
    float *chi, *clo, *cc;                             // cc: the centres' copy the split reads back
    double* cn;
    int* list;
    unsigned int* cnt;                                 // [0] labels changed, [1] rows listed, [2] norms refused
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        chi = cur.take<float>(ce);
        clo = cur.take<float>(ce);
        cc = cur.take<float>(ce);
        cn = cur.take<double>(k);
        list = cur.take<int>(n);
        cnt = cur.take<unsigned int>(3);
    });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaMemcpyAsync(cc, centres, ce * 4, cudaMemcpyDeviceToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(cnt, 0, 12, st));
    rs::normalize_split_kernel<<<(k + rs::NORM_WARPS - 1) / rs::NORM_WARPS, rs::NORM_WARPS * 32, 0, st>>>(
        nullptr, k, d, d, cc, chi, clo, cn, 0);
    ALQ_LAUNCH_CHECK(ctx);
    const unsigned int dblocks = static_cast<unsigned int>((static_cast<long long>(ni) + k + 255) / 256);
    km_domain_kernel<<<dblocks, 256, 0, st>>>(nrm2, ni, cn, k, cnt + 2);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned int bad = 0u;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&bad, cnt + 2, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (bad)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_assign: %u rows or centres have a squared norm that is not in [0, 2]",
                 bad);

    CUtensorMap mxh, mxl, mch, mcl;
    if (!tc::make_map(&mxh, hi, n, d, BM) || !tc::make_map(&mxl, lo, n, d, BM) || !tc::make_map(&mch, chi, k, d, BM) ||
        !tc::make_map(&mcl, clo, k, d, BM))
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_kmeans_assign: cuTensorMapEncodeTiled failed");
    AssignParams P{};
    P.nrm2 = nrm2; P.cn = cn;
    P.n = ni; P.K = k; P.ctiles = (k + BM - 1) / BM; P.kblocks = (d + BK - 1) / BK; P.rblocks = (ni + BM - 1) / BM;
    // DESIGN section 4: with squared norms in [0, 2], d2 <= 8 and the slack covers the fp64 epilogue and the exact
    // sum's own rounding (d 2^-53 of at most 8)
    P.coef = tc::band_coef(d);
    P.slack = 1e-9;
    P.labels = labels; P.list = list; P.counts = cnt;
    const size_t smem = tc::ring_smem_bytes(0);
    ALQ_CUDA(ctx, cudaFuncSetAttribute(km_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    km_assign_kernel<<<std::min(ctx->sm_count, P.rblocks), tc::THREADS, smem, st>>>(mxh, mxl, mch, mcl, P);
    ALQ_LAUNCH_CHECK(ctx);
    km_recheck_kernel<<<ctx->sm_count * 4, RECHECK_WARPS * 32, 0, st>>>(xhat, cc, d, k, list, cnt, labels, cnt);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned int h[2] = {0u, 0u};
    ALQ_CUDA(ctx, cudaMemcpyAsync(h, cnt, 8, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    counts_host[0] = h[0];
    counts_host[1] = h[1];
    return ALQ_OK;
}

extern "C" int alq_kmeans_update(alq_ctx* ctx, const float* xhat, int64_t n, int32_t d, const int32_t* labels, int32_t k,
                                 float* centres, void* stream) {
    using namespace tk;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_update: n=%lld outside [1, 2^31)", (long long)n);
    if (d < 1) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_update: d=%d must be positive", d);
    if (k < 1 || k > K_MAX) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_update: K=%d outside [1, %d]", k, K_MAX);
    if (!xhat || !labels || !centres) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_update: null pointer");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    const int chunks = (ni + CHUNK - 1) / CHUNK;
    int *hist, *count, *start, *order;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        hist = cur.take<int>(static_cast<size_t>(chunks) * k);
        count = cur.take<int>(k);
        start = cur.take<int>(k);
        order = cur.take<int>(n);
    });
    if (rc) return rc;
    const size_t hsm = static_cast<size_t>(k) * 4;
    ALQ_CUDA(ctx, cudaFuncSetAttribute(km_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(hsm)));
    ALQ_CUDA(ctx, cudaFuncSetAttribute(km_place_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(hsm)));
    km_hist_kernel<<<chunks, 256, hsm, st>>>(labels, ni, k, hist);
    ALQ_LAUNCH_CHECK(ctx);
    km_scan_kernel<<<1, 1024, 0, st>>>(hist, chunks, k, count, start);
    ALQ_LAUNCH_CHECK(ctx);
    km_place_kernel<<<chunks, 32, hsm, st>>>(labels, ni, k, hist, order);
    ALQ_LAUNCH_CHECK(ctx);
    km_sum_kernel<<<dim3((d + SUM_THREADS - 1) / SUM_THREADS, k), SUM_THREADS, 0, st>>>(xhat, d, order, count, start, centres);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_typicality(alq_ctx* ctx, const float* xhat, int32_t d, const int32_t* rows, const int64_t* group_off_host,
                              int32_t groups, int32_t k_max, double* typ, int32_t* best, void* stream) {
    using namespace tk;
    if (!ctx) return ALQ_ERR_INVALID;
    if (d < 1) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: d=%d must be positive", d);
    if (k_max < 1 || k_max > 32) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: k=%d outside [1, 32]", k_max);
    if (groups < 1 || !group_off_host) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: need at least one group");
    if (group_off_host[0] != 0) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: group offsets must start at 0");
    std::vector<int> goff(groups + 1), toff(groups + 1);
    long long tiles = 0;
    for (int g = 0; g < groups; ++g) {
        const int64_t m = group_off_host[g + 1] - group_off_host[g];
        if (m < 1 || group_off_host[g + 1] >= (1LL << 31))
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: group %d is empty or the rows reach 2^31", g);
        goff[g] = static_cast<int>(group_off_host[g]);
        toff[g] = static_cast<int>(tiles);
        tiles += (m + TT - 1) / TT;
    }
    goff[groups] = static_cast<int>(group_off_host[groups]);
    toff[groups] = static_cast<int>(tiles);
    if (!xhat || !rows || !typ || !best) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: null pointer");
    if (tiles >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_typicality: too many row tiles");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    int *dg, *dt;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        dg = cur.take<int>(groups + 1);
        dt = cur.take<int>(groups + 1);
    });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaMemcpyAsync(dg, goff.data(), goff.size() * 4, cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(dt, toff.data(), toff.size() * 4, cudaMemcpyHostToDevice, st));
    TypArgs A{};
    A.xhat = xhat; A.d = d; A.groups = groups; A.k_max = k_max;
    A.rows = rows; A.goff = dg; A.toff = dt; A.typ = typ;
    km_typ_kernel<<<static_cast<unsigned int>(tiles), TYP_THREADS, 0, st>>>(A);
    ALQ_LAUNCH_CHECK(ctx);
    km_typ_argmax_kernel<<<groups, 256, 0, st>>>(typ, dg, best);
    ALQ_LAUNCH_CHECK(ctx);
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    return ALQ_OK;
}

extern "C" int alq_kmeans_nearest(alq_ctx* ctx, const float* xhat, int64_t n, int32_t d, const int32_t* labels,
                                  const float* centres, int32_t k, int32_t* nearest, void* stream) {
    using namespace tk;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_nearest: n=%lld outside [1, 2^31)", (long long)n);
    if (d < 4 || d % 4) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_nearest: d=%d must be a positive multiple of 4", d);
    if (k < 1) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_nearest: K=%d must be positive", k);
    if (!xhat || !labels || !centres || !nearest || !aligned16(xhat) || !aligned16(centres))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_kmeans_nearest: null pointer or xhat / centres not 16-byte aligned");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    double* d2;
    unsigned long long* best;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        d2 = cur.take<double>(n);
        best = cur.take<unsigned long long>(k);
    });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaMemsetAsync(best, 0xff, static_cast<size_t>(k) * 8, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(nearest, 0xff, static_cast<size_t>(k) * 4, st));
    km_near_d2_kernel<<<(ni + 255) / 256, 256, 0, st>>>(xhat, ni, d, labels, centres, k, d2, best);
    ALQ_LAUNCH_CHECK(ctx);
    km_near_row_kernel<<<(ni + 255) / 256, 256, 0, st>>>(ni, labels, k, d2, best, reinterpret_cast<unsigned int*>(nearest));
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

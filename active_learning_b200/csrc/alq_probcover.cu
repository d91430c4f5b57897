// K13 / K14: ProbCoverSampler (Yehuda et al., "Active Learning Through a Covering Lens", NeurIPS 2022) on the device.
//
// K13 alq_probcover_graph   the delta-ball graph of the L2-normalised pool rows as CSR.  There is an edge (i, j) iff
//                           scipy's fp64 euclidean distance of the fp32 rows (K7's per-pair arithmetic) is < delta.
//   normalise  one warp per row: lane-strided fp64 sum of squares, a butterfly, norm = sqrt, xhat = fl32(x / norm)
//              (a zero row stays zero); the same kernel splits xhat into TF32 hi / lo (alq_wgmma.cuh) and stores
//              nrm2 = |xhat|^2 in fp64.
//   screen     one CTA per SM, persistent over the upper-triangle 128 x 128 tiles of xhat xhat^T, on the ring of
//              alq_wgmma.cuh that K3 and K9 use: warpgroup 0 is the TMA producer (3-stage ring), warpgroups 1-2 issue
//              the 3xTF32 chain tc::ring_mma.  The epilogue decides each pair from d2 = nrm2_i + nrm2_j - 2 g
//              (g the tensor-core dot product) against the bound
//              |g - <xhat_i, xhat_j>| <= E_ij of DESIGN section 4: clearly inside delta^2 is an edge, clearly outside is
//              not, and a pair inside the band is recomputed exactly with K7's arithmetic.  A pair is decided once per
//              tile, so (i, j) and (j, i) of an off-diagonal tile share one decision; on a diagonal tile both orders are
//              decided separately and agree because every decision equals the exact one.
//   CSR        the tile's decisions go into a 128 x 128 bitmap in shared memory.  Thread t of the consumers then owns
//              tile row t (the edges (i, j), j in the column block) and, on an off-diagonal tile, thread 128 + t owns
//              tile column t (the mirrored edges (j, i)).  Count pass: the number of edges of every (row, column block)
//              into tile_cnt[row][block] (each entry has exactly one writer).  A row scan turns that into offsets inside
//              the row and a row-total scan into row_ptr.  Fill pass (the same screen, bit for bit): each owner writes
//              its edges in ascending column order at row_ptr[row] + tile_cnt[row][block], so every CSR row is ascending
//              without a sort.
// K14 alq_probcover_select  the greedy coverage picks.  Two set-up launches mark every row in a labeled row's ball
//              covered and count deg[x] = |{y in N(x) : y uncovered}|.  Then ONE ordinary launch, one CTA per SM
//              (bracketed by alq_gridsync_begin/end, every wait bounded by "spin_timeout_ms"), runs every pick: each CTA
//              reduces its row segment to (deg, lowest row) and the grid agrees over 8-byte LL words (ll_agree_min); the
//              ball of the pick is split over every thread of the grid, a newly covered y subtracts one from deg[x] of
//              every x in N(y) (atomicSub), and a second round of LL words is the grid barrier before the next step.
//              Work per query: O(B n / SMs + nnz).
#include <math.h>

#include "alq_ll.cuh"
#include "alq_wgmma.cuh"

namespace pc {

using tc::BK;
using tc::BM;                                 // rows and columns of a tile
constexpr int NORM_WARPS = 8;
constexpr int BITS_BYTES = BM * 4 * 4;        // the screen's tile bitmap: [128 rows][4 words]

// ---- normalise + split ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NORM_WARPS * 32)
pc_normalize_kernel(const float* __restrict__ x, int n, int d, long long ldx, float* __restrict__ xhat,
                    float* __restrict__ hi, float* __restrict__ lo, double* __restrict__ nrm2, int normalise) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * NORM_WARPS + (threadIdx.x >> 5);
    if (row >= n) return;
    float* xr = xhat + static_cast<size_t>(row) * d;
    if (normalise) {
        const float* src = x + static_cast<size_t>(row) * ldx;
        double s = 0.0;
        for (int k = lane; k < d; k += 32) {
            const double v = static_cast<double>(src[k]);
            s = __dadd_rn(s, __dmul_rn(v, v));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
        const double norm = __dsqrt_rn(s);
        for (int k = lane; k < d; k += 32)
            xr[k] = norm > 0.0 ? __double2float_rn(__ddiv_rn(static_cast<double>(src[k]), norm)) : 0.f;
    }
    double t = 0.0;
    for (int k = lane; k < d; k += 32) {            // the lane reads back what it wrote
        const float v = xr[k];
        float h, l;
        tc::split_tf32(v, h, l);
        hi[static_cast<size_t>(row) * d + k] = h;
        lo[static_cast<size_t>(row) * d + k] = l;
        t = __dadd_rn(t, __dmul_rn(static_cast<double>(v), static_cast<double>(v)));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = __dadd_rn(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) nrm2[row] = t;
}

struct GraphParams {
    const float* xhat;                 // [n, d]
    const double* nrm2;                // [n]
    int n, d, ntiles, kblocks;
    long long tile_pairs;              // ntiles (ntiles + 1) / 2
    double delta, delta2;
    double coef;                       // d2 error per unit of sqrt(nrm2_i nrm2_j) (DESIGN section 4)
    double slack;                      // absolute slack of the fp64 epilogue and of the exact value's own rounding
    int* tile_cnt;                     // [n][ntiles]: counts (count pass), offsets inside the row (fill pass)
    const long long* row_ptr;          // fill pass
    int* cols;                         // fill pass
    unsigned long long* recheck;       // count pass: pairs decided by the exact recomputation
    int fill;
};

// upper-triangle tile idx -> (ti, tj), row-major: row t starts at t nt - t (t - 1) / 2
__device__ __forceinline__ long long tri_off(long long t, long long nt) { return t * nt - t * (t - 1) / 2; }
__device__ __forceinline__ void tile_of(long long idx, int nt, int& ti, int& tj) {
    const double b = 2.0 * nt + 1.0;
    long long t = static_cast<long long>((b - sqrt(fmax(b * b - 8.0 * static_cast<double>(idx), 0.0))) * 0.5);
    t = t < 0 ? 0 : (t >= nt ? nt - 1 : t);
    while (t > 0 && tri_off(t, nt) > idx) --t;
    while (t + 1 < nt && tri_off(t + 1, nt) <= idx) ++t;
    ti = static_cast<int>(t);
    tj = static_cast<int>(t + (idx - tri_off(t, nt)));
}

// K7's pair arithmetic (scipy's euclidean on fp32 rows): d = a - b in fp64, s = s + d * d, k ascending, no FMA
__device__ __noinline__ bool exact_edge(const float* __restrict__ xhat, int d, int i, int j, double delta) {
    const float* a = xhat + static_cast<size_t>(i) * d;
    const float* b = xhat + static_cast<size_t>(j) * d;
    double s = 0.0;
    for (int k = 0; k < d; ++k) {
        const double df = __dsub_rn(static_cast<double>(__ldg(a + k)), static_cast<double>(__ldg(b + k)));
        s = __dadd_rn(s, __dmul_rn(df, df));
    }
    return __dsqrt_rn(s) < delta;
}

__device__ __forceinline__ uint32_t decide(const GraphParams& P, float g, double ni, double nj, int i, int j,
                                           unsigned int& rech) {
    const double d2 = __dsub_rn(__dadd_rn(ni, nj), 2.0 * static_cast<double>(g));
    const double bnd = __dadd_rn(__dmul_rn(P.coef, __dsqrt_rn(__dmul_rn(ni, nj))), P.slack);
    if (d2 < P.delta2 - bnd) return 1u;
    if (d2 > P.delta2 + bnd) return 0u;
    ++rech;
    return exact_edge(P.xhat, P.d, i, j, P.delta) ? 1u : 0u;
}

__global__ void __launch_bounds__(tc::THREADS, 1)
pc_graph_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                const GraphParams P) {
    extern __shared__ unsigned char smem_dyn[];
    const tc::Role me = tc::ring_role();
    const int nt = P.ntiles;
    const tc::Ring ring = tc::ring_init(smem_dyn);
    uint32_t* bits = reinterpret_cast<uint32_t*>(ring.tail);              // [128 rows][4 words]: the tile's edges

    if (me.wg == 0) {
        tc::producer_regs();
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            for (long long idx = blockIdx.x; idx < P.tile_pairs; idx += gridDim.x) {
                int ti, tj;
                tile_of(idx, nt, ti, tj);
                for (int kb = 0; kb < P.kblocks; ++kb, ++it)
                    tc::ring_load(ring, it, &map_hi, &map_lo, ti * BM, &map_hi, &map_lo, tj * BM, kb * BK);
            }
        }
        return;
    }
    tc::consumer_regs();
    const int ct = threadIdx.x - 128;
    unsigned int rech = 0;
    uint32_t it = 0;
    for (long long idx = blockIdx.x; idx < P.tile_pairs; idx += gridDim.x) {
        int ti, tj;
        tile_of(idx, nt, ti, tj);
        float acc[64];
        int prev = -1;
        for (int kb = 0; kb < P.kblocks; ++kb, ++it) tc::ring_mma(ring, it, me.a_off, acc, kb == 0, prev, me.t);
        tc::ring_drain(ring, prev, me.t);

        // ---- epilogue: the decisions of this thread's 2 x 32 pairs as canonical column masks of its two rows
        const int row0 = ti * BM + me.r_in_tile, row1 = row0 + 8;
        const double n0 = row0 < P.n ? __ldg(P.nrm2 + row0) : 0.0, n1 = row1 < P.n ? __ldg(P.nrm2 + row1) : 0.0;
        uint32_t m0[4] = {0u, 0u, 0u, 0u}, m1[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int cl = 8 * j + me.c_in_tile + e, col = tj * BM + cl;
                if (col >= P.n) continue;
                const double nc = __ldg(P.nrm2 + col);
                if (row0 < P.n) m0[cl >> 5] |= decide(P, acc[4 * j + e], n0, nc, row0, col, rech) << (cl & 31);
                if (row1 < P.n) m1[cl >> 5] |= decide(P, acc[4 * j + 2 + e], n1, nc, row1, col, rech) << (cl & 31);
            }
        }
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1)
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                m0[w] |= __shfl_xor_sync(0xffffffffu, m0[w], o);
                m1[w] |= __shfl_xor_sync(0xffffffffu, m1[w], o);
            }
        if ((me.lane & 3) == 0)
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                bits[me.r_in_tile * 4 + w] = m0[w];
                bits[(me.r_in_tile + 8) * 4 + w] = m1[w];
            }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct < BM) {
            const int row = ti * BM + ct;                  // tile row ct: edges (row, tj * 128 + c)
            if (row < P.n) {
                int* slot = P.tile_cnt + static_cast<size_t>(row) * nt + tj;
                if (!P.fill) {
                    int c = 0;
#pragma unroll
                    for (int w = 0; w < 4; ++w) c += __popc(bits[ct * 4 + w]);
                    *slot = c;
                } else {
                    long long at = P.row_ptr[row] + *slot;
#pragma unroll
                    for (int w = 0; w < 4; ++w)
                        for (uint32_t m = bits[ct * 4 + w]; m; m &= m - 1) P.cols[at++] = tj * BM + 32 * w + (__ffs(m) - 1);
                }
            }
        } else if (ti != tj) {
            const int c = ct - BM, col = tj * BM + c;      // tile column c: mirrored edges (col, ti * 128 + r)
            if (col < P.n) {
                int* slot = P.tile_cnt + static_cast<size_t>(col) * nt + ti;
                const int w = c >> 5;
                const uint32_t bit = 1u << (c & 31);
                if (!P.fill) {
                    int cnt = 0;
                    for (int r = 0; r < BM; ++r) cnt += (bits[r * 4 + w] & bit) ? 1 : 0;
                    *slot = cnt;
                } else {
                    long long at = P.row_ptr[col] + *slot;
                    for (int r = 0; r < BM; ++r)
                        if (bits[r * 4 + w] & bit) P.cols[at++] = ti * BM + r;
                }
            }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");    // the bitmap is rewritten by the next tile
    }
    if (!P.fill && rech) atomicAdd(P.recheck, static_cast<unsigned long long>(rech));
}

// tile_cnt[row][*] -> exclusive offsets inside the row; row_ptr[row + 1] = the row's edges (one warp per row)
__global__ void __launch_bounds__(256) pc_row_scan_kernel(int* __restrict__ tile_cnt, int n, int nt, long long* __restrict__ row_ptr) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n) return;
    int* r = tile_cnt + static_cast<size_t>(row) * nt;
    int run = 0;
    for (int k0 = 0; k0 < nt; k0 += 32) {
        const int v = k0 + lane < nt ? r[k0 + lane] : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += u;
        }
        if (k0 + lane < nt) r[k0 + lane] = run + inc - v;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) row_ptr[row + 1] = run;
}

// row_ptr[0] = 0, row_ptr[i + 1] = sum of the row totals up to i (one block)
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS) pc_ptr_scan_kernel(long long* __restrict__ row_ptr, int n) {
    __shared__ long long part[SCAN_THREADS];
    const int t = threadIdx.x;
    const int per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
    const int lo = min(n, t * per), hi = min(n, lo + per);
    long long s = 0;
    for (int i = lo; i < hi; ++i) s += row_ptr[i + 1];
    part[t] = s;
    __syncthreads();
    if (t == 0) {
        long long run = 0;
        for (int k = 0; k < SCAN_THREADS; ++k) { const long long v = part[k]; part[k] = run; run += v; }
    }
    __syncthreads();
    long long run = part[t];
    for (int i = lo; i < hi; ++i) { run += row_ptr[i + 1]; row_ptr[i + 1] = run; }
    if (t == 0) row_ptr[0] = 0;
}

// ---- K14 --------------------------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 512;                 // >= kPollers: every poller of ll_gather is a thread of the CTA
constexpr int SEL_WARPS = SEL_THREADS / 32;

// every row in a labeled row's ball is covered (one warp per row)
__global__ void __launch_bounds__(256) pc_cover_kernel(const long long* __restrict__ row_ptr, const int* __restrict__ cols, int n,
                                                       const uint8_t* __restrict__ labeled, uint8_t* __restrict__ covered) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n || !labeled[row]) return;
    for (long long e = row_ptr[row] + (threadIdx.x & 31); e < row_ptr[row + 1]; e += 32) covered[cols[e]] = 1;
}

// deg[x] = uncovered rows in N(x) (one warp per row)
__global__ void __launch_bounds__(256) pc_deg_kernel(const long long* __restrict__ row_ptr, const int* __restrict__ cols, int n,
                                                     const uint8_t* __restrict__ covered, int* __restrict__ deg) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= n) return;
    int c = 0;
    for (long long e = row_ptr[row] + lane; e < row_ptr[row + 1]; e += 32) c += covered[cols[e]] ? 0 : 1;
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) deg[row] = c;
}

struct SelArgs {
    const long long* row_ptr;
    const int* cols;
    int n, budget;
    int* deg;
    uint8_t* covered;
    SegShard S;                  // world 1: off = {0, n}
    LLWords W;                   // [2 parities][grid] key words at keyw = 0 of peer[0] (scratch)
    char* barw;                  // [2 parities][grid] barrier words, behind the key words
    int* picks;
    int* steps;
    int* status;
    long long timeout_cycles;
};

__global__ void __launch_bounds__(SEL_THREADS, 1) pc_greedy_kernel(const __grid_constant__ SelArgs A) {
    __shared__ unsigned long long s_key[SEL_WARPS];
    __shared__ int s_pick;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x, G = gridDim.x;
    const int lo = gseg_lo(A.S, b), hi = gseg_lo(A.S, b + 1);
    int steps = 0;
    for (int t = 0; t < A.budget; ++t) {
        // ---- the grid agrees on (largest deg, lowest row): the smallest key (0xffffffff - deg) << 32 | row, deg > 0
        unsigned long long best = ~0ull;
        for (int row = lo + tid; row < hi; row += SEL_THREADS) {
            const int dg = __ldcg(A.deg + row);
            if (dg > 0) {
                const unsigned long long key = (static_cast<unsigned long long>(0xffffffffu - static_cast<uint32_t>(dg)) << 32) | static_cast<uint32_t>(row);
                best = key < best ? key : best;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o);
            best = w < best ? w : best;
        }
        if (lane == 0) s_key[warp] = best;
        __syncthreads();
        const int pick = ll_agree_min<SEL_WARPS>(A, s_key, &s_pick, static_cast<unsigned int>(t), lo, tid);
        if (pick < 0 || pick >= A.n) break;                           // max deg = 0: full coverage (or a failed wait)
        if (b == 0 && tid == 0) A.picks[t] = pick;
        steps = t + 1;
        // ---- cover the ball of the pick, split over every thread of the grid
        const long long e1 = A.row_ptr[pick + 1];
        for (long long e = A.row_ptr[pick] + static_cast<long long>(b) * SEL_THREADS + tid; e < e1;
             e += static_cast<long long>(G) * SEL_THREADS) {
            const int y = __ldg(A.cols + e);
            if (__ldcg(A.covered + y)) continue;                      // y appears once in the ball: one thread owns it
            __stcg(A.covered + y, static_cast<uint8_t>(1));
            const long long f1 = A.row_ptr[y + 1];
            for (long long f = A.row_ptr[y]; f < f1; ++f) atomicSub(A.deg + __ldg(A.cols + f), 1);
        }
        // ---- grid barrier: every deg and covered update of this step is visible before the next arg-max
        __syncthreads();
        const unsigned long long tag = ll_key_tag(A.W, static_cast<unsigned int>(t));
        char* barw = A.barw + static_cast<size_t>(t & 1) * G * 8;
        if (tid == 0) {
            __threadfence();
            ll_store_raw(barw + static_cast<size_t>(b) * 8, tag << 48);
        }
        ll_gather(barw, G, 8, tag, 48, A, tid, [](int, unsigned long long) {});
        __threadfence();
        __syncthreads();
    }
    if (b == 0 && tid == 0) *A.steps = steps;
}

}  // namespace pc

extern "C" int alq_probcover_graph(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, const double* delta_host,
                                   float* xhat, int32_t* tile_cnt, int64_t* row_ptr, int32_t* cols, int64_t* nnz_host,
                                   int64_t* recheck_host, void* stream) {
    using namespace pc;
    if (!ctx) return ALQ_ERR_INVALID;
    const bool fill = cols != nullptr;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_graph: n=%lld outside [1, 2^31)", (long long)n);
    if (d < 4 || d % 4) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_graph: d=%d must be a positive multiple of 4", d);
    if (!delta_host || !(*delta_host > 0.0) || !isfinite(*delta_host))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_graph: delta must be finite and > 0");
    if ((!fill && (!x || ldx < d)) || !xhat || !tile_cnt || !row_ptr || !nnz_host || !recheck_host || !aligned16(xhat))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_graph: null pointer, ldx < d or xhat not 16-byte aligned");
    if (!tc::get_encode()) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_probcover_graph: cuTensorMapEncodeTiled is unavailable");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    const int nt = (ni + BM - 1) / BM;
    const size_t e = static_cast<size_t>(n) * d;
    int rc = alq_scratch_reserve(ctx, scratch_need({e * 4, e * 4, static_cast<size_t>(n) * 8, 8}));
    if (rc) return rc;
    ScratchCursor cur(ctx->scratch);
    float* hi = cur.take<float>(e);
    float* lo = cur.take<float>(e);
    double* nrm2 = cur.take<double>(n);
    unsigned long long* rech = cur.take<unsigned long long>(1);

    pc_normalize_kernel<<<(ni + NORM_WARPS - 1) / NORM_WARPS, NORM_WARPS * 32, 0, st>>>(x, ni, d, ldx, xhat, hi, lo, nrm2, fill ? 0 : 1);
    ALQ_LAUNCH_CHECK(ctx);
    if (!fill) ALQ_CUDA(ctx, cudaMemsetAsync(rech, 0, 8, st));

    CUtensorMap mhi, mlo;
    if (!tc::make_map(&mhi, hi, n, d, BM) || !tc::make_map(&mlo, lo, n, d, BM))
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_probcover_graph: cuTensorMapEncodeTiled failed");
    GraphParams P{};
    P.xhat = xhat; P.nrm2 = nrm2;
    P.n = ni; P.d = d; P.ntiles = nt; P.kblocks = (d + BK - 1) / BK;
    P.tile_pairs = static_cast<long long>(nt) * (nt + 1) / 2;
    P.delta = *delta_host;
    P.delta2 = P.delta * P.delta;
    // DESIGN section 4: |g - <xhat_i, xhat_j>| <= (1 + 3 ceil(d / 8)) 2^-20 sqrt(nrm2_i nrm2_j); d2 carries twice that
    P.coef = 2.0 * (1.0 + 3.0 * ((d + 7) / 8)) * ldexp(1.0, -20) * (1.0 + 1e-6);
    P.slack = 1e-9 * P.delta2 + 1e-10;
    P.tile_cnt = tile_cnt; P.row_ptr = reinterpret_cast<const long long*>(row_ptr); P.cols = cols;
    P.recheck = rech; P.fill = fill ? 1 : 0;
    const size_t smem = tc::ring_smem_bytes(BITS_BYTES);
    ALQ_CUDA(ctx, cudaFuncSetAttribute(pc_graph_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    const int grid = static_cast<int>(std::min<long long>(ctx->sm_count, P.tile_pairs));
    pc_graph_kernel<<<grid, tc::THREADS, smem, st>>>(mhi, mlo, P);
    ALQ_LAUNCH_CHECK(ctx);
    if (fill) {
        ALQ_CUDA(ctx, cudaStreamSynchronize(st));
        return ALQ_OK;
    }
    pc_row_scan_kernel<<<(ni + 7) / 8, 256, 0, st>>>(tile_cnt, ni, nt, reinterpret_cast<long long*>(row_ptr));
    ALQ_LAUNCH_CHECK(ctx);
    pc_ptr_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(reinterpret_cast<long long*>(row_ptr), ni);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned long long rech_h = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(nnz_host, row_ptr + n, 8, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(&rech_h, rech, 8, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    *recheck_host = static_cast<int64_t>(rech_h);
    return ALQ_OK;
}

extern "C" int alq_probcover_select(alq_ctx* ctx, const int64_t* row_ptr, const int32_t* cols, int64_t n,
                                    const uint8_t* labeled, int64_t budget, int32_t* picks, int64_t* n_steps_host,
                                    void* stream) {
    using namespace pc;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_select: n=%lld outside [1, 2^31)", (long long)n);
    if (budget < 0 || budget > n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_select: budget=%lld outside [0, n=%lld]", (long long)budget, (long long)n);
    if (!row_ptr || !cols || !labeled || !n_steps_host || (budget > 0 && !picks))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_select: null pointer");
    *n_steps_host = 0;
    if (budget == 0) return ALQ_OK;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    const int grid = std::max(1, std::min(ctx->sm_count, (ni + 255) / 256));
    if ((ni + grid - 1) / grid > kSegRowsMax)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_probcover_select: n=%d rows over %d CTAs exceed %d rows per CTA segment", ni, grid,
                 kSegRowsMax);
    int rc = alq_scratch_reserve(ctx, scratch_need({static_cast<size_t>(n) * 4, static_cast<size_t>(n),
                                                    static_cast<size_t>(4) * grid * 8, 16}));
    if (rc) return rc;
    ScratchCursor cur(ctx->scratch);
    int* deg = cur.take<int>(n);
    uint8_t* covered = cur.take<uint8_t>(n);
    char* words = cur.take<char>(static_cast<size_t>(4) * grid * 8);
    int* small = cur.take<int>(4);                                   // [0] status, [1] steps
    ALQ_CUDA(ctx, cudaMemsetAsync(covered, 0, static_cast<size_t>(n), st));
    ALQ_CUDA(ctx, cudaMemsetAsync(words, 0, static_cast<size_t>(4) * grid * 8, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(small, 0, 4 * sizeof(int), st));
    const long long* rp = reinterpret_cast<const long long*>(row_ptr);
    pc_cover_kernel<<<(ni + 7) / 8, 256, 0, st>>>(rp, cols, ni, labeled, covered);
    ALQ_LAUNCH_CHECK(ctx);
    pc_deg_kernel<<<(ni + 7) / 8, 256, 0, st>>>(rp, cols, ni, covered, deg);
    ALQ_LAUNCH_CHECK(ctx);
    SelArgs A{};
    A.row_ptr = rp; A.cols = cols; A.n = ni; A.budget = static_cast<int>(budget);
    A.deg = deg; A.covered = covered;
    A.S.world = 1; A.S.rank = 0; A.S.grid = grid;
    A.S.off[0] = 0; A.S.off[1] = ni;
    A.W.peer[0] = words;
    A.W.tag_base = 0x80000000u;
    A.barw = words + static_cast<size_t>(2) * grid * 8;
    A.picks = picks; A.steps = small + 1; A.status = small;
    A.timeout_cycles = ctx->spin_timeout_cycles();
    // every CTA spins on the others' words, so all of them must be resident: grid <= SMs, one CTA per SM
    const cudaError_t le = alq_gridsync_launch(ctx, st, [&] {
        pc_greedy_kernel<<<grid, SEL_THREADS, 0, st>>>(A);
        return cudaGetLastError();
    });
    if (le != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_probcover_select: launch failed: %s", cudaGetErrorString(le));
    int small_h[2] = {0, 0};
    ALQ_CUDA(ctx, cudaMemcpyAsync(small_h, small, sizeof(small_h), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (small_h[0] != 0) ALQ_FAIL(ctx, small_h[0], "alq_probcover_select: timed out waiting for a CTA of the grid");
    *n_steps_host = small_h[1];
    return ALQ_OK;
}

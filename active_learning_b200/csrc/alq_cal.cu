// K18 / K19: CALSampler (Margatina, Vernikos, Barrault & Aletras, "Active Learning by Acquiring Contrastive Examples",
// EMNLP 2021) on the device.
//
// K18 alq_knn        idx[i][0..k) = the k rows j of y with the smallest exact fp64 d2(x_i, y_j) = exact_d2 (K7's pair
//                    arithmetic, alq_common.cuh), ascending (d2, j) = pair_less; the raw rows, not normalised.
//   split      x and y through alq_rows_split.cuh's kernel without normalisation: TF32 hi / lo and nrm2 = |row|^2 in fp64;
//              knn_norms_kernel refuses a squared norm that is not finite or above NRM2_MAX and writes sqrt(nrm2).
//   screen     one CTA per SM, persistent over 128-row blocks of x; for each, every 128-column tile of y on the ring of
//              alq_wgmma.cuh (warpgroup 0 runs tc::ring_produce_rows, warpgroups 1-2 tc::ring_tile).  The epilogue forms
//              d2~ = nrm2_i + nrm2_j - 2 g in fp64 and the band b of DESIGN section 4 (relative to |x_i||y_j| and to
//              (|x_i| + |y_j|)^2), and each row keeps in shared memory the S smallest lower bounds L = d2~ - b (rounded
//              down to fp32) with their columns, and L* = the smallest lower bound it dropped.  The four lanes holding a
//              row's columns insert in turn.  n x m is never formed.
//   recheck    a warp per row, a lane per kept column: the exact d2, a bitonic sort of the 32 (d2, column) pairs, E_k = the
//              k-th.  If L* > E_k every dropped column is strictly farther than the k chosen ones and the row is written;
//              otherwise it goes on the fallback list.
//   fallback   a CTA per listed row: the exact d2 to ALL m rows of y, each warp keeping the k smallest (d2, column) pairs
//              across its lanes, then warp 0 merges the eight lists.
//   Returns the number of rows that took the fallback in one 4-byte copy.
// K19 alq_cal_scores lse_r = m_r + log sum_c exp(z_rc - m_r) (c ascending, fp64) for the candidates and the references,
//              then a thread per (candidate, neighbour): KL(n || i) = sum_c p_nc (lp_nc - lp_ic), c ascending, with
//              lp = z - lse and p = exp(lp); the candidate's thread j = 0 adds the neighbours' KL in list order and divides by
//              their number.  key = -fl32(score) as K1b's ascending key, +0.0 for a zero and +NaN for a NaN score.
#include <math.h>

#include <algorithm>

#include "alq_rows_split.cuh"
#include "alq_wgmma.cuh"

namespace knn {

using tc::BK;
using tc::BM;
constexpr int S = 32;                           // lower bounds kept per row: one per lane of the recheck's warp
constexpr int K_MAX = 32;
constexpr double NRM2_MAX = 0x1p100;            // the band's derivation covers squared norms in [0, 2^100]

// ---- K18 ---------------------------------------------------------------------------------------------------------------
// s[i] = sqrt(nrm2[i]); rows whose nrm2 is NaN, infinite or above NRM2_MAX are counted in *bad
__global__ void __launch_bounds__(256) knn_norms_kernel(const double* __restrict__ nrm2, int n, double* __restrict__ s,
                                                        unsigned int* bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double v = nrm2[i];
    if (!(v <= NRM2_MAX)) atomicAdd(bad, 1u);
    s[i] = __dsqrt_rn(v);
}

struct ScreenParams {
    const double* nx;                  // [n] |x_i|^2
    const double* sx;                  // [n] |x_i|
    const double* ny;                  // [m] |y_j|^2
    const double* sy;                  // [m] |y_j|
    int n, m, ctiles, kblocks, rblocks;
    double coef;                       // per unit of |x_i||y_j|: twice the 3xTF32 bound (DESIGN section 4)
    double rel;                        // per unit of (|x_i| + |y_j|)^2: the fp64 epilogue, the norms, the exact sum
    double abs_;                       // per unit of 1 + |x_i| + |y_j|: underflow of the TF32 operands and products
    int* cand;                         // [n][S] the kept columns, -1 past min(S, m)
    float* lstar;                      // [n] the smallest dropped lower bound, +inf when none was dropped
};

// A row's kept lower bounds in shared memory (Ring::tail).  Each row belongs to one consumer warp.
struct Lists {
    float (*l)[S];                     // [BM][S]
    int (*c)[S];                       // [BM][S]
    float* thr;                        // [BM] the largest kept bound once S are kept, +inf before
    int* cnt;                          // [BM]
    int* at;                           // [BM] the position of thr
};
constexpr size_t LISTS_BYTES = static_cast<size_t>(BM) * S * 8 + BM * 12;

__device__ __forceinline__ Lists lists_at(unsigned char* tail) {
    Lists s;
    s.l = reinterpret_cast<float(*)[S]>(tail);
    s.c = reinterpret_cast<int(*)[S]>(tail + BM * S * 4);
    s.thr = reinterpret_cast<float*>(tail + BM * S * 8);
    s.cnt = reinterpret_cast<int*>(s.thr + BM);
    s.at = s.cnt + BM;
    return s;
}

// the position and value of the largest of a full list
__device__ __forceinline__ void lists_rescan(const Lists& s, int r) {
    float best = s.l[r][0];
    int at = 0;
#pragma unroll 4
    for (int q = 1; q < S; ++q)
        if (s.l[r][q] > best) { best = s.l[r][q]; at = q; }
    s.thr[r] = best;
    s.at[r] = at;
}

// offer (v, col) to row r's list; a bound that does not stay (v itself or the one it evicts) lowers ls
__device__ __forceinline__ void lists_offer(const Lists& s, int r, float v, int col, float& ls) {
    if (!(v < s.thr[r])) { ls = fminf(ls, v); return; }
    const int q = s.cnt[r];
    if (q < S) {
        s.l[r][q] = v;
        s.c[r][q] = col;
        s.cnt[r] = q + 1;
        if (q + 1 == S) lists_rescan(s, r);
        return;
    }
    const int a = s.at[r];
    ls = fminf(ls, s.l[r][a]);
    s.l[r][a] = v;
    s.c[r][a] = col;
    lists_rescan(s, r);
}

__global__ void __launch_bounds__(tc::THREADS, 1)
knn_screen_kernel(const __grid_constant__ CUtensorMap map_xhi, const __grid_constant__ CUtensorMap map_xlo,
                  const __grid_constant__ CUtensorMap map_yhi, const __grid_constant__ CUtensorMap map_ylo,
                  const ScreenParams P) {
    extern __shared__ unsigned char smem_dyn[];
    const tc::Role me = tc::ring_role();
    const tc::Ring ring = tc::ring_init(smem_dyn);

    if (me.wg == 0) {
        tc::producer_regs();
        if (threadIdx.x == 0) tc::ring_produce_rows(ring, &map_xhi, &map_xlo, &map_yhi, &map_ylo, P.rblocks, P.ctiles, P.kblocks);
        return;
    }
    tc::consumer_regs();
    const Lists L = lists_at(ring.tail);
    const int q4 = me.lane & 3;
    uint32_t it = 0;
    for (int rb = blockIdx.x; rb < P.rblocks; rb += gridDim.x) {
        const int row0 = rb * BM + me.r_in_tile;
        if (q4 == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                L.thr[me.r_in_tile + 8 * h] = INFINITY;
                L.cnt[me.r_in_tile + 8 * h] = 0;
            }
        }
        __syncwarp();
        double nr[2], sr[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = row0 + 8 * h;
            nr[h] = row < P.n ? __ldg(P.nx + row) : 0.0;
            sr[h] = row < P.n ? __ldg(P.sx + row) : 0.0;
        }
        float ls[2] = {INFINITY, INFINITY};
        for (int ct = 0; ct < P.ctiles; ++ct) {
            float acc[64];
            tc::ring_tile(ring, it, me, acc, P.kblocks);
            // acc becomes the lower bounds L, rounded down to fp32; columns past m get +inf and are never kept
            float lo = INFINITY;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = ct * BM + 8 * j + me.c_in_tile + e;
                    if (c >= P.m) {
                        acc[4 * j + e] = INFINITY;
                        acc[4 * j + 2 + e] = INFINITY;
                        continue;
                    }
                    const double nc = __ldg(P.ny + c), sc = __ldg(P.sy + c);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const double g = static_cast<double>(acc[4 * j + 2 * h + e]);
                        const double d2 = __dsub_rn(__dadd_rn(nr[h], nc), 2.0 * g);
                        const double t = __dadd_rn(sr[h], sc);
                        const double b = __dadd_rn(__dadd_rn(__dmul_rn(P.coef, __dmul_rn(sr[h], sc)),
                                                             __dmul_rn(P.rel, __dmul_rn(t, t))),
                                                   __dmul_rn(P.abs_, __dadd_rn(1.0, t)));
                        const float v = __double2float_rd(__dsub_rn(d2, b));
                        acc[4 * j + 2 * h + e] = v;
                        lo = fminf(lo, v);
                    }
                }
            }
            // the quad's lanes offer their columns in turn: the rows' lists see one writer at a time
            const bool mine = lo < fmaxf(L.thr[me.r_in_tile], L.thr[me.r_in_tile + 8]);
            if (__any_sync(0xffffffffu, mine)) {
                for (int turn = 0; turn < 4; ++turn) {
                    if (turn == q4) {
#pragma unroll 1
                        for (int h = 0; h < 2; ++h) {           // h stays a loop (selects, not indexing): one copy
                            const int r = me.r_in_tile + 8 * h;
                            float lh = h ? ls[1] : ls[0];
#pragma unroll
                            for (int j = 0; j < 16; ++j)
#pragma unroll
                                for (int e = 0; e < 2; ++e)
                                    lists_offer(L, r, h ? acc[4 * j + 2 + e] : acc[4 * j + e],
                                                ct * BM + 8 * j + me.c_in_tile + e, lh);
                            if (h) ls[1] = lh; else ls[0] = lh;
                        }
                    }
                    __syncwarp();
                }
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        ls[0] = fminf(ls[0], acc[4 * j + e]);
                        ls[1] = fminf(ls[1], acc[4 * j + 2 + e]);
                    }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            ls[h] = fminf(ls[h], __shfl_xor_sync(0xffffffffu, ls[h], 1));
            ls[h] = fminf(ls[h], __shfl_xor_sync(0xffffffffu, ls[h], 2));
            const int row = row0 + 8 * h, r = me.r_in_tile + 8 * h;
            if (row < P.n) {
                const int cnt = L.cnt[r];
                for (int q = q4; q < S; q += 4)
                    P.cand[static_cast<size_t>(row) * S + q] = q < cnt ? L.c[r][q] : -1;
                if (q4 == 0) P.lstar[row] = ls[h];
            }
        }
        __syncwarp();
    }
}

constexpr int RECHECK_WARPS = 8;
__global__ void __launch_bounds__(RECHECK_WARPS * 32)
knn_recheck_kernel(const float* __restrict__ x, const float* __restrict__ y, int n, int d, int k, const int* __restrict__ cand,
                   const float* __restrict__ lstar, int32_t* __restrict__ idx, double* __restrict__ d2, int* __restrict__ list,
                   unsigned int* listed) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * RECHECK_WARPS + (threadIdx.x >> 5);
    if (row >= n) return;
    const int c = cand[static_cast<size_t>(row) * S + lane];
    double e = INFINITY;
    int col = 0x7fffffff;
    if (c >= 0) {
        e = exact_d2(x + static_cast<size_t>(row) * d, y + static_cast<size_t>(c) * d, d);
        col = c;
    }
    // bitonic sort of the warp's (e, col) pairs, ascending
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1)
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            const double oe = __shfl_xor_sync(0xffffffffu, e, stride);
            const int oc = __shfl_xor_sync(0xffffffffu, col, stride);
            const bool keep_min = ((lane & size) == 0) == ((lane & stride) == 0);
            if (keep_min ? pair_less(oe, oc, e, col) : pair_less(e, col, oe, oc)) { e = oe; col = oc; }
        }
    const double ek = __shfl_sync(0xffffffffu, e, k - 1);
    const double ls = static_cast<double>(lstar[row]);
    if (ls == INFINITY || ls > ek) {                  // nothing dropped, or every dropped column lies beyond E_k
        if (lane < k) {
            idx[static_cast<size_t>(row) * k + lane] = e == INFINITY ? -1 : col;
            d2[static_cast<size_t>(row) * k + lane] = e;
        }
    } else if (lane == 0) {
        list[atomicAdd(listed, 1u)] = row;
    }
}

// (v, vc) into the warp's ascending list (lane l holds the l-th smallest pair)
__device__ __forceinline__ void pair_insert(double& le, int& lc, double v, int vc, int lane) {
    const int pos = __popc(__ballot_sync(0xffffffffu, pair_less(le, lc, v, vc)));
    const double ue = __shfl_up_sync(0xffffffffu, le, 1);
    const int uc = __shfl_up_sync(0xffffffffu, lc, 1);
    if (lane == pos) { le = v; lc = vc; }
    else if (lane > pos) { le = ue; lc = uc; }
}

// offer each lane's (v, vc) to the warp's list of the k smallest, lowest lane first
__device__ __forceinline__ void pair_offer(double& le, int& lc, double v, int vc, int k, int lane) {
    double te = __shfl_sync(0xffffffffu, le, k - 1);
    int tcol = __shfl_sync(0xffffffffu, lc, k - 1);
    unsigned int want = __ballot_sync(0xffffffffu, pair_less(v, vc, te, tcol));
    while (want) {
        const int src = __ffs(want) - 1;
        pair_insert(le, lc, __shfl_sync(0xffffffffu, v, src), __shfl_sync(0xffffffffu, vc, src), lane);
        te = __shfl_sync(0xffffffffu, le, k - 1);
        tcol = __shfl_sync(0xffffffffu, lc, k - 1);
        want &= ~(1u << src);
        want &= __ballot_sync(0xffffffffu, pair_less(v, vc, te, tcol));
    }
}

constexpr int FB_WARPS = 8;
__global__ void __launch_bounds__(FB_WARPS * 32)
knn_fallback_kernel(const float* __restrict__ x, const float* __restrict__ y, int m, int d, int k, const int* __restrict__ list,
                    const unsigned int* listed, int32_t* __restrict__ idx, double* __restrict__ d2) {
    __shared__ double se[FB_WARPS][32];
    __shared__ int sc[FB_WARPS][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int count = *listed;
    for (unsigned int w = blockIdx.x; w < count; w += gridDim.x) {
        const int row = list[w];
        const float* a = x + static_cast<size_t>(row) * d;
        double le = INFINITY;
        int lc = 0x7fffffff;
        for (int c0 = warp * 32; c0 < m; c0 += FB_WARPS * 32) {
            const int c = c0 + lane;
            const double v = c < m ? exact_d2(a, y + static_cast<size_t>(c) * d, d) : INFINITY;
            pair_offer(le, lc, v, c < m ? c : 0x7fffffff, k, lane);
        }
        se[warp][lane] = le;
        sc[warp][lane] = lc;
        __syncthreads();
        if (warp == 0) {
            for (int o = 1; o < FB_WARPS; ++o)
                pair_offer(le, lc, lane < k ? se[o][lane] : INFINITY, lane < k ? sc[o][lane] : 0x7fffffff, k, lane);
            if (lane < k) {
                idx[static_cast<size_t>(row) * k + lane] = le == INFINITY ? -1 : lc;
                d2[static_cast<size_t>(row) * k + lane] = le;
            }
        }
        __syncthreads();
    }
}

// ---- K19 ---------------------------------------------------------------------------------------------------------------
// lse[r] = m + log(sum_c exp(z_rc - m)), m = max_c z_rc, c ascending in fp64 (a thread per row)
__global__ void __launch_bounds__(256) cal_lse_kernel(const float* __restrict__ z, int rows, int C, double* __restrict__ lse) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    lse[r] = row_lse(z + static_cast<size_t>(r) * C, C);
}

constexpr int KL_THREADS = 256;
struct KlArgs {
    const float* zc;                   // [n][C] candidates' logits
    const float* zr;                   // [m][C] references' logits
    const double* lse_c;
    const double* lse_r;
    const int32_t* idx;                // [n][k]
    int n, m, C, k;
    double* score;
    float* key;
};

__global__ void __launch_bounds__(KL_THREADS) cal_kl_kernel(const KlArgs A) {
    __shared__ double kl[KL_THREADS];
    __shared__ unsigned char ok[KL_THREADS];
    const int rows = KL_THREADS / A.k;
    const int r = threadIdx.x / A.k, j = threadIdx.x % A.k;
    const int i = blockIdx.x * rows + r;
    const bool live = r < rows && i < A.n;
    double s = 0.0;
    bool valid = false;
    if (live) {
        const int nb = __ldg(A.idx + static_cast<size_t>(i) * A.k + j);
        valid = nb >= 0 && nb < A.m;
        if (valid) {
            const float* zn = A.zr + static_cast<size_t>(nb) * A.C;
            const float* zi = A.zc + static_cast<size_t>(i) * A.C;
            const double ln = __ldg(A.lse_r + nb), li = __ldg(A.lse_c + i);
            for (int c = 0; c < A.C; ++c) {
                const double lpn = __dsub_rn(static_cast<double>(__ldg(zn + c)), ln);
                const double lpi = __dsub_rn(static_cast<double>(__ldg(zi + c)), li);
                s = __dadd_rn(s, __dmul_rn(exp(lpn), __dsub_rn(lpn, lpi)));
            }
        }
    }
    kl[threadIdx.x] = s;
    ok[threadIdx.x] = valid;
    __syncthreads();
    if (live && j == 0) {
        double t = 0.0;
        int cnt = 0;
        for (int q = 0; q < A.k; ++q)
            if (ok[threadIdx.x + q]) { t = __dadd_rn(t, kl[threadIdx.x + q]); ++cnt; }
        const double sc = cnt ? __ddiv_rn(t, static_cast<double>(cnt)) : 0.0;
        const float f = __double2float_rn(sc);
        A.score[i] = sc;
        A.key[i] = sc != sc ? __int_as_float(0x7fffffff) : (f == 0.0f ? 0.0f : -f);
    }
}

}  // namespace knn

extern "C" int alq_knn(alq_ctx* ctx, const float* x, int64_t n, const float* y, int64_t m, int32_t d, int32_t k,
                       int32_t* idx, double* d2, int64_t* fallback_rows_host, void* stream) {
    using namespace knn;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_knn: n=%lld outside [1, 2^31)", (long long)n);
    if (m < 1 || m >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_knn: m=%lld outside [1, 2^31)", (long long)m);
    if (d < 4 || d % 4) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_knn: d=%d must be a positive multiple of 4", d);
    if (k < 1 || k > K_MAX) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_knn: k=%d outside [1, %d]", k, K_MAX);
    if (!x || !y || !idx || !d2 || !fallback_rows_host || !aligned16(x) || !aligned16(y))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_knn: null pointer or x / y not 16-byte aligned");
    if (!tc::get_encode()) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_knn: cuTensorMapEncodeTiled is unavailable");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n), mi = static_cast<int>(m);
    const size_t xe = static_cast<size_t>(n) * d, ye = static_cast<size_t>(m) * d;
    float *xhi, *xlo, *yhi, *ylo, *lstar;
    double *nx, *sx, *ny, *sy;
    int *cand, *list;
    unsigned int* cnt;                                      // [0] rows refused by their norm, [1] rows listed
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        xhi = cur.take<float>(xe);
        xlo = cur.take<float>(xe);
        yhi = cur.take<float>(ye);
        ylo = cur.take<float>(ye);
        nx = cur.take<double>(n);
        sx = cur.take<double>(n);
        ny = cur.take<double>(m);
        sy = cur.take<double>(m);
        cand = cur.take<int>(static_cast<size_t>(n) * S);
        lstar = cur.take<float>(n);
        list = cur.take<int>(n);
        cnt = cur.take<unsigned int>(2);
    });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaMemsetAsync(cnt, 0, 8, st));
    rs::normalize_split_kernel<<<(ni + rs::NORM_WARPS - 1) / rs::NORM_WARPS, rs::NORM_WARPS * 32, 0, st>>>(
        nullptr, ni, d, d, const_cast<float*>(x), xhi, xlo, nx, 0);
    ALQ_LAUNCH_CHECK(ctx);
    rs::normalize_split_kernel<<<(mi + rs::NORM_WARPS - 1) / rs::NORM_WARPS, rs::NORM_WARPS * 32, 0, st>>>(
        nullptr, mi, d, d, const_cast<float*>(y), yhi, ylo, ny, 0);
    ALQ_LAUNCH_CHECK(ctx);
    knn_norms_kernel<<<(ni + 255) / 256, 256, 0, st>>>(nx, ni, sx, cnt);
    ALQ_LAUNCH_CHECK(ctx);
    knn_norms_kernel<<<(mi + 255) / 256, 256, 0, st>>>(ny, mi, sy, cnt);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned int h[2] = {0u, 0u};
    ALQ_CUDA(ctx, cudaMemcpyAsync(h, cnt, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (h[0])
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_knn: %u rows have a squared norm that is not finite or exceeds 2^100", h[0]);

    CUtensorMap mxh, mxl, myh, myl;
    if (!tc::make_map(&mxh, xhi, n, d, BM) || !tc::make_map(&mxl, xlo, n, d, BM) || !tc::make_map(&myh, yhi, m, d, BM) ||
        !tc::make_map(&myl, ylo, m, d, BM))
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_knn: cuTensorMapEncodeTiled failed");
    ScreenParams P{};
    P.nx = nx; P.sx = sx; P.ny = ny; P.sy = sy;
    P.n = ni; P.m = mi; P.ctiles = (mi + BM - 1) / BM; P.kblocks = (d + BK - 1) / BK; P.rblocks = (ni + BM - 1) / BM;
    // DESIGN section 4: the fp64 roundings of the norms, of the epilogue and of the exact sum are < (2d + 13) 2^-53
    // (|x| + |y|)^2, of which the band takes twice; flushed or underflowing TF32 operands and products move 2g by
    // < 2^-118 d (1 + |x| + |y|), of which it takes 2^18 times.
    P.coef = tc::band_coef(d);
    P.rel = (4.0 * d + 32.0) * ldexp(1.0, -53);
    P.abs_ = d * ldexp(1.0, -100);
    P.cand = cand; P.lstar = lstar;
    const size_t smem = tc::ring_smem_bytes(LISTS_BYTES);
    ALQ_CUDA(ctx, cudaFuncSetAttribute(knn_screen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    knn_screen_kernel<<<std::min(ctx->sm_count, P.rblocks), tc::THREADS, smem, st>>>(mxh, mxl, myh, myl, P);
    ALQ_LAUNCH_CHECK(ctx);
    knn_recheck_kernel<<<(ni + RECHECK_WARPS - 1) / RECHECK_WARPS, RECHECK_WARPS * 32, 0, st>>>(
        x, y, ni, d, k, cand, lstar, idx, d2, list, cnt + 1);
    ALQ_LAUNCH_CHECK(ctx);
    knn_fallback_kernel<<<ctx->sm_count * 4, FB_WARPS * 32, 0, st>>>(x, y, mi, d, k, list, cnt + 1, idx, d2);
    ALQ_LAUNCH_CHECK(ctx);
    ALQ_CUDA(ctx, cudaMemcpyAsync(h + 1, cnt + 1, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    *fallback_rows_host = h[1];
    return ALQ_OK;
}

extern "C" int alq_cal_scores(alq_ctx* ctx, const float* cand_logits, int64_t n, const float* ref_logits, int64_t m,
                              int32_t c, const int32_t* idx, int32_t k, double* score, float* key, void* stream) {
    using namespace knn;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_cal_scores: n=%lld outside [1, 2^31)", (long long)n);
    if (m < 1 || m >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_cal_scores: m=%lld outside [1, 2^31)", (long long)m);
    if (c < 1) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_cal_scores: C=%d must be positive", c);
    if (k < 1 || k > K_MAX) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_cal_scores: k=%d outside [1, %d]", k, K_MAX);
    if (!cand_logits || !ref_logits || !idx || !score || !key) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_cal_scores: null pointer");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n), mi = static_cast<int>(m);
    double *lse_c, *lse_r;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        lse_c = cur.take<double>(n);
        lse_r = cur.take<double>(m);
    });
    if (rc) return rc;
    cal_lse_kernel<<<(ni + 255) / 256, 256, 0, st>>>(cand_logits, ni, c, lse_c);
    ALQ_LAUNCH_CHECK(ctx);
    cal_lse_kernel<<<(mi + 255) / 256, 256, 0, st>>>(ref_logits, mi, c, lse_r);
    ALQ_LAUNCH_CHECK(ctx);
    KlArgs A{};
    A.zc = cand_logits; A.zr = ref_logits; A.lse_c = lse_c; A.lse_r = lse_r; A.idx = idx;
    A.n = ni; A.m = mi; A.C = c; A.k = k; A.score = score; A.key = key;
    const int rows = KL_THREADS / k;
    cal_kl_kernel<<<(ni + rows - 1) / rows, KL_THREADS, 0, st>>>(A);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

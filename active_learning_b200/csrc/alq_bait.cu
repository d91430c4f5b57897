// K24-K26: BAITSampler (Ash, Goel, Krishnamurthy & Kakade, "Gone Fishing: Neural Active Learning with Fisher
// Embeddings", NeurIPS 2021) in fp64.  The NumPy statement is tests/bait_oracle.py.
//
// A row's Fisher embedding is V_x = R_x (x) h_x^T, R_x = diag(sqrt p_x)(I - 1 p_x^T), coordinate (c, d) at c D + d; it is
// never materialised.  dim = C D.
//   K24 alq_bait_fisher  p_x in fp64 (row_lse) and the weights w^ab_x = (diag p_x - p_x p_x^T)_ab / n; then F's blocks
//                        F_ab = H^T diag(w^ab) H for a <= b as fp64 tile products (one launch, a block per z), mirrored into
//                        an exactly symmetric dim x dim matrix.
//   K25 alq_bait_init    A = I / lamb; per row At_x = |h_x|^2 / lamb I and Gt_x[a, b] = h_x^T F_ab h_x / lamb^2 (T = H F_ab
//                        by the tile product over a chunk of rows, then a row contraction).
//   K26 alq_bait_select  the labeled rows absorbed, then the forward and backward passes.  A step is ordinary launches on
//                        one stream, the pick never leaving the device:
//     score   a warp per live row: M = s^2 R At R^T, G = s^2 R Gt R^T, Cholesky of I + sigma M, score = sigma tr(G (I +
//             sigma M)^-1) = tr(G (sigma I + M)^-1);
//     argmax  per CTA the best (score, lowest index into the row list); `pick` (one warp) reduces the partials, records
//             the pick and forms Sigma = (sigma I + M_*)^-1 and s R_*;
//     update  U = A Vt_*^T (a pass over A: y_c = A_{:, c} h_*, U = y (s R_*)^T), FU = F U (a pass over F), Q = U^T F U,
//             then one pass over A that forms P = A FU from the old rows and writes A - U Sigma U^T; [W | Z] = H [U | P]
//             (the tile product, the columns read as D x C^2 blocks); every row's forms:
//             At -= W Sigma W^T, Gt -= W Sigma Z^T + Z Sigma W^T - W Sigma Q Sigma W^T.
// Ties: (score, index) is a total order while the scores are not NaN (a failed Cholesky scores -inf and sets the status
// word), so every reduction order gives the lowest index of the largest score.
#include <math.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

#include "alq_common.cuh"

namespace bait {

constexpr int CMAX = 16;             // classes: the per-row C x C forms live in shared memory, C accumulators in registers
constexpr int TM = 64, TN = 64, TK = 16, GT = 256;   // tile product: 64 x 64 outputs, 16-deep k slabs, 4 x 4 per thread
constexpr int WARPS = 8;             // per-row kernels: a warp per row, 8 per CTA
constexpr int RPW = 2;               // dense passes: rows per warp
constexpr int RPC = RPW * WARPS;     // rows per CTA
constexpr int JCH = 256;             // dense passes: columns staged per round
constexpr int ARG_THREADS = 512;

struct Step {                        // what `pick` hands the update
    int row;                         // the pool row absorbed
    int status;                      // ALQ_ERR_NUMERIC once a Cholesky failed
    double sig[CMAX * CMAX];         // Sigma = (sigma I + M_*)^-1
    double rs[CMAX * CMAX];          // s R_*
};

// ---- the fp64 tile product ----------------------------------------------------------------------------------------------
// out(z, m, j) = sum over k ascending of a(z, m, k) * b(z, k, j) (one fma chain per output).  A loader's K_FAST says
// whether consecutive k are adjacent in memory (then a thread walks k), else consecutive m (or j) are.
template <class AL, class BL, class ST>
__global__ void __launch_bounds__(GT) tile_product(AL a, BL b, ST st, int M, int N, int K) {
    __shared__ double As[TK][TM + 1];
    __shared__ double Bs[TK][TN + 1];
    const int z = blockIdx.z;
    const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    for (int k0 = 0; k0 < K; k0 += TK) {
        for (int e = threadIdx.x; e < TK * TM; e += GT) {
            const int kk = AL::K_FAST ? e % TK : e / TM, mm = AL::K_FAST ? e / TK : e % TM;
            const int m = m0 + mm, k = k0 + kk;
            As[kk][mm] = (m < M && k < K) ? a(z, m, k) : 0.0;
        }
        for (int e = threadIdx.x; e < TK * TN; e += GT) {
            const int kk = BL::K_FAST ? e % TK : e / TN, jj = BL::K_FAST ? e / TK : e % TN;
            const int j = n0 + jj, k = k0 + kk;
            Bs[kk][jj] = (j < N && k < K) ? b(z, k, j) : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < TK; ++kk) {
            double av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = As[kk][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = Bs[kk][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + ty + 16 * i, jn = n0 + tx + 16 * j;
            if (m < M && jn < N) st(z, m, jn, acc[i][j]);
        }
}

template <class AL, class BL, class ST>
void launch_product(AL a, BL b, ST st, int M, int N, int K, int Z, cudaStream_t s) {
    const dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM, Z);
    tile_product<<<grid, GT, 0, s>>>(a, b, st, M, N, K);
}

__host__ __device__ inline void pair_of(int z, int C, int& a, int& b) {   // z -> (a, b), a <= b, row-major upper triangle
    a = 0;
    while (z >= C - a) { z -= C - a; ++a; }
    b = a + z;
}

// ---- K24: the Fisher ------------------------------------------------------------------------------------------------------
__global__ void fisher_prep_kernel(const float* __restrict__ logits, int64_t ldl, const float* __restrict__ emb, int n,
                                   int C, int D, double* __restrict__ p, double* __restrict__ w,
                                   unsigned int* __restrict__ bad) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= n) return;
    const float* zr = logits + static_cast<int64_t>(x) * ldl;
    bool ok = true;
    for (int c = 0; c < C; ++c) ok &= isfinite(__ldg(zr + c));
    const float* hr = emb + static_cast<int64_t>(x) * D;
    for (int d = 0; d < D; ++d) ok &= isfinite(__ldg(hr + d));
    if (!ok) atomicAdd(bad, 1u);
    const double lse = row_lse(zr, C);
    double pr[CMAX];
#pragma unroll
    for (int c = 0; c < CMAX; ++c)
        if (c < C) {
            pr[c] = exp(__dsub_rn(static_cast<double>(__ldg(zr + c)), lse));
            p[static_cast<int64_t>(x) * C + c] = pr[c];
        }
    const int np = C * (C + 1) / 2;
    int z = 0;
#pragma unroll
    for (int a = 0; a < CMAX; ++a)
#pragma unroll
        for (int b = 0; b < CMAX; ++b)
            if (a < C && b < C && b >= a) {
                const double v = (a == b ? pr[a] : 0.0) - pr[a] * pr[b];
                w[static_cast<int64_t>(x) * np + z] = v / n;
                ++z;
            }
}

struct HdLoad {          // (z, m = d, k = x) -> h[x, d]
    static constexpr bool K_FAST = false;
    const float* h;
    int D;
    __device__ double operator()(int, int m, int k) const { return static_cast<double>(__ldg(h + static_cast<int64_t>(k) * D + m)); }
};
struct WhLoad {          // (z, k = x, j = e) -> w^ab_x h[x, e]
    static constexpr bool K_FAST = false;
    const float* h;
    const double* w;
    int D, np;
    __device__ double operator()(int z, int k, int j) const {
        return w[static_cast<int64_t>(k) * np + z] * static_cast<double>(__ldg(h + static_cast<int64_t>(k) * D + j));
    }
};
struct FBlockStore {     // F[a D + m, b D + j] for the z-th pair (a, b)
    double* F;
    int C, D;
    __device__ void operator()(int z, int m, int j, double v) const {
        int a, b;
        pair_of(z, C, a, b);
        const int64_t dim = static_cast<int64_t>(C) * D;
        F[(static_cast<int64_t>(a) * D + m) * dim + static_cast<int64_t>(b) * D + j] = v;
    }
};

// F[j, i] = F[i, j] for i < j: 32 x 32 tiles through shared memory
__global__ void mirror_kernel(double* __restrict__ F, int64_t dim) {
    __shared__ double t[32][33];
    const int64_t bi = blockIdx.y, bj = blockIdx.x;
    if (bj < bi) return;
    const int64_t i0 = bi * 32, j0 = bj * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t i = i0 + r, j = j0 + threadIdx.x;
        t[r][threadIdx.x] = (i < dim && j < dim) ? F[i * dim + j] : 0.0;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t j = j0 + r, i = i0 + threadIdx.x;      // writes row j (> i) of the lower triangle
        if (i < dim && j < dim && i < j) F[j * dim + i] = t[threadIdx.x][r];
    }
}

// ---- K25: the initial forms --------------------------------------------------------------------------------------------
__global__ void eye_kernel(double* __restrict__ A, int64_t dim, double v) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e < dim * dim) A[e] = (e / dim == e % dim) ? v : 0.0;
}

struct HkLoad {          // (z, m = x, k = d) -> h[x0 + x, d]
    static constexpr bool K_FAST = true;
    const float* h;
    int D;
    __device__ double operator()(int, int m, int k) const { return static_cast<double>(__ldg(h + static_cast<int64_t>(m) * D + k)); }
};
struct FabLoad {         // (z, k = d, j = e) -> F[a D + d, b D + e]
    static constexpr bool K_FAST = false;
    const double* F;
    int64_t dim;
    int a, b, D;
    __device__ double operator()(int, int k, int j) const {
        return F[(static_cast<int64_t>(a) * D + k) * dim + static_cast<int64_t>(b) * D + j];
    }
};
struct RowStore {        // out[m, j] with leading dimension ld
    double* out;
    int64_t ld;
    __device__ void operator()(int, int m, int j, double v) const { out[static_cast<int64_t>(m) * ld + j] = v; }
};

// Gt_x[a, b] = Gt_x[b, a] = (sum over e ascending of h[x, e] T[x, e]) / lamb^2; with a == b also At_x = |h_x|^2 / lamb I
__global__ void contract_kernel(const float* __restrict__ h, const double* __restrict__ T, int rows, int D, int C, int a,
                                int b, double lamb, double* __restrict__ at, double* __restrict__ gt) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= rows) return;
    const float* hr = h + static_cast<int64_t>(x) * D;
    const double* tr = T + static_cast<int64_t>(x) * D;
    double s = 0.0;
    for (int e = 0; e < D; ++e) s = fma(static_cast<double>(__ldg(hr + e)), tr[e], s);
    const int64_t cc = static_cast<int64_t>(C) * C;
    const double g = s / (lamb * lamb);
    gt[x * cc + a * C + b] = g;
    gt[x * cc + b * C + a] = g;
    if (a == 0 && b == 0) {
        double nn = 0.0;
        for (int e = 0; e < D; ++e) {
            const double v = static_cast<double>(__ldg(hr + e));
            nn = fma(v, v, nn);
        }
        const double d = nn / lamb;
        for (int i = 0; i < C; ++i)
            for (int j = 0; j < C; ++j) at[x * cc + i * C + j] = i == j ? d : 0.0;
    }
}

// ---- K26: small dense algebra of one warp on C x C matrices in shared memory (row-major, C <= CMAX) --------------------
// R X R^T for R = diag(sqrt p)(I - 1 p^T): (X[k, l] - (X p)_k - (p^T X)_l + p^T X p) sqrt(p_k p_l), times s2
__device__ void sandwich(const double* X, const double* p, int C, double s2, double* out, double* tmp) {
    const int l = threadIdx.x & 31;
    if (l < C) {                                     // tmp[0..C) = X p, tmp[C..2C) = p^T X
        double u = 0.0, v = 0.0;
        for (int j = 0; j < C; ++j) {
            u = fma(X[l * C + j], p[j], u);
            v = fma(p[j], X[j * C + l], v);
        }
        tmp[l] = u;
        tmp[C + l] = v;
    }
    __syncwarp();
    double c0 = 0.0;
    for (int j = 0; j < C; ++j) c0 = fma(p[j], tmp[j], c0);
    for (int e = l; e < C * C; e += 32) {
        const int k = e / C, m = e % C;
        out[e] = s2 * (((X[e] - tmp[k]) - tmp[C + m]) + c0) * sqrt(p[k] * p[m]);
    }
    __syncwarp();
}

// In place: B (C x C, symmetric positive definite) -> its Cholesky factor L (lower triangle).  false if a pivot is not > 0.
__device__ bool cholesky(double* B, int C) {
    const int l = threadIdx.x & 31;
    bool ok = true;
    for (int j = 0; j < C; ++j) {
        double djj = B[j * C + j];
        for (int k = 0; k < j; ++k) djj -= B[j * C + k] * B[j * C + k];
        ok &= djj > 0.0;                             // also false for NaN
        const double ljj = sqrt(fmax(djj, 0.0));
        __syncwarp();
        if (l > j && l < C) {
            double v = B[l * C + j];
            for (int k = 0; k < j; ++k) v -= B[l * C + k] * B[j * C + k];
            B[l * C + j] = v / ljj;
        }
        if (l == j) B[j * C + j] = ljj;
        __syncwarp();
    }
    return ok;
}

// Z = (L L^T)^-1 G column by column (lane j solves column j); Z may alias G
__device__ void chol_solve(const double* L, const double* G, double* Z, int C) {
    const int j = threadIdx.x & 31;
    if (j < C) {
        for (int i = 0; i < C; ++i) {                // L y = g
            double v = G[i * C + j];
            for (int k = 0; k < i; ++k) v -= L[i * C + k] * Z[k * C + j];
            Z[i * C + j] = v / L[i * C + i];
        }
        for (int i = C - 1; i >= 0; --i) {           // L^T z = y
            double v = Z[i * C + j];
            for (int k = i + 1; k < C; ++k) v -= L[k * C + i] * Z[k * C + j];
            Z[i * C + j] = v / L[i * C + i];
        }
    }
    __syncwarp();
}

__device__ __forceinline__ bool better(double g, int p, double bg, int bp) { return g > bg || (g == bg && p < bp); }

__device__ __forceinline__ void warp_best(double& g, int& p) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double og = __shfl_xor_sync(0xffffffffu, g, o);
        const int op = __shfl_xor_sync(0xffffffffu, p, o);
        if (better(og, op, g, p)) { g = og; p = op; }
    }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// per-warp scratch of the score: B, G, tmp (2C) and p
constexpr int SCORE_WARP_DOUBLES = 2 * CMAX * CMAX + 3 * CMAX;

// score[i] for every live entry i of rows[0..m)
__global__ void __launch_bounds__(32 * WARPS) score_kernel(const int* __restrict__ rows, const uint8_t* __restrict__ live,
                                                           int m, const double* __restrict__ p,
                                                           const double* __restrict__ at, const double* __restrict__ gt,
                                                           int C, double s2, double sigma, double* __restrict__ score,
                                                           Step* __restrict__ step) {
    extern __shared__ double sm[];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    double* Bm = sm + w * SCORE_WARP_DOUBLES;
    double* Gm = Bm + CMAX * CMAX;
    double* tmp = Gm + CMAX * CMAX;
    double* pr = tmp + 2 * CMAX;
    const int i = blockIdx.x * WARPS + w;
    if (i >= m || !live[i]) return;                  // warp-uniform
    const int64_t x = rows[i];
    const int64_t cc = static_cast<int64_t>(C) * C;
    if (l < C) pr[l] = p[x * C + l];
    __syncwarp();
    sandwich(at + x * cc, pr, C, s2 * sigma, Bm, tmp);
    for (int e = l; e < C * C; e += 32)
        if (e / C == e % C) Bm[e] += 1.0;            // B = I + sigma M
    sandwich(gt + x * cc, pr, C, s2, Gm, tmp);
    __syncwarp();
    const bool ok = cholesky(Bm, C);
    double tr = -INFINITY;
    if (ok) {
        chol_solve(Bm, Gm, Gm, C);
        double v = l < C ? Gm[l * C + l] : 0.0;
        tr = sigma * warp_sum_d(v);                  // the butterfly: every lane holds the same sum
    } else if (l == 0) {
        step->status = ALQ_ERR_NUMERIC;
    }
    if (l == 0) score[i] = tr;
}

__global__ void __launch_bounds__(ARG_THREADS) argmax_kernel(const double* __restrict__ score,
                                                             const uint8_t* __restrict__ live, int m,
                                                             double* __restrict__ part_g, int* __restrict__ part_p) {
    __shared__ double sg[32];
    __shared__ int sp[32];
    double g = -INFINITY;
    int p = INT_MAX;
    for (int i = blockIdx.x * ARG_THREADS + threadIdx.x; i < m; i += gridDim.x * ARG_THREADS)
        if (live[i] && better(score[i], i, g, p)) { g = score[i]; p = i; }
    warp_best(g, p);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { sg[w] = g; sp[w] = p; }
    __syncthreads();
    if (w == 0) {
        g = l < ARG_THREADS / 32 ? sg[l] : -INFINITY;
        p = l < ARG_THREADS / 32 ? sp[l] : INT_MAX;
        warp_best(g, p);
        if (l == 0) { part_g[blockIdx.x] = g; part_p[blockIdx.x] = p; }
    }
}

// One warp.  fixed >= 0: absorb rows[fixed]; otherwise the best of the partials.  Records the pick, then forms Sigma and
// s R_* of the row.
__global__ void pick_kernel(const int* __restrict__ rows, uint8_t* __restrict__ live, int fixed,
                            const double* __restrict__ part_g, const int* __restrict__ part_p, int n_part,
                            const double* __restrict__ p, const double* __restrict__ at, int C, double s, double sigma,
                            int* __restrict__ list, int list_at, double* __restrict__ scores, int score_at,
                            Step* __restrict__ step) {
    __shared__ double Bm[CMAX * CMAX], Z[CMAX * CMAX], tmp[2 * CMAX], pr[CMAX];
    const int l = threadIdx.x;
    int idx = fixed;
    if (fixed < 0) {
        double g = -INFINITY;
        int q = INT_MAX;
        for (int b = l; b < n_part; b += 32)
            if (better(part_g[b], part_p[b], g, q)) { g = part_g[b]; q = part_p[b]; }
        warp_best(g, q);
        idx = q;
        if (l == 0 && scores) scores[score_at] = g;
    }
    if (idx < 0 || idx == INT_MAX) {                 // nothing live: cannot happen for a valid step count
        if (l == 0) step->status = ALQ_ERR_NUMERIC;
        return;
    }
    const int64_t x = rows[idx];
    if (l == 0) {
        live[idx] = 0;
        step->row = static_cast<int>(x);
        if (list) list[list_at] = static_cast<int>(x);
    }
    if (l < C) pr[l] = p[x * C + l];
    __syncwarp();
    sandwich(at + x * static_cast<int64_t>(C) * C, pr, C, s * s * sigma, Bm, tmp);
    for (int e = l; e < C * C; e += 32) {
        const int k = e / C, c = e % C;
        if (k == c) Bm[e] += 1.0;
        Z[e] = k == c ? 1.0 : 0.0;
        step->rs[e] = s * sqrt(pr[k]) * ((k == c ? 1.0 : 0.0) - pr[c]);
    }
    __syncwarp();
    if (!cholesky(Bm, C) && l == 0) step->status = ALQ_ERR_NUMERIC;
    chol_solve(Bm, Z, Z, C);
    for (int e = l; e < C * C; e += 32) step->sig[e] = sigma * Z[e];
}

// U[i, k] = sum_c (s R_*)[k, c] y_c, y_c = sum_d A[i, c D + d] h_*[d]: a warp per row of A
__global__ void __launch_bounds__(32 * WARPS) u_kernel(const double* __restrict__ A, int64_t dim, int C, int D,
                                                       const float* __restrict__ emb, const Step* __restrict__ step,
                                                       double* __restrict__ U) {
    const int l = threadIdx.x & 31;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * WARPS + (threadIdx.x >> 5);
    if (i >= dim) return;
    const float* hs = emb + static_cast<int64_t>(step->row) * D;
    const double* ar = A + i * dim;
    double y[CMAX];
#pragma unroll
    for (int c = 0; c < CMAX; ++c) {
        y[c] = 0.0;
        if (c < C) {
            double v = 0.0;
            for (int d = l; d < D; d += 32) v = fma(ar[static_cast<int64_t>(c) * D + d], static_cast<double>(__ldg(hs + d)), v);
            y[c] = warp_sum_d(v);
        }
    }
    if (l < C) {
        double u = 0.0;
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < C) u = fma(step->rs[l * C + c], y[c], u);
        U[i * C + l] = u;
    }
}

// A pass over the rows of a dense dim x dim matrix X, RPC rows per CTA, the columns staged JCH at a time:
//   out[i, k] = sum_j X[i, j] V[j, k] (V dim x C), and with `upd` also X[i, j] -= sum_k (U Sigma)[i, k] U[j, k] (after
//   the row's products read it).  Dynamic shared memory: 2 C JCH doubles.
template <bool UPD>
__global__ void __launch_bounds__(32 * WARPS) dense_pass_kernel(double* __restrict__ X, int64_t dim, int C,
                                                                const double* __restrict__ V, double* __restrict__ out,
                                                                const double* __restrict__ U,
                                                                const Step* __restrict__ step) {
    extern __shared__ double sm[];
    double* Vs = sm;                                 // [C][JCH]
    double* Us = sm + static_cast<size_t>(C) * JCH;  // [C][JCH]
    __shared__ double us[RPC][CMAX];                 // (U Sigma)[i, :] of this CTA's rows
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const int64_t r0 = static_cast<int64_t>(blockIdx.x) * RPC;
    if (UPD) {
        for (int e = threadIdx.x; e < RPC * CMAX; e += blockDim.x) {
            const int r = e / CMAX, k = e % CMAX;
            double v = 0.0;
            if (k < C && r0 + r < dim)
                for (int q = 0; q < C; ++q) v = fma(U[(r0 + r) * C + q], step->sig[q * C + k], v);
            us[r][k] = v;
        }
    }
    double acc[RPW][CMAX];
#pragma unroll
    for (int r = 0; r < RPW; ++r)
#pragma unroll
        for (int k = 0; k < CMAX; ++k) acc[r][k] = 0.0;
    for (int64_t j0 = 0; j0 < dim; j0 += JCH) {
        const int len = static_cast<int>(dim - j0 < JCH ? dim - j0 : JCH);
        __syncthreads();
        for (int e = threadIdx.x; e < C * JCH; e += blockDim.x) {
            const int k = e / JCH, j = e % JCH;
            Vs[e] = j < len ? V[(j0 + j) * C + k] : 0.0;
            if (UPD) Us[e] = j < len ? U[(j0 + j) * C + k] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < RPW; ++r) {
            const int64_t i = r0 + w * RPW + r;
            if (i >= dim) continue;
            double* xr = X + i * dim + j0;
            for (int j = l; j < len; j += 32) {
                const double xv = xr[j];
                double dv = 0.0;
#pragma unroll
                for (int k = 0; k < CMAX; ++k)
                    if (k < C) {
                        acc[r][k] = fma(xv, Vs[k * JCH + j], acc[r][k]);
                        if (UPD) dv = fma(us[w * RPW + r][k], Us[k * JCH + j], dv);
                    }
                if (UPD) xr[j] = xv - dv;
            }
        }
    }
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
        const int64_t i = r0 + w * RPW + r;
#pragma unroll
        for (int k = 0; k < CMAX; ++k)
            if (k < C) {
                const double v = warp_sum_d(acc[r][k]);
                if (l == 0 && i < dim) out[i * C + k] = v;
            }
    }
}

// Q[k, l] = sum_i U[i, k] FU[i, l]: one CTA, a warp per entry
__global__ void q_kernel(const double* __restrict__ U, const double* __restrict__ FU, int64_t dim, int C,
                         double* __restrict__ Q) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int e = w; e < C * C; e += nw) {
        const int k = e / C, m = e % C;
        double v = 0.0;
        for (int64_t i = l; i < dim; i += 32) v = fma(U[i * C + k], FU[i * C + m], v);
        v = warp_sum_d(v);
        if (l == 0) Q[e] = v;
    }
}

struct WzLoad {          // (z, k = d, j) -> U or P at row (a D + d), column k', j = which C^2 + a C + k'
    static constexpr bool K_FAST = false;
    const double* U;
    const double* P;
    int C, D;
    __device__ double operator()(int, int k, int j) const {
        const int cc = C * C;
        const double* src = j < cc ? U : P;
        const int r = j < cc ? j : j - cc;
        const int a = r / C, q = r % C;
        return src[(static_cast<int64_t>(a) * D + k) * C + q];
    }
};

// per-warp scratch of the form update: W, Z, S1 = W Sigma, T = S1 Q
constexpr int FORM_WARP_DOUBLES = 4 * CMAX * CMAX;

// every row's forms: At -= S1 W^T, Gt -= S1 Z^T + Z S1^T - S1 Q S1^T
__global__ void __launch_bounds__(32 * WARPS) forms_kernel(const double* __restrict__ wz, int n, int C,
                                                           const double* __restrict__ Q, const Step* __restrict__ step,
                                                           double* __restrict__ at, double* __restrict__ gt) {
    extern __shared__ double sm[];
    __shared__ double sig[CMAX * CMAX], qs[CMAX * CMAX];
    const int cc = C * C;
    for (int e = threadIdx.x; e < cc; e += blockDim.x) {
        sig[e] = step->sig[e];
        qs[e] = Q[e];
    }
    __syncthreads();
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const int64_t x = static_cast<int64_t>(blockIdx.x) * WARPS + w;
    if (x >= n) return;
    double* W = sm + w * FORM_WARP_DOUBLES;
    double* Z = W + CMAX * CMAX;
    double* S1 = Z + CMAX * CMAX;
    double* T = S1 + CMAX * CMAX;
    const double* src = wz + x * 2 * cc;
    for (int e = l; e < cc; e += 32) {
        W[e] = src[e];
        Z[e] = src[cc + e];
    }
    __syncwarp();
    for (int e = l; e < cc; e += 32) {
        const int a = e / C, k = e % C;
        double v = 0.0;
        for (int q = 0; q < C; ++q) v = fma(W[a * C + q], sig[q * C + k], v);
        S1[e] = v;
    }
    __syncwarp();
    for (int e = l; e < cc; e += 32) {
        const int a = e / C, k = e % C;
        double v = 0.0;
        for (int q = 0; q < C; ++q) v = fma(S1[a * C + q], qs[q * C + k], v);
        T[e] = v;
    }
    __syncwarp();
    double* ar = at + x * cc;
    double* gr = gt + x * cc;
    for (int e = l; e < cc; e += 32) {
        const int a = e / C, b = e % C;
        double sw = 0.0, sz = 0.0, zs = 0.0, tt = 0.0;
        for (int q = 0; q < C; ++q) {
            sw = fma(S1[a * C + q], W[b * C + q], sw);
            sz = fma(S1[a * C + q], Z[b * C + q], sz);
            zs = fma(Z[a * C + q], S1[b * C + q], zs);
            tt = fma(T[a * C + q], S1[b * C + q], tt);
        }
        ar[e] -= sw;
        gr[e] = gr[e] - sz - zs + tt;
    }
}

bool shapes_ok(int64_t n, int32_t c, int32_t d) {
    return n >= 1 && n < (1LL << 31) && c >= 2 && c <= CMAX && d >= 1 && static_cast<int64_t>(c) * d < (1LL << 31) / 32;
}

}  // namespace bait

extern "C" int alq_bait_fisher(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ldl, const float* emb,
                               int32_t d, double* p, double* fisher, void* stream) {
    using namespace bait;
    if (!ctx) return ALQ_ERR_INVALID;
    if (!logits || !emb || !p || !fisher || !shapes_ok(n, c, d) || ldl < c)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_bait_fisher: bad arguments (n=%lld C=%d D=%d ldl=%lld; 2 <= C <= %d)",
                 (long long)n, c, d, (long long)ldl, CMAX);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n), np = c * (c + 1) / 2;
    const int64_t dim = static_cast<int64_t>(c) * d;
    double* w;
    unsigned int* bad;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        w = cur.take<double>(static_cast<size_t>(n) * np);
        bad = cur.take<unsigned int>(1);
    });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    ALQ_CUDA(ctx, cudaMemsetAsync(bad, 0, 4, st));
    fisher_prep_kernel<<<(ni + 255) / 256, 256, 0, st>>>(logits, ldl, emb, ni, c, d, p, w, bad);
    ALQ_LAUNCH_CHECK(ctx);
    launch_product(HdLoad{emb, d}, WhLoad{emb, w, d, np}, FBlockStore{fisher, c, d}, d, d, ni, np, st);
    ALQ_LAUNCH_CHECK(ctx);
    const int nt = static_cast<int>((dim + 31) / 32);
    mirror_kernel<<<dim3(nt, nt), dim3(32, 8), 0, st>>>(fisher, dim);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned int h = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h, bad, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (h) ALQ_FAIL(ctx, ALQ_ERR_NUMERIC, "alq_bait_fisher: %u rows hold a NaN or infinite logit or embedding entry", h);
    return ALQ_OK;
}

extern "C" int alq_bait_init(alq_ctx* ctx, const float* emb, int64_t n, int32_t c, int32_t d, const double* fisher,
                             const double* lamb_host, double* a, double* at, double* gt, void* stream) {
    using namespace bait;
    if (!ctx) return ALQ_ERR_INVALID;
    if (!emb || !fisher || !lamb_host || !a || !at || !gt || !shapes_ok(n, c, d) || !std::isfinite(*lamb_host) ||
        !(*lamb_host > 0))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_bait_init: bad arguments (n=%lld C=%d D=%d lamb=%g)", (long long)n, c, d,
                 lamb_host ? *lamb_host : 0.0);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const double lamb = *lamb_host;
    const int64_t dim = static_cast<int64_t>(c) * d;
    // T = H F_ab over a chunk of rows at a time: at most dim^2 doubles (the memory rule's scratch), at least 64 rows
    const int chunk = static_cast<int>(std::min<int64_t>(n, std::max<int64_t>(64, dim * dim / d)));
    double* T;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) { T = cur.take<double>(static_cast<size_t>(chunk) * d); });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    eye_kernel<<<static_cast<unsigned>((dim * dim + 255) / 256), 256, 0, st>>>(a, dim, 1.0 / lamb);
    ALQ_LAUNCH_CHECK(ctx);
    const int64_t cc = static_cast<int64_t>(c) * c;
    for (int64_t x0 = 0; x0 < n; x0 += chunk) {
        const int rows = static_cast<int>(std::min<int64_t>(chunk, n - x0));
        const float* h0 = emb + x0 * d;
        for (int a_ = 0; a_ < c; ++a_)
            for (int b_ = a_; b_ < c; ++b_) {
                launch_product(HkLoad{h0, d}, FabLoad{fisher, dim, a_, b_, d}, RowStore{T, d}, rows, d, d, 1, st);
                ALQ_LAUNCH_CHECK(ctx);
                contract_kernel<<<(rows + 255) / 256, 256, 0, st>>>(h0, T, rows, d, c, a_, b_, lamb, at + x0 * cc,
                                                                    gt + x0 * cc);
                ALQ_LAUNCH_CHECK(ctx);
            }
    }
    return ALQ_OK;
}

extern "C" int alq_bait_select(alq_ctx* ctx, const float* emb, const double* p, int64_t n, int32_t c, int32_t d,
                               const double* fisher, double* a, double* at, double* gt, const int32_t* lab_pos,
                               int64_t n_lab, const int32_t* cand_pos, int64_t n_cand, int64_t budget, int32_t* picks,
                               int64_t* n_picks_host, int32_t* fwd_list, double* fwd_scores, double* bwd_scores,
                               float* phase_ms_host, void* stream) {
    using namespace bait;
    if (!ctx) return ALQ_ERR_INVALID;
    if (!emb || !p || !fisher || !a || !at || !gt || !picks || !n_picks_host || !shapes_ok(n, c, d) || n_lab < 0 ||
        n_cand < 0 || n_lab + n_cand > n || (n_lab && !lab_pos) || (n_cand && !cand_pos) || budget < 0 ||
        budget > n_cand)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID,
                 "alq_bait_select: bad arguments (n=%lld C=%d D=%d labeled=%lld candidates=%lld budget=%lld)",
                 (long long)n, c, d, (long long)n_lab, (long long)n_cand, (long long)budget);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    const int64_t dim = static_cast<int64_t>(c) * d;
    const int cc = c * c;
    const int T = static_cast<int>(std::min<int64_t>(2 * budget, n_cand));
    const int mc = static_cast<int>(n_cand);
    const int n_part = std::max(1, std::min(ctx->sm_count, (mc + ARG_THREADS - 1) / ARG_THREADS));
    const int n_rows = static_cast<int>(std::max<int64_t>(std::max<int64_t>(n_cand, n_lab), 1));   // the row lists
    double *score, *part_g, *U, *FU, *P, *Q, *wz;
    int *part_p, *rows, *list;
    uint8_t* live;
    Step* step;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        score = cur.take<double>(std::max(mc, 1));
        part_g = cur.take<double>(n_part);
        part_p = cur.take<int>(n_part);
        rows = cur.take<int>(n_rows);
        live = cur.take<uint8_t>(n_rows);
        list = cur.take<int>(std::max(T, 1));
        U = cur.take<double>(dim * c);
        FU = cur.take<double>(dim * c);
        P = cur.take<double>(dim * c);
        Q = cur.take<double>(cc);
        wz = cur.take<double>(static_cast<size_t>(n) * 2 * cc);
        step = cur.take<Step>(1);
    });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    ALQ_CUDA(ctx, cudaMemsetAsync(step, 0, sizeof(Step), st));

    const double s_lab = 1.0 / std::sqrt(static_cast<double>(n_lab + budget));
    const double s_f = std::sqrt(static_cast<double>(budget) / static_cast<double>(n_lab + budget));
    const unsigned dense_grid = static_cast<unsigned>((dim + RPC - 1) / RPC);
    const size_t dense_smem = 2 * static_cast<size_t>(c) * JCH * sizeof(double);
    const unsigned warp_grid_n = static_cast<unsigned>((n + WARPS - 1) / WARPS);
    const size_t form_smem = WARPS * FORM_WARP_DOUBLES * sizeof(double);
    const size_t score_smem = WARPS * SCORE_WARP_DOUBLES * sizeof(double);
    ALQ_CUDA(ctx, cudaFuncSetAttribute(dense_pass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(dense_smem)));
    ALQ_CUDA(ctx, cudaFuncSetAttribute(dense_pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(dense_smem)));
    ALQ_CUDA(ctx, cudaFuncSetAttribute(forms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(form_smem)));

    // the rank-C update by the row `pick` recorded
    auto update = [&]() -> int {
        u_kernel<<<static_cast<unsigned>((dim + WARPS - 1) / WARPS), 32 * WARPS, 0, st>>>(a, dim, c, d, emb, step, U);
        ALQ_LAUNCH_CHECK(ctx);
        dense_pass_kernel<false><<<dense_grid, 32 * WARPS, dense_smem, st>>>(const_cast<double*>(fisher), dim, c, U, FU,
                                                                              nullptr, step);
        ALQ_LAUNCH_CHECK(ctx);
        q_kernel<<<1, 1024, 0, st>>>(U, FU, dim, c, Q);
        ALQ_LAUNCH_CHECK(ctx);
        dense_pass_kernel<true><<<dense_grid, 32 * WARPS, dense_smem, st>>>(a, dim, c, FU, P, U, step);
        ALQ_LAUNCH_CHECK(ctx);
        launch_product(HkLoad{emb, d}, WzLoad{U, P, c, d}, RowStore{wz, 2 * cc}, ni, 2 * cc, d, 1, st);
        ALQ_LAUNCH_CHECK(ctx);
        forms_kernel<<<warp_grid_n, 32 * WARPS, form_smem, st>>>(wz, ni, c, Q, step, at, gt);
        ALQ_LAUNCH_CHECK(ctx);
        return ALQ_OK;
    };
    // one scored step over rows[0..m): score, argmax, pick; the update unless it is the last
    auto scored = [&](int m, double sigma, int* to_list, int list_at, double* scores, int score_at, bool upd) -> int {
        score_kernel<<<static_cast<unsigned>((m + WARPS - 1) / WARPS), 32 * WARPS, score_smem, st>>>(
            rows, live, m, p, at, gt, c, s_f * s_f, sigma, score, step);
        ALQ_LAUNCH_CHECK(ctx);
        const int np_ = std::max(1, std::min(n_part, (m + ARG_THREADS - 1) / ARG_THREADS));
        argmax_kernel<<<np_, ARG_THREADS, 0, st>>>(score, live, m, part_g, part_p);
        ALQ_LAUNCH_CHECK(ctx);
        pick_kernel<<<1, 32, 0, st>>>(rows, live, -1, part_g, part_p, np_, p, at, c, s_f, sigma, to_list, list_at,
                                      scores, score_at, step);
        ALQ_LAUNCH_CHECK(ctx);
        return upd ? update() : ALQ_OK;
    };

    // phase_ms_host: events around the absorption, the forward and the backward pass
    cudaEvent_t ev[4] = {};
    if (phase_ms_host)
        for (auto& e : ev) ALQ_CUDA(ctx, cudaEventCreate(&e));
    struct Events {
        cudaEvent_t* e;
        ~Events() {
            for (int i = 0; i < 4; ++i)
                if (e[i]) cudaEventDestroy(e[i]);
        }
    } guard{ev};
    auto mark = [&](int i) -> int {
        if (phase_ms_host) ALQ_CUDA(ctx, cudaEventRecord(ev[i], st));
        return ALQ_OK;
    };
    if ((rc = mark(0))) return rc;
    // the labeled rows, in the order given
    if (n_lab) {
        ALQ_CUDA(ctx, cudaMemcpyAsync(rows, lab_pos, static_cast<size_t>(n_lab) * 4, cudaMemcpyDeviceToDevice, st));
        for (int t = 0; t < n_lab; ++t) {
            pick_kernel<<<1, 32, 0, st>>>(rows, live, t, nullptr, nullptr, 0, p, at, c, s_lab, 1.0, nullptr, 0, nullptr,
                                          0, step);
            ALQ_LAUNCH_CHECK(ctx);
            if ((rc = update())) return rc;
        }
    }
    if ((rc = mark(1))) return rc;
    // forward: T picks among the candidates (ascending positions: the lowest index is the lowest position)
    if (T > 0) {
        ALQ_CUDA(ctx, cudaMemcpyAsync(rows, cand_pos, static_cast<size_t>(mc) * 4, cudaMemcpyDeviceToDevice, st));
        ALQ_CUDA(ctx, cudaMemsetAsync(live, 1, mc, st));
        for (int t = 0; t < T; ++t)
            if ((rc = scored(mc, 1.0, list, t, fwd_scores, t, t + 1 < T || T > budget))) return rc;
    }
    if ((rc = mark(2))) return rc;
    // backward: T - B removals from the list, in list order
    const int nb = T - static_cast<int>(budget);
    if (nb > 0) {
        ALQ_CUDA(ctx, cudaMemcpyAsync(rows, list, static_cast<size_t>(T) * 4, cudaMemcpyDeviceToDevice, st));
        ALQ_CUDA(ctx, cudaMemsetAsync(live, 1, T, st));
        for (int t = 0; t < nb; ++t)
            if ((rc = scored(T, -1.0, nullptr, 0, bwd_scores, t, t + 1 < nb))) return rc;
    }
    if ((rc = mark(3))) return rc;
    std::vector<int> h_list(std::max(T, 1));
    std::vector<uint8_t> h_live(std::max(T, 1), 1);
    int h_status = 0;
    if (T > 0) ALQ_CUDA(ctx, cudaMemcpyAsync(h_list.data(), list, static_cast<size_t>(T) * 4, cudaMemcpyDeviceToHost, st));
    if (T > 0 && fwd_list)
        ALQ_CUDA(ctx, cudaMemcpyAsync(fwd_list, list, static_cast<size_t>(T) * 4, cudaMemcpyDeviceToDevice, st));
    if (nb > 0) ALQ_CUDA(ctx, cudaMemcpyAsync(h_live.data(), live, T, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h_status, &step->status, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (h_status)
        ALQ_FAIL(ctx, ALQ_ERR_NUMERIC, "alq_bait_select: a C x C Cholesky factorisation met a pivot that is not > 0");
    if (phase_ms_host)
        for (int i = 0; i < 3; ++i) ALQ_CUDA(ctx, cudaEventElapsedTime(phase_ms_host + i, ev[i], ev[i + 1]));
    std::vector<int> out;
    for (int i = 0; i < T; ++i)
        if (h_live[i]) out.push_back(h_list[i]);
    if (!out.empty())
        ALQ_CUDA(ctx, cudaMemcpy(picks, out.data(), out.size() * 4, cudaMemcpyHostToDevice));
    *n_picks_host = static_cast<int64_t>(out.size());
    return ALQ_OK;
}

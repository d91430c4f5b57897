// K20: ALFAMixSampler (Parvaneh, Abbasnejad, Teney, Haffari, van den Hengel & Shi, "Active Learning by Feature Mixing",
// CVPR 2022) on the device: the closed-form feature-mixing test with the algebra carried out, one number per row.
//
// K20 alq_alfamix_rho   for every candidate row u (logits l_u [C], raw embedding z_u [Dp]) against the head W [C, D] and
//                       the class anchors a_c [C, Dp], in fp64:
//   check      every logit, embedding, anchor and weight finite (one 4-byte copy), otherwise ALQ_ERR_INVALID.
//   gram       G = W W^T: 64 x 64 tiles of the upper triangle, a fixed ascending-d chain per entry (products of fp32
//              values are exact in fp64, the adds rounded one by one), each off-diagonal entry written to both halves.
//   radius     R2_u = max_c exact_d2(z_u, a_c) (K7's pair arithmetic through d2_step, ascending columns): 64 x 64 tiles,
//              a block per 64 rows walking every anchor tile, the max kept per row.  n x C is never formed.
//   rows       in chunks of rows: lse (row_lse, K19's), yhat = argmax l (lowest class on ties) and r = p - e_yhat with
//              p_c = exp(l_c - lse) (a thread per row); w = r G (64 x 64 tiles, an ascending-c chain per entry; G is
//              symmetric, so row k of G is column k); then a thread per row: s2 = sum_k r_k w_k (ascending k),
//              t* = min over {k : w_k > w_yhat} of ((l_yhat - l_k) s) / (w_k - w_yhat) with s = sqrt(s2), +inf when
//              s2 <= 0 or no k qualifies; rho = (sqrt(D) t*) / sqrt(R2), +inf when R2 = 0 or t* = +inf.
//   The NumPy statement, operation for operation, is tests/alfamix_oracle.py; only CUDA's exp / log differ from it.
#include <math.h>

#include <algorithm>

#include "alq_common.cuh"

namespace afm {

constexpr int TT = 64;                          // rows and columns of a tile
constexpr int KC = 16;                          // columns of the contraction staged per step
constexpr int TILE_THREADS = 256;

// acc[q][r] over columns [0, d) of a-row i0 + ty + 16 q and b-row j0 + tx + 16 r, ascending, one chain per entry:
// D2 ? d2_step (K7's pair arithmetic) : s + a * b (no FMA).  Rows past na / nb and columns past d read as 0.
template <bool D2, typename T>
__device__ __forceinline__ void tile_acc(const T* __restrict__ a, int64_t lda, int na, int i0, const T* __restrict__ b,
                                         int64_t ldb, int nb, int j0, int d, T (*sI)[KC + 1], T (*sJ)[KC + 1],
                                         double (&acc)[4][4]) {
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[q][r] = 0.0;
    for (int k0 = 0; k0 < d; k0 += KC) {
        for (int e = tid; e < TT * KC; e += TILE_THREADS) {
            const int rr = e / KC, kk = e % KC, col = k0 + kk;
            const int pi = i0 + rr, pj = j0 + rr;
            sI[rr][kk] = (pi < na && col < d) ? a[static_cast<int64_t>(pi) * lda + col] : T(0);
            sJ[rr][kk] = (pj < nb && col < d) ? b[static_cast<int64_t>(pj) * ldb + col] : T(0);
        }
        __syncthreads();
        const int kn = min(KC, d - k0);                 // the chain stops at d: no padded term is added
#pragma unroll 4
        for (int kk = 0; kk < kn; ++kk) {
            double x[4], y[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                x[q] = static_cast<double>(sI[ty + 16 * q][kk]);
                y[q] = static_cast<double>(sJ[tx + 16 * q][kk]);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int r = 0; r < 4; ++r)
                    acc[q][r] = D2 ? d2_step(acc[q][r], x[q], y[r]) : __dadd_rn(acc[q][r], __dmul_rn(x[q], y[r]));
        }
        __syncthreads();
    }
}

// G[i][j] = G[j][i] = sum_d W_id W_jd for the tiles on and above the diagonal
__global__ void __launch_bounds__(TILE_THREADS) afm_gram_kernel(const float* __restrict__ w, int C, int d,
                                                                double* __restrict__ g) {
    if (blockIdx.y > blockIdx.x) return;
    __shared__ float sI[TT][KC + 1], sJ[TT][KC + 1];
    const int i0 = blockIdx.y * TT, j0 = blockIdx.x * TT;
    double acc[4][4];
    tile_acc<false>(w, d, C, i0, w, d, C, j0, d, sI, sJ, acc);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int i = i0 + ty + 16 * q, j = j0 + tx + 16 * r;
            if (i < C && j < C) {
                g[static_cast<size_t>(i) * C + j] = acc[q][r];
                g[static_cast<size_t>(j) * C + i] = acc[q][r];
            }
        }
}

// R2[i] = max_c exact_d2(z_i, a_c): a block per 64 rows, every anchor tile in turn
__global__ void __launch_bounds__(TILE_THREADS) afm_radius_kernel(const float* __restrict__ z, int n, int dp,
                                                                  const float* __restrict__ anc, int C,
                                                                  double* __restrict__ r2) {
    __shared__ float sI[TT][KC + 1], sJ[TT][KC + 1];
    const int i0 = blockIdx.x * TT;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double mx[4] = {0.0, 0.0, 0.0, 0.0};
    for (int j0 = 0; j0 < C; j0 += TT) {
        double acc[4][4];
        tile_acc<true>(z, dp, n, i0, anc, dp, C, j0, dp, sI, sJ, acc);
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int r = 0; r < 4; ++r)
                if (j0 + tx + 16 * r < C) mx[q] = fmax(mx[q], acc[q][r]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) mx[q] = fmax(mx[q], __shfl_xor_sync(0xffffffffu, mx[q], o));   // the 16 tx lanes
        const int i = i0 + ty + 16 * q;
        if (tx == 0 && i < n) r2[i] = mx[q];
    }
}

// per row of the chunk: yhat and r = p - e_yhat (a thread per row)
__global__ void __launch_bounds__(256) afm_resid_kernel(const float* __restrict__ logits, int rows, int C,
                                                        double* __restrict__ r, int* __restrict__ yhat) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= rows) return;
    const float* zr = logits + static_cast<size_t>(u) * C;
    const double lse = row_lse(zr, C);
    float best = __ldg(zr);
    int y = 0;
    for (int c = 1; c < C; ++c) {
        const float v = __ldg(zr + c);
        if (v > best) { best = v; y = c; }
    }
    double* ru = r + static_cast<size_t>(u) * C;
    for (int c = 0; c < C; ++c) {
        const double p = exp(__dsub_rn(static_cast<double>(__ldg(zr + c)), lse));
        ru[c] = c == y ? __dsub_rn(p, 1.0) : p;
    }
    yhat[u] = y;
}

// w[u][k] = sum_c r[u][c] G[k][c], c ascending
__global__ void __launch_bounds__(TILE_THREADS) afm_gr_kernel(const double* __restrict__ r, int rows, const double* __restrict__ g,
                                                              int C, double* __restrict__ w) {
    __shared__ double sI[TT][KC + 1], sJ[TT][KC + 1];
    const int i0 = blockIdx.y * TT, j0 = blockIdx.x * TT;
    double acc[4][4];
    tile_acc<false>(r, C, rows, i0, g, C, C, j0, C, sI, sJ, acc);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int i = i0 + ty + 16 * q, j = j0 + tx + 16 * s;
            if (i < rows && j < C) w[static_cast<size_t>(i) * C + j] = acc[q][s];
        }
}

// s2, t* and rho per row of the chunk (a thread per row)
__global__ void __launch_bounds__(256) afm_rho_kernel(const float* __restrict__ logits, const double* __restrict__ r,
                                                      const double* __restrict__ w, const int* __restrict__ yhat,
                                                      const double* __restrict__ r2, int rows, int C, double sqrt_d,
                                                      double* __restrict__ rho, double* __restrict__ tstar) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= rows) return;
    const float* zr = logits + static_cast<size_t>(u) * C;
    const double* ru = r + static_cast<size_t>(u) * C;
    const double* wu = w + static_cast<size_t>(u) * C;
    const int y = yhat[u];
    double s2 = 0.0;
    for (int k = 0; k < C; ++k) s2 = __dadd_rn(s2, __dmul_rn(ru[k], wu[k]));
    double t = INFINITY;
    if (s2 > 0.0) {
        const double s = __dsqrt_rn(s2), wy = wu[y], ly = static_cast<double>(__ldg(zr + y));
        for (int k = 0; k < C; ++k) {
            const double wk = wu[k];
            if (wk > wy)
                t = fmin(t, __ddiv_rn(__dmul_rn(__dsub_rn(ly, static_cast<double>(__ldg(zr + k))), s), __dsub_rn(wk, wy)));
        }
    }
    const double rr = __dsqrt_rn(r2[u]);
    rho[u] = (rr > 0.0 && t != INFINITY) ? __ddiv_rn(__dmul_rn(sqrt_d, t), rr) : INFINITY;
    if (tstar) tstar[u] = t;
}

// entries that are NaN or infinite are counted in *bad
__global__ void __launch_bounds__(256) afm_finite_kernel(const float* __restrict__ x, int64_t total, unsigned int* bad) {
    unsigned int cnt = 0;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<int64_t>(gridDim.x) * blockDim.x)
        cnt += !isfinite(__ldg(x + e));
    if (cnt) atomicAdd(bad, cnt);
}

}  // namespace afm

extern "C" int alq_alfamix_rho(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, const float* emb, int32_t dp,
                               const float* anchors, const float* weight, int32_t d, double* rho, double* r2,
                               double* tstar, void* stream) {
    using namespace afm;
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 1 || n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_alfamix_rho: n=%lld outside [1, 2^31)", (long long)n);
    if (c < 2) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_alfamix_rho: C=%d, need at least 2 classes", c);
    if (d < 1 || dp < d || dp % 4)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_alfamix_rho: D=%d and the padded width %d: need 1 <= D <= Dp, Dp %% 4 == 0", d, dp);
    if (!logits || !emb || !anchors || !weight || !rho)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_alfamix_rho: null pointer");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    // rows per chunk of the residual and w = r G pass: r and w stay below 2^25 entries each, and w = r G's row tiles
    // (gridDim.y) within CUDA's 65 535
    const int chunk = std::min({ni, 65535 * TT, std::max(TT, static_cast<int>(((1LL << 25) / c) / TT * TT))});
    const size_t cc = static_cast<size_t>(c) * c, rc = static_cast<size_t>(chunk) * c;
    double *g, *r, *w, *r2s;
    int* yhat;
    unsigned int* bad;
    int rcode = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        g = cur.take<double>(cc);
        r = cur.take<double>(rc);
        w = cur.take<double>(rc);
        yhat = cur.take<int>(chunk);
        r2s = cur.take<double>(n);
        bad = cur.take<unsigned int>(1);
    });
    if (rcode) return rcode;
    if (!r2) r2 = r2s;

    ALQ_CUDA(ctx, cudaMemsetAsync(bad, 0, 4, st));
    const int fb = ctx->sm_count * 8;
    afm_finite_kernel<<<fb, 256, 0, st>>>(logits, n * c, bad);
    ALQ_LAUNCH_CHECK(ctx);
    afm_finite_kernel<<<fb, 256, 0, st>>>(emb, n * dp, bad);
    ALQ_LAUNCH_CHECK(ctx);
    afm_finite_kernel<<<fb, 256, 0, st>>>(anchors, static_cast<int64_t>(c) * dp, bad);
    ALQ_LAUNCH_CHECK(ctx);
    afm_finite_kernel<<<fb, 256, 0, st>>>(weight, static_cast<int64_t>(c) * d, bad);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned int h = 0u;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h, bad, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (h)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_alfamix_rho: %u logits, embedding, anchor or weight entries are not finite", h);

    const int ct = (c + TT - 1) / TT;
    afm_gram_kernel<<<dim3(ct, ct), TILE_THREADS, 0, st>>>(weight, c, d, g);
    ALQ_LAUNCH_CHECK(ctx);
    afm_radius_kernel<<<(ni + TT - 1) / TT, TILE_THREADS, 0, st>>>(emb, ni, dp, anchors, c, r2);
    ALQ_LAUNCH_CHECK(ctx);
    const double sqrt_d = sqrt(static_cast<double>(d));
    for (int lo = 0; lo < ni; lo += chunk) {
        const int rows = std::min(chunk, ni - lo);
        const float* lg = logits + static_cast<size_t>(lo) * c;
        afm_resid_kernel<<<(rows + 255) / 256, 256, 0, st>>>(lg, rows, c, r, yhat);
        ALQ_LAUNCH_CHECK(ctx);
        afm_gr_kernel<<<dim3(ct, (rows + TT - 1) / TT), TILE_THREADS, 0, st>>>(r, rows, g, c, w);
        ALQ_LAUNCH_CHECK(ctx);
        afm_rho_kernel<<<(rows + 255) / 256, 256, 0, st>>>(lg, r, w, yhat, r2 + lo, rows, c, sqrt_d, rho + lo,
                                                           tstar ? tstar + lo : nullptr);
        ALQ_LAUNCH_CHECK(ctx);
    }
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    return ALQ_OK;
}

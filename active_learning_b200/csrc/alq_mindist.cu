// K3: out[i] = min_j (or max_j) of the squared L2 distance between candidate row i and every row
// of a second set, without ever forming the N x M matrix.  Device replacement of
// get_pairwise_l2_dist + `[:, labeled].min(dim=1)` (coreset_sampler.py:59-64,79) and of the
// minimax cold start `.max(dim=1).values.min(dim=0)` (coreset_sampler.py:100), all under
// active_learning/src/query_strategies.
//
// This is the one dense contraction on the path (2*N*M*D flop).  This translation unit is the
// exact-fp32 SIMT version: a 128x128x16 shared-memory tiled SGEMM (8x8 register micro-tiles,
// register-prefetch double buffering) whose epilogue turns each dot product into
// fl(fl(n_i + n_j) - 2*dot) -- the reference's own expression order -- and folds the row-wise
// min/max in registers, so the only HBM traffic is the two operand matrices.
// BADGE rows are rank-1 factors: <g_i, g_j> = <a_i, a_j> * <h_i, h_j>, |g|^2 = |a|^2 |h|^2; the kernel
// then runs two K loops (over c and over d) into two accumulator sets and multiplies them.
#include "alq_common.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 16;
constexpr int LDS_PAD = 4;
constexpr int kThreads = 256;

struct Operand {
    const float* p;
    int64_t ld;
    int64_t rows;
};

// Load this thread's two float4 of a (128 x 16) operand tile: rows row0.., columns k0..k0+15.
__device__ __forceinline__ void load_tile(const Operand& op, int64_t row0, int k0, int kdim, float4 (&r)[2]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int idx = threadIdx.x + h * kThreads;
        const int rr = idx >> 2, kq = (idx & 3) << 2;
        const int64_t row = row0 + rr;
        if (row < op.rows && k0 + kq < kdim)
            r[h] = __ldg(reinterpret_cast<const float4*>(op.p + row * op.ld + k0 + kq));
        else
            r[h] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}
__device__ __forceinline__ void store_tile(float (*s)[BM + LDS_PAD], const float4 (&r)[2]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int idx = threadIdx.x + h * kThreads;
        const int rr = idx >> 2, kq = (idx & 3) << 2;
        s[kq + 0][rr] = r[h].x;
        s[kq + 1][rr] = r[h].y;
        s[kq + 2][rr] = r[h].z;
        s[kq + 3][rr] = r[h].w;
    }
}

// acc[8][8] += X_tile(row0..) * Y_tile(col0..)^T over the full K dimension.
__device__ __forceinline__ void gemm_tile(const Operand& X, const Operand& Y, int64_t row0, int64_t col0,
                                          int kdim, float (*As)[BK][BM + LDS_PAD],
                                          float (*Bs)[BK][BN + LDS_PAD], float (&acc)[8][8]) {
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float4 ra[2], rb[2];
    load_tile(X, row0, 0, kdim, ra);
    load_tile(Y, col0, 0, kdim, rb);
    __syncthreads();  // previous users of the smem buffers are done
    store_tile(As[0], ra);
    store_tile(Bs[0], rb);
    __syncthreads();
    int buf = 0;
    for (int k0 = 0; k0 < kdim; k0 += BK) {
        const bool more = k0 + BK < kdim;
        if (more) {
            load_tile(X, row0, k0 + BK, kdim, ra);
            load_tile(Y, col0, k0 + BK, kdim, rb);
        }
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (more) {
            store_tile(As[buf ^ 1], ra);
            store_tile(Bs[buf ^ 1], rb);
            __syncthreads();
            buf ^= 1;
        }
    }
}

template <bool FACTORED, bool RED_MAX>
__global__ void __launch_bounds__(kThreads, FACTORED ? 1 : 2)
min_dist_kernel(Operand X, const float* __restrict__ xn, Operand Y, const float* __restrict__ yn, int d,
                Operand XA, const float* __restrict__ xan, Operand YA, const float* __restrict__ yan, int c,
                int col_tiles_per_cta, float* __restrict__ out) {
    __shared__ __align__(16) float As[2][BK][BM + LDS_PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + LDS_PAD];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t row0 = static_cast<int64_t>(blockIdx.x) * BM;
    const int64_t n = X.rows, m = Y.rows;
    const int64_t total_col_tiles = (m + BN - 1) / BN;
    const int64_t t_begin = static_cast<int64_t>(blockIdx.y) * col_tiles_per_cta;
    const int64_t t_end = min(total_col_tiles, t_begin + col_tiles_per_cta);

    float rn[8];     // |row|^2 of this thread's 8 rows
    float best[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        float v = 0.f;
        if (r < n) v = FACTORED ? xn[r] * xan[r] : xn[r];
        rn[i] = v;
        best[i] = RED_MAX ? ALQ_NEG_INF : ALQ_POS_INF;
    }
    const float pad_norm = RED_MAX ? ALQ_NEG_INF : ALQ_POS_INF;

    for (int64_t t = t_begin; t < t_end; ++t) {
        const int64_t col0 = t * BN;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        gemm_tile(X, Y, row0, col0, d, As, Bs, acc);
        if (FACTORED) {
            float acc2[8][8];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc2[i][j] = 0.f;
            gemm_tile(XA, YA, row0, col0, c, As, Bs, acc2);
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] *= acc2[i][j];
        }
        float cn[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int64_t cc = col0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
            cn[j] = cc < m ? (FACTORED ? yn[cc] * yan[cc] : yn[cc]) : pad_norm;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float dist = (rn[i] + cn[j]) - 2.0f * acc[i][j];
                best[i] = RED_MAX ? fmaxf(best[i], dist) : fminf(best[i], dist);
            }
    }
    // fold across the 16 threads (tx) that share these rows: lanes differ in the low 4 bits
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        float v = best[i];
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            const float w = __shfl_xor_sync(0xffffffffu, v, o);
            v = RED_MAX ? fmaxf(v, w) : fminf(v, w);
        }
        const int64_t r = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        if (tx == 0 && r < n && t_begin < t_end) {
            if (RED_MAX) atomic_max_float(out + r, v);
            else atomic_min_float(out + r, v);
        }
    }
}

__global__ void fill_kernel(float* p, int64_t n, float v) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

__global__ void __launch_bounds__(1024) argmin_kernel(const float* __restrict__ v, int64_t n, int32_t* out) {
    // single CTA: lowest index among the minima.  key = (ord(v) << 32) | index, take the min.
    __shared__ unsigned long long sm[32];
    unsigned long long best = ~0ull;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long k = (static_cast<unsigned long long>(alq_ord(v[i])) << 32) | static_cast<uint32_t>(i);
        best = k < best ? k : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o);
        best = w < best ? w : best;
    }
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
        best = sm[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o);
            best = w < best ? w : best;
        }
        if (threadIdx.x == 0) out[0] = static_cast<int32_t>(best & 0xffffffffu);
    }
}

// balancing_sampler.py:114-119: arg-min of num[i] / den[i] over the rows with avail[i] != 0, lowest index among equal
// ratios (torch's CPU min over the compacted vector).  num == nullptr: the numerator is the constant 1 (:104-107).
__global__ void __launch_bounds__(1024) ratio_argmin_kernel(const float* __restrict__ num, const float* __restrict__ den,
                                                            const unsigned char* __restrict__ avail, int64_t n,
                                                            int32_t* out) {
    __shared__ unsigned long long sm[32];
    unsigned long long best = ~0ull;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
        if (!avail[i]) continue;
        const float r = __fdiv_rn(num ? num[i] : 1.0f, den[i]);
        const unsigned long long k = (static_cast<unsigned long long>(alq_ord(r + 0.0f)) << 32) | static_cast<uint32_t>(i);
        best = k < best ? k : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o);
        best = w < best ? w : best;
    }
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
        best = sm[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o);
            best = w < best ? w : best;
        }
        if (threadIdx.x == 0) out[0] = best == ~0ull ? -1 : static_cast<int32_t>(best & 0xffffffffu);
    }
}

}  // namespace

int alq_min_dist_tc(alq_ctx* ctx, const float* x, int64_t ldx, const float* xn, int64_t n, const float* y,
                    int64_t ldy, const float* yn, int64_t m, int32_t d, const float* xa, int64_t ldxa,
                    const float* xan, const float* ya, int64_t ldya, const float* yan, int32_t c,
                    int32_t reduce_max, int32_t accumulate, float* out, cudaStream_t st);

extern "C" int alq_min_dist(alq_ctx* ctx, const float* x, int64_t ldx, const float* xn, int64_t n,
                            const float* y, int64_t ldy, const float* yn, int64_t m, int32_t d,
                            const float* xa, int64_t ldxa, const float* xan, const float* ya, int64_t ldya,
                            const float* yan, int32_t c, int32_t reduce_max, int32_t accumulate, float* out,
                            void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || m < 0 || d <= 0 || ldx < d || ldy < d)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: bad shape n=%lld m=%lld d=%d", (long long)n, (long long)m, d);
    if (n == 0) return ALQ_OK;
    if (!x || !xn || !out || (m > 0 && (!y || !yn))) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: null pointer");
    const bool factored = xa != nullptr;
    if (factored && (!ya || !xan || !yan || c <= 0 || ldxa < c || ldya < c))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: incomplete factored operands");
    if ((d % 4) || (ldx % 4) || (ldy % 4) || !aligned16(x) || (m > 0 && !aligned16(y)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: d, ldx, ldy must be multiples of 4 and bases 16-byte aligned");
    if (factored && ((c % 4) || (ldxa % 4) || (ldya % 4) || !aligned16(xa) || !aligned16(ya)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: c, ldxa, ldya must be multiples of 4 (pad with zeros)");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // tensor-core path (wgmma 3xTF32) for contractions big enough to amortise the operand split
    {
        const bool tc_shape = d >= 32 && (!factored || c >= 32) && m > 0;
        const double flop = 2.0 * static_cast<double>(n) * static_cast<double>(m) * (d + (factored ? c : 0));
        const bool want_tc = ctx->k3_impl == 2 || (ctx->k3_impl == 0 && flop >= 4e9);
        if (want_tc && tc_shape) {
            const int rc = alq_min_dist_tc(ctx, x, ldx, xn, n, y, ldy, yn, m, d, xa, ldxa, xan, ya, ldya, yan, c,
                                           reduce_max, accumulate, out, st);
            if (rc != ALQ_ERR_STATE) return rc;   // ALQ_ERR_STATE: not available here -> SIMT below
        } else if (ctx->k3_impl == 2) {
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: k3_impl=2 needs d >= 32 (and c >= 32 when factored)");
        }
    }
    if (!accumulate) {
        fill_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(out, n, reduce_max ? -INFINITY : INFINITY);
        ALQ_LAUNCH_CHECK(ctx);
    }
    if (m == 0) return ALQ_OK;
    const int64_t row_blocks = (n + BM - 1) / BM;
    const int64_t col_tiles = (m + BN - 1) / BN;
    // split the column range until the grid covers ~4 waves of CTAs
    int64_t splits = 1;
    const int64_t want = static_cast<int64_t>(ctx->sm_count) * 4;
    if (row_blocks < want) splits = std::min<int64_t>(col_tiles, (want + row_blocks - 1) / row_blocks);
    const int per = static_cast<int>((col_tiles + splits - 1) / splits);
    splits = (col_tiles + per - 1) / per;
    if (row_blocks > 0x7fffffffLL || splits > 65535) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_min_dist: grid too large");
    dim3 grid(static_cast<unsigned>(row_blocks), static_cast<unsigned>(splits));
    Operand X{x, ldx, n}, Y{y, ldy, m}, XA{xa, ldxa, n}, YA{ya, ldya, m};
    if (factored) {
        if (reduce_max) min_dist_kernel<true, true><<<grid, kThreads, 0, st>>>(X, xn, Y, yn, d, XA, xan, YA, yan, c, per, out);
        else min_dist_kernel<true, false><<<grid, kThreads, 0, st>>>(X, xn, Y, yn, d, XA, xan, YA, yan, c, per, out);
    } else {
        if (reduce_max) min_dist_kernel<false, true><<<grid, kThreads, 0, st>>>(X, xn, Y, yn, d, XA, xan, YA, yan, c, per, out);
        else min_dist_kernel<false, false><<<grid, kThreads, 0, st>>>(X, xn, Y, yn, d, XA, xan, YA, yan, c, per, out);
    }
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_ratio_argmin(alq_ctx* ctx, const float* num, const float* den, const unsigned char* avail, int64_t n,
                                int32_t* out_row, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n <= 0 || n >= (1LL << 31) || !den || !avail || !out_row) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ratio_argmin: bad arguments");
    ratio_argmin_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(num, den, avail, n, out_row);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_argmin(alq_ctx* ctx, const float* v, int64_t n, int32_t* out_row, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n <= 0 || n >= (1LL << 31) || !v || !out_row) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_argmin: bad arguments");
    argmin_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(v, n, out_row);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

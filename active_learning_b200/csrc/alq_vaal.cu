// K9: the VAAL discriminator on the Hopper tensor cores (vaal_sampler.py:57-58 and vaal_discriminator.py of the
// reference's query_strategies):  p[i] = sigmoid(w3 . relu(W2 relu(W1 mu_i + b1) + b2) + b3),  hidden width 512.
//
// Two launches of one kernel template per pool slice of at most SLICE_ROWS rows, both on the ring of alq_wgmma.cuh
// that K3, K13, K15 and K18 use: a one-thread TMA producer warpgroup (tc::ring_produce_rows) feeding a 3-stage
// SWIZZLE_128B ring, two consumer warpgroups issuing the 3xTF32 chain tile by tile (tc::ring_tile: hi*hi' + hi*lo' +
// lo*hi', operands split ahead of time).
//   layer 1  X = mu [rows, z] (z zero-padded to a multiple of 32), Y = W1 [512, z].  Epilogue: relu(acc + b1),
//            stored as the TF32 hi/lo pair layer 2 reads, so the [rows, 512] intermediate needs no split pass.
//   layer 2  X = H1 [rows, 512], Y = W2 [512, 512].  Epilogue: relu(acc + b2_j) * w3_j summed over all 512
//            columns by the thread that holds them, in a fixed order, then across the four lanes of a quad by
//            shuffles: no atomics, so a row's p depends on its own values only (equal rows give equal p).
// A CTA owns whole 128-row blocks (grid-stride over the slice) and sweeps the four 128-column tiles of the hidden
// layer in order; the weights (2 MB of hi + lo for W2) stay in L2.
#include "alq_wgmma.cuh"

namespace vaal {

using namespace tc;

constexpr int HID = 512;                          // the reference's only hidden width
constexpr int NT = HID / BN;
constexpr int64_t SLICE_ROWS = 131072;            // bounds the hi + lo intermediate at 512 MB

struct Params {
    const float* bias;                 // b1 (layer 1) or b2 (layer 2), [512]
    const float* w3; const float* b3;  // layer 2: [512], [1]
    float* h_hi; float* h_lo;          // layer 1 output, [rows, 512]
    float* p; float* logit;            // layer 2 output, [rows] (logit may be null)
    int rows;
    int kblocks;                       // K / 32
};

template <int LAYER>
__global__ void __launch_bounds__(THREADS, 1)
vaal_layer_kernel(const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
                  const __grid_constant__ CUtensorMap map_yh, const __grid_constant__ CUtensorMap map_yl, Params P) {
    extern __shared__ unsigned char smem_dyn[];
    const Role me = ring_role();
    const int m_blocks = (P.rows + BM - 1) / BM;
    const Ring ring = ring_init(smem_dyn);

    if (me.wg == 0) {
        producer_regs();
        if (threadIdx.x == 0) ring_produce_rows(ring, &map_xh, &map_xl, &map_yh, &map_yl, m_blocks, NT, P.kblocks);
    } else {
        consumer_regs();
        uint32_t it = 0;
        for (int mb = blockIdx.x; mb < m_blocks; mb += gridDim.x) {
            const int row0 = mb * BM + me.r_in_tile, row1 = row0 + 8;
            float s0 = 0.f, s1 = 0.f;                 // layer 2: this thread's share of the w3 dot product
            for (int nt = 0; nt < NT; ++nt) {
                float acc[64];
                ring_tile(ring, it, me, acc, P.kblocks);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = nt * BN + 8 * j + me.c_in_tile;
                    const float bb0 = __ldg(P.bias + col), bb1 = __ldg(P.bias + col + 1);
                    const float h00 = fmaxf(acc[4 * j] + bb0, 0.f), h01 = fmaxf(acc[4 * j + 1] + bb1, 0.f);
                    const float h10 = fmaxf(acc[4 * j + 2] + bb0, 0.f), h11 = fmaxf(acc[4 * j + 3] + bb1, 0.f);
                    if constexpr (LAYER == 1) {
                        float hi0, lo0, hi1, lo1;
                        if (row0 < P.rows) {
                            split_tf32(h00, hi0, lo0); split_tf32(h01, hi1, lo1);
                            const size_t o = static_cast<size_t>(row0) * HID + col;
                            *reinterpret_cast<float2*>(P.h_hi + o) = make_float2(hi0, hi1);
                            *reinterpret_cast<float2*>(P.h_lo + o) = make_float2(lo0, lo1);
                        }
                        if (row1 < P.rows) {
                            split_tf32(h10, hi0, lo0); split_tf32(h11, hi1, lo1);
                            const size_t o = static_cast<size_t>(row1) * HID + col;
                            *reinterpret_cast<float2*>(P.h_hi + o) = make_float2(hi0, hi1);
                            *reinterpret_cast<float2*>(P.h_lo + o) = make_float2(lo0, lo1);
                        }
                    } else {
                        const float w0 = __ldg(P.w3 + col), w1 = __ldg(P.w3 + col + 1);
                        s0 = fmaf(h00, w0, s0); s0 = fmaf(h01, w1, s0);
                        s1 = fmaf(h10, w0, s1); s1 = fmaf(h11, w1, s1);
                    }
                }
            }
            if constexpr (LAYER == 2) {
                // the four lanes of a quad hold the same two rows, 128 columns each
                s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
                s0 += __shfl_xor_sync(0xffffffffu, s0, 2); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
                if ((me.lane & 3) == 0) {
                    const float b3 = __ldg(P.b3);
                    if (row0 < P.rows) {
                        const float x = s0 + b3;
                        P.p[row0] = 1.f / (1.f + expf(-x));
                        if (P.logit) P.logit[row0] = x;
                    }
                    if (row1 < P.rows) {
                        const float x = s1 + b3;
                        P.p[row1] = 1.f / (1.f + expf(-x));
                        if (P.logit) P.logit[row1] = x;
                    }
                }
            }
        }
    }
}

// hi/lo TF32 pair of x[rows, d] (leading dimension ld) as contiguous [rows, kp] rows, columns d..kp-1 zero
__global__ void __launch_bounds__(256)
split_pad_kernel(const float* __restrict__ x, int64_t rows, int d, int64_t ld, int kp, float* __restrict__ hi,
                 float* __restrict__ lo) {
    const int64_t total = rows * kp;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t r = i / kp;
        const int k = static_cast<int>(i - r * kp);
        float h = 0.f, l = 0.f;
        if (k < d) split_tf32(x[r * ld + k], h, l);
        hi[i] = h;
        lo[i] = l;
    }
}

}  // namespace vaal

extern "C" int alq_vaal_scores(alq_ctx* ctx, const float* mu, int64_t n, int32_t z, int64_t ldmu, const float* w1,
                               int64_t ldw1, const float* b1, const float* w2, int64_t ldw2, const float* b2,
                               const float* w3, const float* b3, int32_t hidden, float* p, float* logits,
                               void* stream) {
    using namespace vaal;
    if (!ctx) return ALQ_ERR_INVALID;
    if (hidden != HID)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_vaal_scores: hidden width %d, the kernel is built for %d", hidden, HID);
    if (n < 0 || n >= (1LL << 31) || z < 1 || ldmu < z || ldw1 < z || ldw2 < HID || ldmu % 4 || ldw1 % 4 || ldw2 % 4)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_vaal_scores: bad shape (n=%lld z=%d ldmu=%lld ldw1=%lld ldw2=%lld)",
                 (long long)n, z, (long long)ldmu, (long long)ldw1, (long long)ldw2);
    if (!w1 || !b1 || !w2 || !b2 || !w3 || !b3 || (n > 0 && (!mu || !p)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_vaal_scores: null pointer");
    if (!aligned16(w1) || !aligned16(w2) || (n > 0 && !aligned16(mu)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_vaal_scores: mu, w1 and w2 must be 16-byte aligned");
    if (n == 0) return ALQ_OK;
    if (!get_encode()) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_vaal_scores: cuTensorMapEncodeTiled is unavailable");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);

    const int kp = (z + BK - 1) / BK * BK;
    const int64_t slice = std::min<int64_t>(n, SLICE_ROWS);
    const size_t w1e = static_cast<size_t>(HID) * kp, w2e = static_cast<size_t>(HID) * HID;
    const size_t xe = static_cast<size_t>(slice) * kp, he = static_cast<size_t>(slice) * HID;
    float *w1h, *w1l, *w2h, *w2l, *xh, *xl, *hh, *hl;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        w1h = cur.take<float>(w1e); w1l = cur.take<float>(w1e);
        w2h = cur.take<float>(w2e); w2l = cur.take<float>(w2e);
        xh = cur.take<float>(xe); xl = cur.take<float>(xe);
        hh = cur.take<float>(he); hl = cur.take<float>(he);
    });
    if (rc) return rc;

    auto split = [&](const float* src, int64_t rows, int d, int64_t ld, int kpad, float* hi, float* lo) -> int {
        const int blocks = static_cast<int>(std::min<int64_t>((rows * kpad + 255) / 256, static_cast<int64_t>(ctx->sm_count) * 16));
        split_pad_kernel<<<blocks, 256, 0, st>>>(src, rows, d, ld, kpad, hi, lo);
        ALQ_LAUNCH_CHECK(ctx);
        return ALQ_OK;
    };
    if ((rc = split(w1, HID, z, ldw1, kp, w1h, w1l))) return rc;
    if ((rc = split(w2, HID, HID, ldw2, HID, w2h, w2l))) return rc;

    CUtensorMap mw1h, mw1l, mw2h, mw2l;
    if (!(make_map(&mw1h, w1h, HID, kp, BN) && make_map(&mw1l, w1l, HID, kp, BN) && make_map(&mw2h, w2h, HID, HID, BN) &&
          make_map(&mw2l, w2l, HID, HID, BN)))
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_vaal_scores: cuTensorMapEncodeTiled failed");
    const size_t smem = ring_smem_bytes(0);
    ALQ_CUDA(ctx, cudaFuncSetAttribute(vaal_layer_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    ALQ_CUDA(ctx, cudaFuncSetAttribute(vaal_layer_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));

    for (int64_t r0 = 0; r0 < n; r0 += slice) {
        const int rows = static_cast<int>(std::min<int64_t>(slice, n - r0));
        if ((rc = split(mu + r0 * ldmu, rows, z, ldmu, kp, xh, xl))) return rc;
        CUtensorMap mxh, mxl, mhh, mhl;
        if (!(make_map(&mxh, xh, rows, kp, BM) && make_map(&mxl, xl, rows, kp, BM) && make_map(&mhh, hh, rows, HID, BM) &&
              make_map(&mhl, hl, rows, HID, BM)))
            ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_vaal_scores: cuTensorMapEncodeTiled failed");
        const int grid = std::min(ctx->sm_count, (rows + BM - 1) / BM);
        Params P{};
        P.rows = rows;
        P.bias = b1; P.h_hi = hh; P.h_lo = hl; P.kblocks = kp / BK;
        vaal_layer_kernel<1><<<grid, THREADS, smem, st>>>(mxh, mxl, mw1h, mw1l, P);
        ALQ_LAUNCH_CHECK(ctx);
        P.bias = b2; P.w3 = w3; P.b3 = b3; P.p = p + r0; P.logit = logits ? logits + r0 : nullptr; P.kblocks = HID / BK;
        vaal_layer_kernel<2><<<grid, THREADS, smem, st>>>(mhh, mhl, mw2h, mw2l, P);
        ALQ_LAUNCH_CHECK(ctx);
    }
    return ALQ_OK;
}

// Rows into the 3xTF32 pipeline's operands (alq_wgmma.cuh), shared by K13 (alq_probcover.cu) and K15
// (alq_typiclust.cu): one warp per row, optionally L2-normalising the row first, then its TF32 hi / lo split and its
// fp64 squared norm.
//   normalise  lane-strided fp64 sum of squares, a butterfly, norm = sqrt, xhat = fl32(x / norm) (a zero row stays
//              zero);  without it xhat is the input.
//   split      hi / lo = tc::split_tf32(xhat), nrm2 = |xhat|^2 in fp64 in the same lane order.
#pragma once
#include "alq_wgmma.cuh"

namespace rs {

constexpr int NORM_WARPS = 8;

// internal linkage: every kernel file that includes this header gets its own copy
namespace {
__global__ void __launch_bounds__(NORM_WARPS * 32)
normalize_split_kernel(const float* __restrict__ x, int n, int d, long long ldx, float* __restrict__ xhat,
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
}  // namespace

}  // namespace rs

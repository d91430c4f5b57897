// K6 row code shared by the direct kernels (alq_mase.cu: the row lives in registers) and the bulk-copy pipelined
// kernel (alq_score.cu: the row lives in a shared-memory stage).  One warp owns one row of C logits.
#pragma once
#include <limits.h>

#include "alq_common.cuh"

struct MaseArgs {            // by-value kernel argument of the pipelined kernel's MASE modes (zero for the others)
    const float* ginv;       // [C, ldg]  1 / |w_a - w_c|
    int64_t ldg;
    const float* gmin;       // [C + 1]   min_c ginv[a, c]; gmin[C] = table-wide ratio bound (see mase_row_min_smem)
    int32_t* pred;           // [N]
    float* radius;           // [N, ldr] or NULL
    int64_t ldr;
};

template <int NV>
struct MaseRowRegs {         // NV float4 per lane, slots past the row end hold -inf
    float4 v[NV];
    __device__ __forceinline__ float4 get(int k, int /*lane*/) const { return v[k]; }
};

struct MaseRowSmem {         // the row sits in shared memory: re-reading it costs less than 32 live registers
    const float4* p;
    int nvec;
    __device__ __forceinline__ float4 get(int k, int lane) const {
        const int idx = lane + 32 * k;
        return idx < nvec ? p[idx] : make_float4(ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF);
    }
};

// The arg-max follows torch.max: NaN ranks above every number, so a row with a NaN predicts its first NaN (and every
// radius of that row is then +inf).  v beats best: v > best, or v is NaN and best is not.
__device__ __forceinline__ bool mase_beats(float v, float best) { return !(v <= best) && best == best; }
__device__ __forceinline__ bool mase_same(float a, float b) { return a == b || (a != a && b != b); }

// NaN-propagating maximum (max.NaN: NaN if either operand is NaN)
__device__ __forceinline__ float mase_fmax_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ void mase_argmax_merge(float& best, int& arg, float ob, int oa) {
    if (mase_beats(ob, best) || (mase_same(ob, best) && oa < arg)) { best = ob; arg = oa; }
}

__device__ __forceinline__ float mase_radius_of(float zp, float z, float g, bool is_pred) {
    float r = fabsf(zp - z) * g;
    r = (r != r) ? ALQ_POS_INF : r;        // 0 * inf (duplicated class rows), inf - inf
    return is_pred ? ALQ_POS_INF : r;
}

__device__ __forceinline__ float mase_warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// All classes: radius[c] for every c (optionally written to rq), the row minimum and the arg-max.
template <int NV, bool WRITE_R, typename Row>
__device__ __forceinline__ void mase_row_full(const Row& row, int lane, int nvec, const float* __restrict__ ginv,
                                              int64_t ldg, float4* __restrict__ rq, float& mn_out, int& arg_out) {
    float best = ALQ_NEG_INF;
    int arg = INT_MAX;
#pragma unroll
    for (int k = 0; k < NV; ++k) {          // ascending index inside a lane: strict > keeps the first maximum
        const int base = (lane + 32 * k) * 4;
        const float4 e = row.get(k, lane);
        if (mase_beats(e.x, best)) { best = e.x; arg = base; }
        if (mase_beats(e.y, best)) { best = e.y; arg = base + 1; }
        if (mase_beats(e.z, best)) { best = e.z; arg = base + 2; }
        if (mase_beats(e.w, best)) { best = e.w; arg = base + 3; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        mase_argmax_merge(best, arg, ob, oa);
    }
    if (arg == INT_MAX) arg = 0;             // a row of -inf / NaN: torch's max returns index 0
    const float4* gi = reinterpret_cast<const float4*>(ginv + static_cast<int64_t>(arg) * ldg);
    float mn = ALQ_POS_INF;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int idx = lane + 32 * k;
        if (idx < nvec) {
            const float4 g = __ldg(gi + idx);
            const float4 e = row.get(k, lane);
            const int base = idx * 4;
            float4 r;
            r.x = mase_radius_of(best, e.x, g.x, base == arg);
            r.y = mase_radius_of(best, e.y, g.y, base + 1 == arg);
            r.z = mase_radius_of(best, e.z, g.z, base + 2 == arg);
            r.w = mase_radius_of(best, e.w, g.w, base + 3 == arg);
            mn = fminf(fminf(mn, r.x), fminf(r.y, fminf(r.z, r.w)));
            if (WRITE_R) rq[idx] = r;
        }
    }
    mn_out = mase_warp_min(mn);
    arg_out = arg;
}

// MASE needs only min_c radius[i, c].  Every lane evaluates its own smallest-gap class exactly, r0 = the warp minimum
// of those, and a class c can only beat r0 if gap_c * gmin[p] < r0, because ginv[p, c] >= gmin[p] and fp32
// multiplication is monotone.  Only those classes (a handful per row) touch the table: 4 bytes of L2 traffic per
// surviving class instead of 4C per row.  The result is the exact minimum, not an approximation.
template <int NV, typename Row>
__device__ __forceinline__ void mase_row_min(const Row& row, int lane, int c, const float* __restrict__ ginv, int64_t ldg,
                                             const float* __restrict__ gmin, float& mn_out, int& arg_out) {
    // lane-local largest (l1, a1) and second largest (l2, a2) logit, lowest index first among equals
    float l1 = ALQ_NEG_INF, l2 = ALQ_NEG_INF;
    int a1 = INT_MAX, a2 = INT_MAX;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int base = (lane + 32 * k) * 4;
        const float4 q = row.get(k, lane);
        const float e[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (mase_beats(e[j], l1)) { l2 = l1; a2 = a1; l1 = e[j]; a1 = base + j; }
            else if (mase_beats(e[j], l2)) { l2 = e[j]; a2 = base + j; }
        }
    }
    float best = l1;
    int arg = a1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        mase_argmax_merge(best, arg, ob, oa);
    }
    if (arg == INT_MAX) arg = 0;
    const float* gi = ginv + static_cast<int64_t>(arg) * ldg;
    const float gm = __ldg(gmin + arg);
    // this lane's closest competitor: its largest logit, or its second largest if it owns the arg-max
    const bool own = (a1 == arg);
    const float lz = own ? l2 : l1;
    const int li = own ? a2 : a1;
    float mn = (li < c) ? mase_radius_of(best, lz, __ldg(gi + li), false) : ALQ_POS_INF;
    const float r0 = mase_warp_min(mn);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int base = (lane + 32 * k) * 4;
        const float4 q = row.get(k, lane);
        const float e[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int idx = base + j;
            const float bound = fabsf(best - e[j]) * gm;
            if (!(bound >= r0) && idx < c && idx != arg && idx != li)      // NaN bound (0 * inf): must look
                mn = fminf(mn, mase_radius_of(best, e[j], __ldg(gi + idx), false));
        }
    }
    mn_out = mase_warp_min(mn);
    arg_out = arg;
}

// The same exact minimum for a row that sits in shared memory, at a fraction of the instructions (the register
// version above is issue-bound: ~37 instructions per logit).  Work is done per 16-byte chunk of 4 classes:
//   1. chunk maxima m4[k]; best = the warp maximum; t2 = the second largest chunk maximum in the warp, i.e. the logit
//      of SOME class other than the arg-max (a lower bound on the runner-up logit);
//   2. a chunk can be skipped when its maximum is below  thr = best - (best - t2) * ratio * (1 + 2^-18),  ratio = the
//      table-wide bound max_p (largest finite ginv[p, :]) / gmin[p]  (gmin[C]): classes that far down cannot come closer
//      than the runner-up even at the most favourable distances;
//   3. the surviving chunks (typically two: the arg-max's and the runner-up's) are walked twice, first to find the
//      arg-max index, then to evaluate their radii against table row ginv[arg, :];
//   4. the pruning is CHECKED, not assumed: every skipped class has radius >= fl(fl(best - thr) * gmin[arg]) by
//      monotonicity of fp32 subtraction and multiplication; if the minimum found is not below that bound (coinciding
//      class rows, non-finite logits, ...), the row is evaluated in full.  The result is always the exact minimum.
template <int NV>
__device__ __forceinline__ void mase_row_min_smem(const float4* __restrict__ p, int nvec, int lane, const float* __restrict__ ginv,
                                                  int64_t ldg, const float* __restrict__ gmin, float ratio, float& mn_out,
                                                  int& arg_out) {
    float m4[NV];
    float t1 = ALQ_NEG_INF, t2 = ALQ_NEG_INF;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int idx = lane + 32 * k;
        float m = ALQ_NEG_INF;
        if (idx < nvec) {
            const float4 e = p[idx];
            m = mase_fmax_nan(mase_fmax_nan(e.x, e.y), mase_fmax_nan(e.z, e.w));   // a NaN makes best NaN: nothing
        }                                                                           // is pruned, every radius is +inf
        m4[k] = m;
        t2 = fmaxf(t2, fminf(t1, m));
        t1 = mase_fmax_nan(t1, m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float o1 = __shfl_xor_sync(0xffffffffu, t1, o);
        const float o2 = __shfl_xor_sync(0xffffffffu, t2, o);
        const float hi = mase_fmax_nan(t1, o1);
        t2 = fmaxf(fminf(t1, o1), fmaxf(t2, o2));
        t1 = hi;
    }
    const float best = t1;
    const float thr = best - (best - t2) * ratio * 1.000003814697265625f;
    unsigned mask = 0;
#pragma unroll
    for (int k = 0; k < NV; ++k)
        if (!(m4[k] < thr)) mask |= 1u << k;            // NaN threshold: everything survives
    // arg-max index: lowest index among the surviving classes equal to best
    int cand = INT_MAX;
    unsigned mm = mask;
    while (__any_sync(0xffffffffu, mm != 0)) {
        if (mm) {
            const int k = __ffs(mm) - 1;
            mm &= mm - 1;
            const int idx = lane + 32 * k;
            if (idx < nvec) {
                const float4 e = p[idx];
                const int base = idx * 4;
                if (mase_same(e.w, best)) cand = min(cand, base + 3);
                if (mase_same(e.z, best)) cand = min(cand, base + 2);
                if (mase_same(e.y, best)) cand = min(cand, base + 1);
                if (mase_same(e.x, best)) cand = min(cand, base);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
    const int arg = cand == INT_MAX ? 0 : cand;
    const float4* gi = reinterpret_cast<const float4*>(ginv + static_cast<int64_t>(arg) * ldg);
    const float gm = __ldg(gmin + arg);
    float mn = ALQ_POS_INF;
    mm = mask;
    while (__any_sync(0xffffffffu, mm != 0)) {
        if (mm) {
            const int k = __ffs(mm) - 1;
            mm &= mm - 1;
            const int idx = lane + 32 * k;
            if (idx < nvec) {
                const float4 e = p[idx];
                const float4 g = __ldg(gi + idx);
                const int base = idx * 4;
                mn = fminf(mn, fminf(fminf(mase_radius_of(best, e.x, g.x, base == arg), mase_radius_of(best, e.y, g.y, base + 1 == arg)),
                                     fminf(mase_radius_of(best, e.z, g.z, base + 2 == arg), mase_radius_of(best, e.w, g.w, base + 3 == arg))));
            }
        }
    }
    mn = mase_warp_min(mn);
    const float skipped_lb = (best - thr) * gm;           // every skipped class: radius >= fl(fl(best - thr) * gmin[arg])
    if (!(mn <= skipped_lb)) {                            // warp-uniform; rare
        mn = ALQ_POS_INF;
        for (int idx = lane; idx < nvec; idx += 32) {
            const float4 e = p[idx];
            const float4 g = __ldg(gi + idx);
            const int base = idx * 4;
            mn = fminf(mn, fminf(fminf(mase_radius_of(best, e.x, g.x, base == arg), mase_radius_of(best, e.y, g.y, base + 1 == arg)),
                                 fminf(mase_radius_of(best, e.z, g.z, base + 2 == arg), mase_radius_of(best, e.w, g.w, base + 3 == arg))));
        }
        mn = mase_warp_min(mn);
    }
    mn_out = mn;
    arg_out = arg;
}

// Implemented in alq_score.cu next to the pipelined row kernel it instantiates.  Returns false when the shape does not
// qualify (the caller then uses its direct kernels); *err carries a launch failure.
bool alq_mase_rows_pipe(alq_ctx* ctx, cudaStream_t st, const float* logits, int64_t n, int c, const MaseArgs& m,
                        float* min_margin, cudaError_t* err);

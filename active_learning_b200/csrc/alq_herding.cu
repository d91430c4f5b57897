// K23: MaxHerdingSampler's greedy (Bae, Noh & Sutherland, "Generalized Coverage for More Robust Low-Budget Active
// Learning", ECCV 2024) over K22's n x n fp32 Gaussian kernel matrix K (alq_ward.cu), with incremental gains.
//
// F(S) = sum_i max_{s in L u S} K_is.  m_i is the current max (fp32) and gain_c = sum_i max(0, K_ic - m_i) (fp64), so a
// pick c* changes m only on the rows S = {i : K[c*, i] > m_i}, and every gain drops by
//   acc_c = sum_{i in S, ascending} (max(0, K_ic - m_i) - max(0, K_ic - K[c*, i]))
// (fp64; every operation rounded on its own: __dadd_rn / __dsub_rn, no contraction).  A step reads |S| n entries of K
// instead of n^2.  The NumPy statement, operation for operation, is tests/maxherding_oracle.py.
//
//   set-up  m_i = the max over the labeled rows l of K[l, i] (0 with none; a thread per column, the labeled rows of each
//           chunk listed in shared memory); gain_c = the ascending sum over i (a thread per column reading K[i, c]:
//           coalesced across c); the available rows counted (one 4-byte copy: the loop's length).
//   a step  three launches on one stream, the pick never leaving the device:
//     argmax   per CTA the best (gain, lowest position) over the candidates (available, not yet picked);
//     cover    every CTA reduces those partials to the same c*, then compacts its 1024 rows of S in ascending order
//              (ballots) into its own segment as (i, old m_i, K[c*, i]) and sets m_i = K[c*, i]; CTA 0 records the pick.
//              Segment b holds rows [1024 b, 1024 b + 1024), so walking the segments in order walks S ascending;
//     update   a thread per candidate column walks the segments in order (staged in shared memory) and subtracts acc_c.
//           Columns that are not candidates keep a stale gain: it is never read again.
// Ties: (gain, position) is a total order (the gains are never NaN: K is finite), so every reduction order gives the
// lowest position of the largest gain.  Once all gains are 0 (an underflowed kernel) that is the lowest free position.
#include <math.h>

#include <algorithm>
#include <climits>

#include "alq_common.cuh"

namespace herd {

constexpr int COL_THREADS = 256;   // set-up and update: a thread per column
constexpr int SEG = 1024;          // rows per cover CTA (and per segment of S)
constexpr int ARG_THREADS = 512;
constexpr int STAGE = 256;         // segment entries staged per round of the update

struct Entry {
    int row;
    float m_old;
    float kc;
};

__device__ __forceinline__ bool better(double g, int p, double bg, int bp) { return g > bg || (g == bg && p < bp); }

__device__ __forceinline__ void warp_best(double& g, int& p) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double og = __shfl_xor_sync(0xffffffffu, g, o);
        const int op = __shfl_xor_sync(0xffffffffu, p, o);
        if (better(og, op, g, p)) { g = og; p = op; }
    }
}

// block-wide best of (g, p); every thread returns it (blockDim.x a multiple of 32, at most 1024)
__device__ __forceinline__ void block_best(double& g, int& p) {
    __shared__ double sg[32];
    __shared__ int sp[32];
    warp_best(g, p);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();                                   // the previous call's readers are done with sg / sp
    if (l == 0) { sg[w] = g; sp[w] = p; }
    __syncthreads();
    g = l < nw ? sg[l] : -INFINITY;
    p = l < nw ? sp[l] : INT_MAX;
    warp_best(g, p);
}

// m_i = max over labeled rows l of K[l, i]
__global__ void __launch_bounds__(COL_THREADS) hs_m_kernel(const float* __restrict__ K, int n, int64_t ld,
                                                           const uint8_t* __restrict__ labeled, float* __restrict__ m) {
    __shared__ int rows[COL_THREADS];
    __shared__ int cnt;
    const int c = blockIdx.x * COL_THREADS + threadIdx.x;
    float v = 0.0f;
    for (int l0 = 0; l0 < n; l0 += COL_THREADS) {
        if (threadIdx.x == 0) cnt = 0;
        __syncthreads();
        const int l = l0 + threadIdx.x;
        if (l < n && labeled[l]) rows[atomicAdd(&cnt, 1)] = l;    // any order: a max
        __syncthreads();
        if (c < n)
            for (int e = 0; e < cnt; ++e) v = fmaxf(v, __ldg(K + static_cast<int64_t>(rows[e]) * ld + c));
        __syncthreads();
    }
    if (c < n) m[c] = v;
}

// gain_c = sum_{i ascending} max(0, K_ic - m_i); n_avail += available rows
__global__ void __launch_bounds__(COL_THREADS) hs_gain_kernel(const float* __restrict__ K, int n, int64_t ld,
                                                              const float* __restrict__ m,
                                                              const uint8_t* __restrict__ avail,
                                                              double* __restrict__ gain, int* __restrict__ n_avail) {
    __shared__ float sm[COL_THREADS];
    const int c = blockIdx.x * COL_THREADS + threadIdx.x;
    double g = 0.0;
    for (int i0 = 0; i0 < n; i0 += COL_THREADS) {
        __syncthreads();
        if (i0 + threadIdx.x < n) sm[threadIdx.x] = m[i0 + threadIdx.x];
        __syncthreads();
        const int len = min(COL_THREADS, n - i0);
        if (c < n) {
            const float* kp = K + static_cast<int64_t>(i0) * ld + c;
#pragma unroll 8
            for (int e = 0; e < len; ++e)
                g = __dadd_rn(g, fmax(0.0, __dsub_rn(static_cast<double>(__ldg(kp + e * ld)), static_cast<double>(sm[e]))));
        }
    }
    if (c < n) {
        gain[c] = g;
        if (avail[c]) atomicAdd(n_avail, 1);
    }
}

// per CTA: the best (gain, position) over the candidates of its columns
__global__ void __launch_bounds__(ARG_THREADS) hs_argmax_kernel(const double* __restrict__ gain,
                                                                const uint8_t* __restrict__ cand, int n,
                                                                double* __restrict__ part_g, int* __restrict__ part_p) {
    double g = -INFINITY;
    int p = INT_MAX;
    for (int c = blockIdx.x * ARG_THREADS + threadIdx.x; c < n; c += gridDim.x * ARG_THREADS)
        if (cand[c] && better(gain[c], c, g, p)) { g = gain[c]; p = c; }
    block_best(g, p);
    if (threadIdx.x == 0) { part_g[blockIdx.x] = g; part_p[blockIdx.x] = p; }
}

// c* from the partials; this CTA's rows of S compacted in order; m updated on them
__global__ void __launch_bounds__(SEG) hs_cover_kernel(const float* __restrict__ K, int n, int64_t ld,
                                                       const double* __restrict__ part_g, const int* __restrict__ part_p,
                                                       int n_part, float* __restrict__ m, uint8_t* __restrict__ cand,
                                                       Entry* __restrict__ seg, int* __restrict__ seg_cnt,
                                                       int32_t* __restrict__ picks, int step,
                                                       unsigned long long* __restrict__ s_total) {
    __shared__ int wcnt[SEG / 32];
    __shared__ int cstar;
    double g = -INFINITY;
    int p = INT_MAX;
    if (threadIdx.x < 32) {
        for (int b = threadIdx.x; b < n_part; b += 32)
            if (better(part_g[b], part_p[b], g, p)) { g = part_g[b]; p = part_p[b]; }
        warp_best(g, p);
        if (threadIdx.x == 0) cstar = p;
    }
    __syncthreads();
    const int c = cstar;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        picks[step] = c;
        cand[c] = 0;
    }
    const int i = blockIdx.x * SEG + threadIdx.x;
    float kc = 0.0f, mi = 0.0f;
    bool in = false;
    if (i < n) {
        kc = __ldg(K + static_cast<int64_t>(c) * ld + i);
        mi = m[i];
        in = kc > mi;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, in);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) wcnt[w] = __popc(bal);
    __syncthreads();
    if (w == 0) {                                      // exclusive scan of the 32 warp counts
        const int v = wcnt[l];
        int s = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, s, o);
            if (l >= o) s += t;
        }
        wcnt[l] = s - v;
        if (l == 31) {
            seg_cnt[blockIdx.x] = s;
            if (s) atomicAdd(s_total, static_cast<unsigned long long>(s));
        }
    }
    __syncthreads();
    if (in) {
        seg[blockIdx.x * SEG + wcnt[w] + __popc(bal & ((1u << l) - 1u))] = Entry{i, mi, kc};
        m[i] = kc;
    }
}

// gain_c -= sum over S ascending of (max(0, K_ic - m_old_i) - max(0, K_ic - K[c*, i])), candidate columns only
__global__ void __launch_bounds__(COL_THREADS) hs_update_kernel(const float* __restrict__ K, int n, int64_t ld,
                                                                const Entry* __restrict__ seg,
                                                                const int* __restrict__ seg_cnt, int n_seg,
                                                                const uint8_t* __restrict__ cand,
                                                                double* __restrict__ gain) {
    __shared__ Entry se[STAGE];
    const int c = blockIdx.x * COL_THREADS + threadIdx.x;
    const bool live = c < n && cand[c];
    double acc = 0.0;
    for (int b = 0; b < n_seg; ++b) {
        const int cnt = seg_cnt[b];
        for (int e0 = 0; e0 < cnt; e0 += STAGE) {
            const int len = min(STAGE, cnt - e0);
            __syncthreads();
            if (threadIdx.x < len) se[threadIdx.x] = seg[b * SEG + e0 + threadIdx.x];
            __syncthreads();
            if (live) {
#pragma unroll 8
                for (int e = 0; e < len; ++e) {
                    const double k = static_cast<double>(__ldg(K + static_cast<int64_t>(se[e].row) * ld + c));
                    const double t1 = fmax(0.0, __dsub_rn(k, static_cast<double>(se[e].m_old)));
                    const double t2 = fmax(0.0, __dsub_rn(k, static_cast<double>(se[e].kc)));
                    acc = __dadd_rn(acc, __dsub_rn(t1, t2));
                }
            }
        }
    }
    if (live) gain[c] = __dsub_rn(gain[c], acc);
}

}  // namespace herd

extern "C" int alq_herding_select(alq_ctx* ctx, const float* k, int64_t n, int64_t ldk, const uint8_t* labeled,
                                  const uint8_t* avail, int64_t budget, int32_t* picks, float* m, int64_t* n_picks_host,
                                  int64_t* sum_s_host, void* stream) {
    using namespace herd;
    if (!ctx) return ALQ_ERR_INVALID;
    if (!k || !labeled || !avail || !picks || !m || !n_picks_host || n < 1 || n >= (1LL << 31) - SEG || ldk < n ||
        budget < 0)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_herding_select: bad arguments (n=%lld ldk=%lld budget=%lld)", (long long)n,
                 (long long)ldk, (long long)budget);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ni = static_cast<int>(n);
    const int n_col = (ni + COL_THREADS - 1) / COL_THREADS;
    const int n_seg = (ni + SEG - 1) / SEG;
    const int n_part = std::min(ctx->sm_count, (ni + ARG_THREADS - 1) / ARG_THREADS);
    double *gain, *part_g;
    uint8_t* cand;
    Entry* seg;
    int *seg_cnt, *part_p, *n_avail;
    unsigned long long* s_total;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        gain = cur.take<double>(n);
        cand = cur.take<uint8_t>(n);
        seg = cur.take<Entry>(static_cast<size_t>(n_seg) * SEG);
        seg_cnt = cur.take<int>(n_seg);
        part_g = cur.take<double>(n_part);
        part_p = cur.take<int>(n_part);
        s_total = cur.take<unsigned long long>(1);
        n_avail = cur.take<int>(1);
    });
    if (rc) return rc;

    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    ALQ_CUDA(ctx, cudaMemcpyAsync(cand, avail, static_cast<size_t>(n), cudaMemcpyDeviceToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(s_total, 0, 8, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(n_avail, 0, 4, st));
    hs_m_kernel<<<n_col, COL_THREADS, 0, st>>>(k, ni, ldk, labeled, m);
    ALQ_LAUNCH_CHECK(ctx);
    hs_gain_kernel<<<n_col, COL_THREADS, 0, st>>>(k, ni, ldk, m, avail, gain, n_avail);
    ALQ_LAUNCH_CHECK(ctx);
    int h_avail = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h_avail, n_avail, 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    const int steps = static_cast<int>(std::min<int64_t>(budget, h_avail));
    for (int t = 0; t < steps; ++t) {
        hs_argmax_kernel<<<n_part, ARG_THREADS, 0, st>>>(gain, cand, ni, part_g, part_p);
        ALQ_LAUNCH_CHECK(ctx);
        hs_cover_kernel<<<n_seg, SEG, 0, st>>>(k, ni, ldk, part_g, part_p, n_part, m, cand, seg, seg_cnt, picks, t,
                                               s_total);
        ALQ_LAUNCH_CHECK(ctx);
        if (t + 1 < steps) {                           // the last pick's gains are never read
            hs_update_kernel<<<n_col, COL_THREADS, 0, st>>>(k, ni, ldk, seg, seg_cnt, n_seg, cand, gain);
            ALQ_LAUNCH_CHECK(ctx);
        }
    }
    unsigned long long h_s = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h_s, s_total, 8, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    *n_picks_host = steps;
    if (sum_s_host) *sum_s_host = static_cast<int64_t>(h_s);
    return ALQ_OK;
}

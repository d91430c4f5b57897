// K6: MASE / BASE (SURVEY.md section 8f rank 2) -- distance of every pool embedding to the pairwise decision
// boundaries of the linear head, and the class-balanced selection built on it.
//
// Reference semantics (under active_learning/src/query_strategies): mase_sampler.py:52-80 broadcasts
// (B, C, M) tensors per loader batch to get  radius[i, c] = | -(w_p - w_c) * lam / 2 |,
// lam = 2 (h_i.(w_p - w_c) + b_p - b_c) / |w_p - w_c|^2,  p = argmax_c z_i.  With the algebra carried out,
// h_i.(w_p - w_c) + b_p - b_c is the logit gap z_ip - z_ic and the radius is |z_ip - z_ic| / |w_p - w_c|:
// a C x C table of head geometry (computed once per query) and one streaming pass over the logits slab, the same
// [N, C] input K1 reads.  NaN (c == p, duplicated class rows: 0/0, x/0 * 0) becomes +inf like :77.
// base_sampler.py:22-38 then selects class by class; alq_base_select runs that loop on the stream with K1b.
#include <limits.h>

#include <algorithm>

#include "alq_common.cuh"
#include "alq_mase_rows.cuh"

namespace {

constexpr int kMaseThreads = 256;
constexpr int kGapTile = 64;
constexpr int kGapK = 32;
constexpr int kGapLd = kGapK + 4;     // row pitch 36 floats: 16-byte aligned, 128-bit loads of 16 consecutive rows hit 8 bank groups x 2

// ginv[a, c] = 1 / |w_a - w_c|  (IEEE sqrt and division; +inf where the rows coincide, incl. the diagonal).
// den is the direct sum of squared differences like mase_sampler.py:71 (not the |a|^2+|c|^2-2ac expansion, which
// cancels for nearby class rows).  64 x 64 output tile per CTA, 4 x 4 per thread (rows ty + 16 i, columns tx + 16 j:
// conflict-free 128-bit shared loads along k), operand chunks of 32 k fetched with coalesced 128-bit loads one chunk
// ahead of the math.  The table is symmetric: only tiles on or above the diagonal are computed, and mirrored on the way out.
__device__ __forceinline__ float4 gap_load4(const float* __restrict__ w, int row, int c, int k, int m, int64_t ldw, bool vec) {
    if (row >= c || k >= m) return make_float4(0.f, 0.f, 0.f, 0.f);
    const float* p = w + static_cast<int64_t>(row) * ldw + k;
    if (vec && k + 3 < m) return *reinterpret_cast<const float4*>(p);
    float4 r = make_float4(p[0], 0.f, 0.f, 0.f);
    if (k + 1 < m) r.y = p[1];
    if (k + 2 < m) r.z = p[2];
    if (k + 3 < m) r.w = p[3];
    return r;
}

__global__ void __launch_bounds__(256)
class_gap_inv_kernel(const float* __restrict__ w, int c, int m, int64_t ldw, int vec, float* __restrict__ ginv, int64_t ldg) {
    // linear block index -> tile (by, bx) with bx >= by: row by holds tiles - by entries
    int by = 0, rem = blockIdx.x;
    const int tiles = (c + kGapTile - 1) / kGapTile;
    while (rem >= tiles - by) { rem -= tiles - by; ++by; }
    const int bx = by + rem;
    __shared__ __align__(16) float sa[kGapTile][kGapLd];
    __shared__ __align__(16) float sb[kGapTile][kGapLd];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int a0 = by * kGapTile, c0 = bx * kGapTile;
    // fill mapping: 512 float4 per operand chunk, two per thread; 8 consecutive threads cover one row's 128 bytes
    const int fr = threadIdx.x >> 3, fq = (threadIdx.x & 7) * 4;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 pa[2], pb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        pa[h] = gap_load4(w, a0 + fr + 32 * h, c, fq, m, ldw, vec);
        pb[h] = gap_load4(w, c0 + fr + 32 * h, c, fq, m, ldw, vec);
    }
    for (int k0 = 0; k0 < m; k0 += kGapK) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            *reinterpret_cast<float4*>(&sa[fr + 32 * h][fq]) = pa[h];
            *reinterpret_cast<float4*>(&sb[fr + 32 * h][fq]) = pb[h];
        }
        __syncthreads();
        if (k0 + kGapK < m) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                pa[h] = gap_load4(w, a0 + fr + 32 * h, c, k0 + kGapK + fq, m, ldw, vec);
                pb[h] = gap_load4(w, c0 + fr + 32 * h, c, k0 + kGapK + fq, m, ldw, vec);
            }
        }
#pragma unroll
        for (int k4 = 0; k4 < kGapK; k4 += 4) {
            float4 av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                av[i] = *reinterpret_cast<const float4*>(&sa[ty + 16 * i][k4]);
                bv[i] = *reinterpret_cast<const float4*>(&sb[tx + 16 * i][k4]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float d = av[i].x - bv[j].x;
                    acc[i][j] = fmaf(d, d, acc[i][j]);
                    d = av[i].y - bv[j].y;
                    acc[i][j] = fmaf(d, d, acc[i][j]);
                    d = av[i].z - bv[j].z;
                    acc[i][j] = fmaf(d, d, acc[i][j]);
                    d = av[i].w - bv[j].w;
                    acc[i][j] = fmaf(d, d, acc[i][j]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int a = a0 + ty + 16 * i, cc = c0 + tx + 16 * j;
            if (a < c && cc < c) {
                const float g = (a != cc) ? __fdiv_rn(1.0f, __fsqrt_rn(acc[i][j])) : ALQ_POS_INF;
                ginv[static_cast<int64_t>(a) * ldg + cc] = g;
                ginv[static_cast<int64_t>(cc) * ldg + a] = g;
            }
        }
}

// gmin[a] = min_c ginv[a, c]: the reciprocal of the largest distance from class a to any other class row, and
// gmin[C] = max_a (largest finite ginv[a, :]) / gmin[a], how unevenly the class rows are spread (>= 1; the pruning
// bound of mase_row_min_smem).  Also fills the pad columns c..ldg-1 of row a with +inf.  One warp per class row.
__global__ void __launch_bounds__(256)
class_gap_rowmin_kernel(float* __restrict__ ginv, int c, int64_t ldg, float* __restrict__ gmin) {
    const int lane = threadIdx.x & 31;
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= c) return;
    float* g = ginv + static_cast<int64_t>(row) * ldg;
    float mn = ALQ_POS_INF, mx = 0.f;
    for (int j = lane; j < c; j += 32) {
        const float v = g[j];
        mn = fminf(mn, v);
        if (v < ALQ_POS_INF) mx = fmaxf(mx, v);
    }
    for (int j = c + lane; j < ldg; j += 32) g[j] = ALQ_POS_INF;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (lane == 0 && gmin) {
        gmin[row] = mn;
        const float ratio = __fdiv_ru(mx, mn);            // mn = 0 or inf, mx = 0: inf / NaN / 0 -> handled below
        if (ratio >= 1.0f)                                // positive floats order like their bit patterns
            atomicMax(reinterpret_cast<int*>(gmin + c), ratio < ALQ_POS_INF ? __float_as_int(ratio) : 0x7f800000);
    }
}

__global__ void gap_ratio_init_kernel(float* __restrict__ gmin, int c) { gmin[c] = 1.0f; }

// One warp per row, the row held as NV float4 per lane between the arg-max pass and the radius pass
// (row code: alq_mase_rows.cuh).
template <int NV>
__device__ __forceinline__ void load_row_regs(const float* logits, int64_t row, int64_t ld, int lane, int nvec,
                                              MaseRowRegs<NV>& r) {
    const float4* p = reinterpret_cast<const float4*>(logits + row * ld);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int idx = lane + 32 * k;
        r.v[k] = idx < nvec ? ld_stream_f4(p + idx) : make_float4(ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF);
    }
}

template <int NV, bool WRITE_R>
__global__ void __launch_bounds__(kMaseThreads)
mase_rows_vec_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, const float* __restrict__ ginv,
                     int64_t ldg, float* __restrict__ minm, int32_t* __restrict__ pred, float* __restrict__ radius,
                     int64_t ldr) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int nvec = c >> 2;
    for (int64_t row = warp; row < n; row += nwarps) {
        MaseRowRegs<NV> r;
        load_row_regs<NV>(logits, row, ld, lane, nvec, r);
        float mn;
        int arg;
        mase_row_full<NV, WRITE_R>(r, lane, nvec, ginv, ldg, WRITE_R ? reinterpret_cast<float4*>(radius + row * ldr) : nullptr,
                                   mn, arg);
        if (lane == 0) { minm[row] = mn; pred[row] = arg; }
    }
}

template <int NV>
__global__ void __launch_bounds__(kMaseThreads)
mase_rows_min_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, const float* __restrict__ ginv,
                     int64_t ldg, const float* __restrict__ gmin, float* __restrict__ minm, int32_t* __restrict__ pred) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int nvec = c >> 2;
    for (int64_t row = warp; row < n; row += nwarps) {
        MaseRowRegs<NV> r;
        load_row_regs<NV>(logits, row, ld, lane, nvec, r);
        float mn;
        int arg;
        mase_row_min<NV>(r, lane, c, ginv, ldg, gmin, mn, arg);
        if (lane == 0) { minm[row] = mn; pred[row] = arg; }
    }
}

// Any c / alignment: two passes over the row, the second one hits L1/L2.
__global__ void __launch_bounds__(kMaseThreads)
mase_rows_generic_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, const float* __restrict__ ginv,
                         int64_t ldg, float* __restrict__ minm, int32_t* __restrict__ pred, float* __restrict__ radius,
                         int64_t ldr) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t row = warp; row < n; row += nwarps) {
        const float* p = logits + row * ld;
        float best = ALQ_NEG_INF;
        int arg = INT_MAX;
        for (int j = lane; j < c; j += 32) {
            const float z = p[j];
            if (mase_beats(z, best)) { best = z; arg = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            mase_argmax_merge(best, arg, ob, oa);
        }
        if (arg == INT_MAX) arg = 0;
        const float* gi = ginv + static_cast<int64_t>(arg) * ldg;
        float mn = ALQ_POS_INF;
        for (int j = lane; j < c; j += 32) {
            const float r = mase_radius_of(best, p[j], __ldg(gi + j), j == arg);
            mn = fminf(mn, r);
            if (radius) radius[row * ldr + j] = r;
        }
        if (radius)
            for (int j = c + lane; j < ldr; j += 32) radius[row * ldr + j] = ALQ_POS_INF;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        if (lane == 0) { minm[row] = mn; pred[row] = arg; }
    }
}

// base_sampler.py:29-33: the key class `cls` sorts by; rows taken by earlier classes are pushed to +inf.
__global__ void __launch_bounds__(256)
base_keys_kernel(const float* __restrict__ minm, const float* __restrict__ radius, int64_t ldr,
                 const int32_t* __restrict__ pred, const unsigned char* __restrict__ taken, int64_t n, int cls,
                 float* __restrict__ keys) {
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float k = (pred[i] == cls) ? minm[i] : radius[i * ldr + cls];
        keys[i] = taken[i] ? ALQ_POS_INF : k;
    }
}

// marks this class's picks; a row picked twice (only possible once every free key is +inf) is what the
// reference's `assert len(labeled_idxs) == len(set(labeled_idxs))` (:40) trips on -> counted in dup[0].
__global__ void base_mark_kernel(const int32_t* __restrict__ picks, int cnt, unsigned char* __restrict__ taken,
                                 unsigned int* __restrict__ dup) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cnt) {
        const int32_t r = picks[i];
        if (taken[r]) atomicAdd(dup, 1u);
        taken[r] = 1;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// BASE with many classes and few picks per class (ImageNet: 1000 classes x 10): the class loop above is 1000 dependent
// selections of ~30 us.  The dependence is only through the set of rows already taken, so it is split in two:
//
//   base_candidates_kernel  every class at once: the kBaseList smallest (key, row) pairs of each class, ignoring what
//                           other classes take.  One CTA owns 8 adjacent classes (the 32-byte sector of a radius row),
//                           streams the pool once, and every thread keeps the 3 smallest pairs it has seen per class in
//                           shared memory plus, in a register, the smallest pair it dropped; the class's true top list
//                           is inside the union of the kept pairs unless a dropped pair sorts before the list's last
//                           entry -- checked exactly and reported in fail[class] (about 1e-4 per class).
//   base_resolve_kernel     one warp walks the classes in order against a shared-memory bitset of taken rows: the first
//                           cnt free rows of a class's list are what the sequential loop would have selected, provided
//                           the list holds that many free rows with a finite key.  Otherwise it stops at that class; the
//                           host runs the ordinary step for it and resumes after it.
// The result is identical to the sequential loop (tests compare both with the oracle).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kBaseGroup = 8;          // classes per CTA
constexpr int kBaseThreads = 1024;
constexpr int kBaseKeep = 3;           // pairs kept per thread and class
constexpr int kBaseList = 64;          // candidate list length per class
constexpr int kBaseMaxCnt = 32;        // picks per class the parallel path accepts (list = cnt + 32 spare)
constexpr unsigned long long kBaseEmpty = ~0ull;

__device__ __forceinline__ unsigned long long base_pack(float key, uint32_t row) {
    return (static_cast<unsigned long long>(alq_ord(key + 0.0f)) << 32) | row;
}

__global__ void __launch_bounds__(kBaseThreads, 1)
base_candidates_kernel(const float* __restrict__ minm, const float* __restrict__ radius, int64_t ldr,
                       const int32_t* __restrict__ pred, int n, int c, int64_t budget,
                       unsigned long long* __restrict__ cand_out, int* __restrict__ fail_out) {
    extern __shared__ __align__(16) unsigned char smem_base[];
    unsigned long long* cand = reinterpret_cast<unsigned long long*>(smem_base);          // [group][keep][threads]
    unsigned long long* tmp = cand + kBaseGroup * kBaseKeep * kBaseThreads;                // [2 * kBaseList]
    const int tid = threadIdx.x;
    const int c0 = blockIdx.x * kBaseGroup;
    for (int i = tid; i < kBaseGroup * kBaseKeep * kBaseThreads; i += kBaseThreads) cand[i] = kBaseEmpty;
    __syncthreads();
    unsigned long long fourth[kBaseGroup];       // smallest pair this thread did NOT keep, per class
#pragma unroll
    for (int j = 0; j < kBaseGroup; ++j) fourth[j] = kBaseEmpty;
    for (int i = tid; i < n; i += kBaseThreads) {
        const int p = pred[i];
        const float mm = minm[i];
        const float* rrow = radius + static_cast<int64_t>(i) * ldr + c0;
#pragma unroll
        for (int j = 0; j < kBaseGroup; ++j) {
            if (c0 + j < c) {
                const float key = (p == c0 + j) ? mm : rrow[j];
                const unsigned long long w = base_pack(key, static_cast<uint32_t>(i));
                if (w < fourth[j]) {                            // rare after the first few rows
                    unsigned long long* slot = cand + static_cast<size_t>(j) * kBaseKeep * kBaseThreads + tid;
                    const unsigned long long k0 = slot[0], k1 = slot[kBaseThreads], k2 = slot[2 * kBaseThreads];
                    if (w < k2) {                               // joins the kept three; the largest of them is dropped
                        fourth[j] = k2;
                        if (w < k0) { slot[0] = w; slot[kBaseThreads] = k0; slot[2 * kBaseThreads] = k1; }
                        else if (w < k1) { slot[kBaseThreads] = w; slot[2 * kBaseThreads] = k1; }
                        else slot[2 * kBaseThreads] = w;
                    } else {
                        fourth[j] = w;
                    }
                }
            }
        }
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < kBaseGroup; ++j) {
        const int cls = c0 + j;
        if (cls >= c) break;
        const int64_t cnt = budget / c + (cls < budget % c ? 1 : 0);
        if (cnt == 0) continue;                                 // uniform per CTA
        unsigned long long* mine = cand + static_cast<size_t>(j) * kBaseKeep * kBaseThreads;
        unsigned long long my_dropped = fourth[0];              // fourth[j] without dynamic indexing (keeps it in registers)
#pragma unroll
        for (int q = 1; q < kBaseGroup; ++q)
            if (j == q) my_dropped = fourth[q];
        const int len = static_cast<int>(cnt < kBaseList - 32 ? cnt + 32 : kBaseList);
        alq_bitonic_sort_smem(mine, 2 * kBaseThreads);          // slots 0 and 1 of every thread
        alq_bitonic_sort_smem(mine + 2 * kBaseThreads, kBaseThreads);   // slot 2
        if (tid < kBaseList) { tmp[tid] = mine[tid]; tmp[kBaseList + tid] = mine[2 * kBaseThreads + tid]; }
        __syncthreads();
        alq_bitonic_sort_smem(tmp, 2 * kBaseList);
        const unsigned long long last = tmp[len - 1];
        // the list is the exact top-`len` unless some thread dropped a pair that sorts before the list's last entry
        const int bad = __syncthreads_or(my_dropped < last);
        if (tid < kBaseList) cand_out[static_cast<size_t>(cls) * kBaseList + tid] = tid < len ? tmp[tid] : kBaseEmpty;
        if (tid == 0) fail_out[cls] = bad;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kBaseThreads, 1)
base_resolve_kernel(const unsigned long long* __restrict__ cand, const int* __restrict__ fail, unsigned char* __restrict__ taken,
                    int n, int c, int64_t budget, int c_begin, int chunk, int32_t* __restrict__ out_pos, int* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char smem_base[];
    const int words = (n + 31) / 32;
    unsigned long long* lst = reinterpret_cast<unsigned long long*>(smem_base);            // [chunk][kBaseList]
    int* lfail = reinterpret_cast<int*>(lst + static_cast<size_t>(chunk) * kBaseList);     // [chunk]
    uint32_t* bits = reinterpret_cast<uint32_t*>(lfail + chunk);                           // [words]
    __shared__ int s_stop;
    for (int w = threadIdx.x; w < words; w += kBaseThreads) {
        uint32_t v = 0;
        const int lo = w * 32, hi = min(n, lo + 32);
        for (int i = lo; i < hi; ++i) v |= (taken[i] ? 1u : 0u) << (i - lo);
        bits[w] = v;
    }
    if (threadIdx.x == 0) s_stop = -1;
    const int lane = threadIdx.x & 31;
    const int64_t per = budget / c, extra = budget % c;
    const uint32_t ord_inf = 0xff800000u;                        // alq_ord(+inf)
    for (int base = c_begin; base < c; base += chunk) {
        // every thread stages the candidate lists of the next `chunk` classes; one warp then resolves them in order
        const int cnt_cls = min(chunk, c - base);
        for (int i = threadIdx.x; i < cnt_cls * kBaseList; i += kBaseThreads) lst[i] = cand[static_cast<size_t>(base) * kBaseList + i];
        for (int i = threadIdx.x; i < cnt_cls; i += kBaseThreads) lfail[i] = fail[base + i];
        __syncthreads();
        if (threadIdx.x < 32) {
            for (int q = 0; q < cnt_cls; ++q) {
                const int cls = base + q;
                const int cnt = static_cast<int>(per + (cls < extra ? 1 : 0));
                if (cnt == 0) continue;
                const int64_t off = static_cast<int64_t>(cls) * per + min(static_cast<int64_t>(cls), extra);
                const int len = min(cnt + 32, kBaseList);
                const unsigned long long e0 = lst[q * kBaseList + lane], e1 = lst[q * kBaseList + 32 + lane];
                const uint32_t r0 = static_cast<uint32_t>(e0), r1 = static_cast<uint32_t>(e1);
                const bool v0 = lane < len && static_cast<uint32_t>(e0 >> 32) < ord_inf && !((bits[r0 >> 5] >> (r0 & 31)) & 1u);
                const bool v1 = lane + 32 < len && static_cast<uint32_t>(e1 >> 32) < ord_inf && !((bits[r1 >> 5] >> (r1 & 31)) & 1u);
                const uint32_t b0 = __ballot_sync(0xffffffffu, v0), b1 = __ballot_sync(0xffffffffu, v1);
                if (lfail[q] || __popc(b0) + __popc(b1) < cnt) {          // list not provably complete, or too few free rows
                    if (lane == 0) s_stop = cls;
                    break;
                }
                const uint32_t lt = (1u << lane) - 1u;
                const int k0 = __popc(b0 & lt), k1 = __popc(b0) + __popc(b1 & lt);
                if (v0 && k0 < cnt) { out_pos[off + k0] = static_cast<int32_t>(r0); atomicOr(&bits[r0 >> 5], 1u << (r0 & 31)); taken[r0] = 1; }
                if (v1 && k1 < cnt) { out_pos[off + k1] = static_cast<int32_t>(r1); atomicOr(&bits[r1 >> 5], 1u << (r1 & 31)); taken[r1] = 1; }
                __syncwarp();
            }
        }
        __syncthreads();
        if (s_stop >= 0) break;
    }
    if (threadIdx.x == 0) *status = s_stop >= 0 ? s_stop : c;
}

int rows_grid(const alq_ctx* ctx, int64_t n, int warps_per_block) {
    int64_t need = (n + warps_per_block - 1) / warps_per_block;
    const int64_t cap = static_cast<int64_t>(ctx->sm_count) * 8;
    if (need < 1) need = 1;
    return static_cast<int>(need < cap ? need : cap);
}

template <int NV>
void launch_mase_vec(int grid, cudaStream_t st, const float* logits, int64_t n, int c, int64_t ld, const float* ginv,
                     int64_t ldg, float* minm, int32_t* pred, float* radius, int64_t ldr) {
    if (radius)
        mase_rows_vec_kernel<NV, true><<<grid, kMaseThreads, 0, st>>>(logits, n, c, ld, ginv, ldg, minm, pred, radius, ldr);
    else
        mase_rows_vec_kernel<NV, false><<<grid, kMaseThreads, 0, st>>>(logits, n, c, ld, ginv, ldg, minm, pred, radius, ldr);
}

template <int NV>
void launch_mase_min(int grid, cudaStream_t st, const float* logits, int64_t n, int c, int64_t ld, const float* ginv,
                     int64_t ldg, const float* gmin, float* minm, int32_t* pred) {
    mase_rows_min_kernel<NV><<<grid, kMaseThreads, 0, st>>>(logits, n, c, ld, ginv, ldg, gmin, minm, pred);
}

}  // namespace

extern "C" int alq_class_gap_inv(alq_ctx* ctx, const float* weight, int32_t c, int32_t m, int64_t ldw, float* ginv,
                                 int64_t ldg, float* gmin, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (c <= 0 || m <= 0 || ldw < m || ldg < c) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_gap_inv: bad shape (c=%d m=%d ldw=%lld ldg=%lld)", c, m, (long long)ldw, (long long)ldg);
    if (!weight || !ginv) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_gap_inv: null pointer");
    const unsigned tiles = static_cast<unsigned>((c + kGapTile - 1) / kGapTile);
    class_gap_inv_kernel<<<tiles * (tiles + 1) / 2, 256, 0, static_cast<cudaStream_t>(stream)>>>(weight, c, m, ldw, (ldw % 4 == 0) && aligned16(weight), ginv, ldg);
    ALQ_LAUNCH_CHECK(ctx);
    if (gmin) {
        gap_ratio_init_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(gmin, c);
        ALQ_LAUNCH_CHECK(ctx);
    }
    class_gap_rowmin_kernel<<<(c + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(ginv, c, ldg, gmin);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_mase_margins(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, const float* ginv,
                                int64_t ldg, const float* gmin, float* min_margin, int32_t* pred, float* radius, int64_t ldr,
                                void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || c <= 0 || ld < c || ldg < c || (radius && ldr < c)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_mase_margins: bad shape");
    if (n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_mase_margins: n must be < 2^31");
    if (n == 0) return ALQ_OK;
    if (!logits || !ginv || !min_margin || !pred) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_mase_margins: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = rows_grid(ctx, n, kMaseThreads / 32);
    const bool vec = (c % 4 == 0) && (ld % 4 == 0) && (ldg % 4 == 0) && aligned16(logits) && aligned16(ginv) &&
                     (!radius || ((ldr % 4 == 0) && ldr == c && aligned16(radius))) && c <= 1024;
    if (vec && ld == c && (radius ? ldr == c : gmin != nullptr) && n >= 4096) {
        // bulk-copy pipelined kernel (the K1 / K2 pipeline with the K6 row code)
        const MaseArgs margs{ginv, ldg, gmin, pred, radius, ldr};
        cudaError_t e = cudaSuccess;
        if (alq_mase_rows_pipe(ctx, st, logits, n, c, margs, min_margin, &e)) {
            ctx->launches++;
            if (e != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "rows_pipe_kernel (K6) launch failed: %s", cudaGetErrorString(e));
            return ALQ_OK;
        }
    }
    if (vec && !radius && gmin) {       // MASE: exact minimum with table reads pruned by gmin
        const int nv = (c / 4 + 31) / 32;
        switch (nv) {
            case 1: launch_mase_min<1>(grid, st, logits, n, c, ld, ginv, ldg, gmin, min_margin, pred); break;
            case 2: launch_mase_min<2>(grid, st, logits, n, c, ld, ginv, ldg, gmin, min_margin, pred); break;
            case 3: case 4: launch_mase_min<4>(grid, st, logits, n, c, ld, ginv, ldg, gmin, min_margin, pred); break;
            default: launch_mase_min<8>(grid, st, logits, n, c, ld, ginv, ldg, gmin, min_margin, pred); break;
        }
    } else if (vec) {
        const int nv = (c / 4 + 31) / 32;
        switch (nv) {
            case 1: launch_mase_vec<1>(grid, st, logits, n, c, ld, ginv, ldg, min_margin, pred, radius, ldr); break;
            case 2: launch_mase_vec<2>(grid, st, logits, n, c, ld, ginv, ldg, min_margin, pred, radius, ldr); break;
            case 3: case 4: launch_mase_vec<4>(grid, st, logits, n, c, ld, ginv, ldg, min_margin, pred, radius, ldr); break;
            default: launch_mase_vec<8>(grid, st, logits, n, c, ld, ginv, ldg, min_margin, pred, radius, ldr); break;
        }
    } else {
        mase_rows_generic_kernel<<<grid, kMaseThreads, 0, st>>>(logits, n, c, ld, ginv, ldg, min_margin, pred, radius, ldr);
    }
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_base_select(alq_ctx* ctx, const float* min_margin, const float* radius, int64_t ldr, const int32_t* pred,
                               int64_t n, int32_t c, int64_t budget, int32_t* out_pos, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || c <= 0 || ldr < c || budget < 0 || budget > n || n >= (1LL << 31))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_base_select: need 0 <= budget <= n < 2^31, ldr >= c (n=%lld budget=%lld)", (long long)n, (long long)budget);
    if (budget == 0) return ALQ_OK;
    if (!min_margin || !radius || !pred || !out_pos) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_base_select: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t cnt_max = budget / c + (budget % c ? 1 : 0);
    const size_t bitset_bytes = (static_cast<size_t>(n) + 31) / 32 * 4;
    const size_t cand_smem = (static_cast<size_t>(kBaseGroup) * kBaseKeep * kBaseThreads + 2 * kBaseList) * sizeof(unsigned long long);
    // many classes, few picks each: candidate lists for every class at once + an in-order resolve (base_impl: 1 = never)
    const size_t per_class_smem = kBaseList * sizeof(unsigned long long) + sizeof(int);
    const bool parallel = ctx->base_impl != 1 && cnt_max <= kBaseMaxCnt && (c >= 16 || ctx->base_impl == 2) &&
                          bitset_bytes + 8 * per_class_smem + 1024 <= ctx->smem_optin && cand_smem + 1024 <= ctx->smem_optin;
    // the resolve kernel stages `chunk` candidate lists at a time next to its bitset of taken rows
    const int chunk = parallel ? static_cast<int>(std::min<size_t>(256, (ctx->smem_optin - 1024 - bitset_bytes) / per_class_smem)) : 0;
    const size_t resolve_smem = chunk * per_class_smem + bitset_bytes;
    // private arena: alq_select_smallest re-carves the shared scratch on every call
    int rc = alq_arena2_reserve(ctx, scratch_need({static_cast<size_t>(n) * sizeof(float), static_cast<size_t>(n), sizeof(unsigned int),
                                                   static_cast<size_t>(c) * kBaseList * sizeof(unsigned long long),
                                                   static_cast<size_t>(c) * sizeof(int), sizeof(int)}));
    if (rc) return rc;
    ScratchCursor cur(ctx->arena2);
    float* keys = cur.take<float>(n);
    unsigned char* taken = cur.take<unsigned char>(n);
    unsigned int* dup = cur.take<unsigned int>(1);
    unsigned long long* cand = cur.take<unsigned long long>(static_cast<size_t>(c) * kBaseList);
    int* fail = cur.take<int>(c);
    int* status = cur.take<int>(1);
    ALQ_CUDA(ctx, cudaMemsetAsync(taken, 0, static_cast<size_t>(n), st));
    ALQ_CUDA(ctx, cudaMemsetAsync(dup, 0, sizeof(unsigned int), st));
    int kgrid = static_cast<int>((n + 255) / 256);
    if (kgrid > ctx->sm_count * 8) kgrid = ctx->sm_count * 8;
    // one ordinary step of the class loop (base_sampler.py:29-38) for class `cls`
    auto class_step = [&](int cls) -> int {
        const int64_t cnt = budget / c + (cls < budget % c ? 1 : 0);      // base_sampler.py:24-25
        if (cnt == 0) return ALQ_OK;
        const int64_t at = static_cast<int64_t>(cls) * (budget / c) + std::min<int64_t>(cls, budget % c);
        base_keys_kernel<<<kgrid, 256, 0, st>>>(min_margin, radius, ldr, pred, taken, n, cls, keys);
        ALQ_LAUNCH_CHECK(ctx);
        const int r = alq_select_smallest(ctx, keys, n, cnt, out_pos + at, stream);
        if (r) return r;
        base_mark_kernel<<<static_cast<int>((cnt + 255) / 256), 256, 0, st>>>(out_pos + at, static_cast<int>(cnt), taken, dup);
        ALQ_LAUNCH_CHECK(ctx);
        return ALQ_OK;
    };
    if (parallel) {
        ALQ_CUDA(ctx, cudaFuncSetAttribute(base_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(cand_smem)));
        ALQ_CUDA(ctx, cudaFuncSetAttribute(base_resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(resolve_smem)));
        base_candidates_kernel<<<(c + kBaseGroup - 1) / kBaseGroup, kBaseThreads, cand_smem, st>>>(
            min_margin, radius, ldr, pred, static_cast<int>(n), c, budget, cand, fail);
        ALQ_LAUNCH_CHECK(ctx);
        int cls = 0;
        while (cls < c) {
            base_resolve_kernel<<<1, kBaseThreads, resolve_smem, st>>>(cand, fail, taken, static_cast<int>(n), c, budget, cls, chunk, out_pos, status);
            ALQ_LAUNCH_CHECK(ctx);
            int stopped = c;
            ALQ_CUDA(ctx, cudaMemcpyAsync(&stopped, status, sizeof(int), cudaMemcpyDeviceToHost, st));
            ALQ_CUDA(ctx, cudaStreamSynchronize(st));
            if (stopped >= c) break;
            rc = class_step(stopped);          // a list that was too short (or not provably complete): the ordinary step
            if (rc) return rc;
            cls = stopped + 1;
        }
    } else {
        for (int cls = 0; cls < c; ++cls) {
            rc = class_step(cls);
            if (rc) return rc;
        }
    }
    unsigned int dup_host = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&dup_host, dup, sizeof(dup_host), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (dup_host) ALQ_FAIL(ctx, ALQ_ERR_NUMERIC, "alq_base_select: %u rows were selected twice (every free key is +inf; base_sampler.py:40 asserts here)", dup_host);
    return ALQ_OK;
}

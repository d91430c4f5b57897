// K4 / K5: the sequential selection loop of CoreSet (greedy k-center) and BADGE (k-means++ D^2
// seeding) -- the device replacement of `CoresetSampler.coreset` (coreset_sampler.py:66-105 under
// active_learning/src/query_strategies).
//
// Per step the reference re-gathers an N x L slice of the dense distance matrix and re-mins it
// (:79).  Here each step streams the candidate rows once: d2(i, centre) in the reference's own
// expression order fl(fl(n_i + n_q) - 2*dot), a running min into mind[i], and then either
//   * arg-max (lowest row on ties, :94): per-CTA best key -> atomicMax on a 64-bit slot per step, or
//   * D^2 sampling (:84-92): clip/zero -> NumPy's fp32 pairwise-sum tree -> p = c/S -> fp64 cdf ->
//     first k with cdf[k]/total > u  (np.random.choice), with the `+= 1e-5` NaN retry.
// Rows are either dense (x[n,d]) or BADGE's rank-1 factors (a[n,c], x[n,d]); the 2048*1000-d
// gradient embedding is never formed:  <g_i,g_q> = <a_i,a_q><h_i,h_q>,  |g|^2 = |a|^2|h|^2.
// Partitions are a batch dimension: every launch advances all partitions by one step.
//
// This file holds the entry point and the ONE-LAUNCH-PER-STEP variants (single GPU; kept as fallback and as the
// comparison the persistent kernel is tested against).  The default, and the only multi-GPU form, is variant 3 in
// alq_greedy_persist.cu: one persistent cooperative launch for the whole loop.
// The streaming kernel is HBM-bound: 4*d (+4*c) + 12 bytes per row per step.  Two variants here:
//   variant 1  direct 128-bit L1-bypassing loads, one warp per row;
//   variant 2  warp-specialised: one producer lane feeds a ring of shared-memory stages with
//              cp.async.bulk (TMA bulk copies, mbarrier complete_tx), consumer warps do the dots.
#include <math.h>
#include <stdlib.h>

#include "alq_greedy.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// shared argument blocks
// ------------------------------------------------------------------------------------------------
struct StepArgs {
    const float* x;  int64_t ldx; int d;
    const float* a;  int64_t lda; int c;
    const float* xn; const float* an;
    float* mind;
    const BlockSeg* segs;
    const int* budget;              // [P]
    int P;
    int t;                          // this launch consumes pick t-1 as the centre
    unsigned long long* best;       // [Bmax * P]   arg-max slots
    const int* cur;                 // [P]          current centre (sampling variant)
    const int* vpos;                // [n]
    float* cfull;                   // concatenated per-partition full arrays
    const int* cfull_off;           // [P]
    int* status;
    int* picks;
};

// final per-row bookkeeping, executed by one lane
template <bool SAMPLE>
__device__ __forceinline__ void finish_row(const StepArgs& A, int row, int centre, float m_old, float d2,
                                           int cf_off, unsigned long long& best_key) {
    float m = fminf(m_old, d2);
    if (row == centre) m = ALQ_NEG_INF;   // a picked row is never a candidate again
    A.mind[row] = m;
    if (SAMPLE) {
        A.cfull[cf_off + A.vpos[row]] = m;          // raw running min; the sampling stage clips at 0
    } else {
        const unsigned long long k = alq_maxkey(m, static_cast<uint32_t>(row));
        best_key = k > best_key ? k : best_key;
    }
}

// ---- centre of this step, read from the candidate rows.  Called by every thread of the CTA, followed by
//      __syncthreads() in the caller.
struct CentreInfo { int local; float qn; };

template <bool FACTORED, bool SAMPLE>
__device__ __forceinline__ CentreInfo load_centre(const StepArgs& A, int part, float* sq) {
    const int dv = A.d >> 2, cv = FACTORED ? (A.c >> 2) : 0;
    float4* dst = reinterpret_cast<float4*>(sq);
    const int centre = SAMPLE ? A.cur[part]
                              : static_cast<int>(alq_maxkey_row(__ldcg(&A.best[static_cast<size_t>(A.t - 1) * A.P + part])));
    const float4* src = reinterpret_cast<const float4*>(A.x + static_cast<int64_t>(centre) * A.ldx);
    for (int k = threadIdx.x; k < dv; k += blockDim.x) dst[k] = src[k];
    if (FACTORED) {
        const float4* sa = reinterpret_cast<const float4*>(A.a + static_cast<int64_t>(centre) * A.lda);
        for (int k = threadIdx.x; k < cv; k += blockDim.x) dst[dv + k] = sa[k];
    }
    return CentreInfo{centre, FACTORED ? A.xn[centre] * A.an[centre] : A.xn[centre]};
}

// ------------------------------------------------------------------------------------------------
// variant 1: direct loads
// ------------------------------------------------------------------------------------------------
constexpr int kV1Threads = 256;

template <bool FACTORED, bool SAMPLE>
__global__ void __launch_bounds__(kV1Threads)
step_direct_kernel(StepArgs A) {
    extern __shared__ __align__(16) float sq[];   // centre row: x part then a part
    __shared__ unsigned long long sbest[kV1Threads / 32];
    const BlockSeg seg = A.segs[blockIdx.x];
    if (A.t >= A.budget[seg.part]) return;
    const int dv = A.d >> 2, cv = FACTORED ? (A.c >> 2) : 0;
    const CentreInfo ci = load_centre<FACTORED, SAMPLE>(A, seg.part, sq);
    __syncthreads();
    const int centre = ci.local;
    const float qn = ci.qn;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int cf_off = SAMPLE ? A.cfull_off[seg.part] : 0;
    const float4* q4 = reinterpret_cast<const float4*>(sq);
    unsigned long long best_key = 0ull;
    for (int row = seg.row_lo + wib; row < seg.row_hi; row += kV1Threads / 32) {
        float m_old = 0.f, n_i = 0.f;
        if (lane == 0) {
            m_old = A.mind[row];
            n_i = FACTORED ? A.xn[row] * A.an[row] : A.xn[row];
        }
        const float4* p = reinterpret_cast<const float4*>(A.x + static_cast<int64_t>(row) * A.ldx);
        float dot = 0.f;
#pragma unroll 8
        for (int k = lane; k < dv; k += 32) {
            const float4 v = ld_stream_f4(p + k);
            const float4 w = q4[k];
            dot = fmaf(v.x, w.x, dot);
            dot = fmaf(v.y, w.y, dot);
            dot = fmaf(v.z, w.z, dot);
            dot = fmaf(v.w, w.w, dot);
        }
        dot = warp_sum(dot);
        if (FACTORED) {
            const float4* pa = reinterpret_cast<const float4*>(A.a + static_cast<int64_t>(row) * A.lda);
            float da = 0.f;
#pragma unroll 8
            for (int k = lane; k < cv; k += 32) {
                const float4 v = ld_stream_f4(pa + k);
                const float4 w = q4[dv + k];
                da = fmaf(v.x, w.x, da);
                da = fmaf(v.y, w.y, da);
                da = fmaf(v.z, w.z, da);
                da = fmaf(v.w, w.w, da);
            }
            dot *= warp_sum(da);
        }
        if (lane == 0) finish_row<SAMPLE>(A, row, centre, m_old, dist_dense(n_i, qn, dot), cf_off, best_key);
    }
    if (!SAMPLE) {
        if (lane == 0) sbest[wib] = best_key;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long b = 0ull;
            for (int w = 0; w < kV1Threads / 32; ++w) b = sbest[w] > b ? sbest[w] : b;
            if (b) atomicMax(&A.best[static_cast<size_t>(A.t) * A.P + seg.part], b);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// variant 2: bulk-copy (TMA) pipeline
// ------------------------------------------------------------------------------------------------
template <bool FACTORED, bool SAMPLE>
__global__ void __launch_bounds__(32 * 17, 1)
step_pipe_kernel(StepArgs A, PipeCfg cfg) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int d = A.d, c = FACTORED ? A.c : 0;
    const int dv = d >> 2, cv = c >> 2;
    float* sq = reinterpret_cast<float*>(smem_raw);                          // centre: d + c floats
    float* tiles = sq + ((d + c + 31) & ~31);                                // stage ring
    uint64_t* full = reinterpret_cast<uint64_t*>(tiles + static_cast<size_t>(cfg.stages) * cfg.tile_floats);
    uint64_t* empty = full + cfg.stages;
    unsigned long long* sbest = reinterpret_cast<unsigned long long*>(empty + cfg.stages);

    const BlockSeg seg = A.segs[blockIdx.x];
    if (A.t >= A.budget[seg.part]) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const CentreInfo ci = load_centre<FACTORED, SAMPLE>(A, seg.part, sq);
    const int centre = ci.local;
    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int R = cfg.rows_per_tile;
    const int nrows = seg.row_hi - seg.row_lo;
    const int ntiles = (nrows + R - 1) / R;

    if (warp == 0) {
        // ===== producer: one lane issues every bulk copy =====
        if (lane == 0) {
            const bool contig_x = (A.ldx == d), contig_a = FACTORED && (A.lda == c);
            for (int i = 0; i < ntiles; ++i) {
                const int s = i % cfg.stages;
                const uint32_t round = static_cast<uint32_t>(i / cfg.stages);
                if (round > 0) mbar_wait(&empty[s], (round - 1) & 1u);
                const int row0 = seg.row_lo + i * R;
                const int rr = min(R, seg.row_hi - row0);
                float* tx = tiles + static_cast<size_t>(s) * cfg.tile_floats;
                float* ta = tx + static_cast<size_t>(R) * d;
                mbar_expect_tx(&full[s], static_cast<uint32_t>(rr) * static_cast<uint32_t>(d + c) * 4u);
                if (contig_x) {
                    bulk_g2s(tx, A.x + static_cast<int64_t>(row0) * A.ldx, static_cast<uint32_t>(rr) * d * 4u, &full[s]);
                } else {
                    for (int r = 0; r < rr; ++r)
                        bulk_g2s(tx + static_cast<size_t>(r) * d, A.x + static_cast<int64_t>(row0 + r) * A.ldx, d * 4u, &full[s]);
                }
                if (FACTORED) {
                    if (contig_a) {
                        bulk_g2s(ta, A.a + static_cast<int64_t>(row0) * A.lda, static_cast<uint32_t>(rr) * c * 4u, &full[s]);
                    } else {
                        for (int r = 0; r < rr; ++r)
                            bulk_g2s(ta + static_cast<size_t>(r) * c, A.a + static_cast<int64_t>(row0 + r) * A.lda, c * 4u, &full[s]);
                    }
                }
            }
        }
    } else {
        // ===== consumers: warp w owns tiles w-1, w-1+C, ... =====
        const int cw = warp - 1;
        const float qn = ci.qn;
        const int cf_off = SAMPLE ? A.cfull_off[seg.part] : 0;
        const float4* q4 = reinterpret_cast<const float4*>(sq);
        unsigned long long best_key = 0ull;
        for (int i = cw; i < ntiles; i += cfg.consumers) {
            const int s = i % cfg.stages;
            const uint32_t round = static_cast<uint32_t>(i / cfg.stages);
            const int row0 = seg.row_lo + i * R;
            const int rr = min(R, seg.row_hi - row0);
            // per-row scalars do not depend on the tile: fetch them while the copy is in flight
            float m_old = 0.f, n_i = 0.f;
            if (lane < rr) {
                m_old = A.mind[row0 + lane];
                n_i = FACTORED ? A.xn[row0 + lane] * A.an[row0 + lane] : A.xn[row0 + lane];
            }
            mbar_wait(&full[s], round & 1u);
            const float* tx = tiles + static_cast<size_t>(s) * cfg.tile_floats;
            const float* ta = tx + static_cast<size_t>(R) * d;
            float my_d2 = 0.f;
            for (int r = 0; r < rr; ++r) {
                const float4* p = reinterpret_cast<const float4*>(tx + static_cast<size_t>(r) * d);
                float dot = 0.f;
#pragma unroll 4
                for (int k = lane; k < dv; k += 32) {
                    const float4 v = p[k];
                    const float4 w = q4[k];
                    dot = fmaf(v.x, w.x, dot);
                    dot = fmaf(v.y, w.y, dot);
                    dot = fmaf(v.z, w.z, dot);
                    dot = fmaf(v.w, w.w, dot);
                }
                dot = warp_sum(dot);
                if (FACTORED) {
                    const float4* pa = reinterpret_cast<const float4*>(ta + static_cast<size_t>(r) * c);
                    float da = 0.f;
#pragma unroll 4
                    for (int k = lane; k < cv; k += 32) {
                        const float4 v = pa[k];
                        const float4 w = q4[dv + k];
                        da = fmaf(v.x, w.x, da);
                        da = fmaf(v.y, w.y, da);
                        da = fmaf(v.z, w.z, da);
                        da = fmaf(v.w, w.w, da);
                    }
                    dot *= warp_sum(da);
                }
                if (lane == r) my_d2 = dot;   // every lane holds the full sum after warp_sum
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);   // smem reads of this stage are complete
            if (lane < rr)
                finish_row<SAMPLE>(A, row0 + lane, centre, m_old, dist_dense(n_i, qn, my_d2), cf_off, best_key);
        }
        if (!SAMPLE) {
            best_key = warp_max_u64(best_key);
            if (lane == 0) sbest[cw] = best_key;
        }
    }
    if (!SAMPLE) {
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long b = 0ull;
            for (int w = 0; w < cfg.consumers; ++w) b = sbest[w] > b ? sbest[w] : b;
            if (b) atomicMax(&A.best[static_cast<size_t>(A.t) * A.P + seg.part], b);
        }
    }
}

__global__ void fill_f32_kernel(float* p, int n, float v) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ------------------------------------------------------------------------------------------------
// t = 0 helpers
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
argmax_init_kernel(StepArgs A, const int* first_pick) {
    __shared__ unsigned long long sb[8];
    const BlockSeg seg = A.segs[blockIdx.x];
    if (A.budget[seg.part] <= 0 || first_pick[seg.part] >= 0) return;
    unsigned long long b = 0ull;
    for (int r = seg.row_lo + threadIdx.x; r < seg.row_hi; r += blockDim.x) {
        const unsigned long long k = alq_maxkey(A.mind[r], static_cast<uint32_t>(r));
        b = k > b ? k : b;
    }
    b = warp_max_u64(b);
    if ((threadIdx.x & 31) == 0) sb[threadIdx.x >> 5] = b;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) b = sb[w] > b ? sb[w] : b;
        if (b) atomicMax(&A.best[seg.part], b);
    }
}

__global__ void first_pick_kernel(const int* first_pick, const int* budget, const int* pick_off, int P,
                                  unsigned long long* best, int* cur, int* picks) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P || budget[p] <= 0 || first_pick[p] < 0) return;
    if (best) best[p] = alq_maxkey(0.0f, static_cast<uint32_t>(first_pick[p]));
    else picks[pick_off[p]] = first_pick[p];   // arg-max picks are decoded from `best` at the end
    cur[p] = first_pick[p];
}

__global__ void decode_picks_kernel(const unsigned long long* best, const int* budget, const int* pick_off,
                                    int P, int bmax, int* picks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P * bmax) return;
    const int t = i / P, p = i % P;
    if (t < budget[p]) picks[pick_off[p] + t] = static_cast<int>(alq_maxkey_row(best[i]));
}

// cfull[off[p] + vpos[i]] = mind[i] (labeled / padding slots stay -inf);  posinv[...] = i
__global__ void __launch_bounds__(256)
sample_setup_kernel(StepArgs A, int* posinv) {
    const BlockSeg seg = A.segs[blockIdx.x];
    const int off = A.cfull_off[seg.part];
    for (int r = seg.row_lo + threadIdx.x; r < seg.row_hi; r += blockDim.x) {
        const int k = off + A.vpos[r];
        A.cfull[k] = A.mind[r];
        posinv[k] = r;
    }
}

// ------------------------------------------------------------------------------------------------
// D^2 sampling stage: one CTA per partition
// ------------------------------------------------------------------------------------------------
struct PartSched {
    int full_n;        // length of the partition's full (labeled + unlabeled) array
    int cfull_off;     // offset of that array inside cfull / posinv (multiple of 4)
    int n_leaves;      // leaves of NumPy's pairwise-sum tree
    int leaf_base;     // into leaf_off (n_leaves + 1 entries)
    int n_levels;      // combine levels of the tree
    int level_base;    // into level_off (n_levels + 1 entries)
    int comb_base;     // into comb (3 ints per internal node)
    int root;          // node id holding the total
    int row_lo, row_hi;  // candidate rows of this partition
    int pick_off, budget;
};

struct SampleArgs {
    const PartSched* sched;
    const int* leaf_off;
    const int* level_off;
    const int* comb;
    float* cfull;
    const int* posinv;
    float* leafval;              // leaf sums, same indexing as leaf_off
    double* cta_part;            // [P * kCL] per-CTA probability mass
    const double* uniforms;      // [sum budget]
    const int* first_pick;       // [P]
    int* cur;                    // [P]
    int* picks;
    int* status;                 // sticky error flag
    int t;
};

constexpr int kSampThreads = 1024;
constexpr int kCL = 8;             // CTAs per cluster == per partition (portable cluster size)


// One thread-block CLUSTER (kCL CTAs on kCL SMs) per partition.  The three dependent stages of a
// D^2 draw -- np.sum(prob) -> prob = c / S -> inverse-CDF search -- are separated by two cluster
// barriers instead of kernel boundaries:
//   A  leaves of NumPy's pairwise tree, split over the cluster  -> barrier -> every CTA folds the
//      (small) combine tree itself, so all agree on S bit for bit;
//   B  each CTA turns its slice into fp64 probability mass       -> barrier -> the one CTA whose
//      prefix interval contains u * total scans its slice and writes the pick.
// Prefixes are built as ONE sequential chain (rank order, then warp order, then lane order), so the
// "interval contains u" predicates of neighbouring CTAs / warps / threads are computed from
// identical values and exactly one thread claims the draw.
__global__ void __cluster_dims__(kCL, 1, 1) __launch_bounds__(kSampThreads, 1)
sample_cluster_kernel(SampleArgs A) {
    extern __shared__ float val[];                 // 2*n_leaves tree nodes, then the combine schedule (ints)
    __shared__ double sh_w[32];
    __shared__ int sh_hit;
    __shared__ int s_level_off[40];
    const int p = blockIdx.x / kCL;
    const int rank = static_cast<int>(cluster_rank());
    const PartSched S = A.sched[p];
    const int t = A.t;
    if (t >= S.budget) return;                     // uniform over the cluster
    if (t == 0 && A.first_pick[p] >= 0) return;    // chosen by the caller (nothing labeled yet)
    float* cf = A.cfull + S.cfull_off;
    const int n = S.full_n, K = S.n_leaves;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int* leaf_off = A.leaf_off + S.leaf_base;
    float* leafval = A.leafval + S.leaf_base;
    // The combine schedule (3 ints per internal node) is needed only after the leaf sums: start copying it
    // into shared memory now (cp.async, no register staging) so the tree folds without global-load latency.
    int* s_comb = reinterpret_cast<int*>(val + 2 * K);
    {
        const int n_int = 3 * (K - 1);
        const int* g_comb = A.comb + 3 * S.comb_base;
        for (int i = threadIdx.x; i < n_int; i += kSampThreads)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(s_comb + i)), "l"(g_comb + i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (threadIdx.x <= S.n_levels && threadIdx.x < 40) s_level_off[threadIdx.x] = A.level_off[S.level_base + threadIdx.x];
    }

    float total32 = 0.f;
    for (int attempt = 0;; ++attempt) {
        // ---- stage A: np.sum(prob) ---------------------------------------------------------------
        const int kc = (K + kCL - 1) / kCL;
        const int k_lo = rank * kc, k_hi = min(K, k_lo + kc);
        const int grp = lane >> 3, g_lane = lane & 7;
        const unsigned gmask = 0xffu << (grp * 8);
        for (int leaf0 = k_lo + warp * 4; leaf0 < k_hi; leaf0 += (kSampThreads / 32) * 4) {
            const int leaf = leaf0 + grp;
            if (leaf < k_hi) {
                const int lo = leaf_off[leaf], len = leaf_off[leaf + 1] - lo;
                const float v = leaf_sum_group(cf + lo, len, g_lane, gmask);
                if (g_lane == 0) leafval[leaf] = v;
            }
        }
        cluster_sync_all();
        for (int i = threadIdx.x; i < K; i += kSampThreads) val[i] = __ldcg(leafval + i);
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();
        for (int h = 0; h < S.n_levels; ++h) {
            const int lo = s_level_off[h], hi = s_level_off[h + 1];
            for (int j = lo + threadIdx.x; j < hi; j += kSampThreads) {
                const int* cb = s_comb + 3 * j;
                val[cb[0]] = val[cb[1]] + val[cb[2]];
            }
            __syncthreads();
        }
        total32 = val[S.root];
        if (total32 > 0.f && total32 <= 3.4028234e38f) break;
        if (!(total32 == 0.f) || attempt > (1 << 20)) {          // NaN / inf mass: not recoverable
            if (threadIdx.x == 0 && rank == 0) {
                atomicExch(A.status, ALQ_ERR_NUMERIC);
                A.cur[p] = S.row_lo;
                A.picks[S.pick_off + t] = S.row_lo;
            }
            return;                                              // same decision in every CTA
        }
        // ---- sum == 0 -> prob is NaN -> `min_dist_labeled += 0.00001` and retry (:87-90) --------
        // In place: labeled / picked slots hold -inf and stay there; candidate slots are rewritten from
        // `mind` by the next step kernel, so the bump never outlives this draw (like the reference's
        // per-step temporary).
        const int npad_r = (n + 3) & ~3, per_r = (npad_r + kCL - 1) / kCL;
        for (int k = rank * per_r + threadIdx.x; k < min(npad_r, (rank + 1) * per_r); k += kSampThreads)
            cf[k] = cf[k] + 0.00001f;
        cluster_sync_all();
    }

    // ---- stage B: np.random.choice == first k with cumsum64(p)[k] / total > u ---------------------
    const double u = A.uniforms[S.pick_off + t];
    const int npad = (n + 3) & ~3;
    const int per = (((n + kCL - 1) / kCL) + 4 * kSampThreads - 1) / (4 * kSampThreads) * (4 * kSampThreads);
    const int E = per / kSampThreads;                              // multiple of 4
    const int my_lo = rank * per + threadIdx.x * E;
    double loc = 0.0;
    float4 keep[4];                                                 // this thread's slice when E <= 16
    const bool small = E <= 16;
    if (small) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int base = my_lo + 4 * j;
            keep[j] = (4 * j < E && base < npad) ? __ldcg(reinterpret_cast<const float4*>(cf + base))
                                                 : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            loc += prob64(keep[j].x, total32);
            loc += prob64(keep[j].y, total32);
            loc += prob64(keep[j].z, total32);
            loc += prob64(keep[j].w, total32);
        }
    } else {
        for (int j = 0; j < E; j += 4) {
            const int base = my_lo + j;
            if (base < npad) {
                const float4 c4 = *reinterpret_cast<const float4*>(cf + base);   // zero padded to x4
                loc += prob64(c4.x, total32);
                loc += prob64(c4.y, total32);
                loc += prob64(c4.z, total32);
                loc += prob64(c4.w, total32);
            }
        }
    }
    double inc = loc;                                               // inclusive scan inside the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) sh_w[warp] = inc;
    if (threadIdx.x == 0) sh_hit = -1;
    __syncthreads();
    double woff = 0.0, cta_total = 0.0;                             // one sequential chain over warps
    for (int w = 0; w < 32; ++w) {
        if (w == warp) woff = cta_total;
        cta_total += sh_w[w];
    }
    if (threadIdx.x == 0) A.cta_part[p * kCL + rank] = cta_total;
    cluster_sync_all();
    double pre = 0.0, total = 0.0;                                  // ... and over CTAs
    for (int q = 0; q < kCL; ++q) {
        if (q == rank) pre = total;
        total += __ldcg(&A.cta_part[p * kCL + q]);
    }
    const double cta_after = pre + cta_total;
    const bool cta_claims = !(rank > 0 && (pre / total) > u) && ((cta_after / total) > u || rank == kCL - 1);
    if (!cta_claims) return;
    const double inc_prev = __shfl_up_sync(0xffffffffu, inc, 1);
    const double t_base = lane == 0 ? pre + woff : pre + (woff + inc_prev);
    const double t_after = pre + (woff + inc);
    const bool first_thread = threadIdx.x == 0;
    const bool last_thread = threadIdx.x == kSampThreads - 1;
    const bool claims = loc > 0.0 && !(!first_thread && (t_base / total) > u) &&
                        ((t_after / total) > u || last_thread);
    if (claims) {
        double run = t_base;
        int hit = -1, last_nz = -1;
        if (small) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float4 q4 = keep[j >> 2];
                const float raw = (j & 3) == 0 ? q4.x : (j & 3) == 1 ? q4.y : (j & 3) == 2 ? q4.z : q4.w;
                const int k = my_lo + j;
                if (j < E && k < n && hit < 0) {
                    if (raw > 0.f) last_nz = k;
                    run += prob64(raw, total32);
                    if ((run / total) > u) hit = k;
                }
            }
        } else {
            for (int j = 0; j < E && hit < 0; ++j) {
                const int k = my_lo + j;
                if (k >= n) break;
                const float raw = cf[k];
                if (raw > 0.f) last_nz = k;
                run += prob64(raw, total32);
                if ((run / total) > u) hit = k;
            }
        }
        if (hit < 0) hit = last_nz;        // fp64 re-association moved the crossing by an ulp
        atomicMax(&sh_hit, hit);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int k = sh_hit;
        if (k < 0) {
            // no thread of the claiming CTA holds mass after `pre` (u beyond the last entry by an ulp):
            // what a sequential cumsum returns is the last entry with mass
            for (int i = min(n, rank * per + per) - 1; i >= 0; --i)
                if (cf[i] > 0.f) { k = i; break; }
        }
        int row = k >= 0 ? A.posinv[S.cfull_off + k] : -1;
        if (row < 0) { atomicExch(A.status, ALQ_ERR_NUMERIC); row = S.row_lo; }
        A.cur[p] = row;
        A.picks[S.pick_off + t] = row;
        sh_hit = row;
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// A partition's tree as sample_cluster_kernel reads it: leaf offsets, then the internal nodes as (dst, l, r) triples
// grouped by height, internal node k (creation order) being node K + k.  Returns the leaf count K.
int append_sample_tree(const PairTree& tb, PartSched& S, std::vector<int>& leaf_off_all, std::vector<int>& level_off_all,
                       std::vector<int>& comb_all) {
    const int K = tb.n_leaves();
    auto node_id = [K](int v) { return v >= 0 ? v : K + (-v - 1); };
    S.n_leaves = K;
    S.leaf_base = static_cast<int>(leaf_off_all.size());
    leaf_off_all.insert(leaf_off_all.end(), tb.leaf_off.begin(), tb.leaf_off.end());
    S.root = tb.internal.empty() ? 0 : K + static_cast<int>(tb.internal.size()) - 1;
    S.n_levels = tb.n_levels();
    S.level_base = static_cast<int>(level_off_all.size());
    level_off_all.insert(level_off_all.end(), tb.level_off.begin(), tb.level_off.end());
    S.comb_base = static_cast<int>(comb_all.size() / 3);
    for (int k : tb.order) {
        comb_all.push_back(K + k);
        comb_all.push_back(node_id(tb.internal[k].l));
        comb_all.push_back(node_id(tb.internal[k].r));
    }
    return K;
}

template <bool FACTORED, bool SAMPLE>
void launch_step(int variant, int grid, cudaStream_t st, const StepArgs& A, const PipeCfg& cfg, size_t smem_v1,
                 size_t smem_v2) {
    if (variant == 2)
        step_pipe_kernel<FACTORED, SAMPLE><<<grid, 32 * (1 + cfg.consumers), smem_v2, st>>>(A, cfg);
    else
        step_direct_kernel<FACTORED, SAMPLE><<<grid, kV1Threads, smem_v1, st>>>(A);
}

template <bool FACTORED, bool SAMPLE>
cudaError_t set_step_attrs(size_t smem_v1, size_t smem_v2) {
    cudaError_t e = cudaSuccess;
    if (smem_v1 > 48 * 1024)
        e = cudaFuncSetAttribute(step_direct_kernel<FACTORED, SAMPLE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_v1));
    if (e == cudaSuccess && smem_v2 > 48 * 1024)
        e = cudaFuncSetAttribute(step_pipe_kernel<FACTORED, SAMPLE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_v2));
    return e;
}

}  // namespace

extern "C" int alq_greedy_select(alq_ctx* ctx, const alq_greedy_desc* D, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!D || D->struct_size != sizeof(alq_greedy_desc))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: descriptor size mismatch (header/library skew)");
    const int P = D->n_parts;
    const int64_t n = D->n;
    const bool factored = D->a != nullptr;
    const bool sample = D->uniforms_host != nullptr;
    if (P <= 0 || n <= 0 || n >= (1LL << 31) || !D->x || !D->xn || !D->mind || !D->part_off_host ||
        !D->budget_host || !D->picks || D->d <= 0)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: missing or empty arguments");
    if ((D->d % 4) || (D->ldx % 4) || D->ldx < D->d || !aligned16(D->x))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: d and ldx must be multiples of 4, x 16-byte aligned");
    if (factored && (!D->an || D->c <= 0 || (D->c % 4) || (D->lda % 4) || D->lda < D->c || !aligned16(D->a)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: factored rows need an, c %% 4 == 0, lda %% 4 == 0");
    if (sample && (!D->vpos || !D->full_n_host))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: D^2 sampling needs vpos and full_n");
    if (D->part_off_host[0] != 0 || D->part_off_host[P] != n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: part_off must span [0, n]");
    // ---- group path? shard_off on a context with a peer-memory group, of any size (a group of one rank included):
    //      every array is global and replicated, rank r streams its shard (include/alq.h) ----
    const AlqComm& G = ctx->comm;
    const bool comm = D->shard_off_host != nullptr && G.window != nullptr;
    if (D->shard_off_host && !comm && D->shard_off_host[1] != n)
        ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_greedy_select: shard_off given but no multi-GPU group (alq_comm_create/connect)");
    if (comm) {
        if (!G.connected) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_greedy_select: alq_comm_connect has not been called");
        if (P != 1) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: the multi-GPU loop is for one global partition");
        const int v = D->variant ? D->variant : ctx->greedy_variant;
        if (v == 1 || v == 2)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: variant %d with shard_off: the multi-GPU loop has no other variant "
                                           "than the persistent one", v);
        if (D->shard_off_host[0] != 0 || D->shard_off_host[G.world] != n)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: shard_off must span the n global candidate rows");
        for (int r = 0; r < G.world; ++r)
            if (D->shard_off_host[r + 1] < D->shard_off_host[r])
                ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: shard_off must be non-decreasing");
    }
    std::vector<int> pick_off(P + 1, 0), first_pick(P, -1);
    int bmax = 0;
    for (int p = 0; p < P; ++p) {
        const int rows = D->part_off_host[p + 1] - D->part_off_host[p];
        const int b = D->budget_host[p];
        if (rows < 0 || b < 0 || b > rows)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: partition %d has %d rows but budget %d", p, rows, b);
        if (sample && (D->full_n_host[p] < rows || D->full_n_host[p] > (2 << 20)))
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: full_n[%d]=%d out of range", p, D->full_n_host[p]);
        pick_off[p + 1] = pick_off[p] + b;
        bmax = std::max(bmax, b);
        if (D->first_pick_host) {
            first_pick[p] = D->first_pick_host[p];
            if (first_pick[p] >= 0 && (first_pick[p] < D->part_off_host[p] || first_pick[p] >= D->part_off_host[p + 1]))
                ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: first_pick[%d] outside its partition", p);
        }
    }
    const int total_picks = pick_off[P];
    if (total_picks == 0) return ALQ_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));

    // ---- kernel variant and its shared-memory plan ------------------------------------------------
    const int d = D->d, c = factored ? D->c : 0;
    const size_t smem_v1 = static_cast<size_t>(d + c) * sizeof(float);
    PipeCfg cfg{};
    size_t smem_v2 = 0;
    int variant = D->variant ? D->variant : ctx->greedy_variant;
    if (variant == 0 || variant == 3 || comm) {
        // the whole loop as one persistent cooperative launch (alq_greedy_persist.cu)
        const int rc3 = alq_greedy_persist(ctx, D, stream);
        if (rc3 != kPersistNotApplicable) return rc3;
        if (variant == 3 || comm)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: the persistent loop does not fit this problem "
                                           "(more active partitions than SMs, a partition beyond %d tree leaves, or a row too large for the ring)%s",
                     4096, comm ? "; the multi-GPU loop has no other variant" : "");
        variant = 0;
    }
    {
        const size_t row_bytes = static_cast<size_t>(d + c) * 4;
        const size_t centre_bytes = static_cast<size_t>((d + c + 31) & ~31) * 4;
        const size_t budget_bytes = ctx->smem_optin > 8192 ? ctx->smem_optin - 2048 : 0;
        size_t tile_target = 32 * 1024;    // sweep (tools/tune_step.py): 24-32 KB tiles beat 16 KB by 4-8 %
        int max_stages = 16;
        if (const char* e = getenv("ALQ_TILE_KB")) tile_target = std::max(1, atoi(e)) * 1024;      // tuning aids
        if (const char* e = getenv("ALQ_MAX_STAGES")) max_stages = std::max(3, std::min(16, atoi(e)));
        int R = static_cast<int>(std::max<size_t>(1, tile_target / row_bytes));
        R = std::min(R, 32);
        const size_t tile_bytes = R * row_bytes;
        int stages = budget_bytes > centre_bytes ? static_cast<int>((budget_bytes - centre_bytes) / tile_bytes) : 0;
        stages = std::min(stages, max_stages);
        cfg.rows_per_tile = R;
        cfg.stages = stages;
        cfg.tile_floats = static_cast<int>(tile_bytes / 4);
        cfg.consumers = std::max(1, std::min(16, stages));
        smem_v2 = centre_bytes + stages * tile_bytes + 2 * stages * sizeof(uint64_t) + 16 * sizeof(unsigned long long) + 64;
        const bool v2_ok = stages >= 3 && (row_bytes % 16 == 0) && (static_cast<size_t>(d) * 4 % 16 == 0);
        if (variant == 0) variant = v2_ok ? 2 : 1;
        if (variant == 2 && !v2_ok) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: variant 2 does not fit (row too large)");
        if (variant != 1 && variant != 2) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: unknown variant");
        if (smem_v1 > ctx->smem_optin) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: row does not fit shared memory");
    }
    std::vector<BlockSeg> segs;
    build_segments(P, D->part_off_host, D->budget_host, variant == 2 ? ctx->sm_count : ctx->sm_count * 6, segs);
    const int grid = static_cast<int>(segs.size());

    // ---- D^2-sampling schedule (NumPy pairwise tree per partition) ----------------------------------
    std::vector<PartSched> sched(P);
    std::vector<int> leaf_off_all, level_off_all, comb_all, cfull_off(P, 0);
    int cfull_total = 0, max_nodes = 1;
    if (sample) {
        for (int p = 0; p < P; ++p) {
            PartSched& S = sched[p];
            S.full_n = D->full_n_host[p];
            S.cfull_off = cfull_total;
            cfull_off[p] = cfull_total;
            cfull_total += (S.full_n + 3) & ~3;
            S.row_lo = D->part_off_host[p];
            S.row_hi = D->part_off_host[p + 1];
            S.pick_off = pick_off[p];
            S.budget = D->budget_host[p];
            const int K = append_sample_tree(PairTree(S.full_n), S, leaf_off_all, level_off_all, comb_all);
            max_nodes = std::max(max_nodes, 2 * K);
        }
        if (static_cast<size_t>(max_nodes) * sizeof(float) * 5 / 2 > ctx->smem_optin - 16 * 1024)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: partition too long for the sampling stage");
    }

    // ---- scratch --------------------------------------------------------------------------------------
    const size_t n_best = sample ? 0 : static_cast<size_t>(bmax) * P;
    BlockSeg* d_segs;
    PartSched* d_sched;
    int *d_budget, *d_pick_off, *d_first, *d_cur, *d_cfull_off, *d_leaf_off, *d_level_off, *d_comb, *d_posinv, *d_status;
    unsigned long long* d_best;
    double *d_unif, *d_cta_part;
    float *d_cfull, *d_leafval;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        d_segs = cur.take<BlockSeg>(segs.size());
        d_budget = cur.take<int>(P);
        d_pick_off = cur.take<int>(P);
        d_first = cur.take<int>(P);
        d_cur = cur.take<int>(P);
        d_cfull_off = cur.take<int>(P);
        d_best = cur.take<unsigned long long>(n_best);
        d_unif = cur.take<double>(total_picks);
        d_sched = cur.take<PartSched>(sched.size());
        d_leaf_off = cur.take<int>(leaf_off_all.size() + 1);
        d_level_off = cur.take<int>(level_off_all.size() + 1);
        d_comb = cur.take<int>(comb_all.size() + 1);
        d_cfull = cur.take<float>(cfull_total + 4);
        d_posinv = cur.take<int>(cfull_total + 4);
        d_leafval = cur.take<float>(leaf_off_all.size() + 1);
        d_cta_part = cur.take<double>(static_cast<size_t>(P) * kCL);
        d_status = cur.take<int>(1);
    });
    if (rc) return rc;

    // pageable sources: the runtime stages them before returning, so the vectors may die afterwards
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_segs, segs.data(), segs.size() * sizeof(BlockSeg), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_budget, D->budget_host, P * sizeof(int), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_pick_off, pick_off.data(), P * sizeof(int), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_first, first_pick.data(), P * sizeof(int), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(d_status, 0, sizeof(int), st));
    ALQ_CUDA(ctx, cudaMemsetAsync(d_cur, 0, P * sizeof(int), st));
    if (sample) {
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_cfull_off, cfull_off.data(), P * sizeof(int), cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_unif, D->uniforms_host, total_picks * sizeof(double), cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_sched, sched.data(), sched.size() * sizeof(PartSched), cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_leaf_off, leaf_off_all.data(), leaf_off_all.size() * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_level_off, level_off_all.data(), level_off_all.size() * 4, cudaMemcpyHostToDevice, st));
        if (!comb_all.empty())
            ALQ_CUDA(ctx, cudaMemcpyAsync(d_comb, comb_all.data(), comb_all.size() * 4, cudaMemcpyHostToDevice, st));
        fill_f32_kernel<<<(cfull_total + 4 + 255) / 256, 256, 0, st>>>(d_cfull, cfull_total + 4, -INFINITY);
        ALQ_LAUNCH_CHECK(ctx);
        ALQ_CUDA(ctx, cudaMemsetAsync(d_posinv, 0xff, static_cast<size_t>(cfull_total + 4) * 4, st));
    } else {
        ALQ_CUDA(ctx, cudaMemsetAsync(d_best, 0, n_best * 8, st));
    }

    StepArgs A{};
    A.x = D->x; A.ldx = D->ldx; A.d = d;
    A.a = D->a; A.lda = D->lda; A.c = c;
    A.xn = D->xn; A.an = D->an;
    A.mind = D->mind;
    A.segs = d_segs; A.budget = d_budget; A.P = P;
    A.best = d_best; A.cur = d_cur;
    A.vpos = D->vpos; A.cfull = d_cfull; A.cfull_off = d_cfull_off;
    A.status = d_status; A.picks = D->picks;

    cudaError_t ae = cudaSuccess;
    if (factored) ae = sample ? set_step_attrs<true, true>(smem_v1, variant == 2 ? smem_v2 : 0)
                              : set_step_attrs<true, false>(smem_v1, variant == 2 ? smem_v2 : 0);
    else ae = sample ? set_step_attrs<false, true>(smem_v1, variant == 2 ? smem_v2 : 0)
                     : set_step_attrs<false, false>(smem_v1, variant == 2 ? smem_v2 : 0);
    if (ae != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(ae));

    SampleArgs SA{};
    size_t samp_smem = 0;
    if (sample) {
        SA.sched = d_sched; SA.leaf_off = d_leaf_off; SA.level_off = d_level_off; SA.comb = d_comb;
        SA.cfull = d_cfull; SA.posinv = d_posinv;
        SA.leafval = d_leafval; SA.cta_part = d_cta_part; SA.uniforms = d_unif; SA.first_pick = d_first; SA.cur = d_cur;
        SA.picks = D->picks; SA.status = d_status;
        samp_smem = static_cast<size_t>(max_nodes) * sizeof(float) * 5 / 2 + 64;   // nodes + 3 ints per internal node
        if (samp_smem > 32 * 1024)
            ALQ_CUDA(ctx, cudaFuncSetAttribute(sample_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(samp_smem)));
        // alternates with the 200 KB step kernel 10 000 times: keep the same L1/shared split
        cudaFuncSetAttribute(sample_cluster_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                             cudaSharedmemCarveoutMaxShared);
        cudaGetLastError();
    }

    // ---- t = 0 ------------------------------------------------------------------------------------------
    first_pick_kernel<<<(P + 127) / 128, 128, 0, st>>>(d_first, d_budget, d_pick_off, P, sample ? nullptr : d_best,
                                                       d_cur, D->picks);
    ALQ_LAUNCH_CHECK(ctx);
    A.t = 0;
    if (sample) {
        sample_setup_kernel<<<grid, 256, 0, st>>>(A, d_posinv);
        ALQ_LAUNCH_CHECK(ctx);
        SA.t = 0;
        sample_cluster_kernel<<<P * kCL, kSampThreads, samp_smem, st>>>(SA);
        ALQ_LAUNCH_CHECK(ctx);
    } else {
        argmax_init_kernel<<<grid, 256, 0, st>>>(A, d_first);
        ALQ_LAUNCH_CHECK(ctx);
    }

    // ---- steps 1 .. bmax-1 ---------------------------------------------------------------------------------
    constexpr int kMaxTimed = 256;
    std::vector<cudaEvent_t> evs;
    const bool timing = D->step_kernel_ms_host != nullptr;
    const int time_every = std::max(1, (bmax - 1) / kMaxTimed);
    for (int t = 1; t < bmax; ++t) {
        A.t = t;
        const bool timed = timing && ((t - 1) % time_every == 0) && static_cast<int>(evs.size()) < 2 * kMaxTimed;
        if (timed) {
            cudaEvent_t e0, e1;
            cudaEventCreate(&e0);
            cudaEventCreate(&e1);
            evs.push_back(e0);
            evs.push_back(e1);
            cudaEventRecord(e0, st);
        }
        if (factored) {
            if (sample) launch_step<true, true>(variant, grid, st, A, cfg, smem_v1, smem_v2);
            else launch_step<true, false>(variant, grid, st, A, cfg, smem_v1, smem_v2);
        } else {
            if (sample) launch_step<false, true>(variant, grid, st, A, cfg, smem_v1, smem_v2);
            else launch_step<false, false>(variant, grid, st, A, cfg, smem_v1, smem_v2);
        }
        ALQ_LAUNCH_CHECK(ctx);
        if (timed) cudaEventRecord(evs.back(), st);
        if (sample) {
            SA.t = t;
            sample_cluster_kernel<<<P * kCL, kSampThreads, samp_smem, st>>>(SA);
            ALQ_LAUNCH_CHECK(ctx);
        }
    }
    if (!sample) {
        decode_picks_kernel<<<(P * bmax + 255) / 256, 256, 0, st>>>(d_best, d_budget, d_pick_off, P, bmax, D->picks);
        ALQ_LAUNCH_CHECK(ctx);
    }
    int status = 0;
    if (timing || sample) {
        // the sampling variant reports a sticky numeric status; timing needs the events resolved
        ALQ_CUDA(ctx, cudaMemcpyAsync(&status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
        ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    }
    if (timing) {
        double acc = 0.0;
        int cnt = 0;
        for (size_t i = 0; i + 1 < evs.size(); i += 2) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, evs[i], evs[i + 1]) == cudaSuccess) { acc += ms; ++cnt; }
        }
        D->step_kernel_ms_host[0] = cnt ? static_cast<float>(acc / cnt) : 0.f;
        D->step_kernel_ms_host[1] = 0.f;
        D->step_kernel_ms_host[2] = static_cast<float>(cnt);
        D->step_kernel_ms_host[3] = static_cast<float>(variant);
        for (int i = 4; i < 8; ++i) D->step_kernel_ms_host[i] = 0.f;
    }
    for (cudaEvent_t e : evs) cudaEventDestroy(e);
    if (status != 0) ALQ_FAIL(ctx, status, "alq_greedy_select: non-finite or empty probability mass during D^2 sampling");
    return ALQ_OK;
}

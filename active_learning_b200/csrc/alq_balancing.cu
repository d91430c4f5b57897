// K11: the whole query of BalancingSampler (balancing_sampler.py:58-134 of active_learning/src/query_strategies) as
// one persistent launch.
//
// The reference takes one row per step, and every step decides on the labeled class histogram whether to balance
// (nearest to the rarest class centre relative to the farthest majority centre) or to draw at random.  Run as a host
// loop that is about fifteen launches and two host round trips per pick.  Here:
//   set-up   K10's table pass counts the labeled rows per class (and rejects an out-of-range label); one launch
//            counts the available rows of every CTA segment (and rejects an available row's out-of-range label);
//            two launches build the fp64 class sums in a fixed order: per chunk of kSumChunk rows the labeled rows in
//            row order, then the chunks in order;
//   loop     ONE ordinary launch, one CTA per SM (grid <= SMs, bracketed by alq_gridsync_begin/end), every wait bounded
//            by "spin_timeout_ms".  Every CTA keeps the class histogram, the fp32 centres, their norms, the available
//            count of every CTA segment and NumPy's MT19937 state in shared memory and updates them identically after
//            each pick, so the branch, the rarest / majority classes and the random draw need no exchange at all.
//              balancing step: each CTA reduces its segment to one key (ord(ratio + 0), row) and publishes one LL word
//                              {tag16, row offset16, ord32}; every CTA gathers the grid's words and takes the minimum;
//              random step:    every CTA draws the same k (legacy masked rejection on MT19937) and finds the CTA whose
//                              segment holds rank k; that CTA locates the row and announces it in the step's LL word.
//            After the pick: the row leaves `avail` (owner CTA), the class count and the owner's segment count change,
//            and every CTA adds the row to its own fp64 copy of the class sum and recomputes that one centre and norm.
// A row's dot product with a centre is a fixed function of that row: lane l accumulates the float4 chunks l, l + 32, ..
// with fmaf in x, y, z, w order, and a butterfly folds the 32 partials (every lane ends with the same value).  Neither the
// warp, nor the CTA, nor the grid size changes it, so the picks are bit-reproducible.
// Sharded over a group (shard_off_host), the segments above are every rank's CTA segments (SegShard): every CTA of every
// rank keeps all of their counts, the key words go into every rank's window and the owner of a random pick stores its
// word there too; K12 shares the layout.
// The host side of a call is bal_select (alq_balancing.cuh), shared with K12; this file supplies K11's part of it
// (BalLoop: the shared-memory limit, the class-sum scratch and launches) and the segment count of both.
#include "alq_balancing.cuh"

namespace {

constexpr int kBalThreads = 512;                 // >= kPollers: every poller of ll_gather is a thread of the CTA
constexpr int kBalWarps = kBalThreads / 32;
constexpr int kCentresPerPass = 8;               // dot products a lane accumulates at once
constexpr int kSumChunk = 65536;                 // rows per fixed chunk of the fp64 class sums
constexpr int kSumDims = 128;                    // dimensions per CTA of the class-sum pass (one per thread)
struct BalArgs {
    const float* x; long long ldx; int d;
    const float* xn;
    const int* labels;
    uint8_t* avail;              // working copy of the caller's mask
    const double* sums0;         // [c][d] fp64 class sums of the labeled rows
    double* sums;                // [grid][c][d] every CTA's running copy
    const int* counts0;          // [c]
    const int* seg_avail0;       // [world * grid]
    const unsigned int* mt_in;   // [kMtN + 1]: key, pos
    unsigned int* mt_out;        // [kMtN + 1]
    int* picks;
    int* n_bal;
    int* status;
    SegShard S;
    LLWords W;                   // key words of the balancing steps (two parities), one pick word per random step
    int n, c, budget, n_avail;
    long long timeout_cycles;
};

__device__ __forceinline__ float centre_of(double sum, int count) {
    const float denom = bal_den(count);
    return __double2float_rn(sum / static_cast<double>(denom));
}

// <x, q> as the fixed function described above (x, q: d / 4 float4, in any memory)
__device__ __forceinline__ float dot_fixed(const float4* x, const float4* q, int dv, int lane) {
    float acc = 0.f;
    for (int k = lane; k < dv; k += 32) {
        const float4 v = x[k], w = q[k];
        acc = fmaf(v.x, w.x, acc);
        acc = fmaf(v.y, w.y, acc);
        acc = fmaf(v.z, w.z, acc);
        acc = fmaf(v.w, w.w, acc);
    }
    return warp_sum(acc);
}

// available rows per global segment (one block each); the smallest available row with a label outside [0, c) -> *bad
__global__ void __launch_bounds__(256) bal_seg_count_kernel(const int* __restrict__ labels, const uint8_t* __restrict__ avail,
                                                            int c, const __grid_constant__ SegShard S, int* __restrict__ seg_avail,
                                                            unsigned int* __restrict__ bad) {
    __shared__ int wsum[8];
    const int lo = gseg_lo(S, blockIdx.x), hi = gseg_lo(S, blockIdx.x + 1);
    int cnt = 0;
    for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        if (!avail[i]) continue;
        ++cnt;
        if (static_cast<unsigned>(labels[i]) >= static_cast<unsigned>(c)) atomicMin(bad, static_cast<unsigned>(i));
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < 8; ++w) s += wsum[w];
        seg_avail[blockIdx.x] = s;
    }
}

// partial[ch][k][j] = fp64 sum, in row order, of x[r, j] over the labeled rows r of chunk ch with label k (0.0 + ..)
__global__ void __launch_bounds__(kSumDims) bal_class_sum_partial_kernel(const float* __restrict__ x, long long ldx, int d,
                                                                         const int* __restrict__ labels,
                                                                         const uint8_t* __restrict__ labeled, int n, int c,
                                                                         double* __restrict__ partial) {
    extern __shared__ double acc[];              // [c][kSumDims]
    __shared__ int s_row[kSumDims], s_lab[kSumDims], s_wc[kSumDims / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int j = blockIdx.x * kSumDims + tid;
    const int ch = blockIdx.y;
    for (int i = tid; i < c * kSumDims; i += kSumDims) acc[i] = 0.0;
    const int lo = ch * kSumChunk, hi = static_cast<int>(min(static_cast<long long>(n), static_cast<long long>(lo) + kSumChunk));
    for (int r0 = lo; r0 < hi; r0 += kSumDims) {
        const int row = r0 + tid;
        const int y = (row < hi && labeled[row]) ? labels[row] : -1;
        const bool ok = static_cast<unsigned>(y) < static_cast<unsigned>(c);
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) s_wc[warp] = __popc(bal);
        __syncthreads();
        int before = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < kSumDims / 32; ++w) {
            if (w < warp) before += s_wc[w];
            tot += s_wc[w];
        }
        if (ok) {
            const int at = before + __popc(bal & ((1u << lane) - 1u));
            s_row[at] = row;
            s_lab[at] = y;
        }
        __syncthreads();
        if (j < d)
            for (int q = 0; q < tot; ++q) acc[s_lab[q] * kSumDims + tid] += static_cast<double>(__ldg(x + static_cast<long long>(s_row[q]) * ldx + j));
        __syncthreads();
    }
    if (j < d)
        for (int k = 0; k < c; ++k) partial[(static_cast<size_t>(ch) * c + k) * d + j] = acc[k * kSumDims + tid];
}

// sums0[i] = 0.0 + partial[0][i] + partial[1][i] + ..
__global__ void bal_class_sum_reduce_kernel(const double* __restrict__ partial, int nchunks, long long cd, double* __restrict__ sums0) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= cd) return;
    double s = 0.0;
    for (int ch = 0; ch < nchunks; ++ch) s += partial[ch * cd + i];
    sums0[i] = s;
}

__host__ __device__ __forceinline__ size_t bal_loop_smem(int c, int d, int nseg) {
    return static_cast<size_t>(c) * d * 4 + static_cast<size_t>(c) * 12 + static_cast<size_t>(nseg) * 4 + kMtN * 4 + 64;
}

__global__ void __launch_bounds__(kBalThreads, 1) balancing_loop_kernel(const __grid_constant__ BalArgs A) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int c = A.c, d = A.d, dv = d >> 2, nseg = A.S.world * A.S.grid;
    float* cent = reinterpret_cast<float*>(smem_raw);                 // [c][d]
    float* cn = cent + static_cast<size_t>(c) * d;                    // [c]
    int* cnt = reinterpret_cast<int*>(cn + c);                        // [c]
    int* sel = cnt + c;                                               // [c]
    int* seg_av = sel + c;                                            // [nseg]
    unsigned int* mt = reinterpret_cast<unsigned int*>(seg_av + nseg);   // [kMtN]
    __shared__ unsigned long long s_key[kBalWarps];
    __shared__ int s_wc[kBalWarps];
    __shared__ int s_nsel, s_pick, s_owner, s_rank, s_found, s_mtpos, s_navail;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x;
    const int gb = A.S.rank * A.S.grid + b;                           // my global segment
    const int row_lo = gseg_lo(A.S, gb), row_hi = gseg_lo(A.S, gb + 1);
    double* my_sums = A.sums + static_cast<size_t>(b) * c * d;

    for (int i = tid; i < c; i += kBalThreads) cnt[i] = A.counts0[i];
    for (int i = tid; i < nseg; i += kBalThreads) seg_av[i] = A.seg_avail0[i];
    for (int i = tid; i < kMtN; i += kBalThreads) mt[i] = A.mt_in[i];
    if (tid == 0) { s_mtpos = static_cast<int>(A.mt_in[kMtN]); s_navail = A.n_avail; }
    __syncthreads();
    for (int i = tid; i < c * d; i += kBalThreads) {
        const double s = A.sums0[i];
        my_sums[i] = s;
        cent[i] = centre_of(s, cnt[i / d]);
    }
    __syncthreads();
    for (int k = warp; k < c; k += kBalWarps) {
        const float4* q = reinterpret_cast<const float4*>(cent + static_cast<size_t>(k) * d);
        const float v = dot_fixed(q, q, dv, lane);
        if (lane == 0) cn[k] = v;
    }
    if (A.W.ready_tag != 0 && tid < A.S.world) ll_ready_wait(A.W.peer[A.S.rank], tid, A.W.ready_tag, A);
    __syncthreads();

    unsigned int rnd_key = 0;
    int n_bal = 0;
    for (int t = 0; t < A.budget; ++t) {
        if (tid == 0) s_nsel = imbalance_test(cnt, c, A.budget - t, sel);
        __syncthreads();
        const int nsel = s_nsel;
        if (nsel > 0) {
            // ===== balancing step (balancing_sampler.py:85-125) =====
            ++n_bal;
            const bool near1 = cnt[sel[0]] == 0;                          // :106-109: numerator 1
            unsigned long long best = ~0ull;
            for (int row = row_lo + warp; row < row_hi; row += kBalWarps) {
                if (!A.avail[row]) continue;                              // warp-uniform
                const float4* xr = reinterpret_cast<const float4*>(A.x + static_cast<long long>(row) * A.ldx);
                const float xn = __ldg(A.xn + row);
                float near = 1.f, far = ALQ_NEG_INF;
                for (int j0 = near1 ? 1 : 0; j0 < nsel; j0 += kCentresPerPass) {
                    const int jn = min(kCentresPerPass, nsel - j0);
                    const float4* q[kCentresPerPass];
#pragma unroll
                    for (int j = 0; j < kCentresPerPass; ++j)
                        q[j] = reinterpret_cast<const float4*>(cent + static_cast<size_t>(sel[j0 + (j < jn ? j : 0)]) * d);
                    float acc[kCentresPerPass];
#pragma unroll
                    for (int j = 0; j < kCentresPerPass; ++j) acc[j] = 0.f;
                    for (int k = lane; k < dv; k += 32) {
                        const float4 v = __ldg(xr + k);
#pragma unroll
                        for (int j = 0; j < kCentresPerPass; ++j)
                            if (j < jn) {
                                const float4 w = q[j][k];
                                acc[j] = fmaf(v.x, w.x, acc[j]);
                                acc[j] = fmaf(v.y, w.y, acc[j]);
                                acc[j] = fmaf(v.z, w.z, acc[j]);
                                acc[j] = fmaf(v.w, w.w, acc[j]);
                            }
                    }
#pragma unroll
                    for (int j = 0; j < kCentresPerPass; ++j)
                        if (j < jn) {
                            const float dot = warp_sum(acc[j]);
                            const float dist = __fsub_rn(__fadd_rn(xn, cn[sel[j0 + j]]), 2.0f * dot);
                            if (j0 + j == 0) near = dist;
                            else far = fmaxf(far, dist);
                        }
                }
                const float ratio = __fdiv_rn(near, far);
                const unsigned long long key = (static_cast<unsigned long long>(alq_ord(ratio + 0.0f)) << 32) | static_cast<uint32_t>(row);
                best = key < best ? key : best;
            }
            if (lane == 0) s_key[warp] = best;
            __syncthreads();
            ll_agree_min_call<kBalWarps>(A, s_key, &s_pick, ++rnd_key, row_lo, tid);
        } else {
            // ===== random step (balancing_sampler.py:128): np.random.choice over the available rows =====
            if (tid == 0) {
                int k = static_cast<int>(mt_bounded(mt, s_mtpos, static_cast<unsigned int>(s_navail - 1)));
                int o = 0;
                while (o + 1 < nseg && k >= seg_av[o]) { k -= seg_av[o]; ++o; }
                s_owner = o;
                s_rank = k;
                s_found = -1;
            }
            __syncthreads();
            const size_t pw = A.W.pickw + static_cast<size_t>(t) * 8;
            const unsigned int ptag = bal_pick_tag(A.W, t);
            if (s_owner == gb) {                                          // the rank-th available row of this segment
                const int rank = s_rank;
                int base = 0;
                for (int r0 = row_lo; r0 < row_hi; r0 += kBalThreads) {
                    const int row = r0 + tid;
                    const bool av = row < row_hi && A.avail[row];
                    const unsigned bal = __ballot_sync(0xffffffffu, av);
                    if (lane == 0) s_wc[warp] = __popc(bal);
                    __syncthreads();
                    int before = 0, tot = 0;
#pragma unroll
                    for (int w = 0; w < kBalWarps; ++w) {
                        if (w < warp) before += s_wc[w];
                        tot += s_wc[w];
                    }
                    const bool here = rank < base + tot;                  // block-uniform
                    if (here && av && base + before + __popc(bal & ((1u << lane) - 1u)) == rank) s_found = row;
                    __syncthreads();
                    if (here) break;
                    base += tot;
                }
                if (tid < A.S.world) ll_store(A.W.peer[tid] + pw, ptag, static_cast<unsigned int>(s_found));
            }
            if (tid == 0) s_pick = static_cast<int>(ll_wait(A.W.peer[A.S.rank] + pw, ptag, A));
            __syncthreads();
        }

        // ===== update (balancing_sampler.py:131-133) =====
        const int pick = s_pick;
        if (pick < 0 || pick >= A.n) {                                   // a failed wait (status set) or no row: stop
            if (tid == 0) atomicCAS(A.status, 0, ALQ_ERR_STATE);
            break;
        }
        const int cls = __ldg(A.labels + pick);
        const int newc = cnt[cls] + 1;
        const int o = gseg_of(A.S, pick);
        __syncthreads();                                                 // cnt[cls] read by every thread
        if (tid == 0) {
            cnt[cls] = newc;
            seg_av[o] -= 1;
            s_navail -= 1;
            if (o == gb) A.avail[pick] = 0;
            if (b == 0) A.picks[t] = pick;
        }
        float* cc = cent + static_cast<size_t>(cls) * d;
        double* sc = my_sums + static_cast<size_t>(cls) * d;
        const float* xp = A.x + static_cast<long long>(pick) * A.ldx;
        for (int j = tid; j < d; j += kBalThreads) {
            const double s = sc[j] + static_cast<double>(__ldg(xp + j));
            sc[j] = s;
            cc[j] = centre_of(s, newc);
        }
        __syncthreads();
        if (warp == 0) {
            const float v = dot_fixed(reinterpret_cast<const float4*>(cc), reinterpret_cast<const float4*>(cc), dv, lane);
            if (lane == 0) cn[cls] = v;
        }
        __syncthreads();
    }
    if (b == 0) {
        for (int i = tid; i < kMtN; i += kBalThreads) A.mt_out[i] = mt[i];
        if (tid == 0) { A.mt_out[kMtN] = static_cast<unsigned int>(s_mtpos); *A.n_bal = n_bal; }
    }
}

// K11's steps of bal_select
struct BalLoop {
    using Args = BalArgs;
    static constexpr const char* kName = "alq_balancing_select";
    static constexpr int kForce = 2;                 // balancing_loop = 2 forces K11; 1 and 3 make it decline
    static constexpr int kThreads = kBalThreads;
    static constexpr auto kernel = balancing_loop_kernel;
    size_t smem = 0, sum_smem = 0;

    int plan_smem(alq_ctx* ctx, BalCall& B) {
        smem = bal_loop_smem(B.c, B.d, B.nseg);
        sum_smem = static_cast<size_t>(B.c) * kSumDims * sizeof(double);
        if (smem > B.smem_cap || sum_smem > B.smem_cap)
            BAL_LIMIT(B, "%s: the %d centres of %d floats need %zu bytes of shared memory, %zu are available (limit: centres "
                      "in shared memory)", kName, B.c, B.d, std::max(smem, sum_smem), B.smem_cap);
        return ALQ_OK;
    }
    static int nchunks(const BalCall& B) { return (B.n + kSumChunk - 1) / kSumChunk; }
    // all of K11's scratch, reserved with the counts' (the first four) and sized from the shape
    size_t need_with_counts(const BalCall& B) const {
        const size_t cd = static_cast<size_t>(B.c) * B.d;
        return scratch_need({B.entries * 4, static_cast<size_t>(B.c) * 4, 8, static_cast<size_t>(B.nseg) * 4,
                             static_cast<size_t>(nchunks(B)) * cd * 8, cd * 8, static_cast<size_t>(B.S.grid) * cd * 8,
                             static_cast<size_t>(B.n), (kMtN + 1) * 4 * 2, B.sharded ? 0 : B.words_max, 16});
    }
    // the fp64 class sums
    int setup(alq_ctx* ctx, BalCall& B, ScratchCursor& cur, BalArgs& A) {
        const alq_balancing_desc* D = B.D;
        const int n = B.n, c = B.c, d = B.d, nch = nchunks(B);
        const size_t cd = static_cast<size_t>(c) * d;
        double* partial = cur.take<double>(static_cast<size_t>(nch) * cd);
        double* sums0 = cur.take<double>(cd);
        A.sums = cur.take<double>(static_cast<size_t>(B.S.grid) * cd);
        A.sums0 = sums0;
        A.xn = D->xn;
        if (sum_smem > 48u * 1024u)
            ALQ_CUDA(ctx, cudaFuncSetAttribute(bal_class_sum_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sum_smem)));
        bal_class_sum_partial_kernel<<<dim3((d + kSumDims - 1) / kSumDims, nch), kSumDims, sum_smem, B.st>>>(
            D->x, D->ldx, d, D->labels, D->labeled, n, c, partial);
        ALQ_LAUNCH_CHECK(ctx);
        bal_class_sum_reduce_kernel<<<static_cast<int>((cd + 255) / 256), 256, 0, B.st>>>(partial, nch, static_cast<long long>(cd), sums0);
        ALQ_LAUNCH_CHECK(ctx);
        return ALQ_OK;
    }
};

}  // namespace

int bal_seg_count(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int c, const SegShard& S, int32_t* seg_avail,
                  unsigned int* bad, cudaStream_t st) {
    bal_seg_count_kernel<<<S.world * S.grid, 256, 0, st>>>(labels, avail, c, S, seg_avail, bad);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_balancing_select(alq_ctx* ctx, const alq_balancing_desc* D, void* stream) {
    return bal_select<BalLoop>(ctx, D, stream);
}

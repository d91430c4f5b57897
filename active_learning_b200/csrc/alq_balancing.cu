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
// Sharded over a group (shard_off_host), the segments above are every rank's CTA segments (BalShard): every CTA of every
// rank keeps all of their counts, the key words go into every rank's window and the owner of a random pick stores its
// word there too; K12 shares the layout and the host steps below.
#include <limits.h>

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
    BalShard S;
    BalWords W;                  // key words of the balancing steps (two parities), one pick word per random step
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
                                                            int c, const __grid_constant__ BalShard S, int* __restrict__ seg_avail,
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
    bal_ready_wait(A, tid);

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
            bal_agree<kBalWarps>(A, s_key, &s_pick, ++rnd_key, row_lo, tid);
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

constexpr size_t kWordsHead = 128;               // u64 ready[ALQ_MAX_WORLD] in front of a window's words (greedy's layout)

size_t up128(size_t v) { return (v + 127) & ~size_t(127); }

}  // namespace

// descriptors of the shorter, single-GPU layout end here
constexpr size_t kBalDescV1 = offsetof(alq_balancing_desc, shard_off_host);

int alq_bal_shard(alq_ctx* ctx, const alq_balancing_desc* D, int n, BalShard* S, bool* sharded, const char* fn) {
    const int32_t* so = D->struct_size >= sizeof(alq_balancing_desc) ? D->shard_off_host : nullptr;
    *sharded = so != nullptr;
    S->world = 1;
    S->rank = 0;
    S->off[0] = 0;
    S->off[1] = n;
    if (so) {
        const AlqComm& G = ctx->comm;
        if (!G.window || !G.connected)
            ALQ_FAIL(ctx, ALQ_ERR_STATE, "%s: a sharded call (shard_off_host) needs the group of alq_comm_create/connect", fn);
        if (so[0] != 0 || so[G.world] != n)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: shard_off must run from 0 to n=%d, got %d .. %d", fn, n, so[0], so[G.world]);
        for (int r = 0; r < G.world; ++r)
            if (so[r + 1] < so[r]) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: shard_off[%d] = %d < shard_off[%d] = %d", fn, r + 1, so[r + 1], r, so[r]);
        S->world = G.world;
        S->rank = G.rank;
        std::copy(so, so + G.world + 1, S->off);
    }
    int rows_min = n;
    for (int r = 0; r < S->world; ++r) rows_min = std::min(rows_min, S->off[r + 1] - S->off[r]);
    S->grid = std::max(1, std::min(ctx->sm_count, (rows_min + 127) / 128));
    return ALQ_OK;
}

int alq_bal_seg_rows_max(const BalShard& S) {
    int m = 0;
    for (int g = 0; g < S.world * S.grid; ++g) m = std::max(m, gseg_lo(S, g + 1) - gseg_lo(S, g));
    return m;
}

size_t alq_bal_words_bytes(const BalShard& S, int64_t budget, bool sharded) {
    const size_t keyw = sharded ? kWordsHead : 0;
    return up128(keyw + static_cast<size_t>(2) * S.world * S.grid * 8) + static_cast<size_t>(budget) * 8;
}

int alq_bal_words_begin(alq_ctx* ctx, const BalShard& S, bool sharded, int budget, char* scratch, BalWords* W, cudaStream_t st) {
    *W = BalWords{};
    W->keyw = static_cast<unsigned int>(sharded ? kWordsHead : 0);
    W->pickw = static_cast<unsigned int>(up128(W->keyw + static_cast<size_t>(2) * S.world * S.grid * 8));
    const size_t end = alq_bal_words_bytes(S, budget, sharded);
    W->tag_base = 0x80000000u;
    if (!sharded) {
        W->peer[0] = scratch;
        ALQ_CUDA(ctx, cudaMemsetAsync(scratch, 0, end, st));
        return ALQ_OK;
    }
    // the words start without a valid tag; peers write them only after our ready word, which follows the clear
    ALQ_CUDA(ctx, cudaMemsetAsync(ctx->comm.window + kWordsHead, 0, end - kWordsHead, st));
    for (int r = 0; r < S.world; ++r) W->peer[r] = ctx->comm.peer[r];
    ctx->comm.epoch += 1;
    W->ready_tag = ctx->comm.epoch << 32;
    W->tag_base |= static_cast<unsigned int>(ctx->comm.epoch & 0x7fu) << 24;
    return alq_comm_ready(ctx, W->ready_tag, st);
}

int alq_bal_check_desc(alq_ctx* ctx, const alq_balancing_desc* D, const char* fn) {
    if (!D || D->struct_size < kBalDescV1) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: bad descriptor", fn);
    const int64_t n64 = D->n;
    const int c = D->c, d = D->d;
    if (n64 < 0 || n64 >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: n=%lld outside [0, 2^31)", fn, (long long)n64);
    if (c < 1 || c > ALQ_CLASS_MAX) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: C=%d outside [1, %d]", fn, c, ALQ_CLASS_MAX);
    if (d <= 0 || D->ldx < d || D->budget < 0)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: bad shape d=%d ldx=%lld budget=%lld", fn, d, (long long)D->ldx, (long long)D->budget);
    if (!D->mt_key_host || !D->mt_pos_host || !D->n_picks_host || !D->n_balancing_host ||
        (n64 > 0 && (!D->x || !D->xn || !D->labels || !D->avail || !D->labeled)) || (D->budget > 0 && !D->picks))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: null pointer", fn);
    if ((d % 4) || (D->ldx % 4) || (n64 > 0 && !aligned16(D->x)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: d and ldx must be multiples of 4 and x 16-byte aligned", fn);
    if (*D->mt_pos_host < 0 || *D->mt_pos_host > kMtN)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: MT19937 position %d outside [0, %d]", fn, *D->mt_pos_host, kMtN);
    *D->n_picks_host = -1;
    *D->n_balancing_host = 0;
    return ALQ_OK;
}

int alq_bal_counts(alq_ctx* ctx, const alq_balancing_desc* D, int n, int c, const BalShard& S, int32_t* tab, unsigned int* bad,
                   int32_t* counts, int32_t* seg_avail, int32_t* counts_h, int32_t* seg_h, cudaStream_t st, const char* fn) {
    const int nseg = S.world * S.grid;
    ALQ_CUDA(ctx, cudaMemsetAsync(bad, 0xff, 2 * sizeof(unsigned int), st));
    const int rc = alq_class_table_pass(ctx, D->labels, D->labeled, n, c, tab, bad, counts, st);
    if (rc != ALQ_OK) return rc;
    bal_seg_count_kernel<<<nseg, 256, 0, st>>>(D->labels, D->avail, c, S, seg_avail, bad + 1);
    ALQ_LAUNCH_CHECK(ctx);
    unsigned int bad_h[2] = {UINT_MAX, UINT_MAX};
    ALQ_CUDA(ctx, cudaMemcpyAsync(bad_h, bad, sizeof(bad_h), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(counts_h, counts, static_cast<size_t>(c) * 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(seg_h, seg_avail, static_cast<size_t>(nseg) * 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    for (int k = 1; k >= 0; --k)
        if (bad_h[k] != UINT_MAX) {
            int32_t y = 0;
            ALQ_CUDA(ctx, cudaMemcpy(&y, D->labels + bad_h[k], sizeof(int32_t), cudaMemcpyDeviceToHost));
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: %s row %u has label %d, outside [0, %d)", fn,
                     k ? "available" : "labeled", bad_h[k], y, c);
        }
    return ALQ_OK;
}

extern "C" int alq_balancing_select(alq_ctx* ctx, const alq_balancing_desc* D, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    int rc = alq_bal_check_desc(ctx, D, "alq_balancing_select");
    if (rc != ALQ_OK) return rc;
    const int64_t n64 = D->n;
    const int c = D->c, d = D->d;
    if (ctx->balancing_loop == 1 || ctx->balancing_loop == 3) return ALQ_OK;   // the per-step path or K12 runs
    const int n = static_cast<int>(n64);
    const bool forced = ctx->balancing_loop == 2;
    if (n == 0 || D->budget == 0) {
        *D->n_picks_host = 0;
        return ALQ_OK;
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);

    // ---- limits that the shape decides (the same on every rank of a sharded call) -------------------------------------
    BalShard S;
    bool sharded = false;
    rc = alq_bal_shard(ctx, D, n, &S, &sharded, "alq_balancing_select");
    if (rc != ALQ_OK) return rc;
    const int grid = S.grid, nseg = S.world * grid;
    const size_t smem = bal_loop_smem(c, d, nseg);
    const size_t sum_smem = static_cast<size_t>(c) * kSumDims * sizeof(double);
    const size_t smem_cap = ctx->smem_optin > 4096 ? ctx->smem_optin - 1024 : 0;   // the kernels' static shared memory
    if (smem > smem_cap || sum_smem > smem_cap) {
        if (!forced) return ALQ_OK;
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_balancing_select: the %d centres of %d floats need %zu bytes of shared memory, "
                 "%zu are available (limit: centres in shared memory)", c, d, std::max(smem, sum_smem), smem_cap);
    }
    if (alq_bal_seg_rows_max(S) > kSegRowsMax) {
        if (!forced) return ALQ_OK;
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_balancing_select: n=%d rows over %d CTAs exceed %d rows per CTA segment "
                 "(limit: rows per segment)", n, nseg, kSegRowsMax);
    }
    const int64_t budget_req = D->budget;
    const size_t words = alq_bal_words_bytes(S, std::min<int64_t>(budget_req, n), sharded);
    if (sharded && words > ctx->comm.greedy_bytes()) {
        if (!forced) return ALQ_OK;
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_balancing_select: a budget of %lld needs %zu bytes of the peer window, %zu are "
                 "usable (limit: words in the peer window)", (long long)budget_req, words, ctx->comm.greedy_bytes());
    }

    // ---- set-up: counts, segment counts, label checks -----------------------------------------------------------
    const int nchunks = (n + kSumChunk - 1) / kSumChunk;
    const size_t cd = static_cast<size_t>(c) * d;
    const size_t entries = alq_class_table_entries(n, c);
    const size_t need = scratch_need({entries * 4, static_cast<size_t>(c) * 4, 8, static_cast<size_t>(nseg) * 4,
                                      static_cast<size_t>(nchunks) * cd * 8, cd * 8, static_cast<size_t>(grid) * cd * 8,
                                      static_cast<size_t>(n), (kMtN + 1) * 4 * 2, sharded ? 0 : words, 16});
    rc = alq_scratch_reserve(ctx, need);
    if (rc != ALQ_OK) return rc;
    ScratchCursor cur(ctx->scratch);
    int32_t* tab = cur.take<int32_t>(entries);
    int32_t* counts = cur.take<int32_t>(c);
    unsigned int* bad = cur.take<unsigned int>(2);
    int32_t* seg_avail = cur.take<int32_t>(nseg);
    double* partial = cur.take<double>(static_cast<size_t>(nchunks) * cd);
    double* sums0 = cur.take<double>(cd);
    double* sums = cur.take<double>(static_cast<size_t>(grid) * cd);
    uint8_t* avail = cur.take<uint8_t>(n);
    unsigned int* mt = cur.take<unsigned int>(2 * (kMtN + 1));
    char* word_scratch = cur.take<char>(sharded ? 0 : words);
    int* small = cur.take<int>(4);                                     // [0] status, [1] balancing steps

    std::vector<int32_t> counts_h(c), seg_h(nseg);
    rc = alq_bal_counts(ctx, D, n, c, S, tab, bad, counts, seg_avail, counts_h.data(), seg_h.data(), st, "alq_balancing_select");
    if (rc != ALQ_OK) return rc;
    int64_t n_avail = 0, labeled_total = 0;
    for (int g = 0; g < nseg; ++g) n_avail += seg_h[g];
    for (int k = 0; k < c; ++k) labeled_total += counts_h[k];
    const int budget = static_cast<int>(std::min<int64_t>(budget_req, n_avail));
    if (labeled_total + budget >= (1LL << 24)) {
        if (!forced) return ALQ_OK;
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_balancing_select: %lld labeled rows plus a budget of %d reach 2^24 "
                 "(limit: counts plus budget below 2^24)", (long long)labeled_total, budget);
    }
    if (budget == 0) {
        *D->n_picks_host = 0;
        return ALQ_OK;
    }

    // ---- fp64 class sums, the working mask, the RNG state -------------------------------------------------------
    if (sum_smem > 48u * 1024u)
        ALQ_CUDA(ctx, cudaFuncSetAttribute(bal_class_sum_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sum_smem)));
    bal_class_sum_partial_kernel<<<dim3((d + kSumDims - 1) / kSumDims, nchunks), kSumDims, sum_smem, st>>>(
        D->x, D->ldx, d, D->labels, D->labeled, n, c, partial);
    ALQ_LAUNCH_CHECK(ctx);
    bal_class_sum_reduce_kernel<<<static_cast<int>((cd + 255) / 256), 256, 0, st>>>(partial, nchunks, static_cast<long long>(cd), sums0);
    ALQ_LAUNCH_CHECK(ctx);
    std::vector<unsigned int> mt_h(kMtN + 1);
    std::copy(D->mt_key_host, D->mt_key_host + kMtN, mt_h.begin());
    mt_h[kMtN] = static_cast<unsigned int>(*D->mt_pos_host);
    ALQ_CUDA(ctx, cudaMemcpyAsync(mt, mt_h.data(), (kMtN + 1) * 4, cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(avail, D->avail, static_cast<size_t>(n), cudaMemcpyDeviceToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(small, 0, 4 * sizeof(int), st));

    // ---- the loop ---------------------------------------------------------------------------------------------------
    BalArgs A{};
    rc = alq_bal_words_begin(ctx, S, sharded, budget, word_scratch, &A.W, st);
    if (rc != ALQ_OK) return rc;
    A.x = D->x; A.ldx = D->ldx; A.d = d;
    A.xn = D->xn; A.labels = D->labels; A.avail = avail;
    A.sums0 = sums0; A.sums = sums; A.counts0 = counts; A.seg_avail0 = seg_avail;
    A.mt_in = mt; A.mt_out = mt + kMtN + 1;
    A.picks = D->picks; A.n_bal = small + 1; A.status = small;
    A.S = S;
    A.n = n; A.c = c; A.budget = budget; A.n_avail = static_cast<int>(n_avail);
    A.timeout_cycles = static_cast<long long>(ctx->spin_timeout_ms) * ctx->clock_khz;
    ALQ_CUDA(ctx, cudaFuncSetAttribute(balancing_loop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    // every CTA spins on the others' words, so all of them must be resident: grid <= SMs, one CTA per SM at most
    // (see alq_score.cu on why this is an ordinary launch and what alq_gridsync_begin/end guard against)
    alq_gridsync_begin(ctx, st);
    balancing_loop_kernel<<<grid, kBalThreads, smem, st>>>(A);
    const cudaError_t le = cudaGetLastError();
    alq_gridsync_end(ctx, st);
    ctx->launches++;
    if (le != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_balancing_select: launch failed: %s (grid %d, %zu B shared)", cudaGetErrorString(le), grid, smem);

    int small_h[2] = {0, 0};
    ALQ_CUDA(ctx, cudaMemcpyAsync(small_h, small, sizeof(small_h), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(mt_h.data(), A.mt_out, (kMtN + 1) * 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (small_h[0] != 0) ALQ_FAIL(ctx, small_h[0], "alq_balancing_select: timed out waiting for a peer GPU or a CTA of the grid");
    std::copy(mt_h.begin(), mt_h.begin() + kMtN, D->mt_key_host);
    *D->mt_pos_host = static_cast<int32_t>(mt_h[kMtN]);
    *D->n_picks_host = budget;
    *D->n_balancing_host = small_h[1];
    return ALQ_OK;
}

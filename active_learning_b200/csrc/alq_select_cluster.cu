// K1b, cluster-resident: the whole stable top-B selection in ONE launch for pools that fit the shared
// memory of a thread-block cluster (n <= 8 * 32768 scores, b <= 16384).  Same contract and same result as
// the multi-kernel path in alq_select.cu (`torch.sort(scores).indices[:B]` of margin_sampler.py:42 under
// active_learning/src/query_strategies, ties by lowest position).
//
// One cluster of 8 CTAs; every CTA keeps its slice of the order-preserving uint32 score keys in shared
// memory for the whole kernel.  Stages are separated by cluster barriers (~0.4 us) instead of kernel
// boundaries (~7 us each in the multi-kernel path, which is latency-bound: 320 KB of data):
//   1-3  three MSB radix levels (11+11+10 bits): per-CTA histogram (warp-aggregated shared atomics) ->
//        global partials -> barrier -> every CTA reduces the 8 partials and locates the bin itself;
//   4    per-CTA counts of {key < T} and {key == T} -> barrier -> exclusive offsets;
//   5    compaction of the B winners as 64-bit words (key << 32 | position); ties with T are taken in
//        position order by one warp walking the slice with ballots;
//   6    every CTA sorts its share (B/8 words) in shared memory (bitonic network) -> barrier;
//   7    every CTA pulls all sorted shares into shared memory and places its own words by binary searches.
#include "alq_common.cuh"

namespace selc {

constexpr int CL = 8;
constexpr int THREADS = 1024;
constexpr int MAX_SLICE = 32768;          // keys per CTA
constexpr int BINS = 2048;
constexpr int MAX_B = 16384;

struct Scratch {
    uint32_t* hist_part;        // [3][CL][BINS]
    uint32_t* counts;           // [CL][2]  (lt, eq)
    unsigned long long* words;  // [MAX_B]      winners, unordered
    unsigned long long* sorted; // [MAX_B + 2]  per-CTA sorted shares
};

__device__ __forceinline__ uint32_t score_key(float s) { return alq_ord(s + 0.0f); }

__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(THREADS, 1)
select_cluster_kernel(const float* __restrict__ scores, int n, int b, Scratch S, int32_t* __restrict__ out_pos) {
    extern __shared__ __align__(16) unsigned char smem_sel[];
    uint32_t* keys = reinterpret_cast<uint32_t*>(smem_sel);                       // [slice]  (later: all runs)
    __shared__ uint32_t hist[BINS];
    __shared__ unsigned long long part[THREADS / 32];
    __shared__ uint32_t sh_prefix;
    __shared__ unsigned long long sh_k;
    __shared__ uint32_t w_lt[THREADS / 32], w_eq[THREADS / 32];
    __shared__ __align__(8) uint64_t sh_bar;
    const int rank = static_cast<int>(cluster_rank());
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int per = ((n + CL - 1) / CL + 3) & ~3;
    const int lo = rank * per, hi = min(n, lo + per);
    const int cnt = max(0, hi - lo);

    // ---- stage 0: slice -> keys in shared memory, level-0 histogram on the way -------------------------------
    for (int i = threadIdx.x; i < BINS; i += THREADS) hist[i] = 0;
    if (threadIdx.x == 0) { sh_prefix = 0; sh_k = static_cast<unsigned long long>(b); }
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += THREADS) {
        const uint32_t key = score_key(scores[lo + i]);
        keys[i] = key;
        atomicAdd(&hist[key >> 21], 1u);
    }
    __syncthreads();

    // ---- stages 1-3: radix levels ---------------------------------------------------------------------------
#pragma unroll 1
    for (int level = 0; level < 3; ++level) {
        const uint32_t prefix = sh_prefix;
        if (level > 0) {
            for (int i = threadIdx.x; i < BINS; i += THREADS) hist[i] = 0;
            __syncthreads();
            for (int i = threadIdx.x; i < cnt; i += THREADS) {
                const uint32_t key = keys[i];
                if (level == 1) { if ((key >> 21) == prefix) atomicAdd(&hist[(key >> 10) & 0x7ffu], 1u); }
                else { if ((key >> 10) == prefix) atomicAdd(&hist[key & 0x3ffu], 1u); }
            }
            __syncthreads();
        }
        uint32_t* mine = S.hist_part + (static_cast<size_t>(level) * CL + rank) * BINS;
        for (int i = threadIdx.x; i < BINS; i += THREADS) mine[i] = hist[i];
        cluster_sync_all();
        // every CTA reduces the CL partial histograms itself: 2 bins per thread (one 8-byte load per partial)
        unsigned long long c0 = 0, c1 = 0;
        uint2 pv[CL];
#pragma unroll
        for (int q = 0; q < CL; ++q)
            pv[q] = __ldcg(reinterpret_cast<const uint2*>(S.hist_part + (static_cast<size_t>(level) * CL + q) * BINS) + threadIdx.x);
#pragma unroll
        for (int q = 0; q < CL; ++q) { c0 += pv[q].x; c1 += pv[q].y; }
        unsigned long long inc = c0 + c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) part[warp] = inc;
        __syncthreads();
        unsigned long long woff = 0;
        for (int w = 0; w < warp; ++w) woff += part[w];
        const unsigned long long incl = woff + inc, excl = incl - (c0 + c1);
        const unsigned long long k = sh_k;
        __syncthreads();
        if (excl < k && k <= incl) {
            const bool first = k <= excl + c0;
            const uint32_t bin = 2 * threadIdx.x + (first ? 0 : 1);
            sh_prefix = level == 2 ? ((prefix << 10) | bin) : ((prefix << 11) | bin);
            sh_k = first ? k - excl : k - excl - c0;
        }
        __syncthreads();
    }
    const uint32_t T = sh_prefix;
    const unsigned long long ties = sh_k;                       // how many keys equal to T are inside the budget
    const unsigned long long n_less = static_cast<unsigned long long>(b) - ties;

    // ---- stage 4: counts and offsets.  Warp w owns the contiguous chunk [w*chunk, (w+1)*chunk) of the slice, so
    //      "ties by position" is an exclusive prefix over (CTA, warp, ballot lane) ----------------------------------
    const int chunk = ((cnt + 31) / 32 + 31) & ~31;
    const int c_lo = min(cnt, warp * chunk), c_hi = min(cnt, c_lo + chunk);
    uint32_t lt = 0, eq = 0;
    for (int i = c_lo + lane; i < c_hi; i += 32) {
        const uint32_t key = keys[i];
        lt += key < T;
        eq += key == T;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lt += __shfl_xor_sync(0xffffffffu, lt, o);
        eq += __shfl_xor_sync(0xffffffffu, eq, o);
    }
    if (lane == 0) { w_lt[warp] = lt; w_eq[warp] = eq; }
    __syncthreads();
    uint32_t lt_before = 0, eq_before = 0, lt_cta = 0, eq_cta = 0;
    for (int w = 0; w < THREADS / 32; ++w) {
        if (w == warp) { lt_before = lt_cta; eq_before = eq_cta; }
        lt_cta += w_lt[w];
        eq_cta += w_eq[w];
    }
    if (threadIdx.x == 0) { S.counts[rank * 2] = lt_cta; S.counts[rank * 2 + 1] = eq_cta; }
    cluster_sync_all();
    uint32_t lt_off = 0, eq_off = 0;
    for (int q = 0; q < rank; ++q) {
        lt_off += __ldcg(&S.counts[q * 2]);
        eq_off += __ldcg(&S.counts[q * 2 + 1]);
    }

    // ---- stage 5: compaction of the B winners as (key << 32 | position) words ------------------------------------
    {
        uint32_t lt_run = lt_off + lt_before;
        unsigned long long eq_run = static_cast<unsigned long long>(eq_off) + eq_before;
        for (int i0 = c_lo; i0 < c_hi; i0 += 32) {
            const int i = i0 + lane;
            const uint32_t key = i < c_hi ? keys[i] : 0xffffffffu;
            const bool is_lt = i < c_hi && key < T, is_eq = i < c_hi && key == T;
            const unsigned m_lt = __ballot_sync(0xffffffffu, is_lt), m_eq = __ballot_sync(0xffffffffu, is_eq);
            const unsigned below = (1u << lane) - 1u;
            const unsigned long long word = (static_cast<unsigned long long>(key) << 32) | static_cast<uint32_t>(lo + i);
            if (is_lt) S.words[lt_run + __popc(m_lt & below)] = word;
            if (is_eq) {
                const unsigned long long r = eq_run + __popc(m_eq & below);
                if (r < ties) S.words[n_less + r] = word;
            }
            lt_run += __popc(m_lt);
            eq_run += __popc(m_eq);
        }
    }
    cluster_sync_all();

    // ---- stage 6: every CTA sorts its share of the words (<= MAX_B / CL = 2048, padded with ~0) with a bitonic
    //      network in shared memory (an all-pairs rank count was measured 3x slower: 79k vs 27k cycles) ---------
    unsigned long long* sk = reinterpret_cast<unsigned long long*>(smem_sel);      // the key slice is no longer needed
    const int share = (b + CL - 1) / CL;
    const int s_lo = min(b, rank * share), s_hi = min(b, s_lo + share), s_cnt = s_hi - s_lo;
    int npad = 64;
    while (npad < share) npad <<= 1;                         // same in every CTA; <= 2048 = 2 * THREADS
    for (int i = threadIdx.x; i < npad; i += THREADS) sk[i] = i < s_cnt ? __ldcg(&S.words[s_lo + i]) : ~0ull;
    __syncthreads();
    alq_bitonic_sort_smem(sk, npad);
    for (int i = threadIdx.x; i < s_cnt; i += THREADS) S.sorted[s_lo + i] = sk[i];
    cluster_sync_all();

    // ---- stage 7: all sorted shares into shared memory, place this CTA's share by rank counting -------------------
    {
        // one TMA bulk copy per CTA brings all sorted shares (<= 128 KB) into shared memory
        if (threadIdx.x == 0) {
            mbar_init(&sh_bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t bytes = static_cast<uint32_t>(((b + 1) & ~1) * 8);
            mbar_expect_tx(&sh_bar, bytes);
            bulk_g2s(sk, S.sorted, bytes, &sh_bar);
        }
        mbar_wait(&sh_bar, 0);
    }
    for (int i = s_lo + threadIdx.x; i < s_hi; i += THREADS) {
        const unsigned long long key = sk[i];
        int rk = i - s_lo;
        // the searches in the other CL-1 shares are independent: advance them in lock step (12 rounds)
        int l[CL], h[CL], base[CL];
#pragma unroll
        for (int r = 0; r < CL; ++r) {
            base[r] = min(b, r * share);
            l[r] = 0;
            h[r] = r == rank ? 0 : min(b, base[r] + share) - base[r];
        }
#pragma unroll 1
        for (int step = 0; step < 12; ++step) {
#pragma unroll
            for (int r = 0; r < CL; ++r) {
                if (l[r] < h[r]) {
                    const int mid = (l[r] + h[r]) >> 1;
                    if (sk[base[r] + mid] < key) l[r] = mid + 1; else h[r] = mid;
                }
            }
        }
#pragma unroll
        for (int r = 0; r < CL; ++r) rk += l[r];
        out_pos[rk] = static_cast<int32_t>(key & 0xffffffffu);
    }
}

}  // namespace selc

// Returns ALQ_ERR_STATE when the problem does not fit this kernel (caller uses the multi-kernel path).
int alq_select_smallest_cluster(alq_ctx* ctx, const float* scores, int64_t n, int64_t b, int32_t* out_pos,
                                cudaStream_t st) {
    using namespace selc;
    if (n > static_cast<int64_t>(CL) * MAX_SLICE || b > MAX_B || n < 1 || b < 1) return ALQ_ERR_STATE;
    const size_t hist_bytes = static_cast<size_t>(3) * CL * BINS * sizeof(uint32_t);
    int rc = alq_scratch_reserve(ctx, scratch_need({hist_bytes, CL * 2 * sizeof(uint32_t), MAX_B * sizeof(unsigned long long),
                                                    (MAX_B + 2) * sizeof(unsigned long long)}));
    if (rc) return rc;
    ScratchCursor cur(ctx->scratch);
    Scratch S;
    S.hist_part = cur.take<uint32_t>(3 * CL * BINS);
    S.counts = cur.take<uint32_t>(CL * 2);
    S.words = cur.take<unsigned long long>(MAX_B);
    S.sorted = cur.take<unsigned long long>(MAX_B + 2);
    const int per = ((static_cast<int>(n) + CL - 1) / CL + 3) & ~3;
    size_t smem = std::max<size_t>(std::max<size_t>(static_cast<size_t>(per) * 4, static_cast<size_t>(b + 2) * 8), 2048 * 8) + 64;
    if (smem > ctx->smem_optin - 24 * 1024) return ALQ_ERR_STATE;
    static size_t attr_set = 0;
    if (smem > attr_set) {
        ALQ_CUDA(ctx, cudaFuncSetAttribute(select_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        attr_set = smem;
    }
    select_cluster_kernel<<<CL, THREADS, smem, st>>>(scores, static_cast<int>(n), static_cast<int>(b), S, out_pos);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

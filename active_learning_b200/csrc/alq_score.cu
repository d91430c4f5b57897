// K1 (softmax-uncertainty scores), K2 (BADGE gradient-embedding factors), K2p (pooled embedding)
// and row norms.  All are one-pass HBM-streaming kernels: one warp owns one row, the row lives in
// registers between the max pass and the exp pass, loads are 128-bit and L1-bypassing.
//
// Reference semantics: margin_sampler.py:33-35, confidence_sampler.py:31-33,
// badge_sampler.py:33-44, coreset_sampler.py:61 (all under active_learning/src/query_strategies).
#include <initializer_list>
#include <stdlib.h>

#include "alq_ll.cuh"
#include "alq_mase_rows.cuh"

namespace {

constexpr int kScoreThreads = 256;

struct RowStats {
    float m;    // max logit
    float t2;   // second largest logit (== m when the max is repeated)
    float s;    // sum exp(z - m)
    float w;    // sum exp(z - m) * (z - m)      (entropy only)
    int arg;    // lowest index attaining m       (BADGE only)
};

__device__ __forceinline__ void top2_push(float v, float& t1, float& t2) {
    if (v > t1) { t2 = t1; t1 = v; }
    else if (v > t2) t2 = v;
}

// exp(x) for x <= 0 as one FMUL + one MUFU.EX2 (ex2.approx: 2^-22 relative error; the product's
// rounding adds <= 6e-8*|x*log2e| to the exponent, i.e. it only matters where exp(x) is tiny).
// K1 is issue-bound with libdevice expf (25 instr/element, ncu r01); this keeps it memory-bound.
__device__ __forceinline__ float exp_neg(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x * 1.4426950408889634f));
    return r;
}

// Row held as NV float4 per lane (vector path); slots past the row end hold -inf ------------------
template <int NV, bool WANT_T2, bool WANT_ARG, bool WANT_W>
__device__ __forceinline__ RowStats row_stats_vec(const float4 (&v)[NV], int lane, int nvec) {
    float t1 = ALQ_NEG_INF, t2 = ALQ_NEG_INF;
    int arg = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const float e[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (WANT_ARG && e[j] > t1) arg = (lane + 32 * k) * 4 + j;   // strict: first occurrence wins
            if (WANT_T2) t2 = fmaxf(t2, fminf(t1, e[j]));               // branch-free running top-2
            t1 = fmaxf(t1, e[j]);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float o1 = __shfl_xor_sync(0xffffffffu, t1, o);
        if (WANT_ARG) {
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (o1 > t1 || (o1 == t1 && oa < arg)) arg = oa;
        }
        if (WANT_T2) {
            const float o2 = __shfl_xor_sync(0xffffffffu, t2, o);
            t2 = fmaxf(fminf(t1, o1), fmaxf(t2, o2));
        }
        t1 = fmaxf(t1, o1);
    }
    float s = 0.f, w = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const float e[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float dz = e[j] - t1;          // -inf in padded slots and masked classes -> exp 0
            const float ex = exp_neg(dz);
            s += ex;
            if (WANT_W) w = ex > 0.f ? fmaf(ex, dz, w) : w;   // 0 log 0 = 0: no 0 * -inf
        }
    }
    s = warp_sum(s);
    if (WANT_W) w = warp_sum(w);
    return RowStats{t1, t2, s, w, arg};
}

template <int NV>
__device__ __forceinline__ void load_row_vec(const float4* p, int lane, int nvec, float4 (&v)[NV]) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int idx = lane + 32 * k;
        v[k] = idx < nvec ? ld_stream_f4(p + idx) : make_float4(ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF);
    }
}

__device__ __forceinline__ float score_from_stats(const RowStats& r, int mode) {
    if (mode == ALQ_MODE_MARGIN) {
        // p(1) - p(2) with p = exp(z - max) / sum, each quotient rounded like torch's softmax
        return 1.0f / r.s - exp_neg(r.t2 - r.m) / r.s;
    }
    if (mode == ALQ_MODE_LEAST_CONFIDENCE) return 1.0f / r.s;
    // sum_c p_c log p_c = (sum e*(z-m))/s - log s
    float sc = r.w / r.s - logf(r.s);
    return sc + 0.0f;  // canonical +0
}

template <int NV, int MODE>
__global__ void __launch_bounds__(kScoreThreads)
score_rows_vec_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld,
                      float* __restrict__ scores) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int nvec = c >> 2;
    for (int64_t row = warp; row < n; row += nwarps) {
        const float4* p = reinterpret_cast<const float4*>(logits + row * ld);
        float4 v[NV];
        load_row_vec<NV>(p, lane, nvec, v);
        const RowStats r = row_stats_vec<NV, MODE == ALQ_MODE_MARGIN, false, MODE == ALQ_MODE_ENTROPY>(v, lane, nvec);
        if (lane == 0) scores[row] = score_from_stats(r, MODE);
    }
}

// `row` and `n` are positions in the loader order of the WHOLE pool (a shard passes its row offset)
__device__ __forceinline__ float batch_scale(int64_t row, int64_t n, int bs) {
    const int64_t tail = n % bs;
    const int64_t cut = n - tail;
    return 1.0f / static_cast<float>(row < cut ? bs : static_cast<int>(tail));
}

// ---------------------------------------------------------------------------------------------
// K1 / K2, pipelined: one CTA per SM, a producer lane streams tiles of contiguous rows into a ring of
// shared-memory stages with cp.async.bulk (TMA bulk copy, mbarrier complete_tx); every consumer warp
// owns whole tiles, pulls each row smem -> registers and runs the same row code as the direct kernel.
// ~200 KB of loads in flight per SM independent of register pressure: this is what took the step
// kernel of alq_greedy.cu to 0.93-0.97 of the HBM peak.
// ---------------------------------------------------------------------------------------------
struct RowPipeCfg {
    int rows_per_tile, stages, consumers, tile_floats;
    int split;      // consumer warps per tile (rows of a tile are dealt round-robin to them)
};

template <int NV>
__device__ __forceinline__ void load_row_smem(const float4* p, int lane, int nvec, float4 (&v)[NV]) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int idx = lane + 32 * k;
        v[k] = idx < nvec ? p[idx] : make_float4(ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF, ALQ_NEG_INF);
    }
}

// ---- fused stable top-B (K1 + K1b in ONE cooperative launch) ---------------------------------------------------
// The scoring kernel already runs one CTA per SM; with the selection as a separate launch the step paid a 43 us
// 8-SM cluster kernel plus launch gaps behind a 56 us stream.  Fused: every CTA keeps the (key, row) words of the rows
// it scored in shared memory and counts their 11 top key bits on the way; after the stream
//   E1 the per-CTA histograms are added into a global one (red.add), grid barrier;
//   E2 every CTA finds the bin T that holds the b-th smallest key;
//   E3 keeps its words with bin <= T (all of the winners plus the few other keys of bin T) and appends them to a
//      global candidate list (one atomicAdd per CTA reserves the slots), grid barrier;
//   E4 pulls the whole candidate list (b + a few words) into the shared memory the tile ring no longer needs and ranks
//      its OWN candidates against it by counting (warp per candidate): rank < b  ->  out_pos[rank] = row.
// Words are key << 32 | row, so the order is (score, position): exactly K1b's stable order
// (`torch.sort(scores).indices[:B]`, margin_sampler.py:42), whatever the order the candidates were appended in.
struct SelArgs {
    int b;                          // 0: plain scoring kernel
    int list_cap;                   // (key, row) words a CTA can hold
    int list_off;                   // byte offset of that list in dynamic shared memory (everything below it becomes the
                                    // epilogue's buffer once the stream is over: at least 80 KB, more with a big tile ring)
    unsigned int* g_hist;           // [2 * 2048] zeroed: level-0 and level-1 histograms
    unsigned int* g_ctr;            // [4] zeroed: [0] grid-barrier arrivals, [1] candidates appended
    unsigned long long* g_cand;     // [n]
    int32_t* out_pos;               // [b]
    // the sharded call (`world` >= 1 ranks; 0, as zero-initialised, for the one-GPU call): the histograms are summed and
    // the candidates gathered through the peer-memory windows from inside this kernel, every rank ends with the same list
    int world, rank;
    unsigned int row_base;          // global position of this rank's row 0
    char* peer[ALQ_MAX_WORLD];
    unsigned long long hist_off;    // u64 LL words [2 levels][world][2048]   {tag32, count32}
    unsigned long long cnt_off;     // u64 LL words [world][stride]            {tag32, candidates of that CTA}
    unsigned long long cand_off;    // u64 raw words [world][cand_cap]
    int stride, cand_cap;
    unsigned int tag;               // 0x80000000 | call epoch
    long long timeout_cycles;
    int* status;                    // mapped host word (sticky)
    unsigned int* g_tot;            // [2 * 2048] histograms summed over the ranks (local)
    // bucket route of the ranking stage (one GPU; nullptr: off): candidates are routed to CTA `bucket` by a monotone
    // function of their score, so a CTA only sorts its own bucket -- see select_epilogue
    unsigned long long* g_bucket;   // [grid][kBucketLanes][bucket_cap]
    unsigned int* g_bcnt;           // [grid][kBucketLanes] zeroed
    int bucket_cap;                 // words per sub-list
    int ring_off, ring_bars;        // byte offset and count of the tile ring's full[] / empty[] mbarriers
};
constexpr int kBucketLanes = 16;

// inverse of alq_ord
__device__ __forceinline__ float sel_key_to_float(uint32_t key) {
    return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

__device__ __forceinline__ void sel_grid_barrier(unsigned int* ctr, unsigned int target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        unsigned int v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (static_cast<int>(v - target) < 0);
    }
    __syncthreads();
}

// Bin (of 2048) holding the k-th smallest entry of the histogram in shared memory, and k minus the entries below that
// bin.  The first 32 warps each sum 64 bins (two per lane), warp 0 scans the 32 warp totals, the warp that holds the
// bin scans its lanes.  Called by the whole CTA (needs >= 32 warps ... or loops); ends with a barrier.
__device__ __forceinline__ void sel_find_bin(const uint32_t* hist, uint32_t k, uint32_t* s_wsum, int* out_bin, int* out_rest) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    for (int w = warp; w < 32; w += nwarp) {
        uint32_t v = hist[w * 64 + 2 * lane] + hist[w * 64 + 2 * lane + 1];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_wsum[w] = v;
    }
    __syncthreads();
    if (warp == 0) {
        const uint32_t tot = s_wsum[lane];
        uint32_t inc = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        const uint32_t excl = inc - tot;
        const unsigned hit = __ballot_sync(0xffffffffu, excl < k && k <= inc);
        const int w = hit ? __ffs(hit) - 1 : 31;             // the 64-bin group holding the k-th entry
        const uint32_t before = __shfl_sync(0xffffffffu, excl, w);
        const uint32_t a = hist[w * 64 + 2 * lane], b2 = hist[w * 64 + 2 * lane + 1];
        uint32_t pinc = a + b2;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, pinc, o);
            if (lane >= o) pinc += v;
        }
        const uint32_t pexcl = before + pinc - (a + b2);
        if (pexcl < k && k <= pexcl + a + b2) {
            const bool first = k <= pexcl + a;
            *out_bin = w * 64 + 2 * lane + (first ? 0 : 1);
            *out_rest = static_cast<int>(first ? k - pexcl : k - pexcl - a);
        }
    }
    __syncthreads();
}

// Stages shared by both epilogues.  s_misc: [0] words in s_list, [1] level-0 bin, [2] rank still wanted inside it,
// [3] offset in the candidate list, [4] own candidates, [5] level-1 bin, [6] 2047 - first populated level-0 bin,
// [8..9] the list-streaming mbarrier, [16..47] sel_find_bin's scratch, [48..] the bucket route's counters.

// %globaltimer stamp i of CTA 0, read back by alq_uncertainty_tail_timing: [0] kernel start, [1] every CTA of this GPU
// has streamed its rows, [2] kernel end
__device__ __forceinline__ void sel_stamp(unsigned int* g_ctr, int i) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        reinterpret_cast<unsigned long long*>(g_ctr + 4)[i] = t;
    }
}

// this CTA's 2048-bin histogram added into a global one
__device__ __forceinline__ void sel_push_hist(const uint32_t* s_hist, unsigned int* g) {
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) {
        const uint32_t h = s_hist[i];
        if (h) atomicAdd(g + i, h);
    }
}

// a global 2048-bin histogram -> shared memory; with `first` (zero on entry) also the first populated bin, as
// 2047 - bin in *first
__device__ __forceinline__ void sel_load_hist(const unsigned int* g, uint32_t* s_hist, int* first) {
    const int tid = threadIdx.x, nthr = blockDim.x;
    uint32_t hv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) hv[k] = (tid + k * nthr) < 2048 ? __ldcg(g + tid + k * nthr) : 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if ((tid + k * nthr) < 2048) {
            s_hist[tid + k * nthr] = hv[k];
            if (first && hv[k]) atomicMax(first, 2047 - (tid + k * nthr));
        }
}

// Level 1: the next 11 bits of this CTA's keys inside level-0 bin T0 -> s_hist (a float score has few distinct
// exponents, so one level alone can leave most of the pool in the boundary bin)
__device__ __forceinline__ void sel_level1_hist(const unsigned long long* s_list, int cnt, uint32_t T0, uint32_t* s_hist) {
    const int tid = threadIdx.x, nthr = blockDim.x;
    for (int i = tid; i < 2048; i += nthr) s_hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < cnt; i += nthr) {
        const uint32_t key = static_cast<uint32_t>(s_list[i] >> 32);
        if ((key >> 21) == T0) atomicAdd(&s_hist[(key >> 10) & 0x7ffu], 1u);
    }
    __syncthreads();
}

// This CTA's candidates -- every word whose 22-bit key prefix is <= T: the winners plus the few other keys sharing the
// prefix T -- into buf[0, nc), counted in s_misc[4] (zero on entry); nc slots of the candidate count g_ctr[1] are
// reserved, starting at `off`.  Returns nc.
__device__ __forceinline__ int sel_gather_candidates(const SelArgs& S, const unsigned long long* s_list, int cnt, uint32_t T,
                                                     unsigned long long* buf, int* s_misc, int& off) {
    const int tid = threadIdx.x, nthr = blockDim.x;
    for (int i = tid; i < cnt; i += nthr) {
        const unsigned long long w = s_list[i];
        if (static_cast<uint32_t>(w >> 42) <= T) buf[atomicAdd(&s_misc[4], 1)] = w;
    }
    __syncthreads();
    const int nc = s_misc[4];
    if (tid == 0) s_misc[3] = static_cast<int>(atomicAdd(S.g_ctr + 1, static_cast<unsigned int>(nc)));
    __syncthreads();
    off = s_misc[3];
    return nc;
}

// Score buckets of the bucket route.  Every candidate score lies in [lo, hi] = [lower edge of the first populated
// level-0 bin, upper edge of prefix T]; bucket(score) = floor((score - lo) * nb / (hi - lo)), clamped, is monotone in the
// key, so bucket q holds exactly the ranks [words in the buckets below q, ...).  Scores that do not spread and non-finite
// edges leave `spread` false; every thread of every CTA computes the same value from the same histogram.
struct SelBuckets {
    float lo, scale;
    int nb;
    bool spread;
    __device__ __forceinline__ SelBuckets(int first_bin, uint32_t T, int nbuckets) : nb(nbuckets) {
        lo = sel_key_to_float(static_cast<uint32_t>(first_bin) << 21);
        const float hi = sel_key_to_float((T << 10) | 0x3ffu);
        scale = static_cast<float>(nb) / (hi - lo);
        spread = isfinite(lo) && isfinite(hi) && hi > lo && isfinite(scale);
    }
    __device__ __forceinline__ int of(unsigned long long w) const {
        const float sc = sel_key_to_float(static_cast<uint32_t>(w >> 32));
        return min(nb - 1, max(0, __float2int_rd((sc - lo) * scale)));
    }
};

// One bucket w[0, mine) ordered by counting (the words are distinct: the row is part of them); `base` words lie in the
// buckets below.  Rank < b -> out_pos[rank] = row.
__device__ __forceinline__ void sel_rank_bucket(const unsigned long long* w, int mine, int base, int b, int32_t* out_pos) {
    for (int i = threadIdx.x; i < mine; i += blockDim.x) {
        const unsigned long long x = w[i];
        int r = base;
        for (int q = 0; q < mine; ++q) r += w[q] < x;
        if (r < b) out_pos[r] = static_cast<int32_t>(x & 0xffffffffu);
    }
}

// Streams src[0, total) through buf[0, buf_cap) with the whole CTA: one TMA bulk copy per chunk, completing on `bar`,
// then body(words in the chunk).  overlap() runs while the first chunk is in flight.  `bar` is initialised here and
// invalidated before the return; buf must be free on entry.
template <class Overlap, class Body>
__device__ __forceinline__ void sel_stream_list(const unsigned long long* src, int total, unsigned long long* buf, int buf_cap,
                                                uint64_t* bar, Overlap&& overlap, Body&& body) {
    const int tid = threadIdx.x;
    auto copy = [&](int base, int m) {
        const uint32_t bytes = static_cast<uint32_t>((m + 1) & ~1) * 8u;
        mbar_expect_tx(bar, bytes);
        bulk_g2s(buf, src + base, bytes, bar);
    };
    if (tid == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0 && total > 0) copy(0, min(buf_cap, total));
    overlap();
    uint32_t phase = 0;
    for (int base = 0; base < total; base += buf_cap) {
        const int m = min(buf_cap, total - base);
        __syncthreads();                                    // the previous chunk is consumed
        if (base > 0 && tid == 0) copy(base, m);
        mbar_wait(bar, phase);
        phase ^= 1u;
        body(m);
    }
    __syncthreads();
    if (tid == 0) mbar_inval(bar);
}

// s_diff[number of own candidates <= x] += 1 for every word x of buf[0, m): a binary search in the sorted own[0, nc)
__device__ __forceinline__ void sel_count_into_diff_sorted(const unsigned long long* buf, int m, const unsigned long long* own,
                                                           int nc, uint32_t* s_diff) {
    const int tid = threadIdx.x, nthr = blockDim.x;
    for (int j = tid; j < m; j += nthr) {
        const unsigned long long x = buf[j];
        int lo = 0, hi = nc;                                // first own candidate > x
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (own[mid] <= x) lo = mid + 1; else hi = mid;
        }
        atomicAdd(&s_diff[lo], 1u);
    }
}

// The prefix sum of the difference array is the rank of each sorted own word own[0, nc): rank < b -> out_pos[rank] = row
// (~0 words pad the sharded list and are never written)
__device__ __forceinline__ void sel_write_ranks(uint32_t* s_diff, const unsigned long long* own, int nc, int b, int32_t* out_pos) {
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
    if (tid < 32) {
        uint32_t carry = 0;
        for (int base = 0; base < nc; base += 32) {
            const int i = base + lane;
            uint32_t v = i < nc ? s_diff[i] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v += t;
            }
            if (i < nc) s_diff[i] = carry + v;
            carry += __shfl_sync(0xffffffffu, v, 31);
        }
    }
    __syncthreads();
    for (int i = tid; i < nc; i += nthr) {
        const uint32_t r = s_diff[i];
        const unsigned long long w = own[i];
        if (r < static_cast<uint32_t>(b) && w != ~0ull) out_pos[r] = static_cast<int32_t>(w & 0xffffffffu);
    }
}

__device__ __noinline__ void select_epilogue(const SelArgs& S, uint32_t* s_hist, unsigned long long* s_list, int* s_misc,
                                             unsigned long long* buf, int buf_cap) {
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
    __syncthreads();                                        // every consumer warp has appended its rows
    const int cnt = s_misc[0];
    // ---- level 0: the 11 top key bits were counted while the rows streamed ----
    sel_push_hist(s_hist, S.g_hist);
    sel_grid_barrier(S.g_ctr, gridDim.x);
    sel_stamp(S.g_ctr, 1);                                  // every CTA has finished its rows: the stream ends here
    sel_load_hist(S.g_hist, s_hist, &s_misc[6]);
    __syncthreads();
    sel_find_bin(s_hist, static_cast<uint32_t>(S.b), reinterpret_cast<uint32_t*>(s_misc + 16), &s_misc[1], &s_misc[2]);
    const uint32_t T0 = static_cast<uint32_t>(s_misc[1]);
    // ---- level 1 ----
    sel_level1_hist(s_list, cnt, T0, s_hist);
    sel_push_hist(s_hist, S.g_hist + 2048);
    sel_grid_barrier(S.g_ctr, 2u * gridDim.x);
    sel_load_hist(S.g_hist + 2048, s_hist, nullptr);
    __syncthreads();
    {
        const uint32_t want = static_cast<uint32_t>(s_misc[2]);
        __syncthreads();
        sel_find_bin(s_hist, want, reinterpret_cast<uint32_t*>(s_misc + 16), &s_misc[5], &s_misc[2]);
    }
    if (tid == 0) s_misc[4] = 0;
    __syncthreads();
    const uint32_t T = (T0 << 11) | static_cast<uint32_t>(s_misc[5]);        // 22-bit prefix of the b-th smallest key
    unsigned int barriers = 2;
    // ---- bucket route: each candidate goes to the CTA of its score bucket, a CTA sorts ITS bucket (about b / grid
    //      words) and nobody ranks against the whole list (that stage was bound by ~1 shared-memory atomic per list word
    //      per CTA: 5.5 us).  Scores that do not spread and tie groups (one bucket beyond bucket_cap) fall through to the
    //      general route below; every CTA takes the same decision from the same counts. ----
    if (S.g_bucket) {
        const int G = static_cast<int>(gridDim.x);
        const SelBuckets bk(2047 - s_misc[6], T, G);
        if (bk.spread) {
            // kBucketLanes counters (and sub-lists) per bucket, CTA c appends to lane c % kBucketLanes: ~b appends onto `grid`
            // addresses is a chain of ~b / grid same-address atomics deep (measured 4 us); sixteen lanes cut it to a few
            constexpr int R = kBucketLanes;
            const int lane_id = static_cast<int>(blockIdx.x) % R, sub_cap = S.bucket_cap;
            if (tid < 3 + R) s_misc[48 + tid] = 0;          // [48] largest sub-list, [49] words in the buckets below mine, [51..] my sub-lists
            for (int i = tid; i < cnt; i += nthr) {
                const unsigned long long w = s_list[i];
                if (static_cast<uint32_t>(w >> 42) <= T) {
                    const int q = bk.of(w);
                    const unsigned int slot = atomicAdd(S.g_bcnt + q * R + lane_id, 1u);
                    if (slot < static_cast<unsigned int>(sub_cap))
                        S.g_bucket[(static_cast<size_t>(q) * R + lane_id) * sub_cap + slot] = w;
                }
            }
            sel_grid_barrier(S.g_ctr, ++barriers * gridDim.x);
            // my bucket's sub-lists are fetched together with the counters (one L2 round trip); what lies beyond a
            // sub-list's count is dropped once the counts are known
            const unsigned long long* src = S.g_bucket + static_cast<size_t>(blockIdx.x) * R * sub_cap;
            unsigned long long wv[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) wv[k] = (tid + k * nthr) < R * sub_cap ? __ldcg(src + tid + k * nthr) : 0ull;
            {
                int mx = 0, below = 0;
                for (int idx = tid; idx < G * R; idx += nthr) {
                    const int v = static_cast<int>(__ldcg(S.g_bcnt + idx)), q = idx / R;
                    mx = max(mx, v);
                    if (q < static_cast<int>(blockIdx.x)) below += v;
                    if (q == static_cast<int>(blockIdx.x)) s_misc[51 + idx % R] = v;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
                    below += __shfl_xor_sync(0xffffffffu, below, o);
                }
                if (lane == 0) { atomicMax(&s_misc[48], mx); atomicAdd(&s_misc[49], below); }
            }
            __syncthreads();
            if (s_misc[48] <= sub_cap && R * sub_cap <= 2 * nthr) {
                int mine = 0;
                for (int l = 0; l < R; ++l) mine += s_misc[51 + l];
#pragma unroll
                for (int k = 0; k < 2; ++k) {               // sub-list l -> buf[words of the sub-lists before it ...)
                    const int i = tid + k * nthr;
                    if (i < R * sub_cap) {
                        const int l = i / sub_cap, kk = i - l * sub_cap;
                        if (kk < s_misc[51 + l]) {
                            int at = kk;
                            for (int m2 = 0; m2 < l; ++m2) at += s_misc[51 + m2];
                            buf[at] = wv[k];
                        }
                    }
                }
                __syncthreads();
                sel_rank_bucket(buf, mine, s_misc[49], S.b, S.out_pos);
                sel_stamp(S.g_ctr, 2);
                return;
            }
            __syncthreads();
        }
    }
    // ---- general route: the candidates of every CTA are appended to g_cand ----
    int off;
    const int nc = sel_gather_candidates(S, s_list, cnt, T, buf, s_misc, off);
    for (int i = tid; i < nc; i += nthr) {
        const unsigned long long w = buf[i];
        s_list[i] = w;
        S.g_cand[off + i] = w;
    }
    sel_grid_barrier(S.g_ctr, ++barriers * gridDim.x);
    const int total = static_cast<int>(__ldcg(S.g_ctr + 1));
    // ---- rank this CTA's candidates among all of them.  Own candidates are sorted first (a few dozen words: counting);
    //      then every word of the global list is located in that sorted list by a binary search and bumps ONE entry of a
    //      difference array: x is smaller than exactly the own candidates from upper_bound(x) on.  O(total log nc) instead
    //      of the O(total * nc) of plain counting (measured: 22 us of shared-memory bandwidth).  The searches' probes
    //      fall into few banks and the ~b shared-memory atomics on the difference array dominate the stage: the reason
    //      for the bucket route above. ----
    unsigned long long* const tmp = buf + buf_cap;          // [list_cap] words behind the chunk buffer
    sel_stream_list(S.g_cand, total, buf, buf_cap, reinterpret_cast<uint64_t*>(s_misc + 8),
                    [&] {                                   // while the first chunk (b + a few words = 80 KB) lands: own
                        for (int i = tid; i < nc; i += nthr) {      // candidates sorted (rank by counting; the words are
                            const unsigned long long w = s_list[i]; // distinct: the row id is part of them)
                            int r = 0;
                            for (int q = 0; q < nc; ++q) r += s_list[q] < w;
                            tmp[r] = w;
                        }
                        __syncthreads();
                        for (int i = tid; i < nc; i += nthr) s_list[i] = tmp[i];
                        for (int i = tid; i <= nc; i += nthr) s_hist[i] = 0;    // difference array (nc + 1 <= 2049 entries: s_hist has 2064)
                    },
                    [&](int m) { sel_count_into_diff_sorted(buf, m, s_list, nc, s_hist); });
    sel_write_ranks(s_hist, s_list, nc, S.b, S.out_pos);
    sel_stamp(S.g_ctr, 2);
}

// Bounded spin.  The sticky failure flag that lets every other wait of this launch return at once lives in DEVICE
// memory (g_ctr[12]); the host-visible status word is mapped host memory and is only WRITTEN, once, on a timeout --
// polling it from thousands of spinning threads is a PCIe read storm that delays the very launches being waited for
// (measured at 8 GPUs: once one rank was 30 us late every step took 1-6 ms).
__device__ __forceinline__ unsigned int sel_ll_wait(const void* p, unsigned int tag, const SelArgs& S) {
    unsigned long long v;
    const long long t0 = clock64();
    for (int spin = 0;; ++spin) {
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
        if (static_cast<unsigned int>(v >> 32) == tag) break;
        if ((spin & 255) == 255) {
            if (*reinterpret_cast<volatile unsigned int*>(S.g_ctr + 12) != 0) break;
            if (clock64() - t0 > S.timeout_cycles) {
                if (atomicExch(S.g_ctr + 12, 1u) == 0u) {
                    *reinterpret_cast<volatile int*>(S.status) = ALQ_ERR_STATE;
                    __threadfence_system();
                }
                break;
            }
        }
    }
    return static_cast<unsigned int>(v);
}

// The same selection with the rows sharded over `world` GPUs: K1 + K1b + the exchange in ONE launch per rank.  Both
// histogram levels are summed over the ranks (every CTA publishes a slice of its rank's bins to every window as LL
// words and sums the same slice of all ranks), so every rank finds the same 22-bit threshold; the candidates (b + a few
// words over ALL ranks, not b per rank) are stored into every window, each CTA's count follows behind a system fence
// as an LL word; then every rank ranks the whole list (CTA c takes slice c) -- all ranks end with the same out_pos.
// With one rank the window is this GPU's own memory and the same stores, waits, fences and tags run.
__device__ __noinline__ void select_epilogue_mgpu(const SelArgs& S, uint32_t* s_hist, unsigned long long* s_list, int* s_misc,
                                                  unsigned long long* buf, int buf_cap) {
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
    const int grid = gridDim.x, W = S.world;
    char* const win = S.peer[S.rank];
    uint64_t* const bar = reinterpret_cast<uint64_t*>(s_misc + 8);
    __syncthreads();
    const int cnt = s_misc[0];
    uint32_t want = static_cast<uint32_t>(S.b), T0 = 0;
    const int per = (2048 + grid - 1) / grid, b_lo = min(2048, static_cast<int>(blockIdx.x) * per), b_hi = min(2048, b_lo + per);
    for (int level = 0; level < 2; ++level) {
        if (level == 1) sel_level1_hist(s_list, cnt, T0, s_hist);
        sel_push_hist(s_hist, S.g_hist + level * 2048);
        sel_grid_barrier(S.g_ctr, static_cast<unsigned int>(2 * level + 1) * grid);
        if (level == 0) sel_stamp(S.g_ctr, 1);
        // this CTA's slice of the rank histogram -> every rank; then the same slice summed over the ranks
        for (int i = tid; i < (b_hi - b_lo) * W; i += nthr) {
            const int bin = b_lo + i / W, p = i % W;
            ll_store(S.peer[p] + S.hist_off + (static_cast<size_t>(level * W + S.rank) * 2048 + bin) * 8, S.tag,
                     __ldcg(S.g_hist + level * 2048 + bin));
        }
        uint32_t* s_sum = reinterpret_cast<uint32_t*>(s_misc + 16);           // [per <= 32] (find_bin's scratch, free here)
        if (tid < 32) s_sum[tid] = 0;
        __syncthreads();
        for (int i = tid; i < (b_hi - b_lo) * W; i += nthr) {                 // one word per thread: the waits overlap
            const int k = i / W, r = i % W;
            const uint32_t v = sel_ll_wait(win + S.hist_off + (static_cast<size_t>(level * W + r) * 2048 + b_lo + k) * 8, S.tag, S);
            if (v) atomicAdd(&s_sum[k], v);
        }
        __syncthreads();
        for (int i = tid; i < (b_hi - b_lo); i += nthr) S.g_tot[level * 2048 + b_lo + i] = s_sum[i];
        sel_grid_barrier(S.g_ctr, static_cast<unsigned int>(2 * level + 2) * grid);
        sel_load_hist(S.g_tot + level * 2048, s_hist, level == 0 ? &s_misc[6] : nullptr);     // first populated bin: all ranks
        __syncthreads();
        sel_find_bin(s_hist, want, reinterpret_cast<uint32_t*>(s_misc + 16), &s_misc[level == 0 ? 1 : 5], &s_misc[2]);
        want = static_cast<uint32_t>(s_misc[2]);
        if (level == 0) T0 = static_cast<uint32_t>(s_misc[1]);
        __syncthreads();
    }
    const uint32_t T = (T0 << 11) | static_cast<uint32_t>(s_misc[5]);
    if (tid == 0) s_misc[4] = 0;
    __syncthreads();
    // ---- this CTA's candidates -> the rank's region of every window; the count follows behind a system fence ----
    int off;
    const int nc = sel_gather_candidates(S, s_list, cnt, T, buf, s_misc, off);
    if (off + nc > S.cand_cap && tid == 0) { *reinterpret_cast<volatile int*>(S.status) = ALQ_ERR_STATE; __threadfence_system(); }
    for (int i = tid; i < nc * W; i += nthr) {
        const int k = i / W, p = i % W;
        if (off + k < S.cand_cap)
            reinterpret_cast<unsigned long long*>(S.peer[p] + S.cand_off)[static_cast<size_t>(S.rank) * S.cand_cap + off + k] = buf[k];
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence_system();               // the candidate words are visible in every window before the count is
        for (int p = 0; p < W; ++p)
            ll_store(S.peer[p] + S.cnt_off + (static_cast<size_t>(S.rank) * S.stride + blockIdx.x) * 8, S.tag, static_cast<unsigned int>(nc));
    }
    // ---- counts of every CTA of every rank -> per-rank totals ----
    uint32_t* s_tot = reinterpret_cast<uint32_t*>(s_misc + 24);      // [8]
    if (tid < ALQ_MAX_WORLD) s_tot[tid] = 0;
    __syncthreads();
    for (int i = tid; i < W * S.stride; i += nthr) {
        const int r = i / S.stride;
        const uint32_t v = sel_ll_wait(win + S.cnt_off + static_cast<size_t>(i) * 8, S.tag, S);
        if (v) atomicAdd(&s_tot[r], v);
    }
    __syncthreads();
    // ---- the list = the rank segments one after the other (each padded to an even word count with a ~0 word that sorts
    //      behind everything).  CTA c ranks slice c of it against all of it. ----
    int seg_off[ALQ_MAX_WORLD + 1];
    seg_off[0] = 0;
    bool overflow = false;
    for (int r = 0; r < W; ++r) {
        overflow = overflow || s_tot[r] > static_cast<uint32_t>(S.cand_cap);
        seg_off[r + 1] = seg_off[r] + static_cast<int>((min(s_tot[r], static_cast<uint32_t>(S.cand_cap)) + 1u) & ~1u);
    }
    const int M = seg_off[W];
    const int perc = (M + grid - 1) / grid, s0 = min(M, static_cast<int>(blockIdx.x) * perc), n2 = min(M, s0 + perc) - s0;
    if (overflow || n2 > S.list_cap) {        // a tie group larger than the windows were sized for: every rank sees the same
        if (tid == 0) { *reinterpret_cast<volatile int*>(S.status) = ALQ_ERR_STATE; __threadfence_system(); }   // counts and gives up
        return;
    }
    const unsigned long long* cand = reinterpret_cast<const unsigned long long*>(win + S.cand_off);
    // ---- bucket route (see select_epilogue): the list is complete in this rank's window, so CTA c scans it once, keeps
    //      the words of score bucket c (about b / grid of them: the only shared-memory atomics of the stage) and counts
    //      the words of the buckets below; it then orders its bucket alone.  One more grid barrier tells every CTA
    //      whether all buckets fitted; if one did not (tie groups), the general ranking below runs instead. ----
    {
        const SelBuckets bk(2047 - s_misc[6], T, grid);
        if (bk.spread && S.bucket_cap > 0) {
            if (tid == 0) { s_misc[48] = 0; s_misc[49] = 0; s_misc[50] = 0; }
            int below = 0;
            const int me = static_cast<int>(blockIdx.x);
            for (int r = 0; r < W; ++r)
                sel_stream_list(cand + static_cast<size_t>(r) * S.cand_cap, static_cast<int>(s_tot[r]), buf, buf_cap, bar, [] {},
                                [&](int m) {
                                    for (int j = tid; j < m; j += nthr) {
                                        const unsigned long long x = buf[j];
                                        const int q = bk.of(x);
                                        if (q < me) ++below;
                                        else if (q == me) {
                                            const int slot = atomicAdd(&s_misc[48], 1);
                                            if (slot < S.list_cap) s_list[slot] = x;
                                        }
                                    }
                                });
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) below += __shfl_xor_sync(0xffffffffu, below, o);
            if (lane == 0 && below) atomicAdd(&s_misc[49], below);
            __syncthreads();
            if (tid == 0) S.g_hist[me] = static_cast<unsigned int>(s_misc[48]);          // the rank's level-0 bins are no longer read
            sel_grid_barrier(S.g_ctr, 5u * grid);
            {
                int mx = 0;
                for (int q = tid; q < grid; q += nthr) mx = max(mx, static_cast<int>(__ldcg(S.g_hist + q)));
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
                if (lane == 0 && mx) atomicMax(&s_misc[50], mx);
            }
            __syncthreads();
            if (s_misc[50] <= S.list_cap) {
                sel_rank_bucket(s_list, s_misc[48], s_misc[49], S.b, S.out_pos);
                sel_stamp(S.g_ctr, 2);
                return;
            }
            __syncthreads();
        }
    }
    auto list_word = [&](int j) -> unsigned long long {     // word j of the padded list, from this rank's window
        int r = 0;
        while (r + 1 < W && j >= seg_off[r + 1]) ++r;
        const int k = j - seg_off[r];
        return k < static_cast<int>(s_tot[r]) ? __ldcg(cand + static_cast<size_t>(r) * S.cand_cap + k) : ~0ull;
    };
    {
        unsigned long long* tmp = buf + buf_cap;            // [list_cap] words behind the chunk buffer
        for (int i = tid; i < n2; i += nthr) tmp[i] = list_word(s0 + i);
        __syncthreads();
        for (int i = tid; i < n2; i += nthr) {              // own slice sorted (rank by counting; equal pad words keep
            const unsigned long long w = tmp[i];            // distinct slots)
            int r = 0;
            for (int q = 0; q < n2; ++q) {
                const unsigned long long x = tmp[q];
                r += (x < w) || (x == w && q < i);
            }
            s_list[r] = w;
        }
    }
    __syncthreads();
    for (int i = tid; i <= n2; i += nthr) s_hist[i] = 0;
    for (int r = 0; r < W; ++r)                             // the rank segments one after the other
        sel_stream_list(cand + static_cast<size_t>(r) * S.cand_cap, static_cast<int>(s_tot[r]), buf, buf_cap, bar, [] {},
                        [&](int m) { sel_count_into_diff_sorted(buf, m, s_list, n2, s_hist); });
    sel_write_ranks(s_hist, s_list, n2, S.b, S.out_pos);
    sel_stamp(S.g_ctr, 2);
}

// MODE 0..2: scores; MODE 3: BADGE factors (writes a[row, :] and a_norm2[row]);
// MODE 4: MASE minimum margin + predicted class (K6, table reads pruned); MODE 5: MASE with the per-class radii written
constexpr int MODE_MASE_MIN = 4, MODE_MASE_FULL = 5;
template <int NV, int MODE>
__global__ void __launch_bounds__(1024, 1)
rows_pipe_kernel(const float* __restrict__ logits, int64_t n, int c, RowPipeCfg cfg, float* __restrict__ scores,
                 int bs, int64_t grow0, int64_t n_total, float* __restrict__ a, int64_t lda,
                 unsigned int* __restrict__ tile_counter, MaseArgs mase, const __grid_constant__ SelArgs sel) {
    extern __shared__ __align__(128) unsigned char smem_rows[];
    float* tiles = reinterpret_cast<float*>(smem_rows);
    uint64_t* full = reinterpret_cast<uint64_t*>(tiles + static_cast<size_t>(cfg.stages) * cfg.tile_floats);
    uint64_t* empty = full + cfg.stages;
    int* s_tile = reinterpret_cast<int*>(empty + cfg.stages);          // tile index carried by each stage (-1: done)
    // fused selection (sel.b > 0): level-0 histogram, this CTA's (key, row) words, a few counters
    unsigned long long* s_list = reinterpret_cast<unsigned long long*>(smem_rows + sel.list_off);
    uint32_t* s_hist = reinterpret_cast<uint32_t*>(s_list + sel.list_cap);
    int* s_misc = reinterpret_cast<int*>(s_hist + 2064);
    if (sel.b > 0) {
        for (int i = threadIdx.x; i < 2048; i += blockDim.x) s_hist[i] = 0;
        if (threadIdx.x < 48) s_misc[threadIdx.x] = 0;
        sel_stamp(sel.g_ctr, 0);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int R = cfg.rows_per_tile;
    // Tiles are claimed dynamically (runs of kClaim consecutive tiles per atomicAdd): a CTA that starts late --
    // e.g. because another stream's small kernel still holds its SM -- simply claims fewer tiles, so this
    // kernel can overlap with the top-B kernel of the previous query without a straggler tail.
    constexpr int kClaim = 8;
    const int tiles_total = static_cast<int>((n + R - 1) / R);
    const int teams = cfg.consumers / cfg.split;
    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], cfg.split); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int nvec = c >> 2;
    if (warp == 0) {
        if (lane == 0) {
            int claim_lo = 0, claim_hi = 0, sentinels = 0, claimed = 0;
            bool exhausted = false;
            for (int i = 0;; ++i) {
                const int s = i % cfg.stages;
                const uint32_t round = static_cast<uint32_t>(i / cfg.stages);
                if (round > 0) mbar_wait(&empty[s], (round - 1) & 1u);
                if (claim_lo == claim_hi && !exhausted && sel.b > 0 && (claimed + kClaim) * R > sel.list_cap) exhausted = true;
                if (claim_lo == claim_hi && !exhausted) {
                    claimed += kClaim;
                    const unsigned int got = atomicAdd(tile_counter, static_cast<unsigned int>(kClaim));
                    if (got >= static_cast<unsigned int>(tiles_total)) exhausted = true;
                    else { claim_lo = static_cast<int>(got); claim_hi = min(tiles_total, claim_lo + kClaim); }
                }
                if (claim_lo < claim_hi) {
                    const int tile = claim_lo++;
                    const int64_t row0 = static_cast<int64_t>(tile) * R;
                    const int rr = static_cast<int>(min(static_cast<int64_t>(R), n - row0));
                    const uint32_t bytes = static_cast<uint32_t>(rr) * static_cast<uint32_t>(c) * 4u;
                    s_tile[s] = tile;
                    mbar_expect_tx(&full[s], bytes);
                    bulk_g2s(tiles + static_cast<size_t>(s) * cfg.tile_floats, logits + row0 * c, bytes, &full[s]);
                } else {
                    s_tile[s] = -1;                       // one sentinel per consumer team, then stop
                    mbar_arrive(&full[s]);
                    if (++sentinels == teams) break;
                }
            }
        }
    } else {
        const int cw = warp - 1;
        const int team = cw / cfg.split, sub = cw % cfg.split;
        const float mase_ratio = (MODE == MODE_MASE_MIN) ? __ldg(mase.gmin + c) : 0.f;
        for (int i = team;; i += teams) {
            const int s = i % cfg.stages;
            mbar_wait(&full[s], static_cast<uint32_t>(i / cfg.stages) & 1u);
            const int tile_idx = s_tile[s];
            if (tile_idx < 0) break;
            const int64_t row0 = static_cast<int64_t>(tile_idx) * R;
            const int rr = static_cast<int>(min(static_cast<int64_t>(R), n - row0));
            const float* tile = tiles + static_cast<size_t>(s) * cfg.tile_floats;
            float my_score = 0.f;
            int my_pred = 0;
            for (int r = sub; r < rr; r += cfg.split) {
                if (MODE >= MODE_MASE_MIN) {
                    const MaseRowSmem srow{reinterpret_cast<const float4*>(tile + static_cast<size_t>(r) * c), nvec};
                    float mn;
                    int arg;
                    if (MODE == MODE_MASE_MIN) mase_row_min_smem<NV>(srow.p, nvec, lane, mase.ginv, mase.ldg, mase.gmin, mase_ratio, mn, arg);
                    else mase_row_full<NV, true>(srow, lane, nvec, mase.ginv, mase.ldg,
                                                 reinterpret_cast<float4*>(mase.radius + (row0 + r) * mase.ldr), mn, arg);
                    if (lane == r) { my_score = mn; my_pred = arg; }
                    continue;
                }
                float4 v[NV];
                load_row_smem<NV>(reinterpret_cast<const float4*>(tile + static_cast<size_t>(r) * c), lane, nvec, v);
                if (MODE < 3) {
                    const RowStats st = row_stats_vec<NV, MODE == ALQ_MODE_MARGIN, false, MODE == ALQ_MODE_ENTROPY>(v, lane, nvec);
                    if (lane == r) my_score = score_from_stats(st, MODE);
                } else {
                    const RowStats st = row_stats_vec<NV, false, true, false>(v, lane, nvec);
                    const int64_t row = row0 + r;
                    const float inv_bs = batch_scale(grow0 + row, n_total, bs);
                    const float inv_s = 1.0f / st.s;          // one division per row; p = e * (1/s) is within 1 ulp of e / s
                    float4* q = reinterpret_cast<float4*>(a + row * lda);
                    float nn = 0.f;
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                        const int idx = lane + 32 * k;
                        if (idx < nvec) {
                            float e[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const float pj = exp_neg(e[j] - st.m) * inv_s;
                                const float g = (pj - ((idx * 4 + j) == st.arg ? 1.0f : 0.0f)) * inv_bs;
                                e[j] = g;
                                nn += g * g;
                            }
                            q[idx] = make_float4(e[0], e[1], e[2], e[3]);
                        }
                    }
                    nn = warp_sum(nn);
                    if (lane == r) my_score = nn;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);       // this warp's smem reads of the stage are done
            if (lane < rr && (lane % cfg.split) == sub) {
                scores[row0 + lane] = my_score;
                if (MODE >= MODE_MASE_MIN) mase.pred[row0 + lane] = my_pred;
                if (sel.b > 0) {
                    const uint32_t key = alq_ord(my_score + 0.0f);
                    s_list[atomicAdd(&s_misc[0], 1)] = (static_cast<unsigned long long>(key) << 32) | (sel.row_base + static_cast<uint32_t>(row0 + lane));
                    atomicAdd(&s_hist[key >> 21], 1u);
                }
            }
        }
    }
    if (sel.b > 0) {     // every thread of the CTA (the tile ring is free now: it becomes the candidate buffer)
        // Every warp has left the stream, so every bulk copy into the ring has completed and been waited on: the ring's
        // full[] / empty[] barriers are invalidated before the epilogue reuses their words as plain memory (it starts
        // with a barrier).
        __syncthreads();
        if (threadIdx.x == 0) {                          // full[] and empty[] (SelArgs: nothing stays live across the loop)
            uint64_t* ring = reinterpret_cast<uint64_t*>(smem_rows + sel.ring_off);
            for (int s = 0; s < sel.ring_bars; ++s) mbar_inval(&ring[s]);
        }
        if (sel.world > 0) select_epilogue_mgpu(sel, s_hist, s_list, s_misc, reinterpret_cast<unsigned long long*>(tiles),
                                                sel.list_off / 8 - sel.list_cap - 2);
        else select_epilogue(sel, s_hist, s_list, s_misc, reinterpret_cast<unsigned long long*>(tiles),
                             sel.list_off / 8 - sel.list_cap - 2);
    }
}

// Any c / alignment: two passes over the row, the second one hits L1/L2.
__global__ void __launch_bounds__(kScoreThreads)
score_rows_generic_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, int mode,
                          float* __restrict__ scores) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t row = warp; row < n; row += nwarps) {
        const float* p = logits + row * ld;
        float t1 = ALQ_NEG_INF, t2 = ALQ_NEG_INF;
        for (int j = lane; j < c; j += 32) top2_push(p[j], t1, t2);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float o1 = __shfl_xor_sync(0xffffffffu, t1, o);
            const float o2 = __shfl_xor_sync(0xffffffffu, t2, o);
            const float hi = fmaxf(t1, o1);
            t2 = fmaxf(fminf(t1, o1), fmaxf(t2, o2));
            t1 = hi;
        }
        float s = 0.f, w = 0.f;
        for (int j = lane; j < c; j += 32) {
            const float dz = p[j] - t1;
            const float ex = exp_neg(dz);
            s += ex;
            w = ex > 0.f ? fmaf(ex, dz, w) : w;   // 0 log 0 = 0 for masked (-inf) classes
        }
        s = warp_sum(s);
        w = warp_sum(w);
        if (lane == 0) scores[row] = score_from_stats(RowStats{t1, t2, s, w, 0}, mode);
    }
}

// ---------------------------------------------------------------------------------------------
// K2: a = (softmax - onehot(argmax)) * (1 / bs_i)
// ---------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(kScoreThreads)
badge_factors_vec_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, int bs, int64_t row0,
                         int64_t n_total, float* __restrict__ a, int64_t lda, float* __restrict__ a_norm2) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int nvec = c >> 2;
    for (int64_t row = warp; row < n; row += nwarps) {
        const float4* p = reinterpret_cast<const float4*>(logits + row * ld);
        float4 v[NV];
        load_row_vec<NV>(p, lane, nvec, v);
        const RowStats r = row_stats_vec<NV, false, true, false>(v, lane, nvec);
        const float inv_bs = batch_scale(row0 + row, n_total, bs);
        const float inv_s = 1.0f / r.s;
        float4* q = reinterpret_cast<float4*>(a + row * lda);
        float nn = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int idx = lane + 32 * k;
            if (idx < nvec) {
                float e[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float pj = exp_neg(e[j] - r.m) * inv_s;
                    const float g = (pj - ((idx * 4 + j) == r.arg ? 1.0f : 0.0f)) * inv_bs;
                    e[j] = g;
                    nn += g * g;
                }
                q[idx] = make_float4(e[0], e[1], e[2], e[3]);
            }
        }
        nn = warp_sum(nn);
        if (lane == 0) a_norm2[row] = nn;
    }
}

__global__ void __launch_bounds__(kScoreThreads)
badge_factors_generic_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, int bs, int64_t row0,
                             int64_t n_total, float* __restrict__ a, int64_t lda, int cpad,
                             float* __restrict__ a_norm2) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t row = warp; row < n; row += nwarps) {
        const float* p = logits + row * ld;
        float m = ALQ_NEG_INF;
        int arg = 0x7fffffff;
        for (int j = lane; j < c; j += 32) {
            const float z = p[j];
            if (z > m) { m = z; arg = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, m, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (om > m || (om == m && oa < arg)) { m = om; arg = oa; }
        }
        float s = 0.f;
        for (int j = lane; j < c; j += 32) s += exp_neg(p[j] - m);
        s = warp_sum(s);
        const float inv_bs = batch_scale(row0 + row, n_total, bs);
        float nn = 0.f;
        for (int j = lane; j < cpad; j += 32) {
            float g = 0.f;
            if (j < c) g = (exp_neg(p[j] - m) / s - (j == arg ? 1.0f : 0.0f)) * inv_bs;
            a[row * lda + j] = g;
            nn += g * g;
        }
        nn = warp_sum(nn);
        if (lane == 0) a_norm2[row] = nn;
    }
}

// ---------------------------------------------------------------------------------------------
// K2p: pooled gradient embedding out[i, r*pw + s] = mean_{bin r}(a_i) * mean_{bin s}(h_i)
// (adaptive_avg_pool2d of a rank-1 matrix is the outer product of the 1-D pools).
// ---------------------------------------------------------------------------------------------
constexpr int kPoolWarps = 4;

__global__ void __launch_bounds__(kPoolWarps * 32)
badge_pooled_kernel(const float* __restrict__ logits, int64_t n, int c, int64_t ld, int bs,
                    const float* __restrict__ emb, int d, int64_t lde, int ph, int pw,
                    float* __restrict__ out, int64_t ldo) {
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    float* sa = smem + static_cast<size_t>(wib) * (c + ph + pw);
    float* spa = sa + c;
    float* sph = spa + ph;
    const int64_t warp = static_cast<int64_t>(blockIdx.x) * kPoolWarps + wib;
    const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kPoolWarps;
    for (int64_t row = warp; row < n; row += nwarps) {
        const float* p = logits + row * ld;
        float m = ALQ_NEG_INF;
        int arg = 0x7fffffff;
        for (int j = lane; j < c; j += 32) {
            const float z = p[j];
            if (z > m) { m = z; arg = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, m, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (om > m || (om == m && oa < arg)) { m = om; arg = oa; }
        }
        float s = 0.f;
        for (int j = lane; j < c; j += 32) s += exp_neg(p[j] - m);
        s = warp_sum(s);
        const float inv_bs = batch_scale(row, n, bs);
        for (int j = lane; j < c; j += 32)
            sa[j] = (exp_neg(p[j] - m) / s - (j == arg ? 1.0f : 0.0f)) * inv_bs;
        __syncwarp();
        for (int r = lane; r < ph; r += 32) {
            const int lo = static_cast<int>((static_cast<int64_t>(r) * c) / ph);
            const int hi = static_cast<int>((static_cast<int64_t>(r + 1) * c + ph - 1) / ph);
            float acc = 0.f;
            for (int j = lo; j < hi; ++j) acc += sa[j];
            spa[r] = acc / static_cast<float>(hi - lo);
        }
        const float* h = emb + row * lde;
        for (int q = lane; q < pw; q += 32) {
            const int lo = static_cast<int>((static_cast<int64_t>(q) * d) / pw);
            const int hi = static_cast<int>((static_cast<int64_t>(q + 1) * d + pw - 1) / pw);
            float acc = 0.f;
            for (int j = lo; j < hi; ++j) acc += h[j];
            sph[q] = acc / static_cast<float>(hi - lo);
        }
        __syncwarp();
        float* o = out + row * ldo;
        for (int k = lane; k < ph * pw; k += 32) o[k] = spa[k / pw] * sph[k % pw];
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// row norms
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kScoreThreads)
row_norm2_kernel(const float* __restrict__ x, int64_t n, int d, int64_t ld, int vec,
                 float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    for (int64_t row = warp; row < n; row += nwarps) {
        float acc = 0.f;
        if (vec) {
            const float4* p = reinterpret_cast<const float4*>(x + row * ld);
            for (int k = lane; k < (d >> 2); k += 32) {
                const float4 v = ld_stream_f4(p + k);
                acc += v.x * v.x;
                acc += v.y * v.y;
                acc += v.z * v.z;
                acc += v.w * v.w;
            }
        } else {
            const float* p = x + row * ld;
            for (int k = lane; k < d; k += 32) acc += p[k] * p[k];
        }
        acc = warp_sum(acc);
        if (lane == 0) out[row] = acc;
    }
}

int rows_grid(const alq_ctx* ctx, int64_t n, int warps_per_block) {
    int64_t need = (n + warps_per_block - 1) / warps_per_block;
    int64_t cap = static_cast<int64_t>(ctx->sm_count) * 8;
    if (need < 1) need = 1;
    return static_cast<int>(need < cap ? need : cap);
}

// shared-memory plan of the pipelined kernels; false if the row does not fit
bool plan_row_pipe(const alq_ctx* ctx, int c, RowPipeCfg& cfg, size_t& smem, size_t reserve = 0) {
    const size_t row_bytes = static_cast<size_t>(c) * 4;
    if (row_bytes % 16 || row_bytes > 16384 || ctx->smem_optin < 64 * 1024) return false;
    size_t tile_target = 16384;
    if (const char* e = getenv("ALQ_ROW_TILE_KB")) tile_target = static_cast<size_t>(std::max(1, atoi(e))) * 1024;   // tuning aid
    int R = static_cast<int>(std::max<size_t>(1, tile_target / row_bytes));
    R = std::min(R, 32);
    const size_t tile = R * row_bytes;
    int stages = static_cast<int>((ctx->smem_optin - 4096 - reserve) / tile);
    stages = std::min(stages, 16);
    if (stages < 3) return false;
    int split = 2;
    if (const char* e = getenv("ALQ_ROW_SPLIT")) split = std::max(1, std::min(4, atoi(e)));                       // tuning aid
    while (split > 1 && (stages * split > 31 || split > R)) --split;
    cfg.rows_per_tile = R; cfg.stages = stages; cfg.consumers = stages * split; cfg.split = split;
    cfg.tile_floats = static_cast<int>(tile / 4);
    smem = stages * tile + 2 * stages * sizeof(uint64_t) + (stages + 1) * sizeof(int) + 128 + reserve;
    return true;
}

// a zeroed tile counter for one launch: slots of a ring that is cleared once and again whenever it wraps
unsigned int* next_tile_counter(alq_ctx* ctx, cudaStream_t st) {
    constexpr int kSlots = 16384;
    if (!ctx->tile_counters) {
        if (cudaMalloc(&ctx->tile_counters, kSlots * sizeof(unsigned int)) != cudaSuccess) return nullptr;
        cudaMemset(ctx->tile_counters, 0, kSlots * sizeof(unsigned int));
        ctx->tile_counter_next = 0;
    }
    if (ctx->tile_counter_next == kSlots) {
        cudaMemsetAsync(ctx->tile_counters, 0, kSlots * sizeof(unsigned int), st);   // stream-ordered after its last users
        ctx->tile_counter_next = 0;
    }
    return ctx->tile_counters + ctx->tile_counter_next++;
}

template <int NV, int MODE>
cudaError_t launch_rows_pipe(alq_ctx* ctx, cudaStream_t st, const RowPipeCfg& cfg, size_t smem, const float* logits,
                             int64_t n, int c, float* scores, int bs, int64_t row0, int64_t n_total, float* a, int64_t lda,
                             const MaseArgs& mase = MaseArgs{}, const SelArgs& sel = SelArgs{}) {
    cudaError_t e = cudaFuncSetAttribute(rows_pipe_kernel<NV, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    const int64_t tiles_total = (n + cfg.rows_per_tile - 1) / cfg.rows_per_tile;
    const int grid = static_cast<int>(std::min<int64_t>(ctx->sm_count, tiles_total));
    unsigned int* counter = next_tile_counter(ctx, st);
    if (!counter) return cudaErrorMemoryAllocation;
    if (sel.b > 0) {
        // The fused selection synchronises the grid (and, sharded, the GPUs), so all of its CTAs must become resident: one CTA
        // per SM by construction (grid <= SM count, > 113 KB of shared memory each).  A cooperative launch would guarantee that,
        // but cooperative launches are not pipelined by the driver -- every step then waits for a host round trip, and with
        // one process per GPU a descheduled host thread stalls all ranks for milliseconds (measured at 8 GPUs: steps of
        // 1-5 ms instead of 0.1).  Ordinary launches are safe as long as no two grid-synchronising kernels of this process
        // share the device at the same time: they are chained through one event per device (other kernels merely delay the
        // moment the last CTA becomes resident; they never wait for ours).
        if (grid > ctx->sm_count) return cudaErrorInvalidConfiguration;
        return alq_gridsync_launch(ctx, st, [&] {
            rows_pipe_kernel<NV, MODE><<<grid, 32 * (1 + cfg.consumers), smem, st>>>(logits, n, c, cfg, scores, bs, row0, n_total,
                                                                                  a, lda, counter, mase, sel);
            return cudaGetLastError();
        });
    }
    rows_pipe_kernel<NV, MODE><<<grid, 32 * (1 + cfg.consumers), smem, st>>>(logits, n, c, cfg, scores, bs, row0, n_total, a, lda,
                                                                          counter, mase, sel);
    return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_rows_pipe_nv(alq_ctx* ctx, cudaStream_t st, const RowPipeCfg& cfg, size_t smem, const float* logits,
                                int64_t n, int c, float* scores, int bs, int64_t row0, int64_t n_total, float* a, int64_t lda,
                                const MaseArgs& mase = MaseArgs{}, const SelArgs& sel = SelArgs{}) {
    const int nv = (c / 4 + 31) / 32;
    if (nv <= 1) return launch_rows_pipe<1, MODE>(ctx, st, cfg, smem, logits, n, c, scores, bs, row0, n_total, a, lda, mase, sel);
    if (nv <= 2) return launch_rows_pipe<2, MODE>(ctx, st, cfg, smem, logits, n, c, scores, bs, row0, n_total, a, lda, mase, sel);
    if (nv <= 4) return launch_rows_pipe<4, MODE>(ctx, st, cfg, smem, logits, n, c, scores, bs, row0, n_total, a, lda, mase, sel);
    if (nv <= 8) return launch_rows_pipe<8, MODE>(ctx, st, cfg, smem, logits, n, c, scores, bs, row0, n_total, a, lda, mase, sel);
    return launch_rows_pipe<16, MODE>(ctx, st, cfg, smem, logits, n, c, scores, bs, row0, n_total, a, lda, mase, sel);
}

template <int NV>
void launch_score_vec(int mode, int grid, cudaStream_t st, const float* logits, int64_t n, int c,
                      int64_t ld, float* scores) {
    if (mode == ALQ_MODE_MARGIN)
        score_rows_vec_kernel<NV, ALQ_MODE_MARGIN><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, scores);
    else if (mode == ALQ_MODE_LEAST_CONFIDENCE)
        score_rows_vec_kernel<NV, ALQ_MODE_LEAST_CONFIDENCE><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, scores);
    else
        score_rows_vec_kernel<NV, ALQ_MODE_ENTROPY><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, scores);
}

}  // namespace

// K6 through the same pipeline (declared in alq_mase_rows.cuh, called from alq_mase.cu)
bool alq_mase_rows_pipe(alq_ctx* ctx, cudaStream_t st, const float* logits, int64_t n, int c, const MaseArgs& m,
                        float* min_margin, cudaError_t* err) {
    RowPipeCfg cfg{};
    size_t smem = 0;
    if (c > 2048 || !plan_row_pipe(ctx, c, cfg, smem)) return false;
    *err = m.radius ? launch_rows_pipe_nv<MODE_MASE_FULL>(ctx, st, cfg, smem, logits, n, c, min_margin, 1, 0, n, nullptr, 0, m)
                    : launch_rows_pipe_nv<MODE_MASE_MIN>(ctx, st, cfg, smem, logits, n, c, min_margin, 1, 0, n, nullptr, 0, m);
    return true;
}

extern "C" int alq_score_softmax(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld,
                                 int32_t mode, float* scores, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || c <= 0 || ld < c || mode < 0 || mode > 2)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_score_softmax: bad shape n=%lld c=%d ld=%lld mode=%d",
                 (long long)n, c, (long long)ld, mode);
    if (n == 0) return ALQ_OK;
    if (!logits || !scores) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_score_softmax: null pointer");
    if (n >= (1LL << 31)) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_score_softmax: n must be < 2^31");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = rows_grid(ctx, n, kScoreThreads / 32);
    const bool vec = (c % 4 == 0) && (ld % 4 == 0) && aligned16(logits) && c <= 2048;
    RowPipeCfg cfg{};
    size_t smem = 0;
    if (vec && ld == c && n >= 4096 && plan_row_pipe(ctx, c, cfg, smem)) {
        cudaError_t e;
        if (mode == ALQ_MODE_MARGIN) e = launch_rows_pipe_nv<ALQ_MODE_MARGIN>(ctx, st, cfg, smem, logits, n, c, scores, 1, 0, n, nullptr, 0);
        else if (mode == ALQ_MODE_LEAST_CONFIDENCE) e = launch_rows_pipe_nv<ALQ_MODE_LEAST_CONFIDENCE>(ctx, st, cfg, smem, logits, n, c, scores, 1, 0, n, nullptr, 0);
        else e = launch_rows_pipe_nv<ALQ_MODE_ENTROPY>(ctx, st, cfg, smem, logits, n, c, scores, 1, 0, n, nullptr, 0);
        ctx->launches++;
        if (e != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "rows_pipe_kernel launch failed: %s", cudaGetErrorString(e));
        return ALQ_OK;
    }
    if (vec) {
        const int nv = (c / 4 + 31) / 32;
        if (nv <= 1) launch_score_vec<1>(mode, grid, st, logits, n, c, ld, scores);
        else if (nv <= 2) launch_score_vec<2>(mode, grid, st, logits, n, c, ld, scores);
        else if (nv <= 4) launch_score_vec<4>(mode, grid, st, logits, n, c, ld, scores);
        else if (nv <= 8) launch_score_vec<8>(mode, grid, st, logits, n, c, ld, scores);
        else launch_score_vec<16>(mode, grid, st, logits, n, c, ld, scores);
    } else {
        score_rows_generic_kernel<<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, mode, scores);
    }
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

// zeroed scratch of one fused launch (2048-bin histogram + counters): slots of a ring cleared in bulk
static unsigned int* next_sel_slot(alq_ctx* ctx, cudaStream_t st) {
    constexpr int kSlots = 64, kWords = 4 * 2048 + 16;      // 2 level histograms, their cross-rank sums, counters
    if (!ctx->sel_ring) {
        if (cudaMalloc(&ctx->sel_ring, static_cast<size_t>(kSlots) * kWords * 4) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        cudaMemset(ctx->sel_ring, 0, static_cast<size_t>(kSlots) * kWords * 4);
        ctx->sel_ring_next = 0;
    }
    if (ctx->sel_ring_next == kSlots) {
        cudaMemsetAsync(ctx->sel_ring, 0, static_cast<size_t>(kSlots) * kWords * 4, st);   // stream-ordered after its last users
        ctx->sel_ring_next = 0;
    }
    return ctx->sel_ring + static_cast<size_t>(ctx->sel_ring_next++) * kWords;
}

// shared implementation: world_rows == nullptr -> single GPU
static int uncertainty_tail_impl(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, int32_t mode,
                                 int64_t b, float* scores, int32_t* out_pos, void* stream, bool sharded, int64_t row_lo,
                                 int64_t rows_min, int64_t rows_max) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || c <= 0 || ld < c || mode < 0 || mode > 2 || b < 0 || (!sharded && b > n))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_tail: bad shape n=%lld c=%d ld=%lld mode=%d b=%lld", (long long)n, c,
                 (long long)ld, mode, (long long)b);
    if ((!sharded && n == 0) || b == 0) return ALQ_OK;
    if (!logits || !scores || !out_pos) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_tail: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    AlqComm& G = ctx->comm;
    if (sharded && (G.world < 1 || !G.connected)) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_uncertainty_tail_sharded: no peer-memory group (alq_comm_create/connect)");
    if (!sharded) { rows_min = rows_max = n; }
    constexpr int kListCap = 2048;
    const size_t reserve = static_cast<size_t>(kListCap) * 8 + 2064 * 4 + 512;      // list, histogram / difference array, s_misc[128]
    RowPipeCfg cfg{};
    size_t smem = 0;
    const bool vec = (c % 4 == 0) && (ld == c) && aligned16(logits) && c <= 2048;
    // every rank must take the same path: the decision only uses what all ranks know (c, b, the smallest and largest shard)
    bool fused = vec && rows_min >= 4096 && rows_max < (1LL << 31) && ctx->select_impl != 1 &&
                 rows_max * 5 <= static_cast<int64_t>(ctx->sm_count) * kListCap * 4 &&     // the per-CTA lists absorb any imbalance
                 plan_row_pipe(ctx, c, cfg, smem, reserve);
    if (fused && sharded) {
        const int64_t tiles_min = (rows_min + cfg.rows_per_tile - 1) / cfg.rows_per_tile;
        const size_t need = 2 * (static_cast<size_t>(2) * G.world * 2048 * 8 + static_cast<size_t>(G.world) * ctx->sm_count * 8 +
                                 static_cast<size_t>(G.world) * (b / G.world + 4096) * 8 + 1024);
        fused = tiles_min >= ctx->sm_count && need <= AlqComm::kTailRegionBytes &&
                G.bytes > G.topb_region_bytes() + AlqComm::kTailRegionBytes && ctx->xchg_status_dev != nullptr;
    }
    if (!fused) {                                   // separate launches: K1, K1b (and the window exchange of the local winners)
        ctx->sel_last_ctr = nullptr;
        // the window exchange takes at most kTopbWords words per rank: a larger budget is declined before anything runs,
        // and on every rank alike (the decision only uses c, b, rows_min and rows_max)
        if (sharded && b > static_cast<int64_t>(AlqComm::kTopbWords))
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_tail_sharded: the launch does not fuse and b = %lld exceeds the %zu "
                     "words of the window exchange (gather the local winners with alq_topb_pack / alq_topb_merge)", (long long)b,
                     AlqComm::kTopbWords);
        int rc = alq_score_softmax(ctx, logits, n, c, ld, mode, scores, stream);
        if (rc) return rc;
        if (!sharded) return alq_select_smallest(ctx, scores, n, b, out_pos, stream);
        const int64_t k = std::min<int64_t>(b, n);
        rc = alq_scratch_reserve(ctx, scratch_need({static_cast<size_t>(n) * 8 + 16, static_cast<size_t>(k + 1) * 4}));   // the selects below reuse the front
        if (rc) return rc;
        int32_t* pos_loc = nullptr;
        if (cudaMallocAsync(reinterpret_cast<void**>(&pos_loc), static_cast<size_t>(k + 1) * 4, st) != cudaSuccess) {
            cudaGetLastError();
            ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "alq_uncertainty_tail_sharded: allocation failed");
        }
        rc = k > 0 ? alq_select_smallest(ctx, scores, n, k, pos_loc, stream) : ALQ_OK;
        if (!rc) rc = alq_topb_exchange(ctx, scores, pos_loc, k, row_lo, b, out_pos, stream);
        cudaFreeAsync(pos_loc, st);
        return rc;
    }
    if (sharded)
        if (int rc0 = alq_comm_check(ctx)) return rc0;       // a previous asynchronous exchange that timed out
    constexpr int kBucketCap = 48;          // per sub-list: a bucket holds up to 16 x 48 words (about b / grid = 68 expected)
    static_assert(132 * kBucketLanes <= 2 * 2048, "bucket counters live in the slot's cross-rank words");
    int rc = alq_scratch_reserve(ctx, scratch_need({static_cast<size_t>(n) * 8 + 16, static_cast<size_t>(ctx->sm_count) * kBucketLanes * kBucketCap * 8}));
    if (rc) return rc;
    SelArgs sel{};
    sel.b = static_cast<int>(b);
    sel.list_cap = kListCap;
    {   // the pipe plan put `reserve` bytes behind the ring: the list starts there, but never below 128 KB + scratch
        const size_t ring_end = (smem - reserve + 15) & ~size_t(15);
        const size_t off = std::max<size_t>(ring_end, 128 * 1024 + static_cast<size_t>(kListCap) * 8);
        sel.list_off = static_cast<int>(off);
        smem = off + reserve;
        if (smem > ctx->smem_optin) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_tail: shared-memory plan does not fit");
    }
    unsigned int* slot = next_sel_slot(ctx, st);
    if (!slot) ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "alq_uncertainty_tail: scratch allocation failed");
    sel.g_hist = slot;
    sel.g_ctr = slot + 4 * 2048;
    sel.g_tot = slot + 2 * 2048;
    ctx->sel_last_ctr = sel.g_ctr;
    {
        ScratchCursor cur(ctx->scratch);
        sel.g_cand = cur.take<unsigned long long>(n + 2);
        if (sharded) sel.bucket_cap = ctx->tail_buckets ? kBucketCap : 0;      // sharded: the route needs no global lists, only the switch
        if (!sharded && ctx->tail_buckets && ctx->sm_count * kBucketLanes <= 2 * 2048) {
            sel.bucket_cap = kBucketCap;
            sel.g_bucket = cur.take<unsigned long long>(static_cast<size_t>(ctx->sm_count) * kBucketLanes * kBucketCap);
            sel.g_bcnt = sel.g_tot;          // the cross-rank sums are not used on one GPU: zeroed words of the slot
        }
    }
    sel.out_pos = out_pos;
    sel.ring_off = cfg.stages * cfg.tile_floats * 4;        // behind the stages' tiles
    sel.ring_bars = 2 * cfg.stages;
    if (sharded) {
        G.epoch += 1;
        sel.world = G.world; sel.rank = G.rank;
        sel.row_base = static_cast<unsigned int>(row_lo);
        for (int r = 0; r < G.world; ++r) sel.peer[r] = G.peer[r];
        sel.stride = ctx->sm_count;
        const size_t hist_bytes = static_cast<size_t>(2) * G.world * 2048 * 8, cnt_bytes = (static_cast<size_t>(G.world) * sel.stride * 8 + 127) & ~size_t(127);
        const size_t base = G.tail_region_off() + (G.epoch & 1) * (AlqComm::kTailRegionBytes / 2);
        // a rank's candidate region: whatever the slot leaves (a rank sends at most its rows; normally about b / world words --
        // only a huge tie group at the threshold can overflow it, and then every rank reports ALQ_ERR_STATE)
        const size_t room = (AlqComm::kTailRegionBytes / 2 - hist_bytes - cnt_bytes - 256) / (static_cast<size_t>(G.world) * 8);
        sel.cand_cap = static_cast<int>(std::min<size_t>(room & ~size_t(1), static_cast<size_t>((rows_max + 1) & ~1LL)));
        sel.hist_off = base;
        sel.cnt_off = base + hist_bytes;
        sel.cand_off = sel.cnt_off + cnt_bytes;
        sel.tag = 0x80000000u | static_cast<unsigned int>(G.epoch & 0x7fffffffu);
        sel.timeout_cycles = ctx->spin_timeout_cycles();
        sel.status = ctx->xchg_status_dev;
    }
    cudaError_t e;
    if (mode == ALQ_MODE_MARGIN) e = launch_rows_pipe_nv<ALQ_MODE_MARGIN>(ctx, st, cfg, smem, logits, n, c, scores, 1, 0, n, nullptr, 0, MaseArgs{}, sel);
    else if (mode == ALQ_MODE_LEAST_CONFIDENCE) e = launch_rows_pipe_nv<ALQ_MODE_LEAST_CONFIDENCE>(ctx, st, cfg, smem, logits, n, c, scores, 1, 0, n, nullptr, 0, MaseArgs{}, sel);
    else e = launch_rows_pipe_nv<ALQ_MODE_ENTROPY>(ctx, st, cfg, smem, logits, n, c, scores, 1, 0, n, nullptr, 0, MaseArgs{}, sel);
    if (e != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_uncertainty_tail: cooperative launch failed: %s", cudaGetErrorString(e));
    }
    return ALQ_OK;
}

// %globaltimer stamps CTA 0 left in the scratch of the LAST fused launch: out_ms[0] = kernel start -> every CTA of this
// GPU has finished streaming its rows (first grid barrier), out_ms[1] = kernel start -> end.  The caller must have
// synchronised the stream of that launch.  ALQ_ERR_STATE if the last tail call did not take the fused path.
extern "C" int alq_uncertainty_tail_timing(alq_ctx* ctx, float* out_ms_host) {
    if (!ctx || !out_ms_host) return ALQ_ERR_INVALID;
    if (!ctx->sel_last_ctr) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_uncertainty_tail_timing: no fused launch yet");
    unsigned long long t[3] = {};
    ALQ_CUDA(ctx, cudaMemcpy(t, ctx->sel_last_ctr + 4, sizeof(t), cudaMemcpyDeviceToHost));
    out_ms_host[0] = t[1] > t[0] ? static_cast<float>((t[1] - t[0]) * 1e-6) : 0.f;
    out_ms_host[1] = t[2] > t[0] ? static_cast<float>((t[2] - t[0]) * 1e-6) : 0.f;
    return ALQ_OK;
}

extern "C" int alq_uncertainty_tail(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, int32_t mode,
                                    int64_t b, float* scores, int32_t* out_pos, void* stream) {
    return uncertainty_tail_impl(ctx, logits, n, c, ld, mode, b, scores, out_pos, stream, false, 0, n, n);
}

extern "C" int alq_uncertainty_tail_sharded(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, int32_t mode,
                                            int64_t b, int64_t row_lo, int64_t rows_min, int64_t rows_max, float* scores,
                                            int32_t* out_gpos, void* stream) {
    if (rows_min < 0 || rows_max < rows_min || n < rows_min || n > rows_max || row_lo < 0) {
        if (!ctx) return ALQ_ERR_INVALID;
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_tail_sharded: n = %lld outside [rows_min, rows_max] = [%lld, %lld]", (long long)n,
                 (long long)rows_min, (long long)rows_max);
    }
    return uncertainty_tail_impl(ctx, logits, n, c, ld, mode, b, scores, out_gpos, stream, true, row_lo, rows_min, rows_max);
}

extern "C" int alq_badge_factors(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld,
                                 int32_t batch_size, int64_t row0, int64_t n_total, float* a, int64_t lda,
                                 float* a_norm2, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    const int cpad = (c + 3) & ~3;
    if (n_total <= 0) { n_total = n; row0 = 0; }
    if (n < 0 || c <= 0 || ld < c || lda < cpad || batch_size <= 0 || row0 < 0 || row0 + n > n_total)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_badge_factors: bad shape n=%lld c=%d ld=%lld lda=%lld bs=%d",
                 (long long)n, c, (long long)ld, (long long)lda, batch_size);
    if (n == 0) return ALQ_OK;
    if (!logits || !a || !a_norm2) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_badge_factors: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = rows_grid(ctx, n, kScoreThreads / 32);
    const bool vec = (c % 4 == 0) && (ld % 4 == 0) && (lda % 4 == 0) && aligned16(logits) &&
                     aligned16(a) && c <= 2048;
    RowPipeCfg cfg{};
    size_t smem = 0;
    if (vec && ld == c && n >= 4096 && plan_row_pipe(ctx, c, cfg, smem)) {
        cudaError_t e = launch_rows_pipe_nv<3>(ctx, st, cfg, smem, logits, n, c, a_norm2, batch_size, row0, n_total, a, lda);
        ctx->launches++;
        if (e != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "rows_pipe_kernel launch failed: %s", cudaGetErrorString(e));
        return ALQ_OK;
    }
    if (vec) {
        const int nv = (c / 4 + 31) / 32;
        if (nv <= 1) badge_factors_vec_kernel<1><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, batch_size, row0, n_total, a, lda, a_norm2);
        else if (nv <= 2) badge_factors_vec_kernel<2><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, batch_size, row0, n_total, a, lda, a_norm2);
        else if (nv <= 4) badge_factors_vec_kernel<4><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, batch_size, row0, n_total, a, lda, a_norm2);
        else if (nv <= 8) badge_factors_vec_kernel<8><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, batch_size, row0, n_total, a, lda, a_norm2);
        else badge_factors_vec_kernel<16><<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, batch_size, row0, n_total, a, lda, a_norm2);
    } else {
        badge_factors_generic_kernel<<<grid, kScoreThreads, 0, st>>>(logits, n, c, ld, batch_size, row0, n_total, a, lda,
                                                                    cpad, a_norm2);
    }
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_badge_pooled_embedding(alq_ctx* ctx, const float* logits, int64_t n, int32_t c,
                                          int64_t ld, int32_t batch_size, const float* emb, int32_t d,
                                          int64_t lde, float* out, int64_t ldo, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    const int ph = c < 16 ? c : 16;          // badge_sampler.py:42  min(POOLING_H, C)
    const int pw = 512 / ph;                 // badge_sampler.py:43  int(POOLING_AREA / pool_h)
    if (n < 0 || c <= 0 || d <= 0 || ld < c || lde < d || ldo < ph * pw || batch_size <= 0)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_badge_pooled_embedding: bad shape n=%lld c=%d d=%d",
                 (long long)n, c, d);
    if (n == 0) return ALQ_OK;
    if (!logits || !emb || !out) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_badge_pooled_embedding: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = static_cast<size_t>(kPoolWarps) * (c + ph + pw) * sizeof(float);
    if (smem > ctx->smem_optin)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_badge_pooled_embedding: c=%d too large for shared memory", c);
    if (smem > 48 * 1024)
        ALQ_CUDA(ctx, cudaFuncSetAttribute(badge_pooled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(smem)));
    const int grid = rows_grid(ctx, n, kPoolWarps);
    badge_pooled_kernel<<<grid, kPoolWarps * 32, smem, st>>>(logits, n, c, ld, batch_size, emb, d, lde,
                                                           ph, pw, out, ldo);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_row_norm2(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ld, float* out,
                             void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || d <= 0 || ld < d) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_row_norm2: bad shape");
    if (n == 0) return ALQ_OK;
    if (!x || !out) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_row_norm2: null pointer");
    const int vec = (d % 4 == 0) && (ld % 4 == 0) && aligned16(x);
    const int grid = rows_grid(ctx, n, kScoreThreads / 32);
    row_norm2_kernel<<<grid, kScoreThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, n, d, ld, vec, out);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

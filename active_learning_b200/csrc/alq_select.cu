// K1b: positions of the B smallest scores in ascending (score, position) order -- the device
// replacement of `torch.sort(scores).indices[:B]` (margin_sampler.py:42, confidence_sampler.py:42
// under active_learning/src/query_strategies) with the fixed tie-break "lowest position first".
//
//   1. 3-level MSB radix select (11+11+10 bits) over the order-preserving uint32 image of the
//      scores finds T, the B-th smallest key, and how many keys tie with it inside the budget.
//   2. One counting pass + one writing pass compact {key < T} (any order) and the first ties
//      {key == T} in position order into B 64-bit keys (key << 32 | position).
//   3. A bitonic network sorts those B keys (single CTA in shared memory for B <= 16384).
//
// Work is O(N) reads of 4 bytes per level: 4*N*5 bytes in total, negligible next to K1's 4*C*N.
#include <initializer_list>

#include "alq_common.cuh"

namespace {

constexpr int kSelThreads = 256;
constexpr int kSelItems = 8;                       // consecutive positions per thread
constexpr int kSelChunk = kSelThreads * kSelItems; // positions per block in the compaction passes
constexpr int kBins = 2048;

struct SelState {
    unsigned long long k;     // 1-based rank still to resolve inside the current prefix
    uint32_t prefix;          // resolved high bits of T
    uint32_t ticket;          // last-block election
    uint32_t lt_counter;      // slots handed out to keys < T
    uint32_t pad;
};

__device__ __forceinline__ uint32_t score_key(float s) { return alq_ord(s + 0.0f); }

// LEVEL 0: bits 31..21, LEVEL 1: bits 20..10, LEVEL 2: bits 9..0
template <int LEVEL>
__global__ void __launch_bounds__(kSelThreads)
select_hist_kernel(const float* __restrict__ scores, int64_t n, SelState* st, uint32_t* hist) {
    __shared__ uint32_t sh[kBins];
    __shared__ unsigned long long part[kSelThreads];
    __shared__ bool last;
    for (int i = threadIdx.x; i < kBins; i += kSelThreads) sh[i] = 0;
    __syncthreads();
    const uint32_t prefix = st->prefix;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kSelThreads;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * kSelThreads + threadIdx.x; i < n; i += stride) {
        const uint32_t key = score_key(scores[i]);
        if (LEVEL == 0) atomicAdd(&sh[key >> 21], 1u);
        else if (LEVEL == 1) { if ((key >> 21) == prefix) atomicAdd(&sh[(key >> 10) & 0x7ffu], 1u); }
        else { if ((key >> 10) == prefix) atomicAdd(&sh[key & 0x3ffu], 1u); }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kBins; i += kSelThreads)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = (atomicAdd(&st->ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    // the last block resolves this level: find the bin holding rank k
    unsigned long long mine[kBins / kSelThreads];
    unsigned long long tot = 0;
#pragma unroll
    for (int j = 0; j < kBins / kSelThreads; ++j) {
        mine[j] = __ldcg(&hist[threadIdx.x * (kBins / kSelThreads) + j]);
        tot += mine[j];
    }
    part[threadIdx.x] = tot;
    __syncthreads();
    for (int off = 1; off < kSelThreads; off <<= 1) {  // inclusive Hillis-Steele scan
        unsigned long long v = threadIdx.x >= off ? part[threadIdx.x - off] : 0ull;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    const unsigned long long k = st->k;
    const unsigned long long incl = part[threadIdx.x];
    const unsigned long long excl = incl - tot;
    __syncthreads();
    if (excl < k && k <= incl) {
        unsigned long long run = excl;
#pragma unroll
        for (int j = 0; j < kBins / kSelThreads; ++j) {
            if (run < k && k <= run + mine[j]) {
                const uint32_t bin = threadIdx.x * (kBins / kSelThreads) + j;
                st->prefix = LEVEL == 2 ? ((prefix << 10) | bin) : ((prefix << 11) | bin);
                st->k = k - run;
            }
            run += mine[j];
        }
    }
    for (int i = threadIdx.x; i < kBins; i += kSelThreads) hist[i] = 0;
    if (threadIdx.x == 0) st->ticket = 0;
}

// Counting pass: ties with T per chunk, then (last block) exclusive offsets.
__global__ void __launch_bounds__(kSelThreads)
select_count_kernel(const float* __restrict__ scores, int64_t n, SelState* st,
                    uint32_t* __restrict__ eq_count, int nblocks) {
    __shared__ uint32_t wsum[kSelThreads / 32];
    __shared__ bool last;
    const uint32_t T = st->prefix;
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kSelChunk + threadIdx.x * kSelItems;
    uint32_t c = 0;
#pragma unroll
    for (int j = 0; j < kSelItems; ++j)
        if (base + j < n) c += (score_key(scores[base + j]) == T);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < kSelThreads / 32; ++w) t += wsum[w];
        eq_count[blockIdx.x] = t;
        __threadfence();
        last = (atomicAdd(&st->ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (threadIdx.x < 32) {  // one warp turns counts into exclusive offsets, 32 blocks at a time
        uint32_t carry = 0;
        for (int b0 = 0; b0 < nblocks; b0 += 32) {
            const int b = b0 + threadIdx.x;
            const uint32_t v = b < nblocks ? __ldcg(&eq_count[b]) : 0u;
            uint32_t inc = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
                if (threadIdx.x >= o) inc += u;
            }
            if (b < nblocks) eq_count[b] = carry + inc - v;
            carry += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (threadIdx.x == 0) st->ticket = 0;
    }
}

__global__ void __launch_bounds__(kSelThreads)
select_write_kernel(const float* __restrict__ scores, int64_t n, int64_t b, SelState* st,
                    const uint32_t* __restrict__ eq_off, unsigned long long* __restrict__ keys) {
    __shared__ uint32_t wsum[kSelThreads / 32];
    const uint32_t T = st->prefix;
    const unsigned long long ties = st->k;                 // ties taken inside the budget
    const unsigned long long n_less = static_cast<unsigned long long>(b) - ties;
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kSelChunk + threadIdx.x * kSelItems;
    uint32_t key[kSelItems];
    uint32_t eq = 0;
#pragma unroll
    for (int j = 0; j < kSelItems; ++j) {
        key[j] = base + j < n ? score_key(scores[base + j]) : 0xffffffffu;
        if (base + j < n && key[j] == T) ++eq;
    }
    // block-exclusive scan of the per-thread tie counts (threads own consecutive positions)
    uint32_t inc = eq;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if ((threadIdx.x & 31) >= o) inc += u;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = inc;
    __syncthreads();
    uint32_t woff = 0;
    for (int w = 0; w < (threadIdx.x >> 5); ++w) woff += wsum[w];
    unsigned long long rank = static_cast<unsigned long long>(eq_off[blockIdx.x]) + woff + inc - eq;
#pragma unroll
    for (int j = 0; j < kSelItems; ++j) {
        if (base + j >= n) break;
        const unsigned long long packed =
            (static_cast<unsigned long long>(key[j]) << 32) | static_cast<uint32_t>(base + j);
        if (key[j] < T) {
            const uint32_t slot = atomicAdd(&st->lt_counter, 1u);
            keys[slot] = packed;
        } else if (key[j] == T) {
            if (rank < ties) keys[n_less + rank] = packed;
            ++rank;
        }
    }
}

// ---- bitonic sorting of the B selected 64-bit keys ---------------------------------------------
__device__ __forceinline__ void cmpxchg(unsigned long long& a, unsigned long long& b, bool up) {
    if ((a > b) == up) { const unsigned long long t = a; a = b; b = t; }
}

// General path for B > 65536: tiles of 4096 keys in shared memory + global exchange steps.
constexpr int kTile = 4096;

__global__ void __launch_bounds__(1024)
sort_pad_kernel(unsigned long long* keys, int64_t b, int64_t npad) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= b && i < npad) keys[i] = ~0ull;
}

// Runs every (k, j) step with j < kTile for k in [k_lo, k_hi] on one tile (k_hi <= kTile means a
// full local sort of the tile up to k_hi; k_lo == k_hi > kTile means only the tail of stage k).
__global__ void __launch_bounds__(1024)
sort_tile_kernel(unsigned long long* keys, int64_t k_lo, int64_t k_hi) {
    __shared__ unsigned long long sk[kTile];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kTile;
    for (int i = threadIdx.x; i < kTile; i += blockDim.x) sk[i] = keys[base + i];
    __syncthreads();
    for (int64_t k = k_lo; k <= k_hi; k <<= 1) {
        int j0 = static_cast<int>(k >> 1 < kTile ? k >> 1 : kTile >> 1);
        for (int j = j0; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (kTile >> 1); t += blockDim.x) {
                const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                const bool up = ((base + lo) & k) == 0;
                cmpxchg(sk[lo], sk[lo | j], up);
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < kTile; i += blockDim.x) keys[base + i] = sk[i];
}

__global__ void __launch_bounds__(256)
sort_global_step_kernel(unsigned long long* keys, int64_t npad, int64_t k, int64_t j) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= (npad >> 1)) return;
    const int64_t lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
    const bool up = (lo & k) == 0;
    unsigned long long a = keys[lo], c = keys[lo | j];
    if ((a > c) == up) { keys[lo] = c; keys[lo | j] = a; }
}

__global__ void __launch_bounds__(256)
sort_emit_kernel(const unsigned long long* __restrict__ keys, int64_t b, int32_t* __restrict__ out_pos) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < b) out_pos[i] = static_cast<int32_t>(keys[i] & 0xffffffffu);
}

// B <= 64k: sort runs of 2048 keys in shared memory (one CTA each), then place every key at
//   rank = (index in own run) + sum over the other runs of #keys smaller than it   (keys are unique)
// by binary search.  Two launches of a few microseconds instead of one 160 us single-CTA network.
constexpr int kRun = 2048;           // keys per run; one CTA of kRun/2 threads sorts a run

// Bitonic network over one run in shared memory.  Thread t owns the pair (lo, lo | j); for j <= 32 all
// pairs of a warp lie inside that warp's own 64-key chunk, so those 51 of the 66 steps need only
// __syncwarp(); the 15 steps with j >= 64 use the block barrier.
__global__ void __launch_bounds__(kRun / 2)
sort_runs_kernel(unsigned long long* __restrict__ keys, int64_t b) {
    __shared__ unsigned long long sk[kRun];
    const int64_t base = static_cast<int64_t>(blockIdx.x) * kRun;
    for (int i = threadIdx.x; i < kRun; i += kRun / 2) sk[i] = base + i < b ? keys[base + i] : ~0ull;
    __syncthreads();
    alq_bitonic_sort_smem(sk, kRun);
    for (int i = threadIdx.x; i < kRun; i += kRun / 2)
        if (base + i < b) keys[base + i] = sk[i];
}

// rank = index in own run + sum over the other runs of #keys smaller.  The binary searches over the other
// runs are independent, so they advance in lock step, 8 runs at a time: 9 dependent load rounds instead
// of 9 * runs.
__global__ void __launch_bounds__(256)
merge_rank_kernel(const unsigned long long* __restrict__ keys, int64_t b, int runs,
                  int32_t* __restrict__ out_pos, int64_t keep) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= b) return;
    const unsigned long long key = keys[i];
    const int my_run = static_cast<int>(i / kRun);
    int64_t rank = i - static_cast<int64_t>(my_run) * kRun;
    constexpr int W = 8;
    for (int r0 = 0; r0 < runs; r0 += W) {
        int lo[W], hi[W];
#pragma unroll
        for (int w = 0; w < W; ++w) {
            const int r = r0 + w;
            lo[w] = 0;
            hi[w] = (r < runs && r != my_run) ? static_cast<int>(min(static_cast<int64_t>(kRun), b - static_cast<int64_t>(r) * kRun)) : 0;
        }
#pragma unroll 1
        for (int step = 0; step < 12; ++step) {      // 2^11 = kRun: at most 12 rounds
            bool any = false;
#pragma unroll
            for (int w = 0; w < W; ++w) {
                if (lo[w] < hi[w]) {
                    const int mid = (lo[w] + hi[w]) >> 1;
                    if (keys[static_cast<int64_t>(r0 + w) * kRun + mid] < key) lo[w] = mid + 1; else hi[w] = mid;
                    any = true;
                }
            }
            if (!any) break;
        }
#pragma unroll
        for (int w = 0; w < W; ++w) rank += lo[w];
        if (rank >= keep) return;
    }
    out_pos[rank] = static_cast<int32_t>(key & 0xffffffffu);
}

// Every rank's B words arrive already sorted (K1b order), so the G lists are merged by rank counting
// alone: rank = own index + sum over the other lists of #words smaller (binary search), no sorting pass.
__global__ void __launch_bounds__(256)
merge_sorted_lists_kernel(const unsigned long long* __restrict__ keys, int lists, int64_t len,
                          int32_t* __restrict__ out_pos, int64_t keep) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= lists * len) return;
    const unsigned long long key = keys[i];
    if (key == ~0ull) return;                               // padding
    const int mine = static_cast<int>(i / len);
    int64_t rank = i - static_cast<int64_t>(mine) * len;
    if (rank >= keep) return;
    // the searches in the other lists are independent: 8 of them advance in lock step, so a word costs
    // ~log2(len) dependent load rounds instead of lists * log2(len)
    constexpr int W = 8;
    for (int r0 = 0; r0 < lists; r0 += W) {
        int64_t lo[W], hi[W];
#pragma unroll
        for (int w = 0; w < W; ++w) {
            lo[w] = 0;
            hi[w] = (r0 + w < lists && r0 + w != mine) ? len : 0;
        }
#pragma unroll 1
        for (int step = 0; step < 40; ++step) {
            bool any = false;
#pragma unroll
            for (int w = 0; w < W; ++w) {
                if (lo[w] < hi[w]) {
                    const int64_t mid = (lo[w] + hi[w]) >> 1;
                    if (keys[static_cast<int64_t>(r0 + w) * len + mid] < key) lo[w] = mid + 1; else hi[w] = mid;
                    any = true;
                }
            }
            if (!any) break;
        }
#pragma unroll
        for (int w = 0; w < W; ++w) rank += lo[w];
        if (rank >= keep) return;
    }
    out_pos[rank] = static_cast<int32_t>(key & 0xffffffffu);
}

// multi-GPU merge helpers -------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
topb_pack_kernel(const float* __restrict__ scores, const int32_t* __restrict__ pos, int64_t k, int64_t row_lo,
                 int64_t b_pad, unsigned long long* __restrict__ out) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= b_pad) return;
    unsigned long long v = ~0ull;
    if (i < k) {
        const int32_t p = pos[i];
        v = (static_cast<unsigned long long>(score_key(scores[p])) << 32) | static_cast<uint32_t>(row_lo + p);
    }
    out[i] = v;
}

int64_t next_pow2(int64_t v) {
    int64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

}  // namespace

int alq_select_smallest_cluster(alq_ctx* ctx, const float* scores, int64_t n, int64_t b, int32_t* out_pos,
                                cudaStream_t st);

extern "C" int alq_select_smallest(alq_ctx* ctx, const float* scores, int64_t n, int64_t b,
                                   int32_t* out_pos, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || b < 0 || b > n || n >= (1LL << 31))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_select_smallest: need 0 <= b <= n < 2^31 (n=%lld b=%lld)",
                 (long long)n, (long long)b);
    if (b == 0) return ALQ_OK;
    if (!scores || !out_pos) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_select_smallest: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (ctx->select_impl != 1) {      // one cluster-resident launch when the pool fits (n <= 262 144, b <= 16 384)
        const int rc = alq_select_smallest_cluster(ctx, scores, n, b, out_pos, st);
        if (rc != ALQ_ERR_STATE) return rc;
        if (ctx->select_impl == 2) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_select_smallest: select_impl=2 needs n <= 262144 and b <= 16384");
    }
    const int nblocks = static_cast<int>((n + kSelChunk - 1) / kSelChunk);
    const int64_t npad = next_pow2(b < 2 ? 2 : b);
    SelState* state;
    uint32_t *hist, *eq_count;
    unsigned long long* keys;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        state = cur.take<SelState>(1);
        hist = cur.take<uint32_t>(kBins);
        eq_count = cur.take<uint32_t>(nblocks);
        keys = cur.take<unsigned long long>(npad);
    });
    if (rc) return rc;

    SelState init{};
    init.k = static_cast<unsigned long long>(b);
    // small struct: an async copy from a stack temporary is staged by the runtime at call time
    ALQ_CUDA(ctx, cudaMemcpyAsync(state, &init, sizeof(init), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(hist, 0, kBins * sizeof(uint32_t), st));

    // K1 (225 KB of dynamic shared memory) runs right before and after these small kernels: ask for the same
    // max-shared carve-out so the SMs do not re-partition L1/shared memory at every kernel boundary.
    static bool carve_set = false;
    if (!carve_set) {
        carve_set = true;
        const int mx = cudaSharedmemCarveoutMaxShared;
        cudaFuncSetAttribute(select_hist_kernel<0>, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaFuncSetAttribute(select_hist_kernel<1>, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaFuncSetAttribute(select_hist_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaFuncSetAttribute(select_count_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaFuncSetAttribute(select_write_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaFuncSetAttribute(sort_runs_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaFuncSetAttribute(merge_rank_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx);
        cudaGetLastError();
    }
    int hgrid = static_cast<int>((n + kSelThreads * 4 - 1) / (kSelThreads * 4));
    if (hgrid > ctx->sm_count * 4) hgrid = ctx->sm_count * 4;
    if (hgrid < 1) hgrid = 1;
    select_hist_kernel<0><<<hgrid, kSelThreads, 0, st>>>(scores, n, state, hist);
    ALQ_LAUNCH_CHECK(ctx);
    select_hist_kernel<1><<<hgrid, kSelThreads, 0, st>>>(scores, n, state, hist);
    ALQ_LAUNCH_CHECK(ctx);
    select_hist_kernel<2><<<hgrid, kSelThreads, 0, st>>>(scores, n, state, hist);
    ALQ_LAUNCH_CHECK(ctx);
    select_count_kernel<<<nblocks, kSelThreads, 0, st>>>(scores, n, state, eq_count, nblocks);
    ALQ_LAUNCH_CHECK(ctx);
    select_write_kernel<<<nblocks, kSelThreads, 0, st>>>(scores, n, b, state, eq_count, keys);
    ALQ_LAUNCH_CHECK(ctx);

    if (b <= 65536) {
        const int runs = static_cast<int>((b + kRun - 1) / kRun);
        sort_runs_kernel<<<runs, kRun / 2, 0, st>>>(keys, b);
        ALQ_LAUNCH_CHECK(ctx);
        merge_rank_kernel<<<static_cast<int>((b + 255) / 256), 256, 0, st>>>(keys, b, runs, out_pos, b);
        ALQ_LAUNCH_CHECK(ctx);
    } else {
        sort_pad_kernel<<<static_cast<int>((npad + 1023) / 1024), 1024, 0, st>>>(keys, b, npad);
        ALQ_LAUNCH_CHECK(ctx);
        const int tiles = static_cast<int>(npad / kTile);
        sort_tile_kernel<<<tiles, 1024, 0, st>>>(keys, 2, kTile);
        ALQ_LAUNCH_CHECK(ctx);
        const int sgrid = static_cast<int>(((npad >> 1) + 255) / 256);
        for (int64_t k = 2 * kTile; k <= npad; k <<= 1) {
            for (int64_t j = k >> 1; j >= kTile; j >>= 1) {
                sort_global_step_kernel<<<sgrid, 256, 0, st>>>(keys, npad, k, j);
                ALQ_LAUNCH_CHECK(ctx);
            }
            sort_tile_kernel<<<tiles, 1024, 0, st>>>(keys, k, k);
            ALQ_LAUNCH_CHECK(ctx);
        }
        sort_emit_kernel<<<static_cast<int>((b + 255) / 256), 256, 0, st>>>(keys, b, out_pos);
        ALQ_LAUNCH_CHECK(ctx);
    }
    return ALQ_OK;
}

// ---- multi-GPU: every rank contributes its local top-B as packed (score key, global position) words;
//      after one all-gather each rank merges the G*B words with the same run-sort + rank-merge.
extern "C" int alq_topb_pack(alq_ctx* ctx, const float* scores, const int32_t* pos, int64_t k, int64_t row_lo,
                             int64_t b_pad, uint64_t* out, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (k < 0 || b_pad < k || row_lo < 0 || row_lo + (1LL << 31) > (1LL << 32) || !out || (k > 0 && (!scores || !pos)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_topb_pack: bad arguments");
    if (b_pad == 0) return ALQ_OK;
    topb_pack_kernel<<<static_cast<int>((b_pad + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        scores, pos, k, row_lo, b_pad, reinterpret_cast<unsigned long long*>(out));
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_topb_merge(alq_ctx* ctx, const uint64_t* keys, int64_t n, int64_t list_len, int64_t b,
                              int32_t* out_gpos, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || b < 0 || b > n || n > (1 << 24) || !keys || !out_gpos)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_topb_merge: bad arguments (n=%lld b=%lld)", (long long)n, (long long)b);
    if (b == 0) return ALQ_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (list_len > 0) {
        if (n % list_len) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_topb_merge: n is not a multiple of list_len");
        merge_sorted_lists_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(
            reinterpret_cast<const unsigned long long*>(keys), static_cast<int>(n / list_len), list_len, out_gpos, b);
        ALQ_LAUNCH_CHECK(ctx);
        return ALQ_OK;
    }
    unsigned long long* work;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) { work = cur.take<unsigned long long>(n); });
    if (rc) return rc;
    ALQ_CUDA(ctx, cudaMemcpyAsync(work, keys, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToDevice, st));
    const int runs = static_cast<int>((n + kRun - 1) / kRun);
    sort_runs_kernel<<<runs, kRun / 2, 0, st>>>(work, n);
    ALQ_LAUNCH_CHECK(ctx);
    merge_rank_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(work, n, runs, out_gpos, b);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

// ---- the same exchange without NCCL: every rank writes its packed winners straight into every peer's window
//      (st.global on CUDA-IPC mappings over NVLink) and raises an epoch-tagged flag; the merge kernel spins on
//      the G flags of its own window and merges the G sorted lists.  Two launches, no collective call.
namespace {
struct TopbXchg {
    int world, rank;
    char* peer[ALQ_MAX_WORLD];
    size_t words_off, flags_off;      // this call's parity half of the reserved region
    unsigned long long tag;
    unsigned int* ticket;
    int* status;                      // mapped host word: sticky, read by the host at the next group call / alq_comm_check
    long long timeout_cycles;
};

__global__ void __launch_bounds__(256)
topb_push_kernel(const float* __restrict__ scores, const int32_t* __restrict__ pos, int64_t k, int64_t row_lo,
                 int64_t b, TopbXchg X) {
    __shared__ bool last;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < b) {
        unsigned long long v = ~0ull;
        if (i < k) {
            const int32_t p = pos[i];
            v = (static_cast<unsigned long long>(score_key(scores[p])) << 32) | static_cast<uint32_t>(row_lo + p);
        }
        for (int g = 0; g < X.world; ++g)
            reinterpret_cast<unsigned long long*>(X.peer[g] + X.words_off)[static_cast<int64_t>(X.rank) * b + i] = v;
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) last = (atomicAdd(X.ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (last && threadIdx.x < X.world)
        st_release_sys(reinterpret_cast<unsigned long long*>(X.peer[threadIdx.x] + X.flags_off) + X.rank, X.tag);
}

__global__ void __launch_bounds__(256)
topb_wait_merge_kernel(TopbXchg X, int64_t len, int32_t* __restrict__ out_pos, int64_t keep) {
    __shared__ bool ok;
    if (threadIdx.x == 0) {
        ok = true;
        for (int r = 0; r < X.world && ok; ++r)
            ok = wait_flag(reinterpret_cast<const unsigned long long*>(X.peer[X.rank] + X.flags_off) + r, X.tag, X.status, X.timeout_cycles);
    }
    __syncthreads();
    const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(X.peer[X.rank] + X.words_off);
    const int lists = X.world;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (!ok) {                        // a peer never showed up: nothing in the window may be trusted
        if (i < keep) out_pos[i] = -1;
        return;
    }
    if (i >= lists * len) return;
    const unsigned long long key = __ldcg(keys + i);
    if (key == ~0ull) return;
    const int mine = static_cast<int>(i / len);
    int64_t rank = i - static_cast<int64_t>(mine) * len;
    if (rank >= keep) return;
    int64_t lo[ALQ_MAX_WORLD], hi[ALQ_MAX_WORLD];
#pragma unroll
    for (int w = 0; w < ALQ_MAX_WORLD; ++w) { lo[w] = 0; hi[w] = (w < lists && w != mine) ? len : 0; }
#pragma unroll 1
    for (int step = 0; step < 40; ++step) {
        bool any = false;
#pragma unroll
        for (int w = 0; w < ALQ_MAX_WORLD; ++w) {
            if (lo[w] < hi[w]) {
                const int64_t mid = (lo[w] + hi[w]) >> 1;
                if (__ldcg(keys + static_cast<int64_t>(w) * len + mid) < key) lo[w] = mid + 1; else hi[w] = mid;
                any = true;
            }
        }
        if (!any) break;
    }
#pragma unroll
    for (int w = 0; w < ALQ_MAX_WORLD; ++w) rank += lo[w];
    if (rank < keep) out_pos[rank] = static_cast<int32_t>(key & 0xffffffffu);
}
}  // namespace

extern "C" int alq_topb_exchange(alq_ctx* ctx, const float* scores, const int32_t* pos, int64_t k, int64_t row_lo,
                                 int64_t b, int32_t* out_gpos, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    AlqComm& G = ctx->comm;
    if (G.world < 1 || !G.connected) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_topb_exchange: no peer-memory group (alq_comm_create/connect)");
    if (k < 0 || b < 1 || k > b || b > static_cast<int64_t>(AlqComm::kTopbWords) || !out_gpos || (k > 0 && (!scores || !pos)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_topb_exchange: bad arguments (k=%lld b=%lld, b <= %zu)", (long long)k, (long long)b,
                 AlqComm::kTopbWords);
    if (G.bytes < 2 * G.topb_region_bytes()) ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "alq_topb_exchange: peer window too small");
    if (!ctx->xchg_status_dev) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_topb_exchange: no mapped status word (cudaHostAlloc failed at alq_create)");
    // a previous (asynchronous) exchange that timed out is reported here, before its garbage can be built upon
    if (int rc0 = alq_comm_check(ctx)) return rc0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned int* ticket;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) { ticket = cur.take<unsigned int>(1); });
    if (rc) return rc;
    int* status = ctx->xchg_status_dev;
    ALQ_CUDA(ctx, cudaMemsetAsync(ticket, 0, 4, st));
    G.epoch += 1;
    TopbXchg X{};
    X.world = G.world; X.rank = G.rank;
    for (int r = 0; r < G.world; ++r) X.peer[r] = G.peer[r];
    const size_t half = G.topb_region_bytes() / 2;
    const size_t base = G.bytes - G.topb_region_bytes() + (G.epoch & 1) * half;
    X.words_off = base;
    X.flags_off = base + static_cast<size_t>(G.world) * AlqComm::kTopbWords * 8;
    X.tag = G.epoch << 32;
    X.ticket = ticket; X.status = status;
    X.timeout_cycles = ctx->spin_timeout_cycles();
    const int blocks = static_cast<int>((b + 255) / 256);
    topb_push_kernel<<<blocks, 256, 0, st>>>(scores, pos, k, row_lo, b, X);
    ALQ_LAUNCH_CHECK(ctx);
    topb_wait_merge_kernel<<<static_cast<int>((G.world * b + 255) / 256), 256, 0, st>>>(X, b, out_gpos, b);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

// Sticky status of the asynchronous peer-window exchanges (alq_topb_exchange): the kernels write it straight into a
// mapped host word, so reading it costs nothing -- but it is only final once the caller has synchronised the stream
// the exchange ran on (e.g. after copying its result to the host).  Returns ALQ_OK, or ALQ_ERR_STATE (and clears it) if
// a peer's flag never arrived within "spin_timeout_ms": the positions that exchange produced were all set to -1.
extern "C" int alq_comm_check(alq_ctx* ctx) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!ctx->xchg_status_host) return ALQ_OK;
    const int s = *reinterpret_cast<volatile int*>(ctx->xchg_status_host);
    if (s == 0) return ALQ_OK;
    *reinterpret_cast<volatile int*>(ctx->xchg_status_host) = 0;
    ALQ_FAIL(ctx, ALQ_ERR_STATE, "peer-window exchange timed out waiting for a peer GPU's flag (spin_timeout_ms = %d): its result is invalid",
             ctx->spin_timeout_ms);
}

// Host-buffer entry point: H2D of the logits in row chunks on two side streams, K1 on each chunk
// as soon as it lands, then the select on the second stream and the B positions back.
extern "C" int alq_uncertainty_query_host(alq_ctx* ctx, const float* logits_host, int64_t n, int32_t c,
                                          int32_t mode, int64_t b, int32_t* out_pos_host) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (n < 0 || c <= 0 || b < 0 || b > n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_query_host: bad shape n=%lld c=%d b=%lld",
                 (long long)n, c, (long long)b);
    if (b == 0) return ALQ_OK;
    if (!logits_host || !out_pos_host)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_uncertainty_query_host: null pointer");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    // private arena (not the shared scratch: alq_select_smallest re-carves that one)
    const int64_t chunk_rows = std::max<int64_t>(1, (32ll << 20) / (static_cast<int64_t>(c) * 4));
    const size_t chunk_elems = static_cast<size_t>(chunk_rows) * c;
    float *buf[2], *scores;
    int32_t* pos;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        buf[0] = cur.take<float>(chunk_elems);
        buf[1] = cur.take<float>(chunk_elems);
        scores = cur.take<float>(n);
        pos = cur.take<int32_t>(b);
    }, /*arena2=*/true);
    if (rc) return rc;
    auto cleanup = [&]() {};
    cudaStream_t ss[2] = {ctx->side_stream, ctx->side_stream2};
    int which = 0;
    for (int64_t lo = 0; lo < n && rc == ALQ_OK; lo += chunk_rows, which ^= 1) {
        const int64_t rows = std::min(chunk_rows, n - lo);
        if (cudaMemcpyAsync(buf[which], logits_host + lo * c, static_cast<size_t>(rows) * c * sizeof(float),
                            cudaMemcpyHostToDevice, ss[which]) != cudaSuccess) {
            ctx->err = "alq_uncertainty_query_host: H2D copy failed";
            rc = ALQ_ERR_CUDA;
            break;
        }
        rc = alq_score_softmax(ctx, buf[which], rows, c, c, mode, scores + lo, ss[which]);
    }
    if (rc == ALQ_OK) {
        cudaEventRecord(ctx->ev_a, ss[0]);
        cudaStreamWaitEvent(ss[1], ctx->ev_a, 0);
        rc = alq_select_smallest(ctx, scores, n, b, pos, ss[1]);
    }
    if (rc == ALQ_OK) {
        if (cudaMemcpyAsync(out_pos_host, pos, static_cast<size_t>(b) * sizeof(int32_t),
                            cudaMemcpyDeviceToHost, ss[1]) != cudaSuccess ||
            cudaStreamSynchronize(ss[1]) != cudaSuccess) {
            ctx->err = std::string("alq_uncertainty_query_host: ") + cudaGetErrorString(cudaGetLastError());
            rc = ALQ_ERR_CUDA;
        }
    } else {
        cudaDeviceSynchronize();
    }
    cleanup();
    return rc;
}

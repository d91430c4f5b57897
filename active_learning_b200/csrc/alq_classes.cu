// K10: per-class counts and the class-balanced random picks of BalancedRandomSampler (balanced_random_sampler.py:29-95
// of active_learning/src/query_strategies), from device-resident labels.
//
// The reference builds a float copy of the labels, then for EVERY class runs `torch.where(labels == c, avail, False)`
// and `nonzero()` over the whole pool (O(N * C)).  Here the pool is read once per call:
//   * tile histogram: the pool is cut into tiles of `class_tile(C)` rows; one CTA builds a tile's histogram of the
//     available rows in shared memory and writes it to a table tab[t][c] (scratch);
//   * tile scan: per class, an exclusive prefix over the tiles, in place; row `ntiles` receives the class totals;
//   * pick: one warp per output: a binary search of the budget prefix gives the class, a binary search of the class's
//     column gives the tile, and warp ballots on `labels == c && avail` walk the tile to the wanted row.
// Every output is computed independently and without atomics, so the result is deterministic.
// The tile is 1024 * ceil(C / 1024) rows: at least C, so the table holds at most n + 2C entries whatever C is.
#include <limits.h>

#include "alq_common.cuh"

namespace {

constexpr int kTileBase = ALQ_CLASS_TILE;
constexpr int kHistThreads = 512;
constexpr int kPickThreads = 256;
constexpr int kPickRows = 128;          // rows a warp tests per step of the tile walk (4 ballots)

inline int class_tile(int c) { return kTileBase * ((c + kTileBase - 1) / kTileBase); }

// tab[t * c + k] = number of rows i of tile t with avail[i] != 0 and labels[i] == k.  An available row whose label is
// outside [0, c) is not counted; with `bad` given, the smallest such row is recorded there (atomicMin, UINT_MAX = none).
__global__ void __launch_bounds__(kHistThreads)
class_tile_hist_kernel(const int32_t* __restrict__ labels, const uint8_t* __restrict__ avail, int n, int c, int tile,
                       int ntiles, int32_t* __restrict__ tab, unsigned int* __restrict__ bad) {
    extern __shared__ int hist[];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        for (int k = threadIdx.x; k < c; k += blockDim.x) hist[k] = 0;
        __syncthreads();
        const int lo = t * tile;
        const int hi = static_cast<int>(min(static_cast<int64_t>(n), static_cast<int64_t>(lo) + tile));
        for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            if (avail[i]) {
                const int y = labels[i];
                if (static_cast<unsigned>(y) < static_cast<unsigned>(c)) atomicAdd(&hist[y], 1);
                else if (bad) atomicMin(bad, static_cast<unsigned>(i));
            }
        }
        __syncthreads();
        int32_t* row = tab + static_cast<int64_t>(t) * c;
        for (int k = threadIdx.x; k < c; k += blockDim.x) row[k] = hist[k];
        __syncthreads();
    }
}

// Per class k: tab[t * c + k] <- sum of the tile counts before t (exclusive prefix), tab[ntiles * c + k] <- the total
// (and counts[k], if given).  A 32 x 32 block owns 32 consecutive classes: x = class (coalesced rows of the table),
// y = a contiguous chunk of tiles.
__global__ void __launch_bounds__(1024)
class_tile_scan_kernel(int32_t* __restrict__ tab, int ntiles, int c, int32_t* __restrict__ counts) {
    __shared__ int part[32][33];
    const int k = blockIdx.x * 32 + threadIdx.x;
    const int chunk = (ntiles + 31) / 32;
    const int t0 = threadIdx.y * chunk, t1 = min(ntiles, t0 + chunk);
    int s = 0;
    if (k < c)
        for (int t = t0; t < t1; ++t) s += tab[static_cast<int64_t>(t) * c + k];
    part[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0) {
        int run = 0;
        for (int j = 0; j < 32; ++j) {
            const int v = part[j][threadIdx.x];
            part[j][threadIdx.x] = run;
            run += v;
        }
        if (k < c) {
            tab[static_cast<int64_t>(ntiles) * c + k] = run;
            if (counts) counts[k] = run;
        }
    }
    __syncthreads();
    if (k < c) {
        int run = part[threadIdx.y][threadIdx.x];
        for (int t = t0; t < t1; ++t) {
            const int64_t o = static_cast<int64_t>(t) * c + k;
            const int v = tab[o];
            tab[o] = run;
            run += v;
        }
    }
}

// koff[i] = sum of max(k[j], 0) over j < i, for i = 0 .. c (one CTA; c <= ALQ_CLASS_MAX).
__global__ void __launch_bounds__(1024)
class_budget_prefix_kernel(const int32_t* __restrict__ k, int c, int32_t* __restrict__ koff) {
    __shared__ int wsum[32];
    const int per = (c + 1023) / 1024;
    const int a = threadIdx.x * per, b = min(c, a + per);
    int s = 0;
    for (int i = a; i < b; ++i) s += max(k[i], 0);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int v = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) wsum[w] = v;
    __syncthreads();
    if (w == 0) {
        int x = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += u;
        }
        wsum[lane] = x;
    }
    __syncthreads();
    int run = v - s + (w ? wsum[w - 1] : 0);
    for (int i = a; i < b; ++i) {
        koff[i] = run;
        run += max(k[i], 0);
    }
    if (threadIdx.x == 1023) koff[c] = run;
}

// out[j] = the perm[j]-th available row (ascending row order) of the class cls with koff[cls] <= j < koff[cls + 1];
// -1 if j is past the last budget or perm[j] is not in [0, n_cls).  One warp per output.
__global__ void __launch_bounds__(kPickThreads)
class_pick_kernel(const int32_t* __restrict__ labels, const uint8_t* __restrict__ avail, int n, int c, int tile,
                  int ntiles, const int32_t* __restrict__ pre, const int32_t* __restrict__ koff,
                  const int32_t* __restrict__ perm, int b, int32_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (kPickThreads / 32);
    for (int j = blockIdx.x * (kPickThreads / 32) + (threadIdx.x >> 5); j < b; j += warps) {
        int found = -1;
        if (j < koff[c]) {
            int lo = 0, hi = c;                           // the largest class with koff[class] <= j
            while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (koff[mid] <= j) lo = mid;
                else hi = mid;
            }
            const int cls = lo;
            const int r = perm[j];
            if (r >= 0 && r < pre[static_cast<int64_t>(ntiles) * c + cls]) {
                int tl = 0, th = ntiles;                  // the largest tile whose prefix is <= r
                while (th - tl > 1) {
                    const int mid = (tl + th) >> 1;
                    if (pre[static_cast<int64_t>(mid) * c + cls] <= r) tl = mid;
                    else th = mid;
                }
                int rem = r - pre[static_cast<int64_t>(tl) * c + cls];
                const int base = tl * tile;
                const int end = static_cast<int>(min(static_cast<int64_t>(n), static_cast<int64_t>(base) + tile));
                for (int64_t i0 = base; i0 < end && found < 0; i0 += kPickRows) {
                    unsigned int m[kPickRows / 32];
#pragma unroll
                    for (int u = 0; u < kPickRows / 32; ++u) {
                        const int64_t i = i0 + 32 * u + lane;
                        const bool in = i < end;
                        const int y = in ? labels[i] : -1;
                        const uint8_t a = in ? avail[i] : 0;
                        m[u] = __ballot_sync(0xffffffffu, a != 0 && y == cls);
                    }
#pragma unroll
                    for (int u = 0; u < kPickRows / 32; ++u) {
                        const int pc = __popc(m[u]);
                        if (found < 0 && rem < pc) {
                            unsigned int mm = m[u];
                            for (int q = 0; q < rem; ++q) mm &= mm - 1;
                            found = static_cast<int>(i0) + 32 * u + __ffs(mm) - 1;
                        } else if (found < 0) {
                            rem -= pc;
                        }
                    }
                }
            }
        }
        if (lane == 0) out[j] = found;
    }
}

}  // namespace

// K10's table pass and its size, shared with K11 (alq_balancing.cu): declared in alq_common.cuh
int alq_class_table_pass(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int n, int c, int32_t* tab,
               unsigned int* bad, int32_t* counts, cudaStream_t st) {
    const int tile = class_tile(c);
    const int ntiles = static_cast<int>((static_cast<int64_t>(n) + tile - 1) / tile);
    const size_t smem = static_cast<size_t>(c) * sizeof(int);
    if (smem > 48u * 1024u)
        ALQ_CUDA(ctx, cudaFuncSetAttribute(class_tile_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(smem)));
    const int grid = std::min(ntiles, ctx->sm_count * 4);
    class_tile_hist_kernel<<<grid, kHistThreads, smem, st>>>(labels, avail, n, c, tile, ntiles, tab, bad);
    ALQ_LAUNCH_CHECK(ctx);
    class_tile_scan_kernel<<<(c + 31) / 32, dim3(32, 32), 0, st>>>(tab, ntiles, c, counts);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

size_t alq_class_table_entries(int64_t n, int c) {
    const int tile = class_tile(c);
    return static_cast<size_t>((n + tile - 1) / tile + 1) * static_cast<size_t>(c);
}

extern "C" int alq_class_counts(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int64_t n, int32_t c,
                                int32_t* counts, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (c < 1 || c > ALQ_CLASS_MAX)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_counts: C=%d outside [1, %d]", c, ALQ_CLASS_MAX);
    if (n < 0 || n > INT_MAX) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_counts: n=%lld outside [0, 2^31)", (long long)n);
    if (!counts || (n > 0 && (!labels || !avail))) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_counts: null pointer");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n == 0) {
        ALQ_CUDA(ctx, cudaMemsetAsync(counts, 0, static_cast<size_t>(c) * sizeof(int32_t), st));
        return ALQ_OK;
    }
    const size_t entries = alq_class_table_entries(n, c);
    int32_t* tab;
    unsigned int* bad;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        tab = cur.take<int32_t>(entries);
        bad = cur.take<unsigned int>(1);
    });
    if (rc != ALQ_OK) return rc;
    ALQ_CUDA(ctx, cudaMemsetAsync(bad, 0xff, sizeof(unsigned int), st));
    rc = alq_class_table_pass(ctx, labels, avail, static_cast<int>(n), c, tab, bad, counts, st);
    if (rc != ALQ_OK) return rc;
    unsigned int bad_row = UINT_MAX;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&bad_row, bad, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (bad_row != UINT_MAX) {
        int32_t y = 0;
        ALQ_CUDA(ctx, cudaMemcpy(&y, labels + bad_row, sizeof(int32_t), cudaMemcpyDeviceToHost));
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_counts: available row %u has label %d, outside [0, %d)", bad_row, y, c);
    }
    return ALQ_OK;
}

extern "C" int alq_class_pick(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int64_t n, int32_t c,
                              const int32_t* k, const int32_t* perm, int64_t b, int32_t* out, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (c < 1 || c > ALQ_CLASS_MAX)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_pick: C=%d outside [1, %d]", c, ALQ_CLASS_MAX);
    if (n < 0 || n > INT_MAX || b < 0 || b > INT_MAX)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_pick: n=%lld or B=%lld outside [0, 2^31)", (long long)n, (long long)b);
    if (!k || (b > 0 && (!perm || !out)) || (n > 0 && (!labels || !avail)))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_class_pick: null pointer");
    if (b == 0) return ALQ_OK;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n == 0) {                       // no rows: no output has a row
        ALQ_CUDA(ctx, cudaMemsetAsync(out, 0xff, static_cast<size_t>(b) * sizeof(int32_t), st));
        return ALQ_OK;
    }
    const size_t entries = alq_class_table_entries(n, c);
    int32_t *tab, *koff;
    int rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) {
        tab = cur.take<int32_t>(entries);
        koff = cur.take<int32_t>(static_cast<size_t>(c) + 1);
    });
    if (rc != ALQ_OK) return rc;
    rc = alq_class_table_pass(ctx, labels, avail, static_cast<int>(n), c, tab, nullptr, nullptr, st);
    if (rc != ALQ_OK) return rc;
    class_budget_prefix_kernel<<<1, 1024, 0, st>>>(k, c, koff);
    ALQ_LAUNCH_CHECK(ctx);
    const int tile = class_tile(c);
    const int ntiles = static_cast<int>((n + tile - 1) / tile);
    const int per_cta = kPickThreads / 32;
    const int grid = static_cast<int>(std::min<int64_t>((b + per_cta - 1) / per_cta, static_cast<int64_t>(ctx->sm_count) * 16));
    class_pick_kernel<<<grid, kPickThreads, 0, st>>>(labels, avail, static_cast<int>(n), c, tile, ntiles, tab, koff, perm,
                                                     static_cast<int>(b), out);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

// Shared by K11 (alq_balancing.cu) and K12 (alq_balancing_table.cu), BalancingSampler's persistent query: the segment of
// a row, the pick words, the fp32 imbalance test, the class denominators, NumPy's MT19937 and bal_select, the host driver
// of both entry points.  The CTA segments and the LL-word agreement: alq_ll.cuh.
#pragma once
#include <limits.h>

#include "alq_ll.cuh"

// The driver's one step that lives in K11's file (alq_balancing.cu), beside its kernel: one launch counting the available
// rows of every global segment (seg_avail[world * grid]) and the smallest available row with a label outside [0, c)
// (atomicMin into *bad).
int bal_seg_count(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int c, const SegShard& S, int32_t* seg_avail,
                  unsigned int* bad, cudaStream_t st);

namespace {

constexpr int kMtN = 624;
// the global segment holding `row` (0 <= row < off[world])
__device__ __forceinline__ int gseg_of(const SegShard& S, int row) {
    int r = 0;
    while (r + 1 < S.world && S.off[r + 1] <= row) ++r;
    const int grid = S.grid, rows = S.off[r + 1] - S.off[r], p = row - S.off[r];
    int o = static_cast<int>(static_cast<long long>(p) * grid / rows);
    while (o + 1 < grid && seg_lo(rows, grid, o + 1) <= p) ++o;
    while (o > 0 && seg_lo(rows, grid, o) > p) --o;
    return r * grid + o;
}

__device__ __forceinline__ unsigned int bal_pick_tag(const LLWords& W, int t) {   // t < 2^24: the budget limit
    return W.tag_base | static_cast<unsigned int>(t);
}

// balancing_sampler.py:89 in fp32: fl32(count + 1e-5)
__device__ __forceinline__ float bal_den(int count) { return __fadd_rn(static_cast<float>(count), 1e-5f); }

// balancing_sampler.py:66-84 as torch evaluates it on the CPU, from the exact integer tallies: the fp32 mean of the
// counts, and whether the step balances (remaining <= fl32(#rest) * spread, spread NaN when no class is above the mean)
__device__ __forceinline__ float bal_mean(int total, int c) {
    return __fdiv_rn(static_cast<float>(total), static_cast<float>(c));
}
__device__ __forceinline__ bool bal_balances(int remaining, int na, int sa, int nr, int sr) {
    const float spread = __fsub_rn(__fdiv_rn(static_cast<float>(sa), static_cast<float>(na)),
                                   __fdiv_rn(static_cast<float>(sr), static_cast<float>(nr)));
    return static_cast<float>(remaining) <= __fmul_rn(static_cast<float>(nr), spread);
}

// One thread, O(c): counts (< 2^24) against their fp32 mean, each average fl32(sum) / fl32(n).  Returns the number of
// selected classes (0: random step): sel[0] = the rarest class (first index of the minimum), sel[1..] = the majority
// classes ascending.
__device__ int imbalance_test(const int* cnt, int c, int remaining, int* sel) {
    int total = 0, rare = 0;
    for (int i = 0; i < c; ++i) {
        total += cnt[i];
        if (cnt[i] < cnt[rare]) rare = i;
    }
    const float mean = bal_mean(total, c);
    int na = 0, sa = 0, nr = 0, sr = 0;
    for (int i = 0; i < c; ++i) {
        if (static_cast<float>(cnt[i]) > mean) { ++na; sa += cnt[i]; }
        else { ++nr; sr += cnt[i]; }
    }
    if (!bal_balances(remaining, na, sa, nr, sr)) return 0;
    sel[0] = rare;
    int m = 1;
    for (int i = 0; i < c; ++i)
        if (static_cast<float>(cnt[i]) > mean) sel[m++] = i;
    return m;
}

// NumPy's mt19937_gen / mt19937_next32 (numpy/random/src/mt19937), one thread, state in shared memory
__device__ void mt_twist(unsigned int* mt) {
    for (int i = 0; i < kMtN; ++i) {
        const unsigned int y = (mt[i] & 0x80000000u) | (mt[i + 1 < kMtN ? i + 1 : 0] & 0x7fffffffu);
        const int j = i + 397 < kMtN ? i + 397 : i + 397 - kMtN;
        mt[i] = mt[j] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
}
__device__ __forceinline__ unsigned int mt_next32(unsigned int* mt, int& pos) {
    if (pos >= kMtN) { mt_twist(mt); pos = 0; }
    unsigned int y = mt[pos++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}
// legacy RandomState.randint(0, rng + 1) for rng < 2^32 - 1 (random_bounded_uint64_fill, masked): rng == 0 draws nothing
__device__ unsigned int mt_bounded(unsigned int* mt, int& pos, unsigned int rng) {
    if (rng == 0) return 0;
    unsigned int mask = rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    unsigned int v;
    while ((v = (mt_next32(mt, pos) & mask)) > rng) {}
    return v;
}

// ---- the host driver of both loops ----------------------------------------------------------------------------------
// bal_select<K> runs a whole call: the descriptor checks, the option, the shard layout, the limits in a fixed order, the
// counts, the MT19937 state, the LL words, the launch and the read-back.  K, a struct of each loop's file, supplies
// only what differs: its name and forcing option, its shared-memory plan, its scratch and set-up launches, its own
// kernel arguments, and the kernel.

constexpr size_t kWordsHead = 128;               // u64 ready[ALQ_MAX_WORLD] in front of a window's words (greedy's layout)
constexpr size_t kBalDescV1 = offsetof(alq_balancing_desc, shard_off_host);   // the single-GPU descriptor ends here

// A limit the call exceeds: the call declines (ALQ_OK with *n_picks_host = -1: the caller runs another path) unless the
// option forces this loop, which then fails naming the limit.
#define BAL_LIMIT(B, ...)                                    \
    do {                                                     \
        if (!(B).forced) {                                   \
            (B).declined = true;                             \
            return ALQ_OK;                                   \
        }                                                    \
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, __VA_ARGS__);         \
    } while (0)

// What the driver knows of a call when it hands over to the loop's own steps.
struct BalCall {
    const alq_balancing_desc* D;
    cudaStream_t st;
    int n, c, d;
    bool forced, sharded;
    bool declined;                               // a limit of the loop's own steps declined the call (BAL_LIMIT)
    SegShard S;
    int nseg;
    size_t smem_cap;                             // dynamic shared memory per CTA (the kernels' static shared memory aside)
    size_t entries;                              // K10's table pass (int32)
    size_t words_max;                            // bytes of the LL words at the requested budget (at most n picks)
    // after the counts
    std::vector<int32_t> counts_h, seg_h;
    int64_t n_avail, labeled_total;
    int budget;                                  // at most n_avail
    int32_t* counts;                             // counts_h and seg_h on the device
    int32_t* seg_avail;
    size_t avail_of(int r) const {               // the available rows of rank r's segments
        int64_t a = 0;
        for (int g = r * S.grid; g < (r + 1) * S.grid; ++g) a += seg_h[g];
        return static_cast<size_t>(a);
    }
};

size_t up128(size_t v) { return (v + 127) & ~size_t(127); }

// Bytes of the LL words (from the window's start); sharded calls need them inside the window's greedy region.
size_t bal_words_bytes(const SegShard& S, int64_t budget, bool sharded) {
    const size_t keyw = sharded ? kWordsHead : 0;
    return up128(keyw + static_cast<size_t>(2) * S.world * S.grid * 8) + static_cast<size_t>(budget) * 8;
}

// The body of both entry points, alq_balancing_select (K11) and alq_balancing_table_select (K12).  K's steps, in the
// order they run:
//   int plan_smem(ctx, BalCall&)                       the shared-memory limit; sets smem, the loop's dynamic shared memory
//   int fits(ctx, BalCall&, bytes_for)                 after the counts: the loop's memory limits; bytes_for(na) measures
//                                                      the call's scratch layout with na available rows on the rank
//   void carve(ScratchCursor&, const BalCall&, na, Args&)   the loop's own buffers in that layout
//   int setup(ctx, BalCall&, Args&)                    its set-up uploads and launches
template <class K>
int bal_select(alq_ctx* ctx, const alq_balancing_desc* D, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    const char* const fn = K::kName;
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
    *D->n_picks_host = -1;                                            // from here on an early return declines
    *D->n_balancing_host = 0;
    if (ctx->balancing_loop != 0 && ctx->balancing_loop != K::kForce) return ALQ_OK;   // the per-step path or the other loop
    const int n = static_cast<int>(n64);
    if (n == 0 || D->budget == 0) {
        *D->n_picks_host = 0;
        return ALQ_OK;
    }
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    BalCall B{};
    B.D = D; B.st = st;
    B.n = n; B.c = c; B.d = d;
    B.forced = ctx->balancing_loop == K::kForce;

    // ---- limits that the shape decides (the same on every rank of a sharded call) -------------------------------------
    // The layout (S.grid from the smallest shard, the same on every rank).  A sharded call (the descriptor carries
    // shard_off_host) needs the group of alq_comm_create/connect and shard offsets that start at 0, do not decrease and
    // end at n.
    SegShard& S = B.S;
    const int32_t* so = D->struct_size >= sizeof(alq_balancing_desc) ? D->shard_off_host : nullptr;
    B.sharded = so != nullptr;
    S.world = 1;
    S.rank = 0;
    S.off[0] = 0;
    S.off[1] = n;
    if (so) {
        const AlqComm& G = ctx->comm;
        if (!G.window || !G.connected)
            ALQ_FAIL(ctx, ALQ_ERR_STATE, "%s: a sharded call (shard_off_host) needs the group of alq_comm_create/connect", fn);
        if (so[0] != 0 || so[G.world] != n)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: shard_off must run from 0 to n=%d, got %d .. %d", fn, n, so[0], so[G.world]);
        for (int r = 0; r < G.world; ++r)
            if (so[r + 1] < so[r]) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: shard_off[%d] = %d < shard_off[%d] = %d", fn, r + 1, so[r + 1], r, so[r]);
        S.world = G.world;
        S.rank = G.rank;
        std::copy(so, so + G.world + 1, S.off);
    }
    int rows_min = n;
    for (int r = 0; r < S.world; ++r) rows_min = std::min(rows_min, S.off[r + 1] - S.off[r]);
    S.grid = std::max(1, std::min(ctx->sm_count, (rows_min + 127) / 128));
    const int nseg = B.nseg = S.world * S.grid;
    B.smem_cap = ctx->smem_optin > 4096 ? ctx->smem_optin - 1024 : 0;
    K k;
    int rc = k.plan_smem(ctx, B);
    if (rc != ALQ_OK || B.declined) return rc;
    int seg_rows_max = 0;                                             // the key word carries a 16-bit row offset
    for (int g = 0; g < nseg; ++g) seg_rows_max = std::max(seg_rows_max, gseg_lo(S, g + 1) - gseg_lo(S, g));
    if (seg_rows_max > kSegRowsMax)
        BAL_LIMIT(B, "%s: n=%d rows over %d CTAs exceed %d rows per CTA segment (limit: rows per segment)", fn, n, nseg,
                  kSegRowsMax);
    B.words_max = bal_words_bytes(S, std::min<int64_t>(D->budget, n), B.sharded);
    if (B.sharded && B.words_max > ctx->comm.greedy_bytes())
        BAL_LIMIT(B, "%s: a budget of %lld needs %zu bytes of the peer window, %zu are usable (limit: words in the peer "
                  "window)", fn, (long long)D->budget, B.words_max, ctx->comm.greedy_bytes());

    // ---- set-up: K10's table pass over the labeled rows (the counts) and one launch counting the available rows of
    // every global segment; a labeled or available row whose label is outside [0, c) fails naming the row and its label
    B.entries = alq_class_table_entries(n, c);
    int32_t* tab;
    unsigned int* bad;
    auto counts_layout = [&](ScratchCursor& cur) {
        tab = cur.take<int32_t>(B.entries);
        B.counts = cur.take<int32_t>(c);
        bad = cur.take<unsigned int>(2);
        B.seg_avail = cur.take<int32_t>(nseg);
    };
    rc = alq_scratch_carve(ctx, counts_layout);
    if (rc != ALQ_OK) return rc;
    ALQ_CUDA(ctx, cudaMemsetAsync(bad, 0xff, 2 * sizeof(unsigned int), st));
    rc = alq_class_table_pass(ctx, D->labels, D->labeled, n, c, tab, bad, B.counts, st);
    if (rc != ALQ_OK) return rc;
    rc = bal_seg_count(ctx, D->labels, D->avail, c, S, B.seg_avail, bad + 1, st);
    if (rc != ALQ_OK) return rc;
    B.counts_h.resize(c);
    B.seg_h.resize(nseg);
    unsigned int bad_h[2] = {UINT_MAX, UINT_MAX};
    ALQ_CUDA(ctx, cudaMemcpyAsync(bad_h, bad, sizeof(bad_h), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(B.counts_h.data(), B.counts, static_cast<size_t>(c) * 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(B.seg_h.data(), B.seg_avail, static_cast<size_t>(nseg) * 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    for (int i = 1; i >= 0; --i)
        if (bad_h[i] != UINT_MAX) {
            int32_t y = 0;
            ALQ_CUDA(ctx, cudaMemcpy(&y, D->labels + bad_h[i], sizeof(int32_t), cudaMemcpyDeviceToHost));
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: %s row %u has label %d, outside [0, %d)", fn,
                     i ? "available" : "labeled", bad_h[i], y, c);
        }
    for (int g = 0; g < nseg; ++g) B.n_avail += B.seg_h[g];
    for (int i = 0; i < c; ++i) B.labeled_total += B.counts_h[i];
    B.budget = static_cast<int>(std::min<int64_t>(D->budget, B.n_avail));
    if (B.labeled_total + B.budget >= (1LL << 24))
        BAL_LIMIT(B, "%s: %lld labeled rows plus a budget of %d reach 2^24 (limit: counts plus budget below 2^24)", fn,
                  (long long)B.labeled_total, B.budget);
    if (B.budget == 0) {
        *D->n_picks_host = 0;
        return ALQ_OK;
    }

    // ---- the call's whole scratch: the counts' buffers, the loop's own, the working mask, the RNG state, the words and
    // the status.  The carve may move the arena, so the counts go up again from the host.  Then the loop's own set-up.
    typename K::Args A{};
    const size_t words = bal_words_bytes(S, B.budget, B.sharded);
    uint8_t* avail;
    unsigned int* mt;
    char* word_scratch;
    int* small;
    auto layout = [&](ScratchCursor& cur, size_t na) {
        counts_layout(cur);
        k.carve(cur, B, na, A);
        avail = cur.take<uint8_t>(n);
        mt = cur.take<unsigned int>(2 * (kMtN + 1));
        word_scratch = cur.take<char>(B.sharded ? 0 : words);
        small = cur.take<int>(4);                                     // [0] status, [1] balancing steps
    };
    rc = k.fits(ctx, B, [&](size_t na) { return alq_layout_bytes([&](ScratchCursor& cur) { layout(cur, na); }); });
    if (rc != ALQ_OK || B.declined) return rc;
    rc = alq_scratch_carve(ctx, [&](ScratchCursor& cur) { layout(cur, B.avail_of(S.rank)); });
    if (rc != ALQ_OK) return rc;
    ALQ_CUDA(ctx, cudaMemcpyAsync(B.counts, B.counts_h.data(), static_cast<size_t>(c) * 4, cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(B.seg_avail, B.seg_h.data(), static_cast<size_t>(nseg) * 4, cudaMemcpyHostToDevice, st));
    rc = k.setup(ctx, B, A);
    if (rc != ALQ_OK) return rc;
    std::vector<unsigned int> mt_h(kMtN + 1);
    std::copy(D->mt_key_host, D->mt_key_host + kMtN, mt_h.begin());
    mt_h[kMtN] = static_cast<unsigned int>(*D->mt_pos_host);
    ALQ_CUDA(ctx, cudaMemcpyAsync(mt, mt_h.data(), (kMtN + 1) * 4, cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(avail, D->avail, static_cast<size_t>(n), cudaMemcpyDeviceToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(small, 0, 4 * sizeof(int), st));

    // ---- the LL words: a single GPU keeps them in scratch; a sharded call uses the group's window, bumps the epoch and,
    // after the clear in stream order, stores its ready word into every peer's window ---------------------------------
    LLWords& W = A.W;
    W.keyw = static_cast<unsigned int>(B.sharded ? kWordsHead : 0);
    W.pickw = static_cast<unsigned int>(up128(W.keyw + static_cast<size_t>(2) * nseg * 8));
    W.tag_base = 0x80000000u;
    if (!B.sharded) {
        W.peer[0] = word_scratch;
        ALQ_CUDA(ctx, cudaMemsetAsync(word_scratch, 0, words, st));
    } else {
        // the words start without a valid tag; peers write them only after our ready word, which follows the clear
        ALQ_CUDA(ctx, cudaMemsetAsync(ctx->comm.window + kWordsHead, 0, words - kWordsHead, st));
        for (int r = 0; r < S.world; ++r) W.peer[r] = ctx->comm.peer[r];
        ctx->comm.epoch += 1;
        W.ready_tag = ctx->comm.epoch << 32;
        W.tag_base |= static_cast<unsigned int>(ctx->comm.epoch & 0x7fu) << 24;
        rc = alq_comm_ready(ctx, W.ready_tag, st);
        if (rc != ALQ_OK) return rc;
    }

    // ---- the loop ---------------------------------------------------------------------------------------------------
    A.x = D->x; A.ldx = D->ldx; A.d = d;
    A.labels = D->labels; A.avail = avail;
    A.counts0 = B.counts; A.seg_avail0 = B.seg_avail;
    A.mt_in = mt; A.mt_out = mt + kMtN + 1;
    A.picks = D->picks; A.n_bal = small + 1; A.status = small;
    A.S = S;
    A.n = n; A.c = c; A.budget = B.budget; A.n_avail = static_cast<int>(B.n_avail);
    A.timeout_cycles = ctx->spin_timeout_cycles();
    ALQ_CUDA(ctx, cudaFuncSetAttribute(K::kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(k.smem)));
    // every CTA spins on the others' words, so all of them must be resident: grid <= SMs, one CTA per SM at most
    // (see alq_score.cu on why this is an ordinary launch)
    const cudaError_t le = alq_gridsync_launch(ctx, st, [&] {
        K::kernel<<<S.grid, K::kThreads, k.smem, st>>>(A);
        return cudaGetLastError();
    });
    if (le != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "%s: launch failed: %s (grid %d, %zu B shared)", fn, cudaGetErrorString(le), S.grid, k.smem);

    int small_h[2] = {0, 0};
    ALQ_CUDA(ctx, cudaMemcpyAsync(small_h, small, sizeof(small_h), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(mt_h.data(), A.mt_out, (kMtN + 1) * 4, cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (small_h[0] != 0) ALQ_FAIL(ctx, small_h[0], "%s: timed out waiting for a peer GPU or a CTA of the grid", fn);
    std::copy(mt_h.begin(), mt_h.begin() + kMtN, D->mt_key_host);
    *D->mt_pos_host = static_cast<int32_t>(mt_h[kMtN]);
    *D->n_picks_host = B.budget;
    *D->n_balancing_host = small_h[1];
    return ALQ_OK;
}

}  // namespace

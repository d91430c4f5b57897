// Shared by K11 (alq_balancing.cu) and K12 (alq_balancing_table.cu): the CTA segments, the fp32 imbalance test, the class
// denominators, NumPy's MT19937 and the host set-up steps of BalancingSampler's persistent query.
#pragma once
#include "alq_greedy.cuh"

// The rows of a call and who streams them.  Rank r owns rows [off[r], off[r + 1]) and runs `grid` CTAs on them; global
// segment g = r * grid + b, CTA b of rank r, starts at off[r] + seg_lo(off[r + 1] - off[r], grid, b).  A single GPU is
// world 1, rank 0, off = {0, n}: segment b starts at seg_lo(n, grid, b).  Every array stays global and replicated, so
// every rank derives the same world * grid segments.
struct BalShard {
    int world, rank, grid;
    int off[ALQ_MAX_WORLD + 1];
};

// Where the LL words of a call live.  peer[r] is rank r's window (a single GPU: peer[0] is scratch of this call); every
// window has the same layout: u64 ready[ALQ_MAX_WORLD] (sharded calls), the key words [2 parities][world * grid] at
// `keyw` and one pick word per step at `pickw`.  Tags carry the call's epoch (0 on a single GPU).
struct BalWords {
    char* peer[ALQ_MAX_WORLD];
    unsigned int keyw, pickw;
    unsigned int tag_base;               // 0x80000000 | (epoch & 0x7f) << 24: never 0, a zeroed word is invalid
    unsigned long long ready_tag;        // sharded: epoch << 32, stored into every peer's ready[rank]; 0: no handshake
};

namespace {

constexpr int kMtN = 624;
constexpr int kSegRowsMax = 65535;               // the key word carries a 16-bit row offset (0xffff: empty segment)
constexpr unsigned int kEmptyOff = 0xffffu;

__host__ __device__ __forceinline__ int seg_lo(int n, int grid, int b) {
    return static_cast<int>(static_cast<long long>(n) * b / grid);
}

__host__ __device__ __forceinline__ int gseg_lo(const BalShard& S, int g) {
    const int r = g / S.grid;
    if (r >= S.world) return S.off[S.world];
    return S.off[r] + seg_lo(S.off[r + 1] - S.off[r], S.grid, g - r * S.grid);
}
// the global segment holding `row` (0 <= row < off[world])
__device__ __forceinline__ int gseg_of(const BalShard& S, int row) {
    int r = 0;
    while (r + 1 < S.world && S.off[r + 1] <= row) ++r;
    const int grid = S.grid, rows = S.off[r + 1] - S.off[r], p = row - S.off[r];
    int o = static_cast<int>(static_cast<long long>(p) * grid / rows);
    while (o + 1 < grid && seg_lo(rows, grid, o + 1) <= p) ++o;
    while (o > 0 && seg_lo(rows, grid, o) > p) --o;
    return r * grid + o;
}

__device__ __forceinline__ unsigned int bal_key_tag(const BalWords& W, unsigned int round) {
    return 0x8000u | ((W.tag_base >> 12) & 0x7000u) | (round & 0xfffu);
}
__device__ __forceinline__ unsigned int bal_pick_tag(const BalWords& W, int t) {   // t < 2^24: the budget limit
    return W.tag_base | static_cast<unsigned int>(t);
}

// Sharded calls: no CTA stores into a peer's window before that peer has cleared it for this call (its ready word).
// Called by every thread; ends with a barrier.
template <typename Args>
__device__ __forceinline__ void bal_ready_wait(const Args& A, int tid) {
    if (A.W.ready_tag != 0 && tid < A.S.world) {
        const unsigned long long* rw = reinterpret_cast<const unsigned long long*>(A.W.peer[A.S.rank]) + tid;
        for (const long long t0 = clock64(); ld_acquire_sys(rw) != A.W.ready_tag;) {
            if (clock64() - t0 > A.timeout_cycles) { atomicCAS(A.status, 0, ALQ_ERR_STATE); break; }
            __nanosleep(200);
        }
    }
    __syncthreads();
}

// A balancing step's agreement.  s_key[0 .. kWarps) holds each warp's smallest key (ord(ratio) << 32 | row, ~0: none)
// and a barrier has passed.  The CTA's minimum goes as one word {tag16, row offset16, ord32} into slot rank * grid + b
// of every rank's window; every CTA gathers all world * grid words and returns the smallest key's row (-1: none, or a
// failed wait) to every thread.  Not inlined: K12's loop sits at the 128-register cap of its launch bounds, and the
// exchange inlined into it spills.
template <int kWarps, typename Args>
__device__ __noinline__ int bal_agree(const Args& A, unsigned long long* s_key, int* s_pick, unsigned int round,
                                         int row_lo, int tid) {
    const BalShard& S = A.S;
    const int nseg = S.world * S.grid, lane = tid & 31, warp = tid >> 5;
    const unsigned int tag16 = bal_key_tag(A.W, round);
    const size_t keyw = A.W.keyw + static_cast<size_t>(round & 1u) * nseg * 8;
    if (tid < S.world) {
        unsigned long long m = s_key[0];
        for (int w = 1; w < kWarps; ++w) m = s_key[w] < m ? s_key[w] : m;
        const unsigned long long off = m == ~0ull ? kEmptyOff : static_cast<unsigned long long>(static_cast<uint32_t>(m) - row_lo);
        ll_store_raw(A.W.peer[tid] + keyw + static_cast<size_t>(S.rank * S.grid + blockIdx.x) * 8,
                     (static_cast<unsigned long long>(tag16) << 48) | (off << 32) | (m >> 32));
    }
    unsigned long long mine = ~0ull;
    ll_gather(A.W.peer[S.rank] + keyw, nseg, 8, tag16, 48, A, tid, [&](int i, unsigned long long w) {
        const unsigned int off = static_cast<unsigned int>(w >> 32) & 0xffffu;
        if (off == kEmptyOff) return;
        const unsigned long long key = ((w & 0xffffffffull) << 32) | static_cast<uint32_t>(gseg_lo(S, i) + static_cast<int>(off));
        mine = key < mine ? key : mine;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, mine, o);
        mine = w < mine ? w : mine;
    }
    __syncthreads();                                              // s_key is reused
    if (lane == 0) s_key[warp] = mine;
    __syncthreads();
    if (tid == 0) {
        unsigned long long m = s_key[0];
        for (int w = 1; w < kWarps; ++w) m = s_key[w] < m ? s_key[w] : m;
        *s_pick = m == ~0ull ? -1 : static_cast<int>(static_cast<uint32_t>(m));
    }
    __syncthreads();
    return *s_pick;
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

}  // namespace

// ---- host set-up steps (alq_balancing.cu) ---------------------------------------------------------------------------
// The descriptor checks of both entry points (messages start with `fn`); on success *n_picks_host = -1 and
// *n_balancing_host = 0, so an early return declines.  A descriptor that ends before shard_off_host is accepted.
int alq_bal_check_desc(alq_ctx* ctx, const alq_balancing_desc* D, const char* fn);
// The call's layout (S->grid is set from the smallest shard, the same on every rank) and whether it is sharded: the
// descriptor carries shard_off_host.  A sharded call needs the group of alq_comm_create/connect and shard offsets that
// start at 0, do not decrease and end at n.
int alq_bal_shard(alq_ctx* ctx, const alq_balancing_desc* D, int n, BalShard* S, bool* sharded, const char* fn);
// Rows of the largest global segment (the key word carries a 16-bit offset).
int alq_bal_seg_rows_max(const BalShard& S);
// Bytes of the LL words (from the window's start); sharded calls need them inside the window's greedy region.
size_t alq_bal_words_bytes(const BalShard& S, int64_t budget, bool sharded);
// Clears the words for this call and fills W.  A single GPU keeps them in `scratch` (alq_bal_words_bytes of it).  A
// sharded call uses the group's window: it bumps the epoch and, after the clear in stream order, stores its ready word
// into every peer's window.
int alq_bal_words_begin(alq_ctx* ctx, const BalShard& S, bool sharded, int budget, char* scratch, BalWords* W, cudaStream_t st);
// K10's table pass over the labeled rows (counts[c]) and one launch counting the available rows of every global segment
// (seg_avail[world * grid]); both come back to counts_h / seg_h.  A labeled or available row whose label is outside
// [0, c) fails with ALQ_ERR_INVALID naming the row and its label.  Synchronises `st`.
int alq_bal_counts(alq_ctx* ctx, const alq_balancing_desc* D, int n, int c, const BalShard& S, int32_t* tab, unsigned int* bad,
                   int32_t* counts, int32_t* seg_avail, int32_t* counts_h, int32_t* seg_h, cudaStream_t st, const char* fn);

// Shared by K11 (alq_balancing.cu) and K12 (alq_balancing_table.cu): the CTA segments, the fp32 imbalance test, the class
// denominators, NumPy's MT19937 and the host set-up steps of BalancingSampler's persistent query.
#pragma once
#include "alq_greedy.cuh"

namespace {

constexpr int kMtN = 624;
constexpr int kSegRowsMax = 65535;               // the key word carries a 16-bit row offset (0xffff: empty segment)
constexpr unsigned int kEmptyOff = 0xffffu;

__host__ __device__ __forceinline__ int seg_lo(int n, int grid, int b) {
    return static_cast<int>(static_cast<long long>(n) * b / grid);
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
// *n_balancing_host = 0, so an early return declines.
int alq_bal_check_desc(alq_ctx* ctx, const alq_balancing_desc* D, const char* fn);
// K10's table pass over the labeled rows (counts[c]) and one launch counting the available rows of every CTA segment
// (seg_avail[grid]); both come back to counts_h / seg_h.  A labeled or available row whose label is outside [0, c) fails
// with ALQ_ERR_INVALID naming the row and its label.  Synchronises `st`.
int alq_bal_counts(alq_ctx* ctx, const alq_balancing_desc* D, int n, int c, int grid, int32_t* tab, unsigned int* bad,
                   int32_t* counts, int32_t* seg_avail, int32_t* counts_h, int32_t* seg_h, cudaStream_t st, const char* fn);

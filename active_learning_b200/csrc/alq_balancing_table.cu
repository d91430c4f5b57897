// K12: the whole query of BalancingSampler (balancing_sampler.py:58-134) as one persistent launch at class counts whose
// centres do not fit K11's shared memory (ImageNet-LT: 1 000 classes of 2 048 dimensions).
//
// K11 keeps every class centre in each CTA's shared memory and contracts every row against 1 + C_maj centres per
// balancing step.  K12 keeps instead a row x class table in device memory, T[i, c] = <x_i, S_c> in fp64 (S_c: the fp64
// class sum), plus xn64_i = <x_i, x_i>, so a balancing step reads 8 bytes per (row, selected class) and the distance is
//     d2(i, c) = xn64_i - 2 T[i, c] / den_c + q_c / den_c^2,   den_c = fl32(n_c + 1e-5),  q_c = <S_c, S_c>  (fp64),
// i.e. |x_i - m_c|^2 for the unrounded centre m_c = S_c / den_c.  Everything else is K11's: the branch test, the
// numerator 1, NumPy's draws, the tie rule and the LL-word agreement.
//   set-up   K10's table pass and the segment count (with the label checks, as for K11); one launch groups the
//            labeled rows by class in row order; one launch per class sums them in that order (fp64) and forms q_c;
//   loop     ONE ordinary launch, one CTA per SM (bracketed by alq_gridsync_begin/end, every wait bounded by
//            "spin_timeout_ms").  Every CTA keeps the counts, den, q, the majority list, the per-segment available
//            counts and the MT19937 state in shared memory and its own fp64 copy of the sums ([d][c]) in scratch, and
//            updates them identically after every pick.
//              first balancing step: every CTA lists the available rows of its segment (its table slots) and builds
//                              their table rows from its sums; a query that never balances never builds;
//              after a pick p of class y every available row needs T[i, y] += <x_i, x_p>: the pick's row joins the
//                              CTA's pending list (shared memory, at most pend_cap rows);
//              balancing step: each CTA streams its rows once, applies the pending dot products in pick order, scores
//                              the row against the rarest and majority columns and publishes its best key;
//              random step:    K11's draw; if the pending list is full, the CTA first flushes it over its own rows
//                              (no exchange: a CTA only writes its own rows' table entries).
// Fixed orders, independent of the grid: a table entry is an fp64 fma chain over d ascending; a pending dot product is a
// sum of exact fp32 x fp32 products, lane l taking the float4 chunks l, l + 32, .. in x, y, z, w order, folded by a
// butterfly; S_c sums the class's rows in row order; q_c is a per-thread fma chain (dimensions tid, tid + 512, ..)
// folded by a butterfly and the 16 warp partials in order.  So the picks are bit-reproducible.
// The host side of a call is bal_select (alq_balancing.cuh), shared with K11; this file supplies K12's part of it
// (TabLoop: the pending list's shared-memory plan, the device-memory limit, the table's scratch and set-up launches).
#include "alq_balancing.cuh"

namespace {

constexpr int kTabThreads = 512;                 // >= kPollers: every poller of ll_gather is a thread of the CTA
constexpr int kTabWarps = kTabThreads / 32;
constexpr int kPendMax = 64;                     // pending picks a CTA holds at most
constexpr int kPendPerPass = 4;                  // pending dot products a lane accumulates at once
constexpr int kBuildRows = 32;                   // table rows a thread accumulates at once in the build
constexpr int kBuildDims = 128;                  // dimensions per shared-memory stage of the build
constexpr int kBuildLd = kBuildRows + 1;         // padded stage row (doubles)
constexpr size_t kBuildBytes = static_cast<size_t>(kBuildDims) * kBuildLd * sizeof(double);
constexpr int kGroupThreads = 1024;

struct TabArgs {
    const float* x; long long ldx; int d;
    const int* labels;
    uint8_t* avail;              // working copy of the caller's mask
    const double* sums0;         // [d][c] fp64 class sums of the labeled rows
    const double* q0;            // [c] <S_c, S_c>
    double* sums;                // [grid][d][c] every CTA's running copy
    double* table;               // [n_slots][c]
    double* xn64;                // [n_slots]
    int* slot_row;               // [n_slots] the row of every table slot
    const int* slot_lo;          // [grid]: CTA b owns the slots slot_lo[b] ..
    const int* counts0;          // [c]
    const int* seg_avail0;       // [world * grid]
    const unsigned int* mt_in;   // [kMtN + 1]: key, pos
    unsigned int* mt_out;        // [kMtN + 1]
    int* picks;
    int* n_bal;
    int* status;
    SegShard S;
    LLWords W;                   // key words of the balancing steps (two parities), one pick word per random step
    int n, c, budget, n_avail, pend_cap;
    long long timeout_cycles;
};

__device__ __forceinline__ double warp_sum64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// 0.0 + warp 0's butterfly sum + warp 1's + ..; returned to every thread.  red: kTabWarps doubles of shared memory.
__device__ __forceinline__ double block_sum64(double v, double* red) {
    v = warp_sum64(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kTabWarps; ++w) s += red[w];
    __syncthreads();
    return s;
}

__device__ __forceinline__ double dist_tab(double xn, double t, float den, double q) {
    const double dd = static_cast<double>(den);
    return __dadd_rn(__dsub_rn(xn, __ddiv_rn(2.0 * t, dd)), __ddiv_rn(q, __dmul_rn(dd, dd)));
}

// grp[off[k] ..] = the labeled rows of class k in row order (labels already checked).  One CTA: per chunk of rows the
// warps take their turn at the per-class cursors, and lanes of one class within a warp are ranked by lane.
__global__ void __launch_bounds__(kGroupThreads) bal_table_group_kernel(const int* __restrict__ labels,
                                                                        const uint8_t* __restrict__ labeled, int n, int c,
                                                                        const int* __restrict__ off, int* __restrict__ grp) {
    extern __shared__ int cursor[];              // [c]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < c; i += kGroupThreads) cursor[i] = off[i];
    __syncthreads();
    for (int r0 = 0; r0 < n; r0 += kGroupThreads) {
        const int row = r0 + tid;
        const int y = (row < n && labeled[row]) ? labels[row] : -1;
        const bool ok = static_cast<unsigned>(y) < static_cast<unsigned>(c);
        if (!__syncthreads_or(ok)) continue;
        const unsigned peers = __match_any_sync(0xffffffffu, ok ? y : -1);
        const int leader = __ffs(peers) - 1;
        const int rank = __popc(peers & ((1u << lane) - 1u));
        for (int w = 0; w < kGroupThreads / 32; ++w) {
            if (warp == w) {
                int base = 0;
                if (ok && lane == leader) {
                    base = cursor[y];
                    cursor[y] = base + __popc(peers);
                }
                base = __shfl_sync(0xffffffffu, base, leader);
                if (ok) grp[base + rank] = row;
            }
            __syncthreads();
        }
    }
}

// sums0[j][k] = 0.0 + x[r0, j] + x[r1, j] + .. over the labeled rows r0 < r1 < .. of class k, and q0[k] = <S_k, S_k>
// in the loop's order (thread tid: dimensions tid, tid + 512, .., then block_sum64).  One CTA per class.
__global__ void __launch_bounds__(kTabThreads) bal_table_class_sum_kernel(const float* __restrict__ x, long long ldx, int d,
                                                                          int c, const int* __restrict__ off,
                                                                          const int* __restrict__ grp,
                                                                          double* __restrict__ sums0, double* __restrict__ q0) {
    __shared__ double red[kTabWarps];
    const int k = blockIdx.x;
    const int lo = off[k], hi = off[k + 1];
    double sq = 0.0;
    for (int j = threadIdx.x; j < d; j += kTabThreads) {
        double s = 0.0;
        for (int q = lo; q < hi; ++q) s += static_cast<double>(__ldg(x + static_cast<long long>(grp[q]) * ldx + j));
        sums0[static_cast<size_t>(j) * c + k] = s;
        sq = fma(s, s, sq);
    }
    const double t = block_sum64(sq, red);
    if (threadIdx.x == 0) q0[k] = t;
}

__host__ __device__ __forceinline__ size_t bal_table_region(int pend_cap, int d) {
    const size_t pend = static_cast<size_t>(pend_cap) * d * 4;
    return pend > kBuildBytes ? pend : kBuildBytes;
}
__host__ __device__ __forceinline__ size_t bal_table_smem(int c, int d, int nseg, int pend_cap) {
    return bal_table_region(pend_cap, d) + static_cast<size_t>(c) * 20 + static_cast<size_t>(nseg) * 4 +
           static_cast<size_t>(pend_cap) * 4 + kMtN * 4 + 64;
}

__global__ void __launch_bounds__(kTabThreads, 1) balancing_table_kernel(const __grid_constant__ TabArgs A) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int c = A.c, d = A.d, dv = d >> 2, nseg = A.S.world * A.S.grid, pend_cap = A.pend_cap;
    float* pend_x = reinterpret_cast<float*>(smem_raw);                               // [pend_cap][d] (the build's stage)
    double* stage = reinterpret_cast<double*>(smem_raw);                              // [kBuildDims][kBuildLd]
    double* q = reinterpret_cast<double*>(smem_raw + bal_table_region(pend_cap, d));  // [c]
    int* cnt = reinterpret_cast<int*>(q + c);                                         // [c]
    float* den = reinterpret_cast<float*>(cnt + c);                                   // [c]
    int* sel = reinterpret_cast<int*>(den + c);                                       // [c]
    int* seg_av = sel + c;                                                            // [nseg]
    int* pend_y = seg_av + nseg;                                                      // [pend_cap]
    unsigned int* mt = reinterpret_cast<unsigned int*>(pend_y + pend_cap);            // [kMtN]
    __shared__ unsigned long long s_key[kTabWarps];
    __shared__ int s_wc[kTabWarps], s_red[5 * kTabWarps];
    __shared__ double s_dred[kTabWarps];
    __shared__ int s_pick, s_owner, s_rank, s_found, s_mtpos, s_navail;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x;
    const int gb = A.S.rank * A.S.grid + b;                                           // my global segment
    const int row_lo = gseg_lo(A.S, gb), row_hi = gseg_lo(A.S, gb + 1);
    const int slo = A.slot_lo[b];
    double* my_sums = A.sums + static_cast<size_t>(b) * c * d;

    for (int i = tid; i < c; i += kTabThreads) {
        const int k = A.counts0[i];
        cnt[i] = k;
        den[i] = bal_den(k);
        q[i] = A.q0[i];
    }
    for (int i = tid; i < nseg; i += kTabThreads) seg_av[i] = A.seg_avail0[i];
    for (int i = tid; i < kMtN; i += kTabThreads) mt[i] = A.mt_in[i];
    if (tid == 0) { s_mtpos = static_cast<int>(A.mt_in[kMtN]); s_navail = A.n_avail; }
    for (size_t i = tid; i < static_cast<size_t>(c) * d; i += kTabThreads) my_sums[i] = A.sums0[i];
    if (A.W.ready_tag != 0 && tid < A.S.world) ll_ready_wait(A.W.peer[A.S.rank], tid, A.W.ready_tag, A);
    __syncthreads();

    // the table rows of my slots, streamed once per balancing step: apply the pending picks (in pick order) and,
    // when `score`, return the warp's smallest key (ord(fl32(near / far) + 0) << 32 | row)
    int nslot = 0, npend = 0;
    auto pass = [&](bool score, int nsel) -> unsigned long long {
        unsigned long long best = ~0ull;
        const int rare = sel[0];
        const bool near1 = cnt[rare] == 0;                                // :106-109: numerator 1
        for (int s = slo + warp; s < slo + nslot; s += kTabWarps) {
            const int row = A.slot_row[s];
            if (!A.avail[row]) continue;                                  // warp-uniform
            const float4* xr = reinterpret_cast<const float4*>(A.x + static_cast<long long>(row) * A.ldx);
            double* trow = A.table + static_cast<size_t>(s) * c;
            for (int p0 = 0; p0 < npend; p0 += kPendPerPass) {
                const int pn = min(kPendPerPass, npend - p0);
                double acc[kPendPerPass];
#pragma unroll
                for (int j = 0; j < kPendPerPass; ++j) acc[j] = 0.0;
                for (int k = lane; k < dv; k += 32) {
                    const float4 v = __ldg(xr + k);
#pragma unroll
                    for (int j = 0; j < kPendPerPass; ++j)
                        if (j < pn) {
                            const float4 w = reinterpret_cast<const float4*>(pend_x + static_cast<size_t>(p0 + j) * d)[k];
                            acc[j] = fma(static_cast<double>(v.x), static_cast<double>(w.x), acc[j]);
                            acc[j] = fma(static_cast<double>(v.y), static_cast<double>(w.y), acc[j]);
                            acc[j] = fma(static_cast<double>(v.z), static_cast<double>(w.z), acc[j]);
                            acc[j] = fma(static_cast<double>(v.w), static_cast<double>(w.w), acc[j]);
                        }
                }
#pragma unroll
                for (int j = 0; j < kPendPerPass; ++j)
                    if (j < pn) {
                        const double dot = warp_sum64(acc[j]);
                        if (lane == 0) trow[pend_y[p0 + j]] += dot;
                    }
            }
            if (!score) continue;
            __syncwarp();                                                 // lane 0's table updates, seen by the warp
            const double xn = A.xn64[s];
            const double near = near1 ? 1.0 : dist_tab(xn, trow[rare], den[rare], q[rare]);
            double far = -__longlong_as_double(0x7ff0000000000000ll);
            for (int j = 1 + lane; j < nsel; j += 32) {
                const int k = sel[j];
                far = fmax(far, dist_tab(xn, trow[k], den[k], q[k]));
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) far = fmax(far, __shfl_xor_sync(0xffffffffu, far, o));
            const float ratio = __double2float_rn(near / far);
            const unsigned long long key = (static_cast<unsigned long long>(alq_ord(ratio + 0.0f)) << 32) | static_cast<uint32_t>(row);
            best = key < best ? key : best;
        }
        return best;
    };

    unsigned int rnd_key = 0;
    int n_bal = 0;
    bool built = false;
    for (int t = 0; t < A.budget; ++t) {
        // ===== the imbalance test (balancing_sampler.py:66-84): K11's, from block reductions of the exact tallies =====
        int nsel = 0;
        {
            int tot = 0;
            unsigned int mn = UINT_MAX;
            for (int i = tid; i < c; i += kTabThreads) { tot += cnt[i]; mn = min(mn, static_cast<unsigned int>(cnt[i])); }
            tot = __reduce_add_sync(0xffffffffu, tot);
            mn = __reduce_min_sync(0xffffffffu, mn);
            if (lane == 0) { s_red[warp] = tot; s_red[kTabWarps + warp] = static_cast<int>(mn); }
            __syncthreads();
            int total = 0;
            unsigned int mincnt = UINT_MAX;
#pragma unroll
            for (int w = 0; w < kTabWarps; ++w) { total += s_red[w]; mincnt = min(mincnt, static_cast<unsigned int>(s_red[kTabWarps + w])); }
            const float mean = bal_mean(total, c);
            unsigned int first = UINT_MAX;
            int na = 0, sa = 0;
            for (int i = tid; i < c; i += kTabThreads) {
                if (static_cast<unsigned int>(cnt[i]) == mincnt) first = min(first, static_cast<unsigned int>(i));
                if (static_cast<float>(cnt[i]) > mean) { ++na; sa += cnt[i]; }
            }
            first = __reduce_min_sync(0xffffffffu, first);
            na = __reduce_add_sync(0xffffffffu, na);
            sa = __reduce_add_sync(0xffffffffu, sa);
            if (lane == 0) { s_red[2 * kTabWarps + warp] = static_cast<int>(first); s_red[3 * kTabWarps + warp] = na; s_red[4 * kTabWarps + warp] = sa; }
            __syncthreads();
            unsigned int rare = UINT_MAX;
            int nat = 0, sat = 0;
#pragma unroll
            for (int w = 0; w < kTabWarps; ++w) {
                rare = min(rare, static_cast<unsigned int>(s_red[2 * kTabWarps + w]));
                nat += s_red[3 * kTabWarps + w];
                sat += s_red[4 * kTabWarps + w];
            }
            if (bal_balances(A.budget - t, nat, sat, c - nat, total - sat)) {   // block-uniform
                // sel[0] = the rarest class, sel[1..] = the majority classes ascending (block scan)
                if (tid == 0) sel[0] = static_cast<int>(rare);
                nsel = 1;
                for (int i0 = 0; i0 < c; i0 += kTabThreads) {
                    const int i = i0 + tid;
                    const bool f = i < c && static_cast<float>(cnt[i]) > mean;
                    const unsigned bal = __ballot_sync(0xffffffffu, f);
                    if (lane == 0) s_wc[warp] = __popc(bal);
                    __syncthreads();
                    int before = 0, tt = 0;
#pragma unroll
                    for (int w = 0; w < kTabWarps; ++w) {
                        if (w < warp) before += s_wc[w];
                        tt += s_wc[w];
                    }
                    if (f) sel[nsel + before + __popc(bal & ((1u << lane) - 1u))] = i;
                    nsel += tt;
                    __syncthreads();
                }
            }
        }
        if (nsel > 0) {
            // ===== balancing step (balancing_sampler.py:85-125) =====
            ++n_bal;
            if (!built) {
                // my slots: the available rows of my segment in row order
                int base = 0;
                for (int r0 = row_lo; r0 < row_hi; r0 += kTabThreads) {
                    const int row = r0 + tid;
                    const bool av = row < row_hi && A.avail[row];
                    const unsigned bal = __ballot_sync(0xffffffffu, av);
                    if (lane == 0) s_wc[warp] = __popc(bal);
                    __syncthreads();
                    int before = 0, tot = 0;
#pragma unroll
                    for (int w = 0; w < kTabWarps; ++w) {
                        if (w < warp) before += s_wc[w];
                        tot += s_wc[w];
                    }
                    if (av) A.slot_row[slo + base + before + __popc(bal & ((1u << lane) - 1u))] = row;
                    base += tot;
                    __syncthreads();
                }
                nslot = base;
                __syncthreads();                                          // slot_row written by the CTA, read below
                // T[s, k] = fma chain over j ascending of x[row_s, j] * S_k[j]: thread k, kBuildRows slots at a time
                for (int s0 = 0; s0 < nslot; s0 += kBuildRows) {
                    const int rn = min(kBuildRows, nslot - s0);
                    for (int c0 = 0; c0 < c; c0 += kTabThreads) {
                        const int k = c0 + tid;
                        double acc[kBuildRows];
#pragma unroll
                        for (int r = 0; r < kBuildRows; ++r) acc[r] = 0.0;
                        for (int j0 = 0; j0 < d; j0 += kBuildDims) {
                            const int jn = min(kBuildDims, d - j0);
                            __syncthreads();
                            for (int i = tid; i < kBuildRows * kBuildDims; i += kTabThreads) {
                                const int r = i / kBuildDims, jj = i % kBuildDims;
                                stage[jj * kBuildLd + r] = (r < rn && jj < jn)
                                    ? static_cast<double>(__ldg(A.x + static_cast<long long>(A.slot_row[slo + s0 + r]) * A.ldx + j0 + jj))
                                    : 0.0;
                            }
                            __syncthreads();
                            if (k < c)
                                for (int jj = 0; jj < jn; ++jj) {
                                    const double sv = my_sums[static_cast<size_t>(j0 + jj) * c + k];
#pragma unroll
                                    for (int r = 0; r < kBuildRows; ++r) acc[r] = fma(stage[jj * kBuildLd + r], sv, acc[r]);
                                }
                        }
                        if (k < c)
#pragma unroll
                            for (int r = 0; r < kBuildRows; ++r)
                                if (r < rn) A.table[static_cast<size_t>(slo + s0 + r) * c + k] = acc[r];
                    }
                }
                // xn64: the pending dot product's fixed order
                for (int s = slo + warp; s < slo + nslot; s += kTabWarps) {
                    const float4* xr = reinterpret_cast<const float4*>(A.x + static_cast<long long>(A.slot_row[s]) * A.ldx);
                    double acc = 0.0;
                    for (int k = lane; k < dv; k += 32) {
                        const float4 v = __ldg(xr + k);
                        acc = fma(static_cast<double>(v.x), static_cast<double>(v.x), acc);
                        acc = fma(static_cast<double>(v.y), static_cast<double>(v.y), acc);
                        acc = fma(static_cast<double>(v.z), static_cast<double>(v.z), acc);
                        acc = fma(static_cast<double>(v.w), static_cast<double>(v.w), acc);
                    }
                    acc = warp_sum64(acc);
                    if (lane == 0) A.xn64[s] = acc;
                }
                __syncthreads();                                          // the stage is the pending list's memory
                built = true;
                npend = 0;
            }
            const unsigned long long best = pass(true, nsel);
            npend = 0;
            if (lane == 0) s_key[warp] = best;
            __syncthreads();
            ll_agree_min_call<kTabWarps>(A, s_key, &s_pick, ++rnd_key, row_lo, tid);
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
                for (int r0 = row_lo; r0 < row_hi; r0 += kTabThreads) {
                    const int row = r0 + tid;
                    const bool av = row < row_hi && A.avail[row];
                    const unsigned bal = __ballot_sync(0xffffffffu, av);
                    if (lane == 0) s_wc[warp] = __popc(bal);
                    __syncthreads();
                    int before = 0, tot = 0;
#pragma unroll
                    for (int w = 0; w < kTabWarps; ++w) {
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
        if (built && npend == pend_cap) {                                 // the pick would overflow the pending list
            pass(false, 0);
            npend = 0;
            __syncthreads();                                              // pend_x is rewritten below
        }
        const int cls = __ldg(A.labels + pick);
        const int newc = cnt[cls] + 1;
        const int o = gseg_of(A.S, pick);
        __syncthreads();                                                 // cnt[cls] read by every thread
        if (tid == 0) {
            cnt[cls] = newc;
            den[cls] = bal_den(newc);
            seg_av[o] -= 1;
            s_navail -= 1;
            if (o == gb) A.avail[pick] = 0;
            if (b == 0) A.picks[t] = pick;
            if (built) pend_y[npend] = cls;
        }
        const float* xp = A.x + static_cast<long long>(pick) * A.ldx;
        float* px = pend_x + static_cast<size_t>(npend) * d;
        double sq = 0.0;
        for (int j = tid; j < d; j += kTabThreads) {
            const float v = __ldg(xp + j);
            double* sj = my_sums + static_cast<size_t>(j) * c + cls;
            const double s = *sj + static_cast<double>(v);
            *sj = s;
            sq = fma(s, s, sq);
            if (built) px[j] = v;
        }
        const double qv = block_sum64(sq, s_dred);
        if (tid == 0) q[cls] = qv;
        if (built) ++npend;
        __syncthreads();
    }
    if (b == 0) {
        for (int i = tid; i < kMtN; i += kTabThreads) A.mt_out[i] = mt[i];
        if (tid == 0) { A.mt_out[kMtN] = static_cast<unsigned int>(s_mtpos); *A.n_bal = n_bal; }
    }
}

// K12's steps of bal_select
struct TabLoop {
    using Args = TabArgs;
    static constexpr const char* kName = "alq_balancing_table_select";
    static constexpr int kForce = 3;                 // balancing_loop = 3 forces K12; 1 and 2 make it decline
    static constexpr int kThreads = kTabThreads;
    static constexpr auto kernel = balancing_table_kernel;
    size_t smem = 0, group_smem = 0;
    int pend_cap = 0;

    int plan_smem(alq_ctx* ctx, BalCall& B) {
        const int c = B.c, d = B.d, nseg = B.nseg;
        const size_t smem_cap = B.smem_cap;
        const size_t fixed = bal_table_smem(c, d, nseg, 0) - kBuildBytes;
        pend_cap = fixed < smem_cap ? static_cast<int>(std::min<size_t>(kPendMax, (smem_cap - fixed) / (static_cast<size_t>(d) * 4 + 4))) : 0;
        while (pend_cap > 0 && bal_table_smem(c, d, nseg, pend_cap) > smem_cap) --pend_cap;
        group_smem = static_cast<size_t>(c) * 4;
        if (pend_cap < 1 || group_smem > smem_cap)
            BAL_LIMIT(B, "%s: the tables of %d classes and one pending row of %d floats need %zu bytes of shared memory, %zu "
                      "are available (limit: class tables in shared memory)", kName, c, d, bal_table_smem(c, d, nseg, 1), smem_cap);
        smem = bal_table_smem(c, d, nseg, pend_cap);
        return ALQ_OK;
    }
    // the table's rows are the available rows: sized after the counts
    size_t need_with_counts(const BalCall&) const { return 0; }
    // the table and the per-CTA sums must fit the device's free memory: checked before anything is reserved for them;
    // then the table slots, the fp64 class sums in row order per class and their squared norms
    int setup(alq_ctx* ctx, BalCall& B, ScratchCursor& cur, TabArgs& A) {
        const alq_balancing_desc* D = B.D;
        const SegShard& S = B.S;
        const cudaStream_t st = B.st;
        const int n = B.n, c = B.c, d = B.d, grid = S.grid, nseg = B.nseg;
        std::vector<int64_t> avail_of(S.world, 0);                    // available rows per rank: its table rows
        for (int g = 0; g < nseg; ++g) avail_of[g / grid] += B.seg_h[g];
        const size_t cd = static_cast<size_t>(c) * d;
        const size_t words_b = bal_words_bytes(S, B.budget, B.sharded);
        auto need_for = [&](size_t na) {
            return scratch_need({static_cast<size_t>(c) * 4, static_cast<size_t>(nseg) * 4, static_cast<size_t>(c + 1) * 4,
                                 static_cast<size_t>(grid) * 4, static_cast<size_t>(std::max<int64_t>(B.labeled_total, 1)) * 4,
                                 cd * 8, static_cast<size_t>(c) * 8, static_cast<size_t>(grid) * cd * 8, na * c * 8,
                                 na * 8, na * 4, static_cast<size_t>(n), (kMtN + 1) * 4 * 2, B.sharded ? 0 : words_b, 16});
        };
        const size_t na = static_cast<size_t>(avail_of[S.rank]);
        const size_t need = need_for(na);
        if (B.sharded) {
            // the same decision on every rank: every rank's share against the group's least free memory (the caller's
            // gather; this context's scratch is not counted, so the check is conservative)
            for (int r = 0; r < S.world; ++r) {
                const size_t nr = need_for(static_cast<size_t>(avail_of[r]));
                const size_t want = nr + (nr >> 2) + (1u << 20);            // what alq_scratch_reserve allocates
                if (D->group_free_bytes < 0 || want > static_cast<size_t>(D->group_free_bytes))
                    BAL_LIMIT(B, "%s: rank %d's %lld x %d table (%zu bytes) and %d copies of the class sums (%zu bytes) need "
                              "%zu bytes of device memory, the group has %lld free (limit: table in device memory)", kName, r,
                              (long long)avail_of[r], c, static_cast<size_t>(avail_of[r]) * c * 8, grid,
                              static_cast<size_t>(grid) * cd * 8, want, (long long)D->group_free_bytes);
            }
        } else if (need > ctx->scratch_bytes) {
            size_t free_b = 0, total_b = 0;
            ALQ_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
            const size_t want = need + (need >> 2) + (1u << 20);           // what alq_scratch_reserve allocates
            if (want > free_b + ctx->scratch_bytes)
                BAL_LIMIT(B, "%s: the %lld x %d table (%zu bytes) and %d copies of the class sums (%zu bytes) need %zu bytes "
                          "of device memory, %zu are free (limit: table in device memory)", kName, (long long)B.n_avail, c,
                          na * c * 8, grid, static_cast<size_t>(grid) * cd * 8, want, free_b + ctx->scratch_bytes);
        }
        const int rc = alq_scratch_reserve(ctx, need);
        if (rc != ALQ_OK) return rc;
        cur = ScratchCursor(ctx->scratch);                            // the counts move to the front of the new scratch
        B.counts = cur.take<int32_t>(c);
        B.seg_avail = cur.take<int32_t>(nseg);
        int32_t* off = cur.take<int32_t>(c + 1);
        int32_t* slot_lo = cur.take<int32_t>(grid);
        int32_t* grp = cur.take<int32_t>(static_cast<size_t>(std::max<int64_t>(B.labeled_total, 1)));
        double* sums0 = cur.take<double>(cd);
        double* q0 = cur.take<double>(c);
        A.sums0 = sums0; A.q0 = q0;
        A.sums = cur.take<double>(static_cast<size_t>(grid) * cd);
        A.table = cur.take<double>(na * c);
        A.xn64 = cur.take<double>(na);
        A.slot_row = cur.take<int32_t>(na);
        A.slot_lo = slot_lo;
        A.pend_cap = pend_cap;

        // table slots: the available rows of this rank's segments only
        std::vector<int32_t> off_h(c + 1), slot_lo_h(grid);
        off_h[0] = 0;
        for (int k = 0; k < c; ++k) off_h[k + 1] = off_h[k] + B.counts_h[k];
        for (int b = 0, s = 0; b < grid; ++b) { slot_lo_h[b] = s; s += B.seg_h[S.rank * grid + b]; }
        ALQ_CUDA(ctx, cudaMemcpyAsync(B.counts, B.counts_h.data(), static_cast<size_t>(c) * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(B.seg_avail, B.seg_h.data(), static_cast<size_t>(nseg) * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(off, off_h.data(), static_cast<size_t>(c + 1) * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(slot_lo, slot_lo_h.data(), static_cast<size_t>(grid) * 4, cudaMemcpyHostToDevice, st));

        if (group_smem > 48u * 1024u)
            ALQ_CUDA(ctx, cudaFuncSetAttribute(bal_table_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(group_smem)));
        bal_table_group_kernel<<<1, kGroupThreads, group_smem, st>>>(D->labels, D->labeled, n, c, off, grp);
        ALQ_LAUNCH_CHECK(ctx);
        bal_table_class_sum_kernel<<<c, kTabThreads, 0, st>>>(D->x, D->ldx, d, c, off, grp, sums0, q0);
        ALQ_LAUNCH_CHECK(ctx);
        return ALQ_OK;
    }
};

}  // namespace

extern "C" int alq_balancing_table_select(alq_ctx* ctx, const alq_balancing_desc* D, void* stream) {
    return bal_select<TabLoop>(ctx, D, stream);
}

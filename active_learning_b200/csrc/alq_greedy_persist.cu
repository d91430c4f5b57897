// K4 / K5 as ONE persistent cooperative launch: the whole B-step selection loop of
// `CoresetSampler.coreset` (coreset_sampler.py:66-105 under active_learning/src/query_strategies) runs
// inside one kernel, one CTA per SM, on one GPU or on G GPUs that talk through peer-memory windows.
//
// Why: a step is a 100-150 us HBM stream on one GPU but only 12-19 us on eight, and the rows a step
// streams do not depend on the centre -- only the dot products do.  So the TMA producer of every CTA
// runs free across step boundaries: while the grid (and the other GPUs) agree on the next centre, the
// bulk copies of the next step's first tiles are already landing in the shared-memory ring (~200 KB per
// SM, ~30 MB per GPU in flight), and HBM never idles across the exchange.  With one launch per step that
// window was spent on launch latency, the prologue and a flag chain.
//
// Agreement on the centre never moves a row: every rank holds a replica of the candidate rows (a few
// hundred MB next to 180 GB), so a pick is announced as a row id.  All cross-CTA / cross-GPU traffic is
// "LL" words: 8 bytes = {32-bit tag, 32-bit payload}, written with one plain store (single-copy atomic, so
// no fence and no separate flag: one NVLink one-way latency) and polled at the destination until the tag
// matches.  On one GPU the "window" is local scratch and the very same code runs.
//
//   arg-max (K4)   per CTA best key -> atomicMax + ticket; the last CTA of the rank pushes the rank's key
//                  to every rank; everybody polls `world` keys, the largest wins (lowest row on ties).
//   D^2 draw (K5)  NumPy-exact: (1) rank-local grid barrier; (2) leaves of NumPy's float32 pairwise-sum
//                  tree, one 8-lane group per leaf, pushed to every rank; every CTA folds the combine
//                  tree itself (shared memory) so all agree on S bit for bit; (3) fp64 mass of
//                  prob = clip(mind,0)/S per leaf, pushed; every CTA scans the leaf masses and locates the
//                  leaf holding u * total; (4) the CTA owning that leaf searches inside it and pushes the
//                  picked row id.  Shards are aligned to leaf boundaries, so no leaf needs a peer's rows.
#include "alq_greedy.cuh"

namespace {

constexpr int kMaxLeaves = 4096;          // per partition: 2*K floats + K words of shared memory
constexpr int kConsWarps = 11;          // + 1 producer warp = 12 warps = 3 per SM sub-partition: up to 168 registers per thread, no spills
constexpr int kConsThreads = kConsWarps * 32;
constexpr int kGroups = kConsThreads / 8; // 8-lane groups per CTA == leaves a CTA can own

struct PGroup {                 // one partition = one group of CTAs
    int cta_lo, ncta;
    int row_lo;                 // first row of the partition (pick reported after a numeric failure)
    int budget, pick_off;
    int first_pick;             // >= 0: centre 0 chosen by the caller (nothing labeled), else -1
    int full_n, cfull_off;
    int n_leaves, leaf_base;    // leaf_off[leaf_base .. leaf_base + n_leaves]
    int n_levels, level_base;   // level_off[level_base .. level_base + n_levels]
    int sched_base;             // sched[sched_base .. sched_base + n_leaves - 1): internal node j = (l | r << 16)
    int leaf_lo, leaf_hi;       // leaves summed by THIS rank
    int seg_base, seg_stride;   // segtab[seg_base + r * seg_stride + cta] = first row of CTA `cta` of rank r
    int ncta_base;              // ncta_of_rank[ncta_base + r] = CTAs rank r runs for this partition
    unsigned int keyw, leafw, massw, pickw, umw;   // byte offsets of the LL regions inside a window
};

struct PersistArgs {
    const float* x;  long long ldx; int d;
    const float* a;  long long lda; int c;
    const float* xn; const float* an;
    float* mind;
    const int* vpos;
    const BlockSeg* segs;
    const PGroup* groups;
    unsigned long long* valw;      // [sum full_n] LL word per position of the full array: this step's min-distance
    const int* posinv;
    const int* leaf_off;
    const int* level_off;
    const unsigned int* sched;
    const int* segtab;
    const int* ncta_of_rank;
    const double* uniforms;
    int* picks;
    int* status;
    unsigned long long* prof;      // [8] ns: streaming, selection, steps, then selection sub-phases
    int world, rank;
    char* peer[ALQ_MAX_WORLD];     // windows (one GPU without a group: peer[0] = local scratch)
    int leaf_bound[ALQ_MAX_WORLD + 1];   // multi-GPU D^2: rank r sums leaves [leaf_bound[r], leaf_bound[r+1])
    unsigned int ready_off;        // u64 ready[world] at the head of every window
    unsigned long long ready_tag;  // group path: epoch << 32, stored into every peer's ready[rank]; 0: no handshake
    unsigned int tag_base;         // 0x80000000 | (epoch & 0x7f) << 24
    int resident_rows;             // rows at the head of every CTA's segment fetched L2::evict_last (they stay in L2 across
                                   // steps; the rest is fetched evict_first).  0: no hints
    int fast_path;                 // D^2 draw: certified per-CTA-mass path first (0: always the exact NumPy-tree machinery)
    long long timeout_cycles;
};

// LL words (ll_store, ll_load, ll_wait, ll_gather): alq_ll.cuh

__device__ __forceinline__ void cons_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kConsThreads) : "memory"); }
__device__ __forceinline__ unsigned long long gtime_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// NumPy pairwise_sum leaf (n <= 128) from registers: lane g of an 8-lane group holds a[8j + g] in v[j].
//   r[g] = a[g]; r[g] += a[8i + g] for i = 1, 2, ..; ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7)); then the n % 8 tail
//   (n < 8: 0 + a[0] + a[1] + ..) added one by one.  prob = clip(min_dist, 0) (coreset_sampler.py:84).
__device__ __forceinline__ float leaf_sum_regs(const float (&v)[16], int len, int lane, unsigned gmask) {
    const int stop = len - (len & 7);
    float r = 0.f;
    if (stop > 0) {
        r = fmaxf(v[0], 0.f);
#pragma unroll
        for (int j = 1; j < 16; ++j)
            if (8 * j < stop) r += fmaxf(v[j], 0.f);
        r = r + __shfl_down_sync(gmask, r, 1, 8);
        r = r + __shfl_down_sync(gmask, r, 2, 8);
        r = r + __shfl_down_sync(gmask, r, 4, 8);
    }
    const int jt = stop >> 3;                 // row of the tail elements a[stop + i] = lane i's v[jt]
    float tv = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
        if (j == jt) tv = fmaxf(v[j], 0.f);
    const int g0 = lane & ~7;
    for (int i = 0; i < (len & 7); ++i) r += __shfl_sync(gmask, tv, g0 + i);   // meaningful in the group's lane 0
    return __shfl_sync(gmask, r, g0);
}

// First item i of [0, n) with mass(i) > 0 and (base0 + mass(0) + .. + mass(i)) / total > u_hi, found by the whole
// consumer block: idx (-1: none), base = the prefix before that item (base0 included), sum = mass(0) + .. + mass(n-1).
// One fixed association (thread chunks -> lanes -> warps): every CTA of every rank that runs it on the same masses
// gets the same answer.  total_in < 0: use the sum itself as the total.
template <typename Mass>
__device__ __forceinline__ void block_locate(int n, int ct, int cw, int lane, double u_hi, double base0, double total_in,
                                             Mass mass, double* sh_w, int* sh_hw, double* sh_bw, int& idx, double& base, double& sum) {
    const int per = (n + kConsThreads - 1) / kConsThreads;
    const int i0 = min(n, ct * per), i1 = min(n, i0 + per);
    double loc = 0.0;
    for (int i = i0; i < i1; ++i) loc += mass(i);
    double inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double w = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += w;
    }
    if (lane == 31) sh_w[cw] = inc;
    const double prev = __shfl_up_sync(0xffffffffu, inc, 1);
    cons_bar();
    double woff = 0.0, tot = 0.0;
#pragma unroll
    for (int w = 0; w < kConsWarps; ++w) {
        if (w == cw) woff = tot;
        tot += sh_w[w];
    }
    sum = tot;
    const double total = total_in < 0.0 ? tot : total_in;
    double run = base0 + woff + (lane ? prev : 0.0);
    int hit = -1;
    double hb = 0.0;
    // (run / total) > u_hi decided without the fp64 division wherever that is safe: the product u_hi * total is within
    // one ulp of the real threshold and the quotient is correctly rounded, so outside a band of a few ulps around it the
    // comparison of `run` with the product gives the division's answer; inside the band the division itself is done
    const double thr = u_hi * total, thr_lo = thr * (1.0 - 8e-16), thr_hi = thr * (1.0 + 8e-16);
    for (int i = i0; i < i1; ++i) {
        const double before = run, m = mass(i);
        run += m;
        if (hit < 0 && m > 0.0 && run > thr_lo && (run > thr_hi || (run / total) > u_hi)) { hit = i; hb = before; }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit >= 0);
    const int src = bal ? __ffs(bal) - 1 : 0;
    const int wh = __shfl_sync(0xffffffffu, hit, src);
    const double wb = __shfl_sync(0xffffffffu, hb, src);
    if (lane == 0) { sh_hw[cw] = bal ? wh : -1; sh_bw[cw] = wb; }
    cons_bar();
    idx = -1;
    base = 0.0;
#pragma unroll
    for (int w = 0; w < kConsWarps; ++w)
        if (idx < 0 && sh_hw[w] >= 0) { idx = sh_hw[w]; base = sh_bw[w]; }
    cons_bar();                               // sh_* are reused by the next call
}

// block_locate by ONE warp (n <= 2048 items): no block barrier, one shuffle scan.  Same contract.
template <typename Mass>
__device__ __forceinline__ void warp_locate(int n, int lane, double u_hi, double base0, double total_in, Mass mass,
                                            int& idx, double& base, double& sum) {
    const int per = (n + 31) / 32;
    const int i0 = min(n, lane * per), i1 = min(n, i0 + per);
    double loc = 0.0;
    for (int i = i0; i < i1; ++i) loc += mass(i);
    double inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double w = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += w;
    }
    sum = __shfl_sync(0xffffffffu, inc, 31);
    const double total = total_in < 0.0 ? sum : total_in;
    const double prev = __shfl_up_sync(0xffffffffu, inc, 1);
    double run = base0 + (lane ? prev : 0.0);
    int hit = -1;
    double hb = 0.0;
    const double thr = u_hi * total, thr_lo = thr * (1.0 - 8e-16), thr_hi = thr * (1.0 + 8e-16);   // see block_locate
    for (int i = i0; i < i1; ++i) {
        const double before = run, m = mass(i);
        run += m;
        if (hit < 0 && m > 0.0 && run > thr_lo && (run > thr_hi || (run / total) > u_hi)) { hit = i; hb = before; }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit >= 0);
    const int src = bal ? __ffs(bal) - 1 : 0;
    idx = bal ? __shfl_sync(0xffffffffu, hit, src) : -1;
    base = __shfl_sync(0xffffffffu, hb, src);
}

// The exact D^2 draw, NumPy operation for operation (coreset_sampler.py:84-92): leaf sums of the float32 pairwise
// tree -> S -> fp64 mass of fl32(c / S) per leaf -> the leaf and the element where cumsum / total crosses u.  Taken when
// the certified fast path cannot decide (and always with d2_fast_path = 0); out of line so that its registers (16
// values per lane live across three exchanges) do not weigh on the streaming loop.
struct SelShared {
    double w[kConsWarps];
    double bw[kConsWarps];
    double base, base_nz;
    int hw[kConsWarps];
    int level[40];
    int centre, hit, nz;
    unsigned long long prof[10];   // CTA 0 / thread 0 only: [0] stream [1] select [2..5] phases [6] step start [7] last stamp [8] stream end
};

__device__ __noinline__ int exact_draw(const PersistArgs& A, const PGroup* Gp, SelShared* ss, float* val, const unsigned int* s_sched,
                                       const int* s_rows, int grank, unsigned int vtag, double u, unsigned int* rnd,
                                       int my_leaf, int leaf_pos, int leaf_len, unsigned int cand_mask) {
    const PGroup G = *Gp;                     // a private copy: the caller's stays in registers
    const int ct = threadIdx.x - 32, cw = ct >> 5, lane = ct & 31;
    const int grp = ct >> 3, g_lane = ct & 7;
    const unsigned gmask = 0xffu << ((lane >> 3) * 8);
    char* const win = A.peer[A.rank];
    const int K = G.n_leaves;
    const int root = K > 1 ? 2 * K - 2 : 0;
    unsigned long long* const valw = A.valw + G.cfull_off;
    unsigned int& rnd_leaf = rnd[0];
    unsigned int& rnd_mass = rnd[1];
    unsigned int& rnd_pick = rnd[2];
    int centre = G.row_lo;
    // ---- (1) this group's leaf: wait for this step's min-distance of every candidate position ----
    float v[16];
    {
        // all loads of a round are issued before any tag is looked at: one L2 round trip per round, not 16
        unsigned int pend = cand_mask;
        const unsigned long long* base = valw + leaf_pos + g_lane;
        const long long t0 = clock64();
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = ALQ_NEG_INF;          // labeled / padding positions: prob 0
        if (pend) {                   // one word per lane until it is there: no flood while the rows still stream
            const unsigned long long* sp = base + 8 * (31 - __clz(pend));
            for (int spin = 0; static_cast<unsigned int>(ll_load(sp) >> 32) != vtag; ++spin) {
                if (ll_give_up(spin, t0, A)) break;
                __nanosleep(40);
            }
        }
        for (int spin = 0; pend; ++spin) {
            unsigned long long w[16];
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (pend & (1u << j)) w[j] = ll_load(base + 8 * j);
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if ((pend & (1u << j)) && static_cast<unsigned int>(w[j] >> 32) == vtag) {
                    v[j] = __uint_as_float(static_cast<unsigned int>(w[j]));
                    pend &= ~(1u << j);
                }
            if (pend && ll_give_up(spin, t0, A)) break;
        }
    }
    float total32 = 0.f;
    bool failed = false;
    for (int attempt = 0;; ++attempt) {
        // ---- (2) leaf sums of NumPy's pairwise tree -> every rank; fold the tree in shared memory ----
        const unsigned int tag = A.tag_base | (++rnd_leaf & 0xffffffu);
        const unsigned int slot = rnd_leaf & 1u;
        if (my_leaf >= 0) {
            const float s = leaf_sum_regs(v, leaf_len, lane, gmask);
            if (g_lane < A.world)
                ll_store(A.peer[g_lane] + G.leafw + (static_cast<size_t>(slot) * K + my_leaf) * 8, tag, __float_as_uint(s));
        }
        ll_gather(win + G.leafw + static_cast<size_t>(slot) * K * 8, K, 8, tag, 32, A, ct,
                  [&](int i, unsigned long long w) { val[i] = __uint_as_float(static_cast<unsigned int>(w)); });
        cons_bar();
        {
            int h = 0;
            for (; h < G.n_levels && ss->level[h + 1] - ss->level[h] > 32; ++h) {     // wide levels: the whole block
                const int lo = ss->level[h], hi = ss->level[h + 1];
                for (int j = lo + ct; j < hi; j += kConsThreads) {
                    const unsigned int e = s_sched[j];
                    val[K + j] = val[e & 0xffffu] + val[e >> 16];
                }
                cons_bar();
            }
            if (cw == 0)                                                          // the top of the tree: one warp
                for (; h < G.n_levels; ++h) {
                    const int lo = ss->level[h], hi = ss->level[h + 1];
                    for (int j = lo + lane; j < hi; j += 32) {
                        const unsigned int e = s_sched[j];
                        val[K + j] = val[e & 0xffffu] + val[e >> 16];
                    }
                    __syncwarp();
                }
        }
        cons_bar();
        total32 = val[root];
        cons_bar();                                   // val is reused below
        if (total32 > 0.f && total32 <= 3.4028234e38f) break;
        if (!(total32 == 0.f) || attempt > (1 << 20)) { failed = true; break; }   // NaN / inf mass
        // sum == 0 -> prob is NaN -> `min_dist_labeled += 0.00001` and retry (:87-90): on the register copy of
        // this step's values, so the bump never outlives this draw (the next step brings fresh values)
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] += 0.00001f;
    }
    if (failed) {                                     // the same decision in every CTA of every rank
        if (ct == 0) atomicCAS(A.status, 0, ALQ_ERR_NUMERIC);
        centre = G.row_lo;
    } else {
        // ---- (3) fp64 mass of prob = clip(mind, 0) / S per leaf -> every rank ----
        const unsigned int tag = A.tag_base | (++rnd_mass & 0xffffffu);
        const unsigned int slot = rnd_mass & 1u;
        if (my_leaf >= 0) {
            double m = 0.0;
#pragma unroll
            for (int j = 0; j < 16; ++j) m += prob64(v[j], total32);
            m += __shfl_down_sync(gmask, m, 1, 8);
            m += __shfl_down_sync(gmask, m, 2, 8);
            m += __shfl_down_sync(gmask, m, 4, 8);
            m = __shfl_sync(gmask, m, lane & ~7);
            if (g_lane < A.world) {
                char* dst = A.peer[g_lane] + G.massw + (static_cast<size_t>(slot) * K + my_leaf) * 16;
                ll_store(dst, tag, static_cast<unsigned int>(__double2hiint(m)));
                ll_store(dst + 8, tag, static_cast<unsigned int>(__double2loint(m)));
            }
        }
        double* M = reinterpret_cast<double*>(val);   // K doubles == 2K floats
        {
            unsigned int* M32 = reinterpret_cast<unsigned int*>(M);      // word 2i = hi, 2i + 1 = lo of leaf i
            ll_gather(win + G.massw + static_cast<size_t>(slot) * K * 16, 2 * K, 8, tag, 32, A, ct,
                      [&](int i, unsigned long long w) { M32[i ^ 1] = static_cast<unsigned int>(w); });   // little endian: lo first
        }
        if (ct == 0) { ss->hit = 0x7fffffff; ss->nz = -1; }
        cons_bar();
        // ---- np.random.choice == first k with cumsum64(p)[k] / total > u: locate the leaf.  One fixed
        //      chain (thread chunks -> lanes -> warps), identical in every CTA of every rank. ----
        const int per = (K + kConsThreads - 1) / kConsThreads;
        const int l0 = min(K, ct * per), l1 = min(K, l0 + per);
        double loc = 0.0;
        for (int l = l0; l < l1; ++l) loc += M[l];
        double inc = loc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double w = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += w;
        }
        if (lane == 31) ss->w[cw] = inc;
        const double prev = __shfl_up_sync(0xffffffffu, inc, 1);
        cons_bar();
        double woff = 0.0, total = 0.0;
        for (int w = 0; w < kConsWarps; ++w) {
            if (w == cw) woff = total;
            total += ss->w[w];
        }
        double run = woff + (lane ? prev : 0.0);
        int my_hit = 0x7fffffff, my_nz = -1;
        double hit_base = 0.0, nz_base = 0.0;
        for (int l = l0; l < l1; ++l) {
            const double before = run;
            run += M[l];
            if (M[l] > 0.0) { my_nz = l; nz_base = before; }
            if (my_hit == 0x7fffffff && (run / total) > u) { my_hit = l; hit_base = before; }
        }
        {
            const int wh = __reduce_min_sync(0xffffffffu, my_hit), wn = __reduce_max_sync(0xffffffffu, my_nz);
            if (lane == 0) {
                if (wh != 0x7fffffff) atomicMin(&ss->hit, wh);
                if (wn >= 0) atomicMax(&ss->nz, wn);
            }
        }
        cons_bar();
        if (my_hit != 0x7fffffff && my_hit == ss->hit) ss->base = hit_base;
        if (my_nz >= 0 && my_nz == ss->nz) ss->base_nz = nz_base;
        cons_bar();
        int leaf = ss->hit;
        double base = ss->base;
        if (leaf == 0x7fffffff) { leaf = ss->nz; base = ss->base_nz; }   // u beyond the last mass by an ulp
        // ---- (4) the group that owns the leaf searches inside it (values still in registers) ----
        const unsigned int ptag = A.tag_base | (++rnd_pick & 0xffffffu);
        const unsigned int pslot = rnd_pick & 1u;
        if (leaf < 0 && grank == 0 && A.rank == 0 && cw == 0) {       // no mass at all: cannot happen with S > 0
            if (lane == 0) atomicCAS(A.status, 0, ALQ_ERR_NUMERIC);
            if (lane < A.world) ll_store(A.peer[lane] + G.pickw + pslot * 8, ptag, static_cast<unsigned int>(G.row_lo));
        }
        if (leaf >= 0 && leaf == my_leaf) {           // whole 8-lane group, uniformly
            // sequential order k = 8j + lane: scan 8 lanes per j, carry across j
            double carry = base;
            int hit = -1, nz = -1;
            const int g0 = lane & ~7;
            for (int j = 0; j < 16 && 8 * j < leaf_len; ++j) {
                double pj = 0.0;
#pragma unroll
                for (int jj = 0; jj < 16; ++jj)
                    if (jj == j) pj = prob64(v[jj], total32);
                double sc = pj;
#pragma unroll
                for (int o = 1; o < 8; o <<= 1) {
                    const double w = __shfl_up_sync(gmask, sc, o, 8);
                    if (g_lane >= o) sc += w;
                }
                const double rk = carry + sc;
                const bool cross = pj > 0.0 ? ((rk / total) > u) : false;
                // an element with zero mass can cross only if an earlier one did: ignore it
                const unsigned cb = (__ballot_sync(gmask, cross) >> g0) & 0xffu;
                const unsigned zb = (__ballot_sync(gmask, pj > 0.0) >> g0) & 0xffu;
                if (zb) nz = 8 * j + (31 - __clz(zb));
                if (cb) { hit = 8 * j + (__ffs(cb) - 1); break; }
                carry = __shfl_sync(gmask, rk, g0 + 7);
            }
            const int k = hit >= 0 ? hit : nz;        // no crossing: re-association moved it by an ulp
            int row = k >= 0 ? s_rows[grp * 128 + k] : -1;
            if (row < 0) {
                if (g_lane == 0) atomicCAS(A.status, 0, ALQ_ERR_NUMERIC);
                row = G.row_lo;
            }
            if (g_lane < A.world) ll_store(A.peer[g_lane] + G.pickw + pslot * 8, ptag, static_cast<unsigned int>(row));
        }
        if (ct == 0) ss->centre = static_cast<int>(ll_wait(win + G.pickw + pslot * 8, ptag, A));
        cons_bar();
        centre = ss->centre;
    }

    return centre;
}

template <bool FACTORED, bool SAMPLE>
__global__ void __launch_bounds__(32 * (1 + kConsWarps), 1)
greedy_persist_kernel(const __grid_constant__ PersistArgs A, const PipeCfg cfg, const int k_max, const int lc_max, const int ne_max, const int rm_max) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int d = A.d, c = FACTORED ? A.c : 0;
    const int dv = d >> 2, cv = c >> 2;
    float* sq = reinterpret_cast<float*>(smem_raw);                          // centre: d + c floats
    float* tiles = sq + ((d + c + 31) & ~31);                                // stage ring
    uint64_t* full = reinterpret_cast<uint64_t*>(tiles + static_cast<size_t>(cfg.stages) * cfg.tile_floats);
    uint64_t* empty = full + cfg.stages;
    unsigned long long* sbest = reinterpret_cast<unsigned long long*>(empty + cfg.stages);   // [kConsWarps]
    float* val = reinterpret_cast<float*>(sbest + kConsWarps + 1);                                 // [2 * k_max] (SAMPLE)
    unsigned int* s_sched = reinterpret_cast<unsigned int*>(val + 2 * static_cast<size_t>(k_max));   // [k_max]
    int* s_rows = reinterpret_cast<int*>(s_sched + k_max);                                    // [lc_max * 128] row of each owned position
    double* s_u = reinterpret_cast<double*>(s_rows + static_cast<size_t>(lc_max) * 128);        // [ne_max] per-CTA masses of every rank (SAMPLE)
    float* s_m = reinterpret_cast<float*>(s_u + ne_max);                                        // [rm_max] clip(mind, 0) of this CTA's rows (0: not kept)
    __shared__ SelShared ss;

    const BlockSeg seg = A.segs[blockIdx.x];
    const PGroup G = A.groups[seg.part];
    const int grank = static_cast<int>(blockIdx.x) - G.cta_lo;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int R = cfg.rows_per_tile;
    const int nrows = seg.row_hi - seg.row_lo;
    const int ntiles = (nrows + R - 1) / R;
    const int nstream = G.budget - 1;                 // steps 1 .. budget-1 stream the rows

    if (threadIdx.x == 0) {
        for (int s = 0; s < cfg.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (SAMPLE) {
        for (int i = threadIdx.x; i < G.n_leaves - 1; i += blockDim.x) s_sched[i] = A.sched[G.sched_base + i];
        if (threadIdx.x <= G.n_levels && threadIdx.x < 40) ss.level[threadIdx.x] = A.level_off[G.level_base + threadIdx.x];
    }
    __syncthreads();

    if (warp == 0) {
        // ===== producer: one lane issues every bulk copy of every step; it never needs the centre =====
        if (lane == 0 && ntiles > 0) {
            const bool contig_x = (A.ldx == d), contig_a = FACTORED && (A.lda == c);
            const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
            const bool hints = A.resident_rows > 0;
            int s = 0;
            unsigned int par = 0;                     // parity of the `empty` phase to wait for (first round: none)
            bool first_round = true;
            for (int st = 0; st < nstream; ++st) {
                for (int i = 0; i < ntiles; ++i) {
                    if (!first_round) mbar_wait(&empty[s], par);
                    const int row0 = seg.row_lo + i * R;
                    const int rr = min(R, seg.row_hi - row0);
                    float* tx = tiles + static_cast<size_t>(s) * cfg.tile_floats;
                    float* ta = tx + static_cast<size_t>(R) * d;
                    const uint64_t pol = (i * R < A.resident_rows) ? pol_keep : pol_stream;
                    mbar_expect_tx(&full[s], static_cast<uint32_t>(rr) * static_cast<uint32_t>(d + c) * 4u);
                    if (contig_x) {
                        if (hints) bulk_g2s_hint(tx, A.x + static_cast<long long>(row0) * A.ldx, static_cast<uint32_t>(rr) * d * 4u, &full[s], pol);
                        else bulk_g2s(tx, A.x + static_cast<long long>(row0) * A.ldx, static_cast<uint32_t>(rr) * d * 4u, &full[s]);
                    } else {
                        for (int r = 0; r < rr; ++r)
                            bulk_g2s(tx + static_cast<size_t>(r) * d, A.x + static_cast<long long>(row0 + r) * A.ldx, d * 4u, &full[s]);
                    }
                    if (FACTORED) {
                        if (contig_a) {
                            if (hints) bulk_g2s_hint(ta, A.a + static_cast<long long>(row0) * A.lda, static_cast<uint32_t>(rr) * c * 4u, &full[s], pol);
                            else bulk_g2s(ta, A.a + static_cast<long long>(row0) * A.lda, static_cast<uint32_t>(rr) * c * 4u, &full[s]);
                        } else {
                            for (int r = 0; r < rr; ++r)
                                bulk_g2s(ta + static_cast<size_t>(r) * c, A.a + static_cast<long long>(row0 + r) * A.lda, c * 4u, &full[s]);
                        }
                    }
                    if (++s == cfg.stages) {
                        s = 0;
                        if (first_round) first_round = false; else par ^= 1u;
                    }
                }
            }
        }
        return;
    }

    // ===== consumers =====================================================================================
    const int ct = threadIdx.x - 32;          // 0 .. kConsThreads-1
    const int cw = warp - 1;
    const int C = cfg.consumers;              // warps that take tiles (<= kConsWarps)
    char* const win = A.peer[A.rank];
    const float4* q4 = reinterpret_cast<const float4*>(sq);
    unsigned long long* const valw = A.valw + (SAMPLE ? G.cfull_off : 0);

    // D^2 sampling: the leaf this 8-lane group owns for the whole call (one per group), the rows behind its
    // positions (shared memory) and which of this lane's 16 positions hold a candidate at all
    const int grp = ct >> 3, g_lane = ct & 7;
    int my_leaf = -1, leaf_pos = 0, leaf_len = 0;
    unsigned int cand_mask = 0;
    if (SAMPLE) {
        const int leaf = G.leaf_lo + grank + grp * G.ncta;
        if (leaf < G.leaf_hi) {
            my_leaf = leaf;
            leaf_pos = A.leaf_off[G.leaf_base + leaf];
            leaf_len = A.leaf_off[G.leaf_base + leaf + 1] - leaf_pos;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int k = 8 * j + g_lane;
                const int row = k < leaf_len ? A.posinv[G.cfull_off + leaf_pos + k] : -1;
                s_rows[grp * 128 + k] = row;
                if (row >= 0) cand_mask |= 1u << j;
            }
        }
    }

    if (A.ready_tag != 0 && ct < A.world) ll_ready_wait(win + A.ready_off, ct, A.ready_tag, A);   // peers may still be clearing theirs
    cons_bar();

    // per-warp position in the tile stream (global over all steps): tiles cw, cw + C, cw + 2C, ...
    int my_i = cw;                            // next tile this warp consumes, relative to the current step's first tile
    int my_s = cw % cfg.stages;
    unsigned int my_par = 0;
    for (int q = cw / cfg.stages; q > 0; --q) my_par ^= 1u;

    unsigned int rnd_key = 0, rnd_leaf = 0, rnd_mass = 0, rnd_pick = 0, rnd_u = 0;
    int centre = -1;
    const bool prof = A.prof != nullptr && blockIdx.x == 0 && ct == 0;
    if (prof) { for (int i = 0; i < 10; ++i) ss.prof[i] = 0; ss.prof[9] = gtime_ns(); }

    for (int t = 0; t < G.budget; ++t) {
        unsigned long long best_key = 0ull;   // arg-max: ord(min-distance) << 32 | ~(row - seg.row_lo)
        double usum = 0.0;                    // D^2: fp64 mass clip(mind, 0) of the rows this lane finished
        const unsigned int vtag = A.tag_base | (static_cast<unsigned int>(t + 1) & 0xffffffu);
        double u = 0.0;
        if (SAMPLE) u = __ldg(A.uniforms + G.pick_off + t);           // needed late: issue the load now
        if (prof) ss.prof[6] = gtime_ns();
        if (t == 0) {
            if (G.first_pick >= 0) {          // centre 0 chosen by the caller: no selection
                centre = G.first_pick;
                if (grank == 0 && ct == 0) A.picks[G.pick_off] = centre;
                continue;
            }
            for (int row = seg.row_lo + ct; row < seg.row_hi; row += kConsThreads) {
                const float m = __ldcg(A.mind + row);
                if (SAMPLE) {
                    ll_store(valw + A.vpos[row], vtag, __float_as_uint(m));
                    usum += static_cast<double>(fmaxf(m, 0.f));
                    if (rm_max) s_m[row - seg.row_lo] = fmaxf(m, 0.f);
                } else {
                    const unsigned long long k = (static_cast<unsigned long long>(alq_ord(m)) << 32) | (0xffffffffu - static_cast<uint32_t>(row - seg.row_lo));
                    best_key = k > best_key ? k : best_key;
                }
            }
        } else {
            // ---- centre row -> shared memory (a replica of every candidate row is local) ----
            {
                float4* dst = reinterpret_cast<float4*>(sq);
                const float4* src = reinterpret_cast<const float4*>(A.x + static_cast<long long>(centre) * A.ldx);
                for (int k = ct; k < dv; k += kConsThreads) dst[k] = __ldg(src + k);
                if (FACTORED) {
                    const float4* sa = reinterpret_cast<const float4*>(A.a + static_cast<long long>(centre) * A.lda);
                    for (int k = ct; k < cv; k += kConsThreads) dst[dv + k] = __ldg(sa + k);
                }
            }
            const float qn = FACTORED ? __ldg(A.xn + centre) * __ldg(A.an + centre) : __ldg(A.xn + centre);
            cons_bar();
            // ---- this step's tiles ----
            if (cw < C) {
                for (; my_i < ntiles; my_i += C) {
                    const int row0 = seg.row_lo + my_i * R;
                    const int rr = min(R, seg.row_hi - row0);
                    float m_old = 0.f, n_i = 0.f;
                    int vp = 0;
                    if (lane < rr) {
                        m_old = __ldcg(A.mind + row0 + lane);
                        n_i = FACTORED ? __ldg(A.xn + row0 + lane) * __ldg(A.an + row0 + lane) : __ldg(A.xn + row0 + lane);
                        if (SAMPLE) vp = __ldg(A.vpos + row0 + lane);
                    }
                    mbar_wait(&full[my_s], my_par);
                    const float* tx = tiles + static_cast<size_t>(my_s) * cfg.tile_floats;
                    const float* ta = tx + static_cast<size_t>(R) * d;
                    float my_d2 = 0.f;
                    for (int r = 0; r < rr; ++r) {
                        const float4* pr = reinterpret_cast<const float4*>(tx + static_cast<size_t>(r) * d);
                        float dot = 0.f;
#pragma unroll 4
                        for (int k = lane; k < dv; k += 32) {
                            const float4 v = pr[k];
                            const float4 w = q4[k];
                            dot = fmaf(v.x, w.x, dot);
                            dot = fmaf(v.y, w.y, dot);
                            dot = fmaf(v.z, w.z, dot);
                            dot = fmaf(v.w, w.w, dot);
                        }
                        dot = warp_sum(dot);
                        if (FACTORED) {
                            const float4* pa = reinterpret_cast<const float4*>(ta + static_cast<size_t>(r) * c);
                            float da = 0.f;
#pragma unroll 4
                            for (int k = lane; k < cv; k += 32) {
                                const float4 v = pa[k];
                                const float4 w = q4[dv + k];
                                da = fmaf(v.x, w.x, da);
                                da = fmaf(v.y, w.y, da);
                                da = fmaf(v.z, w.z, da);
                                da = fmaf(v.w, w.w, da);
                            }
                            dot *= warp_sum(da);
                        }
                        if (lane == r) my_d2 = dot;
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[my_s]);
                    if (lane < rr) {
                        const int row = row0 + lane;
                        float m = fminf(m_old, dist_dense(n_i, qn, my_d2));
                        if (row == centre) m = ALQ_NEG_INF;         // a picked row is never a candidate again
                        __stcg(A.mind + row, m);
                        if (SAMPLE) {
                            ll_store(valw + vp, vtag, __float_as_uint(m));   // raw running min (exact path); the draw clips at 0
                            usum += static_cast<double>(fmaxf(m, 0.f));
                            if (rm_max) s_m[row - seg.row_lo] = fmaxf(m, 0.f);
                        } else {
                            const unsigned long long k = (static_cast<unsigned long long>(alq_ord(m)) << 32) | (0xffffffffu - static_cast<uint32_t>(row - seg.row_lo));
                            best_key = k > best_key ? k : best_key;
                        }
                    }
                    my_s += C;
                    if (my_s >= cfg.stages) { my_s -= cfg.stages; my_par ^= 1u; }
                }
            }
            my_i -= ntiles;                   // the stream of tiles continues into the next step
        }

        // =================================== selection of pick t ===================================
        if (!SAMPLE) {
            // every CTA of every rank publishes ONE word {tag16, row offset, ord}; everybody reads all of them
            best_key = warp_max_u64(best_key);
            if (lane == 0) sbest[cw] = best_key;
            cons_bar();
            if (prof) ss.prof[8] = gtime_ns();
            const unsigned int tag16 = 0x8000u | ((A.tag_base >> 12) & 0x7000u) | (++rnd_key & 0xfffu);
            const unsigned int slot = rnd_key & 1u;
            const int stride = G.seg_stride;
            if (cw == 0) {
                unsigned long long b = lane < kConsWarps ? sbest[lane] : 0ull;
                b = warp_max_u64(b);
                const unsigned long long word = (static_cast<unsigned long long>(tag16) << 48) |
                                                (static_cast<unsigned long long>((0xffffffffu - static_cast<uint32_t>(b)) & 0xffffu) << 32) | (b >> 32);
                if (lane < A.world)
                    ll_store_raw(A.peer[lane] + G.keyw + (static_cast<size_t>(slot) * A.world * stride + static_cast<size_t>(A.rank) * stride + grank) * 8, word);
                if (grank == 0)               // slots of this rank beyond its CTA count (uneven shards): empty keys
                    for (int e = G.ncta + (lane >> 3); e < stride; e += 4)
                        if ((lane & 7) < A.world)
                            ll_store_raw(A.peer[lane & 7] + G.keyw + (static_cast<size_t>(slot) * A.world * stride + static_cast<size_t>(A.rank) * stride + e) * 8,
                                         static_cast<unsigned long long>(tag16) << 48);
            }
            unsigned long long k = 0ull;
            ll_gather(win + G.keyw + static_cast<size_t>(slot) * A.world * stride * 8, A.world * stride, 8, tag16, 48, A, ct,
                      [&](int i, unsigned long long w) {
                          const uint32_t row = static_cast<uint32_t>(__ldg(A.segtab + G.seg_base + i)) + static_cast<uint32_t>((w >> 32) & 0xffffu);
                          const unsigned long long key = (static_cast<unsigned long long>(static_cast<uint32_t>(w)) << 32) | (0xffffffffu - row);
                          k = key > k ? key : k;
                      });
            cons_bar();                       // sbest is reused
            k = warp_max_u64(k);
            if (lane == 0) sbest[cw] = k;
            cons_bar();
            unsigned long long kk = sbest[0];
#pragma unroll
            for (int w = 1; w < kConsWarps; ++w) kk = sbest[w] > kk ? sbest[w] : kk;
            centre = static_cast<int>(alq_maxkey_row(kk));
        } else {
            if (prof) ss.prof[8] = gtime_ns();
            // ================= certified fast path =================
            // np.random.choice picks the first k with cdf[k] > u, cdf = cumsum64(fl32(c / S)) / its last entry.  Every
            // fl32(c_i / S) is c_i / S (1 + e_i), |e_i| <= 2^-24 (or an absolute 2^-150 when it underflows), and S cancels
            // in the ratio, so cdf[k] = Q[k] / Q[n-1] (1 + d), |d| <= 2^-23, with Q the plain fp64 prefix sums of
            // c = clip(mind, 0).  If Q[k]/Q[n-1] > u + m and Q[k-1]/Q[n-1] <= u - m (m = 1.3e-7 > 2^-23 + fp64 noise) then k IS
            // NumPy's pick -- no float32 pairwise tree, no per-leaf masses.  Q needs one exchange of one fp64 mass per
            // CTA; the CTA holding the crossing searches its own rows.  A step whose u falls inside a margin (about 2 %
            // of the steps at 80 000 rows), or whose mass is zero / non-finite, takes the exact machinery below.
            bool exact = A.fast_path == 0;
            if (!exact) {
                constexpr double kMargin = 1.3e-7;
                const int stride = G.seg_stride, ne = A.world * stride;
                const unsigned int utag = A.tag_base | (++rnd_u & 0xffffffu);
                const unsigned int uslot = rnd_u & 1u;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) usum += __shfl_xor_sync(0xffffffffu, usum, o);
                if (lane == 0) ss.w[cw] = usum;
                cons_bar();
                if (cw == 0) {
                    double tot = 0.0;
#pragma unroll
                    for (int w = 0; w < kConsWarps; ++w) tot += ss.w[w];
                    const size_t off = G.umw + (static_cast<size_t>(uslot) * ne + static_cast<size_t>(A.rank) * stride + grank) * 16;
                    if (lane < A.world) {
                        ll_store(A.peer[lane] + off, utag, static_cast<unsigned int>(__double2hiint(tot)));
                        ll_store(A.peer[lane] + off + 8, utag, static_cast<unsigned int>(__double2loint(tot)));
                    }
                    if (grank == 0)           // slots of this rank beyond its CTA count: zero mass
                        for (int e = G.ncta + (lane >> 3); e < stride; e += 4)
                            if ((lane & 7) < A.world) {
                                char* q = A.peer[lane & 7] + G.umw + (static_cast<size_t>(uslot) * ne + static_cast<size_t>(A.rank) * stride + e) * 16;
                                ll_store(q, utag, 0u);
                                ll_store(q + 8, utag, 0u);
                            }
                }
                cons_bar();                   // ss.w is reused by block_locate
                {
                    unsigned int* u32 = reinterpret_cast<unsigned int*>(s_u);
                    ll_gather(win + G.umw + static_cast<size_t>(uslot) * ne * 16, 2 * ne, 8, utag, 32, A, ct,
                              [&](int i, unsigned long long w) { u32[i ^ 1] = static_cast<unsigned int>(w); });
                }
                cons_bar();
                int e_hit;
                double e_base, q_tot;
                if (ne <= 2048) {             // one warp, no block barriers
                    if (cw == 0) {
                        warp_locate(ne, lane, u + kMargin, 0.0, -1.0, [&](int i) { return s_u[i]; }, e_hit, e_base, q_tot);
                        if (lane == 0) { ss.hw[0] = e_hit; ss.bw[0] = e_base; ss.w[0] = q_tot; }
                    }
                    cons_bar();
                    e_hit = ss.hw[0]; e_base = ss.bw[0]; q_tot = ss.w[0];
                    cons_bar();
                } else {
                    block_locate(ne, ct, cw, lane, u + kMargin, 0.0, -1.0, [&](int i) { return s_u[i]; }, ss.w, ss.hw, ss.bw, e_hit, e_base, q_tot);
                }
                const bool sane = q_tot > 0.0 && q_tot <= 1.0e300;
                if (!sane || e_hit < 0 || !((e_base / q_tot) <= u - kMargin)) exact = true;     // same verdict in every CTA of every rank
                if (!exact) {
                    const unsigned int ptag = A.tag_base | (++rnd_pick & 0xffffffu);
                    const unsigned int pslot = rnd_pick & 1u;
                    if (e_hit == A.rank * stride + grank) {       // the crossing is inside this CTA's rows
                        int r_hit = -1;
                        double r_base = 0.0, r_sum;
                        if (nrows <= 2048) {                      // one warp; the rows' masses are in shared memory if kept
                            if (cw == 0) {
                                if (rm_max) warp_locate(nrows, lane, u + kMargin, e_base, q_tot, [&](int i) { return static_cast<double>(s_m[i]); }, r_hit, r_base, r_sum);
                                else warp_locate(nrows, lane, u + kMargin, e_base, q_tot,
                                                 [&](int i) { return static_cast<double>(fmaxf(__ldcg(A.mind + seg.row_lo + i), 0.f)); }, r_hit, r_base, r_sum);
                                unsigned int word = 0xffffffffu;  // "not certain": everybody takes the exact path
                                if (r_hit >= 0 && (r_base / q_tot) <= u - kMargin) word = static_cast<unsigned int>(seg.row_lo + r_hit);
                                if (lane < A.world) ll_store(A.peer[lane] + G.pickw + pslot * 8, ptag, word);
                            }
                        } else {
                            block_locate(nrows, ct, cw, lane, u + kMargin, e_base, q_tot,
                                         [&](int i) { return static_cast<double>(fmaxf(__ldcg(A.mind + seg.row_lo + i), 0.f)); },
                                         ss.w, ss.hw, ss.bw, r_hit, r_base, r_sum);
                            unsigned int word = 0xffffffffu;
                            if (r_hit >= 0 && (r_base / q_tot) <= u - kMargin) word = static_cast<unsigned int>(seg.row_lo + r_hit);
                            if (ct < A.world) ll_store(A.peer[ct] + G.pickw + pslot * 8, ptag, word);
                        }
                    }
                    if (ct == 0) ss.centre = static_cast<int>(ll_wait(win + G.pickw + pslot * 8, ptag, A));
                    cons_bar();
                    if (ss.centre == -1) exact = true;
                    else centre = ss.centre;
                    cons_bar();               // ss.centre is rewritten by the exact path
                }
            }
            if (exact) {
                unsigned int rnd[3] = {rnd_leaf, rnd_mass, rnd_pick};
                centre = exact_draw(A, A.groups + seg.part, &ss, val, s_sched, s_rows, grank, vtag, u, rnd, my_leaf, leaf_pos, leaf_len, cand_mask);
                rnd_leaf = rnd[0]; rnd_mass = rnd[1]; rnd_pick = rnd[2];
            }
        }
        if (grank == 0 && ct == 0) A.picks[G.pick_off + t] = centre;
        if (prof) {
            const unsigned long long t_c = gtime_ns();
            if (t > 0) { ss.prof[0] += ss.prof[8] - ss.prof[6]; ss.prof[1] += t_c - ss.prof[8]; }
            else ss.prof[4] = t_c - ss.prof[6];      // the t = 0 selection (no streaming)
        }
    }
    if (prof) {
        A.prof[0] = ss.prof[0];
        A.prof[1] = ss.prof[1];
        A.prof[2] = static_cast<unsigned long long>(G.budget > 1 ? G.budget - 1 : 0);
        for (int i = 0; i < 3; ++i) A.prof[3 + i] = ss.prof[2 + i];
        A.prof[6] = gtime_ns() - ss.prof[9];     // the whole kernel as CTA 0 saw it
    }
}

// posinv[off[p] + vpos[row]] = row for every candidate row of every partition
__global__ void persist_posinv_kernel(const int* __restrict__ vpos, const int* __restrict__ part_off,
                                      const int* __restrict__ cfull_off, int P, int n, int* __restrict__ posinv) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    int p = 0;
    while (p + 1 < P && row >= part_off[p + 1]) ++p;
    posinv[cfull_off[p] + vpos[row]] = row;
}

template <bool FACTORED, bool SAMPLE>
cudaError_t launch_persist(int grid, size_t smem, cudaStream_t st, PersistArgs& A, PipeCfg& cfg, int& k_max, int& lc_max, int& ne_max, int& rm_max) {
    auto* fn = greedy_persist_kernel<FACTORED, SAMPLE>;
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    void* args[] = {&A, &cfg, &k_max, &lc_max, &ne_max, &rm_max};
    return cudaLaunchCooperativeKernel(reinterpret_cast<void*>(fn), dim3(grid), dim3(32 * (1 + kConsWarps)), args, smem, st);
}

}  // namespace

extern "C" int64_t alq_pairwise_leaf_bounds(int64_t n, int32_t* out_host, int64_t cap) {
    if (n <= 0 || n >= (1LL << 31) || !out_host) return -1;
    const PairTree tb(static_cast<int>(n));
    const int64_t k = tb.n_leaves();
    if (cap < k + 1) return -1;
    std::copy(tb.leaf_off.begin(), tb.leaf_off.end(), out_host);
    return k;
}

int alq_greedy_persist(alq_ctx* ctx, const alq_greedy_desc* D, void* stream) {
    const int P = D->n_parts;
    const int64_t n = D->n;
    const bool factored = D->a != nullptr;
    const bool sample = D->uniforms_host != nullptr;
    const int d = D->d, c = factored ? D->c : 0;
    const AlqComm& Gc = ctx->comm;
    const bool comm = D->shard_off_host != nullptr && Gc.window != nullptr && Gc.connected;   // the group path (alq_greedy_select)
    const int world = comm ? Gc.world : 1, rank = comm ? Gc.rank : 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);

    // ---- does the problem fit? --------------------------------------------------------------------------
    const size_t row_bytes = static_cast<size_t>(d + c) * 4;
    if ((row_bytes % 16) || (static_cast<size_t>(d) * 4 % 16)) return kPersistNotApplicable;
    std::vector<int> pick_off(P + 1, 0);
    int bmax = 0, active = 0;
    for (int p = 0; p < P; ++p) {
        pick_off[p + 1] = pick_off[p] + D->budget_host[p];
        bmax = std::max(bmax, D->budget_host[p]);
        if (D->budget_host[p] > 0) ++active;
    }
    if (active == 0) return ALQ_OK;
    if (active > ctx->sm_count) return kPersistNotApplicable;

    // ---- CTAs: at most one per SM in total, split over the partitions by row count.  In multi-GPU mode (P == 1)
    //      every rank derives every rank's segmentation (the arg-max words carry a row offset inside a segment). ----
    std::vector<PGroup> groups(P);
    std::vector<BlockSeg> segs;
    std::vector<int> segtab, ncta_tab;
    {
        std::vector<int64_t> rows(P, 0);
        int64_t total = 0;
        for (int p = 0; p < P; ++p) {
            if (D->budget_host[p] <= 0) continue;
            rows[p] = comm ? (D->shard_off_host[rank + 1] - D->shard_off_host[rank]) : (D->part_off_host[p + 1] - D->part_off_host[p]);
            total += rows[p];
        }
        int left = ctx->sm_count - active;           // one CTA per active partition first, the rest by share
        std::vector<int> nb(P, 0);
        for (int p = 0; p < P; ++p) {
            if (D->budget_host[p] <= 0) continue;
            const int extra = total > 0 ? static_cast<int>(static_cast<int64_t>(ctx->sm_count - active) * rows[p] / total) : 0;
            nb[p] = 1 + std::min(extra, left);
            left -= nb[p] - 1;
        }
        for (int p = 0; p < P && left > 0; ++p)
            if (nb[p] > 0 && rows[p] > nb[p]) { ++nb[p]; --left; }
        auto ncta_for = [&](int want, int64_t r) { return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(want, std::max<int64_t>(r, 1)))); };
        int cta = 0;
        for (int p = 0; p < P; ++p) {
            PGroup& g = groups[p];
            g = PGroup{};
            g.budget = D->budget_host[p];
            g.pick_off = pick_off[p];
            g.first_pick = D->first_pick_host ? D->first_pick_host[p] : -1;
            g.row_lo = comm ? 0 : D->part_off_host[p];
            g.n_leaves = 1;
            if (nb[p] == 0) continue;
            g.seg_base = static_cast<int>(segtab.size());
            g.ncta_base = static_cast<int>(ncta_tab.size());
            int stride = 0;
            for (int r = 0; r < world; ++r) {
                const int64_t rr = comm ? (D->shard_off_host[r + 1] - D->shard_off_host[r]) : rows[p];
                const int k = ncta_for(comm ? ctx->sm_count : nb[p], rr);
                ncta_tab.push_back(k);
                stride = std::max(stride, k);
            }
            g.seg_stride = stride;
            segtab.resize(segtab.size() + static_cast<size_t>(world) * stride, 0);
            for (int r = 0; r < world; ++r) {
                const int lo = comm ? D->shard_off_host[r] : D->part_off_host[p];
                const int64_t rr = comm ? (D->shard_off_host[r + 1] - D->shard_off_host[r]) : rows[p];
                const int k = ncta_tab[g.ncta_base + r];
                for (int b = 0; b < k; ++b) {
                    const int s_lo = lo + static_cast<int>(rr * b / k), s_hi = lo + static_cast<int>(rr * (b + 1) / k);
                    segtab[g.seg_base + static_cast<size_t>(r) * stride + b] = s_lo;
                    if (!sample && s_hi - s_lo > 65535) return kPersistNotApplicable;   // 16-bit row offset in the key word
                    if (r == rank) {
                        BlockSeg s;
                        s.row_lo = s_lo; s.row_hi = s_hi; s.part = p; s.pad = 0;
                        segs.push_back(s);
                    }
                }
            }
            g.cta_lo = cta;
            g.ncta = ncta_tab[g.ncta_base + rank];
            cta += g.ncta;
        }
    }
    const int grid = static_cast<int>(segs.size());
    if (grid > ctx->sm_count || grid == 0) return kPersistNotApplicable;

    // ---- trees (D^2 sampling) ------------------------------------------------------------------------------
    std::vector<int> leaf_off_all, level_off_all, cfull_off(P, 0);
    std::vector<unsigned int> sched_all;
    int cfull_total = 0, k_max = 1, lc_max = 1;
    int leaf_bound[ALQ_MAX_WORLD + 1] = {};
    for (int p = 0; p < P && sample; ++p) {
        PGroup& g = groups[p];
        g.full_n = D->full_n_host[p];
        g.cfull_off = cfull_total;
        cfull_off[p] = cfull_total;
        cfull_total += (g.full_n + 3) & ~3;
        const PairTree tb(g.full_n);
        const int K = tb.n_leaves();
        if (K > kMaxLeaves || tb.n_levels() > 38) return kPersistNotApplicable;
        g.n_leaves = K;
        g.leaf_base = static_cast<int>(leaf_off_all.size());
        leaf_off_all.insert(leaf_off_all.end(), tb.leaf_off.begin(), tb.leaf_off.end());
        // internal nodes in level order; node id = K + position in that order
        g.n_levels = tb.n_levels();
        g.level_base = static_cast<int>(level_off_all.size());
        level_off_all.insert(level_off_all.end(), tb.level_off.begin(), tb.level_off.end());
        std::vector<int> newid(tb.internal.size());
        for (size_t j = 0; j < tb.order.size(); ++j) newid[tb.order[j]] = K + static_cast<int>(j);
        g.sched_base = static_cast<int>(sched_all.size());
        auto nid = [&](int v) { return v >= 0 ? v : newid[-v - 1]; };
        for (int k : tb.order)
            sched_all.push_back(static_cast<unsigned int>(nid(tb.internal[k].l)) | (static_cast<unsigned int>(nid(tb.internal[k].r)) << 16));
        g.leaf_lo = 0;
        g.leaf_hi = K;
        k_max = std::max(k_max, K);
        if (comm) {     // shards must be aligned to leaf boundaries
            if (!D->shard_pos_host) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: multi-GPU D^2 sampling needs shard_pos (leaf-aligned shards)");
            for (int r = 0; r <= world; ++r) {
                const int pos = D->shard_pos_host[r];
                auto it = std::lower_bound(tb.leaf_off.begin(), tb.leaf_off.end(), pos);
                if (it == tb.leaf_off.end() || *it != pos)
                    ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: shard_pos[%d] = %d is not a leaf boundary of the pairwise-sum tree", r, pos);
                leaf_bound[r] = static_cast<int>(it - tb.leaf_off.begin());
            }
            if (leaf_bound[0] != 0 || leaf_bound[world] != K)
                ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_greedy_select: shard_pos must span [0, full_n]");
            g.leaf_lo = leaf_bound[rank];
            g.leaf_hi = leaf_bound[rank + 1];
        }
        if (g.ncta > 0) {
            const int lc = (g.leaf_hi - g.leaf_lo + g.ncta - 1) / g.ncta;
            if (lc > kGroups) return kPersistNotApplicable;       // one leaf per 8-lane group
            lc_max = std::max(lc_max, lc);
        }
    }

    k_max = (k_max + 1) & ~1;                 // keeps the doubles behind the tree schedule 8-byte aligned
    // ---- shared-memory plan: centre + ring + tree ---------------------------------------------------------
    PipeCfg cfg{};
    size_t smem = 0;
    int ne_max = 1, rm_max = 0;
    {
        int seg_rows = 0;
        for (const BlockSeg& sg : segs) seg_rows = std::max(seg_rows, sg.row_hi - sg.row_lo);
        if (sample && seg_rows <= 2048) rm_max = (seg_rows + 3) & ~3;      // clip(mind, 0) of a CTA's rows stays in shared memory
        const size_t centre_bytes = static_cast<size_t>((d + c + 31) & ~31) * 4;
        for (int p = 0; p < P; ++p) ne_max = std::max(ne_max, world * groups[p].seg_stride);
        const size_t tree_bytes = (sample ? static_cast<size_t>(k_max) * 12 + static_cast<size_t>(lc_max) * 512 + 64 : 64 + 12 + 512) + static_cast<size_t>(ne_max) * 8 + static_cast<size_t>(rm_max) * 4;
        const size_t fixed = centre_bytes + tree_bytes + kConsWarps * 16 + 256;
        const size_t budget_bytes = ctx->smem_optin > 8192 ? ctx->smem_optin - 1536 : 0;
        size_t tile_target = 32 * 1024;
        int max_stages = 16;
        if (const char* e = getenv("ALQ_TILE_KB")) tile_target = std::max(1, atoi(e)) * 1024;
        if (const char* e = getenv("ALQ_MAX_STAGES")) max_stages = std::max(3, std::min(16, atoi(e)));
        int R = static_cast<int>(std::max<size_t>(1, tile_target / row_bytes));
        R = std::min(R, 32);
        const size_t tile_bytes = R * row_bytes;
        int stages = budget_bytes > fixed ? static_cast<int>((budget_bytes - fixed) / (tile_bytes + 16)) : 0;
        stages = std::min(stages, max_stages);
        if (stages < 3) return kPersistNotApplicable;
        cfg.rows_per_tile = R;
        cfg.stages = stages;
        cfg.tile_floats = static_cast<int>(tile_bytes / 4);
        cfg.consumers = std::max(1, std::min(kConsWarps, stages));
        smem = centre_bytes + stages * tile_bytes + 2 * stages * sizeof(uint64_t) + kConsWarps * 16 + tree_bytes;
    }

    // ---- LL regions: identical layout in every window ------------------------------------------------------
    auto up = [](size_t v) { return (v + 127) & ~size_t(127); };
    size_t woff = up(8 * ALQ_MAX_WORLD);        // u64 ready[world] at offset 0
    for (int p = 0; p < P; ++p) {
        PGroup& g = groups[p];
        if (g.ncta == 0) continue;
        g.keyw = static_cast<unsigned int>(woff);  woff = up(woff + static_cast<size_t>(2) * world * g.seg_stride * 8);
        g.pickw = static_cast<unsigned int>(woff); woff = up(woff + 2 * 8);
        if (sample) {
            g.leafw = static_cast<unsigned int>(woff); woff = up(woff + static_cast<size_t>(2) * g.n_leaves * 8);
            g.massw = static_cast<unsigned int>(woff); woff = up(woff + static_cast<size_t>(2) * g.n_leaves * 16);
            g.umw = static_cast<unsigned int>(woff);   woff = up(woff + static_cast<size_t>(2) * world * g.seg_stride * 16);
        }
    }
    const size_t win_bytes = woff;
    if (comm && win_bytes > Gc.greedy_bytes())
        ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "alq_greedy_select: peer window too small (%zu needed, %zu usable)", win_bytes, Gc.greedy_bytes());

    // ---- scratch ----------------------------------------------------------------------------------------------
    const int total_picks = pick_off[P];
    const size_t need = scratch_need({segs.size() * sizeof(BlockSeg), groups.size() * sizeof(PGroup),
                                      leaf_off_all.size() * 4 + 4, level_off_all.size() * 4 + 4, sched_all.size() * 4 + 4,
                                      static_cast<size_t>(cfull_total) * 8 + 16, static_cast<size_t>(cfull_total) * 4 + 16,
                                      static_cast<size_t>(total_picks) * 8 + 8, segtab.size() * 4 + 4, ncta_tab.size() * 4 + 4,
                                      static_cast<size_t>(P + 1) * 4, static_cast<size_t>(P) * 4, 64, 64, comm ? 0 : win_bytes});
    int rc = alq_scratch_reserve(ctx, need);
    if (rc) return rc;
    ScratchCursor cur(ctx->scratch);
    BlockSeg* d_segs = cur.take<BlockSeg>(segs.size());
    PGroup* d_groups = cur.take<PGroup>(groups.size());
    int* d_leaf_off = cur.take<int>(leaf_off_all.size() + 1);
    int* d_level_off = cur.take<int>(level_off_all.size() + 1);
    unsigned int* d_sched = cur.take<unsigned int>(sched_all.size() + 1);
    unsigned long long* d_valw = cur.take<unsigned long long>(cfull_total + 2);
    int* d_posinv = cur.take<int>(cfull_total + 4);
    double* d_unif = cur.take<double>(total_picks + 1);
    int* d_segtab = cur.take<int>(segtab.size() + 1);
    int* d_ncta = cur.take<int>(ncta_tab.size() + 1);
    int* d_part_off = cur.take<int>(P + 1);
    int* d_cfull_off = cur.take<int>(P);
    int* d_status = cur.take<int>(1);
    unsigned long long* d_prof = cur.take<unsigned long long>(8);
    char* d_win = comm ? Gc.window : cur.take<char>(win_bytes);

    ALQ_CUDA(ctx, cudaMemcpyAsync(d_segs, segs.data(), segs.size() * sizeof(BlockSeg), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_groups, groups.data(), groups.size() * sizeof(PGroup), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_segtab, segtab.data(), segtab.size() * 4, cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_ncta, ncta_tab.data(), ncta_tab.size() * 4, cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemsetAsync(d_status, 0, sizeof(int), st));
    ALQ_CUDA(ctx, cudaMemsetAsync(d_prof, 0, 8 * sizeof(unsigned long long), st));
    // LL regions start without any valid tag (after the ready[] words; peers only write them after our ready flag)
    ALQ_CUDA(ctx, cudaMemsetAsync(d_win + up(8 * ALQ_MAX_WORLD), 0, win_bytes - up(8 * ALQ_MAX_WORLD), st));
    if (sample) {
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_leaf_off, leaf_off_all.data(), leaf_off_all.size() * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_level_off, level_off_all.data(), level_off_all.size() * 4, cudaMemcpyHostToDevice, st));
        if (!sched_all.empty())
            ALQ_CUDA(ctx, cudaMemcpyAsync(d_sched, sched_all.data(), sched_all.size() * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_unif, D->uniforms_host, static_cast<size_t>(total_picks) * 8, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_part_off, D->part_off_host, static_cast<size_t>(P + 1) * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemcpyAsync(d_cfull_off, cfull_off.data(), static_cast<size_t>(P) * 4, cudaMemcpyHostToDevice, st));
        ALQ_CUDA(ctx, cudaMemsetAsync(d_valw, 0, static_cast<size_t>(cfull_total + 2) * 8, st));
        ALQ_CUDA(ctx, cudaMemsetAsync(d_posinv, 0xff, static_cast<size_t>(cfull_total + 4) * 4, st));
        persist_posinv_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(D->vpos, d_part_off, d_cfull_off, P, static_cast<int>(n), d_posinv);
        ALQ_LAUNCH_CHECK(ctx);
    }

    PersistArgs A{};
    A.x = D->x; A.ldx = D->ldx; A.d = d;
    A.a = D->a; A.lda = D->lda; A.c = c;
    A.xn = D->xn; A.an = D->an;
    A.mind = D->mind; A.vpos = D->vpos;
    A.segs = d_segs; A.groups = d_groups;
    A.valw = d_valw; A.posinv = d_posinv;
    A.leaf_off = d_leaf_off; A.level_off = d_level_off; A.sched = d_sched; A.uniforms = d_unif;
    A.segtab = d_segtab; A.ncta_of_rank = d_ncta;
    A.picks = D->picks; A.status = d_status;
    A.prof = D->step_kernel_ms_host ? d_prof : nullptr;
    A.world = world; A.rank = rank;
    for (int r = 0; r < ALQ_MAX_WORLD; ++r) A.peer[r] = nullptr;
    if (comm) for (int r = 0; r < world; ++r) A.peer[r] = Gc.peer[r];
    else A.peer[0] = d_win;
    for (int r = 0; r <= ALQ_MAX_WORLD; ++r) A.leaf_bound[r] = leaf_bound[std::min(r, world)];
    A.ready_off = 0;
    ctx->comm.epoch += 1;
    A.ready_tag = comm ? ctx->comm.epoch << 32 : 0;   // 0: no handshake (one GPU, the window is scratch)
    A.tag_base = static_cast<unsigned int>(ctx->comm.epoch & 0x7fu) << 24 | 0x80000000u;   // never 0: a zeroed word is invalid
    A.timeout_cycles = ctx->spin_timeout_cycles();
    {   // L2 residency: keep `l2_resident_mb` of the rows this GPU streams in L2 across the steps (evict_last), split evenly over the CTAs
        const long long mb = ctx->l2_resident_mb;
        A.resident_rows = mb > 0 ? static_cast<int>(std::min<long long>((mb << 20) / static_cast<long long>(row_bytes) / std::max(grid, 1), 1 << 30)) : 0;
    }
    A.fast_path = ctx->d2_fast_path;

    if (comm) {
        rc = alq_comm_ready(ctx, A.ready_tag, st);       // after the clears above, in stream order
        if (rc) return rc;
    }
    const cudaError_t le = alq_gridsync_launch(ctx, st, [&] {
        if (factored) return sample ? launch_persist<true, true>(grid, smem, st, A, cfg, k_max, lc_max, ne_max, rm_max) : launch_persist<true, false>(grid, smem, st, A, cfg, k_max, lc_max, ne_max, rm_max);
        return sample ? launch_persist<false, true>(grid, smem, st, A, cfg, k_max, lc_max, ne_max, rm_max) : launch_persist<false, false>(grid, smem, st, A, cfg, k_max, lc_max, ne_max, rm_max);
    });
    if (le != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_greedy_select: cooperative launch failed: %s (grid %d, %zu B shared)", cudaGetErrorString(le), grid, smem);
    }

    int status = 0;
    unsigned long long prof[8] = {};
    if (sample || comm || D->step_kernel_ms_host) {
        ALQ_CUDA(ctx, cudaMemcpyAsync(&status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
        if (D->step_kernel_ms_host) ALQ_CUDA(ctx, cudaMemcpyAsync(prof, d_prof, sizeof(prof), cudaMemcpyDeviceToHost, st));
        ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    }
    if (D->step_kernel_ms_host) {
        const double steps = prof[2] ? static_cast<double>(prof[2]) : 1.0;
        D->step_kernel_ms_host[0] = static_cast<float>(prof[0] * 1e-6 / steps);
        D->step_kernel_ms_host[1] = static_cast<float>(prof[1] * 1e-6 / steps);
        D->step_kernel_ms_host[2] = static_cast<float>(prof[2]);
        D->step_kernel_ms_host[3] = 3.0f;
        D->step_kernel_ms_host[4] = static_cast<float>(prof[3] * 1e-6 / steps);
        D->step_kernel_ms_host[5] = static_cast<float>(prof[4] * 1e-6 / steps);
        D->step_kernel_ms_host[6] = static_cast<float>(prof[5] * 1e-6);      // t = 0 selection, ms
        D->step_kernel_ms_host[7] = static_cast<float>(prof[6] * 1e-6);      // whole kernel, ms
    }
    if (status == ALQ_ERR_STATE) ALQ_FAIL(ctx, status, "alq_greedy_select: timed out waiting for a peer GPU (or a CTA of this grid)");
    if (status != 0) ALQ_FAIL(ctx, status, "alq_greedy_select: non-finite or empty probability mass during D^2 sampling");
    return ALQ_OK;
}

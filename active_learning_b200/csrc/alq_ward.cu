// K7 / K8: Ward agglomerative clustering with a merge tree identical to scipy's, for MarginClusteringSampler
// (margin_clustering_sampler.py:59 under active_learning/src/query_strategies runs
// sklearn.cluster.AgglomerativeClustering(n_clusters=20), i.e. scipy.cluster.hierarchy.ward over the full tree).
//
// K7 alq_pdist_f64   scipy's pdist(X, 'euclidean') in fp64: fp32 rows widened to fp64 (exact), s summed k = 0, 1, ...
//                    by d2_step (alq_common.cuh: `d = a - b; s = s + d*d` with no FMA), then sqrt(s).  Two layouts of
//                    the result (below).
//                    One CTA owns a 64 x 64 tile of pairs of the upper triangle (each pair computed once; written to
//                    (i, j) and (j, i) of the square matrix, or once to the condensed vector);
//                    256 threads x 4 x 4 pairs in registers; k-chunks of both row blocks arrive
//                    with 4-byte cp.async (any ld, any alignment, zero-filled past d and past n) into a two-stage fp32
//                    ring and are widened once into an fp64 tile that the inner loop reads.
// K22 alq_herding_kernel  MaxHerdingSampler's Gaussian kernel matrix: K7's square-layout kernel with another epilogue,
//                    K_ij = K_ji = fl32(exp(-(s / q))) of the same fp64 s, into an n x n fp32 matrix (alq_herding.cu runs
//                    the greedy over it).  The diagonal s_ii is 0 for a finite row and NaN for a row with a NaN or
//                    infinite entry, so the diagonal tiles flag non-finite rows with no extra pass.
// K8 alq_ward_nn_chain  scipy's nn_chain (Ward update) as ONE launch of one thread-block cluster (16 CTAs when the GPU
//                    can place them, else 8).  CTA r owns columns [lo_r, hi_r) with their cluster sizes in shared
//                    memory.  A scan of row x: per-CTA (value, lowest index) -> DSMEM exchange -> every CTA resolves
//                    the same winner -> one cluster barrier.  A merge updates the CTA's slice of row y (and, in the
//                    square layout, the mirrored entries D[i, y] of its rows), then one cluster barrier.
//
// Layouts of D (both kernels are templated on it; nothing else depends on it):
//   square     the full symmetric n x n matrix, row-major with leading dimension ldd (8 n^2 bytes);
//   condensed  scipy's pdist vector: (i, j), i < j, at n i - i (i + 1) / 2 + (j - i - 1) (4 n (n - 1) bytes).  Row x
//              of the symmetric matrix is then the entries (j, x), j < x, one per row j (strided), and (x, j), j > x,
//              contiguous;
//   banded     (K8 only) the condensed vector cut into up to ALQ_MAX_WORLD bands of rows, each at its own pointer --
//              possibly in another GPU's memory, mapped through CUDA IPC (sharding.py: ShardGroup.ward_labels).  Band b
//              holds rows [cut[b], cut[b + 1]): (i, j), i < j, lies in the band of row i at cidx(i, j) - cidx(cut[b],
//              cut[b] + 1), exactly where alq_pdist_f64_condensed_rows puts it.  In a scan of row x the contiguous half
//              lies in x's band and each strided entry (j, x) in j's; a merge's store of (i, b) goes to min(i, b)'s band.
//
// Memory ordering of K8 (entries of D written by one SM and read by another): every write happens before a
// `barrier.cluster.arrive.release` of its CTA and every read after a `barrier.cluster.wait.acquire` of the reader;
// all reads of D go through ld.global.cg (L2, never a possibly stale L1 line) and all writes through st.global.cg.
// In the banded layout some bands live in a peer GPU's memory; the same argument holds there unchanged:
//   * during the launch the CTAs of this one cluster are the only readers and writers of every band: the peer that
//     owns a band synchronised its stream after its K7 before it handed out the band's handle, and it neither reads,
//     writes nor frees the band until this rank has broadcast the labels (after this launch has completed);
//   * the PTX memory model orders accesses by scope, not by where the memory lives: a weak st.global.cg before a
//     cluster-scope release and a weak ld.global.cg after the matching cluster-scope acquire of another thread of the
//     same cluster are ordered for every global address, NVLink peer memory included.  No access of another agent
//     (another GPU, the host) has to be ordered against them, so no gpu- or sys-scope fence is needed.  .cg keeps
//     the loads out of the SM's L1; a peer's bytes are served by the owning GPU's L2, the one point every access of
//     this cluster reaches.
// The peer's K7 writes themselves are complete before the launch: the kernel boundary of K7 and the peer's stream
// synchronisation order them before the host-side handle exchange, which precedes this launch.
//
// Offsets into `dist` are int64 (n^2 passes 2^31 at n = 46 341, n (n - 1) / 2 at n = 65 537); row indices themselves
// are int32.
#include <cooperative_groups.h>
#include <math_constants.h>

#include <climits>
#include <cmath>
#include <numeric>

#include "alq_common.cuh"

namespace cg = cooperative_groups;

namespace ward {

// offset of (i, j), i < j, in the condensed vector
__device__ __forceinline__ int64_t cidx(int i, int j, int n) {
    return static_cast<int64_t>(n) * i - static_cast<int64_t>(i) * (i + 1) / 2 + (j - i - 1);
}
enum class Layout { SQUARE, CONDENSED, BANDED };

// The banded layout's bands, by value (a __grid_constant__ kernel parameter).  base[b] is band b's pointer minus
// cidx(cut[b], cut[b] + 1), formed on the host, so that (i, j) of a row i of band b sits at base[b] + cidx(i, j) (the
// base itself may lie outside the band; only entries of the band's rows are dereferenced).  The cuts past the last
// band are n, so the band of row r is the number of cut[1 .. ALQ_MAX_WORLD) that are <= r.
struct Bands {
    double* base[ALQ_MAX_WORLD];
    int cut[ALQ_MAX_WORLD + 1];
};

__device__ __forceinline__ int band_of(const Bands& B, int r) {
    int b = 0;
#pragma unroll
    for (int k = 1; k < ALQ_MAX_WORLD; ++k) b += B.cut[k] <= r;
    return b;
}

// base[] of the band of row r for rows visited in ascending order (one thread's strided entries (j, x), j < x, of a scan,
// or its rows i of a merge): the band index only moves forward and the band's base is kept in a register, so an entry
// costs one compare and no load
struct BandCursor {
    const Bands& B;
    double* p;
    int b, next;
    __device__ __forceinline__ explicit BandCursor(const Bands& bands)
        : B(bands), p(bands.base[0]), b(0), next(bands.cut[1]) {}
    __device__ __forceinline__ double* base(int r) {
        while (r >= next) {
            next = B.cut[++b + 1];
            p = B.base[b];
        }
        return p;
    }
};

// row x's base: (x, j) sits at row + j -- for every j in the square layout, for j > x in the condensed one (where the
// base itself may lie before D: only row + j, j > x, is ever dereferenced)
template <Layout L>
__device__ __forceinline__ int64_t row_off(int x, int n, int64_t ldd) {
    if constexpr (L != Layout::SQUARE) return cidx(x, x + 1, n) - (x + 1);
    else return static_cast<int64_t>(x) * ldd;
}
template <Layout L>
__device__ __forceinline__ double* row_ptr(double* D, const Bands& B, int x, int n, int64_t ldd) {
    if constexpr (L == Layout::BANDED) return B.base[band_of(B, x)] + row_off<L>(x, n, ldd);
    else return D + row_off<L>(x, n, ldd);
}
// address of the symmetric entry (x, j), j != x, given row x's base (and, banded, the cursor over j's band)
template <Layout L, typename T>
__device__ __forceinline__ T* at(double* D, T* row, int x, int j, int n, BandCursor& bc) {
    if constexpr (L == Layout::BANDED) return j < x ? bc.base(j) + cidx(j, x, n) : row + j;
    else if constexpr (L == Layout::CONDENSED) return j < x ? D + cidx(j, x, n) : row + j;
    else return row + j;
}

// ---------------------------------------------------------------------------------------------------------------
// K7
// ---------------------------------------------------------------------------------------------------------------
constexpr int PD_TILE = 64;
constexpr int PD_KC = 16;
constexpr int PD_THREADS = 256;
constexpr int PD_PAD = PD_TILE + 1;      // fp32 staging row pitch: the transposed cp.async stores hit 32 banks

__device__ __forceinline__ void cp_async4(void* smem, const void* gmem, bool pred) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(pred ? 4 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// The band of rows [b.row_lo, b.row_hi): the grid's tile rows start at b.tile_lo = row_lo / PD_TILE, and in the
// condensed layout (i, j) lands at cidx(i, j) - b.base, base = cidx(row_lo, row_lo + 1), so a band is one contiguous
// slice of scipy's vector.  The square layout always takes the whole matrix and reads no field of b.
struct Band {
    int row_lo, row_hi, tile_lo;
    int64_t base;
};

// What the tile's epilogue writes: K7's sqrt(s) in the square or the condensed layout, or K22's fl32(exp(-(s / q))) in
// the square layout (T = float; `bad` counts the rows whose s_ii is not 0)
enum class PdOut { SQUARE, CONDENSED, GAUSS };
struct Gauss {
    double q;
    unsigned int* bad;
};

template <PdOut OUT, typename T>
__global__ void __launch_bounds__(PD_THREADS, 2)
pdist_f64_kernel(const float* __restrict__ x, int n, int d, int64_t ldx, T* __restrict__ dist, int64_t ldd,
                 const Band band, const Gauss gauss) {
    constexpr bool CONDENSED = OUT == PdOut::CONDENSED;
    const int ti = CONDENSED ? band.tile_lo + static_cast<int>(blockIdx.y) : static_cast<int>(blockIdx.y);
    const int tj = blockIdx.x;
    if (ti > tj) return;                                   // upper triangle of tiles only
    __shared__ float s32[2][2][PD_KC][PD_PAD];             // [stage][operand][k][row]
    __shared__ double s64[2][PD_KC][PD_TILE];              // [operand][k][row]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int row_i = ti * PD_TILE, row_j = tj * PD_TILE;
    const int nch = (d + PD_KC - 1) / PD_KC;

    auto issue = [&](int c, int stage) {
        const int k0 = c * PD_KC;
#pragma unroll
        for (int j = 0; j < (2 * PD_TILE * PD_KC) / PD_THREADS; ++j) {
            const int idx = tid + j * PD_THREADS;          // consecutive threads: consecutive k of one row
            const int op = idx / (PD_TILE * PD_KC), rem = idx % (PD_TILE * PD_KC);
            const int r = rem / PD_KC, k = rem % PD_KC;
            const int gr = (op ? row_j : row_i) + r, gk = k0 + k;
            const bool ok = gr < n && gk < d;
            cp_async4(&s32[stage][op][k][r], ok ? x + static_cast<int64_t>(gr) * ldx + gk : x, ok);
        }
        cp_async_commit();
    };

    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;

    issue(0, 0);
#pragma unroll 1
    for (int c = 0; c < nch; ++c) {
        cp_async_wait_all();
        __syncthreads();                                   // chunk c landed; the previous chunk's fp64 tile is consumed
        for (int idx = tid; idx < 2 * PD_KC * PD_TILE; idx += PD_THREADS) {
            const int op = idx / (PD_KC * PD_TILE), rem = idx % (PD_KC * PD_TILE);
            const int k = rem / PD_TILE, r = rem % PD_TILE;
            s64[op][k][r] = static_cast<double>(s32[c & 1][op][k][r]);
        }
        __syncthreads();
        if (c + 1 < nch) issue(c + 1, (c + 1) & 1);         // overlaps the compute below
#pragma unroll
        for (int k = 0; k < PD_KC; ++k) {
            double av[4], bv[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) av[a] = s64[0][k][ty + 16 * a];
#pragma unroll
            for (int b = 0; b < 4; ++b) bv[b] = s64[1][k][tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] = d2_step(acc[a][b], av[a], bv[b]);
        }
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int i = row_i + ty + 16 * a;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int j = row_j + tx + 16 * b;
            if constexpr (CONDENSED) {                     // no diagonal; consecutive tx: consecutive j
                if (band.row_lo <= i && i < band.row_hi && i < j && j < n)
                    dist[cidx(i, j, n) - band.base] = __dsqrt_rn(acc[a][b]);
            } else if (i < n && j < n && (ti != tj || i <= j)) {
                T v;
                if constexpr (OUT == PdOut::GAUSS) {
                    v = __double2float_rn(exp(-__ddiv_rn(acc[a][b], gauss.q)));
                    if (i == j && acc[a][b] != 0.0) atomicAdd(gauss.bad, 1u);
                } else {
                    v = __dsqrt_rn(acc[a][b]);
                }
                dist[static_cast<int64_t>(i) * ldd + j] = v;
                dist[static_cast<int64_t>(j) * ldd + i] = v;
            }
        }
    }
}

// The square matrix from condensed bands: for i in [row_lo, row_hi), j > i, dist[i, j] = dist[j, i] = the band's entry
// and dist[i, i] = 0.0.  HBM-bound; one CTA per 64 x 64 tile of the upper triangle, staged in shared memory so that the
// row-wise stores (consecutive threads: consecutive j) and the transposed ones (consecutive i) are both coalesced.
constexpr int EX_TILE = 64;
constexpr int EX_THREADS = 256;
constexpr int EX_ROWS = EX_THREADS / EX_TILE;              // tile rows per pass

__global__ void __launch_bounds__(EX_THREADS)
pdist_expand_kernel(const double* __restrict__ rows, int n, int row_lo, int row_hi, double* __restrict__ dist,
                    int64_t ldd) {
    const int ti = blockIdx.y + row_lo / EX_TILE, tj = blockIdx.x;
    if (ti > tj) return;
    __shared__ double t[EX_TILE][EX_TILE + 1];             // odd pitch: the transposed reads are conflict-free
    const int c = threadIdx.x % EX_TILE, r0 = threadIdx.x / EX_TILE;
    const int64_t base = cidx(row_lo, row_lo + 1, n);
    const int j = tj * EX_TILE + c;
#pragma unroll 4
    for (int r = r0; r < EX_TILE; r += EX_ROWS) {
        const int i = ti * EX_TILE + r;
        if (i < row_lo || i >= row_hi || j >= n || j < i) continue;
        if (j == i) {
            dist[static_cast<int64_t>(i) * ldd + i] = 0.0;
            continue;
        }
        const double v = rows[cidx(i, j, n) - base];
        dist[static_cast<int64_t>(i) * ldd + j] = v;
        t[r][c] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int r = r0; r < EX_TILE; r += EX_ROWS) {          // row jj of the tile's mirror, consecutive threads: consecutive i
        const int jj = tj * EX_TILE + r, i = ti * EX_TILE + c;
        if (i < row_lo || i >= row_hi || jj >= n || jj <= i) continue;
        dist[static_cast<int64_t>(jj) * ldd + i] = t[c][r];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// K8
// ---------------------------------------------------------------------------------------------------------------
constexpr int NC_THREADS = 512;
constexpr int NC_WARPS = NC_THREADS / 32;

struct Cand {               // a scan's partial result: value, lowest column attaining it, that column's cluster size
    double v;
    int i;
    int s;
};

__device__ __forceinline__ void cand_min(Cand& c, double v, int i, int s) {
    if (v < c.v || (v == c.v && i < c.i)) { c.v = v; c.i = i; c.s = s; }      // NaN never wins
}
__device__ __forceinline__ void warp_cand_min(Cand& c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double v = __shfl_xor_sync(0xffffffffu, c.v, o);
        const int i = __shfl_xor_sync(0xffffffffu, c.i, o);
        const int s = __shfl_xor_sync(0xffffffffu, c.s, o);
        cand_min(c, v, i, s);
    }
}

// scipy's _ward (_hierarchy_distance_update.pxi), evaluated left to right without contraction
__device__ __forceinline__ double ward_update(double dxi, double dyi, double dxy, int nx, int ny, int ni) {
    const double t = __ddiv_rn(1.0, static_cast<double>(nx + ny + ni));
    const double a = __dmul_rn(__dmul_rn(__dmul_rn(static_cast<double>(ni + nx), t), dxi), dxi);
    const double b = __dmul_rn(__dmul_rn(__dmul_rn(static_cast<double>(ni + ny), t), dyi), dyi);
    const double c = __dmul_rn(__dmul_rn(__dmul_rn(static_cast<double>(ni), t), dxy), dxy);
    return __dsqrt_rn(__dsub_rn(__dadd_rn(a, b), c));
}

// dist: n x n (ldd) or condensed, consumed; banded: D is unused and B names the bands (square and condensed: B is unused).
// chain_all: [cluster size][n] int2 (index, cluster size), one stack per CTA (every CTA
// walks the same chain; private copies need no cross-CTA ordering).  status: 0, or ALQ_ERR_NUMERIC if a scan of a
// one-element chain found no finite candidate (non-finite distances).
template <Layout L>
__global__ void __launch_bounds__(NC_THREADS, 1)
ward_chain_kernel(double* __restrict__ D, int n, int64_t ldd, int2* __restrict__ chain_all, int32_t* __restrict__ merge_xy,
                  double* __restrict__ merge_dist, int* __restrict__ status, const __grid_constant__ Bands B) {
    extern __shared__ int sz[];                            // cluster sizes of this CTA's columns, 0 = merged away
    __shared__ Cand part[2];                               // this CTA's scan result, double-buffered across scans
    __shared__ Cand wpart[NC_WARPS];
    __shared__ int2 first_live;                            // (lowest live column of this CTA, its size) or (INT_MAX, 0)
    cg::cluster_group cluster = cg::this_cluster();
    const int cs = static_cast<int>(cluster.num_blocks()), rank = static_cast<int>(cluster.block_rank());
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int slice = (n + cs - 1) / cs;
    const int lo = min(n, rank * slice), hi = min(n, lo + slice), cnt = hi - lo;
    int2* chain = chain_all + static_cast<int64_t>(rank) * n;

    for (int i = tid; i < cnt; i += NC_THREADS) sz[i] = 1;
    int fl = 0;                                            // first possibly-live local column (only moves forward)
    if (tid == 0) first_live = cnt > 0 ? make_int2(lo, 1) : make_int2(INT_MAX, 0);
    cluster_sync_all();

    int len = 0, par = 0;
    int x = 0, xs = 0, p = -1, ps = 0;                     // chain top and the element below it
#pragma unroll 1
    for (int k = 0; k < n - 1; ++k) {
        if (len == 0) {                                    // the chain restarts at the lowest live index
            int2 f = make_int2(INT_MAX, 0);
            if (lane < cs) f = *cluster.map_shared_rank(&first_live, lane);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const int oi = __shfl_xor_sync(0xffffffffu, f.x, o), os = __shfl_xor_sync(0xffffffffu, f.y, o);
                if (oi < f.x) { f.x = oi; f.y = os; }
            }
            x = f.x; xs = f.y; p = -1; ps = 0;
            if (tid == 0) chain[0] = f;
            len = 1;
        }
        double cur;
#pragma unroll 1
        while (true) {
            // ---- scan row x over this CTA's live columns -------------------------------------------------------
            const double* row = row_ptr<L>(D, B, x, n, ldd);
            BandCursor bc(B);
            Cand c{CUDART_INF, INT_MAX, 0};
            int i = lo + tid;
#pragma unroll 1
            for (; i + 3 * NC_THREADS < hi; i += 4 * NC_THREADS) {
                double v[4];
                bool live[4];
                const double* ad[4];                       // banded: the cursor's branches come before the four
#pragma unroll                                             // loads, not between them
                for (int u = 0; u < 4; ++u) {
                    const int j = i + u * NC_THREADS;
                    live[u] = sz[j - lo] > 0 && j != x;
                    if constexpr (L == Layout::BANDED) ad[u] = at<L>(D, row, x, j, n, bc);
                    else v[u] = live[u] ? __ldcg(at<L>(D, row, x, j, n, bc)) : CUDART_INF;
                }
                if constexpr (L == Layout::BANDED) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) v[u] = live[u] ? __ldcg(ad[u]) : CUDART_INF;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (live[u] && v[u] < c.v) { c.v = v[u]; c.i = i + u * NC_THREADS; c.s = sz[i + u * NC_THREADS - lo]; }
            }
            for (; i < hi; i += NC_THREADS) {
                const int s = sz[i - lo];
                if (s > 0 && i != x) {
                    const double v = __ldcg(at<L>(D, row, x, i, n, bc));
                    if (v < c.v) { c.v = v; c.i = i; c.s = s; }
                }
            }
            warp_cand_min(c);
            if (lane == 0) wpart[warp] = c;
            __syncthreads();
            if (warp == 0) {
                c = lane < NC_WARPS ? wpart[lane] : Cand{CUDART_INF, INT_MAX, 0};
                warp_cand_min(c);
                if (lane == 0) part[par] = c;
            }
            cluster_sync_all();                            // the scan's one cluster barrier
            // ---- every warp resolves the same winner from the cs partial results (DSMEM) ----------------------
            Cand m{CUDART_INF, INT_MAX, 0};
            if (lane < cs) m = *cluster.map_shared_rank(&part[par], lane);
            warp_cand_min(m);
            par ^= 1;                                      // part[par] is rewritten only after one more barrier
            BandCursor pc(B);
            cur = p >= 0 ? __ldcg(at<L>(D, row, x, p, n, pc)) : CUDART_INF;   // scipy starts from D[x, prev]: ties go to prev
            int y, ys;
            if (m.v < cur) { y = m.i; ys = m.s; cur = m.v; }
            else { y = p; ys = ps; }
            if (p >= 0 && y == p) break;
            if (y < 0 || y == INT_MAX) {                   // no finite candidate (non-finite input): give up uniformly
                if (rank == 0 && tid == 0) *status = ALQ_ERR_NUMERIC;
                cluster_sync_all();                        // no CTA exits while a peer still reads its part[] (DSMEM)
                return;
            }
            if (tid == 0) chain[len] = make_int2(y, ys);
            ++len;
            p = x; ps = xs; x = y; xs = ys;
        }
        // ---- merge the mutual nearest neighbours x (top) and p -----------------------------------------------------
        len -= 2;
        const int a = min(x, p), b = max(x, p);            // fastcluster's convention: the new cluster keeps index b
        const int na = a == x ? xs : ps, nb = a == x ? ps : xs;
        if (rank == 0 && tid == 0) {
            merge_xy[2 * static_cast<int64_t>(k)] = a;
            merge_xy[2 * static_cast<int64_t>(k) + 1] = b;
            merge_dist[k] = cur;
        }
        const double* rowa = row_ptr<L>(D, B, a, n, ldd);
        double* rowb = row_ptr<L>(D, B, b, n, ldd);
        BandCursor bc(B);
        for (int i = lo + tid; i < hi; i += NC_THREADS) {
            const int ni = sz[i - lo];
            if (ni > 0 && i != a && i != b) {
                if constexpr (L != Layout::SQUARE) {       // one store per (i, b)
                    double* bi = at<L>(D, rowb, b, i, n, bc);
                    __stcg(bi, ward_update(__ldcg(at<L>(D, rowa, a, i, n, bc)), __ldcg(bi), cur, na, nb, ni));
                } else {                                   // row b and the mirrored column
                    const double v = ward_update(__ldcg(rowa + i), __ldcg(rowb + i), cur, na, nb, ni);
                    __stcg(rowb + i, v);
                    __stcg(D + static_cast<int64_t>(i) * ldd + b, v);
                }
            }
        }
        __syncthreads();
        if (tid == 0) {
            if (a >= lo && a < hi) sz[a - lo] = 0;
            if (b >= lo && b < hi) sz[b - lo] = na + nb;
            while (fl < cnt && sz[fl] == 0) ++fl;
            first_live = fl < cnt ? make_int2(lo + fl, sz[fl]) : make_int2(INT_MAX, 0);
        }
        if (len > 0) {                                     // the stack below the merged pair is unchanged; its entries
            const int2 t = __ldcg(chain + len - 1);        // were written by this CTA's thread 0 before a __syncthreads
            x = t.x; xs = t.y;
            if (len > 1) { const int2 q = __ldcg(chain + len - 2); p = q.x; ps = q.y; }
            else { p = -1; ps = 0; }
        }
        cluster_sync_all();                                // the merge's one cluster barrier
    }
}

template <Layout L>
int ward_cluster_size(alq_ctx* ctx, size_t smem, int* out) {
    auto* kern = ward_chain_kernel<L>;
    ALQ_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    ALQ_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    for (int cs : {16, 8}) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cs);
        cfg.blockDim = dim3(NC_THREADS);
        cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = cs;
        attr.val.clusterDim.y = 1;
        attr.val.clusterDim.z = 1;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        int nclusters = 0;
        if (cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg) == cudaSuccess && nclusters > 0) {
            *out = cs;
            return ALQ_OK;
        }
        (void)cudaGetLastError();
    }
    ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_ward_nn_chain: no thread-block cluster of 8 or 16 CTAs fits this GPU");
}

// ---- host twins of scipy's label() and sklearn's _hc_cut ------------------------------------------------------
struct LinkageUnionFind {                                  // scipy/cluster/_hierarchy.pyx
    std::vector<int64_t> parent, size;
    int64_t next_label;
    explicit LinkageUnionFind(int64_t n) : parent(2 * n - 1), size(2 * n - 1, 1), next_label(n) {
        std::iota(parent.begin(), parent.end(), 0);
    }
    int64_t merge(int64_t x, int64_t y) {
        parent[x] = next_label;
        parent[y] = next_label;
        const int64_t s = size[x] + size[y];
        size[next_label] = s;
        ++next_label;
        return s;
    }
    int64_t find(int64_t x) {
        int64_t p = x;
        while (parent[x] != x) x = parent[x];
        while (parent[p] != x) { const int64_t q = parent[p]; parent[p] = x; p = q; }
        return x;
    }
};

// Python's heapq (_siftdown / _siftup), so that the final heap order -- which numbers sklearn's labels -- matches
void heap_siftdown(std::vector<int64_t>& h, size_t start, size_t pos) {
    const int64_t item = h[pos];
    while (pos > start) {
        const size_t parent = (pos - 1) >> 1;
        if (item < h[parent]) { h[pos] = h[parent]; pos = parent; continue; }
        break;
    }
    h[pos] = item;
}
void heap_siftup(std::vector<int64_t>& h, size_t pos) {
    const size_t end = h.size(), start = pos;
    const int64_t item = h[pos];
    size_t child = 2 * pos + 1;
    while (child < end) {
        const size_t right = child + 1;
        if (right < end && !(h[child] < h[right])) child = right;
        h[pos] = h[child];
        pos = child;
        child = 2 * pos + 1;
    }
    h[pos] = item;
    heap_siftdown(h, start, pos);
}
void heap_push(std::vector<int64_t>& h, int64_t item) {
    h.push_back(item);
    heap_siftdown(h, 0, h.size() - 1);
}
void heap_pushpop(std::vector<int64_t>& h, int64_t item) {
    if (!h.empty() && h[0] < item) {
        h[0] = item;
        heap_siftup(h, 0);
    }
}

// K7 launches for either layout over the rows [row_lo, row_hi) (the square layout always takes [0, n)); `name` is the
// entry point's, for its error messages
template <PdOut OUT, typename T>
int pdist_run(alq_ctx* ctx, const char* name, const float* x, int64_t n, int32_t d, int64_t ldx, T* dist, int64_t ldd,
              int64_t row_lo, int64_t row_hi, void* stream, Gauss gauss = Gauss{1.0, nullptr}) {
    const int64_t nt = (n + PD_TILE - 1) / PD_TILE;
    if (nt > 65535) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: n=%lld exceeds %d rows", name, (long long)n, 65535 * PD_TILE);
    const int64_t t0 = row_lo / PD_TILE, t1 = (row_hi + PD_TILE - 1) / PD_TILE;
    if (t1 <= t0) return ALQ_OK;                           // an empty band writes nothing
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    pdist_f64_kernel<OUT, T><<<dim3(static_cast<unsigned>(nt), static_cast<unsigned>(t1 - t0)), PD_THREADS, 0,
                               static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<int>(n), d, ldx, dist, ldd,
        Band{static_cast<int>(row_lo), static_cast<int>(row_hi), static_cast<int>(t0), row_lo * n - row_lo * (row_lo + 1) / 2},
        gauss);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

template <Layout L>
int nn_chain_run(alq_ctx* ctx, const char* name, double* dist, int64_t n, int64_t ldd, const Bands& bands,
                 int32_t* merge_xy, double* merge_dist, void* stream) {
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = static_cast<size_t>((n + 7) / 8) * sizeof(int) + 16;   // sized for the 8-CTA fallback
    if (smem + 4096 > ctx->smem_optin)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "%s: n=%lld does not fit the shared memory of a cluster", name, (long long)n);
    int cs = 0;
    int rc = ward_cluster_size<L>(ctx, smem, &cs);
    if (rc) return rc;
    rc = alq_scratch_reserve(ctx, scratch_need({static_cast<size_t>(cs) * n * sizeof(int2), sizeof(int)}));
    if (rc) return rc;
    ScratchCursor cur(ctx->scratch);
    int2* chain = cur.take<int2>(static_cast<size_t>(cs) * n);
    int* status = cur.take<int>(1);
    ALQ_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int), st));

    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs);
    cfg.blockDim = dim3(NC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cs;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    ALQ_CUDA(ctx, cudaLaunchKernelEx(&cfg, ward_chain_kernel<L>, dist, static_cast<int>(n), ldd, chain, merge_xy,
                                     merge_dist, status, bands));
    ALQ_LAUNCH_CHECK(ctx);
    int h_status = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h_status, status, sizeof(int), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (h_status) ALQ_FAIL(ctx, ALQ_ERR_NUMERIC, "%s: a chain scan found no finite distance (non-finite input)", name);
    return ALQ_OK;
}

}  // namespace ward

using namespace ward;

extern "C" int alq_pdist_f64(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, double* dist, int64_t ldd,
                             void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!x || !dist || n < 1 || d < 1 || ldx < d || ldd < n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_pdist_f64: bad arguments (n=%lld d=%d ldx=%lld ldd=%lld)", (long long)n, d,
                 (long long)ldx, (long long)ldd);
    return pdist_run<PdOut::SQUARE>(ctx, "alq_pdist_f64", x, n, d, ldx, dist, ldd, 0, n, stream);
}

extern "C" int alq_pdist_f64_condensed(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, double* dist,
                                       void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!x || !dist || n < 1 || d < 1 || ldx < d)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_pdist_f64_condensed: bad arguments (n=%lld d=%d ldx=%lld)", (long long)n, d,
                 (long long)ldx);
    return pdist_run<PdOut::CONDENSED>(ctx, "alq_pdist_f64_condensed", x, n, d, ldx, dist, 0, 0, n, stream);
}

extern "C" int alq_pdist_f64_condensed_rows(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx,
                                            int64_t row_lo, int64_t row_hi, double* dist, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!x || !dist || n < 1 || d < 1 || ldx < d || row_lo < 0 || row_hi > n || row_lo > row_hi)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_pdist_f64_condensed_rows: bad arguments (n=%lld d=%d ldx=%lld rows [%lld, %lld))",
                 (long long)n, d, (long long)ldx, (long long)row_lo, (long long)row_hi);
    return pdist_run<PdOut::CONDENSED>(ctx, "alq_pdist_f64_condensed_rows", x, n, d, ldx, dist, 0, row_lo, row_hi, stream);
}

extern "C" int alq_herding_kernel(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, const double* q_host,
                                  float* k, int64_t ldk, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!x || !k || !q_host || n < 1 || d < 1 || ldx < d || ldk < n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_herding_kernel: bad arguments (n=%lld d=%d ldx=%lld ldk=%lld)", (long long)n, d,
                 (long long)ldx, (long long)ldk);
    const double q = *q_host;
    if (!(std::isfinite(q) && std::fpclassify(q) == FP_NORMAL && q > 0.0))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_herding_kernel: q=%g must be a finite positive normal number", q);
    int rc = alq_scratch_reserve(ctx, scratch_need({sizeof(unsigned int)}));
    if (rc) return rc;
    unsigned int* bad = ScratchCursor(ctx->scratch).take<unsigned int>(1);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    ALQ_CUDA(ctx, cudaMemsetAsync(bad, 0, sizeof(unsigned int), st));
    rc = pdist_run<PdOut::GAUSS>(ctx, "alq_herding_kernel", x, n, d, ldx, k, ldk, 0, n, stream, Gauss{q, bad});
    if (rc) return rc;
    unsigned int h = 0;
    ALQ_CUDA(ctx, cudaMemcpyAsync(&h, bad, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    ALQ_CUDA(ctx, cudaStreamSynchronize(st));
    if (h) ALQ_FAIL(ctx, ALQ_ERR_NUMERIC, "alq_herding_kernel: %u rows hold a NaN or infinite entry", h);
    return ALQ_OK;
}

extern "C" int alq_pdist_f64_expand(alq_ctx* ctx, const double* rows, int64_t n, int64_t row_lo, int64_t row_hi,
                                    double* dist, int64_t ldd, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!rows || !dist || n < 1 || ldd < n || row_lo < 0 || row_hi > n || row_lo > row_hi)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_pdist_f64_expand: bad arguments (n=%lld ldd=%lld rows [%lld, %lld))",
                 (long long)n, (long long)ldd, (long long)row_lo, (long long)row_hi);
    const int64_t nt = (n + EX_TILE - 1) / EX_TILE;
    if (nt > 65535)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_pdist_f64_expand: n=%lld exceeds %d rows", (long long)n, 65535 * EX_TILE);
    const int64_t t0 = row_lo / EX_TILE, t1 = (row_hi + EX_TILE - 1) / EX_TILE;
    if (t1 <= t0) return ALQ_OK;
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    pdist_expand_kernel<<<dim3(static_cast<unsigned>(nt), static_cast<unsigned>(t1 - t0)), EX_THREADS, 0,
                          static_cast<cudaStream_t>(stream)>>>(rows, static_cast<int>(n), static_cast<int>(row_lo),
                                                               static_cast<int>(row_hi), dist, ldd);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_ward_nn_chain(alq_ctx* ctx, double* dist, int64_t n, int64_t ldd, int32_t* merge_xy, double* merge_dist,
                                 void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!dist || !merge_xy || !merge_dist || n < 2 || n >= (1LL << 31) - 1 || ldd < n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ward_nn_chain: bad arguments (n=%lld ldd=%lld)", (long long)n, (long long)ldd);
    return nn_chain_run<Layout::SQUARE>(ctx, "alq_ward_nn_chain", dist, n, ldd, Bands{}, merge_xy, merge_dist, stream);
}

extern "C" int alq_ward_nn_chain_condensed(alq_ctx* ctx, double* dist, int64_t n, int32_t* merge_xy, double* merge_dist,
                                           void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!dist || !merge_xy || !merge_dist || n < 2 || n >= (1LL << 31) - 1)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ward_nn_chain_condensed: bad arguments (n=%lld)", (long long)n);
    return nn_chain_run<Layout::CONDENSED>(ctx, "alq_ward_nn_chain_condensed", dist, n, 0, Bands{}, merge_xy, merge_dist,
                                           stream);
}

extern "C" int alq_ward_nn_chain_banded(alq_ctx* ctx, const int64_t* row_cuts_host, void* const* bands_host,
                                        int32_t nbands, int64_t n, int32_t* merge_xy, double* merge_dist, void* stream) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!row_cuts_host || !bands_host || !merge_xy || !merge_dist || nbands < 1 || nbands > ALQ_MAX_WORLD || n < 2 ||
        n >= (1LL << 31) - 1)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ward_nn_chain_banded: bad arguments (n=%lld nbands=%d, max %d bands)",
                 (long long)n, nbands, ALQ_MAX_WORLD);
    if (row_cuts_host[0] != 0 || row_cuts_host[nbands] != n)
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ward_nn_chain_banded: the cuts must run from 0 to n=%lld (got %lld .. %lld)",
                 (long long)n, (long long)row_cuts_host[0], (long long)row_cuts_host[nbands]);
    Bands B{};
    for (int b = 0; b <= ALQ_MAX_WORLD; ++b) B.cut[b] = static_cast<int>(n);
    for (int b = 0; b < nbands; ++b) {
        const int64_t lo = row_cuts_host[b], hi = row_cuts_host[b + 1];
        if (hi < lo)
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ward_nn_chain_banded: cut %d (%lld) is below cut %d (%lld)", b + 1,
                     (long long)hi, b, (long long)lo);
        const int64_t start = lo * n - lo * (lo + 1) / 2;          // cidx(lo, lo + 1): the band's first entry
        const int64_t pairs = hi * n - hi * (hi + 1) / 2 - start;
        if (pairs > 0 && !bands_host[b])
            ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_ward_nn_chain_banded: band %d (rows [%lld, %lld)) has pairs but no pointer",
                     b, (long long)lo, (long long)hi);
        B.cut[b] = static_cast<int>(lo);
        B.base[b] = reinterpret_cast<double*>(reinterpret_cast<uintptr_t>(bands_host[b]) -
                                              static_cast<uintptr_t>(start) * sizeof(double));
    }
    return nn_chain_run<Layout::BANDED>(ctx, "alq_ward_nn_chain_banded", nullptr, n, 0, B, merge_xy, merge_dist, stream);
}

extern "C" int alq_ward_labels(const int32_t* merge_xy_host, const double* merge_dist_host, int64_t n, int32_t n_clusters,
                               int32_t* labels_host) {
    if (!merge_xy_host || !merge_dist_host || !labels_host || n < 2 || n >= (1LL << 31) || n_clusters < 1 || n_clusters > n)
        return ALQ_ERR_INVALID;
    const int64_t m = n - 1;
    for (int64_t k = 0; k < m; ++k) {
        const int64_t a = merge_xy_host[2 * k], b = merge_xy_host[2 * k + 1];
        if (a < 0 || b < 0 || a >= n || b >= n || a == b || std::isnan(merge_dist_host[k])) return ALQ_ERR_INVALID;
    }
    // scipy's nn_chain epilogue: stable sort by distance (np.argsort kind='mergesort'), then label() by union-find
    std::vector<int64_t> order(m);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(),
                     [&](int64_t u, int64_t v) { return merge_dist_host[u] < merge_dist_host[v]; });
    LinkageUnionFind uf(n);
    std::vector<int64_t> children(2 * m);
    for (int64_t r = 0; r < m; ++r) {
        const int64_t k = order[r];
        const int64_t xr = uf.find(merge_xy_host[2 * k]), yr = uf.find(merge_xy_host[2 * k + 1]);
        // the n - 1 pairs, taken as edges, must form a spanning tree (in any order: no edge closes a cycle), which is
        // what makes every leaf end up under the root and labelled
        if (xr == yr) return ALQ_ERR_INVALID;
        children[2 * r] = std::min(xr, yr);
        children[2 * r + 1] = std::max(xr, yr);
        uf.merge(xr, yr);
    }
    // sklearn's _hc_cut: a heap of negated node ids, labels numbered in the heap's final order
    std::vector<int64_t> nodes{-(std::max(children[2 * (m - 1)], children[2 * (m - 1) + 1]) + 1)};
    for (int32_t t = 0; t < n_clusters - 1; ++t) {
        const int64_t node = -nodes[0] - n;
        heap_push(nodes, -children[2 * node]);
        heap_pushpop(nodes, -children[2 * node + 1]);
    }
    std::vector<int64_t> stack;
    for (size_t l = 0; l < nodes.size(); ++l) {
        stack.assign(1, -nodes[l]);
        while (!stack.empty()) {
            const int64_t v = stack.back();
            stack.pop_back();
            if (v < n) { labels_host[v] = static_cast<int32_t>(l); continue; }
            stack.push_back(children[2 * (v - n)]);
            stack.push_back(children[2 * (v - n) + 1]);
        }
    }
    return ALQ_OK;
}

// K3 on the Hopper tensor cores: out[i] = min_j (max_j) fl(fl(xn_i + yn_j) - 2 <x_i, y_j>)
// for fp32 rows, as a wgmma "3xTF32" contraction with the min-epilogue fused on the register
// accumulators.  Same contract as the SIMT kernel in alq_mindist.cu (coreset_sampler.py:59-64,79,100
// of the reference's query_strategies); this is the one dense contraction on the query path.
//
// fp32 fidelity.  .tf32 keeps 10 mantissa bits, so each operand is split once, ahead of time,
// into two valid TF32 numbers  x = hi + lo + r,  hi = rna_tf32(x), lo = rna_tf32(x - hi), |r| <= 2^-22|x|,
// and every k-step issues three MMAs into the same fp32 accumulator:  hi*hi' + hi*lo' + lo*hi'.
// The dropped lo*lo' and r terms are <= 2^-21 |x||y| per product.  Small integers (the exact-arithmetic
// parity fixtures) have lo == 0 and give bit-identical results to fp32.
//
// Structure (one CTA per SM, persistent over a host-built work list, 3 warpgroups):
//   warpgroup 0   TMA producer (one thread): 4 tensor maps (X_hi, X_lo, Y_hi, Y_lo), boxes of 32 fp32
//                 (=128 B, SWIZZLE_128B) x 128 rows into a 3-stage shared-memory ring, mbarrier complete_tx.
//   warpgroups 1-2 consumers: each owns 64 of the tile's 128 rows and issues
//                 wgmma.mma_async.m64n128k8.f32.tf32.tf32 from shared memory (12 per stage, one stage kept
//                 in flight), then the distance + running row min on its register accumulators; one float
//                 atomic per row at the end of a work item.  The factored/BADGE form keeps two accumulators
//                 (<h,h'> and <a,a'>) and multiplies them in the epilogue.
// Every CTA sweeps the column tiles in the same order, so a Y tile is fetched from HBM once and
// served to the other CTAs from L2.
#include <cuda.h>
#include <stdlib.h>

#include "alq_common.cuh"

namespace tc {

constexpr int BM = 128;          // rows per tile (two m64 warpgroups)
constexpr int BN = 128;          // cols per tile (wgmma N)
constexpr int BK = 32;           // fp32 per stage row = 128 bytes = one swizzle span
constexpr int UK = 8;            // wgmma K for tf32
constexpr int STAGES = 3;
constexpr int A_BYTES = BM * BK * 4;              // 16 KB
constexpr int B_BYTES = BN * BK * 4;              // 16 KB
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;   // hi + lo of both operands = 64 KB
constexpr int THREADS = 384;

struct WorkItem {
    int m_blk, n_begin, n_end, pad;   // row block, [first, last) column tile
};

struct Params {
    const float* xn; const float* yn;      // row norms (already multiplied by the a-norms when factored)
    float* out;
    const WorkItem* items;                 // [grid][items_per_cta]
    const int* item_count;                 // [grid]
    int items_per_cta;
    int n, m;                              // rows of X / Y
    int kblocks_h, kblocks_a;              // ceil(d / 32), ceil(c / 32) (0 when dense)
};

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (PTX ISA, "Matrix Descriptor Format" of wgmma):
//   bits [0,14) start address >> 4, [16,30) leading byte offset >> 4 (= 1, unused for swizzled K-major),
//   [32,46) stride byte offset >> 4 (= 1024 B: 8 rows x 128 B), [62,64) swizzle mode = 1 (128 B).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fff);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// d (64 x 128 fp32, the m64n128 register fragment) += A (64 x 8, smem) * B (128 x 8, smem)^T;  scale_d == 0 overwrites d
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

template <bool FACTORED, bool RED_MAX>
__global__ void __launch_bounds__(THREADS, 1)
min_dist_tc_kernel(const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
                   const __grid_constant__ CUtensorMap map_yh, const __grid_constant__ CUtensorMap map_yl,
                   const __grid_constant__ CUtensorMap map_xah, const __grid_constant__ CUtensorMap map_xal,
                   const __grid_constant__ CUtensorMap map_yah, const __grid_constant__ CUtensorMap map_yal,
                   Params P) {
    extern __shared__ unsigned char smem_dyn[];
    // SWIZZLE_128B tiles must sit on 1024-byte boundaries: align by hand (1 KB of slack is allocated)
    unsigned char* smem_raw = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    unsigned char* stage_base = smem_raw;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;

    const int wg = threadIdx.x >> 7;
    const int n_items = P.item_count[blockIdx.x];
    const WorkItem* items = P.items + static_cast<size_t>(blockIdx.x) * P.items_per_cta;
    const int kb_total = P.kblocks_h + (FACTORED ? P.kblocks_a : 0);

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ================= TMA producer =================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            for (int w = 0; w < n_items; ++w) {
                const WorkItem wi = items[w];
                for (int nt = wi.n_begin; nt < wi.n_end; ++nt) {
                    for (int kb = 0; kb < kb_total; ++kb, ++it) {
                        const int s = it % STAGES;
                        const uint32_t round = it / STAGES;
                        if (round > 0) mbar_wait(&empty[s], (round - 1) & 1u);
                        unsigned char* st = stage_base + static_cast<size_t>(s) * STAGE_BYTES;
                        mbar_expect_tx(&full[s], STAGE_BYTES);
                        const bool apart = FACTORED && kb >= P.kblocks_h;
                        const int k0 = (apart ? kb - P.kblocks_h : kb) * BK;
                        tma_load_2d(st, apart ? &map_xah : &map_xh, k0, wi.m_blk * BM, &full[s]);
                        tma_load_2d(st + A_BYTES, apart ? &map_xal : &map_xl, k0, wi.m_blk * BM, &full[s]);
                        tma_load_2d(st + 2 * A_BYTES, apart ? &map_yah : &map_yh, k0, nt * BN, &full[s]);
                        tma_load_2d(st + 2 * A_BYTES + B_BYTES, apart ? &map_yal : &map_yl, k0, nt * BN, &full[s]);
                    }
                }
            }
        }
    } else {
        // ================= consumers: warpgroup wg - 1 owns rows [64 (wg - 1), 64 wg) of the tile =================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
        const uint32_t a_off = static_cast<uint32_t>(wg - 1) * 64 * BK * 4;     // 8 KB: a whole number of swizzle atoms
        // m64nN fp32 fragment: d[4j + {0,1}] = (r, 8j + 2 (lane % 4) + {0,1}), d[4j + {2,3}] = (r + 8, same cols),
        // r = 16 warp + lane / 4
        const int r_in_tile = (wg - 1) * 64 + warp * 16 + (lane >> 2);
        const int c_in_tile = 2 * (lane & 3);
        uint32_t it = 0;
        for (int w = 0; w < n_items; ++w) {
            const WorkItem wi = items[w];
            const int row0 = wi.m_blk * BM + r_in_tile, row1 = row0 + 8;
            const float rn0 = row0 < P.n ? P.xn[row0] : 0.f, rn1 = row1 < P.n ? P.xn[row1] : 0.f;
            float best0 = RED_MAX ? ALQ_NEG_INF : ALQ_POS_INF, best1 = best0;
            for (int nt = wi.n_begin; nt < wi.n_end; ++nt) {
                float acc[64];
                float acc_a[FACTORED ? 64 : 1];
                int prev = -1;
                for (int kb = 0; kb < kb_total; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&full[s], (it / STAGES) & 1u);
                    const bool apart = FACTORED && kb >= P.kblocks_h;
                    const bool first_kb = apart ? (kb == P.kblocks_h) : (kb == 0);
                    const uint32_t a_hi = smem_u32(stage_base + static_cast<size_t>(s) * STAGE_BYTES) + a_off;
                    const uint32_t a_lo = a_hi + A_BYTES, b_hi = a_hi - a_off + 2 * A_BYTES, b_lo = b_hi + B_BYTES;
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / UK; ++k) {
                        const uint32_t off = k * UK * 4;    // bytes along K inside the 128-byte swizzle span
                        const uint64_t dah = make_desc(a_hi + off), dal = make_desc(a_lo + off);
                        const uint64_t dbh = make_desc(b_hi + off), dbl = make_desc(b_lo + off);
                        const uint32_t sc = (first_kb && k == 0) ? 0u : 1u;
                        if constexpr (FACTORED) {
                            if (apart) {
                                wgmma_tf32(acc_a, dah, dbh, sc);
                                wgmma_tf32(acc_a, dah, dbl, 1u);
                                wgmma_tf32(acc_a, dal, dbh, 1u);
                                continue;
                            }
                        }
                        wgmma_tf32(acc, dah, dbh, sc);
                        wgmma_tf32(acc, dah, dbl, 1u);
                        wgmma_tf32(acc, dal, dbh, 1u);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                          // the previous stage's MMAs have retired: hand it back
                    if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);
                    prev = s;
                }
                wgmma_wait<0>();
                if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = nt * BN + 8 * j + c_in_tile;
                    const float pad = RED_MAX ? ALQ_NEG_INF : ALQ_POS_INF;
                    const float cn0 = col < P.m ? __ldg(P.yn + col) : pad;
                    const float cn1 = col + 1 < P.m ? __ldg(P.yn + col + 1) : pad;
                    float v[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};
                    if constexpr (FACTORED) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) v[e] = v[e] * acc_a[4 * j + e];
                    }
                    const float d00 = (rn0 + cn0) - 2.0f * v[0], d01 = (rn0 + cn1) - 2.0f * v[1];
                    const float d10 = (rn1 + cn0) - 2.0f * v[2], d11 = (rn1 + cn1) - 2.0f * v[3];
                    if (RED_MAX) { best0 = fmaxf(best0, fmaxf(d00, d01)); best1 = fmaxf(best1, fmaxf(d10, d11)); }
                    else { best0 = fminf(best0, fminf(d00, d01)); best1 = fminf(best1, fminf(d10, d11)); }
                }
            }
            // the four lanes of a quad hold the same two rows
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                const float b0 = __shfl_xor_sync(0xffffffffu, best0, o), b1 = __shfl_xor_sync(0xffffffffu, best1, o);
                best0 = RED_MAX ? fmaxf(best0, b0) : fminf(best0, b0);
                best1 = RED_MAX ? fmaxf(best1, b1) : fminf(best1, b1);
            }
            if ((lane & 3) == 0 && wi.n_end > wi.n_begin) {
                if (row0 < P.n) { if (RED_MAX) atomic_max_float(P.out + row0, best0); else atomic_min_float(P.out + row0, best0); }
                if (row1 < P.n) { if (RED_MAX) atomic_max_float(P.out + row1, best1); else atomic_min_float(P.out + row1, best1); }
            }
        }
    }
}

// hi = rna_tf32(x), lo = rna_tf32(x - hi): two valid TF32 operands whose sum is x to 2^-22 relative
__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, int64_t rows, int d, int64_t ld, float* __restrict__ hi,
                  float* __restrict__ lo) {
    const int64_t total = rows * (d >> 2);
    const int dv = d >> 2;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t r = i / dv;
        const int k = static_cast<int>(i - r * dv);
        const float4 v = ld_stream_f4(reinterpret_cast<const float4*>(x + r * ld) + k);
        const float e[4] = {v.x, v.y, v.z, v.w};
        float h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            uint32_t hb, lb;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(e[j]));
            h[j] = __uint_as_float(hb);
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(e[j] - h[j]));
            l[j] = __uint_as_float(lb);
        }
        reinterpret_cast<float4*>(hi + r * d)[k] = make_float4(h[0], h[1], h[2], h[3]);
        reinterpret_cast<float4*>(lo + r * d)[k] = make_float4(l[0], l[1], l[2], l[3]);
    }
}

__global__ void mul_norms_kernel(const float* a, const float* b, float* o, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) o[i] = a[i] * b[i];
}
__global__ void fill_kernel(float* p, int64_t n, float v) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
    static EncodeFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeFn>(p);
    }
    return fn;
}

// 2-D fp32 [rows, cols] row-major (contiguous: pitch == cols), box = [32 cols, box_rows], 128-byte swizzle
bool make_map(CUtensorMap* map, const float* base, int64_t rows, int cols, int box_rows) {
    EncodeFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * 4};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tc

// Called by alq_min_dist (alq_mindist.cu).  Returns ALQ_OK, or ALQ_ERR_STATE if the tensor-core path
// cannot be used here (caller then runs the SIMT kernel); other codes are real failures.
int alq_min_dist_tc(alq_ctx* ctx, const float* x, int64_t ldx, const float* xn, int64_t n, const float* y,
                    int64_t ldy, const float* yn, int64_t m, int32_t d, const float* xa, int64_t ldxa,
                    const float* xan, const float* ya, int64_t ldya, const float* yan, int32_t c,
                    int32_t reduce_max, int32_t accumulate, float* out, cudaStream_t st) {
    using namespace tc;
    const bool factored = xa != nullptr;
    if (!get_encode()) return ALQ_ERR_STATE;
    if (n >= (1LL << 31) || m >= (1LL << 31)) return ALQ_ERR_STATE;
    const int cpad = factored ? c : 0;
    // scratch: split operands (contiguous rows) + fused norms + work list
    const size_t xe = static_cast<size_t>(n) * d, ye = static_cast<size_t>(m) * d;
    const size_t xae = static_cast<size_t>(n) * cpad, yae = static_cast<size_t>(m) * cpad;
    const int grid = ctx->sm_count;
    const int m_blocks = static_cast<int>((n + BM - 1) / BM), n_tiles = static_cast<int>((m + BN - 1) / BN);
    // Work list.  A CTA re-reads its row block (hi + lo = 2 MB at d = 2048) for every column tile, so the row
    // blocks that are live at the same time must fit the 50 MB L2 next to the streamed Y tiles: with one row block
    // per CTA (132 x 2 MB) they do not.  Instead `split` CTAs share a row block and divide its column tiles, so only
    // live_mb / 2 MB row blocks are live per round (each Y tile is then read from HBM once per round).
    const size_t blk_bytes = static_cast<size_t>(BM) * (d + cpad) * 8;
    size_t live_mb = 16;
    if (const char* e = getenv("ALQ_K3_LIVE_MB")) live_mb = static_cast<size_t>(std::max(1, atoi(e)));   // tuning aid
    int live = static_cast<int>(std::max<size_t>(1, (live_mb << 20) / std::max<size_t>(blk_bytes, 1)));
    live = std::max(1, std::min(live, grid));
    const int rounds = (m_blocks + live - 1) / live;
    const int items_per_cta = rounds + 1;
    int rc = alq_scratch_reserve(ctx, scratch_need({xe * 4, xe * 4, ye * 4, ye * 4, xae * 4, xae * 4, yae * 4, yae * 4,
                                                    static_cast<size_t>(n) * 4, static_cast<size_t>(m) * 4,
                                                    static_cast<size_t>(grid) * items_per_cta * sizeof(WorkItem),
                                                    static_cast<size_t>(grid) * 4}));
    if (rc) return rc;
    ScratchCursor cur(ctx->scratch);
    float* xh = cur.take<float>(xe); float* xl = cur.take<float>(xe);
    float* yh = cur.take<float>(ye); float* yl = cur.take<float>(ye);
    float* xah = cur.take<float>(xae); float* xal = cur.take<float>(xae);
    float* yah = cur.take<float>(yae); float* yal = cur.take<float>(yae);
    float* xnn = cur.take<float>(n); float* ynn = cur.take<float>(m);
    WorkItem* d_items = cur.take<WorkItem>(static_cast<size_t>(grid) * items_per_cta);
    int* d_counts = cur.take<int>(grid);

    // ---- work list (see above): round r covers row blocks [r*live, r*live + mbs); CTA c takes part c % split of
    //      the column tiles of row block c / split
    std::vector<WorkItem> items(static_cast<size_t>(grid) * items_per_cta);
    std::vector<int> counts(grid, 0);
    for (int r = 0; r < rounds; ++r) {
        const int mb0 = r * live, mbs = std::min(live, m_blocks - mb0);
        const int split = std::max(1, grid / mbs);
        for (int cta = 0; cta < grid; ++cta) {
            const int which = cta / split, part = cta % split;
            if (which >= mbs) continue;
            const int nb = static_cast<int>(static_cast<int64_t>(n_tiles) * part / split);
            const int ne = static_cast<int>(static_cast<int64_t>(n_tiles) * (part + 1) / split);
            if (ne > nb) items[static_cast<size_t>(cta) * items_per_cta + counts[cta]++] = WorkItem{mb0 + which, nb, ne, 0};
        }
    }
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_items, items.data(), items.size() * sizeof(WorkItem), cudaMemcpyHostToDevice, st));
    ALQ_CUDA(ctx, cudaMemcpyAsync(d_counts, counts.data(), counts.size() * sizeof(int), cudaMemcpyHostToDevice, st));

    // ---- split operands
    auto split = [&](const float* src, int64_t rows, int dd, int64_t ld, float* hi, float* lo) {
        if (rows == 0 || dd == 0) return;
        int blocks = static_cast<int>(std::min<int64_t>((rows * (dd / 4) + 255) / 256, static_cast<int64_t>(ctx->sm_count) * 16));
        split_tf32_kernel<<<blocks, 256, 0, st>>>(src, rows, dd, ld, hi, lo);
        ctx->launches++;
    };
    split(x, n, d, ldx, xh, xl);
    split(y, m, d, ldy, yh, yl);
    const float* xn_use = xn; const float* yn_use = yn;
    if (factored) {
        split(xa, n, c, ldxa, xah, xal);
        split(ya, m, c, ldya, yah, yal);
        mul_norms_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(xn, xan, xnn, n);
        mul_norms_kernel<<<static_cast<int>((m + 255) / 256), 256, 0, st>>>(yn, yan, ynn, m);
        ctx->launches += 2;
        xn_use = xnn; yn_use = ynn;
    }
    if (!accumulate) {
        fill_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, st>>>(out, n, reduce_max ? -INFINITY : INFINITY);
        ctx->launches++;
    }
    CUtensorMap mxh, mxl, myh, myl, mxah, mxal, myah, myal;
    bool ok = make_map(&mxh, xh, n, d, BM) && make_map(&mxl, xl, n, d, BM) && make_map(&myh, yh, m, d, BN) &&
              make_map(&myl, yl, m, d, BN);
    if (factored)
        ok = ok && make_map(&mxah, xah, n, c, BM) && make_map(&mxal, xal, n, c, BM) && make_map(&myah, yah, m, c, BN) &&
             make_map(&myal, yal, m, c, BN);
    else { mxah = mxh; mxal = mxl; myah = myh; myal = myl; }
    if (!ok) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_min_dist: cuTensorMapEncodeTiled failed");

    Params P{};
    P.xn = xn_use; P.yn = yn_use; P.out = out; P.items = d_items; P.item_count = d_counts; P.items_per_cta = items_per_cta;
    P.n = static_cast<int>(n); P.m = static_cast<int>(m);
    P.kblocks_h = (d + BK - 1) / BK; P.kblocks_a = factored ? (c + BK - 1) / BK : 0;
    const size_t smem = static_cast<size_t>(STAGES) * STAGE_BYTES + 256 + 1024;
    auto launch = [&](auto kern) -> cudaError_t {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        if (e != cudaSuccess) return e;
        kern<<<grid, THREADS, smem, st>>>(mxh, mxl, myh, myl, mxah, mxal, myah, myal, P);
        return cudaGetLastError();
    };
    cudaError_t e;
    if (factored) e = reduce_max ? launch(min_dist_tc_kernel<true, true>) : launch(min_dist_tc_kernel<true, false>);
    else e = reduce_max ? launch(min_dist_tc_kernel<false, true>) : launch(min_dist_tc_kernel<false, false>);
    ctx->launches++;
    if (e != cudaSuccess) ALQ_FAIL(ctx, ALQ_ERR_CUDA, "min_dist_tc_kernel launch failed: %s", cudaGetErrorString(e));
    return ALQ_OK;
}

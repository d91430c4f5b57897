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
// Structure: the ring of alq_wgmma.cuh (one CTA per SM, a TMA producer warpgroup, two consumer warpgroups issuing
// tc::ring_mma), persistent over a host-built work list of (row block, column-tile range).  The producer loads
// 4 tensor maps (X_hi, X_lo, Y_hi, Y_lo); the consumers compute the distance + running row min on their register
// accumulators and issue one float atomic per row at the end of a work item.  The factored/BADGE form keeps two
// accumulators (<h,h'> and <a,a'>) in the same ring, k-blocks of h first, and multiplies them in the epilogue.
// Every CTA sweeps the column tiles in the same order, so a Y tile is fetched from HBM once and
// served to the other CTAs from L2.
#include <stdlib.h>

#include "alq_wgmma.cuh"

namespace tc {

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

template <bool FACTORED, bool RED_MAX>
__global__ void __launch_bounds__(THREADS, 1)
min_dist_tc_kernel(const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
                   const __grid_constant__ CUtensorMap map_yh, const __grid_constant__ CUtensorMap map_yl,
                   const __grid_constant__ CUtensorMap map_xah, const __grid_constant__ CUtensorMap map_xal,
                   const __grid_constant__ CUtensorMap map_yah, const __grid_constant__ CUtensorMap map_yal,
                   Params P) {
    extern __shared__ unsigned char smem_dyn[];
    const Role me = ring_role();
    const int n_items = P.item_count[blockIdx.x];
    const WorkItem* items = P.items + static_cast<size_t>(blockIdx.x) * P.items_per_cta;
    const int kb_total = P.kblocks_h + (FACTORED ? P.kblocks_a : 0);
    const Ring ring = ring_init(smem_dyn);

    if (me.wg == 0) {
        producer_regs();
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            for (int w = 0; w < n_items; ++w) {
                const WorkItem wi = items[w];
                for (int nt = wi.n_begin; nt < wi.n_end; ++nt) {
                    for (int kb = 0; kb < kb_total; ++kb, ++it) {
                        const bool apart = FACTORED && kb >= P.kblocks_h;
                        ring_load(ring, it, apart ? &map_xah : &map_xh, apart ? &map_xal : &map_xl, wi.m_blk * BM,
                                  apart ? &map_yah : &map_yh, apart ? &map_yal : &map_yl, nt * BN,
                                  (apart ? kb - P.kblocks_h : kb) * BK);
                    }
                }
            }
        }
    } else {
        consumer_regs();
        uint32_t it = 0;
        for (int w = 0; w < n_items; ++w) {
            const WorkItem wi = items[w];
            const int row0 = wi.m_blk * BM + me.r_in_tile, row1 = row0 + 8;
            const float rn0 = row0 < P.n ? P.xn[row0] : 0.f, rn1 = row1 < P.n ? P.xn[row1] : 0.f;
            float best0 = RED_MAX ? ALQ_NEG_INF : ALQ_POS_INF, best1 = best0;
            for (int nt = wi.n_begin; nt < wi.n_end; ++nt) {
                float acc[64];
                float acc_a[FACTORED ? 64 : 1];
                int prev = -1;
                // one pipeline for both contractions: a k-block of the a-part goes into acc_a, and the stage hand-back
                // runs across the boundary
                for (int kb = 0; kb < kb_total; ++kb, ++it) {
                    if constexpr (FACTORED) {
                        if (kb >= P.kblocks_h) {
                            ring_mma(ring, it, me.a_off, acc_a, kb == P.kblocks_h, prev, me.t);
                            continue;
                        }
                    }
                    ring_mma(ring, it, me.a_off, acc, kb == 0, prev, me.t);
                }
                ring_drain(ring, prev, me.t);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = nt * BN + 8 * j + me.c_in_tile;
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
            if ((me.lane & 3) == 0 && wi.n_end > wi.n_begin) {
                if (row0 < P.n) { if (RED_MAX) atomic_max_float(P.out + row0, best0); else atomic_min_float(P.out + row0, best0); }
                if (row1 < P.n) { if (RED_MAX) atomic_max_float(P.out + row1, best1); else atomic_min_float(P.out + row1, best1); }
            }
        }
    }
}

// every row of x as its TF32 hi/lo pair (split_tf32)
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
        for (int j = 0; j < 4; ++j) split_tf32(e[j], h[j], l[j]);
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
    const size_t smem = ring_smem_bytes(0);
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

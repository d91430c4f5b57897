// The Hopper 3xTF32 tile pipeline of the wgmma kernels (K3 in alq_mindist_tc.cu, K9 in alq_vaal.cu, K13 in
// alq_probcover.cu, K15 in alq_typiclust.cu, K18 in alq_cal.cu): TMA tile loads, SWIZZLE_128B shared-memory
// descriptors, the m64n128k8 TF32 MMA, the host-side tensor-map encoder, the ring that connects them, and the
// coefficient of the chain's error bound.  Operands are fp32 rows already split into TF32 hi/lo pairs; a stage row is
// BK = 32 fp32 = 128 bytes, one swizzle span.
//
// The ring (one CTA per SM, 3 warpgroups):
//   warpgroup 0    TMA producer (one thread): per k-block, the hi and lo boxes of a 128-row block of X and of a
//                  128-row block of Y into one of 3 shared-memory stages (ring_load), mbarrier complete_tx on `full`.
//   warpgroups 1-2 consumers: each owns 64 of the tile's 128 rows and issues hi*hi' + hi*lo' + lo*hi' per 8-wide
//                  k-step, k ascending, into one m64n128 fp32 register fragment (ring_mma), keeping one stage in
//                  flight and handing the previous one back on `empty`.
// The producer and the consumers walk the same sequence of k-blocks, counted by `it`.  K9, K15 and K18 run the
// row-block schedule: ring_produce_rows on the producer, ring_tile per tile on the consumers.  K13 keeps its own
// producer loop over the upper-triangle tiles and consumes each tile with ring_tile.  K3 keeps both loops (its factored
// form switches accumulators inside a tile) around ring_load, ring_mma and ring_drain.  Each kernel keeps its own
// epilogue.  All five issue this one chain, so the 3xTF32 error bound of DESIGN section 4 (band_coef), measured
// through K3, holds for all of them.
#pragma once
#include <cuda.h>

#include "alq_common.cuh"

namespace tc {

constexpr int BK = 32;           // fp32 per stage row = 128 bytes = one swizzle span
constexpr int UK = 8;            // wgmma K for tf32
constexpr int BM = 128;          // rows per tile (two m64 consumer warpgroups)
constexpr int BN = 128;          // columns per tile (wgmma N)
constexpr int STAGES = 3;
constexpr int OP_BYTES = BM * BK * 4;             // 16 KB: one operand's k-block (BM == BN)
constexpr int STAGE_BYTES = 4 * OP_BYTES;         // hi + lo of the row block and of the column block = 64 KB
constexpr int THREADS = 384;
static_assert(BM == BN, "the four operand boxes of a stage share OP_BYTES");

// dynamic shared memory of a ring kernel: the stages, the 1 KB SWIZZLE_128B alignment slack, the full / empty
// barriers, and `extra` bytes the kernel places after them (Ring::tail)
__host__ __device__ constexpr size_t ring_smem_bytes(size_t extra) {
    return static_cast<size_t>(STAGES) * STAGE_BYTES + 1024 + 2 * STAGES * sizeof(uint64_t) + extra;
}

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

// hi = rna_tf32(v), lo = rna_tf32(v - hi): two valid TF32 operands whose sum is v to 2^-22 relative
__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
    uint32_t hb, lb;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
    hi = __uint_as_float(hb);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - hi));
    lo = __uint_as_float(lb);
}

// ---- the ring ----------------------------------------------------------------------------------------------------------
struct Ring {
    unsigned char* stage;        // STAGES x STAGE_BYTES, 1 KB aligned: [X hi | X lo | Y hi | Y lo] per stage
    uint64_t* full;              // [STAGES] the producer's TMA bytes have landed
    uint64_t* empty;             // [STAGES] both consumer warpgroups have retired the stage's MMAs
    unsigned char* tail;         // the first byte after the barriers (ring_smem_bytes' `extra`)
};

// every thread of the CTA, before the role split
__device__ __forceinline__ Ring ring_init(unsigned char* smem_dyn) {
    Ring r;
    // SWIZZLE_128B tiles must sit on 1024-byte boundaries: align by hand (ring_smem_bytes allocates 1 KB of slack)
    r.stage = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    r.full = reinterpret_cast<uint64_t*>(r.stage + STAGES * STAGE_BYTES);
    r.empty = r.full + STAGES;
    r.tail = reinterpret_cast<unsigned char*>(r.empty + STAGES);
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&r.full[s], 1); mbar_init(&r.empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    return r;
}

// A thread's role.  Warpgroup 0 produces, warpgroups 1-2 consume; warpgroup wg - 1 owns rows [64 (wg - 1), 64 wg) of the
// tile.  m64nN fp32 fragment: d[4j + {0,1}] = (r, 8j + 2 (lane % 4) + {0,1}), d[4j + {2,3}] = (r + 8, same cols),
// r = 16 warp + lane / 4 inside the warpgroup's 64 rows.
struct Role {
    int wg, t, lane;
    uint32_t a_off;              // the warpgroup's 64 rows inside an X box: 8 KB, a whole number of swizzle atoms
    int r_in_tile, c_in_tile;    // the fragment's first row and first column inside the 128 x 128 tile
};
__device__ __forceinline__ Role ring_role() {
    Role r;
    r.wg = threadIdx.x >> 7;
    r.t = threadIdx.x & 127;
    r.lane = threadIdx.x & 31;
    r.a_off = static_cast<uint32_t>(r.wg - 1) * 64 * BK * 4;
    r.r_in_tile = (r.wg - 1) * 64 + (r.t >> 5) * 16 + (r.lane >> 2);
    r.c_in_tile = 2 * (r.lane & 3);
    return r;
}
// the producer warpgroup gives its registers to the consumers: 40 + 2 x 232 = 3 x 168, the launch's budget per thread
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

// Producer, k-block `it` of the CTA's sequence: columns [k0, k0 + 32) of rows [a_row, a_row + 128) of X (a_hi, a_lo) and
// of rows [b_row, b_row + 128) of Y (b_hi, b_lo) into stage it % STAGES, once the consumers have handed it back.
__device__ __forceinline__ void ring_load(const Ring& r, uint32_t it, const CUtensorMap* a_hi, const CUtensorMap* a_lo,
                                          int a_row, const CUtensorMap* b_hi, const CUtensorMap* b_lo, int b_row, int k0) {
    const int s = it % STAGES;
    const uint32_t round = it / STAGES;
    if (round > 0) mbar_wait(&r.empty[s], (round - 1) & 1u);
    unsigned char* st = r.stage + static_cast<size_t>(s) * STAGE_BYTES;
    mbar_expect_tx(&r.full[s], STAGE_BYTES);
    tma_load_2d(st, a_hi, k0, a_row, &r.full[s]);
    tma_load_2d(st + OP_BYTES, a_lo, k0, a_row, &r.full[s]);
    tma_load_2d(st + 2 * OP_BYTES, b_hi, k0, b_row, &r.full[s]);
    tma_load_2d(st + 3 * OP_BYTES, b_lo, k0, b_row, &r.full[s]);
}

// Consumer, k-block `it`: acc (+)= X Y^T over the stage's 32 columns as 4 k-steps of hi*hi' + hi*lo' + lo*hi'; `first`
// overwrites acc on the first MMA.  The MMAs stay in flight; the previous stage (`prev`, -1 for none) is handed back
// once its own have retired, and `prev` becomes this stage.  After a tile's last k-block, ring_drain.
__device__ __forceinline__ void ring_mma(const Ring& r, uint32_t it, uint32_t a_off, float (&acc)[64], bool first,
                                         int& prev, int t) {
    const int s = it % STAGES;
    mbar_wait(&r.full[s], (it / STAGES) & 1u);
    const uint32_t a_hi = smem_u32(r.stage + static_cast<size_t>(s) * STAGE_BYTES) + a_off;
    const uint32_t a_lo = a_hi + OP_BYTES, b_hi = a_hi - a_off + 2 * OP_BYTES, b_lo = b_hi + OP_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / UK; ++k) {
        const uint32_t off = k * UK * 4;    // bytes along K inside the 128-byte swizzle span
        const uint64_t dah = make_desc(a_hi + off), dal = make_desc(a_lo + off);
        const uint64_t dbh = make_desc(b_hi + off), dbl = make_desc(b_lo + off);
        wgmma_tf32(acc, dah, dbh, (first && k == 0) ? 0u : 1u);
        wgmma_tf32(acc, dah, dbl, 1u);
        wgmma_tf32(acc, dal, dbh, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && t == 0) mbar_arrive(&r.empty[prev]);
    prev = s;
}
// every MMA of the tile has retired: the accumulators are readable and the last stage goes back
__device__ __forceinline__ void ring_drain(const Ring& r, int prev, int t) {
    wgmma_wait<0>();
    if (prev >= 0 && t == 0) mbar_arrive(&r.empty[prev]);
}

// Consumer, one 128 x 128 tile: its `kblocks` k-blocks from `it` on through ring_mma (acc overwritten), then ring_drain.
__device__ __forceinline__ void ring_tile(const Ring& r, uint32_t& it, const Role& me, float (&acc)[64], int kblocks) {
    int prev = -1;
    for (int kb = 0; kb < kblocks; ++kb, ++it) ring_mma(r, it, me.a_off, acc, kb == 0, prev, me.t);
    ring_drain(r, prev, me.t);
}

// Producer thread of the row-block schedule: the CTA's 128-row blocks of X rb = blockIdx.x, blockIdx.x + gridDim.x, ...
// below `rblocks`, for each every 128-row tile of Y ct = 0 .. ctiles - 1, for each its k-blocks.  The consumers walk
// the same sequence: per row block, one ring_tile per ct in ascending order.
__device__ __forceinline__ void ring_produce_rows(const Ring& r, const CUtensorMap* x_hi, const CUtensorMap* x_lo,
                                                  const CUtensorMap* y_hi, const CUtensorMap* y_lo, int rblocks,
                                                  int ctiles, int kblocks) {
    uint32_t it = 0;
    for (int rb = blockIdx.x; rb < rblocks; rb += gridDim.x)
        for (int ct = 0; ct < ctiles; ++ct)
            for (int kb = 0; kb < kblocks; ++kb, ++it) ring_load(r, it, x_hi, x_lo, rb * BM, y_hi, y_lo, ct * BN, kb * BK);
}

// DESIGN section 4: ring_mma's chain over d columns gives |g - <x, y>| <= (1 + 3 ceil(d / 8)) 2^-20 |x||y|.  A d2
// formed as nrm2_x + nrm2_y - 2g carries twice that; the 1e-6 covers |x||y| formed in fp64 from the norms.  The band of
// K13, K15 and K18 is band_coef(d) |x||y| plus each kernel's own slack for its fp64 terms.
inline double band_coef(int d) { return 2.0 * (1.0 + 3.0 * ((d + 7) / 8)) * ldexp(1.0, -20) * (1.0 + 1e-6); }

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeFn get_encode() {
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

// 2-D fp32 [rows, cols] row-major (contiguous: pitch == cols), box = [32 cols, box_rows], 128-byte swizzle.
// Boxes reaching past the last row or column are zero-filled.
inline bool make_map(CUtensorMap* map, const float* base, int64_t rows, int cols, int box_rows) {
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

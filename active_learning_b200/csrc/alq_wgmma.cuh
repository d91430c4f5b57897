// Hopper tensor-core building blocks shared by the wgmma kernels (K3 in alq_mindist_tc.cu, K9 in alq_vaal.cu):
// TMA tile loads, SWIZZLE_128B shared-memory descriptors, the m64n128k8 TF32 MMA and the host-side tensor-map
// encoder.  Operands are fp32 rows already split into TF32 hi/lo pairs; a stage row is BK = 32 fp32 = 128 bytes,
// one swizzle span.
#pragma once
#include <cuda.h>

#include "alq_common.cuh"

namespace tc {

constexpr int BK = 32;           // fp32 per stage row = 128 bytes = one swizzle span
constexpr int UK = 8;            // wgmma K for tf32

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

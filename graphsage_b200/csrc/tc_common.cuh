// wgmma / shared-memory-descriptor helpers shared by the Hopper tensor-core kernels (gemm_tc.cu, maxpool_tc.cu).
//
// Operand tiles in shared memory are K-major with the 128-byte swizzle: 128 rows of 128 bytes, 16-byte chunk c of row r
// at r * 128 + ((c ^ (r & 7)) << 4), the image 1024-byte aligned.  A warpgroup's wgmma.m64n128 reads 64 rows of the A
// image and all 128 rows of the B image.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace gs {

constexpr int TC_BM = 128;       // output tile rows (two warpgroups of 64)
constexpr int TC_BN = 128;       // output tile columns (wgmma N)
constexpr int TC_TILE_BYTES = TC_BM * 128;   // one operand tile image: 128 rows x 128 B (one SW128 atom wide)

// K-major, 128-byte-swizzled shared-memory matrix descriptor (sm_90 wgmma):
//   [0,14) start address >> 4, [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1),
//   [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024 B), [62,64) layout = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define GS_WGMMA_D64                                                                                                       \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,"   \
  "%61,%62,%63}"
#define GS_WGMMA_OUT64(d)                                                                                                 \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),             \
      "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),             \
      "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]),             \
      "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]),             \
      "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),             \
      "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]),             \
      "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] (+)= A[64 x K] * B[128 x K]^T, both operands K-major in shared memory, fp32 accumulate in registers.
// kBf16: one K = 16 step of bf16 operands; else one K = 8 step of tf32 operands.  accumulate = 0 overwrites D.
// Thread t of the warpgroup holds d[4j + e] = D[16 (t / 32) + (t % 32) / 4 + 8 (e / 2)][8 j + 2 (t % 4) + (e % 2)].
// kTransA (bf16 only): A is MN-major instead - the 64 M values of one K index are one 128-byte row of the SW128 image
// (K-rows at 128 B, 8-row groups at the descriptor's 1024-byte stride), i.e. the same bytes as a K-major 64-column
// image read the other way round; the descriptor is unchanged (one 64-wide atom along M, so its leading offset is unused).
template <bool kBf16, int kTransA = 0>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(kBf16 || kTransA == 0, "transposed operands are bf16 only");
  if constexpr (kBf16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " GS_WGMMA_D64 ", %64, %65, p, 1, 1, %67, 0;\n\t}"
        : GS_WGMMA_OUT64(d)
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(kTransA)
        : "memory");
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " GS_WGMMA_D64 ", %64, %65, p, 1, 1;\n\t}"
        : GS_WGMMA_OUT64(d)
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
  }
}

// D[64 x 64] (+)= A[64 x K] * B[64 x K]^T, one K = 16 step of bf16 operands, both K-major in shared memory (B: 64 rows
// of an SW128 image).  Thread t holds d[4j + e] = D[16 (t / 32) + (t % 32) / 4 + 8 (e / 2)][8 j + 2 (t % 4) + (e % 2)].
__device__ __forceinline__ void wgmma_m64n64_bf16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ uint32_t tf32_mask(float x) { return __float_as_uint(x) & 0xFFFFE000u; }

// byte offset of 16-byte chunk c (0..7) of row r (0..127) inside a SW128 K-major tile image
__host__ __device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4));
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

}  // namespace gs

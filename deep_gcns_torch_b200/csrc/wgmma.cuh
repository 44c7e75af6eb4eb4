// Hopper warpgroup MMA (wgmma.mma_async, sm_90a): bf16 x bf16 or fp16 x fp16 -> fp32, both operands in shared memory, the
// accumulator in the registers of the 128 threads of one warpgroup.
#pragma once
#include <stdint.h>

namespace dgcn {

// Shared-memory matrix descriptor: [0,14) start >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte
// offset >> 4 | [62,64) layout, 1 = SWIZZLE_128B, 2 = SWIZZLE_64B.
//   MN-major operand: 64 elements (128 B) along MN per row, leading offset = stride between 64-wide MN blocks,
//                     stride offset = stride between groups of 8 K rows (1024 B inside a block).
//   K-major operand:  rows of 64 K elements (128 B), stride offset = stride between groups of 8 rows; the leading
//                     offset is not used by swizzled K-major layouts.
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t lead, uint32_t stride, uint32_t layout) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>((lead >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((stride >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(layout) << 62;
  return d;
}
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr, uint32_t lead, uint32_t stride) {
  return wg_desc(smem_addr, lead, stride, 1u);
}
// SWIZZLE_64B: the same with rows of 64 B - an MN-major block is 32 elements wide and a group of 8 K rows 512 B
// (the atom must sit on a 512-byte boundary).
__device__ __forceinline__ uint64_t wg_desc_sw64(uint32_t smem_addr, uint32_t lead, uint32_t stride) {
  return wg_desc(smem_addr, lead, stride, 2u);
}

// before the first wgmma of a batch: earlier register writes of the accumulators are ordered before it
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// every committed wgmma of this warpgroup has completed: accumulators readable, operand memory reusable
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Element type of the A and B operands; the accumulator is fp32 either way, so chains of both types may add into the
// same fragments.
enum WgElem : int { WG_BF16 = 0, WG_F16 = 1 };

// D[64 x 64] (+)= A[64 x 16] * B[16 x 64]; TA / TB = 1 for MN-major operands, 0 for K-major.  accumulate = 0
// overwrites D.
#define DGCN_WGMMA_M64N64(TYPES)                                                                                   \
  asm volatile(                                                                                                     \
      "{\n"                                                                                                         \
      ".reg .pred p;\n"                                                                                             \
      "setp.ne.b32 p, %34, 0;\n"                                                                                    \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPES " "                                                       \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                     \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "                           \
      "%32, %33, p, 1, 1, %35, %36;\n"                                                                              \
      "}\n"                                                                                                         \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),     \
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),    \
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])                  \
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)                                                        \
      : "memory")
template <int TA, int TB, int ELEM = WG_BF16>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  static_assert(ELEM == WG_BF16 || ELEM == WG_F16, "operand type");
  if constexpr (ELEM == WG_F16) DGCN_WGMMA_M64N64("f16.f16");
  else DGCN_WGMMA_M64N64("bf16.bf16");
}
#undef DGCN_WGMMA_M64N64
// D[64 x 32] (+)= A[64 x 16] * B[16 x 32]
#define DGCN_WGMMA_M64N32(TYPES)                                                                                   \
  asm volatile(                                                                                                     \
      "{\n"                                                                                                         \
      ".reg .pred p;\n"                                                                                             \
      "setp.ne.b32 p, %18, 0;\n"                                                                                    \
      "wgmma.mma_async.sync.aligned.m64n32k16.f32." TYPES " "                                                       \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "                                     \
      "%16, %17, p, 1, 1, %19, %20;\n"                                                                              \
      "}\n"                                                                                                         \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])                   \
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)                                                        \
      : "memory")
template <int TA, int TB, int ELEM = WG_BF16>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  static_assert(ELEM == WG_BF16 || ELEM == WG_F16, "operand type");
  if constexpr (ELEM == WG_F16) DGCN_WGMMA_M64N32("f16.f16");
  else DGCN_WGMMA_M64N32("bf16.bf16");
}
#undef DGCN_WGMMA_M64N32

// Accumulator fragment of an m64nN wgmma: register i of thread (warp w of the warpgroup, lane l) holds
// row 16 w + l / 4 + 8 ((i / 2) & 1), column 8 (i / 4) + 2 (l & 3) + (i & 1).
__device__ __forceinline__ int wg_frag_row(int i) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int wg_frag_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }

// The 64 x 64 fragment -> rows row0 .. row0 + 63 of a row-major fp32 tile with leading dimension ld (floats).
__device__ __forceinline__ void wg_store_m64n64(const float (&d)[32], float* tile, int ld, int row0) {
#pragma unroll
  for (int i = 0; i < 32; i += 2)
    *reinterpret_cast<float2*>(tile + (row0 + wg_frag_row(i)) * ld + wg_frag_col(i)) = make_float2(d[i], d[i + 1]);
}
// The 64 x 32 fragment -> rows row0 .. row0 + 63, columns 0 .. 31.
__device__ __forceinline__ void wg_store_m64n32(const float (&d)[16], float* tile, int ld, int row0) {
#pragma unroll
  for (int i = 0; i < 16; i += 2)
    *reinterpret_cast<float2*>(tile + (row0 + wg_frag_row(i)) * ld + wg_frag_col(i)) = make_float2(d[i], d[i + 1]);
}

}  // namespace dgcn

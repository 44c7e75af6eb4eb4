// Hopper warpgroup MMA (wgmma.mma_async, sm_90a): bf16 x bf16 -> fp32, both operands in shared memory, the
// accumulator in the registers of the 128 threads of one warpgroup.
#pragma once
#include <stdint.h>

namespace dgcn {

// Shared-memory matrix descriptor: [0,14) start >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte
// offset >> 4 | [62,64) layout, 1 = SWIZZLE_128B.
//   MN-major operand: 64 elements (128 B) along MN per row, leading offset = stride between 64-wide MN blocks,
//                     stride offset = stride between groups of 8 K rows (1024 B inside a block).
//   K-major operand:  rows of 64 K elements (128 B), stride offset = stride between groups of 8 rows; the leading
//                     offset is not used by swizzled K-major layouts.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr, uint32_t lead, uint32_t stride) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>((lead >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((stride >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// before the first wgmma of a batch: earlier register writes of the accumulators are ordered before it
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// every committed wgmma of this warpgroup has completed: accumulators readable, operand memory reusable
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 64] (+)= A[64 x 16] * B[16 x 64]; TA / TB = 1 for MN-major operands, 0 for K-major.  accumulate = 0
// overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}
// D[64 x 32] (+)= A[64 x 16] * B[16 x 32]
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, %19, %20;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

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

}  // namespace dgcn

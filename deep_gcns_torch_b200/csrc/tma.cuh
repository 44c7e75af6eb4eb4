// Hopper TMA (cp.async.bulk.tensor) and mbarrier helpers (sm_90a) for the kernels that feed the tensor cores through
// them, and the host-side encoder of their tensor maps.
#pragma once
#include <cuda.h>          // CUtensorMap (type only: the encoder comes from cudaGetDriverEntryPoint)
#include <stdint.h>

namespace dgcn {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// after the mbar_init calls, before any other thread or the TMA unit uses the barriers
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // bounded spin: a tensor-core pipeline that never signals must trap, not hang the GPU
  for (uint32_t spin = 0;; ++spin) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    if (spin > (1u << 26)) __trap();
  }
}
// the same wait with a suspend-time hint (ns): a warp that expects to wait long sleeps in the barrier unit instead of
// spending issue slots on the retry loop
__device__ __forceinline__ void mbar_wait_hint(uint64_t* bar, uint32_t parity, uint32_t hint_ns) {
  for (uint32_t spin = 0;; ++spin) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns)
        : "memory");
    if (done) return;
    if (spin > (1u << 24)) __trap();
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {   // non-blocking
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}
// a tensor map passed as a kernel parameter: fetch it into the descriptor cache before the first load
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// TMA: one 2-D box of the tensor behind `map` (coordinates innermost first) -> shared memory, completion
// counted in bytes on `bar`
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (TMA, wgmma)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Host: 16-bit matrix (rows, cols) row-major, elements of type `dtype` (bf16 or fp16) -> tensor map with boxes of
// box_cols columns x box_rows rows.  box_cols = 64 (128 bytes), SWIZZLE_128B: a box lands in shared memory as box_rows
// x 128 B rows with the 16-byte chunks XOR-swizzled by (row & 7), which is the canonical wgmma layout of one 64-wide
// block; box_cols = 32 (64 bytes), SWIZZLE_64B: box_rows x 64 B rows, chunks XOR-swizzled by ((row >> 1) & 3), the
// canonical layout of one 32-wide block.  DGCN_ERR_UNSUPPORTED when the driver has no tiled tensor-map encoder,
// DGCN_ERR_CUDA when it rejects the map.
int make_tensor_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int box_cols, int box_rows,
                    CUtensorMapDataType dtype);

}  // namespace dgcn

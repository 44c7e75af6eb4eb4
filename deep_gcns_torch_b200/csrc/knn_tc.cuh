// Tensor-core (wgmma) path of the dilated kNN selection for K <= 48, C <= 64, N % 128 == 0:  the N x N x C
// contraction runs on the Hopper tensor cores as a CERTIFIED PRE-FILTER, the ranking itself stays exact fp32
// (DESIGN.md 6).
//
//   tc_prologue(_pq)  one pass over x: x = hi + mid (two bf16 planes, channel-major like x, channels
//                     zero-padded to a multiple of 16; the three products hi*hi, hi*mid, mid*hi
//                     reproduce x_i.x_j to ~2^-16 relative), |x|^2, the operand block that folds
//                     -|x_j|^2/2 into the product, the node-major fp32 copy, max |x|^2 (and the
//                     EdgeConv node GEMM).
//   knn_tc_kernel     one 128-thread CTA (one warpgroup) = 128 queries of a cloud.  Query planes stay
//                     resident in shared memory; candidate tiles of 128 points are brought in by TMA
//                     (cp.async.bulk.tensor, 64-point x Cpad-channel boxes with SWIZZLE_128B = the
//                     canonical MN-major wgmma layout: x is channel-major = MN-major, so no
//                     transposition anywhere, and no thread spends instructions on the copy).  Per
//                     64-candidate block the warpgroup runs two m64n64k16 wgmma chains (query rows 0..63 and
//                     64..127) and puts the accumulators into a shared-memory stage, row = query; the TMA
//                     of tile t+1 is started as soon as the last wgmma of tile t has completed and lands
//                     under the filter.  Thread r = query r filters its row in 16-column chunks against the
//                     thread's private threshold; survivors go to a private candidate buffer
//                     and from there into the query's register-resident sorted list of the KP best
//                     APPROXIMATE keys (no atomics in the filter).
//                     Afterwards each thread re-evaluates its KP candidates with the exact fp32
//                     FMA chain (same values as knn_small_kernel), sorts them, and certifies:
//                       exact_K-th + eps < approx_KP-th     (eps = bound on |approx - exact|)
//                     i.e. nothing outside the list can belong to the true K best.  Certified
//                     queries run the fused consumer; the others are appended to a fail list.
//   knn_exact_rows_kernel  completes the (rare) uncertified queries with the exact fp32 brute
//                     force, one CTA per query.
#pragma once
#include <cuda.h>          // CUtensorMap (type only: the encoder comes from cudaGetDriverEntryPoint)
#include <cuda_bf16.h>
#include "knn.cuh"
#include "wgmma.cuh"

namespace dgcn {

constexpr int TC_MAX_C = 64;
constexpr int TC_K_MAX = 48;

// ---- PTX wrappers -------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// Arrive (release) and report whether this arrival - or one that raced with it - completed the phase.
__device__ __forceinline__ bool mbar_arrive_completes(uint64_t* bar) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .b64 st;\n"
      ".reg .pred P1;\n"
      "mbarrier.arrive.shared::cta.b64 st, [%1];\n"
      "mbarrier.test_wait.shared::cta.b64 P1, [%1], st;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}"
      : "=r"(done)
      : "r"(smem_u32(bar))
      : "memory");
  return done != 0;
}
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
// TMA: one 2-D box of the tensor behind `map` (coordinates innermost first) -> shared memory, completion
// counted in bytes on `bar`
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void cp_async16_addr(uint32_t smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// ---- operand split ----------------------------------------------------------------------------
// planes (B, TC_PLANES, Cpad, N) bf16: x = hi + mid with |mid| <= 2^-8 |x| and |x - hi - mid| <= 2^-17 |x|;
// channels >= C are zero.  Three bf16 products hi*hi, hi*mid, mid*hi reproduce x_i.x_j to
// 2^-15 relative to |x_i||x_j| in the worst case (two split residuals 2^-16 + the dropped mid*mid
// term 2^-16) - a pre-filter accuracy, the ranking itself is redone in exact fp32.
constexpr int TC_PLANES = 2;

// One pass over x for everything the tensor-core path needs: sq (B,N) (same FMA chain as sqnorm_kernel),
// the bf16 planes, the extra operand block sqp that folds -|x_j|^2/2 into the tensor-core product, the
// node-major copy xt (optional) and the per-cloud max of sq (atomicMax on the bits of a non-negative
// float; sqmax must be zero-initialised).  Block = 32 points x all channels (C <= 64).
#ifndef DGCN_TEMPLATES_ONLY
__global__ void __launch_bounds__(256) tc_prologue_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C,
                                                         int Cpad, int N, float* __restrict__ sq,
                                                         __nv_bfloat16* __restrict__ planes, float* __restrict__ xt,
                                                         float* __restrict__ sqmax, __nv_bfloat16* __restrict__ sqp) {
  __shared__ float tile[TC_MAX_C][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int b = blockIdx.y, n0 = blockIdx.x * 32, n = n0 + tx;
  const int64_t plane = static_cast<int64_t>(Cpad) * N;
  __nv_bfloat16* pb = planes + static_cast<int64_t>(b) * TC_PLANES * plane;
  for (int c = ty; c < Cpad; c += 8) {
    float v = 0.f;
    if (c < C && n < N) v = __ldg(x + b * sb + c * sc + n);
    if (c < C) tile[c][tx] = v;
    if (n < N) {
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      pb[static_cast<int64_t>(c) * N + n] = hi;
      pb[plane + static_cast<int64_t>(c) * N + n] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
  __syncthreads();
  if (ty == 0) {
    float s = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(tile[c][tx], tile[c][tx], s);
    if (n < N) {
      sq[static_cast<int64_t>(b) * N + n] = s;
      // rows 0..2 of the (B, 8, N) extra operand block: -|x|^2 / 2 as three bf16 terms (2^-24 relative)
      __nv_bfloat16* sp = sqp + static_cast<int64_t>(b) * 8 * N + n;
      float rem = -0.5f * s;
#pragma unroll
      for (int t3 = 0; t3 < 3; ++t3) {
        const __nv_bfloat16 h = __float2bfloat16_rn(rem);
        sp[static_cast<int64_t>(t3) * N] = h;
        rem -= __bfloat162float(h);
      }
#pragma unroll
      for (int t3 = 3; t3 < 8; ++t3) sp[static_cast<int64_t>(t3) * N] = __float2bfloat16_rn(0.f);
    }
    float m = n < N ? s : 0.f;
    m = warp_max(m);
    if (tx == 0) atomicMax(reinterpret_cast<unsigned int*>(sqmax + b), __float_as_uint(m));
  }
  if (xt) {
    for (int i = threadIdx.x; i < 32 * C; i += 256) {
      const int rr = i / C, c = i % C;
      if (n0 + rr < N) xt[(static_cast<int64_t>(b) * N + n0 + rr) * C + c] = tile[c][rr];
    }
  }
}
#endif  // DGCN_TEMPLATES_ONLY

// tc_prologue_kernel fused with the EdgeConv node GEMM PQ[b][n][m] = sum_c x[b][c][n] wk[c][m] + bk[m]
// (node_pq_kernel's result bit for bit: fp32 FMA chain over c ascending from 0, bias added last), so x is
// read once for everything the layer needs.  Block = 64 points x all channels (C <= 64); M % 128 == 0,
// N % 64 == 0.  Dynamic shared memory: xs[C][68] + ws[C][M] floats.
struct ProloguePq {
  const float* wk;   // [C][M] packed weights (pack_edge_weights_kernel)
  const float* bk;   // [M]
  float* pq;         // (B, N, M)
  int M;
};
#ifndef DGCN_TEMPLATES_ONLY
__global__ void __launch_bounds__(256, 4) tc_prologue_pq_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C,
                                                            int Cpad, int N, float* __restrict__ sq,
                                                            __nv_bfloat16* __restrict__ planes, float* __restrict__ xt,
                                                            float* __restrict__ sqmax, __nv_bfloat16* __restrict__ sqp,
                                                            const ProloguePq g) {
  extern __shared__ __align__(16) float pq_smem[];
  constexpr int XLD = 68;
  float* xs = pq_smem;                       // [C][XLD]
  float* ws = pq_smem + TC_MAX_C * XLD;      // [C][M]
  const int tid = threadIdx.x;
  const int b = blockIdx.y, n0 = blockIdx.x * 64;
  const int M = g.M;
  const int64_t plane = static_cast<int64_t>(Cpad) * N;
  __nv_bfloat16* pb = planes + static_cast<int64_t>(b) * TC_PLANES * plane;
  if (((reinterpret_cast<uintptr_t>(x) & 7) | (sb & 1) | (sc & 1)) == 0) {
    // two adjacent points per thread: 8-byte loads, one bf16x2 store per plane (each half rounded like the scalar path)
    const int lane = tid & 31, wrp = tid >> 5, n = n0 + 2 * lane;
    for (int c = wrp; c < Cpad; c += 8) {
      const float2 v = c < C ? __ldg(reinterpret_cast<const float2*>(x + b * sb + c * sc + n)) : make_float2(0.f, 0.f);
      if (c < C) *reinterpret_cast<float2*>(xs + c * XLD + 2 * lane) = v;
      const __nv_bfloat162 hi = __floats2bfloat162_rn(v.x, v.y);
      const __nv_bfloat162 mid = __floats2bfloat162_rn(v.x - __low2float(hi), v.y - __high2float(hi));
      *reinterpret_cast<__nv_bfloat162*>(pb + static_cast<int64_t>(c) * N + n) = hi;
      *reinterpret_cast<__nv_bfloat162*>(pb + plane + static_cast<int64_t>(c) * N + n) = mid;
    }
  } else {
    const int tx = tid & 63, ty = tid >> 6, n = n0 + tx;
    for (int c = ty; c < Cpad; c += 4) {
      const float v = c < C ? __ldg(x + b * sb + c * sc + n) : 0.f;
      if (c < C) xs[c * XLD + tx] = v;
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      pb[static_cast<int64_t>(c) * N + n] = hi;
      pb[plane + static_cast<int64_t>(c) * N + n] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
  for (int i = tid * 4; i < C * M; i += 256 * 4)
    *reinterpret_cast<float4*>(ws + i) = __ldg(reinterpret_cast<const float4*>(g.wk + i));
  __syncthreads();
  if (tid < 64) {
    const int n = n0 + tid;
    float s = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(xs[c * XLD + tid], xs[c * XLD + tid], s);
    sq[static_cast<int64_t>(b) * N + n] = s;
    __nv_bfloat16* sp = sqp + static_cast<int64_t>(b) * 8 * N + n;
    float rem = -0.5f * s;
#pragma unroll
    for (int t3 = 0; t3 < 3; ++t3) {
      const __nv_bfloat16 h = __float2bfloat16_rn(rem);
      sp[static_cast<int64_t>(t3) * N] = h;
      rem -= __bfloat162float(h);
    }
#pragma unroll
    for (int t3 = 3; t3 < 8; ++t3) sp[static_cast<int64_t>(t3) * N] = __float2bfloat16_rn(0.f);
    const float m = warp_max(s);
    if ((tid & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(sqmax + b), __float_as_uint(m));
  }
  if (xt && (C & 7) == 0 && (reinterpret_cast<uintptr_t>(xt) & 15) == 0) {
    // node-major copy: a warp step covers 16 points x 8 channels - lane pairs write one full 32-byte sector of a row,
    // and the transposed shared-memory reads ((c0 + 4 (lane & 1) + j) * 68 + lane / 2) hit 32 distinct banks
    const int lane = tid & 31, wrp = tid >> 5;
    for (int it = wrp; it < 4 * (C >> 3); it += 8) {
      const int rr = (lane >> 1) + 16 * (it & 3), c = (it >> 2) * 8 + 4 * (lane & 1);
      const float4 v = make_float4(xs[c * XLD + rr], xs[(c + 1) * XLD + rr], xs[(c + 2) * XLD + rr], xs[(c + 3) * XLD + rr]);
      *reinterpret_cast<float4*>(xt + (static_cast<int64_t>(b) * N + n0 + rr) * C + c) = v;
    }
  } else if (xt) {
    for (int i = tid; i < 64 * C; i += 256) {
      const int rr = i / C, c = i - rr * C;
      xt[(static_cast<int64_t>(b) * N + n0 + rr) * C + c] = xs[c * XLD + rr];
    }
  }
  // node GEMM: thread (tx, ty) owns points 4 ty .. 4 ty + 3 and outputs {4 tx .. +3} U {64 + 4 tx .. +3} of each
  // 128-wide pass
  const int tx = tid & 15, ty = tid >> 4;
  for (int m0 = 0; m0 < M; m0 += 128) {
    // the chain per output - c ascending from 0 - and its bits are those of node_pq_kernel
    float2 acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = make_float2(0.f, 0.f);
#pragma unroll 4
    for (int c = 0; c < C; ++c) {
      const float4 a = *reinterpret_cast<const float4*>(xs + c * XLD + ty * 4);
      const float4 w0 = *reinterpret_cast<const float4*>(ws + c * M + m0 + tx * 4);
      const float4 w1 = *reinterpret_cast<const float4*>(ws + c * M + m0 + 64 + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float2 wv[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[i][j].x = fmaf(av[i], wv[j].x, acc[i][j].x);
          acc[i][j].y = fmaf(av[i], wv[j].y, acc[i][j].y);
        }
    }
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(g.bk + m0 + tx * 4));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(g.bk + m0 + 64 + tx * 4));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float* row = g.pq + (static_cast<int64_t>(b) * N + n0 + ty * 4 + i) * M + m0;
      *reinterpret_cast<float4*>(row + tx * 4) =
          make_float4(acc[i][0].x + b0.x, acc[i][0].y + b0.y, acc[i][1].x + b0.z, acc[i][1].y + b0.w);
      *reinterpret_cast<float4*>(row + 64 + tx * 4) =
          make_float4(acc[i][2].x + b1.x, acc[i][2].y + b1.y, acc[i][3].x + b1.z, acc[i][3].y + b1.w);
    }
  }
}
#endif  // DGCN_TEMPLATES_ONLY



// ---- the tensor-core kernel ------------------------------------------------------------------------
// eight consecutive floats as two 128-bit read-only loads; p must be 16-byte aligned
__device__ __forceinline__ void ldg_f8(const float* p, float (&w)[8]) {
  const float4 u = __ldg(reinterpret_cast<const float4*>(p)), v = __ldg(reinterpret_cast<const float4*>(p) + 1);
  w[0] = u.x; w[1] = u.y; w[2] = u.z; w[3] = u.w;
  w[4] = v.x; w[5] = v.y; w[6] = v.z; w[7] = v.w;
}

struct TcArgs {
  CUtensorMap tm_planes;         // bf16 (B*2*Cpad rows, N) row-major, box 64 points x Cpad rows, SWIZZLE_128B
  CUtensorMap tm_sqp;            // bf16 (B*8 rows, N), box 64 points x 8 rows, SWIZZLE_128B
  KnnArgs a;
  const __nv_bfloat16* planes;   // (B,2,Cpad,N)
  const __nv_bfloat16* sqp;      // (B,8,N): rows 0..2 = bf16 split of -|x|^2/2, rest zero
  const float* xt;               // (B,N,C) node-major fp32 copy (exact re-rank)
  const float* sqmax;            // (B)
  int Cpad;
  int wide;                      // consumer variant (cta_epilogue_wide)
  int work_bytes;                // size of the work area, see tc_work_bytes
  int xt32;                      // xt is 32-byte aligned: 8-float row loads in the exact re-rank
  int flush_early, flush_late;   // packed path: buffered candidates per lane that trigger a flush (tiles 0-1 / later)
  int* fail_count;               // device counter
  int* fail_list;                // (B*N) encoded b*N + q
};

constexpr int TC_THREADS = 128;                       // one warpgroup: thread r = query r
constexpr int TC_FLUSH_AT = 1;                        // unpacked (8-byte entries): flush whenever a lane buffered anything
constexpr int TC_BUF = 16;                            // 8-byte slots per thread, >= TC_FLUSH_AT - 1 + 16 (checked every 16 columns)
constexpr int TC_FLUSH_EARLY = 16;                    // packed 4-byte entries: 32 slots; tight threshold while the
constexpr int TC_FLUSH_LATE = 16;                     // list still moves a lot (first tiles), fuller batches afterwards
constexpr int TC_STAGE_BYTES = TC_PLANES * 2 * TC_MAX_C * 128;   // 32 KB: planes x 2 MN blocks x 64 rows x 128 B
constexpr int TC_XBLOCK_BYTES = 2 * 16 * 128;                    // 4 KB: one extra K=16 block, 2 MN blocks x 16 rows x 128 B
constexpr int TC_ACC_LD = 68;                                     // accumulator stage: 64 columns + 4 (conflict-free row reads)

// Shared memory of one CTA (128 queries of one cloud).
//   work (1024-aligned, work_bytes): while streaming [query planes 32 KB | candidate stage 32 KB |
//   query extra block 4 KB | candidate extra block 4 KB], all canonical MN-major SWIZZLE_128B:
//   [plane][mn_block(2)][Cpad rows][128 B]; the extra K=16 blocks hold ones (query side, rows 0..2) and the
//   bf16 split of -|x_j|^2/2 (candidate side), so the accumulator is x_i.x_j - |x_j|^2/2; afterwards
//   [exact-sorted lists KP x 128 x 8 B | sel 128 x sel_ld x 4 B | consumer scratch].
//   tail: the fixed-size part below.
struct TcTail {
  uint64_t cbuf[TC_BUF * TC_THREADS];               // 16 KB private candidate buffers, slot-major
  float acc[TILE][TC_ACC_LD];                       // 34 KB: one 128-query x 64-candidate accumulator block, row = query
  uint64_t mbar_tma;                                // the next tile's operands have landed (TMA complete_tx)
  uint64_t mbar_q;                                  // query planes + tile 0 have landed
  unsigned char ok[TILE];
};

// Bytes of the work area for list length KP, k kept neighbours and the chosen consumer.
__host__ __device__ inline int tc_sel_ld(int k) { return k | 1; }
__host__ __device__ inline size_t tc_work_bytes(int KP, int k, bool wide, int nch) {
  size_t after = static_cast<size_t>(KP) * TILE * 8 + static_cast<size_t>(TILE) * tc_sel_ld(k) * 4;
  after = (after + 15) & ~static_cast<size_t>(15);
  if (wide) after += static_cast<size_t>(TC_THREADS / 32) * 2 * nch * 4;             // red
  else after += 2 * static_cast<size_t>(32) * STAGE_LD * 4 + 2 * (TC_THREADS / 32) * 32 * 4 + 256;   // stage_max, stage_min, red
  const size_t stream = 2 * static_cast<size_t>(TC_STAGE_BYTES) + 2 * TC_XBLOCK_BYTES;
  const size_t w = after > stream ? after : stream;
  return (w + 1023) & ~static_cast<size_t>(1023);
}

// Branch-free insertion of (nk, nv) into the ascending register-resident list (k, v):
// k[i] <- nk < k[i-1] ? k[i-1] : (nk < k[i] ? nk : k[i]).  All indices are compile-time.
template <int KP>
__device__ __forceinline__ void reg_insert(uint32_t (&k)[KP], uint32_t (&v)[KP], uint32_t nk, uint32_t nv) {
  bool lt[KP];
#pragma unroll
  for (int i = 0; i < KP; ++i) lt[i] = nk < k[i];
#pragma unroll
  for (int i = KP - 1; i > 0; --i) {
    k[i] = lt[i - 1] ? k[i - 1] : (lt[i] ? nk : k[i]);
    v[i] = lt[i - 1] ? v[i - 1] : (lt[i] ? nv : v[i]);
  }
  k[0] = lt[0] ? nk : k[0];
  v[0] = lt[0] ? nv : v[0];
}

// Packed variant for N <= 4096: one register per entry = (float bits of the approximate squared
// distance, low 12 mantissa bits replaced by the candidate index).  Truncating the distance can only
// lower the certificate's cut, never invalidate it.
template <int KP>
__device__ __forceinline__ void reg_insert_packed(uint32_t (&k)[KP], uint32_t nk) {
  // k[i] <- min(max(nk, k[i-1]), k[i]) with the OLD k[i-1]: two integer min/max per entry, no predicates
#pragma unroll
  for (int i = KP - 1; i > 0; --i) k[i] = min(max(nk, k[i - 1]), k[i]);
  k[0] = min(nk, k[0]);
}

template <int KP, bool PACKED>
__global__ void __launch_bounds__(TC_THREADS, 1) knn_tc_kernel(const __grid_constant__ TcArgs t) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // SWIZZLE_128B atoms must sit on 1024-byte boundaries of the shared address space
  unsigned char* work = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  TcTail& sm = *reinterpret_cast<TcTail*>(work + t.work_bytes);
  const KnnArgs& a = t.a;
  const int tid = threadIdx.x;
  const int r = tid;                                    // query row
  const int b = blockIdx.y, q0 = blockIdx.x * TILE;
  const int N = a.N, Cpad = t.Cpad;
  const int plane_bytes = 2 * Cpad * 128;
  const float* sqb = a.sq + static_cast<int64_t>(b) * N;
  unsigned char* qstage = work;
  unsigned char* stage = work + TC_STAGE_BYTES;

  if (tid == 0) {
    // the TMA descriptors live in kernel-parameter space: fetch them into the descriptor cache before the first load
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&t.tm_planes)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&t.tm_sqp)) : "memory");
    mbar_init(&sm.mbar_tma, 1);
    mbar_init(&sm.mbar_q, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int ntiles = N / TILE;
  unsigned char* qx = work + 2 * TC_STAGE_BYTES;          // query-side extra block: ones in K rows 0..2
  unsigned char* sx = qx + TC_XBLOCK_BYTES;               // candidate-side extra block: -|x_j|^2/2 split in rows 0..2
  for (int ch = tid; ch < TC_XBLOCK_BYTES / 16; ch += TC_THREADS) {   // whole rows are constant: no swizzle needed
    const int row = (ch >> 3) & 15;
    const uint32_t one2 = row < 3 ? 0x3F803F80u : 0u;
    reinterpret_cast<uint4*>(qx)[ch] = make_uint4(one2, one2, one2, one2);
    reinterpret_cast<uint4*>(sx)[ch] = make_uint4(0u, 0u, 0u, 0u);        // rows 8..15 stay zero, TMA refreshes rows 0..7
  }
  fence_proxy_async();                                    // generic-proxy fills above -> visible to TMA / wgmma
  __syncthreads();                                        // barriers initialised, fills done
  // One elected thread moves operands.  A tile = 2 planes x 2 MN blocks (boxes of 64 points x Cpad channels) plus
  // the 2 x (64 points x 8 rows) boxes of the -|x_j|^2/2 block.
  const uint32_t tile_bytes = static_cast<uint32_t>(2 * plane_bytes + 2 * 8 * 128);
  auto tma_planes = [&](unsigned char* dst, int p0, uint64_t* bar) {
#pragma unroll
    for (int pl = 0; pl < TC_PLANES; ++pl)
#pragma unroll
      for (int blk = 0; blk < 2; ++blk)
        tma_load_2d(smem_u32(dst) + pl * plane_bytes + blk * (Cpad * 128), &t.tm_planes, p0 + blk * 64,
                    (b * TC_PLANES + pl) * Cpad, bar);
  };
  auto tma_sx = [&](int p0, uint64_t* bar) {
#pragma unroll
    for (int blk = 0; blk < 2; ++blk) tma_load_2d(smem_u32(sx) + blk * 2048, &t.tm_sqp, p0 + blk * 64, b * 8, bar);
  };
  if (tid == 0) {
    mbar_expect_tx(&sm.mbar_q, static_cast<uint32_t>(2 * plane_bytes) + tile_bytes);
    tma_planes(qstage, q0, &sm.mbar_q);
    tma_planes(stage, 0, &sm.mbar_q);
    tma_sx(0, &sm.mbar_q);
  }
  // The warpgroup multiplies the 128 queries against one 64-candidate MN block of the staged tile: rows 0..63 and
  // 64..127 as two m64n64 chains of 3 x Cpad/16 + 1 wgmma each, then the accumulators go to the shared stage where
  // thread r reads row r.
  const uint32_t abase = smem_u32(qstage), bbase = smem_u32(stage);
  auto mma_block = [&](int cb, float (&d0)[32], float (&d1)[32]) {
    const int pa[3] = {0, 0, 1};   // hi*hi, hi*mid, mid*hi  (mid*mid <= 2^-16 |x_i||x_j| is inside eps)
    const int pb[3] = {0, 1, 0};
    wg_fence();
    uint32_t acc = 0;
#pragma unroll 1
    for (int kk = 0; kk < Cpad / 16; ++kk) {
#pragma unroll
      for (int term = 0; term < 3; ++term) {
        const uint32_t ao = abase + pa[term] * plane_bytes + kk * 2048;
        const uint64_t db = wg_desc_sw128(bbase + pb[term] * plane_bytes + cb * (Cpad * 128) + kk * 2048, Cpad * 128, 1024);
        wgmma_m64n64<1, 1>(d0, wg_desc_sw128(ao, Cpad * 128, 1024), db, acc);
        wgmma_m64n64<1, 1>(d1, wg_desc_sw128(ao + Cpad * 128, Cpad * 128, 1024), db, acc);
        acc = 1;
      }
    }
    // + 1 x (-|x_j|^2/2): the accumulator becomes x_i.x_j - |x_j|^2/2 = -key/2
    const uint64_t dsx = wg_desc_sw128(smem_u32(sx) + cb * 2048, 2048, 1024);
    wgmma_m64n64<1, 1>(d0, wg_desc_sw128(smem_u32(qx), 2048, 1024), dsx, 1u);
    wgmma_m64n64<1, 1>(d1, wg_desc_sw128(smem_u32(qx) + 2048, 2048, 1024), dsx, 1u);
    wg_commit();
    wg_wait_all();
  };
  mbar_wait(&sm.mbar_q, 0u);

  const int qg = q0 + r;
  // the KP best approximate keys, ascending, in registers
  uint32_t lk[KP], lv[PACKED ? 1 : KP];
#pragma unroll
  for (int i = 0; i < KP; ++i) {
    lk[i] = 0xFFFFFFFFu;
    if (!PACKED) lv[i] = 0xFFFFFFFFu;
  }
  const float sqq = __ldg(sqb + qg);
  float tau_f = __uint_as_float(0x7FC00000u);     // NaN admits everything until the list is full
  float thr_acc = tau_f;
  // private candidate buffer, slot-major: PACKED 32 slots x 4 B (key bits | 12-bit index), else 16 x 8 B
  constexpr uint32_t ESZ = PACKED ? 4u : 8u;
  const uint32_t cb_addr0 = smem_u32(sm.cbuf) + tid * ESZ;
  uint32_t cb_addr = cb_addr0;      // next free slot of the private buffer (shared-space byte address)
  // Warp-synchronous flush: every lane merges ITS buffered candidates in lockstep.
  auto flush = [&]() {
    const int cnt = static_cast<int>((cb_addr - cb_addr0) / (TC_THREADS * ESZ));
    int mx = cnt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    // buffer reads are volatile asm so that they stay ordered behind the filter's (volatile asm) stores
    auto ld_entry32 = [&](int e) {
      uint32_t v;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(cb_addr0 + static_cast<uint32_t>(e) * (TC_THREADS * 4u)));
      return v;
    };
    auto ld_entry64 = [&](int e) {
      uint64_t v;
      asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(cb_addr0 + static_cast<uint32_t>(e) * (TC_THREADS * 8u)));
      return v;
    };
    uint32_t en_next = 0;
    uint64_t kv_next = 0;
    if (PACKED) en_next = ld_entry32(0); else kv_next = ld_entry64(0);   // slot 0 always exists
    for (int e = 0; e < mx; ++e) {
      uint32_t nk = 0xFFFFFFFFu, nv = 0u;
      const uint32_t en = en_next;
      const uint64_t kv = kv_next;
      if (e + 1 < mx) {                 // prefetch the next round's entry behind this round's insertion
        if (PACKED) en_next = ld_entry32(e + 1); else kv_next = ld_entry64(e + 1);
      }
      if (e < cnt) {
        if (PACKED) {
          // entry = accumulator bits (acc = -key/2) with the low 12 mantissa bits replaced by the index;
          // restore an UPPER bound of acc, i.e. a lower bound of the key
          const uint32_t ab = (en & 0x80000000u) ? (en & 0xFFFFF000u) : (en | 0xFFFu);
          const float d2 = fmaxf(fmaf(-2.0f, __uint_as_float(ab), sqq), 0.f);
          nk = (__float_as_uint(d2) & 0xFFFFF000u) | (en & 0xFFFu);
        } else {
          nv = static_cast<uint32_t>(kv);              // low word = index, high word = accumulator bits
          nk = float_to_ordered(-2.0f * __uint_as_float(static_cast<uint32_t>(kv >> 32)));
        }
      }
      if (nk < lk[KP - 1]) {
        if constexpr (PACKED) reg_insert_packed<KP>(lk, nk);
        else reg_insert<KP>(lk, lv, nk, nv);
      }
    }
    cb_addr = cb_addr0;
    if (PACKED) {   // admission in key units (distance minus |x_i|^2), one truncation step above the last entry
      tau_f = lk[KP - 1] == 0xFFFFFFFFu ? __uint_as_float(0x7FC00000u)
                                        : __uint_as_float((lk[KP - 1] & 0xFFFFF000u) + 0x1000u) - sqq;
    } else {
      tau_f = ordered_to_float(lk[KP - 1]);        // NaN while the list is not full
    }
    thr_acc = -0.5f * tau_f;                        // the filter compares accumulators: key <= tau  <=>  acc >= -tau/2
  };

  // Per tile t and 64-candidate block cb: wgmma -> barrier (everybody has read the previous block out of the stage;
  // after the last block, nobody reads the operand stage any more: thread 0 starts the TMA of tile t+1, which then
  // lands under the filter) -> accumulators to the stage -> barrier -> thread r filters row r in 16-column chunks.
  for (int tile = 0; tile < ntiles; ++tile) {
    if (tile > 0) mbar_wait(&sm.mbar_tma, static_cast<uint32_t>((tile - 1) & 1));
    // filter: thread = query; the accumulator is -key/2 with key = |x_j|^2 - 2 x_i.x_j
    // (row-constant |x_i|^2 omitted): admit when acc >= -tau/2.  The query itself is an ordinary candidate here
    // even with exclude_self (it is dropped in the exact re-rank below; the list is 8 entries longer than K) -
    // a per-thread column patch would turn the chunk registers into an addressable local-memory array.
    const int j0 = tile * TILE;
    const uint32_t flush_bytes = PACKED ? (tile < 2 ? t.flush_early : t.flush_late) * TC_THREADS * 4u
                                        : TC_FLUSH_AT * TC_THREADS * 8u;
    // One 16-column chunk: test, buffer, flush when a lane's buffer runs full (checked once per chunk).  A macro, not
    // a lambda: the body exists once per register buffer and the chunk registers never become an addressable array.
    // PACKED: one LOP3 builds the entry (key & R & I) | (R ^ I) with R = ~0xFFF | index bits 4..11 (tile, chunk) and
    // the immediate I = ~0xFFF | index bits 0..3.
#define DGCN_TC_FILTER16(V, C16)                                                                                      \
  do {                                                                                                                \
    const uint32_t rbits = 0xFFFFF000u | static_cast<uint32_t>(j0 + (C16) * 16);                                      \
    uint32_t jcur = static_cast<uint32_t>(j0 + (C16) * 16);                                                           \
    _Pragma("unroll") for (int i = 0; i < 16; ++i) {                                                                  \
      const uint32_t accb = V[i];                                                                                     \
      /* if (!(acc < thr_acc)) { buffer[slot] = entry; ++slot; }  - predicated, no branch */                          \
      if (PACKED) {                                                                                                   \
        const uint32_t ibits = 0xFFFFF000u | static_cast<uint32_t>(i);                                                \
        asm volatile(                                                                                                 \
            "{\n"                                                                                                     \
            ".reg .pred p;\n"                                                                                         \
            ".reg .b32 en;\n"                                                                                         \
            "lop3.b32 en, %1, %2, %5, 0xE6;\n" /* (a & b & c) | (b ^ c) */                                            \
            "setp.geu.f32 p, %6, %3;\n"                                                                               \
            "@p st.shared.b32 [%0], en;\n"                                                                            \
            "@p add.u32 %0, %0, %4;\n"                                                                                \
            "}"                                                                                                       \
            : "+r"(cb_addr)                                                                                           \
            : "r"(accb), "r"(rbits), "f"(thr_acc), "n"(TC_THREADS * 4), "r"(ibits), "f"(__uint_as_float(accb)));      \
      } else {                                                                                                        \
        asm volatile(                                                                                                 \
            "{\n"                                                                                                     \
            ".reg .pred p;\n"                                                                                         \
            "setp.geu.f32 p, %1, %3;\n"                                                                               \
            "@p st.shared.v2.b32 [%0], {%2, %1};\n"                                                                   \
            "@p add.u32 %0, %0, %4;\n"                                                                                \
            "}"                                                                                                       \
            : "+r"(cb_addr)                                                                                           \
            : "f"(__uint_as_float(accb)), "r"(jcur), "f"(thr_acc), "n"(TC_THREADS * 8));                              \
        ++jcur;                                                                                                       \
      }                                                                                                               \
    }                                                                                                                 \
    if (__any_sync(0xffffffffu, cb_addr - cb_addr0 >= flush_bytes)) flush();                                          \
  } while (0)
#pragma unroll 1
    for (int cb = 0; cb < 2; ++cb) {
      {
        float d0[32], d1[32];
        mma_block(cb, d0, d1);
        __syncthreads();
        if (cb == 1 && tile + 1 < ntiles && tid == 0) {
          mbar_expect_tx(&sm.mbar_tma, tile_bytes);
          tma_planes(stage, (tile + 1) * TILE, &sm.mbar_tma);
          tma_sx((tile + 1) * TILE, &sm.mbar_tma);
        }
        wg_store_m64n64(d0, &sm.acc[0][0], TC_ACC_LD, 0);
        wg_store_m64n64(d1, &sm.acc[0][0], TC_ACC_LD, 64);
      }
      __syncthreads();
      const float* arow = sm.acc[r];
#pragma unroll 1
      for (int c16 = 0; c16 < 4; ++c16) {
        uint32_t va[16];
#pragma unroll
        for (int i = 0; i < 16; i += 4) {
          const float4 v = *reinterpret_cast<const float4*>(arow + c16 * 16 + i);
          va[i] = __float_as_uint(v.x); va[i + 1] = __float_as_uint(v.y);
          va[i + 2] = __float_as_uint(v.z); va[i + 3] = __float_as_uint(v.w);
        }
        DGCN_TC_FILTER16(va, cb * 4 + c16);
      }
    }
#undef DGCN_TC_FILTER16
  }
  flush();
  __syncthreads();   // every wgmma has completed, nobody touches the operands any more

  // ---- exact re-rank of the listed candidates (fp32 FMA chain, k ascending) --------------------------
  uint64_t* list = reinterpret_cast<uint64_t*>(work);   // [KP][TILE]
  // lower bound of every unlisted candidate's approximate key (PACKED: of its squared distance)
  const float cut = (lk[KP - 1] == 0xFFFFFFFFu) ? INFINITY
                    : (PACKED ? __uint_as_float(lk[KP - 1] & 0xFFFFF000u) : ordered_to_float(lk[KP - 1]));
  const int C = a.C;
  const float* xtb = t.xt + static_cast<int64_t>(b) * N * C;
  {
    // pass 1: exact distances of all listed candidates.  Channels in chunks of 8 in the OUTER loop, candidates in
    // the inner one: every candidate keeps its own accumulator, so KP independent FMA chains are in flight (a single
    // 64-long chain per candidate would expose the FMA latency 64 times) and only 8 query channels are live at a
    // time.  Per candidate the chain is still acc = fma(x_q[c], x_j[c], acc) for c ascending from acc = 0 - the bits
    // of the fp32 kernel.
    float dex[KP];
    uint32_t off[KP];                 // element offset of the candidate's row in the node-major copy
#pragma unroll
    for (int u = 0; u < KP; ++u) {
      const bool listed = PACKED ? (lk[u] != 0xFFFFFFFFu) : (lk[u] != 0xFFFFFFFFu || lv[u] != 0xFFFFFFFFu);
      const uint32_t j = listed ? (PACKED ? (lk[u] & 0xFFFu) : lv[u]) : static_cast<uint32_t>(qg);
      off[u] = j * static_cast<uint32_t>(C);
      dex[u] = 0.f;
    }
    const float* xqp = xtb + static_cast<int64_t>(qg) * C;
    if ((C & 7) == 0 && t.xt32) {
      // one 256-bit load per 8 channels: each lane reads a different row, so every load is its own L1 wavefront
#pragma unroll 1
      for (int c = 0; c < C; c += 8) {
        float q8[8];
        ldg_f8(xqp + c, q8);
#pragma unroll
        for (int u = 0; u < KP; ++u) {
          float w[8];
          ldg_f8(xtb + off[u] + c, w);
#pragma unroll
          for (int i = 0; i < 8; ++i) dex[u] = fmaf(q8[i], w[i], dex[u]);
        }
      }
    } else if ((C & 3) == 0) {
#pragma unroll 1
      for (int c = 0; c < C; c += 4) {
        const float4 q4 = __ldg(reinterpret_cast<const float4*>(xqp + c));
#pragma unroll
        for (int u = 0; u < KP; ++u) {
          const float4 w = __ldg(reinterpret_cast<const float4*>(xtb + off[u] + c));
          dex[u] = fmaf(q4.x, w.x, dex[u]);
          dex[u] = fmaf(q4.y, w.y, dex[u]);
          dex[u] = fmaf(q4.z, w.z, dex[u]);
          dex[u] = fmaf(q4.w, w.w, dex[u]);
        }
      }
    } else {
      for (int c = 0; c < C; ++c) {
        const float q1 = __ldg(xqp + c);
#pragma unroll
        for (int u = 0; u < KP; ++u) dex[u] = fmaf(q1, __ldg(xtb + off[u] + c), dex[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < KP; ++u) {
      const bool listed = PACKED ? (lk[u] != 0xFFFFFFFFu) : (lk[u] != 0xFFFFFFFFu || lv[u] != 0xFFFFFFFFu);
      const uint32_t j = listed ? (PACKED ? (lk[u] & 0xFFFu) : lv[u]) : static_cast<uint32_t>(qg);
      dex[u] = (sqq + (-2.0f * dex[u])) + __ldg(sqb + j);
    }
    // pass 2: insertion by exact key into the exact-sorted prefix [0, e)
    int e = 0;
#pragma unroll
    for (int u = 0; u < KP; ++u) {
      const bool listed = PACKED ? (lk[u] != 0xFFFFFFFFu) : (lk[u] != 0xFFFFFFFFu || lv[u] != 0xFFFFFFFFu);
      const uint32_t j = PACKED ? (lk[u] & 0xFFFu) : lv[u];
      if (listed && !(a.exclude_self && j == static_cast<uint32_t>(qg))) {   // self exclusion (DilatedKnnGraph, loop=False)
        const uint64_t key = make_key(dex[u], j);
        int i = e;
        while (i > 0) {
          const uint64_t prev = list[(i - 1) * TILE + r];
          if (prev < key) break;
          list[i * TILE + r] = prev;
          --i;
        }
        list[i * TILE + r] = key;
        ++e;
      }
    }
    for (int i = e; i < KP; ++i) list[i * TILE + r] = KEY_MAX;
  }
  // ---- certificate (thread = query) ------------------------------------------------------------------
  {
    const uint64_t kth = list[(a.K - 1) * TILE + r];
    bool ok = kth != KEY_MAX;
    if (ok && cut < INFINITY) {
      const float dk = ordered_to_float(static_cast<uint32_t>(kth >> 32));
      const float smax = __ldg(t.sqmax + b);
      // |approx - exact fp32| <= eps.  Split error of x = hi + mid (bf16 round-to-nearest): |mid| <= 2^-8 |x|,
      // |x - hi - mid| <= 2^-17 |x|, so the dropped mid*mid product is <= 2^-16 |x_i||x_j| and the two residual
      // products together <= 2^-16 |x_i||x_j|: <= 2^-15 on x_i.x_j, 2 x 2^-15 = 2^-14 on the key.  Then ~4*Cpad
      // fp32 tensor-core accumulations and Cpad FMA-chain roundings (2^-23 each), the -|x_j|^2/2 term accumulated
      // with them (3-term bf16 split, roundings at magnitude <= smax/2) and the final additions (2^-20).
      const float eps = (2.0f * (3.0518e-5f + (5.0f * Cpad + 8.0f) * 1.1921e-7f)) * sqrtf(sqq * smax) +
                        9.537e-7f * (sqq + smax);
      ok = (dk + eps < (PACKED ? cut : cut + sqq));
    }
    sm.ok[r] = ok ? 1 : 0;
    if (!ok) {
      const int slot = atomicAdd(t.fail_count, 1);
      t.fail_list[slot] = b * N + qg;
    }
  }
  __syncthreads();
  // ---- consumer: sel and scratch follow the lists in the work area ---------------------------------------
  const int sel_ld = tc_sel_ld(a.k);
  int* sel = reinterpret_cast<int*>(work + static_cast<size_t>(KP) * TILE * 8);
  float* scratch = reinterpret_cast<float*>(
      work + ((static_cast<size_t>(KP) * TILE * 8 + static_cast<size_t>(TILE) * sel_ld * 4 + 15) & ~static_cast<size_t>(15)));
  const int cta = blockIdx.y * gridDim.x + blockIdx.x;
  if (t.wide) {
    if (a.epi.mode == EPI_EDGE && a.epi.norm == DGCN_NORM_BATCH_TRAIN)
      cta_epilogue_wide<TC_THREADS / 32, true>(a, b, q0, list, sm.ok, sel, sel_ld, scratch, cta, tid);
    else
      cta_epilogue_wide<TC_THREADS / 32, false>(a, b, q0, list, sm.ok, sel, sel_ld, scratch, cta, tid);
  } else {
    float* stage_max = scratch;
    float* stage_min = stage_max + 32 * STAGE_LD + 32;
    cta_epilogue<TC_THREADS / 32>(a, b, q0, list, sm.ok, sel, stage_max, stage_min, cta, sel_ld);
  }
}

// ---- exact completion of uncertified queries ------------------------------------------------------------
// One CTA per failed query: the 8 warps split the N candidates (lanes over candidates, exact fp32 FMA
// chain over channels, the query's channels broadcast from shared memory), each keeps a warp-wide
// sorted list of its best 64, the 8 lists are merged by one bitonic sort in shared memory, then warp 0
// runs the per-query consumer.  A lone uncertified query therefore costs ~N/256 candidate rounds, not N/32.
#ifndef DGCN_TEMPLATES_ONLY
__global__ void __launch_bounds__(256) knn_exact_rows_kernel(const KnnArgs a, const int* __restrict__ fail_count,
                                                            const int* __restrict__ fail_list,
                                                            float* __restrict__ partial_extra) {
  __shared__ float xq[TC_MAX_C];
  __shared__ uint64_t merged[8 * 64];
  __shared__ int sel[64];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total = *fail_count;
  const Epilogue& e = a.epi;
  const int N = a.N, C = a.C, k = a.k;
  float s1acc[4] = {0.f, 0.f, 0.f, 0.f}, s2acc[4] = {0.f, 0.f, 0.f, 0.f};   // c_out <= 128 covered per lane
  for (int f = blockIdx.x; f < total; f += gridDim.x) {
    const int code = fail_list[f];
    const int b = code / N, q = code % N;
    const float* xb = a.x + b * a.sb;
    const float* sqb = a.sq + static_cast<int64_t>(b) * N;
    const float sqq = sqb[q];
    __syncthreads();                       // the previous query's xq / merged / sel are no longer read
    if (tid < C) xq[tid] = __ldg(xb + tid * a.sc + q);
    __syncthreads();
    uint64_t r0 = KEY_MAX, r1 = KEY_MAX;   // this warp's sorted 64-entry list: r0 = ranks 0..31, r1 = 32..63
    for (int j0 = warp * 32; j0 < N; j0 += 256) {
      const int j = j0 + lane;
      uint64_t key = KEY_MAX;
      if (j < N && !(a.exclude_self && j == q)) {
        const float* xj = xb + j;
        float acc = 0.f;
#pragma unroll 8
        for (int c = 0; c < C; ++c) acc = fmaf(xq[c], __ldg(xj + c * a.sc), acc);
        key = make_key((sqq + (-2.0f * acc)) + sqb[j], static_cast<uint32_t>(j));
      }
      const uint64_t worst = shfl_u64(r1, 31);
      unsigned cand = __ballot_sync(0xffffffffu, key < worst);
      while (cand) {
        const int src = __ffs(cand) - 1;
        cand &= cand - 1;
        uint64_t carry = shfl_u64(key, src);
        // insert into r0, evicted element cascades into r1
        uint64_t last0 = shfl_u64(r0, 31);
        if (carry < last0) {
          int pos = __popc(__ballot_sync(0xffffffffu, r0 < carry));
          uint64_t up = shfl_up_u64(r0, 1);
          r0 = (lane == pos) ? carry : (lane > pos ? up : r0);
          carry = last0;
        }
        uint64_t last1 = shfl_u64(r1, 31);
        if (carry < last1) {
          int pos = __popc(__ballot_sync(0xffffffffu, r1 < carry));
          uint64_t up = shfl_up_u64(r1, 1);
          r1 = (lane == pos) ? carry : (lane > pos ? up : r1);
        }
      }
    }
    merged[warp * 64 + lane] = r0;
    merged[warp * 64 + 32 + lane] = r1;
    __syncthreads();
    if (warp != 0) continue;               // (the loop-top barrier keeps the CTA together)
    warp_bitonic_sort(merged, 512, lane);
    const int64_t node0 = static_cast<int64_t>(b) * N;
    for (int l = lane; l < k; l += 32) {
      const int idx = static_cast<int>(static_cast<uint32_t>(merged[keep_rank(a, l)]));
      sel[l] = idx;
      const int64_t o = (node0 + q) * k + l;
      if (e.nbr) e.nbr[o] = idx;
      if (e.edge_index) {
        e.edge_index[o] = idx;
        e.edge_index[static_cast<int64_t>(a.B) * N * k + o] = q;
      }
    }
    __syncwarp();
    if (e.mode == EPI_EDGE) {
      const float slope = epi_slope(e);
      const bool train = e.norm == DGCN_NORM_BATCH_TRAIN;
      for (int c0 = 0, u = 0; c0 < e.c_out; c0 += 32, ++u) {
        const int c = c0 + lane;
        float vmax, vmin, s1 = 0.f, s2 = 0.f, bs, bt;
        bn_affine(e, c, bs, bt);
        edge_query(e, node0, q, sel, k, c, slope, vmax, vmin, s1, s2);
        if (c < e.c_out) {
          const int64_t o = (static_cast<int64_t>(b) * e.c_out + c) * N + q;
          const int64_t oo = b * e.out_sb + static_cast<int64_t>(c) * N + q;
          if (train) {
            e.out[oo] = vmax;
            e.out_min[o] = vmin;
            if (u < 4) {
              s1acc[u] += s1;
              s2acc[u] += s2;
            }
          } else {
            e.out[oo] = epi_res(e, b, c, q, bs >= 0.f ? fmaf(bs, vmax, bt) : fmaf(bs, vmin, bt));
          }
        }
      }
    } else if (e.mode == EPI_MR) {
      for (int c0 = 0; c0 < e.c_in; c0 += 32) {
        const int c = c0 + lane;
        const float r = mr_query(e, node0, q, sel, k, c);
        if (c < e.c_in) e.r_out[(static_cast<int64_t>(b) * e.c_in + c) * N + q] = r;
      }
    }
    __syncwarp();
  }
  // train-mode statistics of the queries completed here: one extra partial row per CTA (warp 0 holds them)
  if (warp == 0 && e.mode == EPI_EDGE && e.norm == DGCN_NORM_BATCH_TRAIN && partial_extra) {
    const int64_t rowi = blockIdx.x;
    for (int u = 0; u < 4; ++u) {
      const int c = u * 32 + lane;
      if (c < e.c_out) {
        partial_extra[(rowi * 2 + 0) * e.c_out + c] = s1acc[u];
        partial_extra[(rowi * 2 + 1) * e.c_out + c] = s2acc[u];
      }
    }
  }
}
#endif  // DGCN_TEMPLATES_ONLY

// ---- per-list-length launchers --------------------------------------------------------------------------
// Each list length KP is instantiated in its own translation unit (knn_tc_kp*.cu, compiled in parallel with
// DGCN_TEMPLATES_ONLY so that the non-template kernels of these headers are not duplicated).
template <int KP>
inline int launch_knn_tc_inst(bool packed, const TcArgs& t, dim3 grid, size_t smem, cudaStream_t stream) {
  if (packed) {
    DGCN_ENSURE_SMEM((knn_tc_kernel<KP, true>), smem);
    knn_tc_kernel<KP, true><<<grid, TC_THREADS, smem, stream>>>(t);
  } else {
    DGCN_ENSURE_SMEM((knn_tc_kernel<KP, false>), smem);
    knn_tc_kernel<KP, false><<<grid, TC_THREADS, smem, stream>>>(t);
  }
  return DGCN_OK;
}
int launch_knn_tc_kp16(bool packed, const TcArgs& t, dim3 grid, size_t smem, cudaStream_t stream);
int launch_knn_tc_kp28(bool packed, const TcArgs& t, dim3 grid, size_t smem, cudaStream_t stream);
int launch_knn_tc_kp40(bool packed, const TcArgs& t, dim3 grid, size_t smem, cudaStream_t stream);
int launch_knn_tc_kp56(bool packed, const TcArgs& t, dim3 grid, size_t smem, cudaStream_t stream);

}  // namespace dgcn

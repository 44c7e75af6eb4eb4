// Row-wise Linear with fused bias / skip connection on the Hopper tensor cores (wgmma):
//
//     out[n][m] = sum_k a[n][k] * W[m][k]  (+ bias[m])  (+ res[n][m])          a (N,K), W (M,K), out / res (N,M), fp32
//
// = the `Linear` that ends GENConv's MLP (gcn_lib/sparse/torch_nn.py:56-68, mlp_layers = 1) together with the
// `+ h` of DeeperGCN's 'res+' block (examples/ogb/ogbn_arxiv/model.py:91-106).  The GEMM is skinny (K, M <= 256)
// and the rows are many, so it is bound by HBM (read a and res, write out once each), not by the tensor pipe; the
// point of the kernel is that everything else rides on that single pass.
//
// fp32 accuracy on bf16 tensor cores: a = a_hi + a_mid, W = W_hi + W_mid (bf16 round-to-nearest each,
// |x - hi - mid| <= 2^-17 |x|), products a_hi W_hi + a_hi W_mid + a_mid W_hi + a_mid W_mid accumulated in fp32:
// error <= ~2^-16 sum_k |a||W| (1.5e-5 relative to the magnitude sum), two orders below the 1e-3 parity
// tolerance.  W is split once per call by a prep kernel; a is split on the fly by the producer warps.
//
// One persistent CTA per SM, 384 threads:
//   warps 8-11 (producers)  tile of 128 rows: coalesced 128-bit loads of a -> (hi, mid) bf16 -> shared memory in the
//                          canonical K-major SWIZZLE_128B layout [plane][K/64][128 rows][128 B].
//   warps 0-7 (consumers)  warpgroup wg = rows 64 wg .. 64 wg + 63 of the tile: 4 x K/16 wgmma m64n32k16 per 32-column
//                          block of the output into registers (up to 8 blocks = M 256), the A buffer is handed back to
//                          the producers as soon as the wgmma have completed - they fill the next tile under this
//                          epilogue -, then out = acc + bias + res straight from the accumulator fragments (each quad
//                          of lanes covers 8 consecutive floats = one 32-byte sector of a row).
//   W (hi, mid)            resident in shared memory for the life of the CTA, loaded once by TMA.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace dgcn {

constexpr int RL_TILE = 128;          // rows per tile = MMA M
constexpr int RL_MAX = 256;           // K and M upper bound

__device__ __forceinline__ uint32_t rl_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void rl_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(rl_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void rl_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(rl_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void rl_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(rl_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void rl_mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spin = 0;; ++spin) {   // bounded: a pipeline that never signals must trap, not hang the GPU
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
        "selp.u32 %0, 1, 0, P1;\n"
        "}"
        : "=r"(done)
        : "r"(rl_smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    if (spin > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void rl_tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(rl_smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// W (M,K) fp32 -> Wp (2, M, K) bf16 (hi, mid)
__global__ void rl_split_weights_kernel(const float* __restrict__ w, int64_t n, __nv_bfloat16* __restrict__ wp) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = w[i];
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  wp[i] = hi;
  wp[n + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

struct RlArgs {
  CUtensorMap tm_w;         // bf16 (2*M rows, K), box 64 x M, SWIZZLE_128B
  const float* a;
  const float* bias;        // (M) or null
  const float* res;         // (N, M) or null
  float* out;
  int64_t N;
  int K, M;
};

struct RlBars {
  uint64_t w_full;          // W planes landed
  uint64_t a_full;          // all 128 producer threads wrote (and fenced) their part of the A tile
  uint64_t a_free;          // the 256 consumer threads' wgmma on the A tile have completed
};

constexpr int RL_EPI_THREADS = 256;   // warps 0..7
constexpr int RL_NB = RL_MAX / 32;    // 32-column output blocks

__global__ void __launch_bounds__(RL_EPI_THREADS + 128, 1) rowlinear_tc_kernel(const __grid_constant__ RlArgs g) {
  extern __shared__ __align__(16) unsigned char rl_smem[];
  unsigned char* base = rl_smem + ((1024u - (rl_smem_u32(rl_smem) & 1023u)) & 1023u);
  const int K = g.K, M = g.M;
  const int kblocks = K / 64;
  const uint32_t w_plane = static_cast<uint32_t>(M) * K * 2;            // bytes of one W plane
  const uint32_t a_plane = static_cast<uint32_t>(RL_TILE) * K * 2;
  unsigned char* w_s = base;                                            // [2][kblocks][M][128 B]
  unsigned char* a_s = w_s + 2 * w_plane;                               // [2][kblocks][128][128 B]
  RlBars& bar = *reinterpret_cast<RlBars*>(a_s + 2 * a_plane);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int64_t ntiles = (g.N + RL_TILE - 1) / RL_TILE;

  if (tid == 0) {
    rl_mbar_init(&bar.w_full, 1);
    rl_mbar_init(&bar.a_full, 128);
    rl_mbar_init(&bar.a_free, RL_EPI_THREADS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= RL_EPI_THREADS / 32) {
    // ======================= producers ===============================================================================
    const int pt = tid - RL_EPI_THREADS;
    if (pt == 0) {   // W: one box of 64 k x M rows per (plane, k-block)
      rl_mbar_expect_tx(&bar.w_full, 2 * w_plane);
      for (int pl = 0; pl < 2; ++pl)
        for (int kb = 0; kb < kblocks; ++kb)
          rl_tma_load_2d(rl_smem_u32(w_s) + pl * w_plane + kb * (M * 128), &g.tm_w, kb * 64, pl * M, &bar.w_full);
    }
    const int chunks = K / 8;                       // 16-byte bf16 chunks per row
    const int rows_per_pass = 128 / chunks;         // K = 64: 16 rows, 128: 8 rows, 256: 4 rows
    const int cg = pt % chunks, rsub = pt / chunks; // my chunk of the row, my row inside a pass
    const int kb = cg >> 3, c = cg & 7;
    int64_t it = 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int64_t row0 = tile * RL_TILE;
      // eight passes at a time: all sixteen 128-bit loads of a group are issued before the first conversion, so a
      // producer warp keeps 8 KB of the a-stream in flight (the kernel is HBM bound: memory-level parallelism is
      // what matters)
      for (int r0 = 0; r0 < RL_TILE; r0 += 8 * rows_per_pass) {
        float4 lo[8], hi4[8];
#pragma unroll
        for (int p8 = 0; p8 < 8; ++p8) {
          const int row = r0 + p8 * rows_per_pass + rsub;
          lo[p8] = make_float4(0.f, 0.f, 0.f, 0.f);
          hi4[p8] = lo[p8];
          if (row < RL_TILE && row0 + row < g.N) {
            const float4* src = reinterpret_cast<const float4*>(g.a + (row0 + row) * K + cg * 8);
            lo[p8] = __ldg(src);
            hi4[p8] = __ldg(src + 1);
          }
        }
        // the A buffer is still read by the previous tile's wgmma: wait only now, with this tile's first loads in flight
        if (r0 == 0 && it > 0) rl_mbar_wait(&bar.a_free, static_cast<uint32_t>((it - 1) & 1));
#pragma unroll
        for (int p8 = 0; p8 < 8; ++p8) {
          const int row = r0 + p8 * rows_per_pass + rsub;
          if (row >= RL_TILE) continue;
          const float v[8] = {lo[p8].x, lo[p8].y, lo[p8].z, lo[p8].w, hi4[p8].x, hi4[p8].y, hi4[p8].z, hi4[p8].w};
          uint32_t ph[4], pm[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const __nv_bfloat16 h0 = __float2bfloat16_rn(v[2 * i]), h1 = __float2bfloat16_rn(v[2 * i + 1]);
            const __nv_bfloat16 m0 = __float2bfloat16_rn(v[2 * i] - __bfloat162float(h0));
            const __nv_bfloat16 m1 = __float2bfloat16_rn(v[2 * i + 1] - __bfloat162float(h1));
            ph[i] = static_cast<uint32_t>(__bfloat16_as_ushort(h0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h1)) << 16);
            pm[i] = static_cast<uint32_t>(__bfloat16_as_ushort(m0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(m1)) << 16);
          }
          unsigned char* dst = a_s + kb * (RL_TILE * 128) + row * 128 + ((c ^ (row & 7)) << 4);
          *reinterpret_cast<uint4*>(dst) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
          *reinterpret_cast<uint4*>(dst + a_plane) = make_uint4(pm[0], pm[1], pm[2], pm[3]);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // my generic-proxy stores -> tensor-core reads
      rl_mbar_arrive(&bar.a_full);
    }
  } else {
    // ======================= consumers: wgmma, then out = acc + bias + res ==========================================
    const int wg = warp >> 2;
    const int nb = M / 32;
    const uint32_t a_base = rl_smem_u32(a_s) + static_cast<uint32_t>(wg) * (64 * 128);   // rows 64 wg .. of every k-block
    const uint32_t w_base = rl_smem_u32(w_s);
    int64_t it = 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      if (it == 0) rl_mbar_wait(&bar.w_full, 0u);
      rl_mbar_wait(&bar.a_full, static_cast<uint32_t>(it & 1));
      float d[RL_NB][16];
      wg_fence();
#pragma unroll
      for (int j = 0; j < RL_NB; ++j) {
        if (j < nb) {
          for (int kk = 0; kk < K / 16; ++kk) {
            const uint32_t koff = static_cast<uint32_t>(kk >> 2) * (RL_TILE * 128) + static_cast<uint32_t>(kk & 3) * 32;
            const uint32_t woff = static_cast<uint32_t>(kk >> 2) * (M * 128) + static_cast<uint32_t>(j) * (32 * 128) +
                                  static_cast<uint32_t>(kk & 3) * 32;
#pragma unroll
            for (int term = 0; term < 4; ++term) {   // hi*hi, hi*mid, mid*hi, mid*mid
              const uint32_t pa = (term >> 1) * a_plane, pb = (term & 1) * w_plane;
              wgmma_m64n32<0, 0>(d[j], wg_desc_sw128(a_base + pa + koff, 16, 1024), wg_desc_sw128(w_base + pb + woff, 16, 1024),
                                 (kk | term) != 0 ? 1u : 0u);
            }
          }
        }
      }
      wg_commit();
      wg_wait_all();
      rl_mbar_arrive(&bar.a_free);
      const int64_t rbase = tile * RL_TILE + wg * 64;
#pragma unroll
      for (int j = 0; j < RL_NB; ++j) {
        if (j < nb) {
#pragma unroll
          for (int i = 0; i < 16; i += 2) {
            const int64_t row = rbase + wg_frag_row(i);
            const int col = j * 32 + wg_frag_col(i);
            if (row < g.N) {
              float2 v = make_float2(d[j][i], d[j][i + 1]);
              if (g.bias) {   // two scalar loads: bias needs only 4-byte alignment (M floats, L1-resident)
                v.x += __ldg(g.bias + col);
                v.y += __ldg(g.bias + col + 1);
              }
              if (g.res) {
                const float2 rv = __ldg(reinterpret_cast<const float2*>(g.res + row * M + col));
                v.x += rv.x;
                v.y += rv.y;
              }
              *reinterpret_cast<float2*>(g.out + row * M + col) = v;
            }
          }
        }
      }
    }
  }
}

typedef CUresult (*RlEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static RlEncodeFn rl_encoder() {
  static std::atomic<void*> cached{nullptr};
  void* fn = cached.load(std::memory_order_acquire);
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    cached.store(fn, std::memory_order_release);
  }
  return reinterpret_cast<RlEncodeFn>(fn);
}

static size_t rl_smem_bytes(int64_t K, int64_t M) {
  return static_cast<size_t>(2) * M * K * 2 + static_cast<size_t>(2) * RL_TILE * K * 2 + sizeof(RlBars) + 1024;
}
static bool rl_shape_ok(int64_t K, int64_t M) {
  // 128 | rows per pass = 1024 / K; W planes + A planes must fit the 227 KB of one SM
  return (K == 64 || K == 128 || K == 256) && M >= 32 && M <= RL_MAX && M % 32 == 0 && rl_smem_bytes(K, M) <= 227 * 1024;
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

size_t dgcn_linear_residual_workspace_bytes(int64_t K, int64_t M) {
  return rl_shape_ok(K, M) ? align_up(static_cast<size_t>(2) * M * K * 2, 256) + 256 : 0;
}

int dgcn_linear_residual(const float* a, int64_t N, int64_t K, const float* weight, const float* bias, int64_t M,
                         const float* res, float* out, void* wsp, size_t ws_bytes, dgcn_stream_t stream_) {
  if (!a || !weight || !out || N < 0 || K <= 0 || M <= 0) return DGCN_ERR_BAD_ARG;
  if (!rl_shape_ok(K, M)) return DGCN_ERR_UNSUPPORTED;
  if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(res)) & 15) != 0)
    return DGCN_ERR_UNSUPPORTED;
  if (N == 0) return DGCN_OK;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Workspace ws(wsp, ws_bytes);
  __nv_bfloat16* wp = ws.take<__nv_bfloat16>(static_cast<size_t>(2) * M * K);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  RlEncodeFn enc = rl_encoder();
  if (!enc) return DGCN_ERR_UNSUPPORTED;
  rl_split_weights_kernel<<<static_cast<unsigned>(ceil_div(M * K, 256)), 256, 0, stream>>>(weight, M * K, wp);
  DGCN_LAUNCH_CHECK();
  RlArgs g{};
  {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(2 * M)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(K) * 2};
    const cuuint32_t box[2] = {64u, static_cast<cuuint32_t>(M)};
    const cuuint32_t estr[2] = {1u, 1u};
    if (enc(&g.tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, wp, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return DGCN_ERR_CUDA;
  }
  g.a = a; g.bias = bias; g.res = res; g.out = out; g.N = N; g.K = static_cast<int>(K); g.M = static_cast<int>(M);
  const size_t smem = rl_smem_bytes(K, M);
  DGCN_ENSURE_SMEM((rowlinear_tc_kernel), smem);
  int dev = 0, sms = 0;
  DGCN_CUDA_TRY(cudaGetDevice(&dev));
  DGCN_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t ntiles = ceil_div(N, RL_TILE);
  const unsigned grid = static_cast<unsigned>(ntiles < sms ? ntiles : sms);
  {
    KernelTimer timer(stream, "linear");
    rowlinear_tc_kernel<<<grid, RL_EPI_THREADS + 128, smem, stream>>>(g);
  }
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // extern "C"

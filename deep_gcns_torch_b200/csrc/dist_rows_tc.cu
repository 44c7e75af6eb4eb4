// Distance rows of the large-K slab path on the Hopper tensor cores (wgmma).
//
//   D[i][j] = (|x_i|^2 + (-2 x_i.x_j)) + |x_j|^2        gcn_lib/dense/torch_edge.py:32-42 (pairwise_distance)
//
// for all pairs of one cloud, written as fp32 rows of the L2-sized slab that select_rows_fast_kernel consumes
// (K = k * dilation > 48: the 25 dilated layers of ResGCN-28).  The contraction runs as a THREE-plane bf16 split
// x = hi + mid + lo (24 bits: the split is exact) with the six products
//   hi*hi, hi*mid, mid*hi, mid*mid, hi*lo, lo*hi
// accumulated in fp32.  Dropped terms (mid*lo, lo*mid, lo*lo) are <= 2^-23 |x_i||x_j|; what remains is the
// fp32 accumulation of exact bf16 products - an fp32-grade value of the same formula, closer to the fp64 distance
// than a 64-step fp32 FMA chain, NOT bit-identical to it.  The ranking contract of the slab path is the oracle's:
// equal to the reference on tie-free inputs, mismatches only between candidates whose fp64 distances differ by
// < 1e-5 relative (tests adjudicate in fp64).  The certified pre-filter of K <= 48 (knn_tc.cuh) is unaffected; the
// call flag DGCN_KNN_EXACT_FP32 keeps the fp32 FMA rows.
//
// One CTA per (128 queries, chunk of candidate tiles) of a cloud - the candidate range is split so that one cloud
// fills the SMs -, 288 threads: warpgroups 0-1 = query rows 0..63 / 64..127 (wgmma m64n64k16 into registers,
// epilogue straight from the accumulator fragments), warp 8 = producer (one elected thread: TMA).  Query planes
// resident (3 x 16 KB), candidate tiles of 128 points through a 2-stage ring (2 x 48 KB) by TMA (SWIZZLE_128B boxes =
// canonical MN-major wgmma layout, like knn_tc): the TMA of tile t+2 runs under the wgmma and epilogue of tile t+1.
// Epilogue: each quad of lanes stores 8 consecutive floats (one 32-byte sector) of a row of
// (sq_i + (-2 acc)) + sq_j.
#include <cuda.h>
#include <cuda_bf16.h>

#define DGCN_TEMPLATES_ONLY      // device helpers of knn_tc.cuh only: its kernels live in dense_fwd.cu
#include "knn_tc.cuh"
#include "wgmma.cuh"

namespace dgcn {

constexpr int DR_PLANES = 3;
constexpr int DR_PLANE_BYTES = 2 * TC_MAX_C * 128;          // one plane of 128 points: 2 MN blocks x 64 rows x 128 B

// x -> (hi, mid, lo) bf16 planes (B, 3, Cpad, N), channel-major like x; sq (B, N) with sqnorm_kernel's FMA chain.
__global__ void __launch_bounds__(256) dr_planes3_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int Cpad,
                                                        int N, float* __restrict__ sq, __nv_bfloat16* __restrict__ planes) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (n >= N) return;
  const int64_t plane = static_cast<int64_t>(Cpad) * N;
  __nv_bfloat16* pb = planes + static_cast<int64_t>(b) * DR_PLANES * plane + n;
  float s = 0.f;
  for (int c = 0; c < Cpad; ++c) {
    const float v = c < C ? __ldg(x + b * sb + c * sc + n) : 0.f;
    s = fmaf(v, v, s);
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const float r1 = v - __bfloat162float(hi);
    const __nv_bfloat16 mid = __float2bfloat16_rn(r1);
    const __nv_bfloat16 lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
    pb[static_cast<int64_t>(c) * N] = hi;
    pb[plane + static_cast<int64_t>(c) * N] = mid;
    pb[2 * plane + static_cast<int64_t>(c) * N] = lo;
  }
  sq[static_cast<int64_t>(b) * N + n] = s;
}

struct DrArgs {
  CUtensorMap tm_planes;      // bf16 (B*3*Cpad rows, N), box 64 points x Cpad rows, SWIZZLE_128B
  const float* sq;            // (B, N)
  float* drows;               // slab: row (b - b0) * N + q, leading dimension ldd
  int b0, N, Cpad, ldd;
};

struct DrBars {
  uint64_t q_full;            // query planes landed
  uint64_t tma_full[2];       // candidate stage s landed
  uint64_t stage_free[2];     // the 256 consumer threads have finished their wgmma on stage s
};

__global__ void __launch_bounds__(288, 1) dist_rows_tc_kernel(const __grid_constant__ DrArgs g) {
  extern __shared__ __align__(16) unsigned char dr_smem[];
  unsigned char* base = dr_smem + ((1024u - (smem_u32(dr_smem) & 1023u)) & 1023u);
  unsigned char* qs = base;                                        // [3 planes][2 MN][Cpad rows][128 B]
  unsigned char* cs = qs + DR_PLANES * DR_PLANE_BYTES;             // 2 stages of the same
  float* sqq_s = reinterpret_cast<float*>(cs + 2 * DR_PLANES * DR_PLANE_BYTES);   // [128] |x_i|^2 of the queries
  DrBars& bar = *reinterpret_cast<DrBars*>(sqq_s + TILE);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int N = g.N, Cpad = g.Cpad;
  const int bl = blockIdx.z, b = g.b0 + bl, q0 = blockIdx.x * TILE;
  const int ntiles = (N / TILE) / static_cast<int>(gridDim.y);          // candidate tiles of this CTA
  const int tile0 = static_cast<int>(blockIdx.y) * ntiles;              // first of them
  const int plane_bytes = 2 * Cpad * 128;
  if (tid == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&g.tm_planes)) : "memory");
    mbar_init(&bar.q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bar.tma_full[i], 1);
      mbar_init(&bar.stage_free[i], 256);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < TILE) sqq_s[tid] = __ldg(g.sq + static_cast<int64_t>(b) * N + q0 + tid);
  __syncthreads();

  if (warp == 8) {
    if ((tid & 31) == 0) {
      // ===================== producer: TMA =====================================================================
      auto tma_tile = [&](unsigned char* dst, int p0, uint64_t* mb) {
        mbar_expect_tx(mb, static_cast<uint32_t>(DR_PLANES * plane_bytes));
        for (int pl = 0; pl < DR_PLANES; ++pl)
          for (int blk = 0; blk < 2; ++blk)
            tma_load_2d(smem_u32(dst) + pl * plane_bytes + blk * (Cpad * 128), &g.tm_planes, p0 + blk * 64,
                        (b * DR_PLANES + pl) * Cpad, mb);
      };
      tma_tile(qs, q0, &bar.q_full);
      tma_tile(cs, tile0 * TILE, &bar.tma_full[0]);
      if (ntiles > 1) tma_tile(cs + DR_PLANES * plane_bytes, (tile0 + 1) * TILE, &bar.tma_full[1]);
      // the stage of tile t is free once both warpgroups' wgmma on it have completed: refill it with tile t + 2
      for (int t = 0; t + 2 < ntiles; ++t) {
        const int s = t & 1;
        mbar_wait(&bar.stage_free[s], static_cast<uint32_t>((t >> 1) & 1));
        tma_tile(cs + s * DR_PLANES * plane_bytes, (tile0 + t + 2) * TILE, &bar.tma_full[s]);
      }
    }
  } else {
    // ===================== warpgroup wg: query rows 64 wg .. 64 wg + 63 =========================================
    const int wg = warp >> 2;
    const int pa[6] = {0, 0, 1, 1, 0, 2};   // hi*hi, hi*mid, mid*hi, mid*mid, hi*lo, lo*hi
    const int pb[6] = {0, 1, 0, 1, 2, 0};
    const float* sqb = g.sq + static_cast<int64_t>(b) * N;
    float* rows = g.drows + (static_cast<int64_t>(bl) * N + q0 + wg * 64) * g.ldd;
    const uint32_t abase = smem_u32(qs) + wg * (Cpad * 128);
    mbar_wait(&bar.q_full, 0u);
    for (int t = 0; t < ntiles; ++t) {
      const int s = t & 1;
      mbar_wait(&bar.tma_full[s], static_cast<uint32_t>((t >> 1) & 1));
      const uint32_t bbase = smem_u32(cs + s * DR_PLANES * plane_bytes);
      float d0[32], d1[32];                 // candidates 0..63 / 64..127 of the tile
      wg_fence();
      for (int kk = 0; kk < Cpad / 16; ++kk) {
#pragma unroll
        for (int term = 0; term < 6; ++term) {
          const uint32_t acc = (kk | term) != 0 ? 1u : 0u;
          const uint64_t da = wg_desc_sw128(abase + pa[term] * plane_bytes + kk * 2048, Cpad * 128, 1024);
          const uint32_t bo = bbase + pb[term] * plane_bytes + kk * 2048;
          wgmma_m64n64<1, 1>(d0, da, wg_desc_sw128(bo, Cpad * 128, 1024), acc);
          wgmma_m64n64<1, 1>(d1, da, wg_desc_sw128(bo + Cpad * 128, Cpad * 128, 1024), acc);
        }
      }
      wg_commit();
      wg_wait_all();
      mbar_arrive(&bar.stage_free[s]);
      const int col0 = (tile0 + t) * TILE;
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int rr = wg_frag_row(i), c = col0 + wg_frag_col(i);
        const float sqi = sqq_s[wg * 64 + rr];
        const float2 sj0 = __ldg(reinterpret_cast<const float2*>(sqb + c));
        const float2 sj1 = __ldg(reinterpret_cast<const float2*>(sqb + c + 64));
        float* row = rows + static_cast<int64_t>(rr) * g.ldd;
        *reinterpret_cast<float2*>(row + c) = make_float2((sqi + (-2.0f * d0[i])) + sj0.x, (sqi + (-2.0f * d0[i + 1])) + sj0.y);
        *reinterpret_cast<float2*>(row + c + 64) =
            make_float2((sqi + (-2.0f * d1[i])) + sj1.x, (sqi + (-2.0f * d1[i + 1])) + sj1.y);
      }
    }
  }
}

typedef CUresult (*DrEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static DrEncodeFn dr_encoder() {
  static std::atomic<void*> cached{nullptr};
  void* fn = cached.load(std::memory_order_acquire);
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    cached.store(fn, std::memory_order_release);
  }
  return reinterpret_cast<DrEncodeFn>(fn);
}

bool dist_rows_tc_ok(const KnnArgs& a) {
  return !a.exact_fp32 && a.C <= TC_MAX_C && a.N >= TILE && (a.N % TILE) == 0;
}
size_t dist_rows_tc_plane_elems(int64_t B, int64_t C, int64_t N) {
  const int64_t cpad = (C + 15) / 16 * 16;
  return static_cast<size_t>(B) * DR_PLANES * cpad * N;
}

// sq and the three bf16 planes of every cloud (one pass over x); sq overwrites a.sq's buffer
int dist_rows_tc_prepare(const KnnArgs& a, __nv_bfloat16* planes, cudaStream_t stream) {
  const int cpad = (a.C + 15) / 16 * 16;
  dr_planes3_kernel<<<dim3(static_cast<unsigned>(ceil_div(a.N, 256)), a.B), 256, 0, stream>>>(
      a.x, a.sb, a.sc, a.C, cpad, a.N, const_cast<float*>(a.sq), planes);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

// distance rows of clouds [b0, b0 + nb) into the slab
int dist_rows_tc_launch(const KnnArgs& a, const __nv_bfloat16* planes, int b0, int nb, float* drows, int ldd,
                        cudaStream_t stream) {
  DrEncodeFn enc = dr_encoder();
  if (!enc) return DGCN_ERR_UNSUPPORTED;
  const int cpad = (a.C + 15) / 16 * 16;
  DrArgs g{};
  {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(a.N), static_cast<cuuint64_t>(a.B) * DR_PLANES * cpad};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(a.N) * 2};
    const cuuint32_t box[2] = {64u, static_cast<cuuint32_t>(cpad)};
    const cuuint32_t estr[2] = {1u, 1u};
    if (enc(&g.tm_planes, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16*>(planes), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return DGCN_ERR_CUDA;
  }
  g.sq = a.sq; g.drows = drows; g.b0 = b0; g.N = a.N; g.Cpad = cpad; g.ldd = ldd;
  const size_t smem = static_cast<size_t>(3) * DR_PLANES * DR_PLANE_BYTES + TILE * 4 + sizeof(DrBars) + 1024;
  DGCN_ENSURE_SMEM((dist_rows_tc_kernel), smem);
  // split the candidate tiles of a query tile over CTAs until one launch fills the SMs (one CTA per SM: 146 KB smem)
  int dev = 0, sms = 0;
  DGCN_CUDA_TRY(cudaGetDevice(&dev));
  DGCN_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int ntiles = a.N / TILE;
  int split = 1;
  while (split * 2 <= ntiles && ntiles % (split * 2) == 0 && static_cast<int64_t>(ntiles) * nb * split * 2 <= sms) split *= 2;
  dist_rows_tc_kernel<<<dim3(ntiles, split, nb), 288, smem, stream>>>(g);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // namespace dgcn

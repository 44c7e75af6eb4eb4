// Dense path, forward: C ABI entry points dgcn_knn_graph / dgcn_graph_conv_forward /
// dgcn_dyn_conv_forward and the node-level kernels around the selection kernels.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <stdlib.h>
#include "knn_tc4.cuh"

namespace dgcn {

// tensor-core distance rows of the large-K slab path (dist_rows_tc.cu)
bool dist_rows_tc_ok(const KnnArgs& a);
size_t dist_rows_tc_plane_elems(int64_t B, int64_t C, int64_t N);
int dist_rows_tc_prepare(const KnnArgs& a, __nv_bfloat16* planes, cudaStream_t stream);
int dist_rows_tc_launch(const KnnArgs& a, const __nv_bfloat16* planes, int b0, int nb, float* drows, int ldd,
                        cudaStream_t stream);

__global__ void to_node_major_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N,
                                     float* __restrict__ xt);

// ---- launch helpers for the selection kernels -------------------------------------
// Clouds per slab of distance rows: two slabs are in flight (rows of slab s+1 under the select of slab s), so each
// gets half of the L2 (at least one cloud).
static size_t knn_slab_clouds(int64_t B, int64_t N) {
  const int64_t ldd = (N + 3) / 4 * 4;
  const int64_t per_cloud = N * ldd * 4;
  int64_t nb = static_cast<int64_t>(device_l2_bytes() / 2) / (per_cloud > 0 ? per_cloud : 1);
  if (nb < 1) nb = 1;
  if (nb > B) nb = B;
  return static_cast<size_t>(nb);
}

constexpr int TC_FALLBACK_GRID = 132;  // CTAs of the exact completion kernel (one uncertified query at a time each; H100 SXM SMs)

static bool tc_shape_ok(int64_t C, int64_t N, int64_t K) {
  return K <= TC_K_MAX && C <= TC_MAX_C && N >= TILE && (N % TILE) == 0;
}

size_t knn_workspace_bytes(int64_t B, int64_t C, int64_t N, int64_t K) {
  size_t bytes = align_up(static_cast<size_t>(B) * N * 4, 256);
  if (tc_shape_ok(C, N, K)) {
    const int64_t cpad = (C + 15) / 16 * 16;
    bytes += align_up(static_cast<size_t>(B) * TC_PLANES * cpad * N * 2, 256);   // bf16 planes
    bytes += align_up(static_cast<size_t>(B) * N * C * 4, 256);          // node-major copy
    bytes += align_up(static_cast<size_t>(B) * 4, 256);                  // per-cloud max |x|^2
    bytes += align_up(static_cast<size_t>(B) * 8 * N * 2, 256);          // -|x|^2/2 operand block
    bytes += align_up(static_cast<size_t>(B) * N * 4 + 256, 256);        // fail counter + list
  }
  if (K > SMALL_K_MAX) {
    const int64_t ldd = (N + 3) / 4 * 4;
    const size_t nslab = static_cast<size_t>(B) > knn_slab_clouds(B, N) ? 2 : 1;   // two slabs: distance rows of slab s+1 overlap the select of slab s
    bytes += nslab * align_up(knn_slab_clouds(B, N) * N * ldd * 4, 256);
    bytes += nslab * align_up(knn_slab_clouds(B, N) * N * 4 + 256, 256);   // rows the sampled select hands to the exact kernel (one list per slab buffer)
    if (C <= TC_MAX_C && N >= TILE && N % TILE == 0) bytes += align_up(dist_rows_tc_plane_elems(B, C, N) * 2, 256);   // (hi, mid, lo) planes
  }
  return bytes + 256;
}

// Side stream of the large-K slab pipeline, one per device, created on first use (a write-once cache: the stream
// carries no state between calls - every call forks it from and joins it back into the caller's stream by events).
static cudaStream_t slab_side_stream() {
  static std::atomic<cudaStream_t> cached[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  cudaStream_t s = cached[dev].load(std::memory_order_acquire);
  if (!s) {
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    cudaStream_t expected = nullptr;
    if (!cached[dev].compare_exchange_strong(expected, s, std::memory_order_acq_rel)) {
      cudaStreamDestroy(s);
      s = expected;
    }
  }
  return s;
}

static int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// cuTensorMapEncodeTiled through the runtime (no link against libcuda): resolved once, the pointer is a
// write-once cache of a driver symbol.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tensor_map_encoder() {
  static std::atomic<void*> cached{nullptr};
  void* fn = cached.load(std::memory_order_acquire);
  if (!fn) {
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    cached.store(fn, std::memory_order_release);
  }
  return reinterpret_cast<EncodeTiledFn>(fn);
}
// bf16 matrix (rows, cols) row-major -> tensor map with boxes of 64 columns (128 bytes) x box_rows rows, SWIZZLE_128B:
// a box lands in shared memory as box_rows x 128 B rows with the 16-byte chunks XOR-swizzled by (row & 7), which is
// the canonical MN-major wgmma layout of one 64-wide MN block.
static int make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int box_rows) {
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enc) return DGCN_ERR_UNSUPPORTED;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * 2};
  const cuuint32_t box[2] = {64u, static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1u, 1u};
  const CUresult rc = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return rc == CUDA_SUCCESS ? DGCN_OK : DGCN_ERR_CUDA;
}

// Tensor-core pre-filter path (knn_tc.cuh).  xt: node-major copy of x if the caller has one.
static int launch_knn_tc(KnnArgs& a, Workspace& ws, cudaStream_t stream, const float* xt, int64_t* n_partial,
                         const ProloguePq* pqf) {
  const int B = a.B, N = a.N, C = a.C, K = a.K;
  const int cpad = (C + 15) / 16 * 16;
  __nv_bfloat16* planes = ws.take<__nv_bfloat16>(static_cast<size_t>(B) * TC_PLANES * cpad * N);
  float* xt_own = xt ? nullptr : ws.take<float>(static_cast<size_t>(B) * N * C);
  float* sqmax = ws.take<float>(static_cast<size_t>(B));
  __nv_bfloat16* sqp = ws.take<__nv_bfloat16>(static_cast<size_t>(B) * 8 * N);
  int* fail = ws.take<int>(static_cast<size_t>(B) * N + 64);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  DGCN_CUDA_TRY(cudaMemsetAsync(fail, 0, 256, stream));
  DGCN_CUDA_TRY(cudaMemsetAsync(sqmax, 0, static_cast<size_t>(B) * 4, stream));
  // sq, bf16 planes, node-major copy and max |x|^2 in one pass over x (sq overwrites what the caller computed)
  if (pqf) {   // the EdgeConv node GEMM rides on the same pass over x
    const size_t smem = (static_cast<size_t>(TC_MAX_C) * 68 + static_cast<size_t>(C) * pqf->M) * 4;
    DGCN_ENSURE_SMEM((tc_prologue_pq_kernel), smem);
    tc_prologue_pq_kernel<<<dim3(N / 64, B), 256, smem, stream>>>(a.x, a.sb, a.sc, C, cpad, N, const_cast<float*>(a.sq),
                                                                  planes, xt ? nullptr : xt_own, sqmax, sqp, *pqf);
  } else {
    tc_prologue_kernel<<<dim3(ceil_div(N, 32), B), 256, 0, stream>>>(a.x, a.sb, a.sc, C, cpad, N,
                                                                 const_cast<float*>(a.sq), planes,
                                                                 xt ? nullptr : xt_own, sqmax, sqp);
  }
  DGCN_LAUNCH_CHECK();
  if (!xt) xt = xt_own;
  TcArgs t{};
  {
    int rc = make_plane_map(&t.tm_planes, planes, static_cast<int64_t>(B) * TC_PLANES * cpad, N, cpad);
    if (rc == DGCN_OK) rc = make_plane_map(&t.tm_sqp, sqp, static_cast<int64_t>(B) * 8, N, 8);
    if (rc != DGCN_OK) return rc;
  }
  t.a = a;
  t.planes = planes;
  t.sqp = sqp;
  t.xt = xt;
  t.xt32 = (reinterpret_cast<uintptr_t>(xt) & 31) == 0 ? 1 : 0;
  t.sqmax = sqmax;
  t.Cpad = cpad;
  t.fail_count = fail;
  t.fail_list = fail + 64;
  const dim3 grid(N / TILE, B);
  const int64_t n_cta = static_cast<int64_t>(grid.x) * grid.y;
  {
    KernelTimer timer(stream, "knn");
    const int nch = a.epi.mode == EPI_MR ? a.epi.c_in : a.epi.c_out;
    t.wide = epilogue_wide_ok(a) ? 1 : 0;
    t.flush_early = TC_FLUSH_EARLY;
    t.flush_late = TC_FLUSH_LATE;
    // list length = K + certification margin
    // (a margin of 4 ranks leaves ~1e-5 of the queries of a random 64-d cloud uncertified, 8 ranks none)
    const int kp = K <= 9 ? 16 : K <= 20 ? 28 : K <= 32 ? 40 : 56;
    t.work_bytes = static_cast<int>(tc_work_bytes(kp, a.k, t.wide != 0, nch));
    const size_t smem = static_cast<size_t>(t.work_bytes) + sizeof(TcTail) + 1024;
    const bool packed = N <= 4096;
    // T4_GROUPS query tiles per CTA, warp specialised (knn_tc4.cuh), where its smaller work area and fixed consumer fit
    const bool train = a.epi.mode == EPI_EDGE && a.epi.norm == DGCN_NORM_BATCH_TRAIN;
    const bool quad = !a.tc_tile_per_cta && packed && t.wide && !train && t.xt32 && (C & 7) == 0 && knn_tc4_list_ok(kp, a.k);
    int rc;
    if (quad) {
      rc = launch_knn_tc4(kp, t, dim3(static_cast<unsigned>(ceil_div(N / TILE, T4_GROUPS)), B), stream);
    } else
    switch (kp) {
      case 16: rc = launch_knn_tc_kp16(packed, t, grid, smem, stream); break;
      case 28: rc = launch_knn_tc_kp28(packed, t, grid, smem, stream); break;
      case 40: rc = launch_knn_tc_kp40(packed, t, grid, smem, stream); break;
      default: rc = launch_knn_tc_kp56(packed, t, grid, smem, stream); break;
    }
    if (rc != DGCN_OK) return rc;
    DGCN_LAUNCH_CHECK();
    float* extra = a.epi.partial ? a.epi.partial + n_cta * 2 * a.epi.c_out : nullptr;
    knn_exact_rows_kernel<<<TC_FALLBACK_GRID, 256, 0, stream>>>(a, t.fail_count, t.fail_list, extra);
    DGCN_LAUNCH_CHECK();
    if (debug_certification_on()) {
      int failed = 0;
      DGCN_CUDA_TRY(cudaMemcpyAsync(&failed, t.fail_count, sizeof(int), cudaMemcpyDeviceToHost, stream));
      DGCN_CUDA_TRY(cudaStreamSynchronize(stream));
      debug_certification_add(failed, static_cast<int64_t>(B) * N);
    }
  }
  if (n_partial) *n_partial = n_cta + TC_FALLBACK_GRID;
  return DGCN_OK;
}

// Runs the selection (+ fused consumer described by a.epi) on `stream`.
// n_partial (optional out): number of train-mode statistic rows the chosen path wrote.
// true when launch_knn will take the tensor-core path for these arguments
static bool knn_takes_tc(const KnnArgs& a) {
  const bool train_wide = a.epi.mode == EPI_EDGE && a.epi.norm == DGCN_NORM_BATCH_TRAIN && a.epi.c_out > 128;
  return !a.exact_fp32 && tc_shape_ok(a.C, a.N, a.K) && a.k <= SEL_LD && !train_wide;
}
// the fused prologue can also produce PQ (EdgeConv): channel / output counts it supports
static bool prologue_pq_ok(const KnnArgs& a, int64_t M) {
  return knn_takes_tc(a) && M % 128 == 0 && M <= 256 && a.C <= TC_MAX_C;
}

// pqf (optional): produce the EdgeConv node GEMM inside the tensor-core prologue; the caller must have
// checked prologue_pq_ok and skipped node_pq_kernel.
int launch_knn(KnnArgs& a, Workspace& ws, cudaStream_t stream, int64_t* n_partial = nullptr,
               const ProloguePq* pqf = nullptr) {
  const int B = a.B, N = a.N, K = a.K;
  float* sq = ws.take<float>(static_cast<size_t>(B) * N);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  a.sq = sq;
  if (knn_takes_tc(a))
    return launch_knn_tc(a, ws, stream, a.epi.mode == EPI_MR ? a.epi.xt : nullptr, n_partial, pqf);
  if (pqf) return DGCN_ERR_BAD_ARG;   // (internal misuse) nobody would produce PQ
  const bool rows_on_tc = K > 32 && K <= LARGE_K_MAX && dist_rows_tc_ok(a);   // large-K: distance rows on the tensor cores
  __nv_bfloat16* planes3 = nullptr;
  if (rows_on_tc) {
    planes3 = ws.take<__nv_bfloat16>(dist_rows_tc_plane_elems(B, a.C, N));
    if (!ws.ok) return DGCN_ERR_WORKSPACE;
    int rc = dist_rows_tc_prepare(a, planes3, stream);      // sq (same FMA chain as sqnorm_kernel) + the bf16 planes
    if (rc != DGCN_OK) return rc;
  } else {
    sqnorm_kernel<<<dim3(ceil_div(N, 256), B), 256, 0, stream>>>(a.x, a.sb, a.sc, a.C, N, sq);
    DGCN_LAUNCH_CHECK();
  }
  const dim3 grid(ceil_div(N, TILE), B);
  if (n_partial) *n_partial = K <= SMALL_K_MAX ? static_cast<int64_t>(grid.x) * grid.y : static_cast<int64_t>(B) * N;
  if (K <= 32) {
    const size_t smem = sizeof(SmallSmem<1>);
    DGCN_ENSURE_SMEM((knn_small_kernel<1>), smem);
    {
      KernelTimer timer(stream, "knn");
      knn_small_kernel<1><<<grid, NTHREADS, smem, stream>>>(a);
    }
    DGCN_LAUNCH_CHECK();
    return DGCN_OK;
  }
  if (K > LARGE_K_MAX) return DGCN_ERR_UNSUPPORTED;
  const int ldd = (N + 3) / 4 * 4;
  const int nbmax = static_cast<int>(knn_slab_clouds(B, N));
  const size_t slab_elems = static_cast<size_t>(nbmax) * N * ldd;
  float* drows = ws.take<float>(slab_elems);
  float* drows2 = B > nbmax ? ws.take<float>(slab_elems) : nullptr;   // second slab: distance rows run one slab ahead
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  const int KP = next_pow2(K);
  const size_t per_warp = static_cast<size_t>(KP) * 8 + static_cast<size_t>(ldd) * 4 + static_cast<size_t>((a.k + 31) / 32 * 32) * 4;   // ldd = N rounded up to 4 keeps every warp's u64 array 16-byte aligned
  int warps = static_cast<int>((200u << 10) / per_warp);
  if (warps < 1) return DGCN_ERR_UNSUPPORTED;   // a single row does not fit in shared memory
  if (warps > 4) warps = 4;
  const size_t smem = per_warp * warps;
  DGCN_ENSURE_SMEM((select_rows_kernel), smem);
  // sampled fast select: bound = sample_rank-th of 128 samples (mean + 2.5 sigma + 2 of the K/N quantile)
  const double pq = static_cast<double>(K) / N;
  int sample_rank = static_cast<int>(128.0 * pq + 2.5 * sqrt(128.0 * pq * (1.0 - pq)) + 2.0) + 1;
  if (sample_rank > 127) sample_rank = 127;
  // room for every key below the bound (no power of two needed: only the wanted bins get sorted);
  // k > 64 keeps the full sort and needs the padded power of two
  // keys below a bound at sample rank r: mean (r+1)/129 N, relative spread ~ 1/sqrt(r+1); leave 3.5 sigma
  const double wmean = (sample_rank + 1) / 129.0 * N;
  const int64_t wcap = static_cast<int64_t>(wmean * (1.0 + 3.5 / sqrt(sample_rank + 1.0))) + 32;
  int cap = static_cast<int>(wcap > K + 64 ? wcap : K + 64);
  cap = a.k > 64 ? next_pow2(cap > 2 * K ? cap : 2 * K) : (cap + 31) / 32 * 32;
  if (cap < 128) cap = 128;            // the sorted sample lives in the same array
  if (cap > 2048) cap = 2048;
  const bool fast = N >= 512 && cap >= K;
  const size_t per_warp_f = static_cast<size_t>(cap) * 8 + static_cast<size_t>((a.k + 31) / 32 * 32) * 4 + 2560;   // keys, sel, multi-select tables (hist 256, prefix 260 ints, 256 marks -> 2320 B)
  int warps_f = static_cast<int>((56u << 10) / per_warp_f);   // <= 56 KB per CTA: four CTAs per SM
  if (warps_f > 8) warps_f = 8;
  if (warps_f < 1) warps_f = 1;
  const size_t smem_f = per_warp_f * warps_f;
  int* rowlist = nullptr;
  int* rowlist2 = nullptr;
  if (fast) {
    rowlist = ws.take<int>(static_cast<size_t>(nbmax) * N + 64);
    if (drows2) rowlist2 = ws.take<int>(static_cast<size_t>(nbmax) * N + 64);
    if (!ws.ok) return DGCN_ERR_WORKSPACE;
    DGCN_ENSURE_SMEM((select_rows_fast_kernel), smem_f);
  }
  KernelTimer timer(stream, "knn");
  // Two-chain slab pipeline: even slabs run (distance rows -> sampled select -> exact completion) on the caller's
  // stream, odd slabs on a side stream with their own row buffer and completion list.  The chains overlap freely:
  // the tensor-core distance rows of one slab run under the instruction-bound select of the other, and - what pays
  // most - the partial last wave of one select (4096 rows are 1.15 .. 2.3 waves of its CTAs) is filled by the CTAs
  // of the other chain.  An event forks the side stream from the caller's stream and one joins it back, so the call
  // is still one stream-ordered operation for the caller (and capturable in a CUDA graph).
  cudaStream_t side = drows2 ? slab_side_stream() : nullptr;
  cudaEvent_t ev_start = nullptr, ev_join = nullptr;
  if (side) {
    if (cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming) != cudaSuccess)
      side = nullptr;
  }
  struct EventGuard {   // destroying an event that is still in flight is legal: it is released on completion
    cudaEvent_t* e[2];
    ~EventGuard() { for (cudaEvent_t* p : e) if (p && *p) cudaEventDestroy(*p); }
  } guard{{&ev_start, &ev_join}};
  if (side) {
    DGCN_CUDA_TRY(cudaEventRecord(ev_start, stream));
    DGCN_CUDA_TRY(cudaStreamWaitEvent(side, ev_start, 0));
  }
  int slab = 0;
  for (int b0 = 0; b0 < B; b0 += nbmax, ++slab) {
    const int nb = (B - b0 < nbmax) ? (B - b0) : nbmax;
    const int buf = side ? (slab & 1) : 0;
    cudaStream_t st = buf ? side : stream;             // a buffer is only ever touched by its own chain: stream order
    float* drows_s = buf ? drows2 : drows;
    int* rowlist_s = buf ? rowlist2 : rowlist;
    if (rows_on_tc) {
      int rc = dist_rows_tc_launch(a, planes3, b0, nb, drows_s, ldd, st);
      if (rc != DGCN_OK) return rc;
    } else {
      dist_rows_kernel<<<dim3(ceil_div(N, TILE), ceil_div(N, TILE), nb), NTHREADS, 0, st>>>(a, b0, drows_s, ldd);
      DGCN_LAUNCH_CHECK();
    }
    const int64_t rows = static_cast<int64_t>(nb) * N;
    if (fast) {
      DGCN_CUDA_TRY(cudaMemsetAsync(rowlist_s, 0, 256, st));
      select_rows_fast_kernel<<<static_cast<unsigned>(ceil_div(rows, warps_f)), warps_f * 32, smem_f, st>>>(
          a, b0, nb, drows_s, ldd, cap, sample_rank, warps_f, rowlist_s, rowlist_s + 64);
      DGCN_LAUNCH_CHECK();
      select_rows_kernel<<<2 * device_sm_count(), warps * 32, smem, st>>>(a, b0, nb, drows_s, ldd, KP, ldd, warps, rowlist_s + 64,
                                                                      rowlist_s);   // grid-stride over the handed-over rows
      DGCN_LAUNCH_CHECK();
    } else {
      select_rows_kernel<<<static_cast<unsigned>(ceil_div(rows, warps)), warps * 32, smem, st>>>(
          a, b0, nb, drows_s, ldd, KP, ldd, warps, nullptr, nullptr);
      DGCN_LAUNCH_CHECK();
    }
  }
  if (side) {
    DGCN_CUDA_TRY(cudaEventRecord(ev_join, side));
    DGCN_CUDA_TRY(cudaStreamWaitEvent(stream, ev_join, 0));
  }
  return DGCN_OK;
}

int fill_knn_args(KnnArgs& a, const float* x, int64_t B, int64_t C, int64_t N, int64_t stride_b,
                  int64_t stride_c, const dgcn_dilation* dil, int exclude_self) {
  if (!x || !dil || B <= 0 || C <= 0 || N <= 0 || dil->k <= 0 || dil->dilation <= 0) return DGCN_ERR_BAD_ARG;
  if (B > 65535 || N > (1 << 30) || C > (1 << 20)) return DGCN_ERR_UNSUPPORTED;
  const int64_t K = dil->k * dil->dilation;
  if (K > N - (exclude_self ? 1 : 0)) return DGCN_ERR_BAD_ARG;   // torch.topk: k out of range
  if (dil->cols_host && dil->k > MAX_KEEP) return DGCN_ERR_UNSUPPORTED;
  a.x = x; a.sb = stride_b; a.sc = stride_c;
  a.B = static_cast<int>(B); a.C = static_cast<int>(C); a.N = static_cast<int>(N);
  a.vec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0 && stride_b % 4 == 0 && stride_c % 4 == 0 && N % 4 == 0) ? 1 : 0;
  a.sq = nullptr;
  a.K = static_cast<int>(K); a.k = static_cast<int>(dil->k); a.dilation = static_cast<int>(dil->dilation);
  a.exclude_self = exclude_self ? 1 : 0;
  a.exact_fp32 = (dil->flags & DGCN_KNN_EXACT_FP32) ? 1 : 0;
  a.tc_tile_per_cta = (dil->flags & DGCN_KNN_TC_TILE_PER_CTA) ? 1 : 0;
  a.has_cols = dil->cols_host ? 1 : 0;
  for (int l = 0; l < MAX_KEEP; ++l) a.cols[l] = 0;
  if (dil->cols_host) {
    for (int l = 0; l < a.k; ++l) {
      int c = dil->cols_host[l];
      if (c < 0 || c >= K) return DGCN_ERR_BAD_ARG;
      a.cols[l] = c;
    }
  }
  a.epi = Epilogue{};
  a.epi.mode = EPI_INDEX;
  return DGCN_OK;
}

// ---- node-level kernels ---------------------------------------------------------------
// EdgeConv weight split (SURVEY.md 7): W.[x_i ; x_j - x_i] = (W1 - W2) x_i + W2 x_j.
// wk[c][m] (k-major, m < 2*co): m < co -> W1[m][c] - W2[m][c]; else W2[m-co][c].  bk = (bias | 0).
__global__ void pack_edge_weights_kernel(const float* __restrict__ w, const float* __restrict__ bias,
                                         int ci, int co, float* __restrict__ wk, float* __restrict__ bk) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ci * 2 * co) {
    int c = i / (2 * co), m = i % (2 * co);
    float v;
    if (m < co) v = w[m * 2 * ci + c] - w[m * 2 * ci + ci + c];
    else v = w[(m - co) * 2 * ci + ci + c];
    wk[i] = v;
  }
  if (i < 2 * co) bk[i] = (i < co && bias) ? bias[i] : 0.f;
}
// MRConv weight transpose: wk[kk][m] = W[m][kk], kk < 2*ci
__global__ void pack_mr_weights_kernel(const float* __restrict__ w, int ci2, int co, float* __restrict__ wk) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ci2 * co) {
    int kk = i / co, m = i % co;
    wk[i] = w[m * ci2 + kk];
  }
}

// (B,C,N) strided -> (B,N,C) contiguous
__global__ void to_node_major_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N,
                                     float* __restrict__ xt) {
  __shared__ float t[32][33];
  const int b = blockIdx.z, n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int c = c0 + r, n = n0 + threadIdx.x;
    t[r][threadIdx.x] = (c < C && n < N) ? __ldg(x + b * sb + c * sc + n) : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int n = n0 + r, c = c0 + threadIdx.x;
    if (n < N && c < C) xt[(static_cast<int64_t>(b) * N + n) * C + c] = t[threadIdx.x][r];
  }
}

// PQ[b][n][m] = sum_c X[b][c][n] * wk[c][m] + bk[m]      (rows = points, cols = m)
__global__ void __launch_bounds__(NTHREADS, 2)
    node_pq_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N, int vec,
                   const float* __restrict__ wk, const float* __restrict__ bk, int M,
                   float* __restrict__ pq) {
  __shared__ TileSmem ts;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, n0 = blockIdx.y * TILE, m0 = blockIdx.x * TILE;
  KMajor A = kmajor1(x + b * sb, sc, C, N, vec != 0);
  KMajor Bm = kmajor1(wk, M, C, M, (M % 4) == 0);
  float acc[8][8];
  tile_product(ts, A, n0, Bm, m0, acc);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int n = n0 + tile_row(ty, i);
    if (n >= N) continue;
    float* row = pq + (static_cast<int64_t>(b) * N + n) * M;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int m = m0 + tile_col(tx, j);
      if (m < M) row[m] = acc[i][j] + __ldg(bk + m);
    }
  }
}

// MRConv node update: out[b][m][n] = norm(act(sum_kk wk[kk][m] * [x ; r][kk][n] + bias[m]))
// rows = m, cols = points.  Train mode stores act() and per-CTA partial statistics.
struct MrNodeArgs {
  const float* x; int64_t sb, sc; const float* r; int ci, N, vec;
  const float* wk; const float* bias; int co;
  float slope; const float* prelu;
  int norm; const float* bn_w; const float* bn_b; const float* bn_m; const float* bn_v; float bn_eps;
  float* out; float* partial;
  const float* res; int64_t res_sb, res_sc; float res_scale; int64_t out_sb;   // block fusion (eval / no norm)
};
__global__ void __launch_bounds__(NTHREADS, 2) mr_node_kernel(const MrNodeArgs g) {
  __shared__ TileSmem ts;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, m0 = blockIdx.y * TILE, n0 = blockIdx.x * TILE;
  KMajor A = kmajor1(g.wk, g.co, 2 * g.ci, g.co, (g.co % 4) == 0);
  KMajor Bm = kmajor2(g.x + b * g.sb, g.sc, g.ci, g.r + static_cast<int64_t>(b) * g.ci * g.N, g.N, 2 * g.ci,
                      g.N, g.vec != 0);
  float acc[8][8];
  tile_product(ts, A, m0, Bm, n0, acc);
  const float slope = g.prelu ? __ldg(g.prelu) : g.slope;
  const bool train = g.norm == DGCN_NORM_BATCH_TRAIN;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + tile_row(ty, i);
    float s = 1.f, t = 0.f, bias = 0.f;
    if (m < g.co) {
      bias = g.bias ? __ldg(g.bias + m) : 0.f;
      if (g.norm == DGCN_NORM_BATCH_EVAL) {
        float inv = 1.0f / sqrtf(__ldg(g.bn_v + m) + g.bn_eps);
        s = (g.bn_w ? __ldg(g.bn_w + m) : 1.f) * inv;
        t = (g.bn_b ? __ldg(g.bn_b + m) : 0.f) - __ldg(g.bn_m + m) * s;
      }
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + tile_col(tx, j);
      float a = act_apply(acc[i][j] + bias, slope);
      if (m < g.co && n < g.N) {
        float v = fmaf(s, a, t);
        if (g.res) v = __fadd_rn(v, __fmul_rn(__ldg(g.res + b * g.res_sb + m * g.res_sc + n), g.res_scale));
        g.out[b * g.out_sb + static_cast<int64_t>(m) * g.N + n] = v;
        s1 += a;
        s2 += a * a;
      }
    }
    if (train) {   // reduce over the 16 tx lanes that share this row (lanes differ in low 4 bits)
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      }
      if (tx == 0 && m < g.co) {
        const int64_t slot = static_cast<int64_t>(b) * gridDim.x + blockIdx.x;
        g.partial[(slot * 2 + 0) * g.co + m] = s1;
        g.partial[(slot * 2 + 1) * g.co + m] = s2;
      }
    }
  }
}

// Batch statistics from partial sums (fixed order, fp64) -> (scale, shift) and the
// batch mean / biased variance the host needs for the running-stat update
// (torch BatchNorm2d training semantics: normalise with biased variance).
__global__ void bn_finalize_kernel(const float* __restrict__ partial, int64_t np, int C, double count,
                                   const float* __restrict__ bn_w, const float* __restrict__ bn_b, float eps,
                                   float* __restrict__ st, float* __restrict__ mean_out,
                                   float* __restrict__ var_out) {
  __shared__ double r1[256], r2[256];
  const int c = blockIdx.x;
  double a1 = 0.0, a2 = 0.0;
  for (int64_t i = threadIdx.x; i < np; i += blockDim.x) {
    a1 += static_cast<double>(partial[(i * 2 + 0) * C + c]);
    a2 += static_cast<double>(partial[(i * 2 + 1) * C + c]);
  }
  r1[threadIdx.x] = a1;
  r2[threadIdx.x] = a2;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      r1[threadIdx.x] += r1[threadIdx.x + o];
      r2[threadIdx.x] += r2[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double mean = r1[0] / count;
    double var = r2[0] / count - mean * mean;
    if (var < 0.0) var = 0.0;
    float inv = 1.0f / sqrtf(static_cast<float>(var) + eps);
    float s = (bn_w ? bn_w[c] : 1.f) * inv;
    st[c] = s;
    st[C + c] = (bn_b ? bn_b[c] : 0.f) - static_cast<float>(mean) * s;
    if (mean_out) mean_out[c] = static_cast<float>(mean);
    if (var_out) var_out[c] = static_cast<float>(var);
  }
}
// out = s >= 0 ? s*out + t : s*out_min + t   (out_min may be null: plain affine)
__global__ void bn_apply_kernel(float* __restrict__ out, const float* __restrict__ out_min,
                                const float* __restrict__ st, int C, int N, int64_t total) {
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int c = static_cast<int>((i / N) % C);
  float s = st[c], t = st[C + c];
  float v = (s >= 0.f || out_min == nullptr) ? out[i] : out_min[i];
  out[i] = fmaf(s, v, t);
}

// ---- static graph: gather / max over a given edge list -----------------------------
struct GatherArgs {
  Epilogue e;
  const int64_t* edge_index;   // (2,B,N,k) or null
  const int32_t* nbr;          // (B,N,k)   or null
  int B, N, k;
};
__global__ void __launch_bounds__(256) graph_gather_kernel(const GatherArgs g) {
  __shared__ float smax[32][33];
  __shared__ float smin[32][33];
  __shared__ float red[8][2][32];
  const Epilogue& e = g.e;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y, i0 = blockIdx.x * 32;
  const int N = g.N, k = g.k;
  const int64_t node0 = static_cast<int64_t>(b) * N;
  const bool edge = e.mode == EPI_EDGE;
  const bool train = edge && e.norm == DGCN_NORM_BATCH_TRAIN;
  const int nch = edge ? e.c_out : e.c_in;
  const float slope = edge ? epi_slope(e) : 0.f;
  const int64_t plane = static_cast<int64_t>(g.B) * N * k;
  for (int c0 = 0; c0 < nch; c0 += 32) {
    const int c = c0 + lane;
    float s1 = 0.f, s2 = 0.f, bs = 1.f, bt = 0.f;
    if (edge) bn_affine(e, c, bs, bt);
    for (int u = 0; u < 4; ++u) {
      const int il = warp * 4 + u, i = i0 + il;
      if (i >= N) continue;
      float vmax = -INFINITY, vmin = INFINITY;
      if (c < nch) {
        for (int l = 0; l < k; ++l) {
          const int64_t o = (node0 + i) * k + l;
          int64_t j, ic;
          if (g.edge_index) {
            j = g.edge_index[o];
            ic = g.edge_index[plane + o];
          } else {
            j = g.nbr[o];
            ic = i;
          }
          j = j < 0 ? 0 : (j >= N ? N - 1 : j);
          ic = ic < 0 ? 0 : (ic >= N ? N - 1 : ic);
          float a;
          if (edge) {
            const int ld = 2 * e.c_out;
            a = act_apply(__ldg(e.pq + (node0 + ic) * ld + c) + __ldg(e.pq + (node0 + j) * ld + e.c_out + c), slope);
            s1 += a;
            s2 += a * a;
          } else {
            a = __ldg(e.xt + (node0 + j) * e.c_in + c) - __ldg(e.xt + (node0 + ic) * e.c_in + c);
          }
          vmax = fmaxf(vmax, a);
          vmin = fminf(vmin, a);
        }
      }
      if (train || !edge) {
        smax[lane][il] = vmax;
        smin[lane][il] = vmin;
      } else {
        smax[lane][il] = bs >= 0.f ? fmaf(bs, vmax, bt) : fmaf(bs, vmin, bt);
      }
    }
    if (train) {
      red[warp][0][lane] = s1;
      red[warp][1][lane] = s2;
    }
    __syncthreads();
    float* dst = edge ? e.out : e.r_out;
    for (int t = tid; t < 32 * 32; t += 256) {
      const int cc = t >> 5, il = t & 31;
      if (c0 + cc < nch && i0 + il < N) {
        int64_t o = (static_cast<int64_t>(b) * nch + c0 + cc) * N + i0 + il;
        dst[o] = smax[cc][il];
        if (train) e.out_min[o] = smin[cc][il];
      }
    }
    if (train && tid < 64) {
      const int which = tid >> 5, cc = tid & 31;
      float s = 0.f;
      for (int w = 0; w < 8; ++w) s += red[w][which][cc];
      const int64_t cta = static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x;
      if (c0 + cc < nch) e.partial[(cta * 2 + which) * nch + c0 + cc] = s;
    }
    __syncthreads();
  }
}

// ---- planning -----------------------------------------------------------------------------
struct ConvPlan {
  size_t wk, bk, pq, xt, r, out_min, partial, st;   // element counts (floats)
  int64_t n_partial;
};
static ConvPlan conv_plan(int conv, int64_t B, int64_t ci, int64_t co, int64_t N, int64_t K, bool fused) {
  ConvPlan p{};
  p.st = 2 * co;
  if (conv == DGCN_CONV_EDGE) {
    p.wk = ci * 2 * co;
    p.bk = 2 * co;
    p.pq = B * N * 2 * co;
    p.out_min = B * co * N;
    int64_t tiles = fused ? (K <= SMALL_K_MAX ? ceil_div(N, TILE) * B + TC_FALLBACK_GRID : B * N) : ceil_div(N, 32) * B;
    p.n_partial = tiles;
    p.partial = tiles * 2 * co;
  } else {
    p.wk = 2 * ci * co;
    p.xt = B * N * ci;
    p.r = B * ci * N;
    p.n_partial = B * ceil_div(N, TILE);
    p.partial = p.n_partial * 2 * co;
  }
  return p;
}
static size_t conv_plan_bytes(const ConvPlan& p) {
  size_t b = 0;
  for (size_t v : {p.wk, p.bk, p.pq, p.xt, p.r, p.out_min, p.partial, p.st}) b += align_up(v * 4, 256);
  return b + 256;
}

static int check_conv_args(int conv, const float* x, int64_t B, int64_t ci, int64_t N, const dgcn_basic_conv* p,
                           int64_t co, const float* out) {
  if (conv != DGCN_CONV_EDGE && conv != DGCN_CONV_MR) return DGCN_ERR_UNSUPPORTED;
  if (!x || !p || !p->weight || !out || B <= 0 || ci <= 0 || co <= 0 || N <= 0) return DGCN_ERR_BAD_ARG;
  if (p->act < DGCN_ACT_NONE || p->act > DGCN_ACT_PRELU) return DGCN_ERR_UNSUPPORTED;
  if (p->act == DGCN_ACT_PRELU && !p->prelu_weight) return DGCN_ERR_BAD_ARG;
  if (p->norm < DGCN_NORM_NONE || p->norm > DGCN_NORM_BATCH_TRAIN) return DGCN_ERR_UNSUPPORTED;
  if (p->norm == DGCN_NORM_BATCH_EVAL && (!p->bn_mean || !p->bn_var)) return DGCN_ERR_BAD_ARG;
  if (B > 65535) return DGCN_ERR_UNSUPPORTED;
  return DGCN_OK;
}

float act_slope_of(const dgcn_basic_conv* p) {
  switch (p->act) {
    case DGCN_ACT_RELU: return 0.f;
    case DGCN_ACT_LEAKYRELU: return p->slope;
    case DGCN_ACT_PRELU: return 0.f;   // read from prelu_weight on device
    default: return 1.f;
  }
}

// Shared body of graph_conv_forward (graph given) and dyn_conv_forward (graph fused).
static int conv_forward(int conv, const float* x, int64_t B, int64_t ci, int64_t N, int64_t sb, int64_t sc,
                        const int64_t* edge_index, const int32_t* nbr, int64_t k, const dgcn_dilation* dil,
                        const dgcn_basic_conv* p, int64_t co, float* out, int32_t* nbr_out, Workspace& ws,
                        cudaStream_t stream, const dgcn_block_fusion* fus = nullptr) {
  const bool fused = dil != nullptr;
  if (fus) {   // block epilogue: out = conv + residual * scale, out possibly a channel slice of a wider buffer
    if (!fused || p->norm == DGCN_NORM_BATCH_TRAIN) return DGCN_ERR_UNSUPPORTED;
    if (fus->out_stride_b != 0 && fus->out_stride_b < co * N) return DGCN_ERR_BAD_ARG;
  }
  const int64_t K = fused ? dil->k * dil->dilation : k;
  const int64_t keep = fused ? dil->k : k;
  ConvPlan pl = conv_plan(conv, B, ci, co, N, K, fused);
  const bool train = p->norm == DGCN_NORM_BATCH_TRAIN;
  const int vec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0 && sb % 4 == 0 && sc % 4 == 0 && N % 4 == 0) ? 1 : 0;

  Epilogue e{};
  e.nbr = nbr_out;
  e.slope = act_slope_of(p);
  e.prelu = p->act == DGCN_ACT_PRELU ? p->prelu_weight : nullptr;
  e.norm = p->norm;
  e.bn_w = p->bn_weight; e.bn_b = p->bn_bias; e.bn_m = p->bn_mean; e.bn_v = p->bn_var; e.bn_eps = p->bn_eps;
  e.c_out = static_cast<int>(co);
  e.c_in = static_cast<int>(ci);
  e.out_sb = (fus && fus->out_stride_b) ? fus->out_stride_b : co * N;
  if (fus && fus->residual && conv == DGCN_CONV_EDGE) {   // (MRConv adds it in its node kernel)
    e.res = fus->residual; e.res_sb = fus->res_stride_b; e.res_sc = fus->res_stride_c; e.res_scale = fus->res_scale;
  }
  float* wk = ws.take<float>(pl.wk);
  float* st = ws.take<float>(pl.st);
  float* partial = train ? ws.take<float>(pl.partial) : nullptr;
  if (!ws.ok) return DGCN_ERR_WORKSPACE;

  if (conv == DGCN_CONV_EDGE) {
    float* bk = ws.take<float>(pl.bk);
    float* pq = ws.take<float>(pl.pq);
    float* out_min = train ? ws.take<float>(pl.out_min) : nullptr;
    if (!ws.ok) return DGCN_ERR_WORKSPACE;
    const int M = static_cast<int>(2 * co);
    pack_edge_weights_kernel<<<static_cast<unsigned>(ceil_div(ci * M > M ? ci * M : M, 256)), 256, 0, stream>>>(
        p->weight, p->bias, static_cast<int>(ci), static_cast<int>(co), wk, bk);
    DGCN_LAUNCH_CHECK();
    e.mode = EPI_EDGE;
    e.pq = pq;
    e.out = out;
    e.out_min = out_min;
    e.partial = partial;
    KnnArgs a;
    bool pq_in_prologue = false;
    if (fused) {
      int rc = fill_knn_args(a, x, B, ci, N, sb, sc, dil, 0);
      if (rc != DGCN_OK) return rc;
      a.epi = e;
      pq_in_prologue = prologue_pq_ok(a, M);   // the tensor-core prologue computes PQ on its pass over x
    }
    if (!pq_in_prologue) {
      node_pq_kernel<<<dim3(ceil_div(M, TILE), ceil_div(N, TILE), B), NTHREADS, 0, stream>>>(
          x, sb, sc, static_cast<int>(ci), static_cast<int>(N), vec, wk, bk, M, pq);
      DGCN_LAUNCH_CHECK();
    }
    if (fused) {
      const ProloguePq pqf{wk, bk, pq, static_cast<int>(M)};
      int rc = launch_knn(a, ws, stream, &pl.n_partial, pq_in_prologue ? &pqf : nullptr);
      if (rc != DGCN_OK) return rc;
    } else {
      GatherArgs g{e, edge_index, nbr, static_cast<int>(B), static_cast<int>(N), static_cast<int>(k)};
      graph_gather_kernel<<<dim3(ceil_div(N, 32), B), 256, 0, stream>>>(g);
      DGCN_LAUNCH_CHECK();
    }
    if (train) {
      bn_finalize_kernel<<<static_cast<unsigned>(co), 256, 0, stream>>>(
          partial, pl.n_partial, static_cast<int>(co), static_cast<double>(B) * N * keep, p->bn_weight, p->bn_bias,
          p->bn_eps, st, p->batch_mean_out, p->batch_var_out);
      DGCN_LAUNCH_CHECK();
      const int64_t total = B * co * N;
      bn_apply_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(
          out, out_min, st, static_cast<int>(co), static_cast<int>(N), total);
      DGCN_LAUNCH_CHECK();
    }
    return DGCN_OK;
  }

  // MRConv: r = max_j x_j - x_i (gather on a node-major copy), then the node update GEMM
  float* xt = ws.take<float>(pl.xt);
  float* r = ws.take<float>(pl.r);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  pack_mr_weights_kernel<<<static_cast<unsigned>(ceil_div(2 * ci * co, 256)), 256, 0, stream>>>(
      p->weight, static_cast<int>(2 * ci), static_cast<int>(co), wk);
  DGCN_LAUNCH_CHECK();
  to_node_major_kernel<<<dim3(ceil_div(N, 32), ceil_div(ci, 32), B), dim3(32, 8), 0, stream>>>(
      x, sb, sc, static_cast<int>(ci), static_cast<int>(N), xt);
  DGCN_LAUNCH_CHECK();
  e.mode = EPI_MR;
  e.xt = xt;
  e.r_out = r;
  if (fused) {
    KnnArgs a;
    int rc = fill_knn_args(a, x, B, ci, N, sb, sc, dil, 0);
    if (rc != DGCN_OK) return rc;
    a.epi = e;
    rc = launch_knn(a, ws, stream);
    if (rc != DGCN_OK) return rc;
  } else {
    GatherArgs g{e, edge_index, nbr, static_cast<int>(B), static_cast<int>(N), static_cast<int>(k)};
    graph_gather_kernel<<<dim3(ceil_div(N, 32), B), 256, 0, stream>>>(g);
    DGCN_LAUNCH_CHECK();
  }
  MrNodeArgs m{};
  m.x = x; m.sb = sb; m.sc = sc; m.r = r; m.ci = static_cast<int>(ci); m.N = static_cast<int>(N); m.vec = vec;
  m.wk = wk; m.bias = p->bias; m.co = static_cast<int>(co);
  m.slope = e.slope; m.prelu = e.prelu;
  m.norm = p->norm; m.bn_w = p->bn_weight; m.bn_b = p->bn_bias; m.bn_m = p->bn_mean; m.bn_v = p->bn_var;
  m.bn_eps = p->bn_eps;
  m.out = out; m.partial = partial;
  m.out_sb = e.out_sb;
  if (fus && fus->residual) {
    m.res = fus->residual; m.res_sb = fus->res_stride_b; m.res_sc = fus->res_stride_c; m.res_scale = fus->res_scale;
  }
  mr_node_kernel<<<dim3(ceil_div(N, TILE), ceil_div(co, TILE), B), NTHREADS, 0, stream>>>(m);
  DGCN_LAUNCH_CHECK();
  if (train) {
    bn_finalize_kernel<<<static_cast<unsigned>(co), 256, 0, stream>>>(
        partial, pl.n_partial, static_cast<int>(co), static_cast<double>(B) * N, p->bn_weight, p->bn_bias, p->bn_eps,
        st, p->batch_mean_out, p->batch_var_out);
    DGCN_LAUNCH_CHECK();
    const int64_t total = B * co * N;
    bn_apply_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(
        out, nullptr, st, static_cast<int>(co), static_cast<int>(N), total);
    DGCN_LAUNCH_CHECK();
  }
  return DGCN_OK;
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

size_t dgcn_knn_graph_workspace_bytes(int64_t B, int64_t C, int64_t N, int64_t K) {
  return knn_workspace_bytes(B, C, N, K);
}

int dgcn_knn_graph(const float* x, int64_t B, int64_t C, int64_t N, int64_t stride_b, int64_t stride_c,
                   const dgcn_dilation* dil, int32_t exclude_self, int64_t* edge_index, int32_t* nbr, void* wsp,
                   size_t ws_bytes, dgcn_stream_t stream) {
  KnnArgs a;
  int rc = fill_knn_args(a, x, B, C, N, stride_b, stride_c, dil, exclude_self);
  if (rc != DGCN_OK) return rc;
  if (!edge_index && !nbr) return DGCN_ERR_BAD_ARG;
  a.epi.edge_index = edge_index;
  a.epi.nbr = nbr;
  Workspace ws(wsp, ws_bytes);
  return launch_knn(a, ws, static_cast<cudaStream_t>(stream));
}

size_t dgcn_graph_conv_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out, int64_t N, int64_t k) {
  return conv_plan_bytes(conv_plan(conv, B, C_in, C_out, N, k, false));
}

int dgcn_graph_conv_forward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N, int64_t stride_b,
                            int64_t stride_c, const int64_t* edge_index, const int32_t* nbr, int64_t k,
                            const dgcn_basic_conv* p, int64_t C_out, float* out, void* wsp, size_t ws_bytes,
                            dgcn_stream_t stream) {
  int rc = check_conv_args(conv, x, B, C_in, N, p, C_out, out);
  if (rc != DGCN_OK) return rc;
  if ((!edge_index && !nbr) || k <= 0) return DGCN_ERR_BAD_ARG;
  Workspace ws(wsp, ws_bytes);
  return conv_forward(conv, x, B, C_in, N, stride_b, stride_c, edge_index, nbr, k, nullptr, p, C_out, out, nullptr,
                      ws, static_cast<cudaStream_t>(stream));
}

size_t dgcn_dyn_conv_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out, int64_t N, int64_t K) {
  return conv_plan_bytes(conv_plan(conv, B, C_in, C_out, N, K, true)) + knn_workspace_bytes(B, C_in, N, K);
}

int dgcn_dyn_conv_forward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N, int64_t stride_b,
                          int64_t stride_c, const dgcn_dilation* dil, const dgcn_basic_conv* p, int64_t C_out,
                          float* out, int32_t* nbr_out, void* wsp, size_t ws_bytes, dgcn_stream_t stream) {
  return dgcn_dyn_conv_forward_fused(conv, x, B, C_in, N, stride_b, stride_c, dil, p, C_out, out, nbr_out, nullptr, wsp,
                                     ws_bytes, stream);
}

int dgcn_dyn_conv_forward_fused(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N, int64_t stride_b,
                                int64_t stride_c, const dgcn_dilation* dil, const dgcn_basic_conv* p, int64_t C_out,
                                float* out, int32_t* nbr_out, const dgcn_block_fusion* fus, void* wsp, size_t ws_bytes,
                                dgcn_stream_t stream) {
  int rc = check_conv_args(conv, x, B, C_in, N, p, C_out, out);
  if (rc != DGCN_OK) return rc;
  if (!dil) return DGCN_ERR_BAD_ARG;
  Workspace ws(wsp, ws_bytes);
  return conv_forward(conv, x, B, C_in, N, stride_b, stride_c, nullptr, nullptr, 0, dil, p, C_out, out, nbr_out, ws,
                      static_cast<cudaStream_t>(stream), fus);
}

}  // extern "C"

// Dense path, forward: C ABI entry points dgcn_knn_graph / dgcn_graph_conv_forward /
// dgcn_dyn_conv_forward and the node-level kernels around the selection kernels.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include "knn_tc4.cuh"

namespace dgcn {

// tensor-core distance rows of the large-K slab path (dist_rows_tc.cu)
bool dist_rows_tc_ok(const KnnArgs& a);
size_t dist_rows_tc_plane_elems(int64_t B, int64_t C, int64_t N);
int dist_rows_tc_prepare(const KnnArgs& a, __nv_bfloat16* planes, cudaStream_t stream);
int dist_rows_tc_launch(const KnnArgs& a, const __nv_bfloat16* planes, int b0, int nb, float* drows, int ldd,
                        cudaStream_t stream);

// ---- kNN plan: the route of a call, decided once -------------------------------------
constexpr int TC_FALLBACK_GRID = 132;  // CTAs of the exact completion kernel (one uncertified query at a time each; H100 SXM SMs)

// The device limits a plan reads, read once per call so that the workspace query and the launch see the same values.
struct DeviceLimits { int sms; size_t l2_bytes; };
static DeviceLimits device_limits() { return DeviceLimits{device_sm_count(), device_l2_bytes()}; }

static int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

enum KnnRoute {
  KNN_SMALL,   // knn_small_kernel: fp32 distance tiles, K <= SMALL_K_MAX
  KNN_TC,      // tensor-core pre-filter (knn_tc_kernel or knn_tc4_kernel) + exact completion, K <= TC_K_MAX
  KNN_SLAB     // distance rows of a slab of clouds in the workspace + one warp per row, K <= LARGE_K_MAX
};

struct KnnPlan {
  KnnRoute route;
  int64_t n_partial;   // train-mode statistic rows the route's EdgeConv epilogue writes
  dim3 grid;           // query tiles x clouds
  int kp, kp4;         // KNN_TC: list lengths of knn_tc_kernel and knn_tc4_kernel
  bool packed;         // KNN_TC: knn_tc_kernel's packed candidate keys (N <= 4096)
  bool tc4;            // KNN_TC: knn_tc4_kernel, provided the carved rows turn out aligned for it
  bool rows_on_tc;     // KNN_SLAB: distance rows on the tensor cores (dist_rows_tc.cu), else dist_rows_kernel
  bool two_slabs;      // KNN_SLAB: a second slab buffer, the distance rows of slab s+1 run under the select of slab s
  bool fast;           // KNN_SLAB: select_rows_fast_kernel first, handing the rows it cannot finish to the exact select
  int nbmax, ldd;      // KNN_SLAB: clouds per slab, distance row stride
  int KP, warps, cap, sample_rank, warps_f, select_grid;   // KNN_SLAB: select parameters
  size_t smem, smem_f;
};

// The one place that decides how a call selects.  Host arithmetic on the shape, k, the flags and the epilogue's
// mode: nothing here reads a pointer, so a workspace query plans exactly as the launch does.  Returns
// DGCN_ERR_UNSUPPORTED for a slab the kernels do not cover (the plan is filled in all the same).
static int knn_plan(const KnnArgs& a, const DeviceLimits& lim, KnnPlan& p) {
  const int B = a.B, C = a.C, N = a.N, K = a.K;
  p = KnnPlan{};
  p.grid = dim3(static_cast<unsigned>(ceil_div(N, TILE)), B);
  const int64_t n_cta = static_cast<int64_t>(p.grid.x) * p.grid.y;
  const bool train = a.epi.mode == EPI_EDGE && a.epi.norm == DGCN_NORM_BATCH_TRAIN;
  const bool tc_shape = C <= TC_MAX_C && N >= TILE && (N % TILE) == 0;
  if (!a.exact_fp32 && tc_shape && K <= TC_K_MAX && a.k <= SEL_LD && !(train && a.epi.c_out > 128)) {
    p.route = KNN_TC;
    p.n_partial = n_cta + TC_FALLBACK_GRID;   // knn_exact_rows_kernel writes one row per CTA
    // list length = K + certification margin
    // (a margin of 4 ranks leaves ~1e-5 of the queries of a random 64-d cloud uncertified, 8 ranks none)
    p.kp = K <= 9 ? 16 : K <= 20 ? 28 : K <= 32 ? 40 : 56;
    p.kp4 = knn_tc4_list_len(K);
    p.packed = N <= 4096;
    // T4_GROUPS query tiles per CTA, warp specialised (knn_tc4.cuh), where its smaller work area and fixed consumer fit
    p.tc4 = !a.tc_tile_per_cta && p.packed && !train && (C & 7) == 0 && knn_tc4_list_ok(p.kp4, a.k);
    return DGCN_OK;
  }
  if (K <= SMALL_K_MAX) {
    p.route = KNN_SMALL;
    p.n_partial = n_cta;
    return DGCN_OK;
  }
  p.route = KNN_SLAB;
  p.n_partial = static_cast<int64_t>(B) * N;
  p.rows_on_tc = K <= LARGE_K_MAX && dist_rows_tc_ok(a);
  p.ldd = (N + 3) / 4 * 4;
  // Clouds per slab of distance rows: two slabs are in flight (rows of slab s+1 under the select of slab s), so each
  // gets half of the L2 (at least one cloud).
  const int64_t per_cloud = static_cast<int64_t>(N) * p.ldd * 4;
  int64_t nb = static_cast<int64_t>(lim.l2_bytes / 2) / (per_cloud > 0 ? per_cloud : 1);
  if (nb < 1) nb = 1;
  if (nb > B) nb = B;
  p.nbmax = static_cast<int>(nb);
  p.two_slabs = B > p.nbmax;
  p.KP = next_pow2(K);
  const size_t per_warp = static_cast<size_t>(p.KP) * 8 + static_cast<size_t>(p.ldd) * 4 + static_cast<size_t>((a.k + 31) / 32 * 32) * 4;   // ldd = N rounded up to 4 keeps every warp's u64 array 16-byte aligned
  p.warps = static_cast<int>((200u << 10) / per_warp);   // 0: a single row does not fit in shared memory
  if (p.warps > 4) p.warps = 4;
  p.smem = per_warp * p.warps;
  // sampled fast select: bound = sample_rank-th of 128 samples (mean + 2.5 sigma + 2 of the K/N quantile)
  const double pq = static_cast<double>(K) / N;
  p.sample_rank = static_cast<int>(128.0 * pq + 2.5 * sqrt(128.0 * pq * (1.0 - pq)) + 2.0) + 1;
  if (p.sample_rank > 127) p.sample_rank = 127;
  // room for every key below the bound (no power of two needed: only the wanted bins get sorted);
  // k > 64 keeps the full sort and needs the padded power of two
  // keys below a bound at sample rank r: mean (r+1)/129 N, relative spread ~ 1/sqrt(r+1); leave 3.5 sigma
  const double wmean = (p.sample_rank + 1) / 129.0 * N;
  const int64_t wcap = static_cast<int64_t>(wmean * (1.0 + 3.5 / sqrt(p.sample_rank + 1.0))) + 32;
  int cap = static_cast<int>(wcap > K + 64 ? wcap : K + 64);
  cap = a.k > 64 ? next_pow2(cap > 2 * K ? cap : 2 * K) : (cap + 31) / 32 * 32;
  if (cap < 128) cap = 128;            // the sorted sample lives in the same array
  if (cap > 2048) cap = 2048;
  p.cap = cap;
  p.fast = N >= 512 && cap >= K;
  const size_t per_warp_f = static_cast<size_t>(cap) * 8 + static_cast<size_t>((a.k + 31) / 32 * 32) * 4 + 2560;   // keys, sel, multi-select tables (hist 256, prefix 260 ints, 256 marks -> 2320 B)
  p.warps_f = static_cast<int>((56u << 10) / per_warp_f);   // <= 56 KB per CTA: four CTAs per SM
  if (p.warps_f > 8) p.warps_f = 8;
  if (p.warps_f < 1) p.warps_f = 1;
  p.smem_f = per_warp_f * p.warps_f;
  p.select_grid = 2 * lim.sms;   // grid-stride over the rows the fast select hands over
  return K > LARGE_K_MAX || p.warps < 1 ? DGCN_ERR_UNSUPPORTED : DGCN_OK;
}

// the fused prologue can also produce PQ (EdgeConv): channel / output counts it supports
static bool prologue_pq_ok(const KnnPlan& p, int64_t M) {
  return p.route == KNN_TC && M % 128 == 0 && M <= 256;
}

// ---- kNN workspace: one carve per route ------------------------------------------------
struct KnnRegions {
  float* sq;                     // (B,N) squared norms
  __nv_bfloat16 *planes, *sqp;   // KNN_TC: operand planes, -|x|^2/2 operand block
  float *xt_own, *sqmax;         // KNN_TC: node-major copy of x (MRConv brings its own), max |x|^2 and fp16 error per cloud
  int* fail;                     // KNN_TC: uncertified queries, a counter (first 64 ints) then the list
  __nv_bfloat16* planes3;        // KNN_SLAB: (hi, mid, lo) planes of the tensor-core distance rows
  float* drows[2];               // KNN_SLAB: distance rows, one buffer per slab in flight
  int* rowlist[2];               // KNN_SLAB: per buffer, a counter (first 64 ints) then the rows the fast select hands over
};

static void carve_knn_tc(const KnnArgs& a, Workspace& ws, KnnRegions& r) {
  const size_t B = a.B, N = a.N, cpad = (a.C + 15) / 16 * 16;
  r.planes = ws.take<__nv_bfloat16>(B * TC_PLANES * cpad * N);
  r.xt_own = a.epi.mode == EPI_MR ? nullptr : ws.take<float>(B * N * a.C);
  r.sqmax = ws.take<float>(B * 2);
  r.sqp = ws.take<__nv_bfloat16>(B * 8 * N);
  r.fail = ws.take<int>(B * N + 64);
}

static void carve_knn_slab(const KnnArgs& a, const KnnPlan& p, Workspace& ws, KnnRegions& r) {
  if (p.rows_on_tc) r.planes3 = ws.take<__nv_bfloat16>(dist_rows_tc_plane_elems(a.B, a.C, a.N));
  const int nbuf = p.two_slabs ? 2 : 1;
  for (int i = 0; i < nbuf; ++i) r.drows[i] = ws.take<float>(static_cast<size_t>(p.nbmax) * a.N * p.ldd);
  if (p.fast)
    for (int i = 0; i < nbuf; ++i) r.rowlist[i] = ws.take<int>(static_cast<size_t>(p.nbmax) * a.N + 64);
}

static KnnRegions carve_knn(const KnnArgs& a, const KnnPlan& p, Workspace& ws) {
  KnnRegions r{};
  r.sq = ws.take<float>(static_cast<size_t>(a.B) * a.N);
  if (p.route == KNN_TC) carve_knn_tc(a, ws, r);
  if (p.route == KNN_SLAB) carve_knn_slab(a, p, ws, r);
  return r;
}

// Largest carve over every route a call of this shape can take.  Besides the shape, the route depends on
// DGCN_KNN_EXACT_FP32, on train-mode BatchNorm (for the EdgeConv epilogue) and on k; `carve` is run in counting
// mode for each combination.
template <typename Carve>
static size_t max_over_routes(int64_t B, int64_t C, int64_t N, int64_t K, int mode, int64_t c_out, Carve carve) {
  KnnArgs a{};
  a.B = static_cast<int>(B); a.C = static_cast<int>(C); a.N = static_cast<int>(N); a.K = static_cast<int>(K);
  a.epi.mode = mode; a.epi.c_in = a.C; a.epi.c_out = static_cast<int>(c_out);
  const DeviceLimits lim = device_limits();
  size_t most = 0;
  for (int exact = 0; exact < 2; ++exact)
    for (int norm : {DGCN_NORM_NONE, DGCN_NORM_BATCH_TRAIN})
      for (int k : {1, a.K}) {
        a.exact_fp32 = exact; a.epi.norm = norm; a.k = k;
        KnnPlan p;
        knn_plan(a, lim, p);   // an unsupported slab is still sized as planned
        Workspace ws;
        carve(a, p, ws);
        if (ws.off > most) most = ws.off;
      }
  return most;
}

// ---- kNN launch ------------------------------------------------------------------------
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
// 16-bit matrix (rows, cols) row-major, elements of type `dtype` (bf16 or fp16) -> tensor map with boxes of box_cols
// columns x box_rows rows.  box_cols = 64 (128 bytes), SWIZZLE_128B: a box lands in shared memory as box_rows x 128 B
// rows with the 16-byte chunks XOR-swizzled by (row & 7), which is the canonical MN-major wgmma layout of one 64-wide
// MN block; box_cols = 32 (64 bytes), SWIZZLE_64B: box_rows x 64 B rows, chunks XOR-swizzled by ((row >> 1) & 3), the
// canonical layout of one 32-wide MN block.
static int make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int box_cols, int box_rows,
                          CUtensorMapDataType dtype) {
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enc) return DGCN_ERR_UNSUPPORTED;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1u, 1u};
  const CUtensorMapSwizzle swz = box_cols == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  const CUresult rc = enc(map, dtype, 2, const_cast<void*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return rc == CUDA_SUCCESS ? DGCN_OK : DGCN_ERR_CUDA;
}

// Tensor-core pre-filter route (knn_tc.cuh).
static int launch_knn_tc(KnnArgs& a, const KnnPlan& pl, const KnnRegions& r, cudaStream_t stream,
                         const ProloguePq* pqf) {
  const int B = a.B, N = a.N, C = a.C;
  const int cpad = (C + 15) / 16 * 16;
  DGCN_CUDA_TRY(cudaMemsetAsync(r.fail, 0, 256, stream));
  DGCN_CUDA_TRY(cudaMemsetAsync(r.sqmax, 0, static_cast<size_t>(B) * 8, stream));
  const float* xt = a.epi.mode == EPI_MR ? a.epi.xt : r.xt_own;
  // The kernel is chosen before the prologue: knn_tc4_kernel reads one fp16 plane, knn_tc_kernel the two bf16 planes.
  // Its alignment conditions are known only now that the regions are carved.
  const bool wide = epilogue_wide_ok(a);
  const bool xt32 = (reinterpret_cast<uintptr_t>(xt) & 31) == 0;
  const bool quad = pl.tc4 && wide && xt32;
  // sq, operand plane(s), node-major copy and max |x|^2 in one pass over x (sq overwrites what the caller computed)
  if (pqf) {   // the EdgeConv node GEMM rides on the same pass over x
    const size_t smem = (static_cast<size_t>(TC_MAX_C) * 68 + static_cast<size_t>(C) * pqf->M) * 4;
    DGCN_ENSURE_SMEM((tc_prologue_pq_kernel), smem);
    tc_prologue_pq_kernel<<<dim3(N / 64, B), 256, smem, stream>>>(a.x, a.sb, a.sc, C, cpad, N, const_cast<float*>(a.sq),
                                                                  r.planes, r.xt_own, r.sqmax, r.sqp, *pqf, quad);
  } else {
    tc_prologue_kernel<<<dim3(ceil_div(N, 32), B), 256, 0, stream>>>(a.x, a.sb, a.sc, C, cpad, N,
                                                                 const_cast<float*>(a.sq), r.planes,
                                                                 r.xt_own, r.sqmax, r.sqp, quad);
  }
  DGCN_LAUNCH_CHECK();
  TcArgs t{};
  {
    int rc = quad ? make_plane_map(&t.tm_planes, r.planes, static_cast<int64_t>(B) * cpad, N, 64, cpad,
                                   CU_TENSOR_MAP_DATA_TYPE_FLOAT16)
                  : make_plane_map(&t.tm_planes, r.planes, static_cast<int64_t>(B) * TC_PLANES * cpad, N, 64, cpad,
                                   CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    if (rc == DGCN_OK)
      rc = make_plane_map(&t.tm_sqp, r.sqp, static_cast<int64_t>(B) * 8, N, 64, 8, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    if (quad && rc == DGCN_OK)   // knn_tc4_kernel's 32-candidate tiles
      rc = make_plane_map(&t.tm_cand, r.planes, static_cast<int64_t>(B) * cpad, N, T4_CT, cpad, CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
    if (quad && rc == DGCN_OK)
      rc = make_plane_map(&t.tm_sqc, r.sqp, static_cast<int64_t>(B) * 8, N, T4_CT, 8, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    if (rc != DGCN_OK) return rc;
  }
  t.a = a;
  t.planes = r.planes;
  t.sqp = r.sqp;
  t.xt = xt;
  t.xt32 = xt32 ? 1 : 0;
  t.sqmax = r.sqmax;
  t.Cpad = cpad;
  t.fail_count = r.fail;
  t.fail_list = r.fail + 64;
  const dim3 grid = pl.grid;
  const int64_t n_cta = static_cast<int64_t>(grid.x) * grid.y;
  {
    KernelTimer timer(stream, "knn");
    const int nch = a.epi.mode == EPI_MR ? a.epi.c_in : a.epi.c_out;
    t.wide = wide ? 1 : 0;
    t.flush_early = TC_FLUSH_EARLY;
    t.flush_late = TC_FLUSH_LATE;
    t.work_bytes = static_cast<int>(tc_work_bytes(pl.kp, a.k, t.wide != 0, nch));
    const size_t smem = static_cast<size_t>(t.work_bytes) + sizeof(TcTail) + 1024;
    int rc;
    if (quad) {
      rc = launch_knn_tc4(pl.kp4, t, dim3(static_cast<unsigned>(ceil_div(N / TILE, T4_GROUPS)), B), stream);
    } else
    switch (pl.kp) {
      case 16: rc = launch_knn_tc_kp16(pl.packed, t, grid, smem, stream); break;
      case 28: rc = launch_knn_tc_kp28(pl.packed, t, grid, smem, stream); break;
      case 40: rc = launch_knn_tc_kp40(pl.packed, t, grid, smem, stream); break;
      default: rc = launch_knn_tc_kp56(pl.packed, t, grid, smem, stream); break;
    }
    if (rc != DGCN_OK) return rc;
    DGCN_LAUNCH_CHECK();
    float* extra = a.epi.partial ? a.epi.partial + n_cta * BN_PARTIAL_ROWS * a.epi.c_out : nullptr;
    knn_exact_rows_kernel<<<TC_FALLBACK_GRID, 256, 0, stream>>>(a, t.fail_count, t.fail_list, extra);
    DGCN_LAUNCH_CHECK();
    if (debug_certification_on()) {
      int failed = 0;
      DGCN_CUDA_TRY(cudaMemcpyAsync(&failed, t.fail_count, sizeof(int), cudaMemcpyDeviceToHost, stream));
      DGCN_CUDA_TRY(cudaStreamSynchronize(stream));
      debug_certification_add(failed, static_cast<int64_t>(B) * N);
    }
  }
  return DGCN_OK;
}

// Runs the selection (+ fused consumer described by a.epi) on `stream`, by the route of `pl`, in the regions
// carve_knn took for that plan.
// pqf (optional): produce the EdgeConv node GEMM inside the tensor-core prologue; the caller must have
// checked prologue_pq_ok and skipped node_pq_kernel.
static int launch_knn(KnnArgs& a, const KnnPlan& pl, const KnnRegions& r, cudaStream_t stream,
                      const ProloguePq* pqf = nullptr) {
  const int B = a.B, N = a.N;
  a.sq = r.sq;
  if (pl.route == KNN_TC) return launch_knn_tc(a, pl, r, stream, pqf);
  if (pqf) return DGCN_ERR_BAD_ARG;   // (internal misuse) nobody would produce PQ
  if (pl.rows_on_tc) {
    int rc = dist_rows_tc_prepare(a, r.planes3, stream);      // sq (same FMA chain as sqnorm_kernel) + the bf16 planes
    if (rc != DGCN_OK) return rc;
  } else {
    sqnorm_kernel<<<dim3(ceil_div(N, 256), B), 256, 0, stream>>>(a.x, a.sb, a.sc, a.C, N, r.sq);
    DGCN_LAUNCH_CHECK();
  }
  if (pl.route == KNN_SMALL) {
    const size_t smem = sizeof(SmallSmem<1>);
    DGCN_ENSURE_SMEM((knn_small_kernel<1>), smem);
    {
      KernelTimer timer(stream, "knn");
      knn_small_kernel<1><<<pl.grid, NTHREADS, smem, stream>>>(a);
    }
    DGCN_LAUNCH_CHECK();
    return DGCN_OK;
  }
  const int ldd = pl.ldd, nbmax = pl.nbmax, warps = pl.warps, warps_f = pl.warps_f;
  DGCN_ENSURE_SMEM((select_rows_kernel), pl.smem);
  if (pl.fast) DGCN_ENSURE_SMEM((select_rows_fast_kernel), pl.smem_f);
  KernelTimer timer(stream, "knn");
  // Two-chain slab pipeline: even slabs run (distance rows -> sampled select -> exact completion) on the caller's
  // stream, odd slabs on a side stream with their own row buffer and completion list.  The chains overlap freely:
  // the tensor-core distance rows of one slab run under the instruction-bound select of the other, and - what pays
  // most - the partial last wave of one select (4096 rows are 1.15 .. 2.3 waves of its CTAs) is filled by the CTAs
  // of the other chain.  An event forks the side stream from the caller's stream and one joins it back, so the call
  // is still one stream-ordered operation for the caller (and capturable in a CUDA graph).
  cudaStream_t side = pl.two_slabs ? slab_side_stream() : nullptr;
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
    float* drows_s = r.drows[buf];
    int* rowlist_s = r.rowlist[buf];
    if (pl.rows_on_tc) {
      int rc = dist_rows_tc_launch(a, r.planes3, b0, nb, drows_s, ldd, st);
      if (rc != DGCN_OK) return rc;
    } else {
      dist_rows_kernel<<<dim3(ceil_div(N, TILE), ceil_div(N, TILE), nb), NTHREADS, 0, st>>>(a, b0, drows_s, ldd);
      DGCN_LAUNCH_CHECK();
    }
    const int64_t rows = static_cast<int64_t>(nb) * N;
    if (pl.fast) {
      DGCN_CUDA_TRY(cudaMemsetAsync(rowlist_s, 0, 256, st));
      select_rows_fast_kernel<<<static_cast<unsigned>(ceil_div(rows, warps_f)), warps_f * 32, pl.smem_f, st>>>(
          a, b0, nb, drows_s, ldd, pl.cap, pl.sample_rank, warps_f, rowlist_s, rowlist_s + 64);
      DGCN_LAUNCH_CHECK();
      select_rows_kernel<<<pl.select_grid, warps * 32, pl.smem, st>>>(a, b0, nb, drows_s, ldd, pl.KP, ldd, warps,
                                                                    rowlist_s + 64, rowlist_s);
      DGCN_LAUNCH_CHECK();
    } else {
      select_rows_kernel<<<static_cast<unsigned>(ceil_div(rows, warps)), warps * 32, pl.smem, st>>>(
          a, b0, nb, drows_s, ldd, pl.KP, ldd, warps, nullptr, nullptr);
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
    BnAcc st = bn_acc_zero();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + tile_col(tx, j);
      float a = act_apply(acc[i][j] + bias, slope);
      if (m < g.co && n < g.N) {
        float v = fmaf(s, a, t);
        if (g.res) v = __fadd_rn(v, __fmul_rn(__ldg(g.res + b * g.res_sb + m * g.res_sc + n), g.res_scale));
        g.out[b * g.out_sb + static_cast<int64_t>(m) * g.N + n] = v;
        if (train) bn_acc_add(st, a);
      }
    }
    if (train) {   // merge over the 16 tx lanes that share this row (lanes differ in low 4 bits)
      BnMoments mo = bn_acc_moments(st);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) mo = bn_merge(mo, bn_shfl_xor(mo, o));
      if (tx == 0 && m < g.co) bn_store_partial(g.partial, static_cast<int64_t>(b) * gridDim.x + blockIdx.x, g.co, m, mo);
    }
  }
}

// Channel c's batch mean and biased variance -> (scale, shift), and both for the host's running-stat update
// (torch BatchNorm2d training semantics: normalise with biased variance).
__device__ __forceinline__ void bn_finalize_channel(double mean, double var, int C, int c,
                                                    const float* __restrict__ bn_w, const float* __restrict__ bn_b,
                                                    float eps, float* __restrict__ st, float* __restrict__ mean_out,
                                                    float* __restrict__ var_out) {
  if (var < 0.0) var = 0.0;
  float inv = 1.0f / sqrtf(static_cast<float>(var) + eps);
  float s = (bn_w ? bn_w[c] : 1.f) * inv;
  st[c] = s;
  st[C + c] = (bn_b ? bn_b[c] : 0.f) - static_cast<float>(mean) * s;
  if (mean_out) mean_out[c] = static_cast<float>(mean);
  if (var_out) var_out[c] = static_cast<float>(var);
}

// fp64 Chan merge of two disjoint sets' (count, mean, M2); either may be empty
__device__ __forceinline__ void bn_merge64(double& n, double& mean, double& m2, double nb, double meanb, double m2b) {
  const double t = n + nb;
  const double f = t > 0.0 ? nb / t : 0.0;
  const double delta = meanb - mean;
  m2 += m2b + delta * (delta * (n * f));
  mean += delta * f;
  n = t;
}

// Batch statistics from the [np][3][C] partial rows (common.cuh), merged in fp64 in a fixed order, one CTA per
// channel.  Local statistics: (scale, shift), batch mean and variance.  Synced (moments != null): this rank's
// [sum a | sum a^2 | count] of the dgcn_bn_sync ABI, formed in fp64 from the merged (count, mean, M2).
__global__ void bn_merge_kernel(const float* __restrict__ partial, int64_t np, int C, double count,
                                const float* __restrict__ bn_w, const float* __restrict__ bn_b, float eps,
                                float* __restrict__ st, float* __restrict__ mean_out, float* __restrict__ var_out,
                                double* __restrict__ moments) {
  __shared__ double rn[256], rm[256], r2[256];
  const int c = blockIdx.x;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int64_t i = threadIdx.x; i < np; i += blockDim.x) {
    const BnMoments p = bn_load_partial(partial, i, C, c);
    bn_merge64(n, mean, m2, p.n, p.mean, p.m2);
  }
  rn[threadIdx.x] = n;
  rm[threadIdx.x] = mean;
  r2[threadIdx.x] = m2;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      n = rn[threadIdx.x];
      mean = rm[threadIdx.x];
      m2 = r2[threadIdx.x];
      bn_merge64(n, mean, m2, rn[threadIdx.x + o], rm[threadIdx.x + o], r2[threadIdx.x + o]);
      rn[threadIdx.x] = n;
      rm[threadIdx.x] = mean;
      r2[threadIdx.x] = m2;
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  n = rn[0];
  mean = rm[0];
  m2 = r2[0];
  if (moments) {
    const double s1 = n * mean;
    moments[c] = s1;
    moments[C + c] = m2 + s1 * mean;   // bn_finalize_moments_kernel subtracts the same product: M2 comes back exact
    if (c == 0) moments[2 * C] = count;
    return;
  }
  bn_finalize_channel(mean, n > 0.0 ? m2 / n : 0.0, C, c, bn_w, bn_b, eps, st, mean_out, var_out);
}
// Synced statistics (dgcn_bn_sync): the same finalisation from the cross-rank moments [sum a | sum a^2 | count],
// the count read on the device.  After the all-reduce the fp64 cancellation costs ~ (mean / std)^2 * 2^-53.
__global__ void bn_finalize_moments_kernel(const double* __restrict__ moments, int C, const float* __restrict__ bn_w,
                                           const float* __restrict__ bn_b, float eps, float* __restrict__ st,
                                           float* __restrict__ mean_out, float* __restrict__ var_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double count = moments[2 * C], s1 = moments[c];
  const double mean = s1 / count;
  bn_finalize_channel(mean, (moments[C + c] - s1 * mean) / count, C, c, bn_w, bn_b, eps, st, mean_out, var_out);
}

// Train mode: (scale, shift) into st from the partial rows of `count` positions; with sync, from the
// statistics of every rank.
static int bn_finalize(const float* partial, int64_t np, int64_t co, double count, const dgcn_basic_conv* p,
                       const dgcn_bn_sync* sync, float* st, cudaStream_t stream) {
  const int C = static_cast<int>(co);
  bn_merge_kernel<<<static_cast<unsigned>(co), 256, 0, stream>>>(partial, np, C, count, p->bn_weight, p->bn_bias,
                                                                 p->bn_eps, st, p->batch_mean_out, p->batch_var_out,
                                                                 sync ? sync->moments : nullptr);
  DGCN_LAUNCH_CHECK();
  if (!sync) return DGCN_OK;
  if (sync->reduce(sync->user) != 0) return DGCN_ERR_REDUCE;
  bn_finalize_moments_kernel<<<static_cast<unsigned>(ceil_div(co, 128)), 128, 0, stream>>>(
      sync->moments, C, p->bn_weight, p->bn_bias, p->bn_eps, st, p->batch_mean_out, p->batch_var_out);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
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
  __shared__ BnMoments red[8][32];
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
    float bs = 1.f, bt = 0.f;
    BnAcc st = bn_acc_zero();
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
            if (train) bn_acc_add(st, a);
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
    if (train) red[warp][lane] = bn_acc_moments(st);
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
    if (train && tid < 32) {
      BnMoments m = red[0][tid];
      for (int w = 1; w < 8; ++w) m = bn_merge(m, red[w][tid]);
      const int64_t cta = static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x;
      if (c0 + tid < nch) bn_store_partial(e.partial, cta, nch, c0 + tid, m);
    }
    __syncthreads();
  }
}

// ---- convolution workspace ------------------------------------------------------------------
struct ConvRegions {
  int64_t n_partial;         // train-mode statistic rows: one per CTA of whatever writes them
  float* wk;                 // packed weights
  float* st;                 // BatchNorm (scale, shift)
  float* partial;            // train mode: [n_partial][3][co] statistics of act() (common.cuh, BnMoments)
  float* bk;                 // EdgeConv: packed bias
  float* pq;                 // EdgeConv: node GEMM (B,N,2co)
  float* out_min;            // EdgeConv, train mode: min over neighbours of act()
  float* xt;                 // MRConv: node-major copy of x
  float* r;                  // MRConv: max_j x_j - x_i
  KnnRegions knn;            // fused graph: the selection's regions
};

// The regions of conv_forward in the order it uses them; a / kp: the selection's arguments and plan when the graph is
// fused, null for a given graph.
static ConvRegions carve_conv(int conv, int64_t B, int64_t ci, int64_t co, int64_t N, bool train, const KnnArgs* a,
                              const KnnPlan* kp, Workspace& ws) {
  ConvRegions r{};
  const bool edge = conv == DGCN_CONV_EDGE;
  // the statistics come from the selection's epilogue, graph_gather_kernel or mr_node_kernel
  r.n_partial = !edge ? ceil_div(N, TILE) * B : kp ? kp->n_partial : ceil_div(N, 32) * B;
  r.wk = ws.take<float>(2 * ci * co);
  r.st = ws.take<float>(2 * co);
  r.partial = train ? ws.take<float>(r.n_partial * BN_PARTIAL_ROWS * co) : nullptr;
  if (edge) {
    r.bk = ws.take<float>(2 * co);
    r.pq = ws.take<float>(B * N * 2 * co);
    r.out_min = train ? ws.take<float>(B * co * N) : nullptr;
  } else {
    r.xt = ws.take<float>(B * N * ci);
    r.r = ws.take<float>(B * ci * N);
  }
  if (kp) r.knn = carve_knn(*a, *kp, ws);
  return r;
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
                        cudaStream_t stream, const dgcn_block_fusion* fus, const dgcn_bn_sync* sync) {
  const bool fused = dil != nullptr;
  if (fus) {   // block epilogue: out = conv + residual * scale, out possibly a channel slice of a wider buffer
    if (!fused || p->norm == DGCN_NORM_BATCH_TRAIN) return DGCN_ERR_UNSUPPORTED;
    if (fus->out_stride_b != 0 && fus->out_stride_b < co * N) return DGCN_ERR_BAD_ARG;
  }
  const int64_t keep = fused ? dil->k : k;
  const bool train = p->norm == DGCN_NORM_BATCH_TRAIN;
  const bool edge = conv == DGCN_CONV_EDGE;
  const int vec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0 && sb % 4 == 0 && sc % 4 == 0 && N % 4 == 0) ? 1 : 0;

  Epilogue e{};
  e.mode = edge ? EPI_EDGE : EPI_MR;
  e.nbr = nbr_out;
  e.slope = act_slope_of(p);
  e.prelu = p->act == DGCN_ACT_PRELU ? p->prelu_weight : nullptr;
  e.norm = p->norm;
  e.bn_w = p->bn_weight; e.bn_b = p->bn_bias; e.bn_m = p->bn_mean; e.bn_v = p->bn_var; e.bn_eps = p->bn_eps;
  e.c_out = static_cast<int>(co);
  e.c_in = static_cast<int>(ci);
  e.out_sb = (fus && fus->out_stride_b) ? fus->out_stride_b : co * N;
  if (fus && fus->residual && edge) {   // (MRConv adds it in its node kernel)
    e.res = fus->residual; e.res_sb = fus->res_stride_b; e.res_sc = fus->res_stride_c; e.res_scale = fus->res_scale;
  }
  KnnArgs a;
  KnnPlan kp;
  if (fused) {
    int rc = fill_knn_args(a, x, B, ci, N, sb, sc, dil, 0);
    if (rc != DGCN_OK) return rc;
    a.epi = e;
    rc = knn_plan(a, device_limits(), kp);
    if (rc != DGCN_OK) return rc;
  }
  const ConvRegions w = carve_conv(conv, B, ci, co, N, train, fused ? &a : nullptr, fused ? &kp : nullptr, ws);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  bool pq_in_prologue = false;

  if (edge) {
    const int M = static_cast<int>(2 * co);
    pack_edge_weights_kernel<<<static_cast<unsigned>(ceil_div(ci * M > M ? ci * M : M, 256)), 256, 0, stream>>>(
        p->weight, p->bias, static_cast<int>(ci), static_cast<int>(co), w.wk, w.bk);
    DGCN_LAUNCH_CHECK();
    e.pq = w.pq;
    e.out = out;
    e.out_min = w.out_min;
    e.partial = w.partial;
    pq_in_prologue = fused && prologue_pq_ok(kp, M);   // the tensor-core prologue computes PQ on its pass over x
    if (!pq_in_prologue) {
      node_pq_kernel<<<dim3(ceil_div(M, TILE), ceil_div(N, TILE), B), NTHREADS, 0, stream>>>(
          x, sb, sc, static_cast<int>(ci), static_cast<int>(N), vec, w.wk, w.bk, M, w.pq);
      DGCN_LAUNCH_CHECK();
    }
  } else {   // MRConv: r = max_j x_j - x_i (gather on a node-major copy), then the node update GEMM
    pack_mr_weights_kernel<<<static_cast<unsigned>(ceil_div(2 * ci * co, 256)), 256, 0, stream>>>(
        p->weight, static_cast<int>(2 * ci), static_cast<int>(co), w.wk);
    DGCN_LAUNCH_CHECK();
    to_node_major_kernel<<<dim3(ceil_div(N, 32), ceil_div(ci, 32), B), dim3(32, 8), 0, stream>>>(
        x, sb, sc, static_cast<int>(ci), static_cast<int>(N), w.xt);
    DGCN_LAUNCH_CHECK();
    e.xt = w.xt;
    e.r_out = w.r;
  }
  if (fused) {
    a.epi = e;
    const ProloguePq pqf{w.wk, w.bk, w.pq, static_cast<int>(2 * co)};
    int rc = launch_knn(a, kp, w.knn, stream, pq_in_prologue ? &pqf : nullptr);
    if (rc != DGCN_OK) return rc;
  } else {
    GatherArgs g{e, edge_index, nbr, static_cast<int>(B), static_cast<int>(N), static_cast<int>(k)};
    graph_gather_kernel<<<dim3(ceil_div(N, 32), B), 256, 0, stream>>>(g);
    DGCN_LAUNCH_CHECK();
  }
  if (!edge) {
    MrNodeArgs m{};
    m.x = x; m.sb = sb; m.sc = sc; m.r = w.r; m.ci = static_cast<int>(ci); m.N = static_cast<int>(N); m.vec = vec;
    m.wk = w.wk; m.bias = p->bias; m.co = static_cast<int>(co);
    m.slope = e.slope; m.prelu = e.prelu;
    m.norm = p->norm; m.bn_w = p->bn_weight; m.bn_b = p->bn_bias; m.bn_m = p->bn_mean; m.bn_v = p->bn_var;
    m.bn_eps = p->bn_eps;
    m.out = out; m.partial = w.partial;
    m.out_sb = e.out_sb;
    if (fus && fus->residual) {
      m.res = fus->residual; m.res_sb = fus->res_stride_b; m.res_sc = fus->res_stride_c; m.res_scale = fus->res_scale;
    }
    mr_node_kernel<<<dim3(ceil_div(N, TILE), ceil_div(co, TILE), B), NTHREADS, 0, stream>>>(m);
    DGCN_LAUNCH_CHECK();
  }
  if (train) {   // EdgeConv normalises the B*N*keep edge activations, MRConv the B*N node activations
    int rc = bn_finalize(w.partial, w.n_partial, co, static_cast<double>(B) * N * (edge ? keep : 1), p, sync, w.st,
                         stream);
    if (rc != DGCN_OK) return rc;
    const int64_t total = B * co * N;
    bn_apply_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(
        out, w.out_min, w.st, static_cast<int>(co), static_cast<int>(N), total);
    DGCN_LAUNCH_CHECK();
  }
  return DGCN_OK;
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

// The workspace queries run the launch's carve in counting mode and report 256 bytes past its last region (512 for
// the dyn conv, which counts the convolution's regions and the selection's); nothing is placed there.

size_t dgcn_knn_graph_workspace_bytes(int64_t B, int64_t C, int64_t N, int64_t K) {
  return max_over_routes(B, C, N, K, EPI_INDEX, 0,
                         [](const KnnArgs& a, const KnnPlan& p, Workspace& ws) { carve_knn(a, p, ws); }) + 256;
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
  KnnPlan pl;
  rc = knn_plan(a, device_limits(), pl);
  if (rc != DGCN_OK) return rc;
  Workspace ws(wsp, ws_bytes);
  const KnnRegions r = carve_knn(a, pl, ws);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  return launch_knn(a, pl, r, static_cast<cudaStream_t>(stream));
}

size_t dgcn_graph_conv_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out, int64_t N, int64_t k) {
  (void)k;
  Workspace ws;
  carve_conv(conv, B, C_in, C_out, N, true, nullptr, nullptr, ws);   // train mode carves the most
  return ws.off + 256;
}

int dgcn_graph_conv_forward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N, int64_t stride_b,
                            int64_t stride_c, const int64_t* edge_index, const int32_t* nbr, int64_t k,
                            const dgcn_basic_conv* p, int64_t C_out, float* out, const dgcn_bn_sync* sync, void* wsp,
                            size_t ws_bytes, dgcn_stream_t stream) {
  int rc = check_conv_args(conv, x, B, C_in, N, p, C_out, out);
  if (rc != DGCN_OK) return rc;
  if ((!edge_index && !nbr) || k <= 0) return DGCN_ERR_BAD_ARG;
  if (sync && (!sync->moments || !sync->reduce)) return DGCN_ERR_BAD_ARG;
  Workspace ws(wsp, ws_bytes);
  return conv_forward(conv, x, B, C_in, N, stride_b, stride_c, edge_index, nbr, k, nullptr, p, C_out, out, nullptr,
                      ws, static_cast<cudaStream_t>(stream), nullptr, sync);
}

size_t dgcn_dyn_conv_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out, int64_t N, int64_t K) {
  return max_over_routes(B, C_in, N, K, conv == DGCN_CONV_EDGE ? EPI_EDGE : EPI_MR, C_out,
                         [&](const KnnArgs& a, const KnnPlan& p, Workspace& ws) {
                           carve_conv(conv, B, C_in, C_out, N, a.epi.norm == DGCN_NORM_BATCH_TRAIN, &a, &p, ws);
                         }) + 512;
}

int dgcn_dyn_conv_forward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N, int64_t stride_b,
                          int64_t stride_c, const dgcn_dilation* dil, const dgcn_basic_conv* p, int64_t C_out,
                          float* out, int32_t* nbr_out, const dgcn_block_fusion* fus, const dgcn_bn_sync* sync,
                          void* wsp, size_t ws_bytes, dgcn_stream_t stream) {
  int rc = check_conv_args(conv, x, B, C_in, N, p, C_out, out);
  if (rc != DGCN_OK) return rc;
  if (!dil) return DGCN_ERR_BAD_ARG;
  if (sync && (!sync->moments || !sync->reduce)) return DGCN_ERR_BAD_ARG;
  Workspace ws(wsp, ws_bytes);
  return conv_forward(conv, x, B, C_in, N, stride_b, stride_c, nullptr, nullptr, 0, dil, p, C_out, out, nbr_out, ws,
                      static_cast<cudaStream_t>(stream), fus, sync);
}

}  // extern "C"

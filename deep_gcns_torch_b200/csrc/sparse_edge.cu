// Sparse layout, EdgeConv: C ABI entry points dgcn_sparse_edge_conv_forward / dgcn_sparse_edge_conv_backward.
// Reference: gcn_lib/sparse/torch_vertex.py:106-114 (EdgConv over torch_geometric's EdgeConv) with the sparse MLP
// gcn_lib/sparse/torch_nn.py:50-68 (Linear -> norm -> act):
//   out_i = max over edges e = (j -> i) of act(BN(W [x_i ; x_j - x_i] + b)),   0 for a node without in-edges.
//
// The Linear is factorised as on the dense path: z_e = P_i + Q_j with P = (W1 - W2) x + b, Q = W2 x, two node-level
// GEMMs stored node-major as PQ (N, 2 C_out).  With f(z) = act(fmaf(s, z, t)), (s, t) the per-channel BatchNorm
// affine or (1, 0), f is monotone (relu, leaky relu, PReLU weight >= 0) or V-shaped (PReLU weight < 0) in z, and
// fmaf and the multiplication by a fixed slope are monotone in fp32.  So max_e f(z_e) = max(f(z_max), f(z_min))
// exactly in fp32: the edge pass keeps z_max and z_min per (row, channel), and in train mode it also gathers the
// statistics of z over all E edges; the node pass applies f once (bn_merge_kernel between the two produces (s, t)).
// Rows are the CSR rows of dgcn_csr_build (destinations, edges in edge_index order); one warp per row, lanes over
// output channels.
//
// Backward: y_e = f(z_e) is recomputed with the forward's expression and grad_out goes to the first edge of the row
// whose y_e equals the row maximum (torch_scatter's scatter_max).  Train mode spreads it over every edge through the
// BatchNorm backward (two passes: pass 0 forms sum du and sum du * zhat, pass 1 dz for every edge).  dP_i sums over
// row i's edges in registers, dQ_j is accumulated with atomics, both into node-major dPQ; the parameter gradients and
// grad_x are node-level products of dPQ.
//
// Synced statistics (dgcn_bn_sync, nn.SyncBatchNorm): the forward all-reduces this rank's moments of z between the
// edge pass and the (s, t) finalisation (bn_finalize); the backward all-reduces pass 0's sums, and
// pass 1 runs with the global sums over the global count.  The edge kernels are the same on both paths.
#include "basic_conv.cuh"

namespace dgcn {

constexpr int SPE_WARPS = 8;            // warps per CTA of the edge passes
constexpr int SPE_ROWS_PER_WARP = 4;    // CSR rows per warp
constexpr int SPE_ROWS = SPE_WARPS * SPE_ROWS_PER_WARP;
constexpr int64_t SPE_MAX_N = 65535LL * 32;   // the (N, C) <-> (C, N) transposes put N / 32 on grid.y

struct SpEdgeArgs {
  const float* pq;                         // (N, 2co) node-major
  const int32_t* rowptr;                   // (N + 1)
  const int32_t* src;                      // (E) source node per CSR slot
  int N, co;
  float slope; const float* prelu;         // act slope (1: no activation), PReLU weight on the device
  int norm;                                // dgcn_norm
  const float* bn_w; const float* bn_b; const float* bn_m; const float* bn_v; float bn_eps;   // running (eval) or batch (train) statistics
  float* out;                              // (N, co)
  float* zmax; float* zmin;                // train forward: (N, co) each
  float* partial;                          // [n_cta][3][co]: forward (count, mean, M2) of z; backward sum du, sum du*zhat, sum dslope
  const float* gout;                       // backward: (N, co)
  const float* sums;                       // backward pass 1, train: [2][co] = sum du, sum du*zhat
  double inv_count;                        // backward: 1 / E
  float* dpq;                              // backward: (N, 2co) node-major, zero-initialised
};

// y = f(z) = act(s * z + t): the one expression of the forward's output and of the backward's routing
__device__ __forceinline__ float sp_edge_f(float z, float s, float t, float slope) {
  return act_apply(fmaf(s, z, t), slope);
}

// (s, t) and the normalisation (mean, 1 / std) of channel c from running (eval) or batch (train) statistics;
// (1, 0, 0, 1) without BatchNorm.  The forward's train mode takes (s, t) from bn_merge_kernel, whose expressions
// this repeats, so the backward sees the same bits.
__device__ __forceinline__ void sp_edge_affine(const SpEdgeArgs& g, int c, float& s, float& t, float& mean,
                                               float& inv) {
  s = 1.f; t = 0.f; mean = 0.f; inv = 1.f;
  if (g.norm == DGCN_NORM_NONE || c >= g.co) return;
  inv = 1.0f / sqrtf(__ldg(g.bn_v + c) + g.bn_eps);
  mean = __ldg(g.bn_m + c);
  s = (g.bn_w ? __ldg(g.bn_w + c) : 1.f) * inv;
  t = (g.bn_b ? __ldg(g.bn_b + c) : 0.f) - mean * s;
}

// Edge pass of the forward.  TRAIN = 0: (s, t) known, the output is written directly; TRAIN = 1: z_max / z_min per
// (row, channel) and one partial statistics row of z per CTA.
template <int TRAIN>
__global__ void __launch_bounds__(SPE_WARPS * 32) sp_edge_fwd_kernel(const SpEdgeArgs g) {
  __shared__ BnMoments red[SPE_WARPS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int co = g.co, ld = 2 * co;
  const float slope = g.prelu ? __ldg(g.prelu) : g.slope;
  for (int c0 = 0; c0 < co; c0 += 32) {
    const int c = c0 + lane;
    const bool live = c < co;
    float s = 1.f, t = 0.f, mean, inv;
    if (!TRAIN) sp_edge_affine(g, c, s, t, mean, inv);   // (train mode: the statistics come from this pass)
    BnMoments st{0.f, 0.f, 0.f};
    for (int u = 0; u < SPE_ROWS_PER_WARP; ++u) {
      const int i = blockIdx.x * SPE_ROWS + warp * SPE_ROWS_PER_WARP + u;
      if (i >= g.N) break;
      const int beg = __ldg(g.rowptr + i), end = __ldg(g.rowptr + i + 1);
      const float p = live ? __ldg(g.pq + static_cast<int64_t>(i) * ld + c) : 0.f;
      float zmax = -INFINITY, zmin = INFINITY;
      for (int e0 = beg; e0 < end; e0 += 32) {
        const int mine = e0 + lane < end ? __ldg(g.src + e0 + lane) : 0;
        const int n = min(32, end - e0);
        BnAcc acc = bn_acc_zero();
        for (int q = 0; q < n; ++q) {
          const int j = __shfl_sync(0xffffffffu, mine, q);
          if (!live) continue;
          const float z = p + __ldg(g.pq + static_cast<int64_t>(j) * ld + co + c);
          zmax = fmaxf(zmax, z);
          zmin = fminf(zmin, z);
          if (TRAIN) bn_acc_add(acc, z);
        }
        // each 32-edge chunk is summed about its own first z and merged by Chan's formula: one running sum over a
        // long row (or over rows of different P_i) would hold the squares of all its deviations from one pivot
        if (TRAIN) st = bn_merge(st, bn_acc_moments(acc));
      }
      if (!live) continue;
      const int64_t o = static_cast<int64_t>(i) * co + c;
      if (TRAIN) {
        g.zmax[o] = zmax;
        g.zmin[o] = zmin;
      } else {
        g.out[o] = end > beg ? fmaxf(sp_edge_f(zmax, s, t, slope), sp_edge_f(zmin, s, t, slope)) : 0.f;
      }
    }
    if (TRAIN) {
      red[warp][lane] = st;
      __syncthreads();
      if (warp == 0) {
        BnMoments m = red[0][lane];
        for (int w = 1; w < SPE_WARPS; ++w) m = bn_merge(m, red[w][lane]);
        if (live) bn_store_partial(g.partial, blockIdx.x, co, c, m);
      }
      __syncthreads();
    }
  }
}

// Node pass of the train-mode forward: out = max(f(z_max), f(z_min)) with the batch statistics' (s, t) in st.
__global__ void sp_edge_apply_kernel(const SpEdgeArgs g, const float* __restrict__ st) {
  const int64_t k = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k >= static_cast<int64_t>(g.N) * g.co) return;
  const int i = static_cast<int>(k / g.co), c = static_cast<int>(k % g.co);
  const float slope = g.prelu ? __ldg(g.prelu) : g.slope;
  const float s = st[c], t = st[g.co + c];
  const bool any = __ldg(g.rowptr + i + 1) > __ldg(g.rowptr + i);
  g.out[k] = any ? fmaxf(sp_edge_f(g.zmax[k], s, t, slope), sp_edge_f(g.zmin[k], s, t, slope)) : 0.f;
}

// Backward edge pass.  Per (row, channel) the first edge of maximal y_e = f(z_e) carries du = act'(u) g_out,
// u = s z + t (act'(0) = slope, as torch).
// PASS = 0 (train only): partial rows of sum du, sum du * zhat and the PReLU weight's sum u du (u < 0).
// PASS = 1: dz into dPQ - eval / no norm: dz = s du on the routed edge only, and the same partial rows;
//           train: dz_e = s (du_e - sum du / E - zhat_e sum du zhat / E) on every edge.
template <int PASS>
__global__ void __launch_bounds__(SPE_WARPS * 32) sp_edge_bwd_kernel(const SpEdgeArgs g) {
  __shared__ float red[SPE_WARPS][3][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int co = g.co, ld = 2 * co;
  const float slope = g.prelu ? __ldg(g.prelu) : g.slope;
  const bool train = g.norm == DGCN_NORM_BATCH_TRAIN;
  const bool sums_out = PASS == 0 || !train;
  for (int c0 = 0; c0 < co; c0 += 32) {
    const int c = c0 + lane;
    const bool live = c < co;
    float s, t, mean, inv;
    sp_edge_affine(g, c, s, t, mean, inv);
    float dbeta_n = 0.f, dgamma_n = 0.f;
    if (PASS == 1 && train && live) {
      dbeta_n = static_cast<float>(g.sums[c] * g.inv_count);
      dgamma_n = static_cast<float>(g.sums[co + c] * g.inv_count);
    }
    float acc_g = 0.f, acc_gz = 0.f, acc_sl = 0.f;
    for (int u = 0; u < SPE_ROWS_PER_WARP; ++u) {
      const int i = blockIdx.x * SPE_ROWS + warp * SPE_ROWS_PER_WARP + u;
      if (i >= g.N) break;
      const int beg = __ldg(g.rowptr + i), end = __ldg(g.rowptr + i + 1);
      if (end == beg) continue;                        // no in-edges: the output is the constant 0
      const float p = live ? __ldg(g.pq + static_cast<int64_t>(i) * ld + c) : 0.f;
      // routing: the first edge whose y_e is the row maximum
      float best = 0.f, zbest = 0.f;
      int ebest = beg;
      for (int e0 = beg; e0 < end; e0 += 32) {
        const int mine = e0 + lane < end ? __ldg(g.src + e0 + lane) : 0;
        const int n = min(32, end - e0);
        for (int q = 0; q < n; ++q) {
          const int j = __shfl_sync(0xffffffffu, mine, q);
          if (!live) continue;
          const float z = p + __ldg(g.pq + static_cast<int64_t>(j) * ld + co + c);
          const float y = sp_edge_f(z, s, t, slope);
          if (e0 + q == beg || y > best) {
            best = y;
            zbest = z;
            ebest = e0 + q;
          }
        }
      }
      if (!live) continue;
      const float go = __ldg(g.gout + static_cast<int64_t>(i) * co + c);
      const float ub = fmaf(s, zbest, t);
      const float du = ub > 0.f ? go : go * slope;
      if (sums_out) {
        acc_g += du;
        acc_gz += du * ((zbest - mean) * inv);
        if (ub < 0.f) acc_sl += ub * go;
      }
      if (PASS == 0) continue;
      if (!train) {
        const float dz = s * du;
        g.dpq[static_cast<int64_t>(i) * ld + c] = dz;
        atomicAdd(g.dpq + static_cast<int64_t>(__ldg(g.src + ebest)) * ld + co + c, dz);
        continue;
      }
      float dp = 0.f;
      for (int e = beg; e < end; ++e) {
        const int j = __ldg(g.src + e);
        const float z = p + __ldg(g.pq + static_cast<int64_t>(j) * ld + co + c);
        const float due = e == ebest ? du : 0.f;
        const float dz = s * (due - dbeta_n - (z - mean) * inv * dgamma_n);
        dp += dz;
        atomicAdd(g.dpq + static_cast<int64_t>(j) * ld + co + c, dz);
      }
      g.dpq[static_cast<int64_t>(i) * ld + c] = dp;
    }
    if (sums_out) {
      red[warp][0][lane] = acc_g;
      red[warp][1][lane] = acc_gz;
      red[warp][2][lane] = acc_sl;
      __syncthreads();
      if (threadIdx.x < 96) {
        const int which = threadIdx.x >> 5, cc = threadIdx.x & 31;
        float a = 0.f;
        for (int w = 0; w < SPE_WARPS; ++w) a += red[w][which][cc];
        if (c0 + cc < co) g.partial[(static_cast<int64_t>(blockIdx.x) * 3 + which) * co + c0 + cc] = a;
      }
      __syncthreads();
    }
  }
}

// ---- workspace ----------------------------------------------------------------------------------------------
static int64_t sp_edge_ctas(int64_t N) { return ceil_div(N, SPE_ROWS); }

struct SpEdgeRegions {
  float *wk, *bk;        // packed weights (ci x 2co, k-major) and bias (2co)
  float* xt;             // (ci, N) channel-major copy of x
  float* pq;             // (N, 2co) node GEMM
  float* st;             // train forward: (s, t) [2][co]
  float* partial;        // [n_cta][3][co]
  float *zmax, *zmin;    // train forward: (N, co) each
  float *dpq, *dpqt;     // backward: dPQ (N, 2co) and its (2co, N) transpose
  float *wcat, *dwcat;   // backward: (2co x ci) transposed packed weights, their gradient
  double* sums;          // backward: [3][co]
  float* sf;             // backward, train: (sum du, sum du * zhat) as floats for pass 1
};

static SpEdgeRegions carve_sp_edge(bool backward, int64_t N, int64_t ci, int64_t co, bool train, Workspace& ws) {
  SpEdgeRegions r{};
  const int64_t M = 2 * co;
  r.wk = ws.take<float>(ci * M);
  r.bk = ws.take<float>(M);
  r.xt = ws.take<float>(ci * N);
  r.pq = ws.take<float>(N * M);
  if (!backward) {
    r.st = ws.take<float>(2 * co);
    if (train) {
      r.partial = ws.take<float>(sp_edge_ctas(N) * BN_PARTIAL_ROWS * co);
      r.zmax = ws.take<float>(N * co);
      r.zmin = ws.take<float>(N * co);
    }
    return r;
  }
  r.partial = ws.take<float>(sp_edge_ctas(N) * 3 * co);
  r.dpq = ws.take<float>(N * M);
  r.dpqt = ws.take<float>(M * N);
  r.wcat = ws.take<float>(M * ci);
  r.dwcat = ws.take<float>(M * ci);
  r.sums = ws.take<double>(3 * co);
  r.sf = train ? ws.take<float>(2 * co) : nullptr;
  return r;
}

static int check_sp_edge_args(const float* x, int64_t N, int64_t ci, const int32_t* rowptr, const int32_t* src,
                              int64_t E, const dgcn_basic_conv* p, int64_t co, const dgcn_bn_sync* sync,
                              bool backward) {
  if (!x || !rowptr || !src || N <= 0 || ci <= 0 || co <= 0 || E < 0) return DGCN_ERR_BAD_ARG;
  const int rc = check_basic_conv(p, sync, backward);
  if (rc != DGCN_OK) return rc;
  if (N > SPE_MAX_N || E > INT32_MAX || co > 65535 || ci > 65535) return DGCN_ERR_UNSUPPORTED;
  return DGCN_OK;
}

static SpEdgeArgs sp_edge_args(const int32_t* rowptr, const int32_t* src, int64_t N, int64_t co,
                               const dgcn_basic_conv* p) {
  SpEdgeArgs g{};
  g.rowptr = rowptr; g.src = src;
  g.N = static_cast<int>(N); g.co = static_cast<int>(co);
  g.slope = act_slope_of(p);
  g.prelu = p->act == DGCN_ACT_PRELU ? p->prelu_weight : nullptr;
  g.norm = p->norm;
  g.bn_w = p->bn_weight; g.bn_b = p->bn_bias; g.bn_m = p->bn_mean; g.bn_v = p->bn_var; g.bn_eps = p->bn_eps;
  return g;
}

// PQ (N, 2co) = node GEMM of the factorised weights on x (N, ci): x is first transposed to (ci, N), the k-major
// operand the tile engine reads.
static int sp_edge_node_pq(const float* x, int64_t N, int64_t ci, const dgcn_basic_conv* p, int64_t co,
                           const SpEdgeRegions& w, cudaStream_t stream) {
  const int M = static_cast<int>(2 * co), iN = static_cast<int>(N), ici = static_cast<int>(ci);
  pack_edge_weights_kernel<<<static_cast<unsigned>(ceil_div(ci * M, 256)), 256, 0, stream>>>(
      p->weight, p->bias, ici, static_cast<int>(co), w.wk, w.bk);
  DGCN_LAUNCH_CHECK();
  // to_node_major_kernel's (C, N) strided -> (N, C) contiguous, with the roles swapped: x (N, ci) -> xt (ci, N)
  to_node_major_kernel<<<dim3(ceil_div(ci, 32), ceil_div(N, 32), 1), dim3(32, 8), 0, stream>>>(x, 0, ci, iN, ici, w.xt);
  DGCN_LAUNCH_CHECK();
  node_pq_kernel<<<dim3(ceil_div(M, TILE), ceil_div(N, TILE), 1), NTHREADS, 0, stream>>>(
      w.xt, 0, N, ici, iN, (N % 4) == 0 ? 1 : 0, w.wk, w.bk, M, w.pq);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

// The workspace queries run the launch's carve in counting mode (train mode, which carves the most) and report 256
// bytes past its last region; nothing is placed there.
size_t dgcn_sparse_edge_conv_workspace_bytes(int64_t N, int64_t C_in, int64_t C_out) {
  Workspace ws;
  carve_sp_edge(false, N, C_in, C_out, true, ws);
  return ws.off + 256;
}

int dgcn_sparse_edge_conv_forward(const float* x, int64_t N, int64_t C_in, const int32_t* rowptr, const int32_t* src,
                                  int64_t E, const dgcn_basic_conv* p, int64_t C_out, float* out,
                                  const dgcn_bn_sync* sync, void* wsp, size_t ws_bytes, dgcn_stream_t stream_) {
  int rc = check_sp_edge_args(x, N, C_in, rowptr, src, E, p, C_out, sync, false);
  if (rc != DGCN_OK) return rc;
  if (!out) return DGCN_ERR_BAD_ARG;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool train = p->norm == DGCN_NORM_BATCH_TRAIN;
  Workspace ws(wsp, ws_bytes);
  const SpEdgeRegions w = carve_sp_edge(false, N, C_in, C_out, train, ws);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  rc = sp_edge_node_pq(x, N, C_in, p, C_out, w, stream);
  if (rc != DGCN_OK) return rc;
  SpEdgeArgs g = sp_edge_args(rowptr, src, N, C_out, p);
  g.pq = w.pq;
  g.out = out;
  const unsigned grid = static_cast<unsigned>(sp_edge_ctas(N));
  if (!train) {
    sp_edge_fwd_kernel<0><<<grid, SPE_WARPS * 32, 0, stream>>>(g);
    DGCN_LAUNCH_CHECK();
    return DGCN_OK;
  }
  g.zmax = w.zmax; g.zmin = w.zmin; g.partial = w.partial;
  sp_edge_fwd_kernel<1><<<grid, SPE_WARPS * 32, 0, stream>>>(g);
  DGCN_LAUNCH_CHECK();
  // batch statistics of z over the E edges (with sync, over every rank's edges) -> (s, t), batch mean and biased
  // variance; a rank without edges contributes count 0 and still makes its reduce call
  rc = bn_finalize(w.partial, sp_edge_ctas(N), C_out, static_cast<double>(E), p, sync, w.st, stream);
  if (rc != DGCN_OK) return rc;
  sp_edge_apply_kernel<<<static_cast<unsigned>(ceil_div(N * C_out, 256)), 256, 0, stream>>>(g, w.st);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

size_t dgcn_sparse_edge_conv_backward_workspace_bytes(int64_t N, int64_t C_in, int64_t C_out) {
  Workspace ws;
  carve_sp_edge(true, N, C_in, C_out, true, ws);
  return ws.off + 256;
}

int dgcn_sparse_edge_conv_backward(const float* x, int64_t N, int64_t C_in, const int32_t* rowptr,
                                   const int32_t* src, int64_t E, const dgcn_basic_conv* p, int64_t C_out,
                                   const float* grad_out, float* grad_x, float* grad_weight, float* grad_bias,
                                   float* grad_bn_weight, float* grad_bn_bias, float* grad_prelu,
                                   const dgcn_bn_sync* sync, void* wsp, size_t ws_bytes, dgcn_stream_t stream_) {
  int rc = check_sp_edge_args(x, N, C_in, rowptr, src, E, p, C_out, sync, true);
  if (rc != DGCN_OK) return rc;
  if (!grad_out) return DGCN_ERR_BAD_ARG;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool train = p->norm == DGCN_NORM_BATCH_TRAIN;
  Workspace ws(wsp, ws_bytes);
  const SpEdgeRegions w = carve_sp_edge(true, N, C_in, C_out, train, ws);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  rc = sp_edge_node_pq(x, N, C_in, p, C_out, w, stream);
  if (rc != DGCN_OK) return rc;
  const int M = static_cast<int>(2 * C_out), iN = static_cast<int>(N), ici = static_cast<int>(C_in);
  const int ico = static_cast<int>(C_out);
  const int64_t n_cta = sp_edge_ctas(N);
  DGCN_CUDA_TRY(cudaMemsetAsync(w.dpq, 0, static_cast<size_t>(N) * M * sizeof(float), stream));
  SpEdgeArgs g = sp_edge_args(rowptr, src, N, C_out, p);
  g.pq = w.pq;
  g.gout = grad_out;
  g.inv_count = E > 0 ? 1.0 / static_cast<double>(E) : 0.0;
  g.dpq = w.dpq;
  g.partial = w.partial;
  if (train) {
    sp_edge_bwd_kernel<0><<<static_cast<unsigned>(n_cta), SPE_WARPS * 32, 0, stream>>>(g);
    DGCN_LAUNCH_CHECK();
    reduce_partials_kernel<<<dim3(ico, 3), 256, 0, stream>>>(w.partial, n_cta, 3, ico, w.sums);
    DGCN_LAUNCH_CHECK();
    // w.sums keeps this rank's sums: the parameter gradients are local, as in nn.SyncBatchNorm.  With sync, pass 1
    // takes the global sums over the global count, divided in place in sync->moments (each entry is read and
    // written by its own thread, the count at [2 co] by none), with inv_count = 1
    const double* pass1 = w.sums;
    if (sync) {
      rc = bn_sync_moments(w.partial, n_cta, 3, ico, static_cast<double>(E), sync, stream);
      if (rc != DGCN_OK) return rc;
      moments_over_count_kernel<<<static_cast<unsigned>(ceil_div(2 * C_out, 128)), 128, 0, stream>>>(
          sync->moments, ico, sync->moments);
      DGCN_LAUNCH_CHECK();
      pass1 = sync->moments;
      g.inv_count = 1.0;
    }
    // pass 1 wants (sum du, sum du * zhat) as float[2][co]: finish_param_grads_kernel does the conversion
    finish_param_grads_kernel<<<static_cast<unsigned>(ceil_div(C_out, 128)), 128, 0, stream>>>(pass1, ico, 0,
                                                                                                w.sf + C_out, w.sf,
                                                                                                nullptr);
    DGCN_LAUNCH_CHECK();
    g.sums = w.sf;
  }
  sp_edge_bwd_kernel<1><<<static_cast<unsigned>(n_cta), SPE_WARPS * 32, 0, stream>>>(g);
  DGCN_LAUNCH_CHECK();
  if (!train) {   // the eval pass wrote the partial sums
    reduce_partials_kernel<<<dim3(ico, 3), 256, 0, stream>>>(w.partial, n_cta, 3, ico, w.sums);
    DGCN_LAUNCH_CHECK();
  }
  finish_param_grads_kernel<<<static_cast<unsigned>(ceil_div(C_out, 128)), 128, 0, stream>>>(
      w.sums, ico, g.prelu != nullptr, p->norm != DGCN_NORM_NONE ? grad_bn_weight : nullptr,
      p->norm != DGCN_NORM_NONE ? grad_bn_bias : nullptr, grad_prelu);
  DGCN_LAUNCH_CHECK();
  // dPQ (N, 2co) -> (2co, N): the k-major operand of the node products below
  to_node_major_kernel<<<dim3(ceil_div(M, 32), ceil_div(N, 32), 1), dim3(32, 8), 0, stream>>>(w.dpq, 0, M, iN, M,
                                                                                             w.dpqt);
  DGCN_LAUNCH_CHECK();
  if (grad_x) {   // dx[n][c] = sum_m dPQ[n][m] wcat[m][c]: (W1 - W2)^T dP_n + W2^T dQ_n
    pack_mr_weights_kernel<<<static_cast<unsigned>(ceil_div(C_in * M, 256)), 256, 0, stream>>>(w.wk, M, ici, w.wcat);
    DGCN_LAUNCH_CHECK();
    KMajor A = kmajor1(w.dpqt, N, M, iN, (N % 4) == 0);
    KMajor Bm = kmajor1(w.wcat, C_in, M, ici, (C_in % 4) == 0);
    tile_gemm_kernel<<<dim3(ceil_div(C_in, TILE), ceil_div(N, TILE), 1), NTHREADS, 0, stream>>>(
        A, 0, Bm, 0, grad_x, C_in, 0, iN, ici);
    DGCN_LAUNCH_CHECK();
  }
  // xt (ci, N) is x as one channel-major cloud
  return edge_param_grads(w.dpqt, w.xt, 0, N, 1, C_in, C_out, N, w.dwcat, grad_weight, grad_bias, stream);
}

}  // extern "C"

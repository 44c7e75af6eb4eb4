// Dense path, backward (D5 of SURVEY.md 2b): gradients of EdgeConv2d / MRConv2d forward
// w.r.t. x and the BasicConv parameters - what torch autograd derives for
// gcn_lib/dense/torch_vertex.py:16-35 + gcn_lib/dense/torch_nn.py:48-58.
//
// EdgeConv (factorised, see dense_fwd.cu): z_e = P[i'] + Q[j], a_e = act(z_e), y_e = s a_e + t,
// out_i = max_e y_e.  The max routes grad_out to one edge per (i, channel); eval-mode BN keeps
// it there, train-mode BN spreads it over every edge of the batch:
//   da_e = s (g_e - dbeta/n - ahat_e dgamma/n),   dz_e = act'(z_e) da_e,
//   dPQ[i'] += dz_e (P half), dPQ[j] += dz_e (Q half), then two node-level GEMMs.
// MRConv: r_i = max_j x_j - x_i, z = W [x; r] + b: node-level BN/act backward, GEMMs, and a
// scatter of dr through the per-channel argmax.
#include "common.cuh"

namespace dgcn {

float act_slope_of(const dgcn_basic_conv* p);
__global__ void pack_edge_weights_kernel(const float* __restrict__ w, const float* __restrict__ bias, int ci, int co,
                                         float* __restrict__ wk, float* __restrict__ bk);
__global__ void pack_mr_weights_kernel(const float* __restrict__ w, int ci2, int co, float* __restrict__ wk);
__global__ void to_node_major_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N,
                                     float* __restrict__ xt);
__global__ void node_pq_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N, int vec,
                               const float* __restrict__ wk, const float* __restrict__ bk, int M,
                               float* __restrict__ pq);

struct EdgeBwdArgs {
  const float* pq;            // (B,N,2co) node-major, recomputed
  const int64_t* edge_index;  // (2,B,N,k) or null
  const int32_t* nbr;         // (B,N,k) or null
  int B, N, k, co;
  float slope; const float* prelu;
  int norm;                   // dgcn_norm
  const float* bn_w; const float* bn_m; const float* bn_v; float bn_eps;   // mean/var: running (eval) or batch (train)
  const float* gout;          // (B,co,N)
  const float* sums;          // train pass B: [2][co] = dbeta, dgamma (finalised)
  double inv_count;           // 1 / (B*N*k); 1 with synced statistics (sums already divided by the global count)
  float* dpq;                 // (B,2co,N) channel-major, zero-initialised, atomically accumulated
  float* partial;             // [n_cta][3][co]: sum g, sum g*ahat, sum dslope
};

__device__ __forceinline__ void edge_of(const EdgeBwdArgs& g, int64_t node0, int i, int l, int& j, int& ic) {
  const int64_t o = (node0 + i) * g.k + l;
  int64_t jj, cc;
  if (g.edge_index) {
    jj = g.edge_index[o];
    cc = g.edge_index[static_cast<int64_t>(g.B) * g.N * g.k + o];
  } else {
    jj = g.nbr[o];
    cc = i;
  }
  j = static_cast<int>(jj < 0 ? 0 : (jj >= g.N ? g.N - 1 : jj));
  ic = static_cast<int>(cc < 0 ? 0 : (cc >= g.N ? g.N - 1 : cc));
}

// PASS = 0: statistics only (train mode): per channel sum g and sum g*ahat over the arg-max edges.
// PASS = 1: gradient routing into dpq (+ eval-mode statistics, prelu slope gradient).
template <int PASS>
__global__ void __launch_bounds__(256) edge_bwd_kernel(const EdgeBwdArgs g) {
  __shared__ float red[8][3][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y, i0 = blockIdx.x * 32;
  const int N = g.N, k = g.k, co = g.co, ld = 2 * co;
  const int64_t node0 = static_cast<int64_t>(b) * N;
  const float slope = g.prelu ? __ldg(g.prelu) : g.slope;
  const bool train = g.norm == DGCN_NORM_BATCH_TRAIN;
  for (int c0 = 0; c0 < co; c0 += 32) {
    const int c = c0 + lane;
    float s = 1.f, mean = 0.f, inv = 1.f;
    if (g.norm != DGCN_NORM_NONE && c < co) {
      inv = 1.0f / sqrtf(__ldg(g.bn_v + c) + g.bn_eps);
      mean = __ldg(g.bn_m + c);
      s = (g.bn_w ? __ldg(g.bn_w + c) : 1.f) * inv;
    }
    float dbeta_n = 0.f, dgamma_n = 0.f;
    if (PASS == 1 && train && c < co) {
      dbeta_n = static_cast<float>(g.sums[c] * g.inv_count);
      dgamma_n = static_cast<float>(g.sums[co + c] * g.inv_count);
    }
    float acc_g = 0.f, acc_ga = 0.f, acc_sl = 0.f;
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + warp * 4 + u;
      if (i >= N || c >= co) continue;
      const float go = __ldg(g.gout + (static_cast<int64_t>(b) * co + c) * N + i);
      // arg-max edge of y = s*a + t, the first one on a tie as torch.max: first max of a when s > 0, first min when
      // s < 0, edge 0 when s == 0 (every y equals t)
      float best = 0.f;
      int lbest = 0;
      for (int l = 0; l < k; ++l) {
        int j, ic;
        edge_of(g, node0, i, l, j, ic);
        const float a = act_apply(__ldg(g.pq + (node0 + ic) * ld + c) + __ldg(g.pq + (node0 + j) * ld + co + c), slope);
        const bool better = (l == 0) || (s > 0.f ? a > best : s < 0.f && a < best);
        if (better) {
          best = a;
          lbest = l;
        }
      }
      const float ahat_best = (best - mean) * inv;
      acc_g += go;
      acc_ga += go * ahat_best;
      if (PASS == 1) {
        for (int l = 0; l < k; ++l) {
          if (!train && l != lbest) continue;          // eval / no norm: only the arg-max edge carries gradient
          int j, ic;
          edge_of(g, node0, i, l, j, ic);
          const float z = __ldg(g.pq + (node0 + ic) * ld + c) + __ldg(g.pq + (node0 + j) * ld + co + c);
          const float a = act_apply(z, slope);
          const float ge = (l == lbest) ? go : 0.f;
          float da = s * ge;
          if (train) da = s * (ge - dbeta_n - (a - mean) * inv * dgamma_n);
          const float dz = z > 0.f ? da : da * slope;     // act'(0) = slope, as torch (relu'(0) = 0)
          if (z < 0.f) acc_sl += z * da;
          atomicAdd(g.dpq + (static_cast<int64_t>(b) * ld + c) * N + ic, dz);
          atomicAdd(g.dpq + (static_cast<int64_t>(b) * ld + co + c) * N + j, dz);
        }
      }
    }
    red[warp][0][lane] = acc_g;
    red[warp][1][lane] = acc_ga;
    red[warp][2][lane] = acc_sl;
    __syncthreads();
    if (threadIdx.x < 96) {
      const int which = threadIdx.x >> 5, cc = threadIdx.x & 31;
      float t = 0.f;
      for (int w = 0; w < 8; ++w) t += red[w][which][cc];
      const int64_t cta = static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x;
      if (c0 + cc < co) g.partial[(cta * 3 + which) * co + c0 + cc] = t;
    }
    __syncthreads();
  }
}

// fixed-order reduction of [np][nq][C] partials -> sums[nq][C] (double)
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int64_t np, int nq, int C,
                                       double* __restrict__ sums) {
  __shared__ double r[256];
  const int c = blockIdx.x, q = blockIdx.y;
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < np; i += blockDim.x) a += static_cast<double>(partial[(i * nq + q) * C + c]);
  r[threadIdx.x] = a;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) r[threadIdx.x] += r[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[q * C + c] = r[0];
}

__global__ void store_count_kernel(double* __restrict__ dst, double count) { *dst = count; }

// Synced backward sums (dgcn_bn_sync): sync->moments = [the fixed-order fp64 sums of rows q = 0, 1 of the
// [np][nq][C] partials | count], then the caller enqueues their cross-rank sum on `stream`.  (The forward's
// statistics partials are (count, mean, M2) rows: bn_merge_kernel, dense_fwd.cu.)
int bn_sync_moments(const float* partial, int64_t np, int nq, int C, double count, const dgcn_bn_sync* sync,
                    cudaStream_t stream) {
  reduce_partials_kernel<<<dim3(C, 2), 256, 0, stream>>>(partial, np, nq, C, sync->moments);
  DGCN_LAUNCH_CHECK();
  store_count_kernel<<<1, 1, 0, stream>>>(sync->moments + 2 * static_cast<int64_t>(C), count);
  DGCN_LAUNCH_CHECK();
  return sync->reduce(sync->user) == 0 ? DGCN_OK : DGCN_ERR_REDUCE;
}

// Synced backward: the pass-1 operand [sum g | sum g*ahat] / count from the cross-rank moments, so pass 1 runs with
// inv_count = 1 and the global count never visits the host.
__global__ void moments_over_count_kernel(const double* __restrict__ moments, int C, double* __restrict__ sums) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 2 * C) sums[i] = moments[i] / moments[2 * C];
}

// Train mode, after pass 0 wrote its partials: sums[0..2C) = (sum g, sum g*ahat) of this rank, with *inv_count
// left as is, or with sync the global sums already divided by the global count and *inv_count = 1.
static int bn_bwd_pass0_sums(const float* partial, int64_t np, int C, double count, const dgcn_bn_sync* sync,
                             double* sums, double* inv_count, cudaStream_t stream) {
  if (!sync) {
    reduce_partials_kernel<<<dim3(C, 3), 256, 0, stream>>>(partial, np, 3, C, sums);
    DGCN_LAUNCH_CHECK();
    return DGCN_OK;
  }
  int rc = bn_sync_moments(partial, np, 3, C, count, sync, stream);
  if (rc != DGCN_OK) return rc;
  moments_over_count_kernel<<<static_cast<unsigned>(ceil_div(2 * C, 128)), 128, 0, stream>>>(sync->moments, C, sums);
  DGCN_LAUNCH_CHECK();
  *inv_count = 1.0;
  return DGCN_OK;
}

// gradients of the BN affine parameters and of the PReLU slope from the reduced sums
__global__ void finish_param_grads_kernel(const double* __restrict__ sums, int C, int have_slope,
                                          float* __restrict__ grad_bn_w, float* __restrict__ grad_bn_b,
                                          float* __restrict__ grad_prelu) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    if (grad_bn_b) grad_bn_b[c] = static_cast<float>(sums[c]);
    if (grad_bn_w) grad_bn_w[c] = static_cast<float>(sums[C + c]);
  }
  if (grad_prelu && have_slope && blockIdx.x == 0 && threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < C; ++i) t += sums[2 * C + i];
    grad_prelu[0] = static_cast<float>(t);
  }
}

// C[r][c] = sum_k A[k][r] B[k][c]: generic node-level GEMM on the tile engine, plain store.
__global__ void __launch_bounds__(NTHREADS, 2)
    tile_gemm_kernel(KMajor A, int64_t a_batch, KMajor Bm, int64_t b_batch, float* __restrict__ out, int64_t ldo,
                     int64_t o_batch, int rows, int cols) {
  __shared__ TileSmem ts;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, r0 = blockIdx.y * TILE, c0 = blockIdx.x * TILE;
  A.ptr += b * a_batch;
  Bm.ptr += b * b_batch;
  float acc[8][8];
  tile_product(ts, A, r0, Bm, c0, acc);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rr = r0 + tile_row(ty, i);
    if (rr >= rows) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int cc = c0 + tile_col(tx, j);
      if (cc < cols) out[b * o_batch + rr * ldo + cc] = acc[i][j];
    }
  }
}

// Split-K "both operands k-contiguous" GEMM for weight gradients:
//   out[r][c] += sum_{b, n in chunk} A[b][r][n] * Bm[b][c][n]      (atomicAdd, out zero-initialised)
// one CTA = one 128x128 output tile x one chunk of KCH points of one cloud.
constexpr int KCH = 512;
__global__ void __launch_bounds__(NTHREADS, 2)
    wgrad_kernel(const float* __restrict__ A, int64_t a_batch, int64_t lda, int rows, const float* __restrict__ Bm,
                 int64_t b_batch, int64_t ldb, int cols, int N, float* __restrict__ out, int64_t ldo) {
  __shared__ TileSmem ts;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, n0 = blockIdx.x * KCH;
  const int r0 = (blockIdx.y / ((cols + TILE - 1) / TILE)) * TILE, c0 = (blockIdx.y % ((cols + TILE - 1) / TILE)) * TILE;
  const float* Ab = A + b * a_batch;
  const float* Bb = Bm + b * b_batch;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const int nend = min(N, n0 + KCH);
  for (int k0 = n0; k0 < nend; k0 += TK) {
    // transpose-load: element (k, i) of the chunk comes from src[i*ld + k]
    for (int f = tid; f < TK * TILE; f += NTHREADS) {
      const int kk = f & (TK - 1), i = f >> 4;
      const int n = k0 + kk;
      ts.a[0][kk][i] = (r0 + i < rows && n < nend) ? __ldg(Ab + static_cast<int64_t>(r0 + i) * lda + n) : 0.f;
      ts.b[0][kk][i] = (c0 + i < cols && n < nend) ? __ldg(Bb + static_cast<int64_t>(c0 + i) * ldb + n) : 0.f;
    }
    __syncthreads();
    chunk_fma(ts.a[0], ts.b[0], tx, ty, acc);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rr = r0 + tile_row(ty, i);
    if (rr >= rows) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int cc = c0 + tile_col(tx, j);
      if (cc < cols) atomicAdd(out + rr * ldo + cc, acc[i][j]);
    }
  }
}

// EdgeConv: dWcat (2co x ci) -> grad_weight (co x 2ci): W1 = dA, W2 = dW2f - dA; bias from dpq row sums
__global__ void unpack_edge_wgrad_kernel(const float* __restrict__ dwcat, int ci, int co, float* __restrict__ gw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= co * ci) return;
  const int m = i / ci, c = i % ci;
  const float da = dwcat[m * ci + c], dw2 = dwcat[(co + m) * ci + c];
  gw[m * 2 * ci + c] = da;
  gw[m * 2 * ci + ci + c] = dw2 - da;
}
// row sums over (b, n) of a (B, M, N) tensor, rows [0, rows): one block per row
__global__ void row_sum_kernel(const float* __restrict__ t, int B, int M, int N, int rows, float* __restrict__ out) {
  __shared__ double r[256];
  const int m = blockIdx.x;
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < static_cast<int64_t>(B) * N; i += blockDim.x) {
    const int b = static_cast<int>(i / N), n = static_cast<int>(i % N);
    a += static_cast<double>(t[(static_cast<int64_t>(b) * M + m) * N + n]);
  }
  r[threadIdx.x] = a;
  __syncthreads();
  for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
    if (threadIdx.x < o) r[threadIdx.x] += r[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0 && m < rows) out[m] = static_cast<float>(r[0]);
}

// ---- MRConv pieces --------------------------------------------------------------------------------------
// r = max_l x_j - x_i' with the arg-max neighbour / its centre recorded per (b, c, i)
struct MrGatherArgs {
  const float* xt; const int64_t* edge_index; const int32_t* nbr; int B, N, k, ci;
  float* r; int32_t* arg_j; int32_t* arg_i;
};
__global__ void __launch_bounds__(256) mr_gather_arg_kernel(const MrGatherArgs g) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y, i = blockIdx.x * 8 + warp;
  if (i >= g.N) return;
  const int64_t node0 = static_cast<int64_t>(b) * g.N;
  EdgeBwdArgs e{};
  e.edge_index = g.edge_index; e.nbr = g.nbr; e.B = g.B; e.N = g.N; e.k = g.k;
  for (int c = lane; c < g.ci; c += 32) {
    float best = 0.f;
    int bj = 0, bi = i;
    for (int l = 0; l < g.k; ++l) {
      int j, ic;
      edge_of(e, node0, i, l, j, ic);
      const float v = __ldg(g.xt + (node0 + j) * g.ci + c) - __ldg(g.xt + (node0 + ic) * g.ci + c);
      if (l == 0 || v > best) {
        best = v;
        bj = j;
        bi = ic;
      }
    }
    const int64_t o = (static_cast<int64_t>(b) * g.ci + c) * g.N + i;
    g.r[o] = best;
    g.arg_j[o] = bj;
    g.arg_i[o] = bi;
  }
}

// z (B,co,N) pre-activation, gout -> dz in place of z; PASS 0: statistics, PASS 1: apply
struct MrBnArgs {
  float* z; const float* gout; int B, co, N;
  float slope; const float* prelu; int norm;
  const float* bn_w; const float* bn_m; const float* bn_v; float bn_eps;
  const double* sums; double inv_count; float* partial;   // inv_count as in EdgeBwdArgs; partial [n_cta][3][co]
};
template <int PASS>
__global__ void __launch_bounds__(256) mr_bn_bwd_kernel(const MrBnArgs g) {
  __shared__ float red[3][256];
  const int c = blockIdx.y, b = blockIdx.z;
  const float slope = g.prelu ? __ldg(g.prelu) : g.slope;
  const bool train = g.norm == DGCN_NORM_BATCH_TRAIN;
  float s = 1.f, mean = 0.f, inv = 1.f;
  if (g.norm != DGCN_NORM_NONE) {
    inv = 1.0f / sqrtf(__ldg(g.bn_v + c) + g.bn_eps);
    mean = __ldg(g.bn_m + c);
    s = (g.bn_w ? __ldg(g.bn_w + c) : 1.f) * inv;
  }
  float dbeta_n = 0.f, dgamma_n = 0.f;
  if (PASS == 1 && train) {
    dbeta_n = static_cast<float>(g.sums[c] * g.inv_count);
    dgamma_n = static_cast<float>(g.sums[g.co + c] * g.inv_count);
  }
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < g.N) {
    const int64_t o = (static_cast<int64_t>(b) * g.co + c) * g.N + n;
    const float z = g.z[o], go = g.gout[o];
    const float ahat = (act_apply(z, slope) - mean) * inv;
    a0 = go;
    a1 = go * ahat;
    if (PASS == 1) {
      float da = s * go;
      if (train) da = s * (go - dbeta_n - ahat * dgamma_n);
      if (z < 0.f) a2 = z * da;
      g.z[o] = z > 0.f ? da : da * slope;             // act'(0) = slope, as torch (relu'(0) = 0)
    }
  }
  red[0][threadIdx.x] = a0;
  red[1][threadIdx.x] = a1;
  red[2][threadIdx.x] = a2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] += red[0][threadIdx.x + o];
      red[1][threadIdx.x] += red[1][threadIdx.x + o];
      red[2][threadIdx.x] += red[2][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x < 3) {
    const int64_t cta = static_cast<int64_t>(b) * gridDim.x + blockIdx.x;
    g.partial[(cta * 3 + threadIdx.x) * g.co + c] = red[threadIdx.x][0];
  }
}

__global__ void add_bias_kernel(float* __restrict__ z, const float* __restrict__ bias, int co, int N, int64_t total) {
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) z[i] += bias[(i / N) % co];
}

// dx = dxcat[:, :ci] ; dr = dxcat[:, ci:] flows +dr to the arg-max neighbour and -dr to its centre
__global__ void mr_scatter_kernel(const float* __restrict__ dxcat, const int32_t* __restrict__ arg_j,
                                  const int32_t* __restrict__ arg_i, int B, int ci, int N, float* __restrict__ gx) {
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(B) * ci * N) return;
  const int n = static_cast<int>(t % N), c = static_cast<int>((t / N) % ci), b = static_cast<int>(t / (static_cast<int64_t>(N) * ci));
  const float dxd = dxcat[(static_cast<int64_t>(b) * 2 * ci + c) * N + n];
  const float dr = dxcat[(static_cast<int64_t>(b) * 2 * ci + ci + c) * N + n];
  float* row = gx + (static_cast<int64_t>(b) * ci + c) * N;
  atomicAdd(row + n, dxd);
  atomicAdd(row + arg_j[t], dr);
  atomicAdd(row + arg_i[t], -dr);
}

// The regions of dgcn_graph_conv_backward, in the order it uses them.
struct BwdRegions {
  int64_t n_partial;         // statistic rows: one per CTA of edge_bwd_kernel / mr_bn_bwd_kernel
  float* wk;                 // packed weights
  float* partial;            // [n_partial][3][co] partial sums
  double* sums;              // [3][co] their fixed-order reductions
  float *bk, *pq, *dpq;      // EdgeConv: packed bias, node GEMM (B,N,2co), its gradient (B,2co,N)
  float* dwcat;              // EdgeConv: dWcat (2co x ci), first the transposed weights for grad_x
  float* sf;                 // EdgeConv, train mode: (dbeta, dgamma) as floats for pass 1
  float *xt, *r, *z, *dxcat; // MRConv: node-major copy of x, max_j x_j - x_i, z then dz, d[x; r]
  int32_t *argj, *argi;      // MRConv: arg-max neighbour and its centre per (b, c, i)
};
static BwdRegions carve_bwd(int conv, int64_t B, int64_t ci, int64_t co, int64_t N, bool train, Workspace& ws) {
  BwdRegions r{};
  const bool edge = conv == DGCN_CONV_EDGE;
  r.n_partial = edge ? ceil_div(N, 32) * B : ceil_div(N, 256) * B;
  r.wk = ws.take<float>(2 * ci * co);
  r.partial = ws.take<float>(r.n_partial * 3 * co);
  r.sums = ws.take<double>(3 * co);
  if (edge) {
    r.bk = ws.take<float>(2 * co);
    r.pq = ws.take<float>(B * N * 2 * co);
    r.dpq = ws.take<float>(B * 2 * co * N);
    r.dwcat = ws.take<float>(2 * co * ci);
    r.sf = train ? ws.take<float>(2 * co) : nullptr;
  } else {
    r.xt = ws.take<float>(B * N * ci);
    r.r = ws.take<float>(B * ci * N);
    r.argj = ws.take<int32_t>(B * ci * N);
    r.argi = ws.take<int32_t>(B * ci * N);
    r.z = ws.take<float>(B * co * N);
    r.dxcat = ws.take<float>(B * 2 * ci * N);
  }
  return r;
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

size_t dgcn_graph_conv_backward_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out, int64_t N,
                                                int64_t k) {
  (void)k;
  Workspace ws;
  carve_bwd(conv, B, C_in, C_out, N, true, ws);   // train mode carves the most
  return ws.off + 512;   // 512 bytes past the last region; nothing is placed there
}

int dgcn_graph_conv_backward(int32_t conv, const float* x, int64_t B, int64_t ci, int64_t N, int64_t sb, int64_t sc,
                             const int64_t* edge_index, const int32_t* nbr, int64_t k, const dgcn_basic_conv* p,
                             int64_t co, const float* grad_out, float* grad_x, float* grad_weight, float* grad_bias,
                             float* grad_bn_weight, float* grad_bn_bias, float* grad_prelu, const dgcn_bn_sync* sync,
                             void* wsp, size_t ws_bytes, dgcn_stream_t stream_) {
  if (conv != DGCN_CONV_EDGE && conv != DGCN_CONV_MR) return DGCN_ERR_UNSUPPORTED;
  if (!x || !p || !p->weight || !grad_out || (!edge_index && !nbr) || B <= 0 || ci <= 0 || co <= 0 || N <= 0 || k <= 0)
    return DGCN_ERR_BAD_ARG;
  if (p->norm != DGCN_NORM_NONE && (!p->bn_mean || !p->bn_var)) return DGCN_ERR_BAD_ARG;
  if (sync && (!sync->moments || !sync->reduce)) return DGCN_ERR_BAD_ARG;
  if (B > 65535 || co > 65535) return DGCN_ERR_UNSUPPORTED;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  Workspace ws(wsp, ws_bytes);
  const int vec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0 && sb % 4 == 0 && sc % 4 == 0 && N % 4 == 0) ? 1 : 0;
  const bool train = p->norm == DGCN_NORM_BATCH_TRAIN;
  if (!train) sync = nullptr;
  const float slope = act_slope_of(p);
  const float* prelu = p->act == DGCN_ACT_PRELU ? p->prelu_weight : nullptr;
  const BwdRegions w = carve_bwd(conv, B, ci, co, N, train, ws);
  if (!ws.ok) return DGCN_ERR_WORKSPACE;
  float* wk = w.wk;
  float* partial = w.partial;
  double* sums = w.sums;
  const int iN = static_cast<int>(N), ico = static_cast<int>(co), ici = static_cast<int>(ci), iB = static_cast<int>(B);

  if (conv == DGCN_CONV_EDGE) {
    float *bk = w.bk, *pq = w.pq, *dpq = w.dpq, *dwcat = w.dwcat;
    const int M = 2 * ico;
    pack_edge_weights_kernel<<<static_cast<unsigned>(ceil_div(ci * M, 256)), 256, 0, stream>>>(p->weight, p->bias, ici,
                                                                                             ico, wk, bk);
    DGCN_LAUNCH_CHECK();
    node_pq_kernel<<<dim3(ceil_div(M, TILE), ceil_div(N, TILE), B), NTHREADS, 0, stream>>>(x, sb, sc, ici, iN, vec, wk, bk,
                                                                                         M, pq);
    DGCN_LAUNCH_CHECK();
    DGCN_CUDA_TRY(cudaMemsetAsync(dpq, 0, static_cast<size_t>(B) * M * N * sizeof(float), stream));
    EdgeBwdArgs g{};
    g.pq = pq; g.edge_index = edge_index; g.nbr = nbr; g.B = iB; g.N = iN; g.k = static_cast<int>(k); g.co = ico;
    g.slope = slope; g.prelu = prelu; g.norm = p->norm;
    g.bn_w = p->bn_weight; g.bn_m = p->bn_mean; g.bn_v = p->bn_var; g.bn_eps = p->bn_eps;
    g.gout = grad_out; g.sums = nullptr; g.inv_count = 1.0 / (static_cast<double>(B) * N * k);
    g.dpq = dpq; g.partial = partial;
    const dim3 grid(ceil_div(N, 32), B);
    EdgeBwdArgs g1 = g;
    if (train) {
      edge_bwd_kernel<0><<<grid, 256, 0, stream>>>(g);
      DGCN_LAUNCH_CHECK();
      int rc = bn_bwd_pass0_sums(partial, w.n_partial, ico, static_cast<double>(B) * N * k, sync, sums, &g1.inv_count,
                                 stream);
      if (rc != DGCN_OK) return rc;
      // pass B wants (dbeta, dgamma) as float[2][co]: finish_param_grads_kernel does the conversion
      finish_param_grads_kernel<<<static_cast<unsigned>(ceil_div(co, 128)), 128, 0, stream>>>(sums, ico, 0, w.sf + co,
                                                                                           w.sf, nullptr);
      DGCN_LAUNCH_CHECK();
      g1.sums = w.sf;
    }
    edge_bwd_kernel<1><<<grid, 256, 0, stream>>>(g1);
    DGCN_LAUNCH_CHECK();
    reduce_partials_kernel<<<dim3(ico, 3), 256, 0, stream>>>(partial, w.n_partial, 3, ico, sums);
    DGCN_LAUNCH_CHECK();
    finish_param_grads_kernel<<<static_cast<unsigned>(ceil_div(co, 128)), 128, 0, stream>>>(
        sums, ico, prelu != nullptr, p->norm != DGCN_NORM_NONE ? grad_bn_weight : nullptr,
        p->norm != DGCN_NORM_NONE ? grad_bn_bias : nullptr, grad_prelu);
    DGCN_LAUNCH_CHECK();
    if (grad_x) {   // dX[b][c][n] = sum_m wcat[m][c] dpq[b][m][n],  wcat[m][c] = wk[c][m] transposed
      // wk is k-major over c; we need k-major over m: pack a (2co x ci) row-major copy
      float* wcat = dwcat;   // reuse as scratch before the weight gradient is formed
      pack_mr_weights_kernel<<<static_cast<unsigned>(ceil_div(ci * M, 256)), 256, 0, stream>>>(wk, M, ici, wcat);
      DGCN_LAUNCH_CHECK();
      KMajor A = kmajor1(wcat, ci, M, ici, (ci % 4) == 0);
      KMajor Bm = kmajor1(dpq, N, M, iN, (N % 4) == 0);
      tile_gemm_kernel<<<dim3(ceil_div(N, TILE), ceil_div(ci, TILE), B), NTHREADS, 0, stream>>>(
          A, 0, Bm, static_cast<int64_t>(M) * N, grad_x, N, ci * N, ici, iN);
      DGCN_LAUNCH_CHECK();
    }
    if (grad_weight) {
      DGCN_CUDA_TRY(cudaMemsetAsync(dwcat, 0, static_cast<size_t>(M) * ci * sizeof(float), stream));
      const int tiles = static_cast<int>(ceil_div(M, TILE) * ceil_div(ci, TILE));
      wgrad_kernel<<<dim3(ceil_div(N, KCH), tiles, B), NTHREADS, 0, stream>>>(dpq, static_cast<int64_t>(M) * N, N, M, x,
                                                                            sb, sc, ici, iN, dwcat, ci);
      DGCN_LAUNCH_CHECK();
      unpack_edge_wgrad_kernel<<<static_cast<unsigned>(ceil_div(co * ci, 256)), 256, 0, stream>>>(dwcat, ici, ico,
                                                                                                grad_weight);
      DGCN_LAUNCH_CHECK();
    }
    if (grad_bias) {
      row_sum_kernel<<<ico, 256, 0, stream>>>(dpq, iB, M, iN, ico, grad_bias);
      DGCN_LAUNCH_CHECK();
    }
    return DGCN_OK;
  }

  // ---- MRConv ---------------------------------------------------------------------------------------------
  float *xt = w.xt, *r = w.r, *z = w.z, *dxcat = w.dxcat;
  int32_t *argj = w.argj, *argi = w.argi;
  to_node_major_kernel<<<dim3(ceil_div(N, 32), ceil_div(ci, 32), B), dim3(32, 8), 0, stream>>>(x, sb, sc, ici, iN, xt);
  DGCN_LAUNCH_CHECK();
  MrGatherArgs mg{xt, edge_index, nbr, iB, iN, static_cast<int>(k), ici, r, argj, argi};
  mr_gather_arg_kernel<<<dim3(ceil_div(N, 8), B), 256, 0, stream>>>(mg);
  DGCN_LAUNCH_CHECK();
  // z[b][m][n] = sum_kk W[m][kk] [x; r][kk][n] + bias[m]   (wk = W^T, k-major over kk)
  pack_mr_weights_kernel<<<static_cast<unsigned>(ceil_div(2 * ci * co, 256)), 256, 0, stream>>>(p->weight, 2 * ici, ico,
                                                                                              wk);
  DGCN_LAUNCH_CHECK();
  {
    KMajor A = kmajor1(wk, co, 2 * ici, ico, (co % 4) == 0);
    KMajor Bm = kmajor2(x, sc, ici, r, N, 2 * ici, iN, vec != 0);
    // batch strides differ per segment: launch per cloud
    for (int64_t b = 0; b < B; ++b) {
      KMajor Bb = Bm;
      Bb.ptr = x + b * sb;
      Bb.ptr2 = r + b * ci * N;
      tile_gemm_kernel<<<dim3(ceil_div(N, TILE), ceil_div(co, TILE), 1), NTHREADS, 0, stream>>>(
          A, 0, Bb, 0, z + b * co * N, N, 0, ico, iN);
      DGCN_LAUNCH_CHECK();
    }
  }
  if (p->bias) {
    add_bias_kernel<<<static_cast<unsigned>(ceil_div(B * co * N, 256)), 256, 0, stream>>>(z, p->bias, ico, iN, B * co * N);
    DGCN_LAUNCH_CHECK();
  }
  MrBnArgs mb{};
  mb.z = z; mb.gout = grad_out; mb.B = iB; mb.co = ico; mb.N = iN; mb.slope = slope; mb.prelu = prelu; mb.norm = p->norm;
  mb.bn_w = p->bn_weight; mb.bn_m = p->bn_mean; mb.bn_v = p->bn_var; mb.bn_eps = p->bn_eps;
  mb.sums = sums; mb.inv_count = 1.0 / (static_cast<double>(B) * N); mb.partial = partial;
  const dim3 bgrid(ceil_div(N, 256), co, B);
  if (train) {
    mr_bn_bwd_kernel<0><<<bgrid, 256, 0, stream>>>(mb);
    DGCN_LAUNCH_CHECK();
    int rc = bn_bwd_pass0_sums(partial, w.n_partial, ico, static_cast<double>(B) * N, sync, sums, &mb.inv_count, stream);
    if (rc != DGCN_OK) return rc;
  }
  mr_bn_bwd_kernel<1><<<bgrid, 256, 0, stream>>>(mb);   // z now holds dz
  DGCN_LAUNCH_CHECK();
  reduce_partials_kernel<<<dim3(ico, 3), 256, 0, stream>>>(partial, w.n_partial, 3, ico, sums);
  DGCN_LAUNCH_CHECK();
  finish_param_grads_kernel<<<static_cast<unsigned>(ceil_div(co, 128)), 128, 0, stream>>>(
      sums, ico, prelu != nullptr, p->norm != DGCN_NORM_NONE ? grad_bn_weight : nullptr,
      p->norm != DGCN_NORM_NONE ? grad_bn_bias : nullptr, grad_prelu);
  DGCN_LAUNCH_CHECK();
  if (grad_bias) {
    row_sum_kernel<<<ico, 256, 0, stream>>>(z, iB, ico, iN, ico, grad_bias);
    DGCN_LAUNCH_CHECK();
  }
  if (grad_weight) {   // dW[m][kk] = sum dz[b][m][n] * [x; r][b][kk][n]
    DGCN_CUDA_TRY(cudaMemsetAsync(grad_weight, 0, static_cast<size_t>(co) * 2 * ci * 4, stream));
    const int tiles = static_cast<int>(ceil_div(co, TILE) * ceil_div(ci, TILE));
    wgrad_kernel<<<dim3(ceil_div(N, KCH), tiles, B), NTHREADS, 0, stream>>>(z, co * N, N, ico, x, sb, sc, ici, iN,
                                                                          grad_weight, 2 * ci);
    DGCN_LAUNCH_CHECK();
    wgrad_kernel<<<dim3(ceil_div(N, KCH), tiles, B), NTHREADS, 0, stream>>>(z, co * N, N, ico, r, ci * N, N, ici, iN,
                                                                          grad_weight + ci, 2 * ci);
    DGCN_LAUNCH_CHECK();
  }
  if (grad_x) {   // dxcat[b][kk][n] = sum_m W[m][kk] dz[b][m][n]
    KMajor A = kmajor1(p->weight, 2 * ci, ico, 2 * ici, ((2 * ci) % 4) == 0 && (reinterpret_cast<uintptr_t>(p->weight) & 15) == 0);
    KMajor Bm = kmajor1(z, N, ico, iN, (N % 4) == 0);
    tile_gemm_kernel<<<dim3(ceil_div(N, TILE), ceil_div(2 * ci, TILE), B), NTHREADS, 0, stream>>>(
        A, 0, Bm, co * N, dxcat, N, 2 * ci * N, 2 * ici, iN);
    DGCN_LAUNCH_CHECK();
    DGCN_CUDA_TRY(cudaMemsetAsync(grad_x, 0, static_cast<size_t>(B) * ci * N * 4, stream));
    mr_scatter_kernel<<<static_cast<unsigned>(ceil_div(B * ci * N, 256)), 256, 0, stream>>>(dxcat, argj, argi, iB, ici, iN,
                                                                                          grad_x);
    DGCN_LAUNCH_CHECK();
  }
  return DGCN_OK;
}

}  // extern "C"

// The BasicConv lowering shared by the dense graph convolutions and the sparse-layout EdgeConv (basic_conv.cuh):
// validation of dgcn_basic_conv / dgcn_bn_sync, weight packing, node-level GEMMs, train-mode BatchNorm statistics
// and EdgeConv's parameter-gradient tail.
#include "basic_conv.cuh"

namespace dgcn {

int check_basic_conv(const dgcn_basic_conv* p, const dgcn_bn_sync* sync, bool backward) {
  if (!p || !p->weight) return DGCN_ERR_BAD_ARG;
  if (sync && (!sync->moments || !sync->reduce)) return DGCN_ERR_BAD_ARG;
  if (p->act < DGCN_ACT_NONE || p->act > DGCN_ACT_PRELU) return DGCN_ERR_UNSUPPORTED;
  if (p->act == DGCN_ACT_PRELU && !p->prelu_weight) return DGCN_ERR_BAD_ARG;
  if (p->norm < DGCN_NORM_NONE || p->norm > DGCN_NORM_BATCH_TRAIN) return DGCN_ERR_UNSUPPORTED;
  const bool stats = backward ? p->norm != DGCN_NORM_NONE : p->norm == DGCN_NORM_BATCH_EVAL;
  if (stats && (!p->bn_mean || !p->bn_var)) return DGCN_ERR_BAD_ARG;
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
// one CTA = one 128x128 output tile x one chunk of KCH points of one cloud (common.cuh).
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
int bn_finalize(const float* partial, int64_t np, int64_t co, double count, const dgcn_basic_conv* p,
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

__global__ void store_count_kernel(double* __restrict__ dst, double count) {
  *dst = count;
}

// Synced backward sums (dgcn_bn_sync): sync->moments = [the fixed-order fp64 sums of rows q = 0, 1 of the
// [np][nq][C] partials | count], then the caller enqueues their cross-rank sum on `stream`.  (The forward's
// statistics partials are (count, mean, M2) rows: bn_merge_kernel.)
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

int edge_param_grads(const float* dpq, const float* x, int64_t sb, int64_t sc, int64_t B, int64_t ci, int64_t co,
                     int64_t N, float* dwcat, float* grad_weight, float* grad_bias, cudaStream_t stream) {
  const int M = static_cast<int>(2 * co), iN = static_cast<int>(N), ici = static_cast<int>(ci);
  const int ico = static_cast<int>(co);
  if (grad_weight) {   // dWcat[m][c] = sum_{b, n} dPQ[b][m][n] x[b][c][n]; W1 = dA, W2 = dB - dA
    DGCN_CUDA_TRY(cudaMemsetAsync(dwcat, 0, static_cast<size_t>(M) * ci * sizeof(float), stream));
    const int tiles = static_cast<int>(ceil_div(M, TILE) * ceil_div(ci, TILE));
    wgrad_kernel<<<dim3(ceil_div(N, KCH), tiles, B), NTHREADS, 0, stream>>>(dpq, static_cast<int64_t>(M) * N, N, M, x,
                                                                          sb, sc, ici, iN, dwcat, ci);
    DGCN_LAUNCH_CHECK();
    unpack_edge_wgrad_kernel<<<static_cast<unsigned>(ceil_div(co * ci, 256)), 256, 0, stream>>>(dwcat, ici, ico,
                                                                                              grad_weight);
    DGCN_LAUNCH_CHECK();
  }
  if (grad_bias) {   // db = sum_{b, n} dP
    row_sum_kernel<<<ico, 256, 0, stream>>>(dpq, static_cast<int>(B), M, iN, ico, grad_bias);
    DGCN_LAUNCH_CHECK();
  }
  return DGCN_OK;
}

}  // namespace dgcn

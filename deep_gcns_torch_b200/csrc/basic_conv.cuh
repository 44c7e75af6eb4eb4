// The BasicConv lowering shared by the dense graph convolutions (dense_fwd.cu, dense_bwd.cu) and the sparse-layout
// EdgeConv (sparse_edge.cu): Linear / 1x1 conv -> BatchNorm -> activation (dgcn_basic_conv), its validation, the
// factorised EdgeConv weights, the node-level GEMMs and the train-mode BatchNorm statistics.  Defined in basic_conv.cu.
#pragma once
#include "common.cuh"

namespace dgcn {

// ---- dgcn_basic_conv / dgcn_bn_sync ---------------------------------------------------------------------
// The checks every BasicConv entry point makes on p and sync: DGCN_ERR_BAD_ARG for a null p or weight, a PReLU
// without its weight, missing statistics (the forward needs the running ones in eval mode, the backward the
// forward's for any norm) or a sync without moments or reduce; DGCN_ERR_UNSUPPORTED for an act or norm out of range.
int check_basic_conv(const dgcn_basic_conv* p, const dgcn_bn_sync* sync, bool backward);
// act_apply's slope of p->act (0 for PReLU, whose slope is read from prelu_weight on the device)
float act_slope_of(const dgcn_basic_conv* p);

// ---- packing and layout -----------------------------------------------------------------------------------
// EdgeConv weight split W.[x_i ; x_j - x_i] = (W1 - W2) x_i + W2 x_j: wk (ci x 2co, k-major), bk = (bias | 0)
__global__ void pack_edge_weights_kernel(const float* __restrict__ w, const float* __restrict__ bias, int ci, int co,
                                         float* __restrict__ wk, float* __restrict__ bk);
// weight transpose: wk[kk][m] = W[m][kk], kk < ci2
__global__ void pack_mr_weights_kernel(const float* __restrict__ w, int ci2, int co, float* __restrict__ wk);
// (B,C,N) strided -> (B,N,C) contiguous
__global__ void to_node_major_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N,
                                     float* __restrict__ xt);

// ---- node-level GEMMs (tile engine, common.cuh) -------------------------------------------------------------
// PQ[b][n][m] = sum_c X[b][c][n] * wk[c][m] + bk[m]
__global__ void node_pq_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N, int vec,
                               const float* __restrict__ wk, const float* __restrict__ bk, int M,
                               float* __restrict__ pq);
// C[r][c] = sum_k A[k][r] B[k][c], plain store
__global__ void tile_gemm_kernel(KMajor A, int64_t a_batch, KMajor Bm, int64_t b_batch, float* __restrict__ out,
                                 int64_t ldo, int64_t o_batch, int rows, int cols);
// split-K: out[r][c] += sum_{b, n} A[b][r][n] * Bm[b][c][n] (atomicAdd, out zero-initialised)
__global__ void wgrad_kernel(const float* __restrict__ A, int64_t a_batch, int64_t lda, int rows,
                             const float* __restrict__ Bm, int64_t b_batch, int64_t ldb, int cols, int N,
                             float* __restrict__ out, int64_t ldo);
// row sums over (b, n) of a (B, M, N) tensor, rows [0, rows): one block per row
__global__ void row_sum_kernel(const float* __restrict__ t, int B, int M, int N, int rows, float* __restrict__ out);
// EdgeConv's weight and bias gradients from the channel-major dPQ (B, 2co, N) and x (element (b, c, n) at
// x[b * sb + c * sc + n]); dwcat (2co x ci) is scratch.  grad_weight / grad_bias may be null.
int edge_param_grads(const float* dpq, const float* x, int64_t sb, int64_t sc, int64_t B, int64_t ci, int64_t co,
                     int64_t N, float* dwcat, float* grad_weight, float* grad_bias, cudaStream_t stream);

// ---- train-mode BatchNorm statistics ----------------------------------------------------------------------
// (scale, shift) into st from the partial rows of `count` positions; with sync, from the statistics of every rank
int bn_finalize(const float* partial, int64_t np, int64_t co, double count, const dgcn_basic_conv* p,
                const dgcn_bn_sync* sync, float* st, cudaStream_t stream);
// fixed-order reduction of [np][nq][C] partials -> sums[nq][C] (double)
__global__ void reduce_partials_kernel(const float* __restrict__ partial, int64_t np, int nq, int C,
                                       double* __restrict__ sums);
// backward: sync->moments = [fp64 sums of rows 0, 1 of the [np][nq][C] partials | count], then its reduce call
int bn_sync_moments(const float* partial, int64_t np, int nq, int C, double count, const dgcn_bn_sync* sync,
                    cudaStream_t stream);
// sums[0..2C) = moments[0..2C) / moments[2C]
__global__ void moments_over_count_kernel(const double* __restrict__ moments, int C, double* __restrict__ sums);
// gradients of the BN affine parameters and of the PReLU slope from the reduced sums
__global__ void finish_param_grads_kernel(const double* __restrict__ sums, int C, int have_slope,
                                          float* __restrict__ grad_bn_w, float* __restrict__ grad_bn_b,
                                          float* __restrict__ grad_prelu);

}  // namespace dgcn

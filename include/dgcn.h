/*
 * dgcn.h - C ABI of the H100-native message-passing hot path of deep_gcns_torch.
 *
 * The reference (lightaime/deep_gcns_torch) has no FFI / plugin layer: its
 * boundary is the Python nn.Module API (SURVEY.md 8b).  This header is the
 * boundary a binding for that API talks to.  Every entry point names the
 * reference code it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - tensors are fp32 (the sparse entry points with a `dtype` argument also take bf16 / fp16
 *     rows, dgcn_dtype), dense, in the reference's own layouts:
 *       dense path   x (B, C, N, 1)  -> element (b,c,n) at x[b*stride_b + c*stride_c + n]
 *                    edge_index (2, B, N, k) int64, plane 0 = neighbour j, plane 1 = centre i
 *       sparse path  x (N, C) row-major, edge_index (2, E) int64 row 0 = source, row 1 = target
 *   - `stream` is a cudaStream_t; nothing synchronises the host, nothing
 *     allocates: scratch memory is a caller-owned workspace sized by the
 *     matching *_workspace_bytes() query;
 *   - return value: DGCN_OK or a negative dgcn_status; no exceptions cross.
 *   - kernels are compiled for sm_90a (H100) only.
 */
#ifndef DGCN_H_
#define DGCN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dgcn_stream_t; /* cudaStream_t */

enum dgcn_status {
  DGCN_OK = 0,
  DGCN_ERR_BAD_ARG = -1,      /* null pointer / negative or inconsistent size */
  DGCN_ERR_UNSUPPORTED = -2,  /* valid request outside what the kernels cover */
  DGCN_ERR_WORKSPACE = -3,    /* workspace too small                          */
  DGCN_ERR_CUDA = -4,         /* launch failed; see dgcn_last_cuda_error()    */
  DGCN_ERR_REDUCE = -5        /* a dgcn_bn_sync reduce callback returned non-zero */
};

/* gcn_lib/dense/torch_nn.py:9-21 (act_layer) */
enum dgcn_act { DGCN_ACT_NONE = 0, DGCN_ACT_RELU = 1, DGCN_ACT_LEAKYRELU = 2, DGCN_ACT_PRELU = 3 };
/* gcn_lib/dense/torch_nn.py:24-33 (norm_layer): BatchNorm2d in eval (running
 * statistics) or train (batch statistics) mode.  InstanceNorm2d cannot be
 * constructed through the reference's BasicConv (torch_nn.py:71 dereferences a
 * None weight), so it is not part of the path. */
enum dgcn_norm { DGCN_NORM_NONE = 0, DGCN_NORM_BATCH_EVAL = 1, DGCN_NORM_BATCH_TRAIN = 2 };
/* gcn_lib/dense/torch_vertex.py:44-49 (GraphConv2d dispatch) */
enum dgcn_conv { DGCN_CONV_EDGE = 0, DGCN_CONV_MR = 1 };
/* Element type of the node / edge rows the sparse entry points read (their `dtype` argument).  bf16 and
 * fp16 rows are widened to fp32 in registers (exact) and everything is computed in fp32 as for fp32 rows. */
enum dgcn_dtype { DGCN_F32 = 0, DGCN_BF16 = 1, DGCN_F16 = 2 };
/* gcn_lib/sparse/torch_message.py:44-85 (GenMessagePassing.aggregate) */
enum dgcn_aggr {
  DGCN_AGGR_SOFTMAX = 0,     /* 'softmax' and 'softmax_sg' (identical forward) */
  DGCN_AGGR_SOFTMAX_SUM = 1,
  DGCN_AGGR_POWER = 2,
  DGCN_AGGR_POWER_SUM = 3,
  DGCN_AGGR_ADD = 4,
  DGCN_AGGR_MEAN = 5,
  DGCN_AGGR_MAX = 6
};

int dgcn_version(void);
const char* dgcn_status_string(int status);
/* text of the last CUDA error seen by this thread ("" if none) */
const char* dgcn_last_cuda_error(void);

/* ------------------------------------------------------------------------
 * Dense path
 * --------------------------------------------------------------------- */

/* Parameters of `BasicConv([2*C_in, C_out], act, norm, bias)`
 * (gcn_lib/dense/torch_nn.py:48-72; state_dict keys nn.0.weight/bias,
 * nn.<i>.weight/bias/running_mean/running_var). */
typedef struct dgcn_basic_conv {
  const float* weight;       /* (C_out, 2*C_in) row-major = Conv2d 1x1 weight */
  const float* bias;         /* (C_out) or NULL                               */
  int32_t act;               /* dgcn_act                                      */
  float slope;               /* leakyrelu negative slope (reference: 0.2)     */
  const float* prelu_weight; /* device scalar for DGCN_ACT_PRELU, else NULL   */
  int32_t norm;              /* dgcn_norm                                     */
  const float* bn_weight;    /* gamma (C_out) or NULL (=1)                    */
  const float* bn_bias;      /* beta  (C_out) or NULL (=0)                    */
  const float* bn_mean;      /* running mean (eval)                           */
  const float* bn_var;       /* running var  (eval)                           */
  float bn_eps;              /* 1e-5                                          */
  float* batch_mean_out;     /* train: batch mean (C_out) out, may be NULL    */
  float* batch_var_out;      /* train: biased batch variance (C_out) out      */
} dgcn_basic_conv;

/* Which ranks of the sorted neighbour list survive
 * (gcn_lib/dense/torch_edge.py:19-29, DenseDilated): rank l*dilation for
 * l < k, or - stochastic branch - the k ranks listed in cols_host (a HOST
 * array drawn by the caller from the CPU generator, torch_edge.py:22-24). */
/* flags: DGCN_KNN_EXACT_FP32 ranks with the fp32 FMA kernels only (no tensor-core
 * pre-filter); DGCN_KNN_TC_TILE_PER_CTA keeps the tensor-core pre-filter on the
 * one-tile-per-CTA kernel where the multi-tile warp-specialised kernel would be chosen.
 * The result is the same list either way - the switches exist for A/B tests and
 * measurements and are a property of the CALL, not of the process. */
enum dgcn_knn_flags {
  DGCN_KNN_DEFAULT = 0,
  DGCN_KNN_EXACT_FP32 = 1,
  DGCN_KNN_TC_TILE_PER_CTA = 2 /* tensor-core path: always the one-tile-per-CTA kernel, never the multi-tile one */
};
typedef struct dgcn_dilation {
  int64_t k;
  int64_t dilation;
  const int32_t* cols_host; /* NULL or k entries, each in [0, k*dilation) */
  int32_t flags;            /* dgcn_knn_flags */
  int32_t reserved;         /* must be 0 */
} dgcn_dilation;

/* Dilated kNN graph of every cloud of a batch.
 * Replaces gcn_lib/dense/torch_edge.py:32-58 (pairwise_distance +
 * dense_knn_matrix) and :61-76 (DenseDilatedKnnGraph.forward); with
 * exclude_self != 0 it replaces :79-101 (DilatedKnnGraph over
 * torch_cluster.knn_graph, loop=False).
 * Ranking: ascending D = (|x_i|^2 + (-2 x_i.x_j)) + |x_j|^2 evaluated in fp32,
 * ties broken towards the smaller j.  No (B,N,N) matrix is materialised for
 * k*dilation <= 64; above that one L2-sized slab of rows lives in `ws`.
 * Outputs (either may be NULL): edge_index (2,B,N,k) int64 exactly as the
 * reference returns it; nbr (B,N,k) int32 = plane 0 only, for the fused
 * consumers below. */
size_t dgcn_knn_graph_workspace_bytes(int64_t B, int64_t C, int64_t N, int64_t K);
int dgcn_knn_graph(const float* x, int64_t B, int64_t C, int64_t N, int64_t stride_b,
                   int64_t stride_c, const dgcn_dilation* dil, int32_t exclude_self,
                   int64_t* edge_index, int32_t* nbr, void* ws, size_t ws_bytes,
                   dgcn_stream_t stream);

/* Train-mode BatchNorm statistics shared across data-parallel ranks (torch.nn.SyncBatchNorm), the `sync`
 * argument of dgcn_graph_conv_forward, dgcn_dyn_conv_forward, dgcn_graph_conv_backward and
 * dgcn_sparse_edge_conv_forward / _backward.  sync == NULL, or a norm other than DGCN_NORM_BATCH_TRAIN: the
 * statistics are the call's own (reduce is never called).  The workspace sizes do not depend on it.
 * moments: caller-owned DEVICE buffer of 2*C_out + 1 doubles.  Forward: [sum a | sum a^2 | count] over the
 *   positions this rank normalises (EdgeConv: the B*N*k edge activations, MRConv: the B*N node activations, the
 *   sparse EdgeConv: the rank's E edge rows of z, E = 0 included);
 *   backward: [sum g | sum g*ahat | count] over the same positions (the sparse EdgeConv then divides the first
 *   2*C_out entries by the global count in place).
 * reduce(user): called on the calling host thread once per call, after the library has enqueued the LOCAL
 *   values into `moments` on `stream` and before it enqueues the work that reads them.  It must enqueue the
 *   element-wise sum of `moments` over all ranks (an all-reduce, in place) in the stream order of `stream` and
 *   return 0; it must not wait for the device.  Every rank has to make the same sequence of calls, so the
 *   all-reduces pair up.  A non-zero return abandons the call with DGCN_ERR_REDUCE (work already enqueued
 *   still runs; the outputs are undefined).  A sync with a NULL moments or reduce is DGCN_ERR_BAD_ARG.
 * After the reduce the library normalises with the GLOBAL mean and biased variance (forward) and forms grad_x
 * from the GLOBAL sums and count (backward); the count is read on the device, so ranks may hold different
 * batch sizes.  The parameter gradients (weight, bias, bn_weight, bn_bias, prelu) stay LOCAL sums, as in
 * torch.nn.SyncBatchNorm: the data-parallel wrapper averages them.  With the routing of EdgeConv's max fixed
 * by the sign of the synced scale, the backward must be given the batch statistics its forward returned. */
typedef struct dgcn_bn_sync {
  double* moments;
  int32_t (*reduce)(void* user);
  void* user;
} dgcn_bn_sync;

/* Static graph convolution on a given graph.
 * Replaces gcn_lib/dense/torch_vertex.py:38-52 (GraphConv2d.forward) =
 * EdgeConv2d.forward :31-35 / MRConv2d.forward :16-20, including
 * batched_index_select (gcn_lib/dense/torch_nn.py:75-96) and BasicConv
 * (torch_nn.py:48-58: conv1x1 -> act -> norm) and the max over neighbours.
 * The graph comes either as the reference's int64 edge_index (2,B,N,k) with
 * arbitrary centres, or as nbr (B,N,k) int32 with centre = own index.
 * out: (B, C_out, N) contiguous.  sync: dgcn_bn_sync or NULL. */
size_t dgcn_graph_conv_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out,
                                       int64_t N, int64_t k);
int dgcn_graph_conv_forward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N,
                            int64_t stride_b, int64_t stride_c, const int64_t* edge_index,
                            const int32_t* nbr, int64_t k, const dgcn_basic_conv* p,
                            int64_t C_out, float* out, const dgcn_bn_sync* sync /* may be NULL */,
                            void* ws, size_t ws_bytes, dgcn_stream_t stream);

/* Dynamic graph convolution: dilated kNN graph on x, then the convolution, in
 * one call; the neighbour list goes from the selection kernel's shared memory
 * straight into the gather/max and never reaches HBM unless nbr_out != NULL.
 * Replaces gcn_lib/dense/torch_vertex.py:55-72 (DynConv2d.forward with
 * knn='matrix').  fus: dgcn_block_fusion or NULL; sync: dgcn_bn_sync or NULL. */
size_t dgcn_dyn_conv_workspace_bytes(int32_t conv, int64_t B, int64_t C_in, int64_t C_out,
                                     int64_t N, int64_t K);

/* Block epilogue around the dynamic convolution (SURVEY.md 8f rank 1), inference (no train-mode BatchNorm: with
 * DGCN_NORM_BATCH_TRAIN a fusion returns DGCN_ERR_UNSUPPORTED):
 *   residual != NULL: out = conv(x) + residual * res_scale   (ResDynBlock2d.forward, gcn_lib/dense/torch_vertex.py:101;
 *     residual (B, C_out, N) with strides res_stride_b / res_stride_c, unit stride along points)
 *   out_stride_b != 0: batch stride of `out` in floats - `out` is a channel slice of a wider (B, C_total, N) buffer
 *     (DenseDynBlock2d's torch.cat, :116, or a model's fusion buffer, examples/sem_seg_dense/architecture.py:52). */
typedef struct dgcn_block_fusion {
  const float* residual;
  int64_t res_stride_b, res_stride_c;
  float res_scale;
  int64_t out_stride_b;
} dgcn_block_fusion;
int dgcn_dyn_conv_forward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N,
                          int64_t stride_b, int64_t stride_c, const dgcn_dilation* dil,
                          const dgcn_basic_conv* p, int64_t C_out, float* out, int32_t* nbr_out,
                          const dgcn_block_fusion* fus /* may be NULL */,
                          const dgcn_bn_sync* sync /* may be NULL */, void* ws, size_t ws_bytes,
                          dgcn_stream_t stream);

/* Gradient of dgcn_graph_conv_forward w.r.t. x and the BasicConv parameters
 * (what torch autograd derives for torch_vertex.py:16-35 + torch_nn.py:48-58).
 * The graph is the one used in forward (edge_index (2,B,N,k) int64 or nbr
 * (B,N,k) int32 with centre = own index; the kNN graph itself is
 * non-differentiable, torch_edge.py:53-56).  With DGCN_NORM_BATCH_TRAIN,
 * p->bn_mean / p->bn_var must hold the BATCH statistics the forward returned.
 * grad_x is (B, C_in, N) contiguous.
 * grad_weight (C_out,2*C_in), grad_bias (C_out), grad_bn_weight/bias (C_out),
 * grad_prelu (1) are OVERWRITTEN; any of them may be NULL.
 * sync: dgcn_bn_sync or NULL.
 * An act or norm out of range is DGCN_ERR_UNSUPPORTED and a PReLU without prelu_weight DGCN_ERR_BAD_ARG, as in
 * the forward. */
size_t dgcn_graph_conv_backward_workspace_bytes(int32_t conv, int64_t B, int64_t C_in,
                                                int64_t C_out, int64_t N, int64_t k);
int dgcn_graph_conv_backward(int32_t conv, const float* x, int64_t B, int64_t C_in, int64_t N,
                             int64_t stride_b, int64_t stride_c, const int64_t* edge_index,
                             const int32_t* nbr, int64_t k,
                             const dgcn_basic_conv* p, int64_t C_out, const float* grad_out,
                             float* grad_x, float* grad_weight, float* grad_bias,
                             float* grad_bn_weight, float* grad_bn_bias, float* grad_prelu,
                             const dgcn_bn_sync* sync /* may be NULL */, void* ws, size_t ws_bytes,
                             dgcn_stream_t stream);

/* ------------------------------------------------------------------------
 * Sparse path
 * --------------------------------------------------------------------- */

/* One-time COO -> CSR-by-destination build of the graph the reference keeps
 * implicit in edge_index (PyG propagate, gcn_lib/sparse/torch_vertex.py:68).
 * Stable: within a destination row, edges keep their edge_index order.
 * rowptr (N+1) int32, src (E) int32 = source node per CSR slot, eid (E) int32 =
 * position of that edge in edge_index (for edge_attr lookup). */
size_t dgcn_csr_build_workspace_bytes(int64_t N, int64_t E);
int dgcn_csr_build(const int64_t* edge_index, int64_t E, int64_t N, int32_t* rowptr,
                   int32_t* src, int32_t* eid, void* ws, size_t ws_bytes, dgcn_stream_t stream);

/* Scalars that the reference keeps either as python floats or as (1,)
 * nn.Parameters (gcn_lib/sparse/torch_message.py:19-40): if the _dev pointer
 * is non-NULL the kernel reads the device scalar, else the host value. */
typedef struct dgcn_genconv_params {
  int32_t aggr;             /* dgcn_aggr */
  float t; const float* t_dev;
  float p; const float* p_dev;
  float y; const float* y_dev;   /* *_sum only: out *= deg^sigmoid(y) */
  float eps;                /* message eps, 1e-7 (torch_vertex.py:26,85) */
  int32_t msg_norm;         /* MsgNorm on/off (torch_message.py:88-99) */
  float msg_scale; const float* msg_scale_dev;
  int32_t add_residual;     /* 1: out = x + m (torch_vertex.py:73); 0: out = m */
  int32_t raw_message;      /* 1: msg_e = x_src[src_e] as is (GenMessagePassing.aggregate on
                               explicit messages, torch_message.py:44); 0: relu(.)+eps */
} dgcn_genconv_params;

/* Long rows ("hubs" of power-law graphs): rows of in-degree >= min_degree are cut into segments of
 * seg_edges edges.  dgcn_csr_hub_rows lists them once per graph, entirely on the device:
 *   items  (2 * max_items int32): (row, segment) pairs, max_items = E / seg_edges + N_hub <= E/seg + E/min_degree + 1
 *   rows   (3 * max_rows  int32): (row, first item, #segments), max_rows <= E / min_degree + 1
 *   counts (2 int32): number of items, number of rows.
 * Given to dgcn_genconv_aggregate (with `partial`, a scratch of items * 3 * C floats) those rows are
 * aggregated by one CTA per segment plus a fixed-order merge instead of one warp per row. */
typedef struct dgcn_csr_hubs {
  const int32_t* items;
  const int32_t* rows;
  const int32_t* counts;
  int32_t min_degree;
  int32_t seg_edges;
  float* partial;
} dgcn_csr_hubs;
int dgcn_csr_hub_rows(const int32_t* rowptr, int64_t N, int64_t E, int32_t min_degree, int32_t seg_edges,
                      int32_t* items, int32_t* rows, int32_t* counts, dgcn_stream_t stream);

/* Block fusion around the aggregate (SURVEY.md 8f rank 1; DeeperGCN 'res+' block,
 * examples/ogb/ogbn_arxiv/model.py:91-106: h <- GENConv(relu(norm(h))) + h) and the split launch
 * that lets a node-partitioned layer overlap its halo exchange:
 *   pre_scale / pre_shift (C) or both NULL: every row read from x_src and x_dst is taken as
 *     act(pre_scale * x + pre_shift) (eval-mode BatchNorm1d folded to an affine, act = relu when
 *     pre_relu != 0), so the normalised / activated copy of h is never written to HBM;
 *   row_list (n_rows int32) or NULL: destination rows this launch processes (NULL = all N rows):
 *     interior rows (all sources local) first, boundary rows once the halo has arrived;
 *   skip_hubs != 0: rows of degree >= hubs->min_degree are left to a later launch. */
typedef struct dgcn_genconv_fusion {
  const float* pre_scale;
  const float* pre_shift;
  int32_t pre_relu;
  int32_t skip_hubs;
  const int32_t* row_list;
  int64_t n_rows;
} dgcn_genconv_fusion;

/* Dropout folded into the pre-activation of the res+ block in training (examples/ogb/ogbn_arxiv/model.py:91-106:
 * dropout(relu(norm(h)))).  keep_bits (N_src, words_per_row) int32 words, bit c % 32 of word c / 32 set when
 * channel c of that row is kept; words_per_row >= ceil(C / 32).  Row r of x_src and row r of x_dst (the first N
 * rows of x_src's numbering) use bit row r.  With it every row read from x_src and x_dst is taken as
 *   keep ? relu(pre_scale * x + pre_shift) * keep_scale : 0          (keep_scale = 1 / (1 - p)),
 * computed in this order in fp32 by the forward and the backward, so both see the same values. */
typedef struct dgcn_keep_mask {
  const int32_t* keep_bits;
  int64_t words_per_row;
  float keep_scale;
} dgcn_keep_mask;

/* Fused GENConv message + aggregate + MsgNorm + residual:
 *   msg_e = relu(x[src_e] + edge_attr[eid_e]) + eps     torch_vertex.py:78-85
 *   m_i   = aggregate_{e -> i}(msg_e)                   torch_message.py:44-85
 *   m_i   = scale * |x_i|_2 * m_i / max(|m_i|_2, 1e-12) torch_message.py:95-99
 *   out_i = x_i + m_i                                   torch_vertex.py:73
 * x_src (N_src, C) holds the rows that sources index (on one GPU the same array
 * as x_dst; under node partitioning local rows followed by halo rows);
 * x_dst (N, C) the rows of the destinations this call owns (may be NULL when neither
 * msg_norm nor add_residual is set).
 * edge_attr (E, C) in edge_index order or NULL.  out (N, C).
 * dtype (dgcn_dtype): x_src, x_dst and edge_attr are all of that type, out stays fp32.  For DGCN_BF16 / DGCN_F16
 * the result is bit-identical to the fp32 call on the same rows converted to fp32.  Half rows need C % 4 == 0,
 * C <= 1024, 8-byte aligned x_src / x_dst / edge_attr, a 16-byte aligned out and no pre-activation
 * (fus->pre_scale NULL); anything else returns DGCN_ERR_UNSUPPORTED.
 * hubs: dgcn_csr_hubs or NULL; fus: dgcn_genconv_fusion or NULL.
 * keep: dgcn_keep_mask or NULL.  A keep mask needs fp32 rows, a pre-activation with pre_relu != 0 and no
 * edge_attr; anything else returns DGCN_ERR_UNSUPPORTED. */
int dgcn_genconv_aggregate(int32_t dtype, const void* x_src, const void* x_dst, int64_t N, int64_t C,
                           const int32_t* rowptr, const int32_t* src, const int32_t* eid,
                           const void* edge_attr, const dgcn_genconv_params* prm,
                           const dgcn_csr_hubs* hubs /* may be NULL */,
                           const dgcn_genconv_fusion* fus /* may be NULL */,
                           const dgcn_keep_mask* keep /* may be NULL */, float* out,
                           dgcn_stream_t stream);
/* Bit-pack a keep mask: keep (N, C) fp32 (non-zero = kept, what Tensor.bernoulli_ draws) -> keep_bits
 * (N, ceil(C / 32)) int32 in the dgcn_keep_mask layout (bits of channels >= C are 0). */
int dgcn_keep_bits_pack(const float* keep, int64_t N, int64_t C, int32_t* keep_bits, dgcn_stream_t stream);

/* Row-wise Linear with fused bias and skip connection on the tensor cores (wgmma):
 *   out[n][m] = sum_k a[n][k] * weight[m][k] (+ bias[m]) (+ res[n][m])
 * = the Linear that ends GENConv's MLP (gcn_lib/sparse/torch_nn.py:56-68 with mlp_layers = 1; nn.Linear
 * weight layout (M, K)) plus the `+ h` of DeeperGCN's res+ block (examples/ogb/ogbn_arxiv/model.py:104).
 * fp32 in / out; the product runs as a two-plane bf16 split of both operands (4 tensor-core products, fp32
 * accumulation, error <= ~2^-16 * sum_k |a||w|).  K in {64, 128, 256}, M a multiple of 32 up to 256,
 * 16-byte aligned rows; anything else returns DGCN_ERR_UNSUPPORTED (callers keep cuBLAS for those).
 * bias, res may be NULL; out may alias res.  ws: dgcn_linear_residual_workspace_bytes(K, M) (0 = unsupported). */
size_t dgcn_linear_residual_workspace_bytes(int64_t K, int64_t M);
int dgcn_linear_residual(const float* a, int64_t N, int64_t K, const float* weight, const float* bias,
                         int64_t M, const float* res, float* out, void* ws, size_t ws_bytes,
                         dgcn_stream_t stream);

/* Gradient of dgcn_genconv_aggregate w.r.t. x (both roles), edge_attr and the
 * scalar parameters.  The softmax weights carry gradient only when
 * softmax_grad != 0 (reference: learn_t, torch_message.py:51-55).
 * grad_x_src (N_src, C) must be zero-initialised by the caller (rows are
 * accumulated with atomics); grad_x_dst (N, C) is overwritten and may alias
 * nothing.  grad_scalars (4) = d/dt, d/dp, d/dy, d/dmsg_scale, accumulated with
 * atomics into a zero-initialised array; may be NULL.
 * dtype (dgcn_dtype): x_src, x_dst, edge_attr and grad_edge_attr are of that type; grad_out, grad_x_src,
 * grad_x_dst and grad_scalars stay fp32.  For half rows grad_edge_attr is written once per CSR edge, rounded to
 * nearest even (no zero-initialisation needed when eid covers every edge_attr row).  Half rows need C % 4 == 0.
 * pre_scale / pre_shift (C) or both NULL, pre_relu: the forward's pre-activation (see dgcn_genconv_fusion); keep:
 * its keep mask (dgcn_keep_mask) or NULL.  The rows are recomputed from x exactly as the forward read them, and
 * grad_x_src / grad_x_dst are the gradients w.r.t. those activated rows (the caller applies the chain rule through
 * the pre-activation).  A pre-activation needs fp32 rows; a keep mask needs a pre-activation with pre_relu != 0
 * and no edge_attr; C > 512 is unsupported; anything else returns DGCN_ERR_UNSUPPORTED. */
int dgcn_genconv_aggregate_backward(int32_t dtype, const void* x_src, const void* x_dst, int64_t N,
                                    int64_t N_src, int64_t C, const int32_t* rowptr,
                                    const int32_t* src, const int32_t* eid,
                                    const void* edge_attr, const dgcn_genconv_params* prm,
                                    int32_t softmax_grad, const float* pre_scale, const float* pre_shift,
                                    int32_t pre_relu, const dgcn_keep_mask* keep /* may be NULL */,
                                    const float* grad_out, float* grad_x_src, float* grad_x_dst,
                                    void* grad_edge_attr, float* grad_scalars, dgcn_stream_t stream);
/* Backward epilogue of the fused res+ block in training: one pass over (N, C) rows
 *   g_y = (g_src + g_dst) * (keep ? keep_scale : 0) * [pre_scale * h + pre_shift > 0]      written over g_src,
 * the gradient w.r.t. the BatchNorm output (keep may be NULL: all kept, scale 1), and per channel
 *   sums[c] += sum_rows g_y,   sums[C + c] += sum_rows g_y * (h - mean[c]) * invstd[c]
 * (fp64, zero-initialised by the caller; the BatchNorm's d beta and d gamma / gamma). */
int dgcn_res_plus_backward_gy(const float* h, int64_t N, int64_t C, const float* pre_scale, const float* pre_shift,
                              const dgcn_keep_mask* keep /* may be NULL */, const float* mean, const float* invstd,
                              float* grad_src, const float* grad_dst, double* sums, dgcn_stream_t stream);
/* ... and its second pass: grad_h = a[c] * g_y + b[c] * h + d[c] + grad_skip (grad_h may alias g_y or grad_skip), the
 * BatchNorm backward folded per channel by the caller (batch statistics: a = gamma * invstd,
 * b = -a * invstd * mean(g_y * xhat), d = -a * mean(g_y) - b * mean; running statistics: a = scale, b = d = 0). */
int dgcn_res_plus_backward_dh(const float* g_y, const float* h, int64_t N, int64_t C, const float* a, const float* b,
                              const float* d, const float* grad_skip, float* grad_h, dgcn_stream_t stream);

/* GIN and GraphSAGE aggregation in the sparse layout (the message passing of gcn_lib/sparse/torch_vertex.py:224-233,
 * torch_geometric's GINConv with eps not trained, and :136-205, the SAGEConv subclass; the MLP, the weight GEMM, the
 * bias and the normalisation stay with the caller).  Over dgcn_csr_build's rowptr (N+1) / src (E) of edge_index:
 *   DGCN_GIN:   out_i = sum_{j->i} x_j + (1 + eps) * x_i  over every edge as given (self loops and duplicates
 *               included, an empty row sums to 0); the sum first, then + fl(fl(1 + eps) * x_i) - the fp32 order of
 *               torch_geometric's GINConv.  eps: (1) DEVICE scalar (the layer's buffer) or NULL for 0.
 *   DGCN_SAGE:  torch_geometric's remove_self_loops + add_self_loops, folded into the walk: with c_i = (number of
 *               edges j -> i with j != i) + 1, out_i = (sum_{j->i, j != i} x_j + x_i) / c_i;
 *   DGCN_RSAGE: the same set with messages x_j - x_i (the added loop's message is 0):
 *               out_i = (sum_{j->i, j != i} x_j - (c_i - 1) * x_i) / c_i.
 * x (N, C) row-major of element type dtype (dgcn_dtype), out (N, C) fp32, C <= 1024; C > 1024 returns
 * DGCN_ERR_UNSUPPORTED.  fp32 rows: float4 lanes when C % 4 == 0 and x, out are 16-byte aligned, one channel per lane
 * otherwise, with the same result.  DGCN_BF16 / DGCN_F16 rows are widened exactly in registers and the result is
 * bit-identical to the fp32 call on the same rows converted to fp32; they need C % 4 == 0, an 8-byte aligned x and a
 * 16-byte aligned out, and anything else returns DGCN_ERR_UNSUPPORTED.  hubs: dgcn_csr_hubs or NULL (rows of
 * in-degree >= min_degree are then aggregated in segments, with the same result up to fp32 re-association). */
enum dgcn_gin_sage { DGCN_GIN = 0, DGCN_SAGE = 1, DGCN_RSAGE = 2 };
int dgcn_gin_sage_aggregate(int32_t dtype, int32_t rule, const void* x, int64_t N, int64_t C, const int32_t* rowptr,
                            const int32_t* src, const dgcn_csr_hubs* hubs /* may be NULL */, const float* eps,
                            float* out, dgcn_stream_t stream);
/* Gradient of dgcn_gin_sage_aggregate w.r.t. x: grad_x (N, C) must be zero-initialised by the caller (rows are
 * accumulated with atomics, so the order of the additions - and the last bits - varies from run to run).  Every
 * source of an edge j -> i receives grad_out_i (GIN) or grad_out_i / c_i (SAGE, RSAGE; edges with j != i only); row i
 * receives (1 + eps) * grad_out_i (GIN), grad_out_i / c_i (SAGE) or -(c_i - 1) / c_i * grad_out_i (RSAGE).
 * x is not read, so the same call serves fp32 and half rows (the caller rounds grad_x to x's type).  C <= 1024. */
int dgcn_gin_sage_aggregate_backward(int32_t rule, int64_t N, int64_t C, const int32_t* rowptr, const int32_t* src,
                                     const float* eps, const float* grad_out, float* grad_x, dgcn_stream_t stream);

/* EdgeConv in the sparse layout.
 * Replaces gcn_lib/sparse/torch_vertex.py:106-114 (EdgConv = torch_geometric's EdgeConv with aggr 'max' around
 * MLP([2*C_in, C_out], act, norm, bias), gcn_lib/sparse/torch_nn.py:50-68).  The order is Linear -> norm -> act
 * (the dense BasicConv's is conv -> act -> norm):
 *   out_i = max over edges e = (j -> i) of act(BN(W [x_i ; x_j - x_i] + b)),   out_i = 0 without in-edges;
 * duplicate edges and self-loops count as ordinary edges.  With DGCN_NORM_BATCH_TRAIN the BatchNorm normalises
 * with the statistics of the E edge rows (written to p->batch_mean_out / batch_var_out, biased variance).
 * x (N, C_in) row-major fp32; the graph is dgcn_csr_build's rowptr (N+1) / src (E) of the edge_index (rows =
 * targets, edges in edge_index order); p: the MLP's parameters in dgcn_basic_conv (weight = the Linear's
 * (C_out, 2*C_in) weight, bn_* = the BatchNorm1d's); out (N, C_out) row-major fp32.
 * sync: dgcn_bn_sync or NULL; with DGCN_NORM_BATCH_TRAIN the statistics are those of the edge rows of every rank.
 * A rank with E = 0 still makes its reduce call.  N <= 0 is DGCN_ERR_BAD_ARG before any reduce call, so a synced
 * rank without nodes leaves its peers waiting in their all-reduce: every rank must hold at least one node.
 * N <= 65535 * 32; ws: dgcn_sparse_edge_conv_workspace_bytes(N, C_in, C_out). */
size_t dgcn_sparse_edge_conv_workspace_bytes(int64_t N, int64_t C_in, int64_t C_out);
int dgcn_sparse_edge_conv_forward(const float* x, int64_t N, int64_t C_in, const int32_t* rowptr,
                                  const int32_t* src, int64_t E, const dgcn_basic_conv* p, int64_t C_out,
                                  float* out, const dgcn_bn_sync* sync /* may be NULL */, void* ws, size_t ws_bytes,
                                  dgcn_stream_t stream);
/* Gradient of dgcn_sparse_edge_conv_forward w.r.t. x and the MLP's parameters (what torch autograd derives for the
 * reference, with the max's gradient going to the first edge in edge_index order that attains it, per node and
 * channel, as torch_scatter's scatter_max).  With DGCN_NORM_BATCH_TRAIN, p->bn_mean / p->bn_var must hold the
 * BATCH statistics the forward returned.  grad_x (N, C_in), grad_weight (C_out, 2*C_in), grad_bias (C_out),
 * grad_bn_weight / grad_bn_bias (C_out), grad_prelu (1) are OVERWRITTEN; any of them may be NULL.
 * sync: dgcn_bn_sync or NULL, as in the forward; grad_x then comes from the sums and count of every rank, the
 * parameter gradients stay this rank's.
 * ws: dgcn_sparse_edge_conv_backward_workspace_bytes(N, C_in, C_out). */
size_t dgcn_sparse_edge_conv_backward_workspace_bytes(int64_t N, int64_t C_in, int64_t C_out);
int dgcn_sparse_edge_conv_backward(const float* x, int64_t N, int64_t C_in, const int32_t* rowptr,
                                   const int32_t* src, int64_t E, const dgcn_basic_conv* p, int64_t C_out,
                                   const float* grad_out, float* grad_x, float* grad_weight, float* grad_bias,
                                   float* grad_bn_weight, float* grad_bn_bias, float* grad_prelu,
                                   const dgcn_bn_sync* sync /* may be NULL */, void* ws, size_t ws_bytes,
                                   dgcn_stream_t stream);

/* Halo packing for node-partitioned graphs (new functionality; the reference
 * has no multi-GPU sparse path, SURVEY.md 3.4): out[r,:] = x[rows[r],:].
 * x and out are of element type `dtype` (dgcn_dtype); rows are copied as is. */
int dgcn_gather_rows(int32_t dtype, const void* x, int64_t C, const int32_t* rows, int64_t R, void* out,
                     dgcn_stream_t stream);

/* ------------------------------------------------------------------------
 * Measurement hook (bench.py): when enabled, the dominant kernel of each path
 * ("knn" = the fused selection kernel(s), "aggregate" = the GENConv kernel) is
 * bracketed by CUDA events on the launch stream.  _read() synchronises those
 * events, returns the summed duration and launch count for `tag` and resets it.
 * --------------------------------------------------------------------- */
int dgcn_debug_kernel_timing(int32_t enable);
int dgcn_debug_kernel_timing_read(const char* tag, double* total_ms, int64_t* launches);

/* Measurement hook (tests): when enabled, every call that takes the tensor-core
 * kNN pre-filter synchronises its stream after the selection and adds the
 * number of queries the pre-filter could not certify (they were completed by
 * the exact fp32 kernel) and the number of queries to two counters.  _read()
 * returns and resets them.  Off by default: the synchronisation costs time. */
int dgcn_debug_tc_certification(int32_t enable);
int dgcn_debug_tc_certification_read(int64_t* uncertified, int64_t* queries);

#ifdef __cplusplus
}
#endif
#endif /* DGCN_H_ */

// Sparse path, forward: fused GENConv message + aggregate + MsgNorm + residual over a
// CSR-by-destination graph (S2/S3/S4 of SURVEY.md 2b; kernel in sparse_aggr.cuh) and the halo row gather.
#include "sparse_aggr.cuh"

namespace dgcn {

// T: float for fp32 rows, unsigned short for bf16 / fp16 rows (a row copy does not look at the values)
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ x, int C, const int32_t* __restrict__ rows,
                                   int64_t R, T* __restrict__ out) {
  constexpr int V = 16 / sizeof(T);   // elements per 16-byte vector
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  const int lane = threadIdx.x & 31;
  const T* src = x + static_cast<int64_t>(__ldg(rows + r)) * C;
  T* dst = out + r * C;
  if ((C & (V - 1)) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
    for (int c = lane * V; c < C; c += 32 * V)
      *reinterpret_cast<float4*>(dst + c) = __ldg(reinterpret_cast<const float4*>(src + c));
  } else {
    for (int c = lane; c < C; c += 32) dst[c] = __ldg(src + c);
  }
}

// Work list of the long rows: per row ceil(deg / seg_edges) (row, segment) items and one
// (row, first item, #segments) triple.  Order is arbitrary; every entry is processed independently.
static __global__ void hub_rows_kernel(const int32_t* __restrict__ rowptr, int N, int min_degree, int seg_edges,
                                int32_t* __restrict__ items, int32_t* __restrict__ item_count,
                                int32_t* __restrict__ rows, int32_t* __restrict__ row_count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int deg = rowptr[i + 1] - rowptr[i];
  if (deg < min_degree) return;
  const int nseg = (deg + seg_edges - 1) / seg_edges;
  const int base = atomicAdd(item_count, nseg);
  for (int s = 0; s < nseg; ++s) {
    items[2 * (base + s)] = i;
    items[2 * (base + s) + 1] = s;
  }
  const int r = atomicAdd(row_count, 1);
  rows[3 * r] = i;
  rows[3 * r + 1] = base;
  rows[3 * r + 2] = nseg;
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

int dgcn_csr_hub_rows(const int32_t* rowptr, int64_t N, int64_t E, int32_t min_degree, int32_t seg_edges,
                                 int32_t* items, int32_t* rows, int32_t* counts, dgcn_stream_t stream) {
  if (!rowptr || !items || !rows || !counts || N <= 0 || min_degree <= 0 || seg_edges <= 0) return DGCN_ERR_BAD_ARG;
  (void)E;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DGCN_CUDA_TRY(cudaMemsetAsync(counts, 0, 8, s));
  hub_rows_kernel<<<static_cast<unsigned>(ceil_div(N, 256)), 256, 0, s>>>(rowptr, static_cast<int>(N), min_degree,
                                                                         seg_edges, items, counts, rows, counts + 1);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

int dgcn_genconv_aggregate(const float* x_src, const float* x_dst, int64_t N, int64_t C, const int32_t* rowptr,
                           const int32_t* src, const int32_t* eid, const float* edge_attr,
                           const dgcn_genconv_params* prm, const dgcn_csr_hubs* hubs, float* out,
                           dgcn_stream_t stream) {
  return dgcn_genconv_aggregate_fused(x_src, x_dst, N, C, rowptr, src, eid, edge_attr, prm, hubs, nullptr, out, stream);
}

int dgcn_genconv_aggregate_fused(const float* x_src, const float* x_dst, int64_t N, int64_t C, const int32_t* rowptr,
                                 const int32_t* src, const int32_t* eid, const float* edge_attr,
                                 const dgcn_genconv_params* prm, const dgcn_csr_hubs* hubs,
                                 const dgcn_genconv_fusion* fus, float* out, dgcn_stream_t stream) {
  return dgcn_genconv_aggregate_fused_rows(DGCN_F32, x_src, x_dst, N, C, rowptr, src, eid, edge_attr, prm, hubs, fus,
                                           out, stream);
}

int dgcn_genconv_aggregate_fused_rows(int32_t dtype, const void* x_src, const void* x_dst, int64_t N, int64_t C,
                                      const int32_t* rowptr, const int32_t* src, const int32_t* eid,
                                      const void* edge_attr, const dgcn_genconv_params* prm,
                                      const dgcn_csr_hubs* hubs, const dgcn_genconv_fusion* fus, float* out,
                                      dgcn_stream_t stream) {
  return dgcn_genconv_aggregate_fused_keep(dtype, x_src, x_dst, N, C, rowptr, src, eid, edge_attr, prm, hubs, fus,
                                           nullptr, out, stream);
}

int dgcn_genconv_aggregate_fused_keep(int32_t dtype, const void* x_src, const void* x_dst, int64_t N, int64_t C,
                                      const int32_t* rowptr, const int32_t* src, const int32_t* eid,
                                      const void* edge_attr, const dgcn_genconv_params* prm,
                                      const dgcn_csr_hubs* hubs, const dgcn_genconv_fusion* fus,
                                      const dgcn_keep_mask* keep, float* out, dgcn_stream_t stream) {
  if (!x_src || !rowptr || !src || !prm || !out || N < 0 || C <= 0) return DGCN_ERR_BAD_ARG;
  if (dtype != DGCN_F32 && dtype != DGCN_BF16 && dtype != DGCN_F16) return DGCN_ERR_BAD_ARG;
  if (fus && ((fus->pre_scale == nullptr) != (fus->pre_shift == nullptr))) return DGCN_ERR_BAD_ARG;
  if (fus && fus->row_list && (fus->n_rows < 0 || fus->n_rows > N)) return DGCN_ERR_BAD_ARG;
  if (!x_dst && (prm->msg_norm || prm->add_residual)) return DGCN_ERR_BAD_ARG;
  if (edge_attr && !eid) return DGCN_ERR_BAD_ARG;
  if (keep && (!keep->keep_bits || keep->words_per_row < (C + 31) / 32)) return DGCN_ERR_BAD_ARG;
  if (keep && (dtype != DGCN_F32 || !fus || !fus->pre_scale || !fus->pre_relu || edge_attr))
    return DGCN_ERR_UNSUPPORTED;
  if (N == 0) return DGCN_OK;
  if (N > (1ll << 31) - 1) return DGCN_ERR_UNSUPPORTED;
  AggrArgs g{};
  g.x_src = static_cast<const float*>(x_src); g.x_dst = static_cast<const float*>(x_dst);
  g.N = static_cast<int>(N); g.C = static_cast<int>(C);
  g.rowptr = rowptr; g.src = src; g.eid = eid; g.edge_attr = static_cast<const float*>(edge_attr);
  g.aggr = prm->aggr;
  g.t = prm->t; g.t_dev = prm->t_dev; g.p = prm->p; g.p_dev = prm->p_dev; g.y = prm->y; g.y_dev = prm->y_dev;
  g.eps = prm->eps; g.msg_norm = prm->msg_norm; g.msg_scale = prm->msg_scale; g.msg_scale_dev = prm->msg_scale_dev;
  g.add_residual = prm->add_residual;
  g.raw = prm->raw_message;
  g.out = out;
  g.n_rows = static_cast<int>(N);
  g.run_hubs = 1;
  if (fus) {
    g.pre_scale = fus->pre_scale; g.pre_shift = fus->pre_shift; g.pre_relu = fus->pre_relu;
    if (fus->row_list) { g.row_list = fus->row_list; g.n_rows = static_cast<int>(fus->n_rows); }
    g.run_hubs = fus->skip_hubs ? 0 : 1;
  }
  if (keep) {
    g.keep_bits = keep->keep_bits; g.keep_words = static_cast<int>(keep->words_per_row);
    g.keep_scale = keep->keep_scale;
  }
  if (hubs && hubs->rows && hubs->items && hubs->counts && hubs->partial && hubs->min_degree > 0 &&
      hubs->seg_edges > 0) {
    g.hub_items = hubs->items; g.hub_item_count = hubs->counts; g.hub_rows = hubs->rows;
    g.hub_row_count = hubs->counts + 1; g.hub_min_degree = hubs->min_degree; g.hub_seg_edges = hubs->seg_edges;
    g.hub_partial = hubs->partial;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype != DGCN_F32) {   // half rows: 8-byte row loads (4 channels per lane), fp32 out stored as float4
    const bool rows8 = ((reinterpret_cast<uintptr_t>(x_src) | reinterpret_cast<uintptr_t>(x_dst) |
                         reinterpret_cast<uintptr_t>(edge_attr)) & 7) == 0;
    if ((C % 4) != 0 || C > 1024 || g.pre_scale || !rows8 || (reinterpret_cast<uintptr_t>(out) & 15) != 0)
      return DGCN_ERR_UNSUPPORTED;
    return launch_aggr_half(g, dtype, s);
  }
  const bool aligned = ((reinterpret_cast<uintptr_t>(x_src) | reinterpret_cast<uintptr_t>(x_dst) |
                         reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(edge_attr)) & 15) == 0;
  if ((C % 4) == 0 && aligned) {
    if (g.keep_bits) {   // pre-activation + dropout (the res+ block in training)
      if (C <= 128) return launch_aggr<float, 4, 1, true, true>(g, s);
      if (C <= 256) return launch_aggr<float, 4, 2, true, true>(g, s);
      if (C <= 512) return launch_aggr<float, 4, 4, true, true>(g, s);
      return DGCN_ERR_UNSUPPORTED;
    }
    if (g.pre_scale) {   // fused pre-activation: float4 channel blocks only
      if (C <= 128) return launch_aggr<float, 4, 1, true>(g, s);
      if (C <= 256) return launch_aggr<float, 4, 2, true>(g, s);
      if (C <= 512) return launch_aggr<float, 4, 4, true>(g, s);
      return DGCN_ERR_UNSUPPORTED;
    }
    if (C <= 128) return launch_aggr<float, 4, 1, false>(g, s);
    if (C <= 256) return launch_aggr<float, 4, 2, false>(g, s);
    if (C <= 512) return launch_aggr<float, 4, 4, false>(g, s);
    if (C <= 1024) return launch_aggr<float, 4, 8, false>(g, s);
    return DGCN_ERR_UNSUPPORTED;
  }
  if (g.pre_scale) return DGCN_ERR_UNSUPPORTED;   // C % 4 != 0 or unaligned rows: run the block unfused
  if (C <= 32) return launch_aggr<float, 1, 1, false>(g, s);
  if (C <= 64) return launch_aggr<float, 1, 2, false>(g, s);
  if (C <= 128) return launch_aggr<float, 1, 4, false>(g, s);
  if (C <= 256) return launch_aggr<float, 1, 8, false>(g, s);
  return DGCN_ERR_UNSUPPORTED;
}

int dgcn_gather_rows(const float* x, int64_t C, const int32_t* rows, int64_t R, float* out, dgcn_stream_t stream) {
  return dgcn_gather_rows_typed(DGCN_F32, x, C, rows, R, out, stream);
}

int dgcn_gather_rows_typed(int32_t dtype, const void* x, int64_t C, const int32_t* rows, int64_t R, void* out,
                           dgcn_stream_t stream) {
  if (C <= 0 || R < 0) return DGCN_ERR_BAD_ARG;
  if (dtype != DGCN_F32 && dtype != DGCN_BF16 && dtype != DGCN_F16) return DGCN_ERR_BAD_ARG;
  if (R == 0) return DGCN_OK;   // an empty halo list is legal (its tensors have null data pointers)
  if (!x || !rows || !out) return DGCN_ERR_BAD_ARG;
  const unsigned grid = static_cast<unsigned>(ceil_div(R, 8));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == DGCN_F32)
    gather_rows_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(x), static_cast<int>(C), rows, R,
                                                   static_cast<float*>(out));
  else
    gather_rows_kernel<unsigned short><<<grid, 256, 0, s>>>(static_cast<const unsigned short*>(x),
                                                            static_cast<int>(C), rows, R,
                                                            static_cast<unsigned short*>(out));
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // extern "C"

// Sparse path: the aggregation of GIN and GraphSAGE (gcn_lib/sparse/torch_vertex.py:136-205, 224-233) over the
// CSR-by-destination graph, forward and backward.  The forward is the GENConv aggregate kernel (sparse_aggr.cuh) on
// the raw source rows with a RULE for the row's own term: warp per row, float4 lanes, hub segments (bf16 / fp16
// rows: sparse_gin_sage_half.cu).  The backward is linear in the upstream gradient and does not read x: one warp per
// destination row scatters its scaled gradient row to the sources with atomics, as the raw-message backward of
// dgcn_genconv_aggregate_backward does, and adds the self term to its own row.
#include "sparse_aggr.cuh"

namespace dgcn {

template <int RULE>
static int dispatch_gin_sage(const AggrArgs& g, bool vec4, cudaStream_t s) {
  if (vec4) return launch_gin_sage_vec4<float, RULE>(g, s);
  const int C = g.C;
  if (C <= 32) launch_gin_sage<float, 1, 1, RULE>(g, s);
  else if (C <= 64) launch_gin_sage<float, 1, 2, RULE>(g, s);
  else if (C <= 128) launch_gin_sage<float, 1, 4, RULE>(g, s);
  else if (C <= 256) launch_gin_sage<float, 1, 8, RULE>(g, s);
  else if (C <= 512) launch_gin_sage<float, 1, 16, RULE>(g, s);
  else if (C <= 1024) launch_gin_sage<float, 1, 32, RULE>(g, s);
  else return DGCN_ERR_UNSUPPORTED;
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

struct GinSageBwdArgs {
  int N, C, rule;
  const int32_t* rowptr; const int32_t* src;
  const float* eps; const float* gout; float* gx;
};

// NCH channels per lane (c = lane + 32 * u).  Row i's gradient row g_i goes to every source of its edges scaled by
// 1 (GIN) or 1 / c_i (SAGE: non-self edges only), and to row i itself scaled by 1 + eps (GIN), 1 / c_i (SAGE) or
// -(c_i - 1) / c_i (relative SAGE).  SELF_LOOP: c_i is counted from the row's edges first, as in the forward.
template <int NCH, int RULE>
__global__ void __launch_bounds__(256) gin_sage_bwd_kernel(const GinSageBwdArgs g) {
  constexpr bool kLoop = RULE == RULE_SELF_LOOP;
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= g.N) return;
  const int C = g.C;
  const int beg = __ldg(g.rowptr + row), end = __ldg(g.rowptr + row + 1);
  int loops = 0;
  if (kLoop) {
    for (int e0 = beg; e0 < end; e0 += 32) {
      const int s = e0 + lane < end ? __ldg(g.src + e0 + lane) : -1;
      loops += __popc(__ballot_sync(0xffffffffu, s == row));
    }
  }
  const float cnt = static_cast<float>(end - beg - loops + 1);
  float ge[NCH], gs[NCH];   // what each edge's source receives, what row i receives
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    const int c = lane + 32 * u;
    const float gi = c < C ? __ldg(g.gout + static_cast<int64_t>(row) * C + c) : 0.f;
    if (RULE == RULE_GIN) {
      ge[u] = gi;
      gs[u] = __fmul_rn(__fadd_rn(1.f, g.eps ? __ldg(g.eps) : 0.f), gi);
    } else {
      ge[u] = __fdiv_rn(gi, cnt);
      gs[u] = g.rule == DGCN_RSAGE ? __fdiv_rn(-(cnt - 1.f) * gi, cnt) : ge[u];
    }
  }
  for (int e0 = beg; e0 < end; e0 += 32) {
    const int n = min(32, end - e0);
    const int my_src = lane < n ? __ldg(g.src + e0 + lane) : 0;
    for (int k = 0; k < n; ++k) {
      const int s = __shfl_sync(0xffffffffu, my_src, k);
      if (kLoop && s == row) continue;   // warp-uniform
#pragma unroll
      for (int u = 0; u < NCH; ++u) {
        const int c = lane + 32 * u;
        if (c < C) atomicAdd(g.gx + static_cast<int64_t>(s) * C + c, ge[u]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    const int c = lane + 32 * u;
    if (c < C) atomicAdd(g.gx + static_cast<int64_t>(row) * C + c, gs[u]);
  }
}

template <int RULE>
static void launch_gin_sage_bwd(const GinSageBwdArgs& g, cudaStream_t s) {
  const unsigned grid = static_cast<unsigned>(ceil_div(g.N, 8));
  if (g.C <= 32) gin_sage_bwd_kernel<1, RULE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 64) gin_sage_bwd_kernel<2, RULE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 128) gin_sage_bwd_kernel<4, RULE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 256) gin_sage_bwd_kernel<8, RULE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 512) gin_sage_bwd_kernel<16, RULE><<<grid, 256, 0, s>>>(g);
  else gin_sage_bwd_kernel<32, RULE><<<grid, 256, 0, s>>>(g);
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

int dgcn_gin_sage_aggregate(int32_t dtype, int32_t rule, const void* x, int64_t N, int64_t C, const int32_t* rowptr,
                            const int32_t* src, const dgcn_csr_hubs* hubs, const float* eps, float* out,
                            dgcn_stream_t stream) {
  if (!x || !rowptr || !src || !out || N < 0 || C <= 0) return DGCN_ERR_BAD_ARG;
  if (dtype != DGCN_F32 && dtype != DGCN_BF16 && dtype != DGCN_F16) return DGCN_ERR_BAD_ARG;
  if (rule != DGCN_GIN && rule != DGCN_SAGE && rule != DGCN_RSAGE) return DGCN_ERR_BAD_ARG;
  if (N == 0) return DGCN_OK;
  if (N > (1ll << 31) - 1) return DGCN_ERR_UNSUPPORTED;
  AggrArgs g{};
  g.x_src = static_cast<const float*>(x); g.x_dst = g.x_src; g.N = static_cast<int>(N); g.C = static_cast<int>(C);
  g.rowptr = rowptr; g.src = src;
  g.aggr = DGCN_AGGR_ADD; g.raw = 1;
  g.out = out;
  g.n_rows = static_cast<int>(N);
  g.run_hubs = 1;
  g.gin_eps = rule == DGCN_GIN ? eps : nullptr;
  g.relative = rule == DGCN_RSAGE;
  if (hubs && hubs->rows && hubs->items && hubs->counts && hubs->partial && hubs->min_degree > 0 &&
      hubs->seg_edges > 0) {
    g.hub_items = hubs->items; g.hub_item_count = hubs->counts; g.hub_rows = hubs->rows;
    g.hub_row_count = hubs->counts + 1; g.hub_min_degree = hubs->min_degree; g.hub_seg_edges = hubs->seg_edges;
    g.hub_partial = hubs->partial;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype != DGCN_F32) {   // half rows: 8-byte row loads (4 channels per lane), fp32 out stored as float4
    if ((C % 4) != 0 || C > 1024 || (reinterpret_cast<uintptr_t>(x) & 7) != 0 ||
        (reinterpret_cast<uintptr_t>(out) & 15) != 0)
      return DGCN_ERR_UNSUPPORTED;
    return launch_gin_sage_half(g, dtype, rule == DGCN_GIN, s);
  }
  const bool vec4 = (C % 4) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  return rule == DGCN_GIN ? dispatch_gin_sage<RULE_GIN>(g, vec4, s) : dispatch_gin_sage<RULE_SELF_LOOP>(g, vec4, s);
}

int dgcn_gin_sage_aggregate_backward(int32_t rule, int64_t N, int64_t C, const int32_t* rowptr, const int32_t* src,
                                     const float* eps, const float* grad_out, float* grad_x, dgcn_stream_t stream) {
  if (!rowptr || !src || !grad_out || !grad_x || N < 0 || C <= 0) return DGCN_ERR_BAD_ARG;
  if (rule != DGCN_GIN && rule != DGCN_SAGE && rule != DGCN_RSAGE) return DGCN_ERR_BAD_ARG;
  if (N == 0) return DGCN_OK;
  if (N > (1ll << 31) - 1 || C > 1024) return DGCN_ERR_UNSUPPORTED;
  GinSageBwdArgs g{};
  g.N = static_cast<int>(N); g.C = static_cast<int>(C); g.rule = rule;
  g.rowptr = rowptr; g.src = src; g.eps = rule == DGCN_GIN ? eps : nullptr; g.gout = grad_out; g.gx = grad_x;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rule == DGCN_GIN) launch_gin_sage_bwd<RULE_GIN>(g, s);
  else launch_gin_sage_bwd<RULE_SELF_LOOP>(g, s);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // extern "C"

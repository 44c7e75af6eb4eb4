// Sparse path, forward on bf16 / fp16 rows (dgcn_genconv_aggregate_fused_rows): the aggregate kernel of
// sparse_aggr.cuh instantiated for half-precision x_src / x_dst / edge_attr.  A launch uses the (VEC, NBLK) the
// fp32 dispatch picks for the same C, so the lane <-> channel mapping, and with it every fp32 sum (MsgNorm's
// warp-reduced norms included), is the same as on the upcast rows: the output is bit-identical.  Only the loads
// are narrower (4 channels = 8 bytes per lane instead of 16).
#include "sparse_aggr.cuh"

namespace dgcn {

template <typename T>
static int launch_half(const AggrArgs& g, cudaStream_t s) {
  if (g.C <= 128) return launch_aggr<T, 4, 1, false>(g, s);
  if (g.C <= 256) return launch_aggr<T, 4, 2, false>(g, s);
  if (g.C <= 512) return launch_aggr<T, 4, 4, false>(g, s);
  if (g.C <= 1024) return launch_aggr<T, 4, 8, false>(g, s);
  return DGCN_ERR_UNSUPPORTED;
}

int launch_aggr_half(const AggrArgs& g, int dtype, cudaStream_t stream) {
  if (dtype == DGCN_BF16) return launch_half<__nv_bfloat16>(g, stream);
  if (dtype == DGCN_F16) return launch_half<__half>(g, stream);
  return DGCN_ERR_UNSUPPORTED;
}

}  // namespace dgcn

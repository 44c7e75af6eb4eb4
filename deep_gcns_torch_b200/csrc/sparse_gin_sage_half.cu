// Sparse path, GIN / GraphSAGE forward on bf16 / fp16 rows (dgcn_gin_sage_aggregate, DGCN_BF16 / DGCN_F16): the
// RULE instantiations of the aggregate kernel (sparse_aggr.cuh) for half-precision x, launched by the same VEC 4
// ladder as fp32 rows (launch_gin_sage_vec4).  The lane <-> channel mapping, the edge order of every fp32 sum, the
// self-loop count and the self term (GIN's fl(fl(1 + eps) * x_i), SAGE's divisions) are those of the upcast rows:
// the output is bit-identical.  Only the loads are narrower (4 channels = 8 bytes per lane instead of 16).
#include "sparse_aggr.cuh"

namespace dgcn {

template <typename T>
static int launch_rule_half(const AggrArgs& g, bool gin, cudaStream_t s) {
  return gin ? launch_gin_sage_vec4<T, RULE_GIN>(g, s) : launch_gin_sage_vec4<T, RULE_SELF_LOOP>(g, s);
}

int launch_gin_sage_half(const AggrArgs& g, int dtype, bool gin, cudaStream_t stream) {
  if (dtype == DGCN_BF16) return launch_rule_half<__nv_bfloat16>(g, gin, stream);
  if (dtype == DGCN_F16) return launch_rule_half<__half>(g, gin, stream);
  return DGCN_ERR_UNSUPPORTED;
}

}  // namespace dgcn

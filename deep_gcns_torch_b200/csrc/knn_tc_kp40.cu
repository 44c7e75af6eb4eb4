// knn_tc_kernel<40, packed / unpacked>: one translation unit per list length so that the long ptxas runs
// of the register-resident insertion networks compile in parallel.
#include "knn_tc.cuh"

namespace dgcn {
int launch_knn_tc_kp40(bool packed, const TcArgs& t, dim3 grid, size_t smem, cudaStream_t stream) {
  return launch_knn_tc_inst<40>(packed, t, grid, smem, stream);
}
}  // namespace dgcn

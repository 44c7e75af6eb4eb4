// knn_tc4_kernel<20 / 32>: the multi-tile, warp-specialised tensor-core selection (knn_tc4.cuh) in its own
// translation unit (long ptxas runs of the sorting networks compile in parallel with the other kernels).
#include "knn_tc4.cuh"

namespace dgcn {
int launch_knn_tc4(int kp, const TcArgs& t, dim3 grid, cudaStream_t stream) {
  if (kp == 20) return launch_knn_tc4_inst<20>(t, grid, stream);
  if (kp == 32) return launch_knn_tc4_inst<32>(t, grid, stream);
  return DGCN_ERR_UNSUPPORTED;
}
}  // namespace dgcn

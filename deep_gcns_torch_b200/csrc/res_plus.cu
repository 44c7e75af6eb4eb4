// The res+ block in training (gcn_lib/sparse/fused.py): the dropout mask packed to bits for the aggregate's reads,
// and the backward epilogue that takes the aggregate's row gradients back through dropout, ReLU and BatchNorm to
// the block input.
#include <algorithm>

#include "common.cuh"

namespace dgcn {

// one warp per (row, 32-channel word): ballot of the lane's channel
__global__ void keep_bits_pack_kernel(const float* __restrict__ keep, int64_t N, int C, int words,
                                      int32_t* __restrict__ bits) {
  const int64_t w = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= N * words) return;
  const int lane = threadIdx.x & 31;
  const int64_t r = w / words;
  const int c = static_cast<int>(w - r * words) * 32 + lane;
  const bool kept = c < C && __ldg(keep + r * C + c) != 0.f;
  const unsigned b = __ballot_sync(0xffffffffu, kept);
  if (lane == 0) bits[w] = static_cast<int32_t>(b);
}

constexpr int kEpiRows = 128;   // rows per CTA of the g_y pass (8 warps, each row one coalesced 32-channel slice)

// thread (tx, ty) = channel blockIdx.y * 32 + tx, rows ty, ty + 8, ... of the CTA's kEpiRows; the channel's keep bit
// is bit tx of the row's word blockIdx.y
__global__ void __launch_bounds__(256) res_plus_gy_kernel(const float* __restrict__ h, int N, int C,
                                                          const float* __restrict__ pre_scale,
                                                          const float* __restrict__ pre_shift,
                                                          const int32_t* __restrict__ keep_bits, int keep_words,
                                                          float keep_scale, const float* __restrict__ mean,
                                                          const float* __restrict__ invstd, float* gsrc,
                                                          const float* __restrict__ gdst, double* sums) {
  __shared__ float red[2][8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + tx;
  const bool live = c < C;
  const float s = live ? __ldg(pre_scale + c) : 0.f, t = live ? __ldg(pre_shift + c) : 0.f;
  const float mu = (live && sums) ? __ldg(mean + c) : 0.f, is = (live && sums) ? __ldg(invstd + c) : 0.f;
  float s1 = 0.f, s2 = 0.f;
  const int r_end = min(N, static_cast<int>(blockIdx.x + 1) * kEpiRows);
  for (int r = blockIdx.x * kEpiRows + ty; r < r_end; r += 8) {
    const bool kept = keep_bits == nullptr ||
                      ((__ldg(keep_bits + static_cast<int64_t>(r) * keep_words + blockIdx.y) >> tx) & 1);
    if (!live) continue;
    const int64_t i = static_cast<int64_t>(r) * C + c;
    const float x = __ldg(h + i);
    const float z = fmaf(s, x, t);                  // the pre-activation exactly as the aggregate computed it
    const float g = gsrc[i] + (gdst ? __ldg(gdst + i) : 0.f);
    const float gy = (kept && z > 0.f) ? g * keep_scale : 0.f;   // strict >: ReLU's gradient at 0 is 0
    gsrc[i] = gy;
    s1 += gy;
    s2 = fmaf(gy, (x - mu) * is, s2);
  }
  if (!sums) return;
  red[0][ty][tx] = s1;
  red[1][ty][tx] = s2;
  __syncthreads();
  if (ty == 0 && live) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < 8; ++k) { a += red[0][k][tx]; b += red[1][k][tx]; }
    atomicAdd(sums + c, static_cast<double>(a));
    atomicAdd(sums + C + c, static_cast<double>(b));
  }
}

// gh may alias gy or gskip (element i is read before it is written, by the same thread)
__global__ void res_plus_dh_kernel(const float* gy, const float* __restrict__ h, int64_t total, int C,
                                   const float* __restrict__ a, const float* __restrict__ b,
                                   const float* __restrict__ d, const float* gskip, float* gh) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    float v = fmaf(__ldg(a + c), gy[i], gskip ? gskip[i] : 0.f);
    if (b) v = fmaf(__ldg(b + c), __ldg(h + i), v);
    if (d) v += __ldg(d + c);
    gh[i] = v;
  }
}

}  // namespace dgcn

using namespace dgcn;

extern "C" {

int dgcn_keep_bits_pack(const float* keep, int64_t N, int64_t C, int32_t* keep_bits, dgcn_stream_t stream) {
  if (N < 0 || C <= 0 || C > (1 << 30)) return DGCN_ERR_BAD_ARG;
  if (N == 0) return DGCN_OK;
  if (!keep || !keep_bits) return DGCN_ERR_BAD_ARG;
  const int words = static_cast<int>((C + 31) / 32);
  keep_bits_pack_kernel<<<static_cast<unsigned>(ceil_div(N * words, 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      keep, N, static_cast<int>(C), words, keep_bits);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

int dgcn_res_plus_backward_gy(const float* h, int64_t N, int64_t C, const float* pre_scale, const float* pre_shift,
                              const dgcn_keep_mask* keep, const float* mean, const float* invstd, float* grad_src,
                              const float* grad_dst, double* sums, dgcn_stream_t stream) {
  if (N < 0 || C <= 0 || N > (1ll << 31) - 1) return DGCN_ERR_BAD_ARG;
  if (N == 0) return DGCN_OK;
  if (!h || !pre_scale || !pre_shift || !grad_src || (sums && (!mean || !invstd))) return DGCN_ERR_BAD_ARG;
  if (keep && (!keep->keep_bits || keep->words_per_row < (C + 31) / 32)) return DGCN_ERR_BAD_ARG;
  const dim3 grid(static_cast<unsigned>(ceil_div(N, kEpiRows)), static_cast<unsigned>(ceil_div(C, 32)));
  res_plus_gy_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      h, static_cast<int>(N), static_cast<int>(C), pre_scale, pre_shift, keep ? keep->keep_bits : nullptr,
      keep ? static_cast<int>(keep->words_per_row) : 0, keep ? keep->keep_scale : 1.f, mean, invstd, grad_src,
      grad_dst, sums);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

int dgcn_res_plus_backward_dh(const float* g_y, const float* h, int64_t N, int64_t C, const float* a, const float* b,
                              const float* d, const float* grad_skip, float* grad_h, dgcn_stream_t stream) {
  if (N < 0 || C <= 0) return DGCN_ERR_BAD_ARG;
  if (N == 0) return DGCN_OK;
  if (!g_y || !a || !grad_h || (b && !h)) return DGCN_ERR_BAD_ARG;
  const int64_t total = N * C;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(ceil_div(total, 256), 8 * device_sm_count()));
  res_plus_dh_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(g_y, h, total, static_cast<int>(C), a, b, d,
                                                                         grad_skip, grad_h);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // extern "C"

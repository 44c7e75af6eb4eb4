// Sparse path, backward (S6 of SURVEY.md 2b): gradient of dgcn_genconv_aggregate w.r.t. the
// node features (source and destination roles), edge_attr and the scalars t, p, y, msg_scale -
// what torch autograd derives for gcn_lib/sparse/torch_vertex.py:62-85 +
// gcn_lib/sparse/torch_message.py:44-99.  One warp per destination row, like the forward:
// pass A recomputes the row's aggregate (running max / sums), the row-local part (MsgNorm,
// residual, degree scaling) is differentiated in registers, pass B walks the row's edges again
// and scatters d(message) to the source rows with atomics.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace dgcn {

struct AggrBwdArgs {
  // x_src / x_dst / edge_attr / gea hold rows of the kernel's element type T, everything else is fp32; typed float*
  // so that the fp32 kernels compile exactly as they did before T existed
  const float* x_src; const float* x_dst; int N, C;
  const int32_t* rowptr; const int32_t* src; const int32_t* eid; const float* edge_attr;
  int aggr;
  float t; const float* t_dev; float p; const float* p_dev; float y; const float* y_dev;
  float eps; int msg_norm; float msg_scale; const float* msg_scale_dev; int add_residual; int raw;
  int softmax_grad;
  const float* gout; float* gx_src; float* gx_dst; float* gea; float* gscalars;
  // PRE instantiations: rows are recomputed as the forward read them, pre_keep(pre_scale, pre_shift, x, pre_relu,
  // keep bit, keep_scale); without keep bits every channel is kept and keep_scale is 1
  const float* pre_scale; const float* pre_shift; int pre_relu;
  const int32_t* keep_bits; int keep_words; float keep_scale;
};

// one row element, widened exactly to fp32 / rounded to nearest even from fp32 (what Tensor.to does)
__device__ __forceinline__ float ld_row(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld_row(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
__device__ __forceinline__ float ld_row(const __half* p) { return __half2float(__ldg(p)); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// s += v with the rounding error carried in c (Kahan).  Pass A sums a whole row in one fp32 chain per lane; on a row
// of 10^6 edges a plain chain leaves the softmax sum S ~3e-3 off, and every weight e / S with it.
__device__ __forceinline__ void kahan_add(float& s, float& c, float v) {
  const float y = v - c;
  const float sum = s + y;
  c = (sum - s) - y;
  s = sum;
}

// T: element type of the rows (float, __nv_bfloat16, __half); NCH: channels per lane (c = lane + 32*u, so channel
// c's keep bit is bit `lane` of the row's word u); PRE: the forward's pre-activation (+ keep mask), fp32 rows.
template <typename T, int NCH, bool PRE = false>
__global__ void __launch_bounds__(256) genconv_aggregate_bwd_kernel(const AggrBwdArgs g) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= g.N) return;
  const int C = g.C;
  const int beg = __ldg(g.rowptr + row), end = __ldg(g.rowptr + row + 1);
  const int deg = end - beg;
  const float t = g.t_dev ? __ldg(g.t_dev) : g.t;
  const float p = g.p_dev ? __ldg(g.p_dev) : g.p;
  const int aggr = g.aggr;
  const bool softmax = aggr == DGCN_AGGR_SOFTMAX || aggr == DGCN_AGGR_SOFTMAX_SUM;
  const bool power = aggr == DGCN_AGGR_POWER || aggr == DGCN_AGGR_POWER_SUM;
  const bool scaled = aggr == DGCN_AGGR_SOFTMAX_SUM || aggr == DGCN_AGGR_POWER_SUM;
  float ps[NCH], pt[NCH];
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    const int c = lane + 32 * u;
    ps[u] = (PRE && c < C) ? __ldg(g.pre_scale + c) : 1.f;
    pt[u] = (PRE && c < C) ? __ldg(g.pre_shift + c) : 0.f;
  }
  // the activated value of channel lane + 32*u of row r (identity without PRE)
  auto act = [&](float x, int r, int u) {
    if (!PRE) return x;
    const bool kept = g.keep_bits == nullptr ||
                      ((__ldg(g.keep_bits + static_cast<int64_t>(r) * g.keep_words + u) >> lane) & 1);
    return pre_keep(ps[u], pt[u], x, g.pre_relu != 0, kept, g.keep_scale);
  };

  // ---- pass A: recompute the aggregate ---------------------------------------------------------
  float M[NCH], S[NCH], W[NCH], L[NCH];   // running max, sum exp / count, weighted sum, sum u^p ln u
  float cS[NCH], cW[NCH];                 // softmax: Kahan compensations of S and W
  int arg[NCH];
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    M[u] = -INFINITY; S[u] = 0.f; W[u] = (aggr == DGCN_AGGR_MAX) ? -INFINITY : 0.f; L[u] = 0.f; arg[u] = -1;
    cS[u] = 0.f; cW[u] = 0.f;
  }
  for (int e = beg; e < end; ++e) {
    const int s = __ldg(g.src + e);
    const int ei = g.edge_attr ? __ldg(g.eid + e) : 0;
#pragma unroll
    for (int u = 0; u < NCH; ++u) {
      const int c = lane + 32 * u;
      if (c < C) {
        float v = act(ld_row(reinterpret_cast<const T*>(g.x_src) + static_cast<int64_t>(s) * C + c), s, u);
        if (g.edge_attr) v += ld_row(reinterpret_cast<const T*>(g.edge_attr) + static_cast<int64_t>(ei) * C + c);
        const float msg = g.raw ? v : fmaxf(v, 0.f) + g.eps;
        if (softmax) {
          const float z = msg * t, d = z - M[u], ex = __expf(-fabsf(d));
          if (d > 0.f) {   // new running max: rescale the sums with their compensations, then add this edge
            S[u] *= ex; cS[u] *= ex; W[u] *= ex; cW[u] *= ex;
            kahan_add(S[u], cS[u], 1.f);
            kahan_add(W[u], cW[u], msg);
            M[u] = z;
          } else {
            kahan_add(S[u], cS[u], ex);
            kahan_add(W[u], cW[u], ex * msg);
          }
        } else if (power) {
          const float uu = fminf(fmaxf(msg, 1e-7f), 10.f);
          const float up = __powf(uu, p);
          W[u] += up;
          L[u] += up * __logf(uu);
        } else if (aggr == DGCN_AGGR_MAX) {
          if (msg > W[u]) { W[u] = msg; arg[u] = e; }
        } else {
          W[u] += msg;
        }
      }
    }
  }
  float sig = 0.f, gdeg = 1.f;
  if (scaled) {
    const float y = g.y_dev ? __ldg(g.y_dev) : g.y;
    sig = 1.f / (1.f + __expf(-y));
    gdeg = deg > 0 ? __powf(static_cast<float>(deg), sig) : 0.f;
  }
  float m0[NCH], m[NCH], Araw[NCH];
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    float r;
    Araw[u] = 0.f;
    if (softmax) r = deg > 0 ? W[u] / S[u] : 0.f;
    else if (power) {
      Araw[u] = deg > 0 ? W[u] / static_cast<float>(deg) : 0.f;
      r = __powf(fminf(fmaxf(Araw[u], 1e-7f), 10.f), 1.f / p);
    } else if (aggr == DGCN_AGGR_MEAN) r = deg > 0 ? W[u] / static_cast<float>(deg) : 0.f;
    else if (aggr == DGCN_AGGR_MAX) r = deg > 0 ? W[u] : 0.f;
    else r = W[u];
    if (lane + 32 * u >= C) r = 0.f;
    m0[u] = r;
    m[u] = r * gdeg;
  }
  // ---- row-local part: residual + MsgNorm + degree scaling ------------------------------------------
  float gh[NCH], xr[NCH];
  float n2m = 0.f, n2x = 0.f, dot_gm = 0.f;
  const bool need_x = g.msg_norm || g.add_residual;
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    const int c = lane + 32 * u;
    gh[u] = c < C ? __ldg(g.gout + static_cast<int64_t>(row) * C + c) : 0.f;
    xr[u] = (need_x && c < C) ? act(ld_row(reinterpret_cast<const T*>(g.x_dst) + static_cast<int64_t>(row) * C + c), row, u)
                              : 0.f;
    n2m = fmaf(m[u], m[u], n2m);
    n2x = fmaf(xr[u], xr[u], n2x);
    dot_gm = fmaf(gh[u], m[u], dot_gm);
  }
  float dm[NCH];
  float d_scale = 0.f, d_y = 0.f, d_t = 0.f, d_p = 0.f;
  if (g.msg_norm) {
    n2m = warp_sum(n2m);
    n2x = warp_sum(n2x);
    dot_gm = warp_sum(dot_gm);
    const float sc = g.msg_scale_dev ? __ldg(g.msg_scale_dev) : g.msg_scale;
    const float nm = fmaxf(sqrtf(n2m), 1e-12f), nx = sqrtf(n2x);
    const float f = sc * nx / nm;
    const float proj = sqrtf(n2m) > 1e-12f ? dot_gm / (nm * nm) : 0.f;   // clamped norm: no projection term
    const float dnx = nx > 0.f ? sc * dot_gm / (nm * nx) : 0.f;          // d|x| * (1/|x|)
    if (lane == 0) d_scale = nx * dot_gm / nm;
#pragma unroll
    for (int u = 0; u < NCH; ++u) {
      dm[u] = f * (gh[u] - m[u] * proj);
      xr[u] = (g.add_residual ? gh[u] : 0.f) + dnx * xr[u];               // gradient for the destination role
    }
  } else {
#pragma unroll
    for (int u = 0; u < NCH; ++u) {
      dm[u] = gh[u];
      xr[u] = g.add_residual ? gh[u] : 0.f;
    }
  }
  if (g.gx_dst) {
#pragma unroll
    for (int u = 0; u < NCH; ++u) {
      const int c = lane + 32 * u;
      if (c < C) g.gx_dst[static_cast<int64_t>(row) * C + c] = need_x ? xr[u] : 0.f;
    }
  }
  float dm0[NCH];
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    dm0[u] = dm[u] * gdeg;
    if (scaled && deg > 1) d_y += dm[u] * m0[u] * gdeg * __logf(static_cast<float>(deg)) * sig * (1.f - sig);
  }
  // power: dA and dp
  float dA[NCH];
#pragma unroll
  for (int u = 0; u < NCH; ++u) {
    dA[u] = 0.f;
    if (power && deg > 0 && lane + 32 * u < C) {
      const bool inA = Araw[u] >= 1e-7f && Araw[u] <= 10.f;
      const float A = fminf(fmaxf(Araw[u], 1e-7f), 10.f);
      if (inA) dA[u] = dm0[u] * (1.f / p) * m0[u] / A;
      const float dAdp = L[u] / static_cast<float>(deg);
      d_p += dm0[u] * m0[u] * ((inA ? dAdp / (A * p) : 0.f) - __logf(A) / (p * p));
    } else if (power && lane + 32 * u < C) {   // empty row: m0 = (1e-7)^(1/p)
      d_p += dm0[u] * m0[u] * (-__logf(1e-7f) / (p * p));
    }
  }
  // ---- pass B: d(message) per edge -> sources / edge_attr ------------------------------------------------------
  const float inv_deg = deg > 0 ? 1.f / static_cast<float>(deg) : 0.f;
  for (int e = beg; e < end; ++e) {
    const int s = __ldg(g.src + e);
    const int ei = (g.edge_attr || g.gea) ? __ldg(g.eid + e) : 0;
#pragma unroll
    for (int u = 0; u < NCH; ++u) {
      const int c = lane + 32 * u;
      if (c < C) {
        float v = act(ld_row(reinterpret_cast<const T*>(g.x_src) + static_cast<int64_t>(s) * C + c), s, u);
        if (g.edge_attr) v += ld_row(reinterpret_cast<const T*>(g.edge_attr) + static_cast<int64_t>(ei) * C + c);
        const float msg = g.raw ? v : fmaxf(v, 0.f) + g.eps;
        float dmsg;
        if (softmax) {
          const float w = __expf(msg * t - M[u]) / S[u];
          dmsg = w * dm0[u];
          if (g.softmax_grad) {
            dmsg *= 1.f + t * (msg - m0[u]);
            d_t += dm0[u] * w * msg * (msg - m0[u]);
          }
        } else if (power) {
          const bool in = msg >= 1e-7f && msg <= 10.f;
          const float uu = fminf(fmaxf(msg, 1e-7f), 10.f);
          dmsg = in ? dA[u] * inv_deg * p * __powf(uu, p - 1.f) : 0.f;
        } else if (aggr == DGCN_AGGR_MAX) {
          dmsg = (e == arg[u]) ? dm0[u] : 0.f;
        } else if (aggr == DGCN_AGGR_MEAN) {
          dmsg = dm0[u] * inv_deg;
        } else {
          dmsg = dm0[u];
        }
        const float dv = (g.raw || v > 0.f) ? dmsg : 0.f;
        if (g.gx_src) atomicAdd(g.gx_src + static_cast<int64_t>(s) * C + c, dv);
        if (g.gea) reinterpret_cast<T*>(g.gea)[static_cast<int64_t>(ei) * C + c] = from_f32<T>(dv);
      }
    }
  }
  if (g.gscalars) {
    d_t = warp_sum(d_t);
    d_p = warp_sum(d_p);
    d_y = warp_sum(d_y);
    if (lane == 0) {
      if (d_t != 0.f) atomicAdd(g.gscalars + 0, d_t);
      if (d_p != 0.f) atomicAdd(g.gscalars + 1, d_p);
      if (d_y != 0.f) atomicAdd(g.gscalars + 2, d_y);
      if (d_scale != 0.f) atomicAdd(g.gscalars + 3, d_scale);
    }
  }
}

template <typename T, bool PRE = false>
static void launch_bwd(const AggrBwdArgs& g, cudaStream_t s) {
  const unsigned grid = static_cast<unsigned>(ceil_div(g.N, 8));
  if (g.C <= 32) genconv_aggregate_bwd_kernel<T, 1, PRE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 64) genconv_aggregate_bwd_kernel<T, 2, PRE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 128) genconv_aggregate_bwd_kernel<T, 4, PRE><<<grid, 256, 0, s>>>(g);
  else if (g.C <= 256) genconv_aggregate_bwd_kernel<T, 8, PRE><<<grid, 256, 0, s>>>(g);
  else genconv_aggregate_bwd_kernel<T, 16, PRE><<<grid, 256, 0, s>>>(g);
}

}  // namespace dgcn

using namespace dgcn;

extern "C" int dgcn_genconv_aggregate_backward(int32_t dtype, const void* x_src, const void* x_dst, int64_t N,
                                               int64_t N_src, int64_t C, const int32_t* rowptr, const int32_t* src,
                                               const int32_t* eid, const void* edge_attr,
                                               const dgcn_genconv_params* prm, int32_t softmax_grad,
                                               const float* pre_scale, const float* pre_shift, int32_t pre_relu,
                                               const dgcn_keep_mask* keep, const float* grad_out, float* grad_x_src,
                                               float* grad_x_dst, void* grad_edge_attr, float* grad_scalars,
                                               dgcn_stream_t stream) {
  (void)N_src;
  if (!x_src || !rowptr || !src || !prm || !grad_out || N < 0 || C <= 0) return DGCN_ERR_BAD_ARG;
  if (dtype != DGCN_F32 && dtype != DGCN_BF16 && dtype != DGCN_F16) return DGCN_ERR_BAD_ARG;
  if (!x_dst && (prm->msg_norm || prm->add_residual)) return DGCN_ERR_BAD_ARG;
  if ((edge_attr || grad_edge_attr) && !eid) return DGCN_ERR_BAD_ARG;
  if (prm->aggr < DGCN_AGGR_SOFTMAX || prm->aggr > DGCN_AGGR_MAX) return DGCN_ERR_UNSUPPORTED;
  if ((pre_scale == nullptr) != (pre_shift == nullptr)) return DGCN_ERR_BAD_ARG;
  if (keep && (!keep->keep_bits || keep->words_per_row < (C + 31) / 32)) return DGCN_ERR_BAD_ARG;
  if (pre_scale && dtype != DGCN_F32) return DGCN_ERR_UNSUPPORTED;
  if (keep && (!pre_scale || !pre_relu || edge_attr || grad_edge_attr)) return DGCN_ERR_UNSUPPORTED;
  if (N == 0) return DGCN_OK;
  AggrBwdArgs g{};
  g.x_src = static_cast<const float*>(x_src); g.x_dst = static_cast<const float*>(x_dst);
  g.N = static_cast<int>(N); g.C = static_cast<int>(C);
  g.rowptr = rowptr; g.src = src; g.eid = eid; g.edge_attr = static_cast<const float*>(edge_attr);
  g.aggr = prm->aggr;
  g.t = prm->t; g.t_dev = prm->t_dev; g.p = prm->p; g.p_dev = prm->p_dev; g.y = prm->y; g.y_dev = prm->y_dev;
  g.eps = prm->eps; g.msg_norm = prm->msg_norm; g.msg_scale = prm->msg_scale; g.msg_scale_dev = prm->msg_scale_dev;
  g.add_residual = prm->add_residual; g.raw = prm->raw_message; g.softmax_grad = softmax_grad;
  g.gout = grad_out; g.gx_src = grad_x_src; g.gx_dst = grad_x_dst; g.gea = static_cast<float*>(grad_edge_attr); g.gscalars = grad_scalars;
  g.pre_scale = pre_scale; g.pre_shift = pre_shift; g.pre_relu = pre_relu; g.keep_scale = 1.f;
  if (keep) {
    g.keep_bits = keep->keep_bits; g.keep_words = static_cast<int>(keep->words_per_row);
    g.keep_scale = keep->keep_scale;
  }
  if (C > 512 || (dtype != DGCN_F32 && (C % 4) != 0)) return DGCN_ERR_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (pre_scale) launch_bwd<float, true>(g, s);
  else if (dtype == DGCN_BF16) launch_bwd<__nv_bfloat16>(g, s);
  else if (dtype == DGCN_F16) launch_bwd<__half>(g, s);
  else launch_bwd<float>(g, s);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

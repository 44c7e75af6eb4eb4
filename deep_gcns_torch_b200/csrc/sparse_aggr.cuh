// GENConv aggregate kernel (message + aggregate + MsgNorm + residual over a CSR-by-destination graph), shared by
// sparse_fwd.cu (fp32 rows) and sparse_fwd_half.cu (bf16 / fp16 rows, their own translation unit so the build
// compiles both halves in parallel).
//
// One warp owns one destination row; lanes own channels (VEC consecutive channels per
// lane per channel block, so a warp reads a source row as one coalesced segment).
// The softmax family is a single-pass online softmax per (row, channel): running
// max M of t*msg, running sum S of exp(t*msg - M) and running weighted sum WS.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace dgcn {

struct AggrArgs {
  // rows of x_src / x_dst / edge_attr are of the kernel's element type T (fp32, or bf16 / fp16 widened exactly in
  // registers); typed float* so that the fp32 kernels compile exactly as they did before T existed
  const float* x_src; const float* x_dst; int N, C;
  const int32_t* rowptr; const int32_t* src; const int32_t* eid; const float* edge_attr;
  int aggr;
  float t; const float* t_dev; float p; const float* p_dev; float y; const float* y_dev;
  float eps; int msg_norm; float msg_scale; const float* msg_scale_dev; int add_residual; int raw;
  float* out;
  // long rows (hubs): items = (row, segment) pairs, rows = (row, first item, #segments) triples
  const int32_t* hub_items; const int32_t* hub_item_count; const int32_t* hub_rows; const int32_t* hub_row_count;
  int hub_min_degree, hub_seg_edges; float* hub_partial;   // [item][3][C] merged (max, sum, weighted sum) states
  // block fusion (dgcn_genconv_fusion): rows are read as act(pre_scale * x + pre_shift); MODE 0 walks row_list
  const float* pre_scale; const float* pre_shift; int pre_relu;
  const int32_t* row_list; int n_rows; int run_hubs;
  // dropout folded into the pre-activation (dgcn_keep_mask; KEEP instantiations only)
  const int32_t* keep_bits; int keep_words; float keep_scale;
};


__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int VEC>
struct VecF { float v[VEC]; };

template <int VEC>
__device__ __forceinline__ VecF<VEC> load_vec(const float* p) {
  VecF<VEC> r;
  if (VEC == 4) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    r.v[0] = t.x; r.v[1 % VEC] = t.y; r.v[2 % VEC] = t.z; r.v[3 % VEC] = t.w;
  } else {
    r.v[0] = __ldg(p);
  }
  return r;
}

// 4 half-precision channels = one 8-byte load; bf16 -> fp32 and fp16 -> fp32 are exact (subnormals included)
template <int VEC>
__device__ __forceinline__ VecF<VEC> load_vec(const __nv_bfloat16* p) {
  static_assert(VEC == 4, "half rows are read 4 channels per lane");
  const uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
  VecF<VEC> r;
  r.v[0] = __uint_as_float(t.x << 16); r.v[1 % VEC] = __uint_as_float(t.x & 0xffff0000u);
  r.v[2 % VEC] = __uint_as_float(t.y << 16); r.v[3 % VEC] = __uint_as_float(t.y & 0xffff0000u);
  return r;
}

template <int VEC>
__device__ __forceinline__ VecF<VEC> load_vec(const __half* p) {
  static_assert(VEC == 4, "half rows are read 4 channels per lane");
  const uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
  VecF<VEC> r;
  r.v[0] = a.x; r.v[1 % VEC] = a.y; r.v[2 % VEC] = b.x; r.v[3 % VEC] = b.y;
  return r;
}

// x -> act(s * x + t) on the VEC channels a lane owns (identity when no pre-activation is fused)
template <int VEC>
__device__ __forceinline__ void pre_apply(VecF<VEC>& v, const float (&s)[VEC], const float (&t)[VEC], bool on, bool relu) {
  if (!on) return;
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const float z = fmaf(s[j], v.v[j], t[j]);
    v.v[j] = relu ? fmaxf(z, 0.f) : z;
  }
}

// channel owned by (lane, block blk, slot j)
template <int VEC>
__device__ __forceinline__ int chan_of(int lane, int blk, int j) { return blk * 32 * VEC + lane * VEC + j; }

// MODE 0: one warp per destination row (rows of degree >= hub_min_degree are left out when a hub list is
//         given).
// MODE 1: one CTA per (hub row, segment of hub_seg_edges edges): its 8 warps take the segment's 32-edge
//         chunks round robin, their running (max, sum, weighted sum) states are merged in a fixed order and
//         written to hub_partial.
// MODE 2: one warp per hub row: merges the row's segment states in segment order, then finishes the row
//         like MODE 0.  A power-law graph's hubs therefore neither serialise on one warp nor make the
//         result depend on scheduling.
// T: element type of the rows (float, __nv_bfloat16, __half); the arithmetic is fp32 and identical for all three.
// PRE: the block's norm -> relu is folded into the reads (dgcn_genconv_fusion); a separate instantiation so that
// the plain kernel keeps its register budget (occupancy is what hides the gather latency).
// KEEP (with PRE, fp32 rows, no edge features): dropout too - each lane loads its VEC channels' keep bits from the
// row's words next to the row itself and reads the row as pre_keep(...).
// (two CTAs per SM for KEEP: the bits' registers would not fit the 85 of three without spilling at NBLK = 2, 4)
template <typename T, int VEC, int NBLK, int AGGR, int MODE, bool PRE, bool KEEP = false>
__global__ void __launch_bounds__(256, KEEP ? 2 : (PRE ? 3 : 1)) genconv_aggregate_kernel(const AggrArgs g) {
  static_assert(!KEEP || (PRE && VEC == 4), "keep bits ride on the float4 pre-activation kernels");
  constexpr bool HUB = MODE == 1;
  __shared__ float hub_red[HUB ? 8 : 1][3][VEC][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_work = MODE == 1 ? __ldg(g.hub_item_count) : (MODE == 2 ? __ldg(g.hub_row_count) : 0);
  const int work0 = MODE == 2 ? static_cast<int>(blockIdx.x * 8 + warp) : static_cast<int>(blockIdx.x);
  const int work_step = MODE == 2 ? static_cast<int>(gridDim.x * 8) : static_cast<int>(gridDim.x);
  for (int hub_it = work0; MODE != 0 ? hub_it < n_work : hub_it == work0; hub_it += work_step) {
  int row, seg = 0, item0 = 0, nseg = 0;
  if (MODE == 0) {
    const int slot = static_cast<int>(blockIdx.x * (blockDim.x >> 5) + warp);
    if (slot >= g.n_rows) return;
    row = g.row_list ? __ldg(g.row_list + slot) : slot;
  } else if (MODE == 1) { row = __ldg(g.hub_items + 2 * hub_it); seg = __ldg(g.hub_items + 2 * hub_it + 1); }
  else { row = __ldg(g.hub_rows + 3 * hub_it); item0 = __ldg(g.hub_rows + 3 * hub_it + 1); nseg = __ldg(g.hub_rows + 3 * hub_it + 2); }
  const int C = g.C;
  constexpr bool pre = PRE;
  // relu(relu(z) + 0) = relu(z): without edge features the message's own relu covers the pre-activation's
  const bool pre_relu_now = g.pre_relu != 0 && g.edge_attr != nullptr;
  const int rbeg = __ldg(g.rowptr + row), rend = __ldg(g.rowptr + row + 1);
  const int deg = rend - rbeg;
  if (MODE == 0 && g.hub_rows != nullptr && deg >= g.hub_min_degree) return;   // the hub kernels own this row
  const int beg = MODE == 1 ? rbeg + seg * g.hub_seg_edges : rbeg;
  const int end = MODE == 1 ? min(rend, beg + g.hub_seg_edges) : (MODE == 2 ? rbeg : rend);   // MODE 2 reads no edges
  const int e_first = HUB ? beg + 32 * warp : beg, e_step = HUB ? 256 : 32;
  const float t = g.t_dev ? __ldg(g.t_dev) : g.t;
  const float p = g.p_dev ? __ldg(g.p_dev) : g.p;
  const float tl = t * 1.4426950408889634f;   // softmax in base 2
  constexpr bool kSoftmax = (AGGR == DGCN_AGGR_SOFTMAX || AGGR == DGCN_AGGR_SOFTMAX_SUM);
  constexpr bool kPower = (AGGR == DGCN_AGGR_POWER || AGGR == DGCN_AGGR_POWER_SUM);

  float m[NBLK][VEC];
#pragma unroll
  for (int blk = 0; blk < NBLK; ++blk) {
    const int cbase = chan_of<VEC>(lane, blk, 0);
    const bool live = cbase < C;   // C % VEC == 0 so a lane's VEC channels are all in or all out
    float M[VEC], S[VEC], W[VEC], ps[VEC], pt[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      ps[j] = (pre && live) ? __ldg(g.pre_scale + cbase + j) : 1.f;
      pt[j] = (pre && live) ? __ldg(g.pre_shift + cbase + j) : 0.f;
      M[j] = -INFINITY;
      S[j] = 0.f;
      W[j] = (AGGR == DGCN_AGGR_MAX) ? -INFINITY : 0.f;
    }
    if (blk * 32 * VEC < C) {   // warp-uniform: this channel block exists
      for (int e0 = e_first; e0 < end; e0 += e_step) {
        const int cnt = min(32, end - e0);
        int my_src = 0, my_eid = 0;
        if (lane < cnt) {
          my_src = __ldg(g.src + e0 + lane);
          if (g.edge_attr) my_eid = __ldg(g.eid + e0 + lane);
        }
        for (int u0 = 0; u0 < cnt; u0 += 4) {
          VecF<VEC> xv[4], ev[4];
          bool have[4];
          unsigned kb[4];   // KEEP: the lane's VEC keep bits of each edge's source row
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int s = __shfl_sync(0xffffffffu, my_src, (u0 + u) & 31);
            int ei = 0;
            if (g.edge_attr) ei = __shfl_sync(0xffffffffu, my_eid, (u0 + u) & 31);   // warp-uniform branch
            have[u] = live && u0 + u < cnt;
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
              xv[u].v[j] = 0.f;
              ev[u].v[j] = 0.f;
            }
            if (KEEP) kb[u] = 0u;
            if (have[u]) {
              xv[u] = load_vec<VEC>(reinterpret_cast<const T*>(g.x_src) + static_cast<int64_t>(s) * C + cbase);
              if (KEEP) kb[u] = static_cast<unsigned>(__ldg(g.keep_bits + static_cast<int64_t>(s) * g.keep_words +
                                                            (cbase >> 5))) >> (cbase & 31);
              if (g.edge_attr) ev[u] = load_vec<VEC>(reinterpret_cast<const T*>(g.edge_attr) + static_cast<int64_t>(ei) * C + cbase);
            }
          }
#pragma unroll
          for (int j = 0; j < VEC; ++j) {
            float msg[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              float v = xv[u].v[j];
              if (KEEP) {
                v = pre_keep(ps[j], pt[j], v, g.pre_relu != 0, (kb[u] >> j) & 1u, g.keep_scale);
              } else if (pre) {   // applied here, behind all four row loads, so that the loads stay back to back
                v = fmaf(ps[j], v, pt[j]);
                if (pre_relu_now) v = fmaxf(v, 0.f);
              }
              if (g.edge_attr) v += ev[u].v[j];
              msg[u] = g.raw ? v : fmaxf(v, 0.f) + g.eps;   // torch_vertex.py:85
            }
            if (kSoftmax) {
              // Four edges per running-max update, branch-free, 5 exp2 per 4 elements:
              // zl = msg * t * log2(e); newM = max(M, zl0..3); S = S*2^(M-newM) + sum 2^(zl-newM).
              float zl[4];
#pragma unroll
              for (int u = 0; u < 4; ++u) zl[u] = have[u] ? msg[u] * tl : -INFINITY;
              const float newM = fmaxf(fmaxf(M[j], fmaxf(zl[0], zl[1])), fmaxf(zl[2], zl[3]));
              const float sc = fast_exp2(M[j] - newM);          // M = -inf first time: 0
              const float e0 = fast_exp2(zl[0] - newM), e1 = fast_exp2(zl[1] - newM);
              const float e2 = fast_exp2(zl[2] - newM), e3 = fast_exp2(zl[3] - newM);
              S[j] = fmaf(S[j], sc, (e0 + e1) + (e2 + e3));
              W[j] = fmaf(W[j], sc, fmaf(e0, msg[0], e1 * msg[1]) + fmaf(e2, msg[2], e3 * msg[3]));
              M[j] = newM;
            } else {
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                if (have[u]) {
                  if (kPower) {
                    const float uu = fminf(fmaxf(msg[u], 1e-7f), 10.f);  // torch_message.py:69-70
                    W[j] += __powf(uu, p);
                  } else if (AGGR == DGCN_AGGR_MAX) {
                    W[j] = fmaxf(W[j], msg[u]);
                  } else {
                    W[j] += msg[u];
                  }
                }
              }
            }
          }
        }
      }
    }
    if (MODE == 1) {   // merge the 8 warps' states (warp order fixed -> deterministic), publish the segment state
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        hub_red[warp][0][j][lane] = M[j];
        hub_red[warp][1][j][lane] = S[j];
        hub_red[warp][2][j][lane] = W[j];
      }
      __syncthreads();
      if (warp == 0 && live) {
        float* part = g.hub_partial + static_cast<int64_t>(hub_it) * 3 * C;
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          float Mx = hub_red[0][0][j][lane];
          for (int w = 1; w < 8; ++w) Mx = fmaxf(Mx, hub_red[w][0][j][lane]);
          float Ss = 0.f, Ws = (AGGR == DGCN_AGGR_MAX) ? -INFINITY : 0.f;
          for (int w = 0; w < 8; ++w) {
            const float Mw = hub_red[w][0][j][lane], Sw = hub_red[w][1][j][lane], Ww = hub_red[w][2][j][lane];
            if (kSoftmax) {
              const float sc = Mw == -INFINITY ? 0.f : fast_exp2(Mw - Mx);
              Ss = fmaf(Sw, sc, Ss);
              Ws = fmaf(Ww, sc, Ws);
            } else if (AGGR == DGCN_AGGR_MAX) {
              Ws = fmaxf(Ws, Ww);
            } else {
              Ws += Ww;
            }
          }
          part[cbase + j] = Mx;
          part[C + cbase + j] = Ss;
          part[2 * C + cbase + j] = Ws;
        }
      }
      __syncthreads();
      continue;   // next channel block; the row is finished by MODE 2
    }
    if (MODE == 2 && live) {   // merge the row's segment states in segment order
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        float Mx = -INFINITY;
        for (int sg = 0; sg < nseg; ++sg) Mx = fmaxf(Mx, g.hub_partial[static_cast<int64_t>(item0 + sg) * 3 * C + cbase + j]);
        float Ss = 0.f, Ws = (AGGR == DGCN_AGGR_MAX) ? -INFINITY : 0.f;
        for (int sg = 0; sg < nseg; ++sg) {
          const float* part = g.hub_partial + static_cast<int64_t>(item0 + sg) * 3 * C;
          const float Mw = part[cbase + j], Sw = part[C + cbase + j], Ww = part[2 * C + cbase + j];
          if (kSoftmax) {
            const float sc = Mw == -INFINITY ? 0.f : fast_exp2(Mw - Mx);
            Ss = fmaf(Sw, sc, Ss);
            Ws = fmaf(Ww, sc, Ws);
          } else if (AGGR == DGCN_AGGR_MAX) {
            Ws = fmaxf(Ws, Ww);
          } else {
            Ws += Ww;
          }
        }
        M[j] = Mx;
        S[j] = Ss;
        W[j] = Ws;
      }
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      float r;
      if (kSoftmax) {
        r = deg > 0 ? W[j] / S[j] : 0.f;
      } else if (kPower) {
        float mean = deg > 0 ? W[j] / static_cast<float>(deg) : 0.f;
        mean = fminf(fmaxf(mean, 1e-7f), 10.f);                     // torch_message.py:73
        r = __powf(mean, 1.f / p);
      } else if (AGGR == DGCN_AGGR_MEAN) {
        r = deg > 0 ? W[j] / static_cast<float>(deg) : 0.f;
      } else if (AGGR == DGCN_AGGR_MAX) {
        r = deg > 0 ? W[j] : 0.f;
      } else {
        r = W[j];
      }
      m[blk][j] = live ? r : 0.f;
    }
  }
  if (AGGR == DGCN_AGGR_SOFTMAX_SUM || AGGR == DGCN_AGGR_POWER_SUM) {   // torch_message.py:60-63,77-80
    const float y = g.y_dev ? __ldg(g.y_dev) : g.y;
    const float sig = 1.f / (1.f + __expf(-y));
    const float f = deg > 0 ? __powf(static_cast<float>(deg), sig) : 0.f;
#pragma unroll
    for (int blk = 0; blk < NBLK; ++blk)
#pragma unroll
      for (int j = 0; j < VEC; ++j) m[blk][j] *= f;
  }
  if (MODE == 1) continue;   // segments only publish their state
  // MsgNorm (torch_message.py:95-99) + residual (torch_vertex.py:73)
  float xr[NBLK][VEC];
  float n2m = 0.f, n2x = 0.f;
  const bool need_x = g.msg_norm || g.add_residual;
#pragma unroll
  for (int blk = 0; blk < NBLK; ++blk) {
    const int cbase = chan_of<VEC>(lane, blk, 0);
#pragma unroll
    for (int j = 0; j < VEC; ++j) xr[blk][j] = 0.f;
    if (need_x && cbase < C) {
      VecF<VEC> xv = load_vec<VEC>(reinterpret_cast<const T*>(g.x_dst) + static_cast<int64_t>(row) * C + cbase);
      if (pre) {
        float ps[VEC], pt[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          ps[j] = __ldg(g.pre_scale + cbase + j);
          pt[j] = __ldg(g.pre_shift + cbase + j);
        }
        if (KEEP) {
          const unsigned kr = static_cast<unsigned>(__ldg(g.keep_bits + static_cast<int64_t>(row) * g.keep_words +
                                                          (cbase >> 5))) >> (cbase & 31);
#pragma unroll
          for (int j = 0; j < VEC; ++j) xv.v[j] = pre_keep(ps[j], pt[j], xv.v[j], g.pre_relu != 0, (kr >> j) & 1u,
                                                            g.keep_scale);
        } else {
          pre_apply<VEC>(xv, ps, pt, true, g.pre_relu != 0);
        }
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j) xr[blk][j] = xv.v[j];
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      n2m = fmaf(m[blk][j], m[blk][j], n2m);
      n2x = fmaf(xr[blk][j], xr[blk][j], n2x);
    }
  }
  float f = 1.f;
  if (g.msg_norm) {
    n2m = warp_sum(n2m);
    n2x = warp_sum(n2x);
    const float sc = g.msg_scale_dev ? __ldg(g.msg_scale_dev) : g.msg_scale;
    f = sqrtf(n2x) * sc / fmaxf(sqrtf(n2m), 1e-12f);
  }
#pragma unroll
  for (int blk = 0; blk < NBLK; ++blk) {
    const int cbase = chan_of<VEC>(lane, blk, 0);
    if (cbase < C) {
      float o[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) o[j] = g.add_residual ? fmaf(m[blk][j], f, xr[blk][j]) : m[blk][j] * f;
      float* dst = g.out + static_cast<int64_t>(row) * C + cbase;
      if (VEC == 4) {
        *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1 % VEC], o[2 % VEC], o[3 % VEC]);
      } else {
        dst[0] = o[0];
      }
    }
  }
  }   // hub_it
}

template <typename T, int VEC, int NBLK, bool PRE, bool KEEP = false>
static int launch_aggr(const AggrArgs& g, cudaStream_t stream) {
  const int warps = 8;
  const unsigned grid = static_cast<unsigned>(ceil_div(g.n_rows, warps));
#define DGCN_AGGR_CASE(A)                                                                   \
  case A:                                                                                   \
    if (grid) genconv_aggregate_kernel<T, VEC, NBLK, A, 0, PRE, KEEP><<<grid, warps * 32, 0, stream>>>(g); \
    if (g.hub_rows && g.run_hubs) {                                                                     \
      genconv_aggregate_kernel<T, VEC, NBLK, A, 1, PRE, KEEP><<<4 * device_sm_count(), 256, 0, stream>>>(g); \
      genconv_aggregate_kernel<T, VEC, NBLK, A, 2, PRE, KEEP><<<32, 256, 0, stream>>>(g);                 \
    }                                                                                       \
    break;
  KernelTimer timer(stream, "aggregate");
  switch (g.aggr) {
    DGCN_AGGR_CASE(DGCN_AGGR_SOFTMAX)
    DGCN_AGGR_CASE(DGCN_AGGR_SOFTMAX_SUM)
    DGCN_AGGR_CASE(DGCN_AGGR_POWER)
    DGCN_AGGR_CASE(DGCN_AGGR_POWER_SUM)
    DGCN_AGGR_CASE(DGCN_AGGR_ADD)
    DGCN_AGGR_CASE(DGCN_AGGR_MEAN)
    DGCN_AGGR_CASE(DGCN_AGGR_MAX)
    default: return DGCN_ERR_UNSUPPORTED;
  }
#undef DGCN_AGGR_CASE
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

// bf16 / fp16 rows (sparse_fwd_half.cu): VEC = 4 and the NBLK the fp32 dispatch picks for C, no pre-activation
int launch_aggr_half(const AggrArgs& g, int dtype, cudaStream_t stream);

}  // namespace dgcn

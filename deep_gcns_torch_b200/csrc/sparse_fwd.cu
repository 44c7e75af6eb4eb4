// Sparse path, forward: fused GENConv message + aggregate + MsgNorm + residual over a
// CSR-by-destination graph (S2/S3/S4 of SURVEY.md 2b) and the halo row gather.
//
// One warp owns one destination row; lanes own channels (VEC consecutive channels per
// lane per channel block, so a warp reads a source row as one coalesced segment).
// The softmax family is a single-pass online softmax per (row, channel): running
// max M of t*msg, running sum S of exp(t*msg - M) and running weighted sum WS.
#include "common.cuh"

namespace dgcn {

struct AggrArgs {
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
// PRE: the block's norm -> relu is folded into the reads (dgcn_genconv_fusion); a separate instantiation so that
// the plain kernel keeps its register budget (occupancy is what hides the gather latency).
template <int VEC, int NBLK, int AGGR, int MODE, bool PRE>
__global__ void __launch_bounds__(256, PRE ? 3 : 1) genconv_aggregate_kernel(const AggrArgs g) {
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
            if (have[u]) {
              xv[u] = load_vec<VEC>(g.x_src + static_cast<int64_t>(s) * C + cbase);
              if (g.edge_attr) ev[u] = load_vec<VEC>(g.edge_attr + static_cast<int64_t>(ei) * C + cbase);
            }
          }
#pragma unroll
          for (int j = 0; j < VEC; ++j) {
            float msg[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              float v = xv[u].v[j];
              if (pre) {   // applied here, behind all four row loads, so that the loads stay back to back
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
      VecF<VEC> xv = load_vec<VEC>(g.x_dst + static_cast<int64_t>(row) * C + cbase);
      if (pre) {
        float ps[VEC], pt[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          ps[j] = __ldg(g.pre_scale + cbase + j);
          pt[j] = __ldg(g.pre_shift + cbase + j);
        }
        pre_apply<VEC>(xv, ps, pt, true, g.pre_relu != 0);
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

template <int VEC, int NBLK, bool PRE>
static int launch_aggr(const AggrArgs& g, cudaStream_t stream) {
  const int warps = 8;
  const unsigned grid = static_cast<unsigned>(ceil_div(g.n_rows, warps));
#define DGCN_AGGR_CASE(A)                                                                   \
  case A:                                                                                   \
    if (grid) genconv_aggregate_kernel<VEC, NBLK, A, 0, PRE><<<grid, warps * 32, 0, stream>>>(g); \
    if (g.hub_rows && g.run_hubs) {                                                                     \
      genconv_aggregate_kernel<VEC, NBLK, A, 1, PRE><<<4 * device_sm_count(), 256, 0, stream>>>(g); \
      genconv_aggregate_kernel<VEC, NBLK, A, 2, PRE><<<32, 256, 0, stream>>>(g);                 \
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

__global__ void gather_rows_kernel(const float* __restrict__ x, int C, const int32_t* __restrict__ rows,
                                   int64_t R, float* __restrict__ out) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  const int lane = threadIdx.x & 31;
  const float* src = x + static_cast<int64_t>(__ldg(rows + r)) * C;
  float* dst = out + r * C;
  if ((C & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
    for (int c = lane * 4; c < C; c += 128)
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
  if (!x_src || !rowptr || !src || !prm || !out || N < 0 || C <= 0) return DGCN_ERR_BAD_ARG;
  if (fus && ((fus->pre_scale == nullptr) != (fus->pre_shift == nullptr))) return DGCN_ERR_BAD_ARG;
  if (fus && fus->row_list && (fus->n_rows < 0 || fus->n_rows > N)) return DGCN_ERR_BAD_ARG;
  if (!x_dst && (prm->msg_norm || prm->add_residual)) return DGCN_ERR_BAD_ARG;
  if (edge_attr && !eid) return DGCN_ERR_BAD_ARG;
  if (N == 0) return DGCN_OK;
  if (N > (1ll << 31) - 1) return DGCN_ERR_UNSUPPORTED;
  AggrArgs g{};
  g.x_src = x_src; g.x_dst = x_dst; g.N = static_cast<int>(N); g.C = static_cast<int>(C);
  g.rowptr = rowptr; g.src = src; g.eid = eid; g.edge_attr = edge_attr;
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
  if (hubs && hubs->rows && hubs->items && hubs->counts && hubs->partial && hubs->min_degree > 0 &&
      hubs->seg_edges > 0) {
    g.hub_items = hubs->items; g.hub_item_count = hubs->counts; g.hub_rows = hubs->rows;
    g.hub_row_count = hubs->counts + 1; g.hub_min_degree = hubs->min_degree; g.hub_seg_edges = hubs->seg_edges;
    g.hub_partial = hubs->partial;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool aligned = ((reinterpret_cast<uintptr_t>(x_src) | reinterpret_cast<uintptr_t>(x_dst) |
                         reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(edge_attr)) & 15) == 0;
  if ((C % 4) == 0 && aligned) {
    if (g.pre_scale) {   // fused pre-activation: float4 channel blocks only
      if (C <= 128) return launch_aggr<4, 1, true>(g, s);
      if (C <= 256) return launch_aggr<4, 2, true>(g, s);
      if (C <= 512) return launch_aggr<4, 4, true>(g, s);
      return DGCN_ERR_UNSUPPORTED;
    }
    if (C <= 128) return launch_aggr<4, 1, false>(g, s);
    if (C <= 256) return launch_aggr<4, 2, false>(g, s);
    if (C <= 512) return launch_aggr<4, 4, false>(g, s);
    if (C <= 1024) return launch_aggr<4, 8, false>(g, s);
    return DGCN_ERR_UNSUPPORTED;
  }
  if (g.pre_scale) return DGCN_ERR_UNSUPPORTED;   // C % 4 != 0 or unaligned rows: run the block unfused
  if (C <= 32) return launch_aggr<1, 1, false>(g, s);
  if (C <= 64) return launch_aggr<1, 2, false>(g, s);
  if (C <= 128) return launch_aggr<1, 4, false>(g, s);
  if (C <= 256) return launch_aggr<1, 8, false>(g, s);
  return DGCN_ERR_UNSUPPORTED;
}

int dgcn_gather_rows(const float* x, int64_t C, const int32_t* rows, int64_t R, float* out, dgcn_stream_t stream) {
  if (C <= 0 || R < 0) return DGCN_ERR_BAD_ARG;
  if (R == 0) return DGCN_OK;   // an empty halo list is legal (its tensors have null data pointers)
  if (!x || !rows || !out) return DGCN_ERR_BAD_ARG;
  gather_rows_kernel<<<static_cast<unsigned>(ceil_div(R, 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, static_cast<int>(C), rows, R, out);
  DGCN_LAUNCH_CHECK();
  return DGCN_OK;
}

}  // extern "C"

// Dilated kNN selection kernels (D1/D2 of SURVEY.md 2b) with the fused
// gather/max consumers (D3/D4) as epilogues.
//
//   small path  (K = k*dilation <= 32): one CTA owns 128 queries of a cloud and
//     streams all candidates through 128x128 fp32 distance tiles; a register
//     level threshold test feeds per-query candidate buffers in shared memory,
//     which warps merge into per-query sorted lists.  No (N,N) matrix exists.
//   large path  (K > 32): distance rows of an L2-sized slab of clouds are
//     written to the workspace, then one warp per row does an exact
//     bit-bisection select (in-place compaction in shared memory) of the K-th
//     key, gathers the K winners in index order and bitonic-sorts them.
//
// Ranking is on D = (|x_i|^2 + (-2 x_i.x_j)) + |x_j|^2 in fp32
// (gcn_lib/dense/torch_edge.py:40-42), ties to the smaller j.
#pragma once
#include "common.cuh"

namespace dgcn {

constexpr int MAX_KEEP = 128;       // k (kept neighbours) supported with explicit column lists
constexpr int SMALL_K_MAX = 32;     // K handled by the fused fp32 small path (above: slab path)
constexpr int LARGE_K_MAX = 2048;   // K handled by the slab path

enum EpiMode { EPI_INDEX = 0, EPI_EDGE = 1, EPI_MR = 2 };

// What happens to a query's selected neighbour list.
struct Epilogue {
  int mode;
  int64_t* edge_index;   // (2,B,N,k) or null
  int32_t* nbr;          // (B,N,k) or null
  // EPI_EDGE: pq (B,N,2*c_out) node-major: [0,c_out) = (W1-W2)x+b, [c_out,2c_out) = W2 x
  const float* pq;
  int c_out;
  float slope;
  const float* prelu;
  int norm;              // dgcn_norm
  const float* bn_w; const float* bn_b; const float* bn_m; const float* bn_v; float bn_eps;
  float* out;            // (B,c_out,N): final value, or max_l act() in train mode
  float* out_min;        // train mode: min_l act()
  float* partial;        // train mode: [n_cta][2][c_out] sum / sum of squares of act()
  // EPI_MR: xt (B,N,c_in) node-major copy of x ; r_out (B,c_in,N) = max_l x_j - x_i
  const float* xt;
  int c_in;
  float* r_out;
  // block fusion (dgcn_block_fusion; eval / no norm only): out = conv + res * res_scale, written with batch
  // stride out_sb (a channel slice of a wider buffer)
  const float* res; int64_t res_sb, res_sc; float res_scale;
  int64_t out_sb;        // batch stride of `out` in floats (c_out * N when out is contiguous)
};

// final value of output element (b, c, q): + skip connection.  Two roundings (x * scale, then the add) like the
// reference's `self.body(x) + x * self.res_scale`.
__device__ __forceinline__ float epi_res(const Epilogue& e, int b, int c, int q, float v) {
  return e.res ? __fadd_rn(v, __fmul_rn(__ldg(e.res + b * e.res_sb + c * e.res_sc + q), e.res_scale)) : v;
}

struct KnnArgs {
  const float* x; int64_t sb, sc; int B, C, N; int vec;
  const float* sq;          // (B,N) squared norms
  int K, k, dilation, has_cols, exclude_self;
  int exact_fp32;           // dgcn_dilation.flags & DGCN_KNN_EXACT_FP32 (host-side routing only)
  int tc_tile_per_cta;      // dgcn_dilation.flags & DGCN_KNN_TC_TILE_PER_CTA (host-side routing only)
  int cols[MAX_KEEP];
  Epilogue epi;
};

__device__ __forceinline__ int keep_rank(const KnnArgs& a, int l) {
  return a.has_cols ? a.cols[l] : l * a.dilation;
}

// ---- squared norms -----------------------------------------------------------
#ifndef DGCN_TEMPLATES_ONLY
__global__ void sqnorm_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N,
                              float* __restrict__ sq) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  int b = blockIdx.y;
  if (n >= N) return;
  const float* p = x + b * sb + n;
  float s = 0.f;
  for (int c = 0; c < C; ++c) {
    float v = __ldg(p + c * sc);
    s = fmaf(v, v, s);
  }
  sq[static_cast<int64_t>(b) * N + n] = s;
}
#endif  // DGCN_TEMPLATES_ONLY

// ---- per-query consumers -------------------------------------------------------
// One warp, one query (cloud b, point q, already-selected neighbour ids sel[0..k)).
// Lane owns channel c (may be >= channel count: then it idles).  Returns max / min
// over neighbours of act(P_q + Q_j) (EDGE) or of x_j (MR, min unused), plus the
// sum and sum of squares of act() for batch statistics.
__device__ __forceinline__ void edge_query(const Epilogue& e, int64_t node0, int q, const int* sel,
                                           int k, int c, float slope, float& vmax, float& vmin,
                                           float& s1, float& s2) {
  vmax = -INFINITY;
  vmin = INFINITY;
  if (c >= e.c_out) return;
  const int ld = 2 * e.c_out;
  const float p = __ldg(e.pq + (node0 + q) * ld + c);
  const float* qbase = e.pq + node0 * ld + e.c_out + c;
  int l = 0;
  if (e.norm != DGCN_NORM_BATCH_TRAIN && slope >= 0.f) {
    // no statistics needed and act is non-decreasing, like the rounded p + q: max / min commute with
    // them bit for bit, so reduce the raw gathered values and activate once
    float rmax = -INFINITY, rmin = INFINITY;
    for (; l + 8 <= k; l += 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldg(qbase + static_cast<int64_t>(sel[l + u]) * ld);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        rmax = fmaxf(rmax, v[u]);
        rmin = fminf(rmin, v[u]);
      }
    }
    for (; l < k; ++l) {
      const float v = __ldg(qbase + static_cast<int64_t>(sel[l]) * ld);
      rmax = fmaxf(rmax, v);
      rmin = fminf(rmin, v);
    }
    vmax = act_apply(p + rmax, slope);
    vmin = act_apply(p + rmin, slope);
    return;
  }
  for (; l + 8 <= k; l += 8) {   // eight independent row reads in flight per lane
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldg(qbase + static_cast<int64_t>(sel[l + u]) * ld);
#pragma unroll
    for (int u = 0; u < 8; u += 4) {
      float a0 = act_apply(p + v[u], slope), a1 = act_apply(p + v[u + 1], slope);
      float a2 = act_apply(p + v[u + 2], slope), a3 = act_apply(p + v[u + 3], slope);
      vmax = fmaxf(fmaxf(vmax, a0), fmaxf(a1, fmaxf(a2, a3)));
      vmin = fminf(fminf(vmin, a0), fminf(a1, fminf(a2, a3)));
      s1 += (a0 + a1) + (a2 + a3);
      s2 += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
  }
  for (; l + 4 <= k; l += 4) {
    float v0 = __ldg(qbase + static_cast<int64_t>(sel[l + 0]) * ld);
    float v1 = __ldg(qbase + static_cast<int64_t>(sel[l + 1]) * ld);
    float v2 = __ldg(qbase + static_cast<int64_t>(sel[l + 2]) * ld);
    float v3 = __ldg(qbase + static_cast<int64_t>(sel[l + 3]) * ld);
    float a0 = act_apply(p + v0, slope), a1 = act_apply(p + v1, slope);
    float a2 = act_apply(p + v2, slope), a3 = act_apply(p + v3, slope);
    vmax = fmaxf(fmaxf(vmax, a0), fmaxf(a1, fmaxf(a2, a3)));
    vmin = fminf(fminf(vmin, a0), fminf(a1, fminf(a2, a3)));
    s1 += (a0 + a1) + (a2 + a3);
    s2 += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
  }
  for (; l < k; ++l) {
    float a0 = act_apply(p + __ldg(qbase + static_cast<int64_t>(sel[l]) * ld), slope);
    vmax = fmaxf(vmax, a0);
    vmin = fminf(vmin, a0);
    s1 += a0;
    s2 += a0 * a0;
  }
}

__device__ __forceinline__ float mr_query(const Epilogue& e, int64_t node0, int q, const int* sel,
                                          int k, int c) {
  if (c >= e.c_in) return 0.f;
  const float* base = e.xt + node0 * e.c_in + c;
  float vmax = -INFINITY;
  int l = 0;
  for (; l + 4 <= k; l += 4) {
    float v0 = __ldg(base + static_cast<int64_t>(sel[l + 0]) * e.c_in);
    float v1 = __ldg(base + static_cast<int64_t>(sel[l + 1]) * e.c_in);
    float v2 = __ldg(base + static_cast<int64_t>(sel[l + 2]) * e.c_in);
    float v3 = __ldg(base + static_cast<int64_t>(sel[l + 3]) * e.c_in);
    vmax = fmaxf(fmaxf(vmax, v0), fmaxf(v1, fmaxf(v2, v3)));
  }
  for (; l < k; ++l) vmax = fmaxf(vmax, __ldg(base + static_cast<int64_t>(sel[l]) * e.c_in));
  return vmax - __ldg(base + static_cast<int64_t>(q) * e.c_in);
}

// eval-mode BatchNorm folded to y = s*a + t (gcn_lib/dense/torch_nn.py:28; eps 1e-5)
__device__ __forceinline__ void bn_affine(const Epilogue& e, int c, float& s, float& t) {
  s = 1.f;
  t = 0.f;
  if (e.norm == DGCN_NORM_BATCH_EVAL && c < e.c_out) {
    float inv = 1.0f / sqrtf(__ldg(e.bn_v + c) + e.bn_eps);
    s = (e.bn_w ? __ldg(e.bn_w + c) : 1.f) * inv;
    t = (e.bn_b ? __ldg(e.bn_b + c) : 0.f) - __ldg(e.bn_m + c) * s;
  }
}
__device__ __forceinline__ float epi_slope(const Epilogue& e) {
  return e.prelu ? __ldg(e.prelu) : e.slope;
}

// ---- CTA-level consumer of finished neighbour lists --------------------------------------
// list: rank-major sorted keys (list[rank*TILE + query], low 32 bits = neighbour id) of the
// TILE queries [q0, q0+TILE) of cloud b.  ok[query] == 0 (when given) marks queries whose
// list is not final (they are completed by the exact fallback kernel) - nothing is written
// for them.  sel: int [TILE][SEL_LD] scratch; stage_max / stage_min: float [32][STAGE_LD]
// (+ 2*NW*32 floats after stage_min) scratch; stage_min may alias `list` (it is only
// touched after every warp has extracted its ids).  All NW warps of the CTA must call.
constexpr int SEL_LD = 64;
constexpr int STAGE_LD = TILE + 1;         // padded staging row (bank-conflict free)

template <int NW>
__device__ __forceinline__ void cta_epilogue(const KnnArgs& a, int b, int q0, const uint64_t* list,
                                             const unsigned char* ok, int* sel, float* stage_max,
                                             float* stage_min, int cta, int sel_ld = SEL_LD) {
  const Epilogue& e = a.epi;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = a.N, k = a.k;
  constexpr int QPW = TILE / NW;            // queries per warp
  const int64_t node0 = static_cast<int64_t>(b) * N;
  for (int qq = 0; qq < QPW; ++qq) {
    const int ql = warp * QPW + qq;
    const int qg = q0 + ql;
    const bool live = qg < N && (ok == nullptr || ok[ql]);
    for (int l = lane; l < k; l += 32) {
      int idx = static_cast<int>(static_cast<uint32_t>(list[keep_rank(a, l) * TILE + ql]));
      sel[ql * sel_ld + l] = idx;
      if (live) {
        int64_t o = (node0 + qg) * k + l;
        if (e.nbr) e.nbr[o] = idx;
        if (e.edge_index) {
          e.edge_index[o] = idx;
          e.edge_index[static_cast<int64_t>(a.B) * N * k + o] = qg;
        }
      }
    }
  }
  __syncthreads();
  if (e.mode == EPI_INDEX) return;

  float* red = stage_min + 32 * STAGE_LD;                    // [NW][2][32] stat partials
  const bool train = (e.mode == EPI_EDGE && e.norm == DGCN_NORM_BATCH_TRAIN);
  const int nch = (e.mode == EPI_EDGE) ? e.c_out : e.c_in;
  const float slope = (e.mode == EPI_EDGE) ? epi_slope(e) : 0.f;
  for (int c0 = 0; c0 < nch; c0 += 32) {
    const int c = c0 + lane;
    float s1 = 0.f, s2 = 0.f, bs = 1.f, bt = 0.f;
    if (e.mode == EPI_EDGE) bn_affine(e, c, bs, bt);
    for (int qq = 0; qq < QPW; ++qq) {
      const int ql = warp * QPW + qq;
      const int qg = q0 + ql;
      if (qg >= N || (ok != nullptr && !ok[ql])) continue;
      if (e.mode == EPI_EDGE) {
        float vmax, vmin;
        edge_query(e, node0, qg, &sel[ql * sel_ld], k, c, slope, vmax, vmin, s1, s2);
        if (train) {
          stage_max[lane * STAGE_LD + ql] = vmax;
          stage_min[lane * STAGE_LD + ql] = vmin;
        } else {
          stage_max[lane * STAGE_LD + ql] = bs >= 0.f ? fmaf(bs, vmax, bt) : fmaf(bs, vmin, bt);
        }
      } else {
        stage_max[lane * STAGE_LD + ql] = mr_query(e, node0, qg, &sel[ql * sel_ld], k, c);
      }
    }
    if (train) {
      red[(warp * 2 + 0) * 32 + lane] = s1;
      red[(warp * 2 + 1) * 32 + lane] = s2;
    }
    __syncthreads();
    float* dst = (e.mode == EPI_EDGE) ? e.out : e.r_out;
    const int64_t dst_sb = (e.mode == EPI_EDGE) ? e.out_sb : static_cast<int64_t>(nch) * N;
    for (int i = tid; i < 32 * TILE; i += NW * 32) {
      const int cc = i >> 7, ql = i & (TILE - 1);
      if (c0 + cc < nch && q0 + ql < N && (ok == nullptr || ok[ql])) {
        int64_t o = (static_cast<int64_t>(b) * nch + c0 + cc) * N + q0 + ql;
        float v = stage_max[cc * STAGE_LD + ql];
        if (e.mode == EPI_EDGE && !train) v = epi_res(e, b, c0 + cc, q0 + ql, v);
        dst[b * dst_sb + static_cast<int64_t>(c0 + cc) * N + q0 + ql] = v;
        if (train) e.out_min[o] = stage_min[cc * STAGE_LD + ql];
      }
    }
    if (train && tid < 64) {
      const int which = tid >> 5, cc = tid & 31;
      float s = 0.f;
      for (int w = 0; w < NW; ++w) s += red[(w * 2 + which) * 32 + cc];
      if (c0 + cc < nch) e.partial[(static_cast<int64_t>(cta) * 2 + which) * nch + c0 + cc] = s;
    }
    __syncthreads();
  }
}


// ---- wide CTA-level consumer ------------------------------------------------------------------
// Same contract as cta_epilogue for channel counts nch in {32, 64, 128} (nch = c_out for EdgeConv,
// c_in for MRConv) and N % 8 == 0: a group of G = nch/4 lanes owns one query and reads every selected
// row as ONE float4 per lane, up to ten rows in flight, so a warp keeps 32 x 10 x 16 B outstanding
// instead of 8 x 128 B.  A group walks eight consecutive queries and then stores its four channels as
// full 32-byte sectors; no shared-memory staging.  sel: int [TILE][sel_ld]; red: float [NW][2][nch]
// (train statistics only).  Each warp only touches the sel rows of its own queries.
__host__ __device__ __forceinline__ bool epilogue_wide_ok(const KnnArgs& a) {
  const Epilogue& e = a.epi;
  if (e.mode == EPI_INDEX) return true;
  const int nch = (e.mode == EPI_EDGE) ? e.c_out : e.c_in;
  const float* rows = (e.mode == EPI_EDGE) ? e.pq : e.xt;
  return (nch == 32 || nch == 64 || nch == 128) && (a.N & 7) == 0 && (reinterpret_cast<uintptr_t>(rows) & 15) == 0;
}

// LB: neighbour rows a lane keeps in flight (one round trip to L2 per LB neighbours)
template <int NW, bool TRAIN, bool SEL_READY = false, int LB = 10>
__device__ __forceinline__ void cta_epilogue_wide(const KnnArgs& a, int b, int q0, const uint64_t* list,
                                                  const unsigned char* ok, int* sel, int sel_ld, float* red,
                                                  int cta, int tid) {
  // tid: index of the calling thread inside the NW-warp team that owns the 128 queries (threadIdx.x when the
  // team is the CTA; the multi-tile kernel passes the index inside the warpgroup).  TRAIN syncs the whole CTA.
  const Epilogue& e = a.epi;
  const int lane = tid & 31, warp = tid >> 5;
  const int N = a.N, k = a.k;
  constexpr int QPW = TILE / NW;            // queries per warp
  static_assert(QPW == 32 || QPW == 16, "wide consumer: a warp owns 32 or 16 queries (8 | QPW / (32 / G) for G = 16, 32)");
  const int64_t node0 = static_cast<int64_t>(b) * N;
  // SEL_READY: the caller has filled sel (the k neighbours of every live query, any order) and wants no index output
  for (int qq = 0; qq < (SEL_READY ? 0 : QPW); ++qq) {
    const int ql = warp * QPW + qq;
    const int qg = q0 + ql;
    const bool live = qg < N && ok[ql];
    for (int l = lane; l < k; l += 32) {
      const int idx = static_cast<int>(static_cast<uint32_t>(list[keep_rank(a, l) * TILE + ql]));
      sel[ql * sel_ld + l] = idx;
      if (live) {
        const int64_t o = (node0 + qg) * k + l;
        if (e.nbr) e.nbr[o] = idx;
        if (e.edge_index) {
          e.edge_index[o] = idx;
          e.edge_index[static_cast<int64_t>(a.B) * N * k + o] = qg;
        }
      }
    }
  }
  __syncwarp();
  if (e.mode == EPI_INDEX) return;

  const bool edge = e.mode == EPI_EDGE;
  const int nch = edge ? e.c_out : e.c_in;
  const int ld = edge ? 2 * e.c_out : e.c_in;
  const int G = nch >> 2, slots = 32 / G, per_slot = QPW / slots;     // 8 | per_slot
  const int g = lane & (G - 1), slot = lane / G;
  const float* rows = (edge ? e.pq + e.c_out : e.xt) + node0 * ld + 4 * g;   // neighbour rows (Q half / x rows)
  const float* self = (edge ? e.pq : e.xt) + node0 * ld + 4 * g;             // centre rows (P half / x rows)
  const float slope = edge ? epi_slope(e) : 0.f;
  float bs[4] = {1.f, 1.f, 1.f, 1.f}, bt[4] = {0.f, 0.f, 0.f, 0.f};
  if (edge && !TRAIN) {
#pragma unroll
    for (int i = 0; i < 4; ++i) bn_affine(e, 4 * g + i, bs[i], bt[i]);
  }
  float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
  float* dst = edge ? e.out : e.r_out;
  // eval with a non-decreasing activation (or MRConv's plain max): reduce the raw gathered values
  const bool mono = !TRAIN && (!edge || slope >= 0.f);
  const bool need_min = edge && __any_sync(0xffffffffu, bs[0] < 0.f || bs[1] < 0.f || bs[2] < 0.f || bs[3] < 0.f);
  for (int round = 0; round < per_slot; round += 8) {
    const int qlb = warp * QPW + slot * per_slot + round;    // first of eight consecutive queries
    float res[8][4], res2[TRAIN ? 8 : 1][4];
    bool all_live = true;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int ql = qlb + i, qg = q0 + ql;
      const bool live = qg < N && ok[ql];
      all_live = all_live && live;
      float vmax[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
      float vmin[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
      if (live) {
        p = __ldg(reinterpret_cast<const float4*>(self + static_cast<int64_t>(qg) * ld));
        const int* srow = sel + ql * sel_ld;
        for (int l0 = 0; l0 < k; l0 += LB) {
          float4 v[LB];
#pragma unroll
          for (int u = 0; u < LB; ++u) {
            const int idx = srow[min(l0 + u, k - 1)];
            v[u] = __ldg(reinterpret_cast<const float4*>(rows + static_cast<int64_t>(idx) * ld));
          }
          if (mono) {
            // act is non-decreasing (slope >= 0) and so is the rounded p + q: max / min commute with them,
            // bit for bit - one FMNMX per gathered element (tail duplicates are harmless)
#pragma unroll
            for (int u = 0; u < LB; ++u) {
              const float w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                vmax[c] = fmaxf(vmax[c], w[c]);
                if (need_min) vmin[c] = fminf(vmin[c], w[c]);
              }
            }
          } else {
#pragma unroll
            for (int u = 0; u < LB; ++u) {
              if (l0 + u < k) {
                const float w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
                const float pp[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                  const float av = act_apply(pp[c] + w[c], slope);
                  vmax[c] = fmaxf(vmax[c], av);
                  vmin[c] = fminf(vmin[c], av);
                  if (TRAIN) {
                    s1[c] += av;
                    s2[c] = fmaf(av, av, s2[c]);
                  }
                }
              }
            }
          }
        }
        if (mono && edge) {
          const float pp[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            vmax[c] = act_apply(pp[c] + vmax[c], slope);
            vmin[c] = act_apply(pp[c] + vmin[c], slope);
          }
        }
      }
      const float pp[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (!edge) res[i][c] = vmax[c] - pp[c];
        else if (TRAIN) {
          res[i][c] = vmax[c];
          res2[i][c] = vmin[c];
        } else {
          res[i][c] = bs[c] >= 0.f ? fmaf(bs[c], vmax[c], bt[c]) : fmaf(bs[c], vmin[c], bt[c]);
        }
      }
    }
    const int64_t dst_sb = edge ? e.out_sb : static_cast<int64_t>(nch) * N;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int64_t o = (static_cast<int64_t>(b) * nch + 4 * g + c) * N + q0 + qlb;          // contiguous (out_min)
      const int64_t oo = b * dst_sb + static_cast<int64_t>(4 * g + c) * N + q0 + qlb;        // out / r_out
      if (edge && !TRAIN && e.res) {   // skip connection of the block: eight consecutive points of one channel
#pragma unroll
        for (int i = 0; i < 8; ++i) res[i][c] = epi_res(e, b, 4 * g + c, q0 + qlb + i < N ? q0 + qlb + i : q0 + qlb, res[i][c]);
      }
      if (all_live) {
        *reinterpret_cast<float4*>(dst + oo) = make_float4(res[0][c], res[1][c], res[2][c], res[3][c]);
        *reinterpret_cast<float4*>(dst + oo + 4) = make_float4(res[4][c], res[5][c], res[6][c], res[7][c]);
        if (TRAIN) {
          *reinterpret_cast<float4*>(e.out_min + o) = make_float4(res2[0][c], res2[1][c], res2[2][c], res2[3][c]);
          *reinterpret_cast<float4*>(e.out_min + o + 4) =
              make_float4(res2[TRAIN ? 4 : 0][c], res2[TRAIN ? 5 : 0][c], res2[TRAIN ? 6 : 0][c], res2[TRAIN ? 7 : 0][c]);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int ql = qlb + i;
          if (q0 + ql < N && ok[ql]) {
            dst[oo + i] = res[i][c];
            if (TRAIN) e.out_min[o + i] = res2[TRAIN ? i : 0][c];
          }
        }
      }
    }
  }
  if (TRAIN) {
    // fixed-order reduction: slots of a warp (xor shuffles), then the NW warps in order
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      for (int o = G; o < 32; o <<= 1) {
        s1[c] += __shfl_xor_sync(0xffffffffu, s1[c], o);
        s2[c] += __shfl_xor_sync(0xffffffffu, s2[c], o);
      }
      if (slot == 0) {
        red[(warp * 2 + 0) * nch + 4 * g + c] = s1[c];
        red[(warp * 2 + 1) * nch + 4 * g + c] = s2[c];
      }
    }
    __syncthreads();
    for (int i = tid; i < 2 * nch; i += NW * 32) {
      const int which = i / nch, c = i - which * nch;
      float s = 0.f;
      for (int w = 0; w < NW; ++w) s += red[(w * 2 + which) * nch + c];
      e.partial[(static_cast<int64_t>(cta) * 2 + which) * nch + c] = s;
    }
  }
}

// ---- small path ----------------------------------------------------------------
constexpr int SM_CAP = 32;                 // candidate buffer entries per query
template <int R>
struct SmallSmem {
  static constexpr int KP = 32 * R;
  TileSmem tile;                           // 32 KB, reused as output staging
  uint64_t list[KP * TILE];                // sorted keys, rank-major: list[rank*TILE + query]
  uint64_t buf[SM_CAP * TILE];             // unsorted candidates, slot-major; reused as sel[TILE][2*SM_CAP]
  uint64_t taukey[TILE];
  float taud[TILE];
  int cnt[TILE];
};

// One thread per query: insertion of the buffered candidates into the query's sorted
// list (rank-major layout: a warp's 32 queries hit 32 different bank pairs whatever
// their ranks).  ~6 warp-instructions per insertion amortised, against ~25 for a
// warp-cooperative insert of one query at a time.
template <int R>
__device__ __forceinline__ void thread_merge(SmallSmem<R>& sm, int q, int K) {
  const int c = min(sm.cnt[q], SM_CAP);
  if (c <= 0) return;
  uint64_t tau = sm.taukey[q];
  for (int e = 0; e < c; ++e) {
    const uint64_t key = sm.buf[e * TILE + q];
    if (key < tau) {
      int i = K - 1;
      while (i > 0) {
        const uint64_t prev = sm.list[(i - 1) * TILE + q];
        if (prev < key) break;
        sm.list[i * TILE + q] = prev;
        --i;
      }
      sm.list[i * TILE + q] = key;
      tau = sm.list[(K - 1) * TILE + q];
    }
  }
  sm.taukey[q] = tau;
  sm.taud[q] = ordered_to_float(static_cast<uint32_t>(tau >> 32));
  sm.cnt[q] = 0;
}

template <int R>
__global__ void __launch_bounds__(NTHREADS, R == 1 ? 2 : 1) knn_small_kernel(const KnnArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmallSmem<R>& sm = *reinterpret_cast<SmallSmem<R>*>(smem_raw);
  constexpr int KP = SmallSmem<R>::KP;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.y, q0 = blockIdx.x * TILE;
  const int N = a.N;

  for (int i = tid; i < TILE * KP; i += NTHREADS) sm.list[i] = KEY_MAX;
  if (tid < TILE) {
    sm.taukey[tid] = KEY_MAX;
    sm.taud[tid] = __uint_as_float(0x7FC00000u);  // NaN: "!(d > tau)" admits everything
    sm.cnt[tid] = 0;
  }
  KMajor X = kmajor1(a.x + b * a.sb, a.sc, a.C, N, a.vec != 0);
  const float* sqb = a.sq + static_cast<int64_t>(b) * N;
  float sqq[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int q = q0 + tile_row(ty, i);
    sqq[i] = q < N ? __ldg(sqb + q) : 0.f;
  }
  __syncthreads();

  for (int j0 = 0; j0 < N; j0 += TILE) {
    float acc[8][8];
    tile_product(sm.tile, X, q0, X, j0, acc);
    float sqj[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int jg = j0 + tile_col(tx, j);
      sqj[j] = jg < N ? __ldg(sqb + jg) : 0.f;
    }
    // register-level threshold test; bit (i*8+j) of (pend_hi:pend_lo) = element still to be placed
    uint32_t pend_lo = 0, pend_hi = 0;
    const bool edge_tile = (j0 + TILE > N) || (q0 + TILE > N) || (a.exclude_self && j0 == q0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int ql = tile_row(ty, i);
      const float tq = sm.taud[ql];
      uint32_t bits = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float d = (sqq[i] + (-2.0f * acc[i][j])) + sqj[j];
        acc[i][j] = d;
        bits |= (!(d > tq) ? 1u : 0u) << j;
      }
      if (edge_tile) {   // ragged tiles / self exclusion: mask out what may not be selected
        const int qg = q0 + ql;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int jg = j0 + tile_col(tx, j);
          if (jg >= N || qg >= N || (a.exclude_self && jg == qg)) bits &= ~(1u << j);
        }
      }
      if (i < 4) pend_lo |= bits << (i * 8);
      else pend_hi |= bits << ((i - 4) * 8);
    }
    int more = __syncthreads_or((pend_lo | pend_hi) != 0);
    while (more) {
      if (pend_lo | pend_hi) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          uint32_t& word = (i < 4) ? pend_lo : pend_hi;
          if ((word >> ((i & 3) * 8)) & 0xFFu) {
            const int ql = tile_row(ty, i);
            const uint64_t tk = sm.taukey[ql];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const uint32_t bit = 1u << ((i & 3) * 8 + j);
              if (word & bit) {
                uint64_t key = make_key(acc[i][j], static_cast<uint32_t>(j0 + tile_col(tx, j)));
                if (key < tk) {
                  int slot = atomicAdd(&sm.cnt[ql], 1);
                  if (slot < SM_CAP) {
                    sm.buf[slot * TILE + ql] = key;
                    word &= ~bit;
                  }
                } else {
                  word &= ~bit;
                }
              }
            }
          }
        }
      }
      __syncthreads();
      if (tid < TILE) thread_merge<R>(sm, tid, a.K);
      more = __syncthreads_or((pend_lo | pend_hi) != 0);
    }
  }

  // ---- epilogue: selected ranks -> neighbour ids -> consumer ------------------------
  cta_epilogue<NTHREADS / 32>(a, b, q0, sm.list, nullptr, reinterpret_cast<int*>(sm.buf),
                              reinterpret_cast<float*>(&sm.tile), reinterpret_cast<float*>(sm.list) /* after sel */,
                              blockIdx.y * gridDim.x + blockIdx.x);
}

// ---- large path ------------------------------------------------------------------
// distance rows of clouds [b0, b0+nb) into ws rows (row = (b-b0)*N + q, ld = ldd)
#ifndef DGCN_TEMPLATES_ONLY
__global__ void __launch_bounds__(NTHREADS, 2)
    dist_rows_kernel(const KnnArgs a, int b0, float* __restrict__ drows, int ldd) {
  __shared__ TileSmem ts;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = b0 + blockIdx.z, q0 = blockIdx.y * TILE, j0 = blockIdx.x * TILE;
  const int N = a.N;
  KMajor X = kmajor1(a.x + b * a.sb, a.sc, a.C, N, a.vec != 0);
  float acc[8][8];
  tile_product(ts, X, q0, X, j0, acc);
  const float* sqb = a.sq + static_cast<int64_t>(b) * N;
  float sqj[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int jg = j0 + tile_col(tx, j);
    sqj[j] = jg < N ? __ldg(sqb + jg) : 0.f;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int qg = q0 + tile_row(ty, i);
    if (qg >= N) continue;
    const float sqq = __ldg(sqb + qg);
    float* row = drows + (static_cast<int64_t>(blockIdx.z) * N + qg) * ldd;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int jg = j0 + tile_col(tx, h * 4);
      float4 v;
      v.x = (sqq + (-2.0f * acc[i][h * 4 + 0])) + sqj[h * 4 + 0];
      v.y = (sqq + (-2.0f * acc[i][h * 4 + 1])) + sqj[h * 4 + 1];
      v.z = (sqq + (-2.0f * acc[i][h * 4 + 2])) + sqj[h * 4 + 2];
      v.w = (sqq + (-2.0f * acc[i][h * 4 + 3])) + sqj[h * 4 + 3];
      if (jg + 3 < ldd) {
        *reinterpret_cast<float4*>(row + jg) = v;   // ldd % 4 == 0, pad columns are never read
      }
    }
  }
}
#endif  // DGCN_TEMPLATES_ONLY

// warp-level bitonic sort of n (power of two) 64-bit keys in shared memory
__device__ __forceinline__ void warp_bitonic_sort(uint64_t* s, int n, int lane) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = lane; t < (n >> 1); t += 32) {
        int i = ((t & ~(stride - 1)) << 1) | (t & (stride - 1));
        int j = i | stride;
        uint64_t va = s[i], vb = s[j];
        bool up = ((i & size) == 0);
        if ((va > vb) == up) {
          s[i] = vb;
          s[j] = va;
        }
      }
      __syncwarp();
    }
  }
}

// Per-row consumer shared by the slab kernels: sk holds the row's sorted keys (ascending), sel is a
// k-entry scratch.  Writes the selected neighbour ids and runs the fused EdgeConv / MRConv consumer.
// sk == nullptr: sel already holds the k selected neighbour ids.
__device__ __forceinline__ void row_consume(const KnnArgs& a, int b, int q, const uint64_t* sk, int* sel, int lane) {
  const int N = a.N, k = a.k;
  const Epilogue& e = a.epi;
  const int64_t node0 = static_cast<int64_t>(b) * N;
  for (int l = lane; l < k; l += 32) {
    int idx = sk ? static_cast<int>(static_cast<uint32_t>(sk[keep_rank(a, l)])) : sel[l];
    sel[l] = idx;
    int64_t o = (node0 + q) * k + l;
    if (e.nbr) e.nbr[o] = idx;
    if (e.edge_index) {
      e.edge_index[o] = idx;
      e.edge_index[static_cast<int64_t>(a.B) * N * k + o] = q;
    }
  }
  __syncwarp();
  if (e.mode == EPI_INDEX) return;
  if (e.mode == EPI_EDGE) {
    const float slope = epi_slope(e);
    const bool train = e.norm == DGCN_NORM_BATCH_TRAIN;
    for (int c0 = 0; c0 < e.c_out; c0 += 32) {
      const int c = c0 + lane;
      float vmax, vmin, s1 = 0.f, s2 = 0.f, bs, bt;
      bn_affine(e, c, bs, bt);
      edge_query(e, node0, q, sel, k, c, slope, vmax, vmin, s1, s2);
      if (c < e.c_out) {
        int64_t o = (static_cast<int64_t>(b) * e.c_out + c) * N + q;
        const int64_t oo = b * e.out_sb + static_cast<int64_t>(c) * N + q;
        if (train) {
          e.out[oo] = vmax;
          e.out_min[o] = vmin;
          // one partial slot per query row: [row][2][c_out]
          e.partial[(static_cast<int64_t>(node0 + q) * 2 + 0) * e.c_out + c] = s1;
          e.partial[(static_cast<int64_t>(node0 + q) * 2 + 1) * e.c_out + c] = s2;
        } else {
          e.out[oo] = epi_res(e, b, c, q, bs >= 0.f ? fmaf(bs, vmax, bt) : fmaf(bs, vmin, bt));
        }
      }
    }
  } else {
    for (int c0 = 0; c0 < e.c_in; c0 += 32) {
      const int c = c0 + lane;
      float r = mr_query(e, node0, q, sel, k, c);
      if (c < e.c_in) e.r_out[(static_cast<int64_t>(b) * e.c_in + c) * N + q] = r;
    }
  }
}

// One warp per query row: exact K smallest (key = ordered distance, index), sorted.
// dynamic smem per warp: keys[nkeys] (u32) | sk[KP] (u64) | sel[k] (int)
// With row_list != null the kernel instead completes the rows listed there (rows the sampled fast
// kernel could not bound), grid-striding over *row_count entries.
#ifndef DGCN_TEMPLATES_ONLY
__global__ void select_rows_kernel(const KnnArgs a, int b0, int nb, const float* __restrict__ drows,
                                   int ldd, int KP, int nkeys, int warps_per_cta, const int* __restrict__ row_list,
                                   const int* __restrict__ row_count) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int N = a.N, K = a.K, k = a.k;
  const size_t per_warp = static_cast<size_t>(KP) * 8 + static_cast<size_t>(nkeys) * 4 + static_cast<size_t>((k + 31) / 32 * 32) * 4;
  unsigned char* mine = smem_raw + per_warp * warp;
  uint64_t* sk = reinterpret_cast<uint64_t*>(mine);
  uint32_t* keys = reinterpret_cast<uint32_t*>(mine + static_cast<size_t>(KP) * 8);
  int* sel = reinterpret_cast<int*>(mine + static_cast<size_t>(KP) * 8 + static_cast<size_t>(nkeys) * 4);

  const int64_t total_rows = row_list ? static_cast<int64_t>(*row_count) : static_cast<int64_t>(nb) * N;
  for (int64_t it = static_cast<int64_t>(blockIdx.x) * warps_per_cta + warp; it < total_rows;
       it += static_cast<int64_t>(gridDim.x) * warps_per_cta) {
  const int64_t row = row_list ? row_list[it] : it;
  const int b = b0 + static_cast<int>(row / N), q = static_cast<int>(row % N);
  const float* drow = drows + row * ldd;

  // 1. ordered keys of the row + which bits vary at all
  uint32_t vand = 0xFFFFFFFFu, vor = 0u;
  for (int i = lane; i < N; i += 32) {
    uint32_t key = float_to_ordered(__ldg(drow + i));
    if (a.exclude_self && i == q) key = 0xFFFFFFFFu;
    keys[i] = key;
    vand &= key;
    vor |= key;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vand &= __shfl_xor_sync(0xffffffffu, vand, o);
    vor |= __shfl_xor_sync(0xffffffffu, vor, o);
  }
  __syncwarp();
  // 2. bit bisection with in-place compaction: afterwards every active key equals T,
  //    and `need` of them (lowest indices) belong to the K smallest.
  uint32_t vary = vand ^ vor;
  int n = N, need = K;
  uint32_t T = vand;   // bits common to all keys
  for (int bit = 31; bit >= 0 && n > 0; --bit) {
    if (!((vary >> bit) & 1u)) continue;
    int c0 = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      int i = i0 + lane;
      bool z = (i < n) && !((keys[i] >> bit) & 1u);
      c0 += __popc(__ballot_sync(0xffffffffu, z));
    }
    const bool keep_zero = need <= c0;
    if (!keep_zero) {
      need -= c0;
      T |= (1u << bit);
    } else {
      T &= ~(1u << bit);
    }
    if (c0 == 0 || c0 == n) continue;   // nothing to drop
    int w = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      int i = i0 + lane;
      uint32_t key = (i < n) ? keys[i] : 0u;
      bool keep = (i < n) && ((((key >> bit) & 1u) == 0u) == keep_zero);
      unsigned m = __ballot_sync(0xffffffffu, keep);
      __syncwarp();
      if (keep) keys[w + __popc(m & ((1u << lane) - 1u))] = key;
      w += __popc(m);
      __syncwarp();
    }
    n = w;
  }
  // 3. gather the K winners in index order
  int wl = 0, we = 0;   // running counts: taken so far (all) / equal-to-T taken
  for (int i0 = 0; i0 < N; i0 += 32) {
    int i = i0 + lane;
    uint32_t key = 0xFFFFFFFFu;
    float d = 0.f;
    if (i < N) {
      d = __ldg(drow + i);
      key = float_to_ordered(d);
      if (a.exclude_self && i == q) key = 0xFFFFFFFFu;
    }
    bool less = (i < N) && key < T;
    bool eq = (i < N) && key == T && !(a.exclude_self && i == q);
    unsigned me = __ballot_sync(0xffffffffu, eq);
    int eq_rank = we + __popc(me & ((1u << lane) - 1u));
    bool take = less || (eq && eq_rank < need);
    unsigned mt = __ballot_sync(0xffffffffu, take);
    if (take) sk[wl + __popc(mt & ((1u << lane) - 1u))] = (static_cast<uint64_t>(key) << 32) | static_cast<uint32_t>(i);
    wl += __popc(mt);
    we += __popc(me);
  }
  for (int i = wl + lane; i < KP; i += 32) sk[i] = KEY_MAX;
  __syncwarp();
  // 4. sort, 5. consume
  warp_bitonic_sort(sk, KP, lane);
  row_consume(a, b, q, sk, sel, lane);
  __syncwarp();
  }
}
#endif  // DGCN_TEMPLATES_ONLY

// Fast variant: a 128-key sample of the row bounds the K-th distance from above, one pass compacts
// every key below that bound (in index order) into shared memory, a bitonic sort of the next power of
// two finishes.  Exact whenever the compacted set holds >= K and <= CAP keys; other rows go to a list
// that select_rows_kernel completes.  dynamic smem per warp: sk[CAP] (u64) | sel[k] (int).
#ifndef DGCN_TEMPLATES_ONLY
__global__ void select_rows_fast_kernel(const KnnArgs a, int b0, int nb, const float* __restrict__ drows, int ldd,
                                        int CAP, int sample_rank, int warps_per_cta, int* __restrict__ row_count,
                                        int* __restrict__ row_list) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int N = a.N, K = a.K, k = a.k;
  const size_t per_warp = static_cast<size_t>(CAP) * 8 + static_cast<size_t>((k + 31) / 32 * 32) * 4 + 2560;
  unsigned char* mine = smem_raw + per_warp * warp;
  uint64_t* sk = reinterpret_cast<uint64_t*>(mine);
  int* sel = reinterpret_cast<int*>(mine + static_cast<size_t>(CAP) * 8);
  const int64_t row = static_cast<int64_t>(blockIdx.x) * warps_per_cta + warp;
  if (row >= static_cast<int64_t>(nb) * N) return;   // whole warp exits together
  const int b = b0 + static_cast<int>(row / N), q = static_cast<int>(row % N);
  const float* drow = drows + row * ldd;
  // 1. sample 128 keys spread over the row, sort them, take the sample_rank-th as the bound.  The sort runs in
  //    registers: element e = 32 u + lane lives in smp[u] of lane `lane`; exchange distances below 32 are warp
  //    shuffles, 32 and 64 are register pairs (a shared-memory bitonic sort of these 128 keys was a third of this
  //    kernel's time, all of it shared-memory latency between dependent stages).
  uint32_t smp[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int s = lane + 32 * u;
    const int i = static_cast<int>((static_cast<int64_t>(s) * N) >> 7);
    uint32_t key = float_to_ordered(__ldg(drow + i));
    if (a.exclude_self && i == q) key = 0xFFFFFFFFu;
    smp[u] = key;
  }
  // the first 128 distances of the row: in flight under the sample sort
  float first[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) first[u] = (u * 32 + lane < N) ? __ldg(drow + u * 32 + lane) : 0.f;
#pragma unroll
  for (int kk = 2; kk <= 128; kk <<= 1) {
#pragma unroll
    for (int j = kk >> 1; j > 0; j >>= 1) {
      if (j < 32) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const uint32_t other = __shfl_xor_sync(0xffffffffu, smp[u], j);
          const bool up = (((32 * u + lane) & kk) == 0);      // ascending block
          const bool lower = (lane & j) == 0;                   // this element is the lower index of its pair
          smp[u] = (lower == up) ? min(smp[u], other) : max(smp[u], other);
        }
      } else {
        const int jr = j >> 5;                                  // partner register: u ^ jr, same lane
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if ((u & jr) == 0) {
            const bool up = (((32 * u) & kk) == 0);
            const uint32_t lo = min(smp[u], smp[u ^ jr]), hi = max(smp[u], smp[u ^ jr]);
            smp[u] = up ? lo : hi;
            smp[u ^ jr] = up ? hi : lo;
          }
        }
      }
    }
  }
  // lane l now holds the sorted samples l, l+32, l+64, l+96
  // 2. compaction in index order of every distance <= bound; if the sample misjudged the row (too few or too
  //    many below the bound) move the bound along the sorted sample and try again.  The pass is the bulk of
  //    this kernel's instructions, so it works on the raw floats: one FSETP against the bound (a float compare
  //    admits the same set as the ordered-key compare except that -0 and +0 tie, which only widens the superset;
  //    NaN never passes), the entry is stored as (float bits, index) and converted to an ordered key afterwards,
  //    for the ~K..2K survivors only.
  const int q_self = a.exclude_self ? q : -1;
  int w = 0, rank = sample_rank, lo_rank = -1, hi_rank = 128;   // lo_rank: too few, hi_rank: too many
  bool ok = false;
  const bool full_groups = (N & 127) == 0;
  for (int attempt = 0; attempt < 6 && !ok; ++attempt) {
    uint32_t bound = __shfl_sync(0xffffffffu, smp[0], rank & 31);
    if ((rank >> 5) == 1) bound = __shfl_sync(0xffffffffu, smp[1], rank & 31);
    if ((rank >> 5) == 2) bound = __shfl_sync(0xffffffffu, smp[2], rank & 31);
    if ((rank >> 5) == 3) bound = __shfl_sync(0xffffffffu, smp[3], rank & 31);
    const float bound_f = ordered_to_float(bound);
    const unsigned lt_mask = (1u << lane) - 1u;
    w = 0;
    float nxt[4];                        // the next 128 distances are in flight while these are compacted
    if (attempt == 0) {
#pragma unroll
      for (int u = 0; u < 4; ++u) nxt[u] = first[u];             // issued before the sample sort
    } else {
#pragma unroll
      for (int u = 0; u < 4; ++u) nxt[u] = (u * 32 + lane < N) ? __ldg(drow + u * 32 + lane) : 0.f;
    }
    for (int i0 = 0; i0 < N; i0 += 128) {
      float cur[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) cur[u] = nxt[u];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + 128 + u * 32 + lane;
        if (i < N) nxt[u] = __ldg(drow + i);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * 32 + lane;
        bool take = cur[u] <= bound_f && i != q_self;
        if (!full_groups) take = take && i < N;
        const unsigned m = __ballot_sync(0xffffffffu, take);
        const int pos = w + __popc(m & lt_mask);
        if (take && pos < CAP) sk[pos] = (static_cast<uint64_t>(__float_as_uint(cur[u])) << 32) | static_cast<uint32_t>(i);
        w += __popc(m);
      }
    }
    if (w < K) {
      lo_rank = rank;
      rank = min(127, max(rank + 1, (rank * 3) / 2 + 1));
      if (rank >= hi_rank) rank = hi_rank - 1;
      if (rank <= lo_rank) break;          // bracket closed (massive ties): exact kernel
    } else if (w > CAP) {
      hi_rank = rank;
      rank = (lo_rank + rank) / 2;
      if (rank <= lo_rank) break;
    } else {
      ok = true;
    }
    __syncwarp();
  }
  if (ok) {   // raw float bits -> ordered keys (the survivors are never NaN: the compare rejects it)
    for (int i = lane; i < w; i += 32) {
      const uint64_t e = sk[i];
      sk[i] = (static_cast<uint64_t>(float_to_ordered(__uint_as_float(static_cast<uint32_t>(e >> 32)))) << 32) |
              static_cast<uint32_t>(e);
    }
    __syncwarp();
  }
  if (!ok) {   // leave the row to the exact bisection kernel
    if (lane == 0) row_list[atomicAdd(row_count, 1)] = static_cast<int>(row);
    return;
  }
  if (k > 64) {   // many kept ranks: plain sort of everything below the bound
    int KP = 128;
    while (KP < w) KP <<= 1;
    if (KP > CAP) {
      if (lane == 0) row_list[atomicAdd(row_count, 1)] = static_cast<int>(row);
      return;
    }
    for (int i = w + lane; i < KP; i += 32) sk[i] = KEY_MAX;
    __syncwarp();
    warp_bitonic_sort(sk, KP, lane);
    row_consume(a, b, q, sk, sel, lane);
    return;
  }
  // 3. multi-select: only the k ranks keep_rank(l) of the K smallest are wanted (dilation keeps every d-th).
  //    Histogram the w compacted keys over 256 distance bins between the smallest sample and the bound,
  //    find the bins holding wanted ranks, compact those bins' keys in place, sort only them.
  int* hist = sel + (k + 31) / 32 * 32;       // [256] keys per bin, then reused: keys in UNMARKED bins below
  int* pre = hist + 256;                      // [257] exclusive prefix of hist
  unsigned char* mark = reinterpret_cast<unsigned char*>(pre + 260);   // [256]
  const float dlo = ordered_to_float(__shfl_sync(0xffffffffu, smp[0], 0));
  const float dhi = ordered_to_float(__shfl_sync(0xffffffffu, rank < 32 ? smp[0] : rank < 64 ? smp[1] : rank < 96 ? smp[2] : smp[3], rank & 31));
  const float scale = dhi > dlo ? 255.99f / (dhi - dlo) : 0.f;
  auto bin_of = [&](uint64_t key) {
    const float d = ordered_to_float(static_cast<uint32_t>(key >> 32));
    const float t = (d - dlo) * scale;                 // monotone in d; NaN / negative -> bin 0
    return t > 0.f ? min(255, static_cast<int>(t)) : 0;
  };
  for (int i = lane; i < 256; i += 32) {
    hist[i] = 0;
    mark[i] = 0;
  }
  __syncwarp();
  for (int i = lane; i < w; i += 32) atomicAdd(&hist[bin_of(sk[i])], 1);
  __syncwarp();
  {   // exclusive prefix: lane owns bins [8 lane, 8 lane + 8)
    int loc[8], sum = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      loc[u] = sum;
      sum += hist[lane * 8 + u];
    }
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    const int base = inc - sum;
#pragma unroll
    for (int u = 0; u < 8; ++u) pre[lane * 8 + u] = base + loc[u];
    if (lane == 31) pre[256] = inc;
  }
  __syncwarp();
  // bin of every wanted rank (binary search: last b with pre[b] <= r)
  int mybin[2] = {0, 0};
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int l = lane + 32 * j;
    if (l < k) {
      const int r = keep_rank(a, l);
      int lo = 0, hi = 256;            // pre[lo] <= r < pre[hi]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (pre[mid] <= r) lo = mid; else hi = mid;
      }
      mybin[j] = lo;
      mark[lo] = 1;
    }
  }
  __syncwarp();
  {   // hist <- number of keys in unmarked bins below b (exclusive prefix over unmarked bins)
    int loc[8], sum = 0;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      loc[u] = sum;
      sum += mark[lane * 8 + u] ? 0 : hist[lane * 8 + u];
    }
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    const int base = inc - sum;
    __syncwarp();
#pragma unroll
    for (int u = 0; u < 8; ++u) hist[lane * 8 + u] = base + loc[u];
  }
  __syncwarp();
  // in-place compaction of the keys of marked bins (write position never passes the read position)
  int T = 0;
  for (int i0 = 0; i0 < w; i0 += 32) {
    const int i = i0 + lane;
    uint64_t key = KEY_MAX;
    bool take = false;
    if (i < w) {
      key = sk[i];
      take = mark[bin_of(key)] != 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, take);
    __syncwarp();
    if (take) sk[T + __popc(m & ((1u << lane) - 1u))] = key;
    T += __popc(m);
  }
  int TP = 32;
  while (TP < T) TP <<= 1;
  if (TP > CAP) {   // (massive ties inside the wanted bins) no room to pad the sort: exact kernel
    if (lane == 0) row_list[atomicAdd(row_count, 1)] = static_cast<int>(row);
    return;
  }
  __syncwarp();
  for (int i = T + lane; i < TP; i += 32) sk[i] = KEY_MAX;
  __syncwarp();
  warp_bitonic_sort(sk, TP, lane);
  // rank r sits at position r - (#keys in unmarked bins below its bin) of the sorted marked keys
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int l = lane + 32 * j;
    if (l < k) sel[l] = static_cast<int>(static_cast<uint32_t>(sk[keep_rank(a, l) - hist[mybin[j]]]));
  }
  __syncwarp();
  row_consume(a, b, q, nullptr, sel, lane);
}
#endif  // DGCN_TEMPLATES_ONLY

}  // namespace dgcn

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
  float* partial;        // train mode: [n_cta][3][c_out] statistics of act() (common.cuh, BnMoments)
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
__global__ void sqnorm_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C, int N, float* __restrict__ sq);

// ---- per-query consumers -------------------------------------------------------
// One warp, one query (cloud b, point q, already-selected neighbour ids sel[0..k)).
// Lane owns channel c (may be >= channel count: then it idles).  Returns max / min
// over neighbours of act(P_q + Q_j) (EDGE) or of x_j (MR, min unused); in train mode
// act() also goes into the batch statistics st.
__device__ __forceinline__ void edge_query(const Epilogue& e, int64_t node0, int q, const int* sel,
                                           int k, int c, float slope, float& vmax, float& vmin, BnAcc& st) {
  vmax = -INFINITY;
  vmin = INFINITY;
  if (c >= e.c_out) return;
  const int ld = 2 * e.c_out;
  const float p = __ldg(e.pq + (node0 + q) * ld + c);
  const float* qbase = e.pq + node0 * ld + e.c_out + c;
  int l = 0;
  const bool train = e.norm == DGCN_NORM_BATCH_TRAIN;
  if (!train && slope >= 0.f) {
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
      if (train) {
        bn_acc_add(st, a0);
        bn_acc_add(st, a1);
        bn_acc_add(st, a2);
        bn_acc_add(st, a3);
      }
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
    if (train) {
      bn_acc_add(st, a0);
      bn_acc_add(st, a1);
      bn_acc_add(st, a2);
      bn_acc_add(st, a3);
    }
  }
  for (; l < k; ++l) {
    float a0 = act_apply(p + __ldg(qbase + static_cast<int64_t>(sel[l]) * ld), slope);
    vmax = fmaxf(vmax, a0);
    vmin = fminf(vmin, a0);
    if (train) bn_acc_add(st, a0);
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

  BnMoments* red = reinterpret_cast<BnMoments*>(stage_min + 32 * STAGE_LD);   // [NW][32] stat partials
  const bool train = (e.mode == EPI_EDGE && e.norm == DGCN_NORM_BATCH_TRAIN);
  const int nch = (e.mode == EPI_EDGE) ? e.c_out : e.c_in;
  const float slope = (e.mode == EPI_EDGE) ? epi_slope(e) : 0.f;
  for (int c0 = 0; c0 < nch; c0 += 32) {
    const int c = c0 + lane;
    float bs = 1.f, bt = 0.f;
    BnAcc st = bn_acc_zero();
    if (e.mode == EPI_EDGE) bn_affine(e, c, bs, bt);
    for (int qq = 0; qq < QPW; ++qq) {
      const int ql = warp * QPW + qq;
      const int qg = q0 + ql;
      if (qg >= N || (ok != nullptr && !ok[ql])) continue;
      if (e.mode == EPI_EDGE) {
        float vmax, vmin;
        edge_query(e, node0, qg, &sel[ql * sel_ld], k, c, slope, vmax, vmin, st);
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
    if (train) red[warp * 32 + lane] = bn_acc_moments(st);
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
    if (train && tid < 32) {
      BnMoments m = red[tid];
      for (int w = 1; w < NW; ++w) m = bn_merge(m, red[w * 32 + tid]);
      if (c0 + tid < nch) bn_store_partial(e.partial, cta, nch, c0 + tid, m);
    }
    __syncthreads();
  }
}


// ---- wide CTA-level consumer ------------------------------------------------------------------
// Same contract as cta_epilogue for channel counts nch in {32, 64, 128} (nch = c_out for EdgeConv,
// c_in for MRConv) and N % 8 == 0: a group of G = nch/4 lanes owns one query and reads every selected
// row as ONE float4 per lane, up to ten rows in flight, so a warp keeps 32 x 10 x 16 B outstanding
// instead of 8 x 128 B.  A group walks eight consecutive queries and then stores its four channels as
// full 32-byte sectors; no shared-memory staging.  sel: int [TILE][sel_ld]; red: float [NW][3][nch]
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
  BnAcc st[4] = {};
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
                  if (TRAIN) bn_acc_add(st[c], av);
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
    // fixed-order merge: slots of a warp (xor shuffles), then the NW warps in order
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      BnMoments m = bn_acc_moments(st[c]);
      for (int o = G; o < 32; o <<= 1) m = bn_merge(m, bn_shfl_xor(m, o));
      if (slot == 0) bn_store_partial(red, warp, nch, 4 * g + c, m);
    }
    __syncthreads();
    for (int c = tid; c < nch; c += NW * 32) {
      BnMoments m = bn_load_partial(red, 0, nch, c);
      for (int w = 1; w < NW; ++w) m = bn_merge(m, bn_load_partial(red, w, nch, c));
      bn_store_partial(e.partial, cta, nch, c, m);
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
__global__ void dist_rows_kernel(const KnnArgs a, int b0, float* __restrict__ drows, int ldd);

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
      float vmax, vmin, bs, bt;
      BnAcc st = bn_acc_zero();
      bn_affine(e, c, bs, bt);
      edge_query(e, node0, q, sel, k, c, slope, vmax, vmin, st);
      if (c < e.c_out) {
        int64_t o = (static_cast<int64_t>(b) * e.c_out + c) * N + q;
        const int64_t oo = b * e.out_sb + static_cast<int64_t>(c) * N + q;
        if (train) {
          e.out[oo] = vmax;
          e.out_min[o] = vmin;
          bn_store_partial(e.partial, node0 + q, e.c_out, c, bn_acc_moments(st));   // one partial row per query
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
__global__ void select_rows_kernel(const KnnArgs a, int b0, int nb, const float* __restrict__ drows, int ldd, int KP,
                                   int nkeys, int warps_per_cta, const int* __restrict__ row_list,
                                   const int* __restrict__ row_count);

// Fast variant: a 128-key sample of the row bounds the K-th distance from above, one pass compacts
// every key below that bound (in index order) into shared memory, a bitonic sort of the next power of
// two finishes.  Exact whenever the compacted set holds >= K and <= CAP keys; other rows go to a list
// that select_rows_kernel completes.  dynamic smem per warp: sk[CAP] (u64) | sel[k] (int).
__global__ void select_rows_fast_kernel(const KnnArgs a, int b0, int nb, const float* __restrict__ drows, int ldd,
                                        int CAP, int sample_rank, int warps_per_cta, int* __restrict__ row_count,
                                        int* __restrict__ row_list);

}  // namespace dgcn

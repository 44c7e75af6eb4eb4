// The non-template kernels of the tensor-core kNN route, declared and documented in knn_tc.cuh: the two prologues
// and the exact completion of uncertified queries.
#include "knn_tc.cuh"

namespace dgcn {

__global__ void __launch_bounds__(256) tc_prologue_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C,
                                                         int Cpad, int N, float* __restrict__ sq,
                                                         __nv_bfloat16* __restrict__ planes, float* __restrict__ xt,
                                                         float* __restrict__ sqmax, __nv_bfloat16* __restrict__ sqp,
                                                         bool f16) {
  __shared__ float tile[TC_MAX_C][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int b = blockIdx.y, n0 = blockIdx.x * 32, n = n0 + tx;
  const int64_t plane = static_cast<int64_t>(Cpad) * N;
  __nv_bfloat16* pb = planes + static_cast<int64_t>(b) * TC_PLANES * plane;
  __half* ph = reinterpret_cast<__half*>(planes) + static_cast<int64_t>(b) * plane;
  for (int c = ty; c < Cpad; c += 8) {
    float v = 0.f;
    if (c < C && n < N) v = __ldg(x + b * sb + c * sc + n);
    if (c < C) tile[c][tx] = v;
    if (n < N && f16) {
      ph[static_cast<int64_t>(c) * N + n] = tc_to_f16(v);
    } else if (n < N) {
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      pb[static_cast<int64_t>(c) * N + n] = hi;
      pb[plane + static_cast<int64_t>(c) * N + n] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
  __syncthreads();
  if (ty == 0) {
    float s = 0.f, e2 = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(tile[c][tx], tile[c][tx], s);
    if (f16) {
      for (int c = 0; c < C; ++c) e2 += tc_f16_err2(tile[c][tx]);
      const float em = warp_max(n < N ? e2 : 0.f);
      if (tx == 0) atomicMax(reinterpret_cast<unsigned int*>(sqmax + gridDim.y + b), __float_as_uint(em));
    }
    if (n < N) {
      sq[static_cast<int64_t>(b) * N + n] = s;
      // rows 0..2 of the (B, 8, N) extra operand block: -|x|^2 / 2 as three bf16 terms (2^-24 relative)
      __nv_bfloat16* sp = sqp + static_cast<int64_t>(b) * 8 * N + n;
      float rem = -0.5f * s;
#pragma unroll
      for (int t3 = 0; t3 < 3; ++t3) {
        const __nv_bfloat16 h = __float2bfloat16_rn(rem);
        sp[static_cast<int64_t>(t3) * N] = h;
        rem -= __bfloat162float(h);
      }
#pragma unroll
      for (int t3 = 3; t3 < 8; ++t3) sp[static_cast<int64_t>(t3) * N] = __float2bfloat16_rn(0.f);
    }
    float m = n < N ? s : 0.f;
    m = warp_max(m);
    if (tx == 0) atomicMax(reinterpret_cast<unsigned int*>(sqmax + b), __float_as_uint(m));
  }
  if (xt) {
    for (int i = threadIdx.x; i < 32 * C; i += 256) {
      const int rr = i / C, c = i % C;
      if (n0 + rr < N) xt[(static_cast<int64_t>(b) * N + n0 + rr) * C + c] = tile[c][rr];
    }
  }
}

__global__ void __launch_bounds__(256, 4) tc_prologue_pq_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int C,
                                                            int Cpad, int N, float* __restrict__ sq,
                                                            __nv_bfloat16* __restrict__ planes, float* __restrict__ xt,
                                                            float* __restrict__ sqmax, __nv_bfloat16* __restrict__ sqp,
                                                            const ProloguePq g, bool f16) {
  extern __shared__ __align__(16) float pq_smem[];
  constexpr int XLD = 68;
  float* xs = pq_smem;                       // [C][XLD]
  float* ws = pq_smem + TC_MAX_C * XLD;      // [C][M]
  const int tid = threadIdx.x;
  const int b = blockIdx.y, n0 = blockIdx.x * 64;
  const int M = g.M;
  const int64_t plane = static_cast<int64_t>(Cpad) * N;
  __nv_bfloat16* pb = planes + static_cast<int64_t>(b) * TC_PLANES * plane;
  __half* ph = reinterpret_cast<__half*>(planes) + static_cast<int64_t>(b) * plane;
  if (((reinterpret_cast<uintptr_t>(x) & 7) | (sb & 1) | (sc & 1)) == 0) {
    // two adjacent points per thread: 8-byte loads, one bf16x2 store per plane (each half rounded like the scalar path)
    const int lane = tid & 31, wrp = tid >> 5, n = n0 + 2 * lane;
    for (int c = wrp; c < Cpad; c += 8) {
      const float2 v = c < C ? __ldg(reinterpret_cast<const float2*>(x + b * sb + c * sc + n)) : make_float2(0.f, 0.f);
      if (c < C) *reinterpret_cast<float2*>(xs + c * XLD + 2 * lane) = v;
      if (f16) {
        *reinterpret_cast<__half2*>(ph + static_cast<int64_t>(c) * N + n) = __halves2half2(tc_to_f16(v.x), tc_to_f16(v.y));
        continue;
      }
      const __nv_bfloat162 hi = __floats2bfloat162_rn(v.x, v.y);
      const __nv_bfloat162 mid = __floats2bfloat162_rn(v.x - __low2float(hi), v.y - __high2float(hi));
      *reinterpret_cast<__nv_bfloat162*>(pb + static_cast<int64_t>(c) * N + n) = hi;
      *reinterpret_cast<__nv_bfloat162*>(pb + plane + static_cast<int64_t>(c) * N + n) = mid;
    }
  } else {
    const int tx = tid & 63, ty = tid >> 6, n = n0 + tx;
    for (int c = ty; c < Cpad; c += 4) {
      const float v = c < C ? __ldg(x + b * sb + c * sc + n) : 0.f;
      if (c < C) xs[c * XLD + tx] = v;
      if (f16) {
        ph[static_cast<int64_t>(c) * N + n] = tc_to_f16(v);
        continue;
      }
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      pb[static_cast<int64_t>(c) * N + n] = hi;
      pb[plane + static_cast<int64_t>(c) * N + n] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
  for (int i = tid * 4; i < C * M; i += 256 * 4)
    *reinterpret_cast<float4*>(ws + i) = __ldg(reinterpret_cast<const float4*>(g.wk + i));
  __syncthreads();
  if (tid < 64) {
    const int n = n0 + tid;
    float s = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(xs[c * XLD + tid], xs[c * XLD + tid], s);
    sq[static_cast<int64_t>(b) * N + n] = s;
    if (f16) {
      float e2 = 0.f;
      for (int c = 0; c < C; ++c) e2 += tc_f16_err2(xs[c * XLD + tid]);
      const float em = warp_max(e2);
      if ((tid & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(sqmax + gridDim.y + b), __float_as_uint(em));
    }
    __nv_bfloat16* sp = sqp + static_cast<int64_t>(b) * 8 * N + n;
    float rem = -0.5f * s;
#pragma unroll
    for (int t3 = 0; t3 < 3; ++t3) {
      const __nv_bfloat16 h = __float2bfloat16_rn(rem);
      sp[static_cast<int64_t>(t3) * N] = h;
      rem -= __bfloat162float(h);
    }
#pragma unroll
    for (int t3 = 3; t3 < 8; ++t3) sp[static_cast<int64_t>(t3) * N] = __float2bfloat16_rn(0.f);
    const float m = warp_max(s);
    if ((tid & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(sqmax + b), __float_as_uint(m));
  }
  if (xt && (C & 7) == 0 && (reinterpret_cast<uintptr_t>(xt) & 15) == 0) {
    // node-major copy: a warp step covers 16 points x 8 channels - lane pairs write one full 32-byte sector of a row,
    // and the transposed shared-memory reads ((c0 + 4 (lane & 1) + j) * 68 + lane / 2) hit 32 distinct banks
    const int lane = tid & 31, wrp = tid >> 5;
    for (int it = wrp; it < 4 * (C >> 3); it += 8) {
      const int rr = (lane >> 1) + 16 * (it & 3), c = (it >> 2) * 8 + 4 * (lane & 1);
      const float4 v = make_float4(xs[c * XLD + rr], xs[(c + 1) * XLD + rr], xs[(c + 2) * XLD + rr], xs[(c + 3) * XLD + rr]);
      *reinterpret_cast<float4*>(xt + (static_cast<int64_t>(b) * N + n0 + rr) * C + c) = v;
    }
  } else if (xt) {
    for (int i = tid; i < 64 * C; i += 256) {
      const int rr = i / C, c = i - rr * C;
      xt[(static_cast<int64_t>(b) * N + n0 + rr) * C + c] = xs[c * XLD + rr];
    }
  }
  // node GEMM: thread (tx, ty) owns points 4 ty .. 4 ty + 3 and outputs {4 tx .. +3} U {64 + 4 tx .. +3} of each
  // 128-wide pass
  const int tx = tid & 15, ty = tid >> 4;
  for (int m0 = 0; m0 < M; m0 += 128) {
    // the chain per output - c ascending from 0 - and its bits are those of node_pq_kernel
    float2 acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = make_float2(0.f, 0.f);
#pragma unroll 4
    for (int c = 0; c < C; ++c) {
      const float4 a = *reinterpret_cast<const float4*>(xs + c * XLD + ty * 4);
      const float4 w0 = *reinterpret_cast<const float4*>(ws + c * M + m0 + tx * 4);
      const float4 w1 = *reinterpret_cast<const float4*>(ws + c * M + m0 + 64 + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float2 wv[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y), make_float2(w1.z, w1.w)};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[i][j].x = fmaf(av[i], wv[j].x, acc[i][j].x);
          acc[i][j].y = fmaf(av[i], wv[j].y, acc[i][j].y);
        }
    }
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(g.bk + m0 + tx * 4));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(g.bk + m0 + 64 + tx * 4));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float* row = g.pq + (static_cast<int64_t>(b) * N + n0 + ty * 4 + i) * M + m0;
      *reinterpret_cast<float4*>(row + tx * 4) =
          make_float4(acc[i][0].x + b0.x, acc[i][0].y + b0.y, acc[i][1].x + b0.z, acc[i][1].y + b0.w);
      *reinterpret_cast<float4*>(row + 64 + tx * 4) =
          make_float4(acc[i][2].x + b1.x, acc[i][2].y + b1.y, acc[i][3].x + b1.z, acc[i][3].y + b1.w);
    }
  }
}

__global__ void __launch_bounds__(256) knn_exact_rows_kernel(const KnnArgs a, const int* __restrict__ fail_count,
                                                            const int* __restrict__ fail_list,
                                                            float* __restrict__ partial_extra) {
  __shared__ float xq[TC_MAX_C];
  __shared__ uint64_t merged[8 * 64];
  __shared__ int sel[64];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int total = *fail_count;
  const Epilogue& e = a.epi;
  const int N = a.N, C = a.C, k = a.k;
  BnAcc stacc[4];                          // c_out <= 128 covered per lane
#pragma unroll
  for (int u = 0; u < 4; ++u) stacc[u] = bn_acc_zero();
  for (int f = blockIdx.x; f < total; f += gridDim.x) {
    const int code = fail_list[f];
    const int b = code / N, q = code % N;
    const float* xb = a.x + b * a.sb;
    const float* sqb = a.sq + static_cast<int64_t>(b) * N;
    const float sqq = sqb[q];
    __syncthreads();                       // the previous query's xq / merged / sel are no longer read
    if (tid < C) xq[tid] = __ldg(xb + tid * a.sc + q);
    __syncthreads();
    uint64_t r0 = KEY_MAX, r1 = KEY_MAX;   // this warp's sorted 64-entry list: r0 = ranks 0..31, r1 = 32..63
    for (int j0 = warp * 32; j0 < N; j0 += 256) {
      const int j = j0 + lane;
      uint64_t key = KEY_MAX;
      if (j < N && !(a.exclude_self && j == q)) {
        const float* xj = xb + j;
        float acc = 0.f;
#pragma unroll 8
        for (int c = 0; c < C; ++c) acc = fmaf(xq[c], __ldg(xj + c * a.sc), acc);
        key = make_key((sqq + (-2.0f * acc)) + sqb[j], static_cast<uint32_t>(j));
      }
      const uint64_t worst = shfl_u64(r1, 31);
      unsigned cand = __ballot_sync(0xffffffffu, key < worst);
      while (cand) {
        const int src = __ffs(cand) - 1;
        cand &= cand - 1;
        uint64_t carry = shfl_u64(key, src);
        // insert into r0, evicted element cascades into r1
        uint64_t last0 = shfl_u64(r0, 31);
        if (carry < last0) {
          int pos = __popc(__ballot_sync(0xffffffffu, r0 < carry));
          uint64_t up = shfl_up_u64(r0, 1);
          r0 = (lane == pos) ? carry : (lane > pos ? up : r0);
          carry = last0;
        }
        uint64_t last1 = shfl_u64(r1, 31);
        if (carry < last1) {
          int pos = __popc(__ballot_sync(0xffffffffu, r1 < carry));
          uint64_t up = shfl_up_u64(r1, 1);
          r1 = (lane == pos) ? carry : (lane > pos ? up : r1);
        }
      }
    }
    merged[warp * 64 + lane] = r0;
    merged[warp * 64 + 32 + lane] = r1;
    __syncthreads();
    if (warp != 0) continue;               // (the loop-top barrier keeps the CTA together)
    warp_bitonic_sort(merged, 512, lane);
    const int64_t node0 = static_cast<int64_t>(b) * N;
    for (int l = lane; l < k; l += 32) {
      const int idx = static_cast<int>(static_cast<uint32_t>(merged[keep_rank(a, l)]));
      sel[l] = idx;
      const int64_t o = (node0 + q) * k + l;
      if (e.nbr) e.nbr[o] = idx;
      if (e.edge_index) {
        e.edge_index[o] = idx;
        e.edge_index[static_cast<int64_t>(a.B) * N * k + o] = q;
      }
    }
    __syncwarp();
    if (e.mode == EPI_EDGE) {
      const float slope = epi_slope(e);
      const bool train = e.norm == DGCN_NORM_BATCH_TRAIN;
      for (int c0 = 0, u = 0; c0 < e.c_out; c0 += 32, ++u) {
        const int c = c0 + lane;
        float vmax, vmin, bs, bt;
        bn_affine(e, c, bs, bt);
        // the lane's running statistics of channel c accumulate across the queries of this CTA (selected by
        // compile-time indices, so that stacc stays in registers)
        BnAcc st = bn_acc_zero();
#pragma unroll
        for (int v = 0; v < 4; ++v)
          if (v == u) st = stacc[v];
        edge_query(e, node0, q, sel, k, c, slope, vmax, vmin, st);
#pragma unroll
        for (int v = 0; v < 4; ++v)
          if (v == u) stacc[v] = st;
        if (c < e.c_out) {
          const int64_t o = (static_cast<int64_t>(b) * e.c_out + c) * N + q;
          const int64_t oo = b * e.out_sb + static_cast<int64_t>(c) * N + q;
          if (train) {
            e.out[oo] = vmax;
            e.out_min[o] = vmin;
          } else {
            e.out[oo] = epi_res(e, b, c, q, bs >= 0.f ? fmaf(bs, vmax, bt) : fmaf(bs, vmin, bt));
          }
        }
      }
    } else if (e.mode == EPI_MR) {
      for (int c0 = 0; c0 < e.c_in; c0 += 32) {
        const int c = c0 + lane;
        const float r = mr_query(e, node0, q, sel, k, c);
        if (c < e.c_in) e.r_out[(static_cast<int64_t>(b) * e.c_in + c) * N + q] = r;
      }
    }
    __syncwarp();
  }
  // train-mode statistics of the queries completed here: one extra partial row per CTA (warp 0 holds them)
  if (warp == 0 && e.mode == EPI_EDGE && e.norm == DGCN_NORM_BATCH_TRAIN && partial_extra) {
    const int64_t rowi = blockIdx.x;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = u * 32 + lane;
      if (c < e.c_out) bn_store_partial(partial_extra, rowi, e.c_out, c, bn_acc_moments(stacc[u]));
    }
  }
}

}  // namespace dgcn

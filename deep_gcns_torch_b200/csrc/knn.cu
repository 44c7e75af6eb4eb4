// The non-template kernels of the fp32 kNN routes, declared and documented in knn.cuh: squared norms, and the slab
// route's distance rows and row selects.
#include "knn.cuh"

namespace dgcn {

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

}  // namespace dgcn

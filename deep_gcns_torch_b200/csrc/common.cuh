// Shared device helpers for the dgcn kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <atomic>

#include "../../include/dgcn.h"

namespace dgcn {

// ---- host-side error plumbing ---------------------------------------------
void set_last_cuda_error(cudaError_t e, const char* file, int line);

#define DGCN_LAUNCH_CHECK()                                        \
  do {                                                             \
    cudaError_t e__ = cudaGetLastError();                          \
    if (e__ != cudaSuccess) {                                      \
      ::dgcn::set_last_cuda_error(e__, __FILE__, __LINE__);        \
      return DGCN_ERR_CUDA;                                        \
    }                                                              \
  } while (0)

#define DGCN_CUDA_TRY(expr)                                        \
  do {                                                             \
    cudaError_t e__ = (expr);                                      \
    if (e__ != cudaSuccess) {                                      \
      ::dgcn::set_last_cuda_error(e__, __FILE__, __LINE__);        \
      return DGCN_ERR_CUDA;                                        \
    }                                                              \
  } while (0)

// Dynamic shared memory opt-in, once per (call site, device): the attribute is sticky, so it is set on
// first use (or when a larger size is asked for) instead of before every launch.  The table is a
// write-once cache of what the driver already knows, not program state.
#define DGCN_ENSURE_SMEM(kernel, bytes)                                                              \
  do {                                                                                               \
    static std::atomic<int> smem_set__[64];                                                          \
    int dev__ = 0;                                                                                   \
    DGCN_CUDA_TRY(cudaGetDevice(&dev__));                                                            \
    const int want__ = static_cast<int>(bytes);                                                      \
    const bool slot__ = dev__ >= 0 && dev__ < 64;                                                    \
    if (!slot__ || smem_set__[dev__].load(std::memory_order_relaxed) < want__) {                     \
      DGCN_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, want__)); \
      if (slot__) smem_set__[dev__].store(want__, std::memory_order_relaxed);                        \
    }                                                                                                \
  } while (0)

// SM count and L2 size of the current device (write-once per-device cache of what the driver reports; 132 SMs and
// 50 MB, an H100 SXM, if the query fails).  Grid and slab sizes derive from them.
int device_sm_count();
size_t device_l2_bytes();

// Certification counters of the tensor-core kNN pre-filter (see dgcn_debug_tc_certification).
bool debug_certification_on();
void debug_certification_add(int64_t uncertified, int64_t queries);

// Optional event bracket around a path's dominant kernel (see dgcn_debug_kernel_timing).
struct KernelTimer {
  KernelTimer(cudaStream_t stream, const char* tag);
  ~KernelTimer();
  cudaStream_t stream_;
  void* slot_;
};

// The res+ block's activated row in training, keep ? relu(s * x + t) * keep_scale : 0 (dgcn_keep_mask): one
// function for the aggregate's reads and its backward's recomputation, so both see the same bits (__fmul_rn is
// never contracted into an FMA).
__device__ __forceinline__ float pre_keep(float s, float t, float x, bool relu, bool kept, float keep_scale) {
  float z = fmaf(s, x, t);
  if (relu) z = fmaxf(z, 0.f);
  return kept ? __fmul_rn(z, keep_scale) : 0.f;
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Bump allocator over the caller-owned workspace.  A Workspace made without arguments only counts: take()
// advances `off` as it would and returns nullptr, so a *_workspace_bytes() query is the launch's own carve run
// this way, and a carve takes every region of a path before the path's first launch.
struct Workspace {
  char* base;
  size_t size;
  size_t off;
  bool ok;
  bool counting;
  Workspace() : base(nullptr), size(0), off(0), ok(true), counting(true) {}
  Workspace(void* p, size_t n) : base(static_cast<char*>(p)), size(n), off(0), ok(true), counting(false) {}
  template <typename T>
  T* take(size_t count) {
    size_t bytes = align_up(count * sizeof(T), 256);
    if (counting) {
      off += bytes;
      return nullptr;
    }
    if (base == nullptr || off + bytes > size) {
      ok = false;
      return nullptr;
    }
    T* r = reinterpret_cast<T*>(base + off);
    off += bytes;
    return r;
  }
};

// ---- ordering keys ----------------------------------------------------------
// Monotone map fp32 -> uint32 (ascending floats give ascending unsigned keys).
// NaNs are canonicalised to the positive quiet NaN so they rank after +inf.
__device__ __forceinline__ uint32_t float_to_ordered(float f) {
  uint32_t u = __float_as_uint(f);
  if (f != f) u = 0x7FC00000u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(uint32_t k) {
  uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  return __uint_as_float(u);
}
// (distance, index) -> one 64-bit key: ascending distance, ties to smaller index.
__device__ __forceinline__ uint64_t make_key(float d, uint32_t idx) {
  return (static_cast<uint64_t>(float_to_ordered(d)) << 32) | idx;
}
constexpr uint64_t KEY_MAX = 0xFFFFFFFFFFFFFFFFull;

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
  uint32_t lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v), src);
  uint32_t hi = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), src);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_up_u64(uint64_t v, int delta) {
  uint32_t lo = __shfl_up_sync(0xffffffffu, static_cast<uint32_t>(v), delta);
  uint32_t hi = __shfl_up_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), delta);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int mask) {
  uint32_t lo = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(v), mask);
  uint32_t hi = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), mask);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// act(z) of gcn_lib/dense/torch_nn.py:9-21 as one expression: slope = 0 relu,
// 0.2 leakyrelu, learnt prelu weight, 1 identity.
__device__ __forceinline__ float act_apply(float z, float slope) { return z >= 0.f ? z : z * slope; }

// ---- train-mode BatchNorm statistics ------------------------------------------
// A channel's batch statistics travel as (count, mean, M2 = sum of squared deviations from the mean), never as
// (sum a, sum a^2): E[a^2] - E[a]^2 in fp32 loses ~ (mean / std)^2 * 2^-24 of the variance, which a channel with a
// large mean (un-centred coordinates, a ReLU channel dominated by its bias) turns into percent errors.  A thread
// sums a - pivot and (a - pivot)^2, pivot = the first value it saw, so its sums are of the channel's spread only;
// threads and warps merge (count, mean, M2) with Chan's formula in fp32; the partial rows [n_partial][3][C] of a
// launch are merged the same way in fp64 (bn_merge_kernel).  A constant channel stays exact: every deviation and
// every mean difference is 0, so the variance is 0 and the mean the constant.
constexpr int BN_PARTIAL_ROWS = 3;   // a partial row: count, mean, M2 (each [C])

struct BnAcc { float n, pivot, d1, d2; };     // one thread's running sums
struct BnMoments { float n, mean, m2; };

__device__ __forceinline__ BnAcc bn_acc_zero() { return BnAcc{0.f, 0.f, 0.f, 0.f}; }
__device__ __forceinline__ void bn_acc_add(BnAcc& s, float a) {
  s.pivot = s.n == 0.f ? a : s.pivot;
  const float d = a - s.pivot;
  s.n += 1.f;
  s.d1 += d;
  s.d2 = fmaf(d, d, s.d2);
}
__device__ __forceinline__ BnMoments bn_acc_moments(const BnAcc& s) {
  if (s.n == 0.f) return BnMoments{0.f, 0.f, 0.f};
  const float m = s.d1 / s.n;
  return BnMoments{s.n, s.pivot + m, fmaxf(fmaf(-s.d1, m, s.d2), 0.f)};
}
// Chan et al.: merge of two disjoint sets; either (or both) may be empty
__device__ __forceinline__ BnMoments bn_merge(const BnMoments& a, const BnMoments& b) {
  const float n = a.n + b.n;
  const float f = n > 0.f ? b.n / n : 0.f;
  const float delta = b.mean - a.mean;
  return BnMoments{n, fmaf(delta, f, a.mean), a.m2 + b.m2 + delta * (delta * (a.n * f))};
}
__device__ __forceinline__ BnMoments bn_shfl_xor(const BnMoments& m, int o) {
  return BnMoments{__shfl_xor_sync(0xffffffffu, m.n, o), __shfl_xor_sync(0xffffffffu, m.mean, o),
                   __shfl_xor_sync(0xffffffffu, m.m2, o)};
}
// partial row `row`, channel c of C
__device__ __forceinline__ void bn_store_partial(float* partial, int64_t row, int C, int c, const BnMoments& m) {
  float* p = partial + row * BN_PARTIAL_ROWS * C + c;
  p[0] = m.n;
  p[C] = m.mean;
  p[2 * static_cast<int64_t>(C)] = m.m2;
}
__device__ __forceinline__ BnMoments bn_load_partial(const float* partial, int64_t row, int C, int c) {
  const float* p = partial + row * BN_PARTIAL_ROWS * C + c;
  return BnMoments{p[0], p[C], p[2 * static_cast<int64_t>(C)]};
}

// ---- 128x128 fp32 tile engine ------------------------------------------------
// C[r][c] = sum_k A[k][r] * B[k][c] for one 128x128 output tile, A and B both
// "k-major" (row k contiguous along r / c).  256 threads, 8x8 accumulators per
// thread, channels streamed through shared memory in chunks of TK with register
// prefetch (double buffered).  The fp32 accumulation order is k ascending, one
// FMA per k - this is the order the distance ranking is defined on.
constexpr int TILE = 128;   // rows and cols of an output tile
constexpr int TK = 16;      // k-chunk staged per step
constexpr int NTHREADS = 256;
constexpr int KCH = 512;     // points per CTA of the split-K weight-gradient GEMM (wgrad_kernel, basic_conv.cu)

struct KMajor {          // a k-major operand: element (k, i) at ptr[k*ld + i]
  const float* ptr;      // rows k < K1
  int64_t ld;
  const float* ptr2;     // rows K1 <= k < K (second stacked segment), row k-K1
  int64_t ld2;
  int K1;
  int K;                 // valid k rows in total
  int n;                 // valid extent along i
  bool vec;              // every row is 16-byte aligned and n % 4 == 0
};
__host__ __device__ __forceinline__ KMajor kmajor1(const float* p, int64_t ld, int K, int n, bool vec) {
  return KMajor{p, ld, nullptr, 0, K, K, n, vec};
}
__host__ __device__ __forceinline__ KMajor kmajor2(const float* p, int64_t ld, int K1, const float* p2,
                                                   int64_t ld2, int K, int n, bool vec) {
  return KMajor{p, ld, p2, ld2, K1, K, n, vec};
}

struct TileSmem {
  float a[2][TK][TILE];
  float b[2][TK][TILE];
};

// thread -> micro-tile geometry: rows {ty*4..+3, 64+ty*4..+3}, cols likewise with tx.
__device__ __forceinline__ int tile_row(int ty, int i) { return (i < 4 ? 0 : 60) + ty * 4 + i; }
__device__ __forceinline__ int tile_col(int tx, int j) { return (j < 4 ? 0 : 60) + tx * 4 + j; }

__device__ __forceinline__ void chunk_load(const KMajor& m, int k0, int i0, float4 (&r)[2]) {
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    int f = threadIdx.x + u * NTHREADS;  // float4 slot in the TKx128 chunk
    int kr = f >> 5;
    int ci = (f & 31) * 4;
    int k = k0 + kr;
    int i = i0 + ci;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < m.K) {
      const float* src = (k < m.K1) ? m.ptr + static_cast<int64_t>(k) * m.ld + i
                                    : m.ptr2 + static_cast<int64_t>(k - m.K1) * m.ld2 + i;
      if (m.vec && i + 3 < m.n) {
        v = __ldg(reinterpret_cast<const float4*>(src));
      } else {
        if (i + 0 < m.n) v.x = __ldg(src + 0);
        if (i + 1 < m.n) v.y = __ldg(src + 1);
        if (i + 2 < m.n) v.z = __ldg(src + 2);
        if (i + 3 < m.n) v.w = __ldg(src + 3);
      }
    }
    r[u] = v;
  }
}
__device__ __forceinline__ void chunk_store(float (*dst)[TILE], const float4 (&r)[2]) {
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    int f = threadIdx.x + u * NTHREADS;
    *reinterpret_cast<float4*>(&dst[f >> 5][(f & 31) * 4]) = r[u];
  }
}

__device__ __forceinline__ void chunk_fma(const float (*as)[TILE], const float (*bs)[TILE], int tx,
                                          int ty, float (&acc)[8][8]) {
#pragma unroll
  for (int k = 0; k < TK; ++k) {
    float4 a0 = *reinterpret_cast<const float4*>(&as[k][ty * 4]);
    float4 a1 = *reinterpret_cast<const float4*>(&as[k][64 + ty * 4]);
    float4 b0 = *reinterpret_cast<const float4*>(&bs[k][tx * 4]);
    float4 b1 = *reinterpret_cast<const float4*>(&bs[k][64 + tx * 4]);
    float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
}

// Full tile product; on return all threads have passed a barrier and shared
// memory may be reused.  A tile origin r0, B tile origin c0.
__device__ __forceinline__ void tile_product(TileSmem& sm, const KMajor& A, int r0, const KMajor& B,
                                             int c0, float (&acc)[8][8]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const int nchunk = (A.K + TK - 1) / TK;
  float4 ra[2], rb[2];
  chunk_load(A, 0, r0, ra);
  chunk_load(B, 0, c0, rb);
  chunk_store(sm.a[0], ra);
  chunk_store(sm.b[0], rb);
  __syncthreads();
  for (int ch = 0; ch < nchunk; ++ch) {
    const int s = ch & 1;
    if (ch + 1 < nchunk) {
      chunk_load(A, (ch + 1) * TK, r0, ra);
      chunk_load(B, (ch + 1) * TK, c0, rb);
    }
    chunk_fma(sm.a[s], sm.b[s], tx, ty, acc);
    if (ch + 1 < nchunk) {
      chunk_store(sm.a[s ^ 1], ra);
      chunk_store(sm.b[s ^ 1], rb);
    }
    __syncthreads();
  }
}

}  // namespace dgcn

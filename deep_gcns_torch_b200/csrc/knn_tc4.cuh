// Multi-tile variant of the tensor-core kNN selection (knn_tc.cuh): ONE CTA per SM, warp specialised.
//
//   Why: the CTA holds T4_GROUPS query tiles of the SAME cloud, so a candidate tile is brought in once (TMA) and
//   multiplied against every resident query operand, and the filter code of knn_tc_kernel is replaced by a cheaper
//   sorting-network flush.  Two groups: the query planes, the per-group accumulator stage and candidate buffer of a
//   third would not fit the 227 KB of shared memory an H100 block may use.
//
//   producer warp            moves the operands by TMA: the query planes of the groups once, then 64-candidate
//                            half-tiles into a two-stage ring (the stage of half-tile h+1 is refilled as soon as every
//                            group has finished its wgmma on half-tile h-1, stage_free).
//   filter warpgroup g       per half-tile: wait full[s], two m64n64k16 wgmma chains (query rows 0..63 and 64..127,
//                            3*Cpad/16 + 1 each) against the stage, release the stage, the accumulators to the group's
//                            shared-memory stage (row = query); thread r = query r of tile g reads 8 columns at a
//                            time, threshold test -> private candidate buffer (shared memory, slot-major).
//                            FLUSH = sorting network instead of one insertion per entry: the batch (<= 16 entries
//                            per lane, a second pass for slots 16..23) is bitonic-sorted in registers, min-merged
//                            against the upper half of the 32-entry sorted register list and the list re-sorted by
//                            one 32-input bitonic merge - a fixed ~450 instructions per warp-wide flush whatever
//                            the lanes' counts (the insertion loop costs ~80 per ROUND, rounds = the fullest
//                            lane's count).
//                            Then, per warpgroup (named barriers) in the group's own (now idle) query-plane memory:
//                            - set-only consumers (every rank kept, no index output, no self exclusion): membership
//                              by interval arithmetic on the approximate list, exact fp32 chains only inside the
//                              ambiguous band around rank K (DESIGN.md 6);
//                            - otherwise the exact fp32 re-rank of all listed candidates and the certificate of
//                              knn_tc_kernel;
//                            and the fused consumer (cta_epilogue_wide).
//
// Eligibility (host side, launch_knn_tc): packed entries (N <= 4096), K <= 20 (list of 28 or 16), C % 8 == 0,
// 32-byte aligned node-major copy, wide consumer, no train-mode statistics.  Everything else keeps knn_tc_kernel.
#pragma once
#include "knn_tc.cuh"

namespace dgcn {

constexpr int T4_GROUPS = 2;
constexpr int T4_THREADS = T4_GROUPS * 128 + 32;                 // filter warpgroups + the producer warp
constexpr int T4_CT = 64;                                        // candidates per half-tile (wgmma N)
constexpr int T4_STAGES = 2;
constexpr int T4_CAP = 24;                                       // candidate-buffer slots per thread
constexpr int T4_FLUSH_AT = 16;                                  // flush when a lane holds this many (checked every 8 candidates)
constexpr int T4_LIST = 32;                                      // register list length (power of two >= KP)
constexpr int T4_QBYTES = TC_PLANES * 2 * TC_MAX_C * 128;        // 32 KB: query planes of one group
constexpr int T4_STAGE_BYTES = TC_PLANES * TC_MAX_C * 128;       // 16 KB: one 64-candidate half-tile
constexpr int T4_SX_BYTES = 16 * 128;                            // 2 KB: candidate-side extra K=16 block
constexpr int T4_CBUF_BYTES = T4_CAP * 128 * 4;                  // 12 KB per group
constexpr int T4_ACC_LD = 68;                                    // accumulator stage row: 64 columns + 4
constexpr int T4_ACC_BYTES = TILE * T4_ACC_LD * 4;               // 34 KB per group
constexpr uint32_t T4_SLOT_STRIDE = 128u * 4u;                   // bytes between two slots of one thread
static_assert(T4_SLOT_STRIDE == 512u, "the filter's asm bumps the slot pointer by the literal 512");

struct T4Tail {
  uint64_t full[T4_STAGES];               // half-tile operands have landed (TMA complete_tx)
  uint64_t stage_free[T4_STAGES];         // every wgmma reading the stage has completed
  uint64_t q_full;                        // query planes have landed
  unsigned char ok[T4_GROUPS][TILE];
};

constexpr size_t T4_SMEM_BYTES = static_cast<size_t>(T4_GROUPS) * T4_QBYTES + T4_STAGES * (T4_STAGE_BYTES + T4_SX_BYTES) +
                                 TC_XBLOCK_BYTES + static_cast<size_t>(T4_GROUPS) * (T4_CBUF_BYTES + T4_ACC_BYTES) +
                                 sizeof(T4Tail) + 1024;
static_assert(T4_SMEM_BYTES <= 227 * 1024, "one CTA per SM");

// compare-exchange of two register entries (ascending)
__device__ __forceinline__ void t4_ce(uint32_t& x, uint32_t& y) {
  const uint32_t lo = min(x, y), hi = max(x, y);
  x = lo;
  y = hi;
}
// Bitonic sorting network over a register array, ascending.  All indices are compile-time.
template <int NN>
__device__ __forceinline__ void t4_sort(uint32_t (&v)[NN]) {
#pragma unroll
  for (int k = 2; k <= NN; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int i = 0; i < NN; ++i) {
        const int l = i ^ j;
        if (l > i) {
          if ((i & k) == 0) t4_ce(v[i], v[l]);
          else t4_ce(v[l], v[i]);
        }
      }
    }
  }
}
// v bitonic -> ascending
template <int NN>
__device__ __forceinline__ void t4_merge(uint32_t (&v)[NN]) {
#pragma unroll
  for (int j = NN >> 1; j > 0; j >>= 1) {
#pragma unroll
    for (int i = 0; i < NN; ++i) {
      const int l = i ^ j;
      if (l > i) t4_ce(v[i], v[l]);
    }
  }
}
// true on exactly one lane of the (converged) warp
__device__ __forceinline__ bool t4_elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void t4_group_sync(int g) {
  asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "n"(128) : "memory");
}

template <int KP>
__global__ void __launch_bounds__(T4_THREADS, 1) knn_tc4_kernel(const __grid_constant__ TcArgs t) {
  static_assert(KP <= T4_LIST && (KP & 1) == 0, "list length");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SWIZZLE_128B atoms: 1024-aligned
  unsigned char* qbase = base;                                              // [group][plane][mn block][Cpad rows][128 B]
  unsigned char* stage0 = qbase + T4_GROUPS * T4_QBYTES;                    // [stage][plane][Cpad rows][128 B]
  unsigned char* sx0 = stage0 + T4_STAGES * T4_STAGE_BYTES;                 // [stage][16 rows][128 B]
  unsigned char* qx = sx0 + T4_STAGES * T4_SX_BYTES;                        // ones block, shared by the groups
  unsigned char* cbuf0 = qx + TC_XBLOCK_BYTES;                              // [group][slot][128 threads] u32
  float* acc0 = reinterpret_cast<float*>(cbuf0 + T4_GROUPS * T4_CBUF_BYTES); // [group][128 queries][T4_ACC_LD]
  T4Tail& sm = *reinterpret_cast<T4Tail*>(reinterpret_cast<unsigned char*>(acc0) + T4_GROUPS * T4_ACC_BYTES);
  const KnnArgs& a = t.a;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int b = blockIdx.y;
  const int N = a.N, Cpad = t.Cpad;
  const int qt0 = blockIdx.x * T4_GROUPS;                                   // first query tile of this CTA
  const int ngroups = min(T4_GROUPS, N / TILE - qt0);
  const int H = N / T4_CT;
  const int plane_q = 2 * Cpad * 128, plane_c = Cpad * 128;

  if (tid == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&t.tm_planes)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&t.tm_sqp)) : "memory");
    for (int s = 0; s < T4_STAGES; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.stage_free[s], static_cast<uint32_t>(ngroups * 128));
    }
    mbar_init(&sm.q_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // constant operand blocks: ones in K rows 0..2 on the query side; the candidate-side blocks are zero in rows
  // 8..15 (TMA refreshes rows 0..7 of a stage with every half-tile).  Whole rows are constant: no swizzle needed.
  for (int ch = tid; ch < TC_XBLOCK_BYTES / 16; ch += T4_THREADS) {
    const int row = (ch >> 3) & 15;
    const uint32_t one2 = row < 3 ? 0x3F803F80u : 0u;
    reinterpret_cast<uint4*>(qx)[ch] = make_uint4(one2, one2, one2, one2);
  }
  for (int ch = tid; ch < T4_STAGES * T4_SX_BYTES / 16; ch += T4_THREADS)
    reinterpret_cast<uint4*>(sx0)[ch] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async();
  __syncthreads();

  if (warp >= T4_GROUPS * 4) {
    // ================================ producer: TMA ================================
    const uint32_t tile_bytes = static_cast<uint32_t>(2 * plane_c + 8 * 128);
    auto tma_tile = [&](int h) {
      const int s = h & 1;
      mbar_expect_tx(&sm.full[s], tile_bytes);
#pragma unroll
      for (int pl = 0; pl < TC_PLANES; ++pl)
        tma_load_2d(smem_u32(stage0 + s * T4_STAGE_BYTES) + pl * plane_c, &t.tm_planes, h * T4_CT,
                    (b * TC_PLANES + pl) * Cpad, &sm.full[s]);
      tma_load_2d(smem_u32(sx0 + s * T4_SX_BYTES), &t.tm_sqp, h * T4_CT, b * 8, &sm.full[s]);
    };
    if (t4_elect_one()) {
      mbar_expect_tx(&sm.q_full, static_cast<uint32_t>(ngroups * 2 * plane_q));
      for (int g = 0; g < ngroups; ++g)
#pragma unroll
        for (int pl = 0; pl < TC_PLANES; ++pl)
#pragma unroll
          for (int blk = 0; blk < 2; ++blk)
            tma_load_2d(smem_u32(qbase + g * T4_QBYTES) + pl * plane_q + blk * (Cpad * 128), &t.tm_planes,
                        (qt0 + g) * TILE + blk * 64, (b * TC_PLANES + pl) * Cpad, &sm.q_full);
      tma_tile(0);
#pragma unroll 1
      for (int h = 0; h + 1 < H; ++h) {                    // refill the other stage: its wgmma (half-tile h-1) must be done
        if (h >= 1) mbar_wait_hint(&sm.stage_free[(h + 1) & 1], static_cast<uint32_t>(((h - 1) >> 1) & 1), 1000u);
        tma_tile(h + 1);
      }
    }
    __syncwarp();
  } else {
    if ((warp >> 2) < ngroups) {
    // ================================ filter warpgroup ================================
    const int g = warp >> 2;
    const int r = tid & 127;                               // query row of the tile
    const int q0 = (qt0 + g) * TILE, qg = q0 + r;
    const float* sqb = a.sq + static_cast<int64_t>(b) * N;
    uint32_t lk[T4_LIST];                                  // ascending packed entries (key bits | 12-bit index)
#pragma unroll
    for (int i = 0; i < T4_LIST; ++i) lk[i] = 0xFFFFFFFFu;
    const float sqq = __ldg(sqb + qg);
    float tau_f = __uint_as_float(0x7FC00000u);            // NaN admits everything until the list is full
    float thr_acc = tau_f;
    const uint32_t cb_addr0 = smem_u32(cbuf0 + g * T4_CBUF_BYTES) + static_cast<uint32_t>(r) * 4u;
    uint32_t cb_addr = cb_addr0;

    // entry = accumulator bits (acc = -key/2) with the low 12 mantissa bits replaced by the index -> packed list
    // entry: (bits of an UPPER bound of the squared distance's lower bound ... ) exactly as knn_tc_kernel's flush
    auto unpack = [&](uint32_t en) -> uint32_t {
      const uint32_t ab = (en & 0x80000000u) ? (en & 0xFFFFF000u) : (en | 0xFFFu);
      const float d2 = fmaxf(fmaf(-2.0f, __uint_as_float(ab), sqq), 0.f);
      return (__float_as_uint(d2) & 0xFFFFF000u) | (en & 0xFFFu);
    };
    auto ld_slot = [&](int e) -> uint32_t {
      uint32_t v;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(cb_addr0 + static_cast<uint32_t>(e) * T4_SLOT_STRIDE));
      return v;
    };
    // Warp-synchronous flush by sorting network (see the header comment).
    auto flush = [&]() {
      const int cnt = static_cast<int>((cb_addr - cb_addr0) / T4_SLOT_STRIDE);
      {
        uint32_t bv[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          bv[i] = 0xFFFFFFFFu;
          if (i < cnt) bv[i] = unpack(ld_slot(i));
        }
        t4_sort<16>(bv);
#pragma unroll
        for (int i = 0; i < 16; ++i) lk[T4_LIST - 16 + i] = min(lk[T4_LIST - 16 + i], bv[15 - i]);
        t4_merge<T4_LIST>(lk);
      }
      if (__any_sync(0xffffffffu, cnt > 16)) {             // slots 16..23 (a lane can hold 15 + 8 when the check fires)
        uint32_t bv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          bv[i] = 0xFFFFFFFFu;
          if (16 + i < cnt) bv[i] = unpack(ld_slot(16 + i));
        }
        t4_sort<8>(bv);
#pragma unroll
        for (int i = 0; i < 8; ++i) lk[T4_LIST - 8 + i] = min(lk[T4_LIST - 8 + i], bv[7 - i]);
        t4_merge<T4_LIST>(lk);
      }
      cb_addr = cb_addr0;
      // admission in key units (distance minus |x_i|^2), one truncation step above the KP-th entry
      tau_f = lk[KP - 1] == 0xFFFFFFFFu ? __uint_as_float(0x7FC00000u)
                                        : __uint_as_float((lk[KP - 1] & 0xFFFFF000u) + 0x1000u) - sqq;
      thr_acc = -0.5f * tau_f;                             // key <= tau  <=>  acc >= -tau/2
    };

    // Eight candidates: test, buffer; then the flush check.  ONE asm statement (the compiler cannot thread register
    // copies of the slot pointer through it) and a macro (the chunk registers never become an addressable array).
    // Per candidate: one LOP3 builds the entry (key & R & I) | (R ^ I), R = ~0xFFF | index bits 3..11,
    // I = ~0xFFF | index bits 0..2 (immediate); FSETP; predicated STS + pointer bump.
#define DGCN_T4_FILTER8(V, RB)                                                                                        \
  do {                                                                                                                \
    asm volatile(                                                                                                     \
        "{\n"                                                                                                         \
        ".reg .pred p;\n"                                                                                             \
        ".reg .b32 en;\n"                                                                                             \
        "lop3.b32 en, %1, %17, 0xFFFFF000, 0xE6;\n setp.geu.f32 p, %9, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n"  \
        "lop3.b32 en, %2, %17, 0xFFFFF001, 0xE6;\n setp.geu.f32 p, %10, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "lop3.b32 en, %3, %17, 0xFFFFF002, 0xE6;\n setp.geu.f32 p, %11, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "lop3.b32 en, %4, %17, 0xFFFFF003, 0xE6;\n setp.geu.f32 p, %12, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "lop3.b32 en, %5, %17, 0xFFFFF004, 0xE6;\n setp.geu.f32 p, %13, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "lop3.b32 en, %6, %17, 0xFFFFF005, 0xE6;\n setp.geu.f32 p, %14, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "lop3.b32 en, %7, %17, 0xFFFFF006, 0xE6;\n setp.geu.f32 p, %15, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "lop3.b32 en, %8, %17, 0xFFFFF007, 0xE6;\n setp.geu.f32 p, %16, %18;\n @p st.shared.b32 [%0], en;\n @p add.u32 %0, %0, 512;\n" \
        "}"                                                                                                           \
        : "+r"(cb_addr)                                                                                               \
        : "r"(V[0]), "r"(V[1]), "r"(V[2]), "r"(V[3]), "r"(V[4]), "r"(V[5]), "r"(V[6]), "r"(V[7]),                     \
          "f"(__uint_as_float(V[0])), "f"(__uint_as_float(V[1])), "f"(__uint_as_float(V[2])),                         \
          "f"(__uint_as_float(V[3])), "f"(__uint_as_float(V[4])), "f"(__uint_as_float(V[5])),                         \
          "f"(__uint_as_float(V[6])), "f"(__uint_as_float(V[7])), "r"(RB), "f"(thr_acc));                             \
    if (__any_sync(0xffffffffu, cb_addr - cb_addr0 >= T4_FLUSH_AT * T4_SLOT_STRIDE)) flush();                         \
  } while (0)
    // A half-tile is consumed in eight steps of 8 columns, two steps per iteration of a rolled loop (the flush code
    // exists twice plus the final flush, not once per step: the instruction cache matters at ~700 instructions a copy).
    const uint32_t abase = smem_u32(qbase + g * T4_QBYTES);
    const uint64_t dqx0 = wg_desc_sw128(smem_u32(qx), 2048, 1024), dqx1 = wg_desc_sw128(smem_u32(qx) + 2048, 2048, 1024);
    float* accg = acc0 + g * (TILE * T4_ACC_LD);
    const float* arow = accg + r * T4_ACC_LD;
    mbar_wait(&sm.q_full, 0u);
#pragma unroll 1
    for (int h = 0; h < H; ++h) {
      const int s = h & 1;
      mbar_wait_hint(&sm.full[s], static_cast<uint32_t>((h >> 1) & 1), 1000u);
      {
        // query rows 0..63 and 64..127 against the 64 staged candidates: hi*hi, hi*mid, mid*hi (mid*mid <= 2^-16
        // |x_i||x_j| is inside eps), then + 1 x (-|x_j|^2/2)
        const uint32_t bbase = smem_u32(stage0 + s * T4_STAGE_BYTES);
        float d0[32], d1[32];
        wg_fence();
#pragma unroll 1
        for (int kk = 0; kk < Cpad / 16; ++kk) {
          const uint32_t ah = abase + kk * 2048, am = ah + plane_q, bh = bbase + kk * 2048, bm = bh + plane_c;
          const uint64_t dbh = wg_desc_sw128(bh, Cpad * 128, 1024), dbm = wg_desc_sw128(bm, Cpad * 128, 1024);
          const uint32_t acc = kk > 0 ? 1u : 0u;
          wgmma_m64n64<1, 1>(d0, wg_desc_sw128(ah, Cpad * 128, 1024), dbh, acc);
          wgmma_m64n64<1, 1>(d1, wg_desc_sw128(ah + Cpad * 128, Cpad * 128, 1024), dbh, acc);
          wgmma_m64n64<1, 1>(d0, wg_desc_sw128(ah, Cpad * 128, 1024), dbm, 1u);
          wgmma_m64n64<1, 1>(d1, wg_desc_sw128(ah + Cpad * 128, Cpad * 128, 1024), dbm, 1u);
          wgmma_m64n64<1, 1>(d0, wg_desc_sw128(am, Cpad * 128, 1024), dbh, 1u);
          wgmma_m64n64<1, 1>(d1, wg_desc_sw128(am + Cpad * 128, Cpad * 128, 1024), dbh, 1u);
        }
        const uint64_t dsx = wg_desc_sw128(smem_u32(sx0 + s * T4_SX_BYTES), 2048, 1024);
        wgmma_m64n64<1, 1>(d0, dqx0, dsx, 1u);
        wgmma_m64n64<1, 1>(d1, dqx1, dsx, 1u);
        wg_commit();
        wg_wait_all();
        mbar_arrive(&sm.stage_free[s]);                    // my part of the group's reads of the stage is done
        t4_group_sync(g);                                  // the group has read the previous half-tile out of its stage
        wg_store_m64n64(d0, accg, T4_ACC_LD, 0);
        wg_store_m64n64(d1, accg, T4_ACC_LD, 64);
        t4_group_sync(g);
      }
      // eight steps of 8 columns, two per iteration of a rolled loop (the flush code exists twice plus the final
      // flush, not once per step: the instruction cache matters at ~700 instructions a copy)
#pragma unroll 1
      for (int c8 = 0; c8 < T4_CT / 8; c8 += 2) {
        // (the warp stays converged through this loop: the flush branch is taken on a warp-wide vote)
        const uint32_t rbits = 0xFFFFF000u | static_cast<uint32_t>(h * T4_CT + c8 * 8);
        uint32_t va[8], vb[8];
        {
          const float4 u0 = *reinterpret_cast<const float4*>(arow + c8 * 8), u1 = *reinterpret_cast<const float4*>(arow + c8 * 8 + 4);
          const float4 w0 = *reinterpret_cast<const float4*>(arow + c8 * 8 + 8), w1 = *reinterpret_cast<const float4*>(arow + c8 * 8 + 12);
          va[0] = __float_as_uint(u0.x); va[1] = __float_as_uint(u0.y); va[2] = __float_as_uint(u0.z); va[3] = __float_as_uint(u0.w);
          va[4] = __float_as_uint(u1.x); va[5] = __float_as_uint(u1.y); va[6] = __float_as_uint(u1.z); va[7] = __float_as_uint(u1.w);
          vb[0] = __float_as_uint(w0.x); vb[1] = __float_as_uint(w0.y); vb[2] = __float_as_uint(w0.z); vb[3] = __float_as_uint(w0.w);
          vb[4] = __float_as_uint(w1.x); vb[5] = __float_as_uint(w1.y); vb[6] = __float_as_uint(w1.z); vb[7] = __float_as_uint(w1.w);
        }
        DGCN_T4_FILTER8(va, rbits);
        DGCN_T4_FILTER8(vb, rbits + 8u);
      }
    }
#undef DGCN_T4_FILTER8
    flush();
    t4_group_sync(g);   // the group's wgmma have completed and nobody of the group flushes any more: its query
                        // planes and candidate buffer become the work area

    const float cut = (lk[KP - 1] == 0xFFFFFFFFu) ? INFINITY : __uint_as_float(lk[KP - 1] & 0xFFFFF000u);
    const int C = a.C;
    const float* xtb = t.xt + static_cast<int64_t>(b) * N * C;
    const float* xqp = xtb + static_cast<int64_t>(qg) * C;
    const float smax = __ldg(t.sqmax + b);
    // |approx - exact fp32| <= eps: see the certificate of knn_tc_kernel
    const float eps = (2.0f * (3.0518e-5f + (5.0f * Cpad + 8.0f) * 1.1921e-7f)) * sqrtf(sqq * smax) +
                      9.537e-7f * (sqq + smax);
    int* sel = reinterpret_cast<int*>(cbuf0 + g * T4_CBUF_BYTES);
    const int sel_ld = tc_sel_ld(a.k);
    // The consumer reduces over the SET of the K nearest (max over neighbours) when every rank is kept and nobody
    // asked for the index lists: then only membership matters, and exact arithmetic is needed only where the
    // approximate ranking cannot decide it.
    const bool set_only = !a.has_cols && a.dilation == 1 && !a.exclude_self && a.epi.mode != EPI_INDEX &&
                          a.epi.nbr == nullptr && a.epi.edge_index == nullptr;
    if (set_only) {
      // ---- membership by interval arithmetic, exact fp32 chains only inside the ambiguous band --------------------
      // A list entry a_c (its 20 value bits) is a LOWER bound of the approximate squared distance with
      // a_c <= approx_c <= a_c + delta(a_c), delta(v) = 2^-10 (v + |x_i|^2) (12 accumulator bits + 12 distance bits
      // dropped by the packing), and |approx_c - exact_c| <= eps.  With the list ascending in a and vK, vK1 the values
      // at ranks K and K+1 (1-based): every entry below  lo = vK1 - delta(vK1) - 2 eps  beats all but at most K-1
      // candidates (certainly IN), every entry - and every unlisted candidate, whose approximation is >= cut - above
      // hi = vK + delta(vK) + 2 eps  is beaten by K candidates (certainly OUT).  What lies in [lo, hi] is ranked by
      // the exact key (fp32 FMA chain, ties to the smaller index) and fills the remaining places.
      constexpr int MB = 12;                                           // band entries a query may hold
      uint64_t* band = reinterpret_cast<uint64_t*>(qbase + g * T4_QBYTES);   // [MB][TILE] exact keys
      const int K = a.K;
      float vK = INFINITY, vK1 = INFINITY;
#pragma unroll
      for (int u = 0; u < KP; ++u) {
        const float v = lk[u] == 0xFFFFFFFFu ? INFINITY : __uint_as_float(lk[u] & 0xFFFFF000u);
        if (u == K - 1) vK = v;
        if (u == K) vK1 = v;
      }
      const float hi = vK + 9.765625e-4f * (vK + sqq) + 2.0f * eps;
      const float lo = vK1 - 9.765625e-4f * (vK1 + sqq) - 2.0f * eps;
      bool ok = vK < INFINITY && (cut == INFINITY || hi < cut);
      int* selrow = sel + r * sel_ld;
      uint32_t* bandj = reinterpret_cast<uint32_t*>(band + MB * TILE);   // [MB][TILE] candidate indices of the band
      int n_in = 0, nb = 0;
#pragma unroll
      for (int u = 0; u < KP; ++u) {
        const float v = lk[u] == 0xFFFFFFFFu ? INFINITY : __uint_as_float(lk[u] & 0xFFFFF000u);
        const uint32_t j = lk[u] & 0xFFFu;
        const bool in = v < lo;                                        // the list ascends: a prefix
        if (in && u < K) {
          selrow[u] = static_cast<int>(j);
          n_in = u + 1;
        }
        if (ok && !in && v <= hi) {
          if (nb < MB) bandj[nb * TILE + r] = j;
          ++nb;
        }
      }
      if (nb > MB) ok = false;                                         // a cluster of near ties: exact completion kernel
      // exact keys of the band, four independent FMA chains at a time; per candidate the chain is
      // acc = fma(x_q[c], x_j[c], acc) for c ascending from acc = 0 - the bits of the fp32 kernel
      const int nbe = ok ? nb : 0;
      int nb_max = nbe;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) nb_max = max(nb_max, __shfl_xor_sync(0xffffffffu, nb_max, o));
      for (int m0 = 0; m0 < nb_max; m0 += 4) {
        uint32_t jj[4];
        float dot[4];
#pragma unroll
        for (int i4 = 0; i4 < 4; ++i4) {
          jj[i4] = m0 + i4 < nbe ? bandj[(m0 + i4) * TILE + r] : static_cast<uint32_t>(qg);
          dot[i4] = 0.f;
        }
        // idle chains issue no loads: every lane-load is its own 32-byte sector request, and the request rate of
        // such divergent loads - not bytes, not latency - is what bounds this phase
#pragma unroll 1
        for (int c = 0; c < C; c += 8) {
          float q8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (m0 < nbe) ldg_f8(xqp + c, q8);
#pragma unroll
          for (int i4 = 0; i4 < 4; ++i4) {
            float w[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (m0 + i4 < nbe) ldg_f8(xtb + jj[i4] * static_cast<uint32_t>(C) + c, w);
#pragma unroll
            for (int i = 0; i < 8; ++i) dot[i4] = fmaf(q8[i], w[i], dot[i4]);
          }
        }
#pragma unroll
        for (int i4 = 0; i4 < 4; ++i4)
          if (m0 + i4 < nbe) band[(m0 + i4) * TILE + r] = make_key((sqq + (-2.0f * dot[i4])) + __ldg(sqb + jj[i4]), jj[i4]);
      }
      if (ok) {
        const int need = K - n_in;                                     // 0 <= need <= nb
        int pos = n_in;
        for (int i = 0; i < nb; ++i) {
          const uint64_t ki = band[i * TILE + r];
          int rank = 0;
          for (int i2 = 0; i2 < nb; ++i2) rank += band[i2 * TILE + r] < ki ? 1 : 0;
          if (rank < need) selrow[pos++] = static_cast<int>(static_cast<uint32_t>(ki));
        }
      }
      sm.ok[g][r] = ok ? 1 : 0;
      if (!ok) {
        const int slot = atomicAdd(t.fail_count, 1);
        t.fail_list[slot] = b * N + qg;
      }
      t4_group_sync(g);
      cta_epilogue_wide<4, false, true, 10>(a, b, q0, nullptr, sm.ok[g], sel, sel_ld, nullptr, 0, r);
    } else {
    // ---- exact re-rank of the listed candidates (fp32 FMA chain, channels ascending) --------------------------
    uint64_t* list = reinterpret_cast<uint64_t*>(qbase + g * T4_QBYTES);   // [KP][TILE]
    {
      // Two halves of KP/2 candidates (register budget of a 9-warp CTA at one CTA per SM).  Channels in chunks of 8 in the outer
      // loop, candidates in the inner one: KP/2 independent FMA chains in flight; per candidate the chain is
      // acc = fma(x_q[c], x_j[c], acc) for c ascending from acc = 0 - the bits of the fp32 kernel.
      constexpr int HN = KP / 2;
      int e = 0;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        float dex[HN];
#pragma unroll
        for (int u = 0; u < HN; ++u) dex[u] = 0.f;
#pragma unroll 1
        for (int c = 0; c < C; c += 8) {
          float q8[8];
          ldg_f8(xqp + c, q8);
#pragma unroll
          for (int u = 0; u < HN; ++u) {
            const uint32_t en = lk[half * HN + u];
            const uint32_t j = en != 0xFFFFFFFFu ? (en & 0xFFFu) : static_cast<uint32_t>(qg);
            float w[8];
            ldg_f8(xtb + j * static_cast<uint32_t>(C) + c, w);
#pragma unroll
            for (int i = 0; i < 8; ++i) dex[u] = fmaf(q8[i], w[i], dex[u]);
          }
        }
        // insertion by exact key into the exact-sorted prefix [0, e)
#pragma unroll
        for (int u = 0; u < HN; ++u) {
          const uint32_t en = lk[half * HN + u];
          const bool listed = en != 0xFFFFFFFFu;
          const uint32_t j = en & 0xFFFu;
          if (listed && !(a.exclude_self && j == static_cast<uint32_t>(qg))) {   // self exclusion (loop=False)
            const float d = (sqq + (-2.0f * dex[u])) + __ldg(sqb + j);
            const uint64_t key = make_key(d, j);
            int i = e;
            while (i > 0) {
              const uint64_t prev = list[(i - 1) * TILE + r];
              if (prev < key) break;
              list[i * TILE + r] = prev;
              --i;
            }
            list[i * TILE + r] = key;
            ++e;
          }
        }
      }
      for (int i = e; i < KP; ++i) list[i * TILE + r] = KEY_MAX;
    }
    // ---- certificate (thread = query): see knn_tc_kernel -------------------------------------------------------
    {
      const uint64_t kth = list[(a.K - 1) * TILE + r];
      bool ok = kth != KEY_MAX;
      if (ok && cut < INFINITY) {
        const float dk = ordered_to_float(static_cast<uint32_t>(kth >> 32));
        ok = (dk + eps < cut);
      }
      sm.ok[g][r] = ok ? 1 : 0;
      if (!ok) {
        const int slot = atomicAdd(t.fail_count, 1);
        t.fail_list[slot] = b * N + qg;
      }
    }
    t4_group_sync(g);
    // ---- consumer: sel lives in the group's candidate buffer ---------------------------------------------------
    cta_epilogue_wide<4, false, false, 10>(a, b, q0, list, sm.ok[g], sel, sel_ld, nullptr, 0, r);
    }
    }
  }
}

inline bool knn_tc4_list_ok(int kp, int k) {
  return (kp == 16 || kp == 28) && static_cast<size_t>(TILE) * tc_sel_ld(k) * 4 <= static_cast<size_t>(T4_CBUF_BYTES);
}

template <int KP>
inline int launch_knn_tc4_inst(const TcArgs& t, dim3 grid, cudaStream_t stream) {
  DGCN_ENSURE_SMEM((knn_tc4_kernel<KP>), T4_SMEM_BYTES);
  knn_tc4_kernel<KP><<<grid, T4_THREADS, T4_SMEM_BYTES, stream>>>(t);
  return DGCN_OK;
}
int launch_knn_tc4(int kp, const TcArgs& t, dim3 grid, cudaStream_t stream);

}  // namespace dgcn

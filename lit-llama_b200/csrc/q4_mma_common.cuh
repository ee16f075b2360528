// Pieces shared by the mma.sync int4 decode kernels (q4_gemv.cu: one activation row, int8 MMA; q4_gemv_batch.cu:
// 2..8 rows, f16 MMA): tile geometry, mbarrier / TMA / named-barrier wrappers, the MMA wrappers, the f16 unpack.
#pragma once
#include "b2l_common.cuh"

namespace b2l {
namespace q4mv {

constexpr int RB = 16;                        // rows per row block
constexpr int KB = 64;                        // k per k block (4 MMAs)
constexpr int KB_BYTES = 512;                 // one (row block, k block): 32 lanes x 16 B
constexpr int NCW = 8;                        // consumer warps
constexpr int KBP_PER_STAGE = 16;             // k-block positions per stage (2 per consumer warp)
constexpr int MAX_HALVES = 2;                 // a unit is one or two consecutive 16-row blocks sharing the B fragments
constexpr int HALF_STAGE_BYTES = KBP_PER_STAGE * KB_BYTES;   // 8 KB
constexpr int STAGE_BYTES = MAX_HALVES * HALF_STAGE_BYTES;   // 16 KB
constexpr int MAX_STAGES = 13;
constexpr int PRODUCER_WARP = NCW;            // warp 8
constexpr int NTHREADS = (NCW + 2) * 32;      // 320

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t a, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t a) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(a) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t a, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t a, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(a), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(mbar)
      : "memory");
}
// barrier ids are immediates so that ptxas reserves only the 8 barriers this kernel uses
template <int ID> __device__ __forceinline__ void bar_sync_c(int n) { asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(n) : "memory"); }
template <int ID> __device__ __forceinline__ void bar_arrive_c(int n) { asm volatile("bar.arrive %0, %1;" ::"n"(ID), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int n) {
  switch (id) {
    case 1: bar_sync_c<1>(n); break;
    case 2: bar_sync_c<2>(n); break;
    case 3: bar_sync_c<3>(n); break;
    case 4: bar_sync_c<4>(n); break;
    case 5: bar_sync_c<5>(n); break;
    case 6: bar_sync_c<6>(n); break;
    default: bar_sync_c<7>(n); break;
  }
}
__device__ __forceinline__ void named_bar_arrive(int id, int n) {
  switch (id) {
    case 4: bar_arrive_c<4>(n); break;
    case 5: bar_arrive_c<5>(n); break;
    case 6: bar_arrive_c<6>(n); break;
    default: bar_arrive_c<7>(n); break;
  }
}

__device__ __forceinline__ void mma_f16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// IMMA.16832.U8.S8: D (16 x 8, s32) += A (16 x 32, u8, row) * B (32 x 8, s8, col)
__device__ __forceinline__ void mma_u8s8_16832(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// (w & mask) | magic in one LOP3: masks and magic live in registers
__device__ __forceinline__ uint32_t lop_and_or(uint32_t a, uint32_t mask, uint32_t magic) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(mask), "r"(magic));
  return d;
}
// two fp32 -> packed fp16 (lo in bits 0..15), saturating (q4_batch_prep_kernel scales every row below 2^15 first)
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}

// packed fp16 a - b
__device__ __forceinline__ uint32_t hsub2_u32(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}

// One k-block position (64 k) of NH 16-row halves: LDS.128 per half, 1 shift + 4 LOP3 + 2 HADD2 per word, 4 MMAs per
// half.  The lower k half gets q itself (1024 + q - 1024, exact): with the 1024 left in, the fp32 accumulator would
// carry 1024 x for every activation x and round at that magnitude, so an output whose level sits at its zero point on
// a massive channel (|x| ~ 1e4) would be off by many ulps.  The upper half keeps 1024 + 16 q against x / 16, i.e.
// q x + 64 x: a bias 16 times smaller, removed with the exact row sums in the epilogue.
template <int NH>
__device__ __forceinline__ void kblock_mma(float (&acc)[MAX_HALVES][2][4], const uint8_t* wbase, const uint4& xa, const uint4& xb,
                                           uint32_t kmask, uint32_t kmask4, uint32_t kmagic) {
  const uint32_t bb[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
  for (int h = 0; h < NH; ++h) {
    const uint4 wv = *reinterpret_cast<const uint4*>(wbase + h * HALF_STAGE_BYTES);
    const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      uint32_t a[4];
      const uint32_t w8 = ww[c] >> 8;
      a[0] = hsub2_u32(lop_and_or(ww[c], kmask, kmagic), kmagic);   // row g,     k 2t..2t+1 : q
      a[1] = hsub2_u32(lop_and_or(w8, kmask, kmagic), kmagic);      // row g + 8, k 2t..2t+1 : q
      a[2] = lop_and_or(ww[c], kmask4, kmagic);  // row g,     k 2t+8..2t+9   : 1024 + 16 q  (x / 16 in B)
      a[3] = lop_and_or(w8, kmask4, kmagic);     // row g + 8, k 2t+8..2t+9   : 1024 + 16 q
      mma_f16_16816(acc[h][c & 1], a, bb[2 * c], bb[2 * c + 1]);
    }
  }
}

}  // namespace q4mv
}  // namespace b2l

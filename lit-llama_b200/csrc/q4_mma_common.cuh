// Pieces shared by the mma.sync int4 decode kernels (q4_gemv.cu: one activation row, int8 MMA; q4_gemv_batch.cu:
// 2..8 rows, f16 MMA): tile geometry, the named-barrier switches, the f16 MMA and unpack, and the int8 kernels'
// exact activation conversion.
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

// bar_sync_c / bar_arrive_c (b2l_common.cuh) for a barrier id known only at run time: a switch over immediates
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

// ---- the exact activation conversion of the int8-MMA GEMVs (q4_gemv.cu).  q4_gemv_kernel and w8_batch_prep_kernel
// (w8_gemv_batch.cu) both run it on 256 threads, thread tid owning elements 8 (c 256 + tid) .. + 7 of chunk c, and
// reduce in the same order, so row n of a batch gets the batch-1 kernel's sh and X.
// [RMSNorm], power-of-two scaling, balanced digits in B-fragment order, exact sum(X).  Every CTA of the batch-1
// kernel converts the whole row and cannot start its main loop before this is done: the conversion is written for
// instruction count.  Per pair of elements: packed bf16 max / multiplies, ONE fma that both scales and rounds to an
// integer (x * 2^sh + 1.5 * 2^23: the integer sits in the mantissa, |X| < 2^22 -- no F2I, which runs at a quarter of
// the fp32 rate), the balanced digits straight from those bits with one add and one xor.
constexpr uint32_t MAGIC_BITS = 0x4B400000u;   // 1.5 * 2^23
constexpr int MAX_K = 12 * NCW * 32 * 8;       // 24576: 12 chunks of 2048 activations held in registers (MAXC)

// Pass 1 over this thread's MAXC chunks: the sum of bf16-rounded squares (RMSNorm, model.py:274: one HMUL2 is the
// exactly-rounded bf16 product the reference computes) and max |x|, or with RMSNorm max_k |bf16(g_k x_k)|, which
// bounds the normalised values
template <int MAXC>
__device__ __forceinline__ void act_pass1(const uint4 (&xv)[MAXC], const uint4 (&gv)[MAXC], int nchunk, bool norm, float& ss,
                                          float& mx) {
  ss = 0.f;
  __nv_bfloat162 amax2 = __float2bfloat162_rn(0.f);
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    if (c < nchunk) {
      const uint32_t w[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w};
      const uint32_t g[4] = {gv[c].x, gv[c].y, gv[c].z, gv[c].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
        if (norm) {
          amax2 = __hmax2(amax2, __habs2(__hmul2(v, *reinterpret_cast<const __nv_bfloat162*>(&g[q]))));
          const __nv_bfloat162 sq = __hmul2(v, v);
          const uint32_t su = *reinterpret_cast<const uint32_t*>(&sq);
          ss += __uint_as_float(su << 16) + __uint_as_float(su & 0xffff0000u);
        } else {
          amax2 = __hmax2(amax2, __habs2(v));
        }
      }
    }
  }
  mx = fmaxf(__low2float(amax2), __high2float(amax2));
}

struct ActScale {
  __nv_bfloat162 rinv2;   // the RMSNorm factor, a bf16 value (1 without RMSNorm)
  float scale;            // 2^sh
  int sh;
};

// sh and 2^sh from the row's sum of squares and max (pass 1 reduced over the 256 threads)
template <int NDIG>
__device__ __forceinline__ ActScale act_scale(float ss, float mx, bool norm, int K, float eps) {
  float rinv = 1.f;
  if (norm) {
    // The normalised value is v_k = bf16(g_k bf16(x_k rinv)) (rinv is a bf16 value), and pass 1 took
    // p_k = bf16(g_k x_k).  With u = 2^-8, the unit roundoff of bf16:
    //   |v_k| <= |g_k x_k| rinv (1 + u)^2 <= |p_k| rinv (1 + u)^2 / (1 - u) < 1.012 |p_k| rinv,
    // and the two fp32 roundings below lose less than 2^-23, so mx > max_k |v_k|: |X| < 2^22 follows from the
    // choice of sh.  (A product below bf16's normal range 2^-126 may round further; such elements have
    // |v_k| < 2^-125 rinv, and sh <= 126 keeps them below 2^22 for any rinv < 2^21, i.e. eps > 2^-42.)
    // A bound on max|x| max|g| instead overshoots by up to max|g| / g_k when the largest activation carries a small
    // scale (LLaMA's massive channels do), and the digit grid below coarsens by the same factor.
    rinv = rms_rinv(ss, K, eps);
    mx = mx * rinv * 1.02f;
  }
  // 2^sh: the largest power of two with max|v| * 2^sh < 2^(8 NDIG - 2)
  const int e = (int)((__float_as_uint(mx) >> 23) & 0xffu) - 127;   // mx < 2^(e + 1)
  int sh = (8 * NDIG - 3) - e;
  sh = max(-126, min(126, sh));
  ActScale a;
  a.rinv2 = __float2bfloat162_rn(rinv);  // rinv is already a bf16 value
  a.scale = __uint_as_float((uint32_t)(sh + 127) << 23);
  a.sh = sh;
  return a;
}

// Eight activations (xv: 4 bf16 pairs, gv: their RMSNorm scales) -> dj[j][n] = digit n of elements 4j .. 4j+3 (B
// register j of lane t, column n), and sxu += their X (modulo 2^32)
__device__ __forceinline__ void act_digits(const uint4& xv, const uint4& gv, bool norm, const ActScale& a, uint32_t (&dj)[2][3],
                                           uint32_t& sxu) {
  uint32_t w[4] = {xv.x, xv.y, xv.z, xv.w};
  if (norm) {
    const uint32_t g[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
      const __nv_bfloat162 gg = *reinterpret_cast<const __nv_bfloat162*>(&g[q]);
      const __nv_bfloat162 y2 = __hmul2(gg, __hmul2(v, a.rinv2));  // bf16(scale * bf16(x * rinv)), model.py:276-277
      w[q] = *reinterpret_cast<const uint32_t*>(&y2);
    }
  }
  const float magic = __uint_as_float(MAGIC_BITS);
  uint32_t xd[8];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    // x * 2^sh is exact in fp32 (8-bit significand, power-of-two scale): the fma rounds once, to nearest even,
    // and leaves MAGIC_BITS + X in the result's bit pattern
    const uint32_t b0 = __float_as_uint(__fmaf_rn(__uint_as_float(w[q] << 16), a.scale, magic));
    const uint32_t b1 = __float_as_uint(__fmaf_rn(__uint_as_float(w[q] & 0xffff0000u), a.scale, magic));
    sxu += b0 + b1;                                          // the 2 MAGIC_BITS per pair are removed below
    // the balanced base-256 digits of X (byte 3 is unused): ((uint32_t)X + 0x808080) ^ 0x808080
    xd[2 * q] = (b0 + (0x00808080u - MAGIC_BITS)) ^ 0x00808080u;
    xd[2 * q + 1] = (b1 + (0x00808080u - MAGIC_BITS)) ^ 0x00808080u;
  }
  sxu -= 8u * MAGIC_BITS;
  // 4 x 3 byte transposes: word (j, n) = digit n of elements 4j .. 4j+3
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint32_t lo01 = __byte_perm(xd[4 * j], xd[4 * j + 1], 0x5140), hi01 = __byte_perm(xd[4 * j], xd[4 * j + 1], 0x7362);
    const uint32_t lo23 = __byte_perm(xd[4 * j + 2], xd[4 * j + 3], 0x5140), hi23 = __byte_perm(xd[4 * j + 2], xd[4 * j + 3], 0x7362);
    dj[j][0] = __byte_perm(lo01, lo23, 0x5410);
    dj[j][1] = __byte_perm(lo01, lo23, 0x7632);
    dj[j][2] = __byte_perm(hi01, hi23, 0x5410);
  }
}

}  // namespace q4mv
}  // namespace b2l

// Prefill-shaped int4 weight-only GEMM on the Hopper tensor cores (wgmma): y[M, N] = x[M, K] . dequant(W)[N, K]^T
// for M > 16 (prompt processing, no-cache forward, evaluation; BASELINE.json configs[3] prefill 8 x 512).
//
// Replaces ColBlockQuantizedLinear.forward (lit_llama/quantization.py:413-423) and the Triton kernel
// linear_kernel_4bit_weight (quantization.py:187-333: tiles up to 256 x 256, dequantise inside the tile loop) for
// 4-bit weights with one (scale, zero) per output row.
//
// One CTA computes a 128 (tokens) x 128 (output features) tile of y over the full K:
//   warpgroups 0 and 1 (warps 0..7): wgmma.mma_async.m64n128k16 (bf16 x bf16 -> fp32), both operands from shared
//       memory (K-major canonical core-matrix layout, no swizzle); warpgroup h owns token rows 64 h .. 64 h + 63 and
//       keeps its 64 x 128 fp32 accumulator in registers; a stage is released to the producers once the wgmma group
//       that read it has completed (wgmma.wait_group 1 keeps one group in flight);
//   warpgroup 2 (warps 8..11, 128 threads = the 128 weight rows of the tile), per 64-wide k stage:
//       * the activation tile [128 tokens][64 k]: ONE tensor-map TMA copy (cp.async.bulk.tensor.3d) per stage.  x is
//         described to the TMA unit as a 3-D tensor (8 elements = 16 B | M rows, stride ldx | K/8 chunks, stride 16 B),
//         so a box of 8 x 128 x 8 lands in shared memory as [k chunk][row][16 B] -- exactly the no-swizzle
//         K-major core-matrix order wgmma reads; rows beyond M are zero-filled by the TMA unit;
//       * two LDG.128 of packed levels per thread (load-time tiling b2l_q4_tile: a row's 32 levels of a k slab in
//         16 bytes, nibble order chosen so that (w >> 4s) & 0x000f000f | 0x43004300 IS the bf16 pair
//         (128 + level[k], 128 + level[k+1])), dequantised with the reference's own rounding:
//         level = v - 128 (exact), level - zero (bf16), * scale (bf16) -- bit-identical to get_weight
//         (quantization.py:392-411), so the GEMM sees exactly the matrix the reference's dense branch multiplies;
//       * 16-byte st.shared of 8 consecutive k of a row = one row of a core matrix; fence.proxy.async; mbarrier arrive;
//   epilogue: each MMA thread converts its accumulator fragment to bf16 and stores pairs of output features.
// gptq.int8 (b2l_w8_gemm) is the same kernel with W8 = true: only the producers differ (w8_load below).
// SRC = SRC_I8 / SRC_I8_HALF (B2L_F_GEMM_I8 [| _LO / _HI]) swaps the weight source for the batch-1 decode tilings
// (b2l_q4_tile_i8 / b2l_w8_tile_i8, the one resident copy of a compacted model; i8_producer below): the producers
// write the same bf16 values to the same shared-memory positions, so the MMAs and the result are unchanged bit for bit.
// NLL = true (b2l_q4_gemm_nll / b2l_w8_gemm_nll) replaces the epilogue's store: the quad of lanes holding a token row
// reduces the bf16-rounded accumulators of the tile's 128 columns to (max, sum of exp) into a workspace, and the lane
// holding the row's target column records its logit (nll_common.cuh; csrc/nll.cu merges the tiles).
#include "b2l_common.cuh"
#include "nll_common.cuh"

namespace b2l {
namespace q4gm {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int A_BYTES = BM * BK * 2;           // 16 KB: [8 k-columns][128 token rows][16 B]
constexpr int B_BYTES = BN * BK * 2;           // 16 KB: [8 k-columns][128 weight rows][16 B]
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int NSTAGE = 4;
constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + 256;
constexpr int NMMA = 256;                      // two MMA warpgroups
constexpr int NPROD = 128;                     // producer threads = weight rows of the tile
constexpr int NTHREADS = NMMA + NPROD;
constexpr int LBO_A = BM * 16;                 // bytes between adjacent 8-k columns of the activation operand
constexpr int LBO_B = BN * 16;                 // bytes between adjacent 8-k columns of the weight operand
constexpr int SBO = 128;                       // bytes between adjacent 8-row groups
// weight source: b2l_q4_tile (4 bits) / quant_weight (8 bits), the batch-1 tiling, or one half of an interleaved one
constexpr int SRC_OWN = 0, SRC_I8 = 1, SRC_I8_HALF = 2;

struct Params {
  CUtensorMap xmap;        // 3-D view of x (see above); must stay the first member (64-byte alignment)
  const __nv_bfloat16* x; int ldx;
  const uint8_t* qwt;      // b2l_q4_tile layout: [N/128 tiles][K/32 slabs][128 rows][16 B]; 8 bits: quant_weight [K][N]
  const void* scales; const void* zeros; int szdt;
  __nv_bfloat16* y; int ldy;
  int M, N, K;
  int half;                // SRC_I8_HALF only: 0 = rows 0..7, 1 = rows 8..15 of every 16-row block of a 2N-row tiling
  const void* targets; int tgt_i64;   // NLL only: targets [M], partials [N/128][M], target logits [M]
  float2* part; float* tl;
};

// D[64 x 128] (fp32, registers) += A[64 x 16] (smem) * B[16 x 128] (smem), both K-major bf16
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1)
      : "memory");
}
__device__ __forceinline__ void reg_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// 8-bit levels (gptq.int8): producer thread pt owns weight rows n0 + 4 (pt % 32) .. + 3 and k 16 (pt / 32) .. + 15 of
// a stage.  Sixteen 4-byte loads from quant_weight in the reference layout (uint8 [K][N], N-contiguous: a warp reads
// 128 consecutive bytes per k) give 4 rows x 16 k; each level becomes bf16 exactly through the fp32 mantissa
// (2^23 + lv - 2^23: every level 0..255 is a bf16 value, which the int4 trick 0x4300 | lv is not beyond 127).
__device__ __forceinline__ void w8_load(uint32_t (&wq)[16], const uint8_t* qw, int N, int row0, int k0, bool vec) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const uint8_t* src = qw + (size_t)(k0 + j) * N + row0;
    if (vec) {
      wq[j] = __ldg(reinterpret_cast<const uint32_t*>(src));
    } else {   // ragged N (not a multiple of 4) or the last rows: byte loads, zero beyond N
      uint32_t w = 0;
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (row0 + r < N) w |= (uint32_t)__ldg(src + r) << (8 * r);
      wq[j] = w;
    }
  }
}

// (level - zero) * scale of the bf16 level pair in `v` (0x4300 | (128 + level) per half at 4 bits, see below) with
// get_weight's roundings
__device__ __forceinline__ uint32_t q4_pair(uint32_t v, __nv_bfloat162 z2, __nv_bfloat162 sc2) {
  const __nv_bfloat162 c128 = __float2bfloat162_rn(128.f);
  __nv_bfloat162 t = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&v), c128);   // level, exact
  t = __hmul2(__hsub2(t, z2), sc2);
  return *reinterpret_cast<const uint32_t*>(&t);
}
// the same for the 8-bit levels in bytes r and r + 1 of `w` (the 2^23 mantissa trick of the W8 producer)
__device__ __forceinline__ uint32_t w8_pair(uint32_t w, int r, __nv_bfloat162 z2, __nv_bfloat162 sc2) {
  const float two23 = 8388608.f;
  const float f0 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540u | (uint32_t)r)) - two23;
  const float f1 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540u | (uint32_t)(r + 1))) - two23;
  __nv_bfloat162 t = __floats2bfloat162_rn(f0, f1);   // level pair, exact
  t = __hmul2(__hsub2(t, z2), sc2);
  return *reinterpret_cast<const uint32_t*>(&t);
}

template <bool W8, bool NLL, int SRC>
__global__ void __launch_bounds__(NTHREADS, 1) q4_gemm_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bars = sbase + NSTAGE * STAGE_BYTES;      // full[NSTAGE], empty[NSTAGE]
  const uint32_t bar_full = bars, bar_empty = bars + NSTAGE * 8;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int n_kt = p.K / BK;

  if (tid == 0) {
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(bar_full + i * 8, NPROD / 32 + 1);   // one elected arrival per producer warp + the TMA issuer's expect_tx
      mbar_init(bar_empty + i * 8, NMMA / 32);       // one arrival per MMA warp once its wgmma group has completed
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < NMMA / 32) {
    // ===================== MMA warpgroups =====================
    const int h = warp >> 2;                       // token rows 64 h .. 64 h + 63 of the tile
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kt = 0; kt < n_kt; ++kt) {
      const int st = kt % NSTAGE;
      mbar_wait(bar_full + st * 8, (uint32_t)(kt / NSTAGE) & 1u);
      const uint32_t a_base = sbase + st * STAGE_BYTES, b_base = a_base + A_BYTES;
      wgmma_fence();
      reg_fence(acc);
#pragma unroll
      for (int j = 0; j < BK / 16; ++j)
        wgmma_m64n128k16(acc, make_desc(a_base + h * 64 * 16 + j * 2 * LBO_A, LBO_A, SBO), make_desc(b_base + j * 2 * LBO_B, LBO_B, SBO));
      wgmma_commit();
      wgmma_wait<1>();   // the group of stage kt - 1 has completed
      reg_fence(acc);
      if (kt > 0 && lane == 0) mbar_arrive(bar_empty + ((kt - 1) % NSTAGE) * 8);
    }
    wgmma_wait<0>();
    reg_fence(acc);
    // ===================== epilogue: registers -> bf16 -> y.  acc[4 c + e]: token row 16 (warp % 4) + lane / 4
    // (+ 8 for e >= 2), output feature 8 c + 2 (lane % 4) + (e & 1)
    const int mr = m0 + h * 64 + (warp & 3) * 16 + (lane >> 2);
    const int nc = n0 + 2 * (lane & 3);
    if constexpr (NLL) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float v[32];
#pragma unroll
        for (int c = 0; c < BN / 8; ++c) {   // bf16(acc) as the store below would write it; -inf past N
          const int n = nc + 8 * c;
          v[2 * c] = n < p.N ? rbf(acc[4 * c + 2 * hh]) : -INFINITY;
          v[2 * c + 1] = n + 1 < p.N ? rbf(acc[4 * c + 2 * hh + 1]) : -INFINITY;
        }
        nll::tile_row(v, mr + 8 * hh, p.M, blockIdx.x, nc, p.N, p.targets, p.tgt_i64, p.part, p.tl);
      }
    } else {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = mr + 8 * hh;
        if (m >= p.M) continue;
        __nv_bfloat16* dst = p.y + (size_t)m * p.ldy;
#pragma unroll
        for (int c = 0; c < BN / 8; ++c) {
          const int n = nc + 8 * c;
          const float v0 = acc[4 * c + 2 * hh], v1 = acc[4 * c + 2 * hh + 1];
          if (n + 1 < p.N && ((reinterpret_cast<uintptr_t>(dst + n) & 3) == 0)) {
            *reinterpret_cast<__nv_bfloat162*>(dst + n) = __floats2bfloat162_rn(v0, v1);
          } else {
            if (n < p.N) dst[n] = f2bf(v0);
            if (n + 1 < p.N) dst[n + 1] = f2bf(v1);
          }
        }
      }
    }
  } else if constexpr (SRC != SRC_OWN) {
    // ===================== producers, batch-1 tilings: activations (TMA) + dequantised weights =====================
    // A (16-row block rb, k block kb) tile of b2l_q4_tile_i8 is 512 B at (rb * K/64 + kb) * 512: lane (g, t) holds in
    // word 2c + j, byte i, the levels of rows g (low nibble) and g + 8 (high nibble) at k = 64 kb + 32 c + 8 t + 4 j + i.
    // Of b2l_w8_tile_i8 it is 1024 B, [c][32 lanes][16 B]: word w of lane (g, t) holds row g + 8 (w & 1) at
    // k = 64 kb + 32 c + 8 t + 4 (w >> 1) + 0..3.  Either way one lane's 16 B of chunk c are 8 consecutive k (the
    // core-matrix row of k column 4 c + t) of rows g and g + 8.  A 64-wide k stage is one k block; producer warp pw
    // loads NCH consecutive row blocks, 2 of 8 (plain), or 4 of the 16 interleaved blocks whose half p.half holds this
    // layer's 128 rows (SRC_I8_HALF: layer row o is row 16 (o / 8) + o % 8 + 8 half of the 2N-row tiling), which
    // reads twice the bytes it uses.  Thread `lane` takes tile lane (g, t) = (lane % 8, lane / 8): the 8 threads of a
    // shared-memory store phase then write 8 consecutive rows of one k column, 128 contiguous bytes (lane order
    // would put 4 of them 2 KB apart, in the same banks).
    constexpr bool HALF = SRC == SRC_I8_HALF;
    constexpr int NCH = HALF ? 4 : 2;                // row blocks per producer thread and stage
    constexpr int RPB = HALF ? 1 : 2;                // rows of a block this layer owns per lane
    constexpr int NLD = W8 ? 2 : 1;                  // 16-byte loads per lane and block (k chunks c at 8 bits)
    constexpr int TILE_B = W8 ? 1024 : 512;
    const int pw = (tid - NMMA) >> 5, g = lane & 7, t = lane >> 3;
    const int n_kb = p.K / BK;
    const int n_rb = HALF ? p.N / 8 : (p.N + 15) / 16;   // row blocks of the tiling that hold this layer's rows
    const int hsel = HALF ? p.half : 0;
    const uint8_t* src[NCH];
    bool ok[NCH];
    __nv_bfloat162 sc2[NCH][RPB], z2[NCH][RPB];
    int trow[NCH][RPB];                              // row of the 128-row tile
#pragma unroll
    for (int b = 0; b < NCH; ++b) {
      const int q = NCH * pw + b;                    // block of the tile
      const int rb = (HALF ? n0 / 8 : n0 / 16) + q;  // block of the tiling
      ok[b] = rb < n_rb;
      src[b] = p.qwt + (size_t)min(rb, n_rb - 1) * n_kb * TILE_B + (4 * g + t) * 16;
#pragma unroll
      for (int r = 0; r < RPB; ++r) {
        trow[b][r] = HALF ? 8 * q + g : 16 * q + g + 8 * r;
        const int row_n = n0 + trow[b][r];
        float sc_f = 0.f, z_f = 0.f;
        if (row_n < p.N) { sc_f = load_sz(p.scales, p.szdt, row_n); z_f = load_sz(p.zeros, p.szdt, row_n); }
        sc2[b][r] = __float2bfloat162_rn(sc_f); z2[b][r] = __float2bfloat162_rn(z_f);
      }
    }
    uint4 wq[NCH][NLD];
    auto load_w = [&](int kt) {
#pragma unroll
      for (int b = 0; b < NCH; ++b)
#pragma unroll
        for (int c = 0; c < NLD; ++c) {
          wq[b][c] = make_uint4(0, 0, 0, 0);
          if (ok[b]) wq[b][c] = __ldg(reinterpret_cast<const uint4*>(src[b] + (size_t)kt * TILE_B + c * 512));
        }
    };
    load_w(0);
    for (int kt = 0; kt < n_kt; ++kt) {
      const int st = kt % NSTAGE;
      if (kt >= NSTAGE) mbar_wait(bar_empty + st * 8, (uint32_t)(kt / NSTAGE - 1) & 1u);
      const uint32_t a_base = sbase + st * STAGE_BYTES, b_base = a_base + A_BYTES;
      if (tid == NMMA) {
        mbar_expect_tx(bar_full + st * 8, A_BYTES);
        tma_load_3d(a_base, &p.xmap, 0, m0, kt * (BK / 8), bar_full + st * 8);
      }
      uint4 w[NCH][NLD];
#pragma unroll
      for (int b = 0; b < NCH; ++b)
#pragma unroll
        for (int c = 0; c < NLD; ++c) w[b][c] = wq[b][c];
      if (kt + 1 < n_kt) load_w(kt + 1);
#pragma unroll
      for (int b = 0; b < NCH; ++b) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {                // k column 4 c + t
#pragma unroll
          for (int r = 0; r < RPB; ++r) {
            const int hi = HALF ? hsel : r;          // row g + 8 hi of the 16-row block
            uint32_t o[4];
            if constexpr (W8) {
              const uint4 u = w[b][c];
              const uint32_t lo4 = hi ? u.y : u.x, hi4 = hi ? u.w : u.z;   // k 0..3 and 4..7 of the row
              o[0] = w8_pair(lo4, 0, z2[b][r], sc2[b][r]);
              o[1] = w8_pair(lo4, 2, z2[b][r], sc2[b][r]);
              o[2] = w8_pair(hi4, 0, z2[b][r], sc2[b][r]);
              o[3] = w8_pair(hi4, 2, z2[b][r], sc2[b][r]);
            } else {
              const uint4 u = w[b][0];
              const uint32_t wj[2] = {c ? u.z : u.x, c ? u.w : u.y};     // words 2 c, 2 c + 1: k 0..3, 4..7
#pragma unroll
              for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int s = 0; s < 2; ++s) {       // bytes 2 s, 2 s + 1 -> halves of a word, then row g's / g + 8's nibble
                  const uint32_t v = (__byte_perm(wj[j], 0u, s ? 0x4342u : 0x4140u) >> (4 * hi)) & 0x000f000fu;
                  o[2 * j + s] = q4_pair(v | 0x43004300u, z2[b][r], sc2[b][r]);
                }
            }
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(b_base + (4 * c + t) * LBO_B + trow[b][r] * 16),
                         "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
          }
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + st * 8);
    }
  } else if constexpr (W8) {
    // ===================== producers, 8-bit levels: activations (TMA) + dequantised weights =====================
    const int pt = tid - NMMA;
    const int row0 = n0 + 4 * lane, kq = 16 * (pt >> 5);    // 4 rows x 16 k of every stage
    const bool vec = (p.N % 4 == 0) && row0 + 4 <= p.N;
    __nv_bfloat162 sc2[4], z2[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float sc_f = 0.f, z_f = 0.f;
      if (row0 + r < p.N) { sc_f = load_sz(p.scales, p.szdt, row0 + r); z_f = load_sz(p.zeros, p.szdt, row0 + r); }
      sc2[r] = __float2bfloat162_rn(sc_f); z2[r] = __float2bfloat162_rn(z_f);
    }
    const float two23 = 8388608.f;
    uint32_t wq[16];
    if (row0 < p.N) w8_load(wq, p.qwt, p.N, row0, kq, vec);
    for (int kt = 0; kt < n_kt; ++kt) {
      const int st = kt % NSTAGE;
      if (kt >= NSTAGE) mbar_wait(bar_empty + st * 8, (uint32_t)(kt / NSTAGE - 1) & 1u);
      const uint32_t a_base = sbase + st * STAGE_BYTES, b_base = a_base + A_BYTES;
      if (pt == 0) {
        mbar_expect_tx(bar_full + st * 8, A_BYTES);
        tma_load_3d(a_base, &p.xmap, 0, m0, kt * (BK / 8), bar_full + st * 8);
      }
      uint32_t w[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) w[j] = row0 < p.N ? wq[j] : 0u;
      if (kt + 1 < n_kt && row0 < p.N) w8_load(wq, p.qwt, p.N, row0, (kt + 1) * BK + kq, vec);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {       // k-column 2 (pt / 32) + c: 8 consecutive k of row row0 + r
          uint32_t o[4];
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            const uint32_t sel = 0x7540u | (uint32_t)r;   // level byte r under the exponent byte of 2^23
            const float f0 = __uint_as_float(__byte_perm(w[8 * c + 2 * s], 0x4B000000u, sel)) - two23;
            const float f1 = __uint_as_float(__byte_perm(w[8 * c + 2 * s + 1], 0x4B000000u, sel)) - two23;
            __nv_bfloat162 t = __floats2bfloat162_rn(f0, f1);   // level pair, exact
            t = __hmul2(__hsub2(t, z2[r]), sc2[r]);            // (level - zero) * scale with the reference's bf16 roundings
            o[s] = *reinterpret_cast<const uint32_t*>(&t);
          }
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(b_base + (2 * (pt >> 5) + c) * LBO_B + (4 * lane + r) * 16),
                       "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + st * 8);
    }
  } else {
    // ===================== producers: activations (TMA) + dequantised weights =====================
    const int pt = tid - NMMA;                     // 0..127 = weight row of the tile
    const int row_n = n0 + pt;
    const int n_slab = p.K / 32;
    const bool row_ok = row_n < ((p.N + 127) / 128) * 128;     // rows inside the (128-padded) tiling
    const uint8_t* wrow = p.qwt + ((size_t)(row_n >> 7) * n_slab * 128 + (row_n & 127)) * 16;   // + slab * 2048
    float sc_f = 0.f, z_f = 0.f;
    if (row_n < p.N) { sc_f = load_sz(p.scales, p.szdt, row_n); z_f = load_sz(p.zeros, p.szdt, row_n); }
    const __nv_bfloat162 sc2 = __float2bfloat162_rn(sc_f), z2 = __float2bfloat162_rn(z_f);
    const __nv_bfloat162 c128 = __float2bfloat162_rn(128.f);
    uint4 wq[2];
    auto load_w = [&](int kt) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wq[h] = make_uint4(0, 0, 0, 0);
        if (row_ok) wq[h] = __ldg(reinterpret_cast<const uint4*>(wrow + (size_t)(kt * 2 + h) * 2048));
      }
    };
    load_w(0);
    for (int kt = 0; kt < n_kt; ++kt) {
      const int st = kt % NSTAGE;
      if (kt >= NSTAGE) mbar_wait(bar_empty + st * 8, (uint32_t)(kt / NSTAGE - 1) & 1u);
      const uint32_t a_base = sbase + st * STAGE_BYTES, b_base = a_base + A_BYTES;
      // ---- activations: one tensor-map TMA copy of the whole [8 k chunks][128 rows][16 B] tile
      if (pt == 0) {
        mbar_expect_tx(bar_full + st * 8, A_BYTES);
        tma_load_3d(a_base, &p.xmap, 0, m0, kt * (BK / 8), bar_full + st * 8);
      }
      // ---- weights of this stage (loaded one stage ahead), then the next stage's loads
      const uint4 w0 = wq[0], w1 = wq[1];
      if (kt + 1 < n_kt) load_w(kt + 1);
      const uint32_t ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int c = 0; c < 8; ++c) {       // word c = 8 consecutive k = one 16-byte core-matrix row
        uint32_t o[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const uint32_t v = ((ww[c] >> (4 * s)) & 0x000f000fu) | 0x43004300u;          // (128 + level) pair, exact
          __nv_bfloat162 t = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&v), c128);   // level, exact
          t = __hmul2(__hsub2(t, z2), sc2);      // (level - zero) * scale with the reference's bf16 roundings
          o[s] = *reinterpret_cast<const uint32_t*>(&t);
        }
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(b_base + c * LBO_B + pt * 16), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + st * 8);
    }
  }
}

}  // namespace q4gm
}  // namespace b2l

using namespace b2l;
using namespace b2l::q4gm;

namespace {
template <bool W8, bool NLL, int SRC>
int launch(const Params& p, dim3 grid, cudaStream_t stream) {
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(q4_gemm_kernel<W8, NLL, SRC>, SMEM_BYTES, smem_cache)) return rc;
  q4_gemm_kernel<W8, NLL, SRC><<<grid, NTHREADS, SMEM_BYTES, stream>>>(p);
  B2L_LAUNCH_CHECK("q4_gemm_kernel");
  return 0;
}

template <bool W8, bool NLL>
int launch_src(const Params& p, int flags, dim3 grid, cudaStream_t stream) {
  if (flags & (B2L_F_GEMM_I8_LO | B2L_F_GEMM_I8_HI)) return launch<W8, NLL, SRC_I8_HALF>(p, grid, stream);
  if (flags & B2L_F_GEMM_I8) return launch<W8, NLL, SRC_I8>(p, grid, stream);
  return launch<W8, NLL, SRC_OWN>(p, grid, stream);
}

// b2l_q4_gemm (W8 = false: qw_tiled from b2l_q4_tile) and b2l_w8_gemm (W8 = true: quant_weight, uint8 [K][N]), or with
// B2L_F_GEMM_I8 the batch-1 tiling of either width (B2L_F_GEMM_I8_LO / _HI: one half of an interleaved one);
// with `nl` (b2l_*_gemm_nll) the NLL epilogue instead of the store, then the combine kernel
template <bool W8>
int gemm_entry(const b2l_q4_linear_args* a, const b2l_nll_args* nl, b2l_stream_t stream) {
  const bool with_nll = nl != nullptr;
  const char* fn = with_nll ? (W8 ? "b2l_w8_gemm_nll" : "b2l_q4_gemm_nll") : (W8 ? "b2l_w8_gemm" : "b2l_q4_gemm");
  B2L_CHECK_ARG(a != nullptr, "%s: null args", fn);
  B2L_CHECK_ARG(a->x && a->qw_tiled && a->scales && a->zeros && (a->y || with_nll), "%s: null pointer", fn);
  B2L_CHECK_SUPPORTED(a->out_affine.scale == nullptr && a->out_affine.bias == nullptr,
                      "%s: out_affine is not supported (apply b2l_linear_affine to y)", fn);
  B2L_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0, "%s: bad shape", fn);
  B2L_CHECK_SUPPORTED(a->K % BK == 0, "%s: K=%d must be a multiple of %d", fn, a->K, BK);
  B2L_CHECK_ARG(a->ldx >= a->K && a->ldx % 8 == 0 && (a->ldy >= a->N || with_nll), "%s: bad leading dimension (ldx %% 8 == 0)", fn);
  B2L_CHECK_ARG(((uintptr_t)a->x % 16 == 0) && ((uintptr_t)a->qw_tiled % 16 == 0), "%s: x / qw_tiled must be 16-byte aligned", fn);
  B2L_CHECK_ARG(a->sz_dtype == B2L_BF16 || a->sz_dtype == B2L_F32, "%s: bad sz_dtype", fn);
  constexpr int kHalves = B2L_F_GEMM_I8_LO | B2L_F_GEMM_I8_HI;
  B2L_CHECK_SUPPORTED((a->flags & ~(B2L_F_GEMM_I8 | kHalves)) == 0, "%s: unknown flags 0x%x", fn, a->flags);
  B2L_CHECK_ARG((a->flags & kHalves) != kHalves, "%s: B2L_F_GEMM_I8_LO and B2L_F_GEMM_I8_HI exclude each other", fn);
  B2L_CHECK_ARG(!(a->flags & kHalves) || (a->flags & B2L_F_GEMM_I8), "%s: B2L_F_GEMM_I8_LO / _HI need B2L_F_GEMM_I8", fn);
  B2L_CHECK_SUPPORTED(!(a->flags & kHalves) || a->N % 8 == 0,
                      "%s: B2L_F_GEMM_I8_LO / _HI take 8-row groups of an interleaved tiling: N=%d must be a multiple of 8", fn, a->N);
  B2L_CHECK_SUPPORTED(a->prologue == B2L_PRO_NONE && a->epilogue == B2L_EPI_STORE, "%s: plain linear only (no fused prologue / epilogue)", fn);
  if (with_nll) {
    if (int rc = nll::check_args(nl, a->M, fn)) return rc;
  }
  const PFN_cuTensorMapEncodeTiled encode = tensor_map_encoder();
  if (encode == nullptr) {
    set_error("%s: cuTensorMapEncodeTiled is not available from this driver", fn);
    return B2L_E_STATE;
  }
  Params p;
  {
    // x[M, K] (leading dimension ldx) as (8 elements | M rows | K/8 chunks): a box of 8 x 128 x 8 is one stage's tile
    const cuuint64_t dims[3] = {8, (cuuint64_t)a->M, (cuuint64_t)(a->K / 8)};
    const cuuint64_t strides[2] = {(cuuint64_t)a->ldx * 2, 16};
    const cuuint32_t box[3] = {8, (cuuint32_t)BM, (cuuint32_t)(BK / 8)};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult cr = encode(&p.xmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(a->x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("%s: cuTensorMapEncodeTiled failed (%d) for M=%d K=%d ldx=%d", fn, (int)cr, a->M, a->K, a->ldx);
      return B2L_E_ARG;
    }
  }
  p.x = (const __nv_bfloat16*)a->x; p.ldx = a->ldx;
  p.qwt = (const uint8_t*)a->qw_tiled;
  p.scales = a->scales; p.zeros = a->zeros; p.szdt = a->sz_dtype;
  p.y = (__nv_bfloat16*)a->y; p.ldy = a->ldy;
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.half = (a->flags & B2L_F_GEMM_I8_HI) ? 1 : 0;
  p.targets = nullptr; p.tgt_i64 = 0; p.part = nullptr; p.tl = nullptr;
  dim3 grid((a->N + BN - 1) / BN, (a->M + BM - 1) / BM);
  if (!with_nll) return launch_src<W8, false>(p, a->flags, grid, (cudaStream_t)stream);
  uint8_t* ws = (uint8_t*)nl->workspace;
  p.targets = nl->targets; p.tgt_i64 = nl->targets_i64;
  p.part = (float2*)ws; p.tl = (float*)(ws + nll::part_bytes(a->M, a->N));
  if (int rc = launch_src<W8, true>(p, a->flags, grid, (cudaStream_t)stream)) return rc;
  return nll::launch_combine(nl->targets, nl->targets_i64, a->M, a->N, nl->workspace, nl->nll, nl->nll_sum, (cudaStream_t)stream);
}
}  // namespace

extern "C" int b2l_q4_gemm(const b2l_q4_linear_args* a, b2l_stream_t stream) { return gemm_entry<false>(a, nullptr, stream); }

extern "C" int b2l_w8_gemm(const b2l_q4_linear_args* a, b2l_stream_t stream) { return gemm_entry<true>(a, nullptr, stream); }

extern "C" int b2l_q4_gemm_nll(const b2l_q4_linear_args* a, const b2l_nll_args* nl, b2l_stream_t stream) {
  B2L_CHECK_ARG(nl != nullptr, "b2l_q4_gemm_nll: null nll args");
  return gemm_entry<false>(a, nl, stream);
}

extern "C" int b2l_w8_gemm_nll(const b2l_q4_linear_args* a, const b2l_nll_args* nl, b2l_stream_t stream) {
  B2L_CHECK_ARG(nl != nullptr, "b2l_w8_gemm_nll: null nll args");
  return gemm_entry<true>(a, nl, stream);
}

// Batch-1 decode kernel: fused [RMSNorm ->] int4 weight-only GEMV [-> residual | SwiGLU], integer tensor pipe.
//
// Replaces, for gptq.int4 with one (scale, zero) per output row and a single activation row:
//   ColBlockQuantizedLinear.forward      lit_llama/quantization.py:413-423
//   linear_kernel_4bit_weight (Triton)   lit_llama/quantization.py:187-333
//   RMSNorm.forward                      lit_llama/model.py:270-277      (prologue)
//   x + h / silu(a) * b                  lit_llama/model.py:166-167, 252 (epilogue)
//
// The contraction y[o] = scale[o] * sum_k (level[o,k] - zero[o]) * x[k] is evaluated in EXACT integer arithmetic:
//   * the activation row (after the RMSNorm prologue, i.e. the bf16 values the reference feeds its linear) is
//     scaled by a power of two 2^sh chosen from max|x| and rounded to X[k] (|X| < 2^22: 14 bits of dynamic range
//     below the largest element before an 8-bit significand loses a bit, and a rounding unit of 2^-22 max|x| from
//     there on), then split into three balanced base-256 digits X = sum_j d_j 256^j, d_j in [-128, 127];
//   * mma.sync.m16n8k32 (u8 x s8 -> s32, SASS IMMA.16832.U8.S8) has 8 result columns and a single activation row
//     needs one: digit plane j is column j, so all digits cost ONE MMA per 16 x 32 weight tile;
//   * a packed byte holds two levels.  It is fed to the tensor core UNMASKED as the operand of row g (value
//     level[g] + 16 level[g+8]) and with the low nibbles masked off as the operand of row g + 8 (16 level[g+8]):
//     one LOP3 per word, and the epilogue recovers row g = D[g] - D[g+8], row g + 8 = D[g+8] / 16;
//   * int32 accumulators cannot overflow for K <= 65536 (255 * 127 * K < 2^31); digits are recombined in int64 and
//     the zero point is removed with the exact sum of X: y = scale * 2^-sh * (sum level X - zero * sum X).
// An IMMA.16832 consumes 512 levels behind 2 LOP3 where the f16 form (HMMA.16816) consumes 256 behind 5 ALU ops
// (issue rates: tools/diag.py imma_rate / hmma_rate).  Results do not depend on the order of the K split, carry no
// 1024-bias cancellation, and have no fp16 range limit on the activations.
//
// Why not wgmma here: its A operand would first have to be expanded to 16-bit lanes by the same ALUs (>= 4 LOP3 per
// packed word), and a 64-row wgmma tile wastes 63 of 64 rows on a single activation row; the IMMA form needs 1 LOP3
// per packed word.  wgmma carries the M > 8 shapes.
//
// Data movement is unchanged from round 1: a persistent CTA owns 16-row blocks over the FULL K, a producer warp
// streams 16 KB stages with TMA bulk copies into an mbarrier ring (issued before griddepcontrol.wait, so the
// weights of this linear stream while the previous kernel drains), 8 consumer warps split K inside a stage.
//
// Weight layout (b2l_q4_tile_i8): [N/16 row blocks][K/64 k blocks][32 lanes][16 B].  Lane (g = lane/4, t = lane%4),
// word 2c + j (c = k32 chunk of the k block, j = 0/1), byte i: low nibble = level[16 rb + g][k], high nibble =
// level[16 rb + g + 8][k], k = 64 kb + 32 c + 8 t + 4 j + i.  (The k order inside a chunk is a free choice as long as
// the activation digits use the same one; this one gives every prologue thread, which owns 8 consecutive k, both
// B registers of one lane.)
//
// gptq.int8 (8-bit levels, b2l_w8_gemv) runs the same kernel with W8 = true: weight layout b2l_w8_tile_i8,
// [N/16 row blocks][K/64 k blocks][2 chunks][32 lanes][16 B], whose four words per lane are the u8 A fragment itself
// (no LOP3, no row-pair recovery in the epilogue).  The int32 accumulators hold 255 * 128 * K < 2^31 for K <= 24576.
#include <algorithm>

#include "q4_mma_common.cuh"

namespace b2l {
namespace q4mv {

struct Params {
  const __nv_bfloat16* x;
  const uint8_t* qwt;
  const void* scales; const void* zeros; int szdt;
  __nv_bfloat16* y;
  int N, K;              // N rows (padded to a multiple of 16 in the tiled weight), K % 64 == 0
  int n_rb;              // row blocks
  int prologue; const __nv_bfloat16* norm_scale; float eps;
  int epilogue; const __nv_bfloat16* res;
  int nst;               // ring stages
  unsigned long long* tl;  // debug timeline (nullptr = off)
  int nocompute;           // debug: consumers release every stage untouched (pure TMA streaming rate)
  // LLaMA-Adapter v2 affine (AFFINE instantiations only): bf16 [N] in weight row order
  const __nv_bfloat16* aff_scale; const __nv_bfloat16* aff_bias;
};

// digit-plane stride in bytes: one byte per k, padded so that planes n and n + 1 fall into different bank halves
__host__ __device__ inline uint32_t plane_stride(int K) { return (uint32_t)K + ((K % 128 == 0) ? 64u : 0u); }

// shared memory map
struct SmemLayout {
  uint32_t ring, xf, zero, scratch, red, sxp, bars, total;
};
__host__ __device__ inline SmemLayout smem_layout(int nst, int K, int ndig) {
  SmemLayout L;
  uint32_t o = 0;
  L.ring = o;    o += (uint32_t)nst * STAGE_BYTES;
  L.xf = o;      o += (uint32_t)ndig * plane_stride(K);   // digit planes: [digit][k block][t (4)][16 B]
  L.zero = o;    o += 16;                                 // the B operand of the unused MMA columns
  L.scratch = o; o += 2 * NCW * MAX_HALVES * RB * 16;     // [buf][warp][half][row][digit (4)] int32 partials
  L.red = o;     o += 144;                                // reductions: float[8] sumsq, float[8] max, int64[8] sum X, int sh
  L.sxp = o;     o += NCW * 32 * 4;                       // per-thread partial sums of X
  L.bars = o;    o += 2 * MAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

// Weight width W8 (false: 4-bit levels, b2l_q4_tile_i8; true: 8-bit levels, b2l_w8_tile_i8).  A (16-row block, k block)
// tile is 512 B of packed nibbles or 1024 B of bytes; a half stage is 8 KB either way, so the ring, the stage count
// and the producer are shared and a stage carries half as many k-block positions at 8 bits.
template <bool W8> struct WTile {
  static constexpr int KB_BYTES = W8 ? 1024 : 512;
  static constexpr int KBP = HALF_STAGE_BYTES / KB_BYTES;   // k-block positions per half stage: 16 / 8
};

// One tile (16 rows x 64 k) into one accumulator set.  4 bits: one LDS.128, 1 LOP3 + 1 IMMA per packed word pair
// (a byte feeds rows g and g + 8); 8 bits: chunk c is its own LDS.128 whose four words ARE the A fragment.
template <bool W8>
__device__ __forceinline__ void single_imma(int (&a)[2][4], const uint8_t* tile, const uint4& xb) {
  if constexpr (W8) {
    const uint4 w0 = *reinterpret_cast<const uint4*>(tile), w1 = *reinterpret_cast<const uint4*>(tile + 512);
    mma_u8s8_16832(a[0], w0.x, w0.y, w0.z, w0.w, xb.x, xb.y);
    mma_u8s8_16832(a[1], w1.x, w1.y, w1.z, w1.w, xb.z, xb.w);
  } else {
    const uint4 wv = *reinterpret_cast<const uint4*>(tile);
    mma_u8s8_16832(a[0], wv.x, wv.x & 0xf0f0f0f0u, wv.y, wv.y & 0xf0f0f0f0u, xb.x, xb.y);
    mma_u8s8_16832(a[1], wv.z, wv.z & 0xf0f0f0f0u, wv.w, wv.w & 0xf0f0f0f0u, xb.z, xb.w);
  }
}

// One k-block position of NH 16-row halves (the activation fragments are loaded once for all of them).
template <int NH, bool W8>
__device__ __forceinline__ void kblock_imma(int (&acc)[MAX_HALVES][2][4], const uint8_t* wbase, const uint4& xb) {
#pragma unroll
  for (int h = 0; h < NH; ++h) single_imma<W8>(acc[h], wbase + h * HALF_STAGE_BYTES, xb);
}

// MAXC = activation chunks (2048 elements each) a thread block caches in registers during the prologue:
// 6 covers K <= 12288 (every 7B/13B/30B layer), 12 covers K <= 24576 (65B mlp.c_proj, K = 22016).
// NDIG = base-256 digits of the scaled activations: 3 (|X| < 2^22).  W8: 8-bit weight levels (see WTile).
// AFFINE: LLaMA-Adapter v2's v = bf16(s * bf16(v + b)) per row before the epilogue (adapter_v2.py:30-33).
template <int MAXC, int NDIG, bool W8, bool AFFINE>
__global__ void __launch_bounds__(NTHREADS, 2) q4_gemv_kernel(const Params p) {
  constexpr int KB_BYTES = WTile<W8>::KB_BYTES, KBP_PER_STAGE = WTile<W8>::KBP;
  extern __shared__ __align__(128) uint8_t smem[];
  const SmemLayout L = smem_layout(p.nst, p.K, NDIG);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_kb = p.K / KB;                                              // k blocks per 16-row block
  // A 16 KB stage holds 32 tiles of 512 B (16 of 1024 B at 8 bits): KBP_PER_STAGE k-block positions of BOTH 16-row
  // blocks of a pair, or twice as many of a single block (the ring slot is always used in full).  The last stage of
  // a unit may be short.
  const int spu2 = (n_kb + KBP_PER_STAGE - 1) / KBP_PER_STAGE, spu1 = (n_kb + 2 * KBP_PER_STAGE - 1) / (2 * KBP_PER_STAGE);
  // this CTA's contiguous range of 16-row blocks, processed as pairs and at most one single
  const int rb_lo = (int)(((long long)blockIdx.x * p.n_rb) / gridDim.x);
  const int rb_hi = (int)(((long long)(blockIdx.x + 1) * p.n_rb) / gridDim.x);
  const int n_units = (rb_hi - rb_lo + 1) / 2;
  const int total_stages = ((rb_hi - rb_lo) / 2) * spu2 + ((rb_hi - rb_lo) & 1) * spu1;
  const uint32_t bar_full = sbase + L.bars, bar_empty = bar_full + MAX_STAGES * 8;
  const uint32_t PS = plane_stride(p.K);

  if (tid == 0) tl_min(p.tl, 0);
  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) {
      mbar_init(bar_full + i * 8, 1);
      mbar_init(bar_empty + i * 8, NCW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < 4) reinterpret_cast<uint32_t*>(smem + L.zero)[tid] = 0u;
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ===================== TMA producer: the CTA's units, stage by stage =====================
    if (lane == 0) {
      int slot = 0;
      uint32_t phase = 1;  // fresh barriers: waiting on parity 1 passes immediately
      int it = 0;
      for (int u = 0; u < n_units; ++u) {
        const int rb = rb_lo + 2 * u;
        const int halves = min(2, rb_hi - rb);
        const uint8_t* src = p.qwt + (size_t)rb * n_kb * KB_BYTES;
        const int per_stage = halves == 2 ? KBP_PER_STAGE : 2 * KBP_PER_STAGE;
        for (int kb0 = 0; kb0 < n_kb; kb0 += per_stage, ++it) {
          const int nkb = min(per_stage, n_kb - kb0);
          const uint32_t bytes = (uint32_t)nkb * KB_BYTES;
          mbar_wait(bar_empty + slot * 8, phase);
          mbar_expect_tx(bar_full + slot * 8, bytes * halves);
          for (int h = 0; h < halves; ++h) {
            const uint32_t dst = sbase + L.ring + slot * STAGE_BYTES + h * HALF_STAGE_BYTES;
            const uint8_t* from = src + ((size_t)h * n_kb + kb0) * KB_BYTES;
            tma_bulk_g2s(dst, from, bytes, bar_full + slot * 8);
          }
          if (++slot == p.nst) { slot = 0; phase ^= 1; }
          if (it + 1 == min(total_stages, p.nst)) pdl_launch_dependents();  // ring full: next kernel may prefetch
        }
      }
      if (total_stages == 0) pdl_launch_dependents();
    }
  } else if (warp < NCW) {
    // ===================== consumer warps =====================
    float* red = reinterpret_cast<float*>(smem + L.red);   // [0..7] sum of squares, [8..15] max, then int64[8] sum X, int sh
    int* red_sh = reinterpret_cast<int*>(smem + L.red + 128);
    // ---- activations: [RMSNorm], power-of-two scaling, balanced digits in B-fragment order, exact sum(X)
    // (act_pass1 / act_scale / act_digits, q4_mma_common.cuh)
    {
      const bool norm = (p.prologue == B2L_PRO_RMSNORM);
      constexpr int NT = NCW * 32;   // 256 threads, 8 elements each per pass
      uint4 xv[MAXC], gv[MAXC];
      // the RMSNorm scale is a weight: fetch it BEFORE waiting for the producing kernel
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int k = (c * NT + tid) * 8;
        gv[c] = make_uint4(0, 0, 0, 0);
        if (norm && k < p.K) gv[c] = *reinterpret_cast<const uint4*>(p.norm_scale + k);
      }
      pdl_wait();
      if (tid == 0) tl_max(p.tl, 1);
      // written by the previous kernel: coherent loads (p.x is neither const __restrict__ nor read through ld.global.nc)
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int k = (c * NT + tid) * 8;
        xv[c] = make_uint4(0, 0, 0, 0);
        if (k < p.K) xv[c] = ld_coherent_u4(p.x + k);
      }
      const int nchunk = (p.K + NT * 8 - 1) / (NT * 8);  // warp-uniform: chunks that hold data
      float ss, mx;
      act_pass1<MAXC>(xv, gv, nchunk, norm, ss, mx);
      ss = warp_sum(ss);
      mx = warp_max(mx);
      if (lane == 0) { red[warp] = ss; red[8 + warp] = mx; }
      named_bar_sync(1, NT);
      ss = 0.f; mx = 0.f;
#pragma unroll
      for (int w = 0; w < NCW; ++w) { ss += red[w]; mx = fmaxf(mx, red[8 + w]); }
      const ActScale as = act_scale<NDIG>(ss, mx, norm, p.K, p.eps);
      uint32_t sxu = 0;     // sum of this thread's X (<= 48 values below 2^22), modulo 2^32
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        const int k = (c * NT + tid) * 8;
        if (c < nchunk && k < p.K) {
          uint32_t dj[2][3];
          act_digits(xv[c], gv[c], norm, as, dj, sxu);
          // k = 64 kb + 32 c32 + 8 t + (0..7): plane n, k block kb, lane slot t, words 2 c32, 2 c32 + 1
          uint8_t* dst = smem + L.xf + (k >> 6) * 64 + ((k >> 3) & 3) * 16 + ((k >> 5) & 1) * 8;
#pragma unroll
          for (int n = 0; n < NDIG; ++n) *reinterpret_cast<uint2*>(dst + n * PS) = make_uint2(dj[0][n], dj[1][n]);
        }
      }
      // exact sum of X over the row: every thread leaves its int32 partial (<= 48 values below 2^22) in shared memory
      // and goes on to the main loop; the epilogue warp, idle until the first unit is done, adds the 256 partials
      // in int64 (integers: the order does not matter)
      reinterpret_cast<int*>(smem + L.sxp)[tid] = (int)sxu;
      if (tid == 0) *red_sh = as.sh;
      named_bar_sync(3, NT + 32);          // releases the epilogue warp too: digit planes, sum X and sh are ready
      if (tid == 0) tl_max(p.tl, 2);
    }

    // ---- weights: stage -> registers -> mma.sync.  Warp w takes k-block positions w and w + 8 of a stage
    // and, for each, both 16-row halves of the unit (the B fragments are loaded once per position).
    // lanes 0..15 = MMA columns 0..3 = digit planes; lanes 16..31 (columns 4..7) read the zero block
    const int ncol = lane >> 2, t4 = lane & 3;
    const uint8_t* xf_lane = (ncol < NDIG) ? smem + L.xf + ncol * PS + t4 * 16 : smem + L.zero;
    const int xf_step = (ncol < NDIG) ? 64 : 0;
    int slot = 0;
    uint32_t phase = 0;
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    for (int u = 0; u < n_units; ++u) {
      const int halves = min(2, rb_hi - (rb_lo + 2 * u));
      int acc[MAX_HALVES][2][4];
#pragma unroll
      for (int h = 0; h < MAX_HALVES; ++h)
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[h][c][i] = 0;
      const int per_stage = halves == 2 ? KBP_PER_STAGE : 2 * KBP_PER_STAGE;
      for (int kb0 = 0; kb0 < n_kb; kb0 += per_stage) {
        const int nkb = min(per_stage, n_kb - kb0);
        mbar_wait(bar_full + slot * 8, phase);
        // warp w owns tiles w, w + 8, w + 16, w + 24 of the stage (same addresses for pairs and singles):
        // a pair: k-block positions w, w + 8 of block 0 and of block 1 (the digit fragments are shared);
        // a single: positions w, w + 8, w + 16, w + 24 of the one block, accumulated in both accumulator sets
        const uint8_t* st_base = smem + L.ring + slot * STAGE_BYTES + lane * 16;
        const uint8_t* xq = xf_lane + kb0 * xf_step;
        if (!p.nocompute) {
          constexpr int NPAIR = KBP_PER_STAGE / NCW, NSINGLE = 2 * KBP_PER_STAGE / NCW;   // positions per warp
          if (halves == MAX_HALVES) {
            if (nkb == KBP_PER_STAGE) {
#pragma unroll
              for (int i = 0; i < NPAIR; ++i) {
                const int kbl = i * NCW + warp;
                kblock_imma<MAX_HALVES, W8>(acc, st_base + kbl * KB_BYTES, *reinterpret_cast<const uint4*>(xq + kbl * xf_step));
              }
            } else {
#pragma unroll
              for (int i = 0; i < NPAIR; ++i) {
                const int kbl = i * NCW + warp;
                if (kbl < nkb) kblock_imma<MAX_HALVES, W8>(acc, st_base + kbl * KB_BYTES, *reinterpret_cast<const uint4*>(xq + kbl * xf_step));
              }
            }
          } else {
            if (nkb == 2 * KBP_PER_STAGE) {
#pragma unroll
              for (int i = 0; i < NSINGLE; ++i) {
                const int kbl = i * NCW + warp;
                single_imma<W8>(acc[i & 1], st_base + kbl * KB_BYTES, *reinterpret_cast<const uint4*>(xq + kbl * xf_step));
              }
            } else {
#pragma unroll
              for (int i = 0; i < NSINGLE; ++i) {
                const int kbl = i * NCW + warp;
                if (kbl < nkb) single_imma<W8>(acc[i & 1], st_base + kbl * KB_BYTES, *reinterpret_cast<const uint4*>(xq + kbl * xf_step));
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + slot * 8);
        if (++slot == p.nst) { slot = 0; phase ^= 1; }
      }
      // 16 x 8 result: lane (g, t) holds rows g (c0, c1) and g + 8 (c2, c3) of columns 2t, 2t + 1 = digits 2t, 2t + 1.
      // 4 bits: row g = D[g] - D[g+8] (the unmasked byte carried 16 * level[g+8] as well), row g + 8 = D[g+8] / 16
      // (exact); 8 bits: the rows are D[g] and D[g+8] themselves
      const int buf = u & 1;
      named_bar_sync(4 + buf, NCW * 32 + 32);  // the epilogue warp has drained this scratch buffer (two units ago)
      if (t4 < 2) {
        if (halves != MAX_HALVES) {   // a single block: its two accumulator sets hold different k-block positions
#pragma unroll
          for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[0][c][i] += acc[1][c][i];
        }
#pragma unroll
        for (int h = 0; h < MAX_HALVES; ++h) {
          const int c0 = acc[h][0][0] + acc[h][1][0], c1 = acc[h][0][1] + acc[h][1][1];
          const int c2 = acc[h][0][2] + acc[h][1][2], c3 = acc[h][0][3] + acc[h][1][3];
          int* dst = scratch + (((buf * NCW + warp) * MAX_HALVES + h) * RB + (lane >> 2)) * 4 + 2 * t4;
          if constexpr (W8) {
            *reinterpret_cast<int2*>(dst) = make_int2(c0, c1);
            *reinterpret_cast<int2*>(dst + 8 * 4) = make_int2(c2, c3);
          } else {
            *reinterpret_cast<int2*>(dst) = make_int2(c0 - c2, c1 - c3);
            *reinterpret_cast<int2*>(dst + 8 * 4) = make_int2(c2 >> 4, c3 >> 4);
          }
        }
      }
      __syncwarp();
      named_bar_arrive(6 + buf, NCW * 32 + 32);  // partials of this unit are in the scratch buffer
    }
    if (tid == 0) tl_max(p.tl, 3);
  } else {
    // ===================== epilogue warp: lane = row of the 32-row unit =====================
    // the affine vectors are weights: the first unit's are loaded before the wait, later units' ahead of their reduction
    float aff_s = 1.f, aff_b = 0.f;
    auto load_affine = [&](int u) {
      const int orow = (rb_lo + 2 * u + (lane >> 4)) * RB + (lane & 15);
      const int o = min(orow, p.N - 1);
      aff_s = bf2f(p.aff_scale[o]);
      aff_b = bf2f(p.aff_bias[o]);
    };
    if constexpr (AFFINE) {
      if (n_units > 0) load_affine(0);
    }
    pdl_wait();
    const int* red_sh = reinterpret_cast<const int*>(smem + L.red + 128);
    const int* scratch = reinterpret_cast<const int*>(smem + L.scratch);
    named_bar_sync(3, NCW * 32 + 32);
    long long sum_x = 0;
    {
      const int4* sp = reinterpret_cast<const int4*>(smem + L.sxp) + lane * 2;   // 8 partials per lane
      const int4 s0 = sp[0], s1 = sp[1];
      sum_x = (long long)s0.x + s0.y + s0.z + s0.w + s1.x + s1.y + s1.z + s1.w;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum_x += __shfl_xor_sync(0xffffffffu, sum_x, o);
    }
    const double dsum_x = (double)sum_x;
    const int sh = *red_sh;
    const double inv_scale = __longlong_as_double((long long)(1023 - sh) << 52);   // 2^-sh
    // both scratch buffers start free
    if (n_units > 0) named_bar_arrive(4, NCW * 32 + 32);
    if (n_units > 1) named_bar_arrive(5, NCW * 32 + 32);
    for (int u = 0; u < n_units; ++u) {
      const int rb = rb_lo + 2 * u;
      const int halves = min(2, rb_hi - rb);
      const int buf = u & 1;
      const int half = lane >> 4, row = lane & 15;
      const bool active = half < halves;
      const int orow = (rb + half) * RB + row;             // row of the (interleaved) weight matrix
      const int o = min(orow, p.N - 1);
      const float sc = load_sz(p.scales, p.szdt, o);
      const float zero = load_sz(p.zeros, p.szdt, o);
      if constexpr (AFFINE) {
        if (u > 0) load_affine(u);
      }
      float resv = 0.f;
      if (p.epilogue == B2L_EPI_RESIDUAL && active && orow < p.N) resv = bf2f(p.res[orow]);
      named_bar_sync(6 + buf, NCW * 32 + 32);
      int d0 = 0, d1 = 0, d2 = 0, d3 = 0;
#pragma unroll
      for (int w = 0; w < NCW; ++w) {   // integer sums: exact, independent of the order
        const int4 v = *reinterpret_cast<const int4*>(scratch + (((buf * NCW + w) * MAX_HALVES + half) * RB + row) * 4);
        d0 += v.x; d1 += v.y; d2 += v.z; d3 += v.w;
      }
      if (u + 2 < n_units) named_bar_arrive(4 + buf, NCW * 32 + 32);                                   // scratch buffer free again
      // sum_k level X = d0 + 256 d1 + 65536 d2 + 2^24 d3 (exact in int64, < 2^53)
      const long long tq = (long long)d0 + ((long long)d1 << 8) + ((long long)d2 << 16) + ((long long)d3 << 24);
      const float tf = (float)(((double)tq - (double)zero * dsum_x) * inv_scale);   // sum (level - zero) x, one rounding
      float v = rbf(sc * tf);
      if constexpr (AFFINE) v = rbf(aff_s * rbf(v + aff_b));
      if (p.epilogue == B2L_EPI_SWIGLU) {
        // rows 0..7 of a 16-row block are c_fc1[o..o+7], rows 8..15 are c_fc2[o..o+7]
        const float b = __shfl_down_sync(0xffffffffu, v, 8);
        if (active && row < 8) {
          const float sl = rbf(v / (1.0f + expf(-v)));
          p.y[(rb + half) * 8 + row] = f2bf(sl * b);
        }
      } else if (active && orow < p.N) {
        p.y[orow] = f2bf(p.epilogue == B2L_EPI_RESIDUAL ? v + resv : v);
      }
    }
    if (lane == 0) tl_max(p.tl, 4);
  }
}

// ---------------------------------------------------------------- re-tiling for the int8-MMA layout
__global__ void q4_tile_i8_kernel(const uint8_t* __restrict__ qw, uint32_t* __restrict__ out, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one output word
  const int n_kb = K / KB;
  const int n_rb = (N + RB - 1) / RB;
  const size_t total = (size_t)n_rb * n_kb * 32 * 4;
  if (idx >= total) return;
  const int wd = idx & 3, lane = (idx >> 2) & 31;
  const size_t rest = idx >> 7;
  const int kb = (int)(rest % n_kb), rb = (int)(rest / n_kb);
  const int g = lane >> 2, t = lane & 3, c = wd >> 1, j = wd & 1;
  uint32_t w = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = kb * KB + 32 * c + 8 * t + 4 * j + i;
#pragma unroll
    for (int hi = 0; hi < 2; ++hi) {
      const int row = rb * RB + g + 8 * hi;
      if (row < N) {
        const uint8_t b = qw[(size_t)(k >> 1) * N + row];
        w |= (uint32_t)((b >> ((k & 1) * 4)) & 0xF) << (8 * i + 4 * hi);
      }
    }
  }
  out[idx] = w;
}

__global__ void q4_untile_i8_kernel(const uint32_t* __restrict__ tiled, uint8_t* __restrict__ qw, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one packed byte [j][o]
  const size_t total = (size_t)(K / 2) * N;
  if (idx >= total) return;
  const int o = (int)(idx % N), jp = (int)(idx / N);
  const int n_kb = K / KB;
  uint8_t b = 0;
#pragma unroll
  for (int nr = 0; nr < 2; ++nr) {
    const int k = 2 * jp + nr;
    const int kb = k / KB, kl = k % KB, c = kl >> 5, kk = kl & 31;
    const int t = kk >> 3, j = (kk >> 2) & 1, i = kk & 3;
    const int rb = o / RB, rl = o % RB, g = rl & 7, hi = rl >> 3;
    const uint32_t w = tiled[(((size_t)rb * n_kb + kb) * 32 + (g * 4 + t)) * 4 + 2 * c + j];
    b |= (uint8_t)(((w >> (8 * i + 4 * hi)) & 0xF) << (4 * nr));
  }
  qw[idx] = b;
}

// 8-bit levels (reference layout: byte [k][o], quantization.py:386-390 with one entry per byte) ->
// [N/16 row blocks][K/64 k blocks][2 chunks][32 lanes][4 words]: word w of lane (g, t) in chunk c holds row
// g + 8 (w & 1), k = 64 kb + 32 c + 8 t + 4 (w >> 1) + (0..3) -- the A fragment of mma.m16n8k32 against the
// activation words the prologue builds (k = 64 kb + 32 c + 8 t + 4 j + i).  Rows beyond N are zero.
__global__ void w8_tile_i8_kernel(const uint8_t* __restrict__ qw, uint32_t* __restrict__ out, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one output word
  const int n_kb = K / KB;
  const int n_rb = (N + RB - 1) / RB;
  const size_t total = (size_t)n_rb * n_kb * 2 * 32 * 4;
  if (idx >= total) return;
  const int wd = idx & 3, lane = (idx >> 2) & 31, c = (idx >> 7) & 1;
  const size_t rest = idx >> 8;
  const int kb = (int)(rest % n_kb), rb = (int)(rest / n_kb);
  const int row = rb * RB + (lane >> 2) + 8 * (wd & 1);
  const int k0 = kb * KB + 32 * c + 8 * (lane & 3) + 4 * (wd >> 1);
  uint32_t w = 0;
  if (row < N) {
#pragma unroll
    for (int i = 0; i < 4; ++i) w |= (uint32_t)qw[(size_t)(k0 + i) * N + row] << (8 * i);
  }
  out[idx] = w;
}

__global__ void w8_untile_i8_kernel(const uint8_t* __restrict__ tiled, uint8_t* __restrict__ qw, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one byte [k][o]
  const size_t total = (size_t)K * N;
  if (idx >= total) return;
  const int o = (int)(idx % N), k = (int)(idx / N);
  const int kb = k / KB, kl = k % KB, c = kl >> 5, t = (kl >> 3) & 3, j = (kl >> 2) & 1, i = kl & 3;
  const int rb = o / RB, rl = o % RB;
  const size_t word = ((((size_t)rb * (K / KB) + kb) * 2 + c) * 32 + (rl & 7) * 4 + t) * 4 + 2 * j + (rl >> 3);
  qw[idx] = tiled[word * 4 + i];
}

}  // namespace q4mv
}  // namespace b2l

using namespace b2l;
using namespace b2l::q4mv;

extern "C" size_t b2l_q4_tiled_i8_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || K % KB != 0) return 0;
  return (size_t)((N + RB - 1) / RB) * (K / KB) * KB_BYTES;
}

extern "C" int b2l_q4_tile_i8(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_q4_tile_i8: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_q4_tile_i8: in_features %d must be a multiple of %d", K, KB);
  const size_t total = b2l_q4_tiled_i8_bytes(N, K) / 4;
  q4_tile_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)qw, (uint32_t*)qw_tiled, N, K);
  B2L_LAUNCH_CHECK("q4_tile_i8_kernel");
  return 0;
}

extern "C" int b2l_q4_untile_i8(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_q4_untile_i8: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_q4_untile_i8: in_features %d must be a multiple of %d", K, KB);
  const size_t total = (size_t)(K / 2) * N;
  q4_untile_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint32_t*)qw_tiled, (uint8_t*)qw, N, K);
  B2L_LAUNCH_CHECK("q4_untile_i8_kernel");
  return 0;
}

extern "C" size_t b2l_w8_tiled_i8_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || K % KB != 0) return 0;
  return (size_t)((N + RB - 1) / RB) * (K / KB) * WTile<true>::KB_BYTES;
}

extern "C" int b2l_w8_tile_i8(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_w8_tile_i8: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_w8_tile_i8: in_features %d must be a multiple of %d", K, KB);
  const size_t total = b2l_w8_tiled_i8_bytes(N, K) / 4;
  w8_tile_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)qw, (uint32_t*)qw_tiled, N, K);
  B2L_LAUNCH_CHECK("w8_tile_i8_kernel");
  return 0;
}

extern "C" int b2l_w8_untile_i8(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_w8_untile_i8: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_w8_untile_i8: in_features %d must be a multiple of %d", K, KB);
  const size_t total = (size_t)K * N;
  w8_untile_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)qw_tiled, (uint8_t*)qw, N, K);
  B2L_LAUNCH_CHECK("w8_untile_i8_kernel");
  return 0;
}

namespace {
// three digits (|X| < 2^22) everywhere: the prologue's fma conversion needs the integer inside a float mantissa
constexpr int NDIG_GEMV = 3;

// Ring stages that fit `budget` bytes of shared memory at this K (0: not even two)
template <int NDIG>
int ring_stages(int K, uint32_t budget) {
  const uint32_t fixed = smem_layout(0, K, NDIG).total;
  const int nst = fixed + 2 * STAGE_BYTES <= budget ? (int)((budget - fixed) / STAGE_BYTES) : 0;
  return nst > MAX_STAGES ? MAX_STAGES : nst;
}

// CTAs per SM before the small-linear choice in launch_gemv_variant, and the ring stages at that size (0: not even
// two).  That choice only ever moves to one CTA per SM with a deeper ring.
template <int NDIG>
int base_ring_stages(int K, int* ctas_per_sm) {
  *ctas_per_sm = K <= 16384 ? 2 : 1;
  return ring_stages<NDIG>(K, (*ctas_per_sm == 2 ? 110u : 224u) * 1024u);
}

// Stages a CTA owning `rbs` row blocks streams (pairs, then at most one single, as q4_gemv_kernel walks them)
template <bool W8>
int cta_stages(int rbs, int n_kb) {
  constexpr int KBP = WTile<W8>::KBP;
  return (rbs / 2) * ((n_kb + KBP - 1) / KBP) + (rbs & 1) * ((n_kb + 2 * KBP - 1) / (2 * KBP));
}

// Launch shape.  Up to K = 16384, two CTAs per SM with 110 KB of shared memory each; above, the digit planes leave no
// room for a useful ring at that size and one CTA takes the whole SM.  A linear small enough that, at one CTA per SM,
// every CTA's whole share of the weights fits its ring (LLaMA-7B attn.c_proj: 2 row blocks, 4 of 5 stages) runs as
// one 113 KB CTA per SM instead: two such CTAs fit an SM beside each other (228 KB less 1 KB reserved per CTA), so
// the launch needs one free slot, not two, to become resident behind the attention kernel, and each CTA requests all
// of its weights before the dependency resolves.  On H100 that is 3.3 % more 7B tokens/s; one CTA per SM for the
// larger linears, whose stream does not fit, measured slower (DESIGN.md section 3: 8 consumer warps per SM stream less
// than 16).
template <int MAXC, int NDIG, bool W8, bool AFFINE>
int launch_gemv_variant(const Params& p0, int grid_override, bool pdl, cudaStream_t stream) {
  Params p = p0;
  int ctas_per_sm;
  int nst = base_ring_stages<NDIG>(p.K, &ctas_per_sm);   // >= 2: check_gemv
  if (ctas_per_sm == 2) {
    const int sms = sm_count(), n_kb = p.K / KB;
    const int one = ring_stages<NDIG>(p.K, 113u * 1024u);
    const int rb_max = (p.n_rb + sms - 1) / sms, rb_min = p.n_rb / sms;
    if (std::max(cta_stages<W8>(rb_max, n_kb), cta_stages<W8>(rb_min, n_kb)) <= one) {
      ctas_per_sm = 1;
      nst = one;
    }
  }
  p.nst = nst;
  const SmemLayout L = smem_layout(nst, p.K, NDIG);
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(q4_gemv_kernel<MAXC, NDIG, W8, AFFINE>, L.total, smem_cache)) return rc;
  int grid = grid_override > 0 ? grid_override : ctas_per_sm * sm_count();
  if (grid > p.n_rb) grid = p.n_rb;
  LaunchCfg lc(dim3(grid), dim3(NTHREADS), L.total, stream, pdl, 1);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q4_gemv_kernel<MAXC, NDIG, W8, AFFINE>, p));
  return 0;
}

template <int MAXC, int NDIG, bool W8>
int launch_gemv(const Params& p, int grid_override, bool pdl, cudaStream_t stream) {
  if (p.aff_scale != nullptr) return launch_gemv_variant<MAXC, NDIG, W8, true>(p, grid_override, pdl, stream);
  return launch_gemv_variant<MAXC, NDIG, W8, false>(p, grid_override, pdl, stream);
}

}  // namespace

namespace b2l {
// b2l_q4_gemv's (W8 = false) and b2l_w8_gemv's (W8 = true) argument checks: 0, or B2L_E_* with a message
int check_gemv(const b2l_q4_linear_args* a, bool W8) {
  const char* fn = W8 ? "b2l_w8_gemv" : "b2l_q4_gemv";
  B2L_CHECK_ARG(a != nullptr, "%s: null args", fn);
  B2L_CHECK_ARG(a->x && a->qw_tiled && a->scales && a->zeros && a->y, "%s: null pointer", fn);
  B2L_CHECK_SUPPORTED(a->M == 1, "%s: M=%d (this kernel is the batch-1 path; use %s)", fn, a->M,
                      W8 ? "b2l_w8_gemm" : "b2l_q4_gemv_batch / b2l_q4_linear_tc");
  B2L_CHECK_SUPPORTED(a->K > 0 && a->K % KB == 0 && a->K <= MAX_K, "%s: K=%d must be a multiple of %d and <= %d", fn, a->K, KB, MAX_K);
  B2L_CHECK_ARG(a->N > 0, "%s: bad N", fn);
  B2L_CHECK_ARG(((uintptr_t)a->x % 16 == 0) && ((uintptr_t)a->qw_tiled % 16 == 0), "%s: x / qw_tiled must be 16-byte aligned", fn);
  B2L_CHECK_ARG(a->sz_dtype == B2L_BF16 || a->sz_dtype == B2L_F32, "%s: bad sz_dtype", fn);
  if (W8) B2L_CHECK_SUPPORTED((a->flags & ~(B2L_F_PDL | B2L_F_DEBUG_NOCOMPUTE)) == 0, "%s: unknown flags 0x%x", fn, a->flags);
  if (a->prologue == B2L_PRO_RMSNORM)
    B2L_CHECK_ARG(a->norm_scale && ((uintptr_t)a->norm_scale % 16 == 0), "%s: RMSNorm prologue needs a 16-byte aligned scale", fn);
  else
    B2L_CHECK_ARG(a->prologue == B2L_PRO_NONE, "%s: bad prologue %d", fn, a->prologue);
  if (a->epilogue == B2L_EPI_RESIDUAL) B2L_CHECK_ARG(a->res != nullptr, "%s: RESIDUAL epilogue needs res", fn);
  else if (a->epilogue == B2L_EPI_SWIGLU) B2L_CHECK_SUPPORTED(a->N % RB == 0, "%s: SWIGLU needs N %% 16 == 0", fn);
  else B2L_CHECK_ARG(a->epilogue == B2L_EPI_STORE, "%s: bad epilogue %d", fn, a->epilogue);
  B2L_CHECK_ARG((a->out_affine.scale == nullptr) == (a->out_affine.bias == nullptr),
                "%s: out_affine needs both scale and bias (or neither)", fn);
  int ctas_per_sm;
  B2L_CHECK_SUPPORTED(base_ring_stages<NDIG_GEMV>(a->K, &ctas_per_sm) >= 2, "%s: K=%d does not leave room for the weight ring",
                      fn, a->K);
  return 0;
}
}  // namespace b2l

namespace {
// b2l_q4_gemv (W8 = false) and b2l_w8_gemv (W8 = true): the same checks, argument block and launch policy
template <bool W8>
int gemv_entry(const b2l_q4_linear_args* a, b2l_stream_t stream) {
  if (int rc = check_gemv(a, W8)) return rc;
  Params p;
  p.aff_scale = (const __nv_bfloat16*)a->out_affine.scale;
  p.aff_bias = (const __nv_bfloat16*)a->out_affine.bias;
  p.x = (const __nv_bfloat16*)a->x;
  p.qwt = (const uint8_t*)a->qw_tiled;
  p.scales = a->scales; p.zeros = a->zeros; p.szdt = a->sz_dtype;
  p.y = (__nv_bfloat16*)a->y;
  p.N = a->N; p.K = a->K;
  p.n_rb = (a->N + RB - 1) / RB;
  p.prologue = a->prologue; p.norm_scale = (const __nv_bfloat16*)a->norm_scale; p.eps = a->eps;
  p.epilogue = a->epilogue; p.res = (const __nv_bfloat16*)a->res;
  p.nst = 0;
  p.tl = (unsigned long long*)a->trace;
  p.nocompute = (a->flags & B2L_F_DEBUG_NOCOMPUTE) ? 1 : 0;
  const bool pdl = (a->flags & B2L_F_PDL) != 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = a->split_k;  // split_k doubles as a grid override
  if (a->K <= 12288) return launch_gemv<6, NDIG_GEMV, W8>(p, grid, pdl, st);
  return launch_gemv<12, NDIG_GEMV, W8>(p, grid, pdl, st);
}
}  // namespace

extern "C" int b2l_q4_gemv(const b2l_q4_linear_args* a, b2l_stream_t stream) { return gemv_entry<false>(a, stream); }

extern "C" int b2l_w8_gemv(const b2l_q4_linear_args* a, b2l_stream_t stream) { return gemv_entry<true>(a, stream); }

// LLM.int8() linear for one activation row (decode), fused with its activation quantisation.
//
// Replaces Linear8bitLt.forward (lit_llama/quantization.py:38-77 + the bitsandbytes forward it
// inherits: MatMul8bitLt with has_fp16_weights=False, threshold=6.0):
//   a   = fp16(x)
//   out = { k : |a_k| >= threshold }                      (outlier columns, shared by the batch)
//   SCA = max_{k not in out} |a_k| ;  CA_k = round(a_k * 127 / SCA), 0 on outlier columns
//   y   = fp16( (CA . CB[o]) * SCA * SCB[o] / 127^2 ) + fp16( sum_{k in out} a_k * fp16(CB[o][k] * SCB[o] / 127) )
// The int8 x int8 -> int32 contraction runs on the tensor cores (mma.sync.m16n8k32.s8) straight
// from the TMA-staged tile: int8 needs no unpacking at all.  Same skeleton as q4_gemv.cu:
// persistent CTAs over 16-row blocks and the full K, TMA bulk copies into an mbarrier ring
// issued before the PDL dependency, deterministic in-CTA reduction.
//
// Two weight sources, one kernel body (template parameter WS); only how a stage (16 rows x 1024 k) reaches shared
// memory and how a warp fetches its A fragments differ:
//   WS_CB (b2l_q8_gemv_cb, what Linear8bitLt runs): CB itself, int8 (N, K) row-major.  Lanes 0..15 of the producer
//     warp each issue one bulk copy of their row's 1024 bytes, into a ring whose rows are ROW_PITCH = 1040 bytes
//     apart; no tensor map is read.  Each warp builds the m16 x k32 A fragment of chunk c with one ldmatrix.x4: its
//     four 8 x 8 .b16 matrices (rows 0-7 / 8-15 x k 32c..+15 / 32c+16..+31) are exactly registers a0..a3 of the s8
//     fragment, and the 16-byte pad puts each matrix's eight rows in distinct banks.  Rows past N are not copied:
//     their accumulators are never stored.  Measured on an H100, this beat a tensor-map copy of the same stage (with
//     or without the 128-byte swizzle) on every 7B shape and on whole-token 7B decode (DESIGN.md §3).
//   WS_TILED (b2l_q8_gemv): the b2l_q8_tile layout [N/16 row blocks][K/128 k blocks][4 k32 chunks][32 lanes][16 B];
//     the 16 bytes of lane (g, t) are registers a0..a3 of m16n8k32: rows g, g+8 x k = 32c + 4t..+3 and
//     32c + 16 + 4t..+3.  One 16 KB bulk copy per stage.
// Both contract the same int8 values in the same order, so their outputs are bit-identical.
//
// FUSED (b2l_q8_linear, WS_CB only): the whole-token step's llm.int8 linear.  The consumers first apply RMSNorm exactly
// as b2l_rmsnorm does (same 256-thread chunking and reduction order, the scale staged in `ah` before the dependency),
// so the outlier mask and SCA are those of the module path.  For SWIGLU a 16-row block holds 8 rows of cb and the
// same 8 rows of cb2; the epilogue warp rounds each row to bf16 as the module's store would, applies the v2 affine,
// then adds the residual or combines lane r with lane r + 8 through silu_mul1.  The non-FUSED instantiations compile
// to the same SASS as before the FUSED code existed.
//
// parity: the arithmetic restates the published LLM.int8() algorithm (bitsandbytes is not in
// the reference tree and not installed): parity with the reference is unpinned (DESIGN.md).
#include <cuda_fp16.h>

#include "b2l_common.cuh"
#include "q8_common.cuh"

namespace b2l {
namespace q8mv {

enum WeightSource { WS_TILED, WS_CB };

constexpr int RB = 16;
constexpr int KB = 128;                 // k per k block (4 IMMAs of k32)
constexpr int KB_BYTES = 2048;          // one (row block, k block)
constexpr int NCW = 8;
constexpr int KBP_PER_STAGE = 8;        // one k block per consumer warp per stage
constexpr int STAGE_BYTES = KBP_PER_STAGE * KB_BYTES;  // 16 KB
constexpr int ROW_PITCH = KBP_PER_STAGE * KB + 16;     // WS_CB: one weight row of a stage + 16 B (conflict-free ldmatrix)
template <WeightSource WS> __host__ __device__ constexpr uint32_t stage_bytes() { return WS == WS_CB ? RB * ROW_PITCH : STAGE_BYTES; }
constexpr int MAX_STAGES = 6;
constexpr int PRODUCER_WARP = NCW;
constexpr int NTHREADS = (NCW + 2) * 32;
constexpr int MAX_K = 32768;            // LLaMA-65B's n_hidden is 22016

struct Params {
  const __nv_bfloat16* x;     // one row, bf16 [K]
  const uint8_t* wt;          // WS_TILED: tiled CB
  const int8_t* cb;           // reference layout CB (N, K) row-major: WS_CB's weights, and the outlier columns
  const float* scb;           // [N]
  const uint32_t* mask_in;    // optional precomputed outlier mask (K bits), shared by a batch; nullptr = derive from x
  __nv_bfloat16* y;           // [N]
  int N, K, n_rb, nst;
  float threshold;
  // FUSED (b2l_q8_linear) only
  const int8_t* cb2;          // SWIGLU: the second CB / SCB (rows 8..15 of every block; rows 0..7 come from cb)
  const float* scb2;
  const __nv_bfloat16* norm_scale;   // RMSNorm prologue; nullptr = none
  float eps;
  int epilogue;               // B2L_EPI_*
  const __nv_bfloat16* res;   // RESIDUAL
  const __nv_bfloat16* aff_s; // LLaMA-Adapter v2 affine; nullptr = none
  const __nv_bfloat16* aff_b;
};

struct SmemLayout {
  uint32_t ring, xf, ah, mask, scratch, red, bars, total;
};
__host__ __device__ inline SmemLayout smem_layout(int nst, int K, uint32_t stage) {
  SmemLayout L;
  uint32_t o = 0;
  L.ring = o;    o += (uint32_t)nst * stage;
  L.xf = o;      o += (uint32_t)(K / KB) * 128;   // int8 B fragments: [k block][t (4)][32 B]
  L.ah = o;      o += (uint32_t)K * 2;            // fp16 activations (outlier term)
  L.mask = o;    o += (uint32_t)((K + 31) / 32) * 4;
  o = (o + 15u) & ~15u;
  L.scratch = o; o += 2 * NCW * RB * 4;           // [buf][warp][row] int32 partials
  L.red = o;     o += 64;
  o = (o + 7u) & ~7u;
  L.bars = o;    o += 2 * MAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

// One output row of a 16-row block as the FUSED epilogue needs it.  SWIGLU: rows 0..7 are outputs rb*8 .. rb*8+7 of
// cb, rows 8..15 the same outputs of cb2; the affine vectors are interleaved the same way (16 entries per block).
struct FusedRow {
  const int8_t* w;   // the weight row (outlier term)
  float scb, s, b;   // SCB and the affine's scale / bias (1, 0 without one)
  int col;           // output index
  bool valid;
};
__device__ __forceinline__ FusedRow fused_row(const Params& p, int rb, int row) {
  const bool glu = p.epilogue == B2L_EPI_SWIGLU;
  FusedRow r;
  r.col = glu ? rb * 8 + (row & 7) : rb * RB + row;
  r.valid = r.col < p.N;
  const int o = min(r.col, p.N - 1);
  const bool second = glu && row >= 8;
  r.w = (second ? p.cb2 : p.cb) + (size_t)o * p.K;
  r.scb = (second ? p.scb2 : p.scb)[o];
  r.s = 1.f;
  r.b = 0.f;
  if (p.aff_s != nullptr) {
    const int ai = glu ? (r.valid ? rb * 16 + row : 0) : o;
    r.s = bf2f(p.aff_s[ai]);
    r.b = bf2f(p.aff_b[ai]);
  }
  return r;
}

// FUSED = false: b2l_q8_gemv / b2l_q8_gemv_cb.  FUSED = true (WS_CB only): b2l_q8_linear, the same body plus the
// RMSNorm prologue, two weight sources for SWIGLU and the affine / residual / SwiGLU epilogue.
template <WeightSource WS, bool FUSED>
__global__ void __launch_bounds__(NTHREADS, 2) q8_gemv_kernel(const Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr uint32_t SB = stage_bytes<WS>();
  const SmemLayout L = smem_layout(p.nst, p.K, SB);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_kb = p.K / KB;
  const int stages_per_rb = (n_kb + KBP_PER_STAGE - 1) / KBP_PER_STAGE;
  const int rb_lo = (int)(((long long)blockIdx.x * p.n_rb) / gridDim.x);
  const int rb_hi = (int)(((long long)(blockIdx.x + 1) * p.n_rb) / gridDim.x);
  const int n_units = rb_hi - rb_lo;
  const int total_stages = n_units * stages_per_rb;
  const uint32_t bar_full = sbase + L.bars, bar_empty = bar_full + MAX_STAGES * 8;

  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) {
      mbar_init(bar_full + i * 8, 1);
      mbar_init(bar_empty + i * 8, NCW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0 || WS == WS_CB) {
      int slot = 0, it = 0;
      uint32_t phase = 1;
      for (int u = 0; u < n_units; ++u) {
        for (int s = 0; s < stages_per_rb; ++s, ++it) {
          if constexpr (FUSED) {
            // as WS_CB below; SWIGLU: lanes 0..7 copy rows of cb, lanes 8..15 the same rows of cb2
            const bool glu = p.epilogue == B2L_EPI_SWIGLU;
            const int per = glu ? 8 : RB, i = glu ? (lane & 7) : lane;
            const int row0 = (rb_lo + u) * per, nrows = min(per, p.N - row0);
            const uint32_t row_bytes = (uint32_t)min(KBP_PER_STAGE, n_kb - s * KBP_PER_STAGE) * KB;
            if (lane == 0) {
              mbar_wait(bar_empty + slot * 8, phase);
              mbar_expect_tx(bar_full + slot * 8, (uint32_t)(glu ? 2 : 1) * nrows * row_bytes);
            }
            __syncwarp();
            if (lane < RB && i < nrows)
              tma_bulk_g2s(sbase + L.ring + slot * SB + lane * ROW_PITCH,
                           ((glu && lane >= 8) ? p.cb2 : p.cb) + (size_t)(row0 + i) * p.K + (size_t)s * KBP_PER_STAGE * KB,
                           row_bytes, bar_full + slot * 8);
          } else if constexpr (WS == WS_CB) {
            // one bulk copy per weight row (lanes 0..15); rows past N are not copied (their accumulators are never
            // stored), so the transaction count is what is actually copied
            const int row0 = (rb_lo + u) * RB, nrows = min(RB, p.N - row0);
            const uint32_t row_bytes = (uint32_t)min(KBP_PER_STAGE, n_kb - s * KBP_PER_STAGE) * KB;
            if (lane == 0) {
              mbar_wait(bar_empty + slot * 8, phase);
              mbar_expect_tx(bar_full + slot * 8, (uint32_t)nrows * row_bytes);
            }
            __syncwarp();
            if (lane < nrows)
              tma_bulk_g2s(sbase + L.ring + slot * SB + lane * ROW_PITCH, p.cb + (size_t)(row0 + lane) * p.K + (size_t)s * KBP_PER_STAGE * KB,
                           row_bytes, bar_full + slot * 8);
          } else {
            mbar_wait(bar_empty + slot * 8, phase);
            const uint32_t bytes = (uint32_t)min(KBP_PER_STAGE, n_kb - s * KBP_PER_STAGE) * KB_BYTES;
            mbar_expect_tx(bar_full + slot * 8, bytes);
            const uint8_t* src = p.wt + (size_t)(rb_lo + u) * n_kb * KB_BYTES + (size_t)s * STAGE_BYTES;
            tma_bulk_g2s(sbase + L.ring + slot * STAGE_BYTES, src, bytes, bar_full + slot * 8);
          }
          if (++slot == p.nst) { slot = 0; phase ^= 1; }
          if (it + 1 == min(total_stages, p.nst)) pdl_launch_dependents();
        }
      }
      if (total_stages == 0) pdl_launch_dependents();
    }
  } else if (warp < NCW) {
    // ===================== consumer warps =====================
    if constexpr (!FUSED) pdl_wait();
    float* red = reinterpret_cast<float*>(smem + L.red);
    __half* ah = reinterpret_cast<__half*>(smem + L.ah);
    uint32_t* mask = reinterpret_cast<uint32_t*>(smem + L.mask);
    constexpr int NT = NCW * 32;
    float rinv = 0.f;
    if constexpr (FUSED) {
      // RMSNorm: the scale (a weight) is staged in `ah` before the dependency; each thread later overwrites exactly the
      // chunks it staged.  Sum of squares in rmsnorm_kernel's order: these 256 threads take its 256 threads' 8-element
      // chunks, then its block_sum (warp_sum, partials of 8 warps, warp_sum).
      if (p.norm_scale != nullptr)
        for (int k = tid * 8; k < p.K; k += NT * 8)
          *reinterpret_cast<uint4*>(ah + k) = *reinterpret_cast<const uint4*>(p.norm_scale + k);
      pdl_wait();
      if (p.norm_scale != nullptr) {
        float ss = 0.f;
        for (int k = tid * 8; k < p.K; k += NT * 8) {
          const uint4 v = ld_coherent_u4(p.x + k);
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float lo = __uint_as_float(w[q] << 16), hi = __uint_as_float(w[q] & 0xffff0000u);
            ss += rbf(lo * lo) + rbf(hi * hi);
          }
        }
        ss = warp_sum(ss);
        if (lane == 0) red[warp] = ss;
        bar_sync_c<1>(NT);
        ss = warp_sum(lane < NCW ? red[lane] : 0.f);
        rinv = rms_rinv(ss, p.K, p.eps);   // red is next written after two more bar_sync_c<1>
      }
    }
    // ---- activations: fp16 copy, outlier mask, row-wise absmax over inliers, int8 B fragments.  The row lives in
    // shared memory only (ah, which the epilogue needs anyway): each thread re-reads the 8-element chunks it wrote,
    // so no K-sized register array limits K.
    for (int i = tid; i < (p.K + 31) / 32; i += NT) mask[i] = p.mask_in ? p.mask_in[i] : 0u;
    bar_sync_c<1>(NT);
    for (int k = tid * 8; k < p.K; k += NT * 8) {
      uint4 u;
      if constexpr (FUSED) {
        u = ld_coherent_u4(p.x + k);
        if (p.norm_scale != nullptr) {   // x^ = rms_apply (b2l_rmsnorm's bf16 values), scale from `ah`
          const uint4 g = *reinterpret_cast<const uint4*>(ah + k);
          const uint32_t xw[4] = {u.x, u.y, u.z, u.w}, gw[4] = {g.x, g.y, g.z, g.w};
          uint32_t o[4];
#pragma unroll
          for (int q = 0; q < 4; ++q)
            o[q] = pack_bf16x2(rms_apply(__uint_as_float(xw[q] << 16), rinv, __uint_as_float(gw[q] << 16)),
                               rms_apply(__uint_as_float(xw[q] & 0xffff0000u), rinv, __uint_as_float(gw[q] & 0xffff0000u)));
          u = make_uint4(o[0], o[1], o[2], o[3]);
        }
      } else {
        u = *reinterpret_cast<const uint4*>(p.x + k);
      }
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      __half hv[8];
      uint32_t outl = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        hv[2 * q] = __float2half_rn(__uint_as_float(w[q] << 16));
        hv[2 * q + 1] = __float2half_rn(__uint_as_float(w[q] & 0xffff0000u));
      }
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (!p.mask_in && fabsf(__half2float(hv[e])) >= p.threshold) outl |= 1u << e;
      *reinterpret_cast<uint4*>(ah + k) = *reinterpret_cast<const uint4*>(hv);
      if (outl) atomicOr(&mask[k >> 5], outl << (k & 31));
    }
    bar_sync_c<1>(NT);
    float amax = 0.f;
    for (int k = tid * 8; k < p.K; k += NT * 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(ah + k);
      const __half* hv = reinterpret_cast<const __half*>(&u);
      const uint32_t mb = (mask[k >> 5] >> (k & 31)) & 0xFFu;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (!((mb >> e) & 1u)) amax = fmaxf(amax, fabsf(__half2float(hv[e])));
    }
    amax = warp_max(amax);
    if (lane == 0) red[warp] = amax;
    bar_sync_c<1>(NT);
    float sca = 0.f;
#pragma unroll
    for (int w = 0; w < NCW; ++w) sca = fmaxf(sca, red[w]);
    const float qs = sca > 0.f ? 127.0f / sca : 0.f;
    for (int k = tid * 8; k < p.K; k += NT * 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(ah + k);
      const __half* hv = reinterpret_cast<const __half*>(&u);
      const uint32_t mb = (mask[k >> 5] >> (k & 31)) & 0xFFu;
      uint32_t pk[2] = {0u, 0u};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        int qv = ((mb >> e) & 1u) ? 0 : __float2int_rn(__half2float(hv[e]) * qs);
        qv = max(-127, min(127, qv));
        pk[e >> 2] |= (uint32_t)(qv & 0xFF) << (8 * (e & 3));
      }
      // k..k+3 -> lane t = (k % 16) / 4, half = (k % 32) / 16, chunk c32 = (k % 128) / 32; k+4..k+7 -> t + 1
      const int kb = k >> 7, c32 = (k >> 5) & 3, half = (k >> 4) & 1, t0 = (k >> 2) & 3;
      uint32_t* dst = reinterpret_cast<uint32_t*>(smem + L.xf + kb * 128);
      dst[t0 * 8 + c32 * 2 + half] = pk[0];
      dst[(t0 + 1) * 8 + c32 * 2 + half] = pk[1];
    }
    if (tid == 0) red[8] = sca;
    bar_sync_c<3>(NT + 32);  // xf, ah, mask, SCA ready (epilogue warp included)

    // ---- weights: stage -> registers -> mma.sync s8 (no unpacking)
    const int t4 = lane & 3;
    int slot = 0;
    uint32_t phase = 0;
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    const uint8_t* xf_lane = smem + L.xf + t4 * 32;
    // WS_CB: lane i addresses row i % 8 of ldmatrix matrix j = i / 8, i.e. weight row i % 8 + 8 (j % 2) and 16-byte unit
    // 2c + j / 2 of the warp's k block
    const uint32_t lm_row = (uint32_t)((lane & 7) + 8 * ((lane >> 3) & 1)) * ROW_PITCH;
    const uint32_t lm_unit = (uint32_t)(lane >> 4);
    for (int u = 0; u < n_units; ++u) {
      int acc[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
      for (int s = 0; s < stages_per_rb; ++s) {
        const int nkb = min(KBP_PER_STAGE, n_kb - s * KBP_PER_STAGE);
        mbar_wait(bar_full + slot * 8, phase);
        if (warp < nkb) {
          const uint4* xp = reinterpret_cast<const uint4*>(xf_lane + (s * KBP_PER_STAGE + warp) * 128);
          const uint4 xa = xp[0], xb = xp[1];
          const uint32_t bb[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            uint4 a;
            if constexpr (WS == WS_CB)
              a = ldmatrix_x4(sbase + L.ring + slot * SB + lm_row + warp * KB + (2 * c + lm_unit) * 16);
            else
              a = *reinterpret_cast<const uint4*>(smem + L.ring + slot * STAGE_BYTES + warp * KB_BYTES + lane * 16 + c * 512);
            mma_s8s8_16832(acc[c & 1], a, bb[2 * c], bb[2 * c + 1]);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + slot * 8);
        if (++slot == p.nst) { slot = 0; phase ^= 1; }
      }
      const int buf = u & 1;
      if (buf) bar_sync_c<5>(NCW * 32 + 32); else bar_sync_c<4>(NCW * 32 + 32);
      if (t4 == 0) {
        int* dst = scratch + (buf * NCW + warp) * RB + (lane >> 2);
        dst[0] = acc[0][0] + acc[1][0];
        dst[8] = acc[0][2] + acc[1][2];
      }
      __syncwarp();
      if (buf) bar_arrive_c<7>(NCW * 32 + 32); else bar_arrive_c<6>(NCW * 32 + 32);
    }
  } else {
    // ===================== epilogue warp: lanes 0..15 = rows of the block =====================
    FusedRow fr{};
    if constexpr (FUSED)   // the first block's SCB and affine are weights: read before the dependency
      if (n_units > 0) fr = fused_row(p, rb_lo, lane & 15);
    pdl_wait();
    const float* red = reinterpret_cast<const float*>(smem + L.red);
    const int* scratch = reinterpret_cast<const int*>(smem + L.scratch);
    const __half* ah = reinterpret_cast<const __half*>(smem + L.ah);
    const uint32_t* mask = reinterpret_cast<const uint32_t*>(smem + L.mask);
    bar_sync_c<3>(NCW * 32 + 32);
    const float sca = red[8];
    if (n_units > 0) bar_arrive_c<4>(NCW * 32 + 32);
    if (n_units > 1) bar_arrive_c<5>(NCW * 32 + 32);
    const int nwords = (p.K + 31) / 32;
    for (int u = 0; u < n_units; ++u) {
      const int buf = u & 1;
      const int row = lane & 15;
      const int orow = (rb_lo + u) * RB + row;
      const int o = min(orow, p.N - 1);
      if constexpr (FUSED)
        if (u > 0) fr = fused_row(p, rb_lo + u, row);
      const float scb = FUSED ? fr.scb : p.scb[o];
      // outlier term first (global loads overlap the consumers' work): fp16 weights, fp32 accumulate, k ascending
      float term = 0.f;
      bool any = false;
      const float wsc = scb / 127.0f;
      for (int wi = 0; wi < nwords; ++wi) {
        uint32_t mb = mask[wi];
        while (mb) {
          const int e = __ffs(mb) - 1;
          mb &= mb - 1;
          const int k = wi * 32 + e;
          const float wv = q8_outlier_weight(FUSED ? fr.w[k] : p.cb[(size_t)o * p.K + k], wsc);
          term = fmaf(__half2float(ah[k]), wv, term);
          any = true;
        }
      }
      if (buf) bar_sync_c<7>(NCW * 32 + 32); else bar_sync_c<6>(NCW * 32 + 32);
      int t = 0;
#pragma unroll
      for (int w = 0; w < NCW; ++w) t += scratch[(buf * NCW + w) * RB + row];
      if (u + 2 < n_units) { if (buf) bar_arrive_c<5>(NCW * 32 + 32); else bar_arrive_c<4>(NCW * 32 + 32); }
      float v = q8_dequant(t, sca, scb);
      if (any) v = q8_add_outliers(v, term);
      if constexpr (FUSED) {
        // the module path's bf16 output, then b2l_linear_affine, then b2l_add / b2l_silu_mul
        float yv = rbf(v);
        if (p.aff_s != nullptr) yv = rbf(affine1(yv, fr.s, fr.b));
        if (p.epilogue == B2L_EPI_SWIGLU) {
          const float up = __shfl_down_sync(0xffffffffu, yv, 8);   // row r + 8: c_fc2's output of the same column
          if (lane < 8 && fr.valid) p.y[fr.col] = f2bf(silu_mul1(yv, up));
        } else if (lane < 16 && fr.valid) {
          p.y[fr.col] = f2bf(p.epilogue == B2L_EPI_RESIDUAL ? yv + ld_coherent_bf16(p.res + fr.col) : yv);
        }
      } else {
        if (lane < 16 && orow < p.N) p.y[orow] = f2bf(v);
      }
    }
  }
}

// ---- re-tiling: CB (N, K) row-major int8 -> fragment order
__global__ void q8_tile_kernel(const int8_t* __restrict__ cb, uint32_t* __restrict__ out, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one output word
  const int n_kb = K / KB, n_rb = (N + RB - 1) / RB;
  const size_t total = (size_t)n_rb * n_kb * 4 * 32 * 4;
  if (idx >= total) return;
  const int r = idx & 3, lane = (idx >> 2) & 31, c = (idx >> 7) & 3;
  const size_t rest = idx >> 9;
  const int kb = (int)(rest % n_kb), rb = (int)(rest / n_kb);
  const int g = lane >> 2, t = lane & 3;
  const int row = rb * RB + g + 8 * (r & 1);
  const int k0 = kb * KB + 32 * c + 16 * (r >> 1) + 4 * t;
  uint32_t w = 0;
  if (row < N) {
#pragma unroll
    for (int e = 0; e < 4; ++e) w |= (uint32_t)(uint8_t)cb[(size_t)row * K + k0 + e] << (8 * e);
  }
  out[idx] = w;
}

}  // namespace q8mv
}  // namespace b2l

using namespace b2l;
using namespace b2l::q8mv;

extern "C" size_t b2l_q8_tiled_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || K % KB != 0) return 0;
  return (size_t)((N + RB - 1) / RB) * (K / KB) * KB_BYTES;
}

extern "C" int b2l_q8_tile(const void* cb, void* tiled, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(cb && tiled && N > 0 && K > 0, "b2l_q8_tile: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_q8_tile: in_features %d must be a multiple of %d", K, KB);
  const size_t total = b2l_q8_tiled_bytes(N, K) / 4;
  q8_tile_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const int8_t*)cb, (uint32_t*)tiled, N, K);
  B2L_LAUNCH_CHECK("q8_tile_kernel");
  return 0;
}

// stage count, grid and launch, shared by both weight sources; p holds everything but nst
template <WeightSource WS, bool FUSED = false>
static int launch_gemv(Params& p, int flags, b2l_stream_t stream) {
  constexpr uint32_t SB = stage_bytes<WS>();
  const uint32_t fixed = smem_layout(0, p.K, SB).total;
  int nst = (int)((110u * 1024u - fixed) / SB);
  if (nst > MAX_STAGES) nst = MAX_STAGES;
  if (nst < 2) nst = 2;
  p.nst = nst;
  const SmemLayout L = smem_layout(nst, p.K, SB);
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(q8_gemv_kernel<WS, FUSED>, L.total, smem_cache)) return rc;
  // two CTAs per SM while both fit in its 228 KB (1 KB of each reserved by the hardware); above K ~ 26000 only one does
  int grid = (L.total <= 113u * 1024u ? 2 : 1) * sm_count();
  if (grid > p.n_rb) grid = p.n_rb;
  LaunchCfg lc(dim3(grid), dim3(NTHREADS), L.total, (cudaStream_t)stream, (flags & B2L_F_PDL) != 0, 1);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q8_gemv_kernel<WS, FUSED>, p));
  return 0;
}

static void fill_params(Params& p, const void* x, const void* cb, const void* scb, const void* outlier_mask, void* y, int N, int K,
                        float threshold) {
  p = Params{};   // every kernel parameter defined, wt included where it is unused
  p.x = (const __nv_bfloat16*)x; p.cb = (const int8_t*)cb; p.scb = (const float*)scb;
  p.mask_in = (const uint32_t*)outlier_mask; p.y = (__nv_bfloat16*)y;
  p.N = N; p.K = K; p.n_rb = (N + RB - 1) / RB; p.threshold = threshold;
}

extern "C" int b2l_q8_gemv(const void* x, const void* w_tiled, const void* cb, const void* scb, const void* outlier_mask, void* y,
                           int N, int K, float threshold, int flags, b2l_stream_t stream) {
  B2L_CHECK_ARG(x && w_tiled && cb && scb && y && N > 0, "b2l_q8_gemv: bad argument");
  B2L_CHECK_SUPPORTED(K > 0 && K % KB == 0 && K <= MAX_K, "b2l_q8_gemv: K=%d must be a multiple of %d and <= %d", K, KB, MAX_K);
  B2L_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)w_tiled % 16 == 0), "b2l_q8_gemv: x / w_tiled must be 16-byte aligned");
  Params p;
  fill_params(p, x, cb, scb, outlier_mask, y, N, K, threshold);
  p.wt = (const uint8_t*)w_tiled;
  return launch_gemv<WS_TILED>(p, flags, stream);
}

extern "C" int b2l_q8_gemv_cb(const void* x, const void* cb, const void* scb, const void* outlier_mask, void* y, int N, int K,
                              float threshold, int flags, b2l_stream_t stream) {
  B2L_CHECK_ARG(x && cb && scb && y, "b2l_q8_gemv_cb: null pointer");
  B2L_CHECK_SUPPORTED(K > 0 && K % KB == 0 && K <= MAX_K, "b2l_q8_gemv_cb: K=%d must be a multiple of %d and <= %d", K, KB, MAX_K);
  B2L_CHECK_ARG(N > 0, "b2l_q8_gemv_cb: bad shape N=%d", N);
  B2L_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)cb % 16 == 0), "b2l_q8_gemv_cb: x / cb must be 16-byte aligned");
  B2L_CHECK_SUPPORTED((flags & ~B2L_F_PDL) == 0, "b2l_q8_gemv_cb: unknown flags 0x%x (only B2L_F_PDL)", (unsigned)flags);
  Params p;
  fill_params(p, x, cb, scb, outlier_mask, y, N, K, threshold);
  return launch_gemv<WS_CB>(p, flags, stream);
}

namespace b2l {
// b2l_q8_linear's argument checks: 0, or B2L_E_* with a message
int check_q8_linear(const b2l_q8_linear_args* a) {
  B2L_CHECK_ARG(a != nullptr && a->x && a->cb && a->scb && a->y, "b2l_q8_linear: null pointer");
  const int N = a->N, K = a->K;
  B2L_CHECK_SUPPORTED(K > 0 && K % KB == 0 && K <= MAX_K, "b2l_q8_linear: K=%d must be a multiple of %d and <= %d", K, KB, MAX_K);
  B2L_CHECK_ARG(N > 0, "b2l_q8_linear: bad shape N=%d", N);
  B2L_CHECK_ARG(a->prologue == B2L_PRO_NONE || a->prologue == B2L_PRO_RMSNORM, "b2l_q8_linear: bad prologue %d", a->prologue);
  B2L_CHECK_ARG(a->epilogue == B2L_EPI_STORE || a->epilogue == B2L_EPI_RESIDUAL || a->epilogue == B2L_EPI_SWIGLU,
                "b2l_q8_linear: bad epilogue %d", a->epilogue);
  const bool norm = a->prologue == B2L_PRO_RMSNORM, glu = a->epilogue == B2L_EPI_SWIGLU;
  B2L_CHECK_ARG(!norm || a->norm_scale, "b2l_q8_linear: RMSNORM needs norm_scale");
  B2L_CHECK_ARG(a->epilogue != B2L_EPI_RESIDUAL || a->res, "b2l_q8_linear: RESIDUAL needs res");
  B2L_CHECK_ARG(!glu || (a->cb2 && a->scb2), "b2l_q8_linear: SWIGLU needs cb2 and scb2");
  B2L_CHECK_ARG((a->out_affine.scale == nullptr) == (a->out_affine.bias == nullptr),
                "b2l_q8_linear: out_affine needs both scale and bias (or neither)");
  B2L_CHECK_ARG(((uintptr_t)a->x | (uintptr_t)a->cb | (uintptr_t)(glu ? a->cb2 : nullptr) |
                 (uintptr_t)(norm ? a->norm_scale : nullptr)) % 16 == 0,
                "b2l_q8_linear: x / cb / cb2 / norm_scale must be 16-byte aligned");
  B2L_CHECK_SUPPORTED((a->flags & ~B2L_F_PDL) == 0, "b2l_q8_linear: unknown flags 0x%x (only B2L_F_PDL)", (unsigned)a->flags);
  return 0;
}

// b2l_q8_linear's and b2l_q8_linear_batch's M rows of y must not overlap x: the kernels read x after they start writing y
int check_q8_disjoint(const b2l_q8_linear_args* a, int M, const char* who) {
  const uintptr_t x0 = (uintptr_t)a->x, y0 = (uintptr_t)a->y;
  B2L_CHECK_ARG(y0 + 2 * (size_t)M * a->N <= x0 || x0 + 2 * (size_t)M * a->K <= y0, "%s: y overlaps x", who);
  return 0;
}
}  // namespace b2l

extern "C" int b2l_q8_linear(const b2l_q8_linear_args* a, b2l_stream_t stream) {
  if (int rc = check_q8_linear(a)) return rc;
  if (int rc = check_q8_disjoint(a, 1, "b2l_q8_linear")) return rc;
  const int N = a->N, K = a->K;
  const bool norm = a->prologue == B2L_PRO_RMSNORM, glu = a->epilogue == B2L_EPI_SWIGLU;
  Params p;
  fill_params(p, a->x, a->cb, a->scb, nullptr, a->y, N, K, a->threshold);
  p.n_rb = glu ? (N + 7) / 8 : (N + RB - 1) / RB;
  p.cb2 = (const int8_t*)a->cb2; p.scb2 = (const float*)a->scb2;
  p.norm_scale = norm ? (const __nv_bfloat16*)a->norm_scale : nullptr; p.eps = a->eps;
  p.epilogue = a->epilogue; p.res = (const __nv_bfloat16*)a->res;
  p.aff_s = (const __nv_bfloat16*)a->out_affine.scale; p.aff_b = (const __nv_bfloat16*)a->out_affine.bias;
  return launch_gemv<WS_CB, true>(p, a->flags, stream);
}

// outlier columns of a batch: bit k set iff any row has |fp16(x[m][k])| >= threshold
__global__ void q8_outlier_mask_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int M, int K, float threshold, uint32_t* __restrict__ mask) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  bool o = false;
  if (k < K)
    for (int m = 0; m < M; ++m) o |= fabsf(__half2float(__float2half_rn(bf2f(x[(size_t)m * ldx + k])))) >= threshold;
  const uint32_t b = __ballot_sync(0xffffffffu, o);
  if ((threadIdx.x & 31) == 0 && k < K) mask[k >> 5] = b;
}

extern "C" int b2l_q8_outlier_mask(const void* x, int ldx, int M, int K, float threshold, void* mask, b2l_stream_t stream) {
  B2L_CHECK_ARG(x && mask && M > 0 && K > 0 && K % 32 == 0, "b2l_q8_outlier_mask: bad argument");
  q8_outlier_mask_kernel<<<(K + 255) / 256, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, ldx, M, K, threshold, (uint32_t*)mask);
  B2L_LAUNCH_CHECK("q8_outlier_mask_kernel");
  return 0;
}

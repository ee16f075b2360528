// Batched decode kernel for gptq.int8: fused [RMSNorm ->] 8-bit weight-only linear [-> residual | SwiGLU] for 2..16
// activation rows, on the resident batch-1 tiling (b2l_w8_tile_i8) and in the batch-1 kernel's exact integer form.
//
// Replaces the same reference code as b2l_w8_gemv (ColBlockQuantizedLinear.forward, lit_llama/quantization.py:413-423,
// with the RMSNorm of lit_llama/model.py:270-277 in front and x + h / silu(a) * b of model.py:166-167, 252 behind)
// for B > 1 (model.py:76-122 accepts any batch).
//
// Contraction (q4_gemv.cu, W8 = true), extended to columns.  Each activation row n gets its own power of two 2^sh_n
// from max|x_n|, is rounded to X_n (|X_n| < 2^22) and split into three balanced base-256 digit planes, exactly as
// the batch-1 prologue does it.  The 3 M planes are the columns of mma.m16n8k32 (u8 x s8 -> s32): ceil(3M / 8)
// IMMA.16832 per 16 x 32 weight tile (1 at M <= 2, 3 at M = 8, 6 at M = 16).  The int32 sums are exact and do not
// depend on their order, the digits are recombined in int64 and each row's zero point is removed with that row's
// exact sum of X_n: y = scale * 2^-sh_n * (sum level X_n - zero * sum X_n), rounded as in the batch-1 epilogue.  Row
// n of a batch is therefore bit-identical to b2l_w8_gemv on row n alone.
//
// 3 M K bytes of digits (65B mlp.c_proj at M = 16: 1 MB) do not fit beside the weight ring, so, as in
// q4_gemv_batch.cu:
//   1. w8_batch_prep_kernel (one CTA per activation row) applies RMSNorm and writes the digit planes, sh_n and
//      sum X_n to a workspace that stays in L2.  It is the batch-1 prologue with the same 256-thread split and the
//      same reduction order, so sh_n and X_n are the batch-1 kernel's;
//   2. w8_gemv_batch_kernel streams, per stage of 8 k blocks x 2 row blocks of weights (16 KB), the 3 M digit planes
//      of those k blocks (1.5 KB per row) through the same mbarrier ring.  The weight copies of the first ring-full
//      are issued before griddepcontrol.wait, the digit copies after it.
// Every consumer warp owns one k block of a stage; its int32 partials are added into a per-unit shared-memory
// buffer with integer atomics (exact, any order) that the epilogue warp reads, converts and clears.
//
// Workspace (b2l_w8_gemv_batch_workspace_bytes): [K/64 k blocks][3M planes (row n digit d = plane 3n + d)][4 t][16 B]
// in the batch-1 plane order, then int64 sum X [16] and int sh [16].
//
// gptq.int4 (b2l_q4_gemv_batch_i8) runs the same prep kernel, workspace, ring, reduction and epilogue with W8 = false,
// on the resident batch-1 int4 tiling (b2l_q4_tile_i8, q4_gemv.cu): a (16-row block, k block) tile is 512 B of packed
// nibbles, fed to the MMA as in single_imma<false> -- the unmasked word as the operand of row g, the word & 0xf0f0f0f0
// as that of row g + 8, one LOP3 per word shared by every column group -- and each partial is turned back into the
// row pair (row g = D[g] - D[g+8], row g + 8 = D[g+8] >> 4, exact and linear) before it is added into the unit's
// buffer.  Stage geometry: still 8 k blocks per stage, one per consumer warp, so the 4-bit half stages are 4 KB.
// Sixteen k blocks per stage (two per warp) would keep 8 KB half stages but halve the number of stages the same
// shared memory holds; at 8 KB of weights per stage a 110 KB CTA still keeps >= 72 KB of weights in flight.  The
// digits of a stage are the same 3 M x 512 B at either width, so per byte of weights streamed from HBM the kernel
// reads 3 M / 16 bytes of digits from L2 at 4 bits (3 at M = 16) against 3 M / 32 at 8 bits.
#include <cstdlib>

#include "q4_mma_common.cuh"

namespace b2l {
namespace w8mb {
using namespace q4mv;

constexpr int MAXB = 16;                     // activation rows
constexpr int NDIG = 3;                      // base-256 digits per row (|X| < 2^22)
// one (16-row block, k block) tile: 1024 B of 8-bit levels (b2l_w8_tile_i8) or 512 B of packed nibbles (b2l_q4_tile_i8)
__host__ __device__ constexpr int tile_bytes(bool w8) { return w8 ? 1024 : 512; }
constexpr int KBP = HALF_STAGE_BYTES / tile_bytes(true);   // 8 k blocks per stage, one per consumer warp
static_assert(KBP == NCW, "one k block per consumer warp and stage");
constexpr int PLANE_KB_BYTES = 64;           // one digit plane of one k block: [4 t][16 B]
constexpr int BMAX_STAGES = 12;

__host__ __device__ inline uint32_t xkb_bytes(int M) { return (uint32_t)(NDIG * M * PLANE_KB_BYTES); }   // digits of one k block
// weights of a stage: KBP k blocks of both 16-row blocks of a unit (16 KB at 8 bits, 8 KB at 4 bits)
__host__ __device__ constexpr uint32_t wstage_bytes(bool w8) { return (uint32_t)(2 * KBP * tile_bytes(w8)); }
__host__ __device__ inline uint32_t bstage_bytes(int M, bool w8) { return wstage_bytes(w8) + KBP * xkb_bytes(M); }   // [weights][digits]
__host__ __device__ inline int scratch_stride(int M) { return (NDIG * M) | 1; }   // ints per result row (odd: no bank conflicts)
__host__ __device__ inline size_t frag_bytes(int K, int M) { return (size_t)NDIG * M * K; }

struct BParams {
  const uint8_t* qwt;
  const void* scales; const void* zeros; int szdt;
  const uint8_t* xfrag;      // workspace digit planes
  const long long* sum_x;    // workspace sum X [16]
  const int* sh;             // workspace sh [16]
  __nv_bfloat16* y; int ldy;
  int M, N, K, n_rb;
  int epilogue; const __nv_bfloat16* res; int ldres;
  int nst;
};

struct BSmem {
  uint32_t ring, scratch, rowc, bars, total;
};
__host__ __device__ inline BSmem bsmem_layout(int nst, int M, bool w8) {
  BSmem L;
  uint32_t o = 0;
  L.ring = o;    o += (uint32_t)nst * bstage_bytes(M, w8);
  L.scratch = o; o += (2u * 2 * RB * scratch_stride(M) * 4 + 15u) & ~15u;   // [buf][32 result rows][stride] int32
  L.rowc = o;    o += 2 * MAXB * 8;                                        // double[16] sum X, double[16] 2^-sh
  L.bars = o;    o += 2 * BMAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

// ---------------------------------------------------------------- step 1: activation rows -> digit planes
// The consumer-warp prologue of q4_gemv_kernel for one row per CTA: the same activation conversion (act_pass1 /
// act_scale / act_digits, q4_mma_common.cuh), thread split and reduction order.
template <int MAXC>
__global__ void __launch_bounds__(256) w8_batch_prep_kernel(const __nv_bfloat16* x, int ldx, int M, int K,
                                                            const __nv_bfloat16* __restrict__ norm_scale, float eps,
                                                            uint8_t* __restrict__ ws) {
  __shared__ float red[16];          // [0..7] sum of squares, [8..15] max |x| (max |bf16(g x)| with RMSNorm)
  __shared__ long long sred[8];
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NT = 256;
  pdl_launch_dependents();  // the linear may start streaming its weights
  const bool norm = norm_scale != nullptr;
  uint4 xv[MAXC], gv[MAXC];
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int k = (c * NT + tid) * 8;
    gv[c] = make_uint4(0, 0, 0, 0);
    if (norm && k < K) gv[c] = *reinterpret_cast<const uint4*>(norm_scale + k);
  }
  pdl_wait();
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int k = (c * NT + tid) * 8;
    xv[c] = make_uint4(0, 0, 0, 0);
    if (k < K) xv[c] = ld_coherent_u4(x + (size_t)n * ldx + k);   // written by the previous kernel (PDL): coherent load
  }
  const int nchunk = (K + NT * 8 - 1) / (NT * 8);
  float ss, mx;
  act_pass1<MAXC>(xv, gv, nchunk, norm, ss, mx);
  ss = warp_sum(ss);
  mx = warp_max(mx);
  if (lane == 0) { red[warp] = ss; red[8 + warp] = mx; }
  __syncthreads();
  ss = 0.f; mx = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) { ss += red[w]; mx = fmaxf(mx, red[8 + w]); }
  const ActScale as = act_scale<NDIG>(ss, mx, norm, K, eps);
  const uint32_t XKB = xkb_bytes(M);
  uint32_t sxu = 0;
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int k = (c * NT + tid) * 8;
    if (c < nchunk && k < K) {
      uint32_t dj[2][3];
      act_digits(xv[c], gv[c], norm, as, dj, sxu);
      // k = 64 kb + 32 c32 + 8 t + (0..7): k block kb, plane 3n + d, lane slot t, words 2 c32, 2 c32 + 1
      uint8_t* dst = ws + (size_t)(k >> 6) * XKB + (size_t)(NDIG * n) * PLANE_KB_BYTES + ((k >> 3) & 3) * 16 + ((k >> 5) & 1) * 8;
#pragma unroll
      for (int d = 0; d < NDIG; ++d) *reinterpret_cast<uint2*>(dst + d * PLANE_KB_BYTES) = make_uint2(dj[0][d], dj[1][d]);
    }
  }
  // exact sum of X over the row (integers: the order does not matter)
  long long sx = (long long)(int)sxu;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o);
  if (lane == 0) sred[warp] = sx;
  __syncthreads();
  if (tid == 0) {
    long long t = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sred[w];
    long long* sum_x = reinterpret_cast<long long*>(ws + frag_bytes(K, M));
    sum_x[n] = t;
    reinterpret_cast<int*>(sum_x + MAXB)[n] = as.sh;
  }
}

// ---------------------------------------------------------------- step 2: the streaming contraction
// NG = ceil(3M / 8) column groups of the MMA.  Lane (g, t) of group G feeds column g = plane 8G + g (zero past 3M).
// W8: 8-bit levels (b2l_w8_tile_i8); false: 4-bit levels (b2l_q4_tile_i8).
template <int NG, bool W8>
__global__ void __launch_bounds__(NTHREADS, NG <= 2 ? 2 : 1) w8_gemv_batch_kernel(const BParams p) {
  constexpr uint32_t TILE = tile_bytes(W8), WHALF = KBP * TILE, WSTAGE = 2 * WHALF;
  extern __shared__ __align__(128) uint8_t smem[];
  const BSmem L = bsmem_layout(p.nst, p.M, W8);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_kb = p.K / KB;
  const int spu = (n_kb + KBP - 1) / KBP;   // stages per unit
  const int rb_lo = (int)(((long long)blockIdx.x * p.n_rb) / gridDim.x);
  const int rb_hi = (int)(((long long)(blockIdx.x + 1) * p.n_rb) / gridDim.x);
  const int n_units = (rb_hi - rb_lo + 1) / 2;
  const int total_stages = n_units * spu;
  const uint32_t bar_full = sbase + L.bars, bar_empty = bar_full + BMAX_STAGES * 8;
  const uint32_t SB = bstage_bytes(p.M, W8), XKB = xkb_bytes(p.M);
  const int NP = NDIG * p.M, RS = scratch_stride(p.M);

  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) {
      mbar_init(bar_full + i * 8, 1);
      mbar_init(bar_empty + i * 8, NCW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      const int pre = min(total_stages, p.nst);   // stages whose weights are requested before the dependency resolves
      for (int it = 0; it < total_stages; ++it) {
        const int u = it / spu, s = it - u * spu;
        const int slot = it % p.nst;
        const uint32_t phase = ((uint32_t)(it / p.nst) & 1u) ^ 1u;   // fresh barriers: parity 1 passes immediately
        const int rb = rb_lo + 2 * u;
        const int halves = min(2, rb_hi - rb);
        const int nkb = min(KBP, n_kb - s * KBP);
        const uint32_t wbytes = (uint32_t)nkb * TILE, xbytes = (uint32_t)nkb * XKB;
        const uint32_t stage = sbase + L.ring + slot * SB;
        mbar_wait(bar_empty + slot * 8, phase);
        mbar_expect_tx(bar_full + slot * 8, wbytes * halves + xbytes);
        const uint8_t* wsrc = p.qwt + (size_t)rb * n_kb * TILE;
        for (int h = 0; h < halves; ++h)
          tma_bulk_g2s(stage + h * WHALF, wsrc + ((size_t)h * n_kb + (size_t)s * KBP) * TILE, wbytes,
                       bar_full + slot * 8);
        if (it >= pre) {
          tma_bulk_g2s(stage + WSTAGE, p.xfrag + (size_t)s * KBP * XKB, xbytes, bar_full + slot * 8);
        } else if (it + 1 == pre) {
          // ring full of weights: let the next kernel in, wait for the digits' producer, then request the digits of
          // every stage issued so far
          pdl_launch_dependents();
          pdl_wait();
          // the digits were written with ordinary stores by the previous grid and are read by the async proxy
          asm volatile("fence.proxy.async;" ::: "memory");
          for (int j = 0; j < pre; ++j) {
            const int uj = j / spu, sj = j - uj * spu;
            const int nkbj = min(KBP, n_kb - sj * KBP);
            tma_bulk_g2s(sbase + L.ring + (j % p.nst) * SB + WSTAGE, p.xfrag + (size_t)sj * KBP * XKB,
                         (uint32_t)nkbj * XKB, bar_full + (j % p.nst) * 8);
          }
        }
      }
      if (total_stages == 0) pdl_launch_dependents();
    }
  } else if (warp < NCW) {
    // ===================== consumer warps: warp w takes k block w of every stage =====================
    const int g = lane >> 2, t4 = lane & 3;
    int xoff[NG];
#pragma unroll
    for (int G = 0; G < NG; ++G) xoff[G] = (8 * G + g < NP) ? (8 * G + g) * PLANE_KB_BYTES + t4 * 16 : -1;
    int slot = 0;
    uint32_t phase = 0;
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    for (int u = 0; u < n_units; ++u) {
      const int halves = min(2, rb_hi - (rb_lo + 2 * u));
      int acc[NG][MAX_HALVES][4];
#pragma unroll
      for (int G = 0; G < NG; ++G)
#pragma unroll
        for (int h = 0; h < MAX_HALVES; ++h)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[G][h][i] = 0;
      for (int s = 0; s < spu; ++s) {
        const int nkb = min(KBP, n_kb - s * KBP);
        mbar_wait(bar_full + slot * 8, phase);
        if (warp < nkb) {
          const uint8_t* st = smem + L.ring + slot * SB;
          const uint8_t* wt = st + warp * TILE + lane * 16;
          const uint8_t* xs = st + WSTAGE + warp * XKB;
          if constexpr (W8) {
            const uint4 a0 = *reinterpret_cast<const uint4*>(wt), a1 = *reinterpret_cast<const uint4*>(wt + 512);
            uint4 b0 = make_uint4(0, 0, 0, 0), b1 = b0;
            if (halves == MAX_HALVES) {
              b0 = *reinterpret_cast<const uint4*>(wt + WHALF);
              b1 = *reinterpret_cast<const uint4*>(wt + WHALF + 512);
            }
#pragma unroll
            for (int G = 0; G < NG; ++G) {
              uint4 xb = make_uint4(0, 0, 0, 0);
              if (xoff[G] >= 0) xb = *reinterpret_cast<const uint4*>(xs + xoff[G]);
              mma_u8s8_16832(acc[G][0], a0.x, a0.y, a0.z, a0.w, xb.x, xb.y);
              mma_u8s8_16832(acc[G][0], a1.x, a1.y, a1.z, a1.w, xb.z, xb.w);
              if (halves == MAX_HALVES) {
                mma_u8s8_16832(acc[G][1], b0.x, b0.y, b0.z, b0.w, xb.x, xb.y);
                mma_u8s8_16832(acc[G][1], b1.x, b1.y, b1.z, b1.w, xb.z, xb.w);
              }
            }
          } else {
            // a packed byte is level[g] + 16 level[g + 8]: unmasked for row g, high nibble only for row g + 8
            constexpr uint32_t HI = 0xf0f0f0f0u;
            const uint4 a = *reinterpret_cast<const uint4*>(wt);
            uint4 b = make_uint4(0, 0, 0, 0);
            if (halves == MAX_HALVES) b = *reinterpret_cast<const uint4*>(wt + WHALF);
            const uint4 ah = make_uint4(a.x & HI, a.y & HI, a.z & HI, a.w & HI);
            const uint4 bh = make_uint4(b.x & HI, b.y & HI, b.z & HI, b.w & HI);
#pragma unroll
            for (int G = 0; G < NG; ++G) {
              uint4 xb = make_uint4(0, 0, 0, 0);
              if (xoff[G] >= 0) xb = *reinterpret_cast<const uint4*>(xs + xoff[G]);
              mma_u8s8_16832(acc[G][0], a.x, ah.x, a.y, ah.y, xb.x, xb.y);
              mma_u8s8_16832(acc[G][0], a.z, ah.z, a.w, ah.w, xb.z, xb.w);
              if (halves == MAX_HALVES) {
                mma_u8s8_16832(acc[G][1], b.x, bh.x, b.y, bh.y, xb.x, xb.y);
                mma_u8s8_16832(acc[G][1], b.z, bh.z, b.w, bh.w, xb.z, xb.w);
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + slot * 8);
        if (++slot == p.nst) { slot = 0; phase ^= 1; }
      }
      // 16 x 8 tile of group G: lane (g, t) holds rows g (c0, c1) and g + 8 (c2, c3) of columns 8G + 2t, 8G + 2t + 1.
      // 4 bits: row g = D[g] - D[g+8], row g + 8 = D[g+8] >> 4 (every term of D[g+8] is a multiple of 16: exact)
      const int buf = u & 1;
      named_bar_sync(4 + buf, NCW * 32 + 32);   // the epilogue warp has read and cleared this buffer (two units ago)
      int* sb = scratch + buf * 2 * RB * RS;
#pragma unroll
      for (int G = 0; G < NG; ++G) {
        const int col = 8 * G + 2 * t4;
#pragma unroll
        for (int h = 0; h < MAX_HALVES; ++h) {
          if (h < halves) {
            int* r0 = sb + (h * RB + g) * RS + col;
            int* r8 = r0 + 8 * RS;
            int c0 = acc[G][h][0], c1 = acc[G][h][1], c2 = acc[G][h][2], c3 = acc[G][h][3];
            if constexpr (!W8) {
              c0 -= c2; c1 -= c3;
              c2 >>= 4; c3 >>= 4;
            }
            if (col < NP) { atomicAdd(r0, c0); atomicAdd(r8, c2); }
            if (col + 1 < NP) { atomicAdd(r0 + 1, c1); atomicAdd(r8 + 1, c3); }
          }
        }
      }
      __syncwarp();
      named_bar_arrive(6 + buf, NCW * 32 + 32);  // partials of this unit are in the buffer
    }
  } else {
    // ===================== epilogue warp: lane = row of the 32-row unit, all M activation rows =====================
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    for (int i = lane; i < 2 * 2 * RB * RS; i += 32) scratch[i] = 0;
    pdl_wait();
    double* dsum = reinterpret_cast<double*>(smem + L.rowc);
    double* dinv = dsum + MAXB;
    if (lane < p.M) {
      dsum[lane] = (double)p.sum_x[lane];
      dinv[lane] = __longlong_as_double((long long)(1023 - p.sh[lane]) << 52);   // 2^-sh
    }
    __syncwarp();
    // both buffers start free
    if (n_units > 0) named_bar_arrive(4, NCW * 32 + 32);
    if (n_units > 1) named_bar_arrive(5, NCW * 32 + 32);
    for (int u = 0; u < n_units; ++u) {
      const int rb = rb_lo + 2 * u;
      const int halves = min(2, rb_hi - rb);
      const int buf = u & 1;
      const int half = lane >> 4, row = lane & 15;
      const bool active = half < halves;
      const int orow = (rb + half) * RB + row;
      const int o = min(orow, p.N - 1);
      const float sc = load_sz(p.scales, p.szdt, o);
      const float zero = load_sz(p.zeros, p.szdt, o);
      named_bar_sync(6 + buf, NCW * 32 + 32);
      int* r = scratch + buf * 2 * RB * RS + lane * RS;
      for (int n = 0; n < p.M; ++n) {   // warp-uniform (the SwiGLU shuffle needs every lane)
        // sum_k level X_n = d0 + 256 d1 + 65536 d2 (exact in int64, < 2^53)
        const long long tq = (long long)r[3 * n] + ((long long)r[3 * n + 1] << 8) + ((long long)r[3 * n + 2] << 16);
        const float tf = (float)(((double)tq - (double)zero * dsum[n]) * dinv[n]);   // sum (level - zero) x, one rounding
        const float v = rbf(sc * tf);
        if (p.epilogue == B2L_EPI_SWIGLU) {
          // rows 0..7 of a 16-row block are c_fc1[o..o+7], rows 8..15 are c_fc2[o..o+7]
          const float b = __shfl_down_sync(0xffffffffu, v, 8);
          if (active && row < 8) {
            const float sl = rbf(v / (1.0f + expf(-v)));
            p.y[(size_t)n * p.ldy + (rb + half) * 8 + row] = f2bf(sl * b);
          }
        } else if (active && orow < p.N) {
          const float resv = p.epilogue == B2L_EPI_RESIDUAL ? bf2f(p.res[(size_t)n * p.ldres + orow]) : 0.f;
          p.y[(size_t)n * p.ldy + orow] = f2bf(p.epilogue == B2L_EPI_RESIDUAL ? v + resv : v);
        }
      }
      for (int i = 0; i < NP; ++i) r[i] = 0;   // cleared for unit u + 2
      __syncwarp();
      if (u + 2 < n_units) named_bar_arrive(4 + buf, NCW * 32 + 32);   // buffer free again
    }
  }
}

}  // namespace w8mb
}  // namespace b2l

using namespace b2l;
using namespace b2l::q4mv;
using namespace b2l::w8mb;

extern "C" size_t b2l_w8_gemv_batch_workspace_bytes(int K, int M) {
  if (K <= 0 || K % KB != 0 || M < 2 || M > MAXB) return 0;
  return frag_bytes(K, M) + MAXB * (sizeof(long long) + sizeof(int));
}

namespace {
// Column groups of M rows (one instantiation of w8_gemv_batch_kernel each)
int column_groups(int M) { return std::min(6, (NDIG * M + 7) / 8); }

// Ring stages of the batch kernel at M rows (0: not even two).  1..2 column groups (M <= 5): two CTAs per SM; more:
// one CTA per SM with a deeper ring
int batch_ring_stages(int M, bool W8) {
  const uint32_t budget = (column_groups(M) <= 2 ? 110u : 224u) * 1024u;
  const uint32_t fixed = bsmem_layout(0, M, W8).total, sb = bstage_bytes(M, W8);
  const int nst = fixed + 2 * sb <= budget ? (int)((budget - fixed) / sb) : 0;
  return nst > BMAX_STAGES ? BMAX_STAGES : nst;
}

template <int NG, bool W8>
int launch_batch(const BParams& p0, int grid_override, bool pdl, cudaStream_t stream) {
  BParams p = p0;
  const int ctas_per_sm = NG <= 2 ? 2 : 1;
  p.nst = batch_ring_stages(p.M, W8);
  const BSmem L = bsmem_layout(p.nst, p.M, W8);
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(w8_gemv_batch_kernel<NG, W8>, L.total, smem_cache)) return rc;
  int grid = grid_override > 0 ? grid_override : ctas_per_sm * sm_count();
  if (grid > p.n_rb) grid = p.n_rb;
  LaunchCfg lc(dim3(grid), dim3(NTHREADS), L.total, stream, pdl, 1);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, w8_gemv_batch_kernel<NG, W8>, p));
  return 0;
}

}  // namespace

namespace b2l {
// b2l_w8_gemv_batch's (W8 = true) and b2l_q4_gemv_batch_i8's (W8 = false) argument checks: 0, or B2L_E_* with a message
int check_gemv_batch_i8(const b2l_q4_linear_args* a, bool W8) {
  const char* fn = W8 ? "b2l_w8_gemv_batch" : "b2l_q4_gemv_batch_i8";
  B2L_CHECK_ARG(a != nullptr, "%s: null args", fn);
  B2L_CHECK_ARG(a->x && a->qw_tiled && a->scales && a->zeros && a->y, "%s: null pointer", fn);
  B2L_CHECK_ARG(a->workspace != nullptr, "%s: null workspace (b2l_w8_gemv_batch_workspace_bytes(K, M) bytes)", fn);
  B2L_CHECK_SUPPORTED(a->out_affine.scale == nullptr && a->out_affine.bias == nullptr,
                      "%s: out_affine is not supported (apply b2l_linear_affine to y)", fn);
  B2L_CHECK_SUPPORTED(a->M >= 2 && a->M <= MAXB, "%s: M=%d (2..%d activation rows; use %s for 1)", fn, a->M, MAXB,
                      W8 ? "b2l_w8_gemv" : "b2l_q4_gemv");
  B2L_CHECK_SUPPORTED(a->K > 0 && a->K % KB == 0 && a->K <= MAX_K, "%s: K=%d must be a multiple of %d and <= %d", fn, a->K, KB, MAX_K);
  B2L_CHECK_ARG(a->N > 0, "%s: bad N", fn);
  B2L_CHECK_ARG(a->ldx >= a->K && a->ldx % 8 == 0, "%s: ldx=%d must be >= K and a multiple of 8", fn, a->ldx);
  B2L_CHECK_ARG(((uintptr_t)a->x % 16 == 0) && ((uintptr_t)a->qw_tiled % 16 == 0) && ((uintptr_t)a->workspace % 16 == 0),
                "%s: x / qw_tiled / workspace must be 16-byte aligned", fn);
  B2L_CHECK_ARG(a->sz_dtype == B2L_BF16 || a->sz_dtype == B2L_F32, "%s: bad sz_dtype", fn);
  B2L_CHECK_SUPPORTED((a->flags & ~B2L_F_PDL) == 0, "%s: unknown flags 0x%x", fn, a->flags);
  if (a->prologue == B2L_PRO_RMSNORM)
    B2L_CHECK_ARG(a->norm_scale && ((uintptr_t)a->norm_scale % 16 == 0), "%s: RMSNorm prologue needs a 16-byte aligned scale", fn);
  else
    B2L_CHECK_ARG(a->prologue == B2L_PRO_NONE, "%s: bad prologue %d", fn, a->prologue);
  if (a->epilogue == B2L_EPI_RESIDUAL) {
    B2L_CHECK_ARG(a->res != nullptr, "%s: RESIDUAL epilogue needs res", fn);
    B2L_CHECK_ARG(a->ldres >= a->N, "%s: ldres=%d < N=%d", fn, a->ldres, a->N);
  } else if (a->epilogue == B2L_EPI_SWIGLU) {
    B2L_CHECK_SUPPORTED(a->N % RB == 0, "%s: SWIGLU needs N %% 16 == 0", fn);
  } else {
    B2L_CHECK_ARG(a->epilogue == B2L_EPI_STORE, "%s: bad epilogue %d", fn, a->epilogue);
  }
  B2L_CHECK_ARG(a->ldy >= (a->epilogue == B2L_EPI_SWIGLU ? a->N / 2 : a->N), "%s: ldy=%d is too small", fn, a->ldy);
  B2L_CHECK_SUPPORTED(batch_ring_stages(a->M, W8) >= 2, "%s: M=%d does not leave room for the weight ring", fn, a->M);
  return 0;
}
}  // namespace b2l

namespace {
// b2l_w8_gemv_batch (W8 = true) and b2l_q4_gemv_batch_i8 (W8 = false): the same checks, workspace and launches
template <bool W8>
int batch_entry(const b2l_q4_linear_args* a, b2l_stream_t stream) {
  if (int rc = check_gemv_batch_i8(a, W8)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const bool pdl = (a->flags & B2L_F_PDL) != 0;

  uint8_t* ws = (uint8_t*)a->workspace;
  {
    LaunchCfg lc(dim3(a->M), dim3(256), 0, st, pdl, 1);
    const __nv_bfloat16* ns = a->prologue == B2L_PRO_RMSNORM ? (const __nv_bfloat16*)a->norm_scale : nullptr;
    if (a->K > 6 * 256 * 8)
      B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, w8_batch_prep_kernel<12>, (const __nv_bfloat16*)a->x, a->ldx, a->M, a->K, ns, a->eps, ws));
    else
      B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, w8_batch_prep_kernel<6>, (const __nv_bfloat16*)a->x, a->ldx, a->M, a->K, ns, a->eps, ws));
  }

  BParams p;
  p.qwt = (const uint8_t*)a->qw_tiled;
  p.scales = a->scales; p.zeros = a->zeros; p.szdt = a->sz_dtype;
  p.xfrag = ws;
  p.sum_x = (const long long*)(ws + frag_bytes(a->K, a->M));
  p.sh = (const int*)(p.sum_x + MAXB);
  p.y = (__nv_bfloat16*)a->y; p.ldy = a->ldy;
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.n_rb = (a->N + RB - 1) / RB;
  p.epilogue = a->epilogue; p.res = (const __nv_bfloat16*)a->res; p.ldres = a->ldres;
  p.nst = 0;
  const int grid = a->split_k;   // split_k doubles as a grid override
  switch (column_groups(a->M)) {
    case 1: return launch_batch<1, W8>(p, grid, pdl, st);
    case 2: return launch_batch<2, W8>(p, grid, pdl, st);
    case 3: return launch_batch<3, W8>(p, grid, pdl, st);
    case 4: return launch_batch<4, W8>(p, grid, pdl, st);
    case 5: return launch_batch<5, W8>(p, grid, pdl, st);
    default: return launch_batch<6, W8>(p, grid, pdl, st);
  }
}
}  // namespace

extern "C" int b2l_w8_gemv_batch(const b2l_q4_linear_args* a, b2l_stream_t stream) { return batch_entry<true>(a, stream); }

extern "C" int b2l_q4_gemv_batch_i8(const b2l_q4_linear_args* a, b2l_stream_t stream) { return batch_entry<false>(a, stream); }

// Batched decode kernel: fused [RMSNorm ->] int4 weight-only linear [-> residual | SwiGLU] for 2..8
// activation rows (batched generation; BASELINE.json configs[3] decodes 8 sequences at once).
//
// Same replacement as q4_gemv.cu (ColBlockQuantizedLinear.forward lit_llama/quantization.py:413-423 with the
// RMSNorm of lit_llama/model.py:270-277 in front and x + h / silu(a) * b of model.py:166-167, 252 behind) and
// the same contraction: mma.sync.m16n8k16 computes a 16-row x 8-COLUMN tile, and the batch-1 kernel uses one
// of the 8 columns.  Here column n is activation row n, so 8 sequences cost the same MMAs as one.
//
// What changes is the activation side.  8 rows of K fp16 fragments (up to 8 * 24576 * 2 B) do not fit in
// shared memory next to the weight ring, so
//   1. q4_batch_prep_kernel (one CTA per activation row) applies RMSNorm with the reference's bf16 rounding
//      points, scales row n by a power of two 2^sh_n that puts its largest magnitude in [2^14, 2^15), converts
//      to fp16 in MMA B-fragment order (upper k half of every k16 chunk pre-divided by 16, see q4_gemv.cu) and
//      writes them, plus the two per-row sums the zero-point correction needs and 2^-sh_n, to a workspace that
//      stays in L2.  The epilogue multiplies by 2^-sh_n before its bf16 rounding, so a row's result does not
//      depend on its magnitude: y(2^e x) = 2^e y(x) bit for bit, whatever the other rows hold;
//   2. q4_gemv_batch_kernel streams, per 16 KB weight stage, the matching 16 KB of activation fragments
//      through the same mbarrier ring (one more TMA bulk copy per stage).  The weight copies of the first
//      ring-full are issued before griddepcontrol.wait; the fragment copies, which depend on step 1, after.
// Work split, ring, warp roles, reduction order and epilogue are those of q4_gemv.cu; results are
// bit-deterministic.
//
// Workspace (b2l_q4_gemv_batch_workspace_bytes): [K/64 k blocks][2 planes][32 lanes][16 B] fragments, lane
// 4n + t holding row n; then float[8][2] = {sum over the lower k halves, sum over the upper k halves} of the scaled
// values, then float[8] = 2^-sh_n.
#include <cstdlib>

#include "q4_mma_common.cuh"

namespace b2l {
namespace q4mb {
using namespace q4mv;

constexpr int MAXB = 8;                                  // activation rows = MMA columns
constexpr int XKB_BYTES = 1024;                          // fragments of one k block: 2 planes x 32 lanes x 16 B
constexpr int XSTAGE_BYTES = KBP_PER_STAGE * XKB_BYTES;  // 16 KB
constexpr int BSTAGE_BYTES = STAGE_BYTES + XSTAGE_BYTES; // 32 KB: [weights, two halves][activation fragments]
constexpr int BMAX_STAGES = 3;
constexpr int TILE_F = RB * MAXB;                        // 128 fp32 results of a 16-row half

struct BParams {
  const uint8_t* qwt;
  const void* scales; const void* zeros; int szdt;
  const uint8_t* xfrag;   // workspace fragments
  const float* sums;      // workspace sums [8][2]
  __nv_bfloat16* y; int ldy;
  int M, N, K, n_rb;
  int epilogue; const __nv_bfloat16* res; int ldres;
  int nst;
};

struct BSmem {
  uint32_t ring, scratch, bars, total;
};
__host__ __device__ inline BSmem bsmem_layout(int nst) {
  BSmem L;
  uint32_t o = 0;
  L.ring = o;    o += (uint32_t)nst * BSTAGE_BYTES;
  L.scratch = o; o += 2 * NCW * MAX_HALVES * TILE_F * 4;   // [buf][warp][half][row][col] fp32 partials
  L.bars = o;    o += 2 * BMAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

// ---------------------------------------------------------------- step 1: activations -> fragments
template <int MAXC>
__global__ void __launch_bounds__(256) q4_batch_prep_kernel(const __nv_bfloat16* x, int ldx, int M, int K,
                                                            const __nv_bfloat16* __restrict__ norm_scale, float eps,
                                                            uint32_t* __restrict__ xfrag, float* __restrict__ sums) {
  __shared__ float red[32];   // [0..7] sum of squares, [8..23] the two half sums, [24..31] max |v|
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NT = 256;
  pdl_launch_dependents();  // the linear may start streaming its weights
  const bool norm = norm_scale != nullptr;
  const bool live = n < M;   // rows beyond M are written as zeros (their MMA columns are ignored, but must be finite)
  uint4 xv[MAXC], gv[MAXC];
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int k = (c * NT + tid) * 8;
    gv[c] = make_uint4(0, 0, 0, 0);
    if (live && norm && k < K) gv[c] = *reinterpret_cast<const uint4*>(norm_scale + k);
  }
  pdl_wait();
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int k = (c * NT + tid) * 8;
    xv[c] = make_uint4(0, 0, 0, 0);
    if (live && k < K) xv[c] = ld_coherent_u4(x + (size_t)n * ldx + k);   // written by the previous kernel (PDL): coherent load
  }
  const int nchunk = (K + NT * 8 - 1) / (NT * 8);
  float rinv = 1.f;
  if (norm) {   // model.py:270-277 in bf16: HMUL2 is the exactly rounded bf16 product
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nchunk) {
        const uint32_t w[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
          const __nv_bfloat162 sq = __hmul2(v, v);
          const uint32_t su = *reinterpret_cast<const uint32_t*>(&sq);
          ss += __uint_as_float(su << 16) + __uint_as_float(su & 0xffff0000u);
        }
      }
    }
    ss = warp_sum(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    ss = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) ss += red[w];
    rinv = rms_rinv(ss, K, eps);
  }
  // the values the reference feeds its linear (RMSNorm applied in place), and their largest magnitude
  const __nv_bfloat162 rinv2 = __float2bfloat162_rn(rinv);
  __nv_bfloat162 amax2 = __float2bfloat162_rn(0.f);
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    if (c < nchunk) {
      uint32_t w[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w};
      const uint32_t g[4] = {gv[c].x, gv[c].y, gv[c].z, gv[c].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
        if (norm) v = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(&g[q]), __hmul2(v, rinv2));
        amax2 = __hmax2(amax2, __habs2(v));
        w[q] = *reinterpret_cast<const uint32_t*>(&v);
      }
      xv[c] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  const float mx = warp_max(fmaxf(__low2float(amax2), __high2float(amax2)));
  if (lane == 0) red[24 + warp] = mx;
  __syncthreads();
  float rmax = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) rmax = fmaxf(rmax, red[24 + w]);
  // Row scale 2^sh: the largest magnitude lands in [2^14, 2^15).  The fp16 operands and the fp32 sums are then the
  // same numbers for x and 2^e x (power-of-two scaling is exact), nothing saturates (|lower half| < 2^15, upper half
  // < 2^11), and a bf16 element converts to fp16 exactly unless it lies more than 2^27 below the row's largest.
  const int e = (int)((__float_as_uint(rmax) >> 23) & 0xffu) - 127;   // rmax in [2^e, 2^(e + 1)); a zero row: e = -127
  const int sh = max(-126, min(126, 14 - e));
  const float scale = __uint_as_float((uint32_t)(sh + 127) << 23);
  float sx = 0.f;
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int k = (c * NT + tid) * 8;
    if (c < nchunk && k < K) {
      const uint32_t w[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w};
      // 8 consecutive k = one half of a k16 chunk; pair q belongs to lane 4n + q, register (c16, half)
      const int kb = k >> 6, c16 = (k >> 4) & 3, half = (k >> 3) & 1;
      const float pre = half ? 0.0625f : 1.0f;
      uint32_t* dst = xfrag + ((size_t)(kb * 2 + (c16 >> 1)) * 32 + n * 4) * 4 + (c16 & 1) * 2 + half;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float lo = __uint_as_float(w[q] << 16) * scale, hi = __uint_as_float(w[q] & 0xffff0000u) * scale;
        sx += lo + hi;
        dst[q * 4] = pack_f16x2(lo * pre, hi * pre);
      }
    }
  }
  // even threads hold lower-half sums, odd threads upper-half sums (the half is tid & 1)
#pragma unroll
  for (int o = 16; o > 1; o >>= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o);
  if (lane < 2) red[8 + 8 * lane + warp] = sx;
  __syncthreads();
  if (tid < 2) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[8 + 8 * tid + w];   // fixed order
    sums[n * 2 + tid] = t;
    if (tid == 0) sums[2 * MAXB + n] = __uint_as_float((uint32_t)(127 - sh) << 23);   // 2^-sh
  }
}

// ---------------------------------------------------------------- step 2: the streaming contraction
__global__ void __launch_bounds__(NTHREADS, 2) q4_gemv_batch_kernel(const BParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const BSmem L = bsmem_layout(p.nst);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_kb = p.K / KB;
  const int stages_per_unit = (n_kb + KBP_PER_STAGE - 1) / KBP_PER_STAGE;
  const int rb_lo = (int)(((long long)blockIdx.x * p.n_rb) / gridDim.x);
  const int rb_hi = (int)(((long long)(blockIdx.x + 1) * p.n_rb) / gridDim.x);
  const int n_units = (rb_hi - rb_lo + 1) / 2;
  const int total_stages = n_units * stages_per_unit;
  const uint32_t bar_full = sbase + L.bars, bar_empty = bar_full + BMAX_STAGES * 8;

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
      // stage `it` of this CTA: unit it / spu, stage it % spu, ring slot it % nst
      const int pre = min(total_stages, p.nst);   // stages whose weights are requested before the dependency resolves
      for (int it = 0; it < total_stages; ++it) {
        const int u = it / stages_per_unit, s = it - u * stages_per_unit;
        const int slot = it % p.nst;
        const uint32_t phase = ((uint32_t)(it / p.nst) & 1u) ^ 1u;   // fresh barriers: parity 1 passes immediately
        const int rb = rb_lo + 2 * u;
        const int halves = min(2, rb_hi - rb);
        const int nkb = min(KBP_PER_STAGE, n_kb - s * KBP_PER_STAGE);
        const uint32_t wbytes = (uint32_t)nkb * KB_BYTES, xbytes = (uint32_t)nkb * XKB_BYTES;
        const uint32_t stage = sbase + L.ring + slot * BSTAGE_BYTES;
        mbar_wait(bar_empty + slot * 8, phase);
        mbar_expect_tx(bar_full + slot * 8, wbytes * halves + xbytes);
        const uint8_t* wsrc = p.qwt + (size_t)rb * n_kb * KB_BYTES;
        for (int h = 0; h < halves; ++h)
          tma_bulk_g2s(stage + h * HALF_STAGE_BYTES, wsrc + ((size_t)h * n_kb + (size_t)s * KBP_PER_STAGE) * KB_BYTES, wbytes,
                       bar_full + slot * 8);
        if (it >= pre) {
          tma_bulk_g2s(stage + STAGE_BYTES, p.xfrag + (size_t)s * KBP_PER_STAGE * XKB_BYTES, xbytes, bar_full + slot * 8);
        } else if (it + 1 == pre) {
          // ring full of weights: let the next kernel in, wait for the fragments' producer, then request the
          // fragments of every stage issued so far
          pdl_launch_dependents();
          pdl_wait();
          // the fragments were written with ordinary stores by the previous grid and are read by the async proxy
          asm volatile("fence.proxy.async;" ::: "memory");
          for (int j = 0; j < pre; ++j) {
            const int uj = j / stages_per_unit, sj = j - uj * stages_per_unit;
            const int nkbj = min(KBP_PER_STAGE, n_kb - sj * KBP_PER_STAGE);
            tma_bulk_g2s(sbase + L.ring + (j % p.nst) * BSTAGE_BYTES + STAGE_BYTES, p.xfrag + (size_t)sj * KBP_PER_STAGE * XKB_BYTES,
                         (uint32_t)nkbj * XKB_BYTES, bar_full + (j % p.nst) * 8);
          }
        }
      }
      if (total_stages == 0) pdl_launch_dependents();
    }
  } else if (warp < NCW) {
    // ===================== consumer warps =====================
    uint32_t kmask, kmask4, kmagic;
    asm volatile("mov.b32 %0, 0x000f000f;" : "=r"(kmask));
    asm volatile("mov.b32 %0, 0x00f000f0;" : "=r"(kmask4));
    asm volatile("mov.b32 %0, 0x64006400;" : "=r"(kmagic));
    int slot = 0;
    uint32_t phase = 0;
    float* scratch = reinterpret_cast<float*>(smem + L.scratch);
    const int g = lane >> 2, t4 = lane & 3;
    for (int u = 0; u < n_units; ++u) {
      const int halves = min(2, rb_hi - (rb_lo + 2 * u));
      float acc[MAX_HALVES][2][4];
#pragma unroll
      for (int h = 0; h < MAX_HALVES; ++h)
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[h][c][i] = 0.f;
      for (int s = 0; s < stages_per_unit; ++s) {
        const int nkb = min(KBP_PER_STAGE, n_kb - s * KBP_PER_STAGE);
        mbar_wait(bar_full + slot * 8, phase);
        const uint8_t* st_base = smem + L.ring + slot * BSTAGE_BYTES + lane * 16;
        const uint8_t* xs_base = st_base + STAGE_BYTES;
#pragma unroll
        for (int i = 0; i < KBP_PER_STAGE / NCW; ++i) {
          const int kbl = i * NCW + warp;
          if (kbl < nkb) {
            const uint4 xa = *reinterpret_cast<const uint4*>(xs_base + kbl * XKB_BYTES);
            const uint4 xb = *reinterpret_cast<const uint4*>(xs_base + kbl * XKB_BYTES + 512);
            if (halves == MAX_HALVES) kblock_mma<MAX_HALVES>(acc, st_base + kbl * KB_BYTES, xa, xb, kmask, kmask4, kmagic);
            else kblock_mma<1>(acc, st_base + kbl * KB_BYTES, xa, xb, kmask, kmask4, kmagic);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + slot * 8);
        if (++slot == p.nst) { slot = 0; phase ^= 1; }
      }
      // 16x8 tiles: lane (g, t) holds rows g / g + 8, columns 2t / 2t + 1
      const int buf = u & 1;
      named_bar_sync(4 + buf, NCW * 32 + 32);
#pragma unroll
      for (int h = 0; h < MAX_HALVES; ++h) {
        float* dst = scratch + ((buf * NCW + warp) * MAX_HALVES + h) * TILE_F + g * MAXB + 2 * t4;
        *reinterpret_cast<float2*>(dst) = make_float2(acc[h][0][0] + acc[h][1][0], acc[h][0][1] + acc[h][1][1]);
        *reinterpret_cast<float2*>(dst + 8 * MAXB) = make_float2(acc[h][0][2] + acc[h][1][2], acc[h][0][3] + acc[h][1][3]);
      }
      __syncwarp();
      named_bar_arrive(6 + buf, NCW * 32 + 32);
    }
  } else {
    // ===================== epilogue warp: lane = row of the 32-row unit, all 8 columns =====================
    pdl_wait();
    const float* scratch = reinterpret_cast<const float*>(smem + L.scratch);
    float sum_lo[MAXB], sum_hi[MAXB], rscale[MAXB];
#pragma unroll
    for (int n = 0; n < MAXB; ++n) { sum_lo[n] = p.sums[2 * n]; sum_hi[n] = p.sums[2 * n + 1]; rscale[n] = p.sums[2 * MAXB + n]; }
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
      float resv[MAXB];
#pragma unroll
      for (int n = 0; n < MAXB; ++n) {
        resv[n] = 0.f;
        if (p.epilogue == B2L_EPI_RESIDUAL && active && orow < p.N && n < p.M) resv[n] = bf2f(p.res[(size_t)n * p.ldres + orow]);
      }
      named_bar_sync(6 + buf, NCW * 32 + 32);
      float t[MAXB];
#pragma unroll
      for (int n = 0; n < MAXB; ++n) t[n] = 0.f;
#pragma unroll
      for (int w = 0; w < NCW; ++w) {   // fixed order: deterministic
        const float4* src = reinterpret_cast<const float4*>(scratch + ((buf * NCW + w) * MAX_HALVES + half) * TILE_F + row * MAXB);
        const float4 a = src[0], b = src[1];
        t[0] += a.x; t[1] += a.y; t[2] += a.z; t[3] += a.w;
        t[4] += b.x; t[5] += b.y; t[6] += b.z; t[7] += b.w;
      }
      if (u + 2 < n_units) named_bar_arrive(4 + buf, NCW * 32 + 32);
#pragma unroll
      for (int n = 0; n < MAXB; ++n) {
        // t = sum q x + 64 sum_hi (see kblock_mma), in units of 2^-sh_n: exact
        const float v = rbf(sc * ((t[n] - zero * sum_lo[n]) - (64.0f + zero) * sum_hi[n]) * rscale[n]);
        if (p.epilogue == B2L_EPI_SWIGLU) {
          const float b = __shfl_down_sync(0xffffffffu, v, 8);
          if (active && row < 8 && n < p.M) {
            const float sl = rbf(v / (1.0f + expf(-v)));
            p.y[(size_t)n * p.ldy + (rb + half) * 8 + row] = f2bf(sl * b);
          }
        } else if (active && orow < p.N && n < p.M) {
          p.y[(size_t)n * p.ldy + orow] = f2bf(p.epilogue == B2L_EPI_RESIDUAL ? v + resv[n] : v);
        }
      }
    }
  }
}

// ---------------------------------------------------------------- re-tiling for the mma.sync f16 layout (this kernel's operand)
__global__ void q4_tile_mma_kernel(const uint8_t* __restrict__ qw, uint32_t* __restrict__ out, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one output word
  const int n_kb = K / KB;
  const int n_rb = (N + RB - 1) / RB;
  const size_t total = (size_t)n_rb * n_kb * 32 * 4;
  if (idx >= total) return;
  const int c = idx & 3, lane = (idx >> 2) & 31;
  const size_t rest = idx >> 7;
  const int kb = (int)(rest % n_kb), rb = (int)(rest / n_kb);
  const int g = lane >> 2, t = lane & 3;
  uint32_t w = 0;
#pragma unroll
  for (int s = 0; s < 8; ++s) {
    const int ss = s & 3;
    const int row = rb * RB + g + 8 * (ss >> 1);
    const int k = kb * KB + 16 * c + 2 * t + 8 * (ss & 1) + (s >> 2);
    if (row < N) {
      const uint8_t b = qw[(size_t)(k >> 1) * N + row];
      w |= (uint32_t)((b >> ((k & 1) * 4)) & 0xF) << (4 * s);
    }
  }
  out[idx] = w;
}

__global__ void q4_untile_mma_kernel(const uint32_t* __restrict__ tiled, uint8_t* __restrict__ qw, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one packed byte [j][o]
  const size_t total = (size_t)(K / 2) * N;
  if (idx >= total) return;
  const int o = (int)(idx % N), j = (int)(idx / N);
  const int n_kb = K / KB;
  uint8_t b = 0;
#pragma unroll
  for (int nr = 0; nr < 2; ++nr) {
    const int k = 2 * j + nr;
    const int kb = k / KB, kl = k % KB, c = kl >> 4, k16 = kl & 15;
    const int hi8 = k16 >> 3, t = (k16 & 7) >> 1, odd = k16 & 1;
    const int rb = o / RB, rl = o % RB, g = rl & 7, r8 = rl >> 3;
    const int s = (r8 << 1 | hi8) + 4 * odd;
    const uint32_t w = tiled[(((size_t)rb * n_kb + kb) * 32 + (g * 4 + t)) * 4 + c];
    b |= (uint8_t)(((w >> (4 * s)) & 0xF) << (4 * nr));
  }
  qw[idx] = b;
}

}  // namespace q4mb
}  // namespace b2l

using namespace b2l;
using namespace b2l::q4mv;
using namespace b2l::q4mb;

extern "C" size_t b2l_q4_tiled_mma_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || K % KB != 0) return 0;
  return (size_t)((N + RB - 1) / RB) * (K / KB) * KB_BYTES;
}

extern "C" int b2l_q4_tile_mma(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_q4_tile_mma: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_q4_tile_mma: in_features %d must be a multiple of %d", K, KB);
  const size_t total = b2l_q4_tiled_mma_bytes(N, K) / 4;
  q4_tile_mma_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)qw, (uint32_t*)qw_tiled, N, K);
  B2L_LAUNCH_CHECK("q4_tile_mma_kernel");
  return 0;
}

extern "C" int b2l_q4_untile_mma(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_q4_untile_mma: bad argument");
  B2L_CHECK_SUPPORTED(K % KB == 0, "b2l_q4_untile_mma: in_features %d must be a multiple of %d", K, KB);
  const size_t total = (size_t)(K / 2) * N;
  q4_untile_mma_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint32_t*)qw_tiled, (uint8_t*)qw, N, K);
  B2L_LAUNCH_CHECK("q4_untile_mma_kernel");
  return 0;
}

extern "C" size_t b2l_q4_gemv_batch_workspace_bytes(int K) {
  if (K <= 0 || K % KB) return 0;
  return (size_t)(K / KB) * XKB_BYTES + MAXB * 3 * sizeof(float);
}

namespace b2l {
// b2l_q4_gemv_batch's argument checks: 0, or B2L_E_* with a message
int check_q4_gemv_batch(const b2l_q4_linear_args* a) {
  B2L_CHECK_ARG(a != nullptr, "b2l_q4_gemv_batch: null args");
  B2L_CHECK_ARG(a->x && a->qw_tiled && a->scales && a->zeros && a->y && a->workspace, "b2l_q4_gemv_batch: null pointer");
  B2L_CHECK_SUPPORTED(a->out_affine.scale == nullptr && a->out_affine.bias == nullptr,
                      "b2l_q4_gemv_batch: out_affine is not supported (apply b2l_linear_affine to y)");
  B2L_CHECK_SUPPORTED(a->M >= 1 && a->M <= MAXB, "b2l_q4_gemv_batch: M=%d (1..%d activation rows)", a->M, MAXB);
  B2L_CHECK_SUPPORTED(a->K > 0 && a->K % KB == 0 && a->K <= 12 * 256 * 8, "b2l_q4_gemv_batch: K=%d must be a multiple of %d and <= %d", a->K, KB,
                      12 * 256 * 8);
  B2L_CHECK_ARG(a->N > 0 && a->ldx >= a->K && a->ldx % 8 == 0, "b2l_q4_gemv_batch: bad N / ldx (ldx %% 8 == 0)");
  B2L_CHECK_ARG(((uintptr_t)a->x % 16 == 0) && ((uintptr_t)a->qw_tiled % 16 == 0) && ((uintptr_t)a->workspace % 16 == 0),
                "b2l_q4_gemv_batch: x / qw_tiled / workspace must be 16-byte aligned");
  B2L_CHECK_ARG(a->sz_dtype == B2L_BF16 || a->sz_dtype == B2L_F32, "b2l_q4_gemv_batch: bad sz_dtype");
  if (a->prologue == B2L_PRO_RMSNORM)
    B2L_CHECK_ARG(a->norm_scale && ((uintptr_t)a->norm_scale % 16 == 0), "b2l_q4_gemv_batch: RMSNorm prologue needs a 16-byte aligned scale");
  else
    B2L_CHECK_ARG(a->prologue == B2L_PRO_NONE, "b2l_q4_gemv_batch: bad prologue %d", a->prologue);
  if (a->epilogue == B2L_EPI_RESIDUAL) B2L_CHECK_ARG(a->res != nullptr, "b2l_q4_gemv_batch: RESIDUAL epilogue needs res");
  else if (a->epilogue == B2L_EPI_SWIGLU) B2L_CHECK_SUPPORTED(a->N % RB == 0, "b2l_q4_gemv_batch: SWIGLU needs N %% 16 == 0");
  else B2L_CHECK_ARG(a->epilogue == B2L_EPI_STORE, "b2l_q4_gemv_batch: bad epilogue %d", a->epilogue);
  return 0;
}
}  // namespace b2l

extern "C" int b2l_q4_gemv_batch(const b2l_q4_linear_args* a, b2l_stream_t stream) {
  if (int rc = check_q4_gemv_batch(a)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  // programmatic dependent launch for the two kernels (B2L_BATCH_PDL=0: plain stream order)
  static const int env_pdl = [] { const char* e = getenv("B2L_BATCH_PDL"); return e ? atoi(e) : 1; }();
  const bool pdl = (a->flags & B2L_F_PDL) != 0 && env_pdl != 0;

  uint8_t* ws = (uint8_t*)a->workspace;
  float* sums = (float*)(ws + (size_t)(a->K / KB) * XKB_BYTES);
  {
    LaunchCfg lc(dim3(MAXB), dim3(256), 0, st, pdl, 1);
    const __nv_bfloat16* ns = a->prologue == B2L_PRO_RMSNORM ? (const __nv_bfloat16*)a->norm_scale : nullptr;
    if (a->K > 6 * 256 * 8)
      B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q4_batch_prep_kernel<12>, (const __nv_bfloat16*)a->x, a->ldx, a->M, a->K, ns, a->eps, (uint32_t*)ws, sums));
    else
      B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q4_batch_prep_kernel<6>, (const __nv_bfloat16*)a->x, a->ldx, a->M, a->K, ns, a->eps, (uint32_t*)ws, sums));
  }

  BParams p;
  p.qwt = (const uint8_t*)a->qw_tiled;
  p.scales = a->scales; p.zeros = a->zeros; p.szdt = a->sz_dtype;
  p.xfrag = ws; p.sums = sums;
  p.y = (__nv_bfloat16*)a->y; p.ldy = a->ldy;
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.n_rb = (a->N + RB - 1) / RB;
  p.epilogue = a->epilogue; p.res = (const __nv_bfloat16*)a->res; p.ldres = a->ldres;
  p.nst = BMAX_STAGES;
  const BSmem L = bsmem_layout(p.nst);
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(q4_gemv_batch_kernel, L.total, smem_cache)) return rc;
  int grid = a->split_k > 0 ? a->split_k : 2 * sm_count();   // split_k doubles as a grid override
  if (grid > p.n_rb) grid = p.n_rb;
  LaunchCfg lc(dim3(grid), dim3(NTHREADS), L.total, st, pdl, 1);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q4_gemv_batch_kernel, p));
  return 0;
}

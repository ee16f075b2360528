// One persistent kernel per decoded token (batch 1, gptq.int4 per-row scales, head_size 128).
//
// Replaces, for T == 1 with a KV cache, the whole of LLaMA.forward (lit_llama/model.py:76-122): wte lookup, per
// Block [rms_1 + c_attn] -> rope / KV append / attention -> [c_proj + residual] -> [rms_2 + c_fc1|c_fc2 + SwiGLU]
// -> [mlp.c_proj + residual] (model.py:156-168, 171-237, 240-254), ln_f + lm_head; and the roll branch of
// model.py:214-218 as a ring offset.  The per-op kernels of api.cu remain the path for every other shape.
//
// Why one kernel (measured, DESIGN.md section 4): a 2 x 110 KB-per-SM streaming kernel cannot be co-resident with
// its successor, so programmatic dependent launch only overlaps kernel TAILS and every one of the 161 launches of a
// token pays its own ring-fill latency (~2 us of idle HBM per launch at 7B).  Here one CTA per SM stays resident for
// the whole token:
//   * the producer warp of each CTA walks the token's static op list and streams that CTA's share of EVERY op's
//     weights (and K/V rows) through one mbarrier ring with TMA bulk copies.  Weights never depend on activations,
//     so it only ever waits for a free ring slot: HBM keeps streaming through every dependency wait;
//   * a dependency is a global arrival counter per op (red.release.gpu by each CTA when its rows are stored,
//     ld.acquire.gpu polling by one thread per CTA) instead of a kernel boundary;
//   * the contraction is the exact int8-digit MMA of q4_gemv.cu (IMMA.16832.U8.S8), fast enough (10-12 issue cycles
//     per 512 levels) that consumers drain the ring several times faster than HBM fills it after each wait;
//   * attention is a work item (head, 128-key split) of the same CTAs: old K/V rows arrive through the ring as 64-row
//     stages (prefetched ahead like weights), the new token's row is rotated, appended and scored from registers,
//     splits are merged by the last CTA of a head (acq_rel ticket), exactly like attn_decode_fused_kernel.
// Every CTA arrives exactly once on every op's counter, so "counter == grid" means the op's outputs are complete.
// All waits are bounded: a timeout sets a sticky error word and lets every loop fall through (no hang).
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "q4_mma_common.cuh"

namespace b2l {
namespace mega {
using namespace q4mv;

enum { OP_GEMV = 0, OP_ATTN = 1 };

struct Op {
  int kind;
  int N, K, n_rb;
  int prologue, epilogue;
  int rot;                 // rotation of the CTA -> row-range assignment (spreads the uneven split over different CTAs)
  int x_is_emb, res_is_emb;
  const uint8_t* qwt; const void* scales; const void* zeros;
  const __nv_bfloat16* x; __nv_bfloat16* y; const __nv_bfloat16* res; const __nv_bfloat16* norm_scale;
  __nv_bfloat16* k_cache; __nv_bfloat16* v_cache;
};

struct Params {
  const Op* ops; int n_ops;
  unsigned int* counters;   // [n_ops] arrivals per op; zero before the step, re-armed by the last CTA of the step
  unsigned int* error;      // sticky: 0 = ok
  const void* idx; int idx_is_i64; const __nv_bfloat16* wte; int vocab;
  const int64_t* input_pos; int32_t* ring_start;
  const float* rope; int block_size;
  int C, n_head, S;
  const __nv_bfloat16* qkv; __nv_bfloat16* att; float* attn_work; int* tickets; int n_split;
  float eps; int szdt;
  int nst, kmax;
  unsigned long long* tl;   // debug timeline [n_ops][16] (nullptr = off)
};

// One CTA per SM: 16 consumer warps + producer warp + epilogue warp.  (Two 10-warp CTAs per SM, the per-op kernels'
// shape, were measured first: both CTAs of an SM ran the same activation prologue -- ~150 instructions per 8
// elements, 1.6 us for K = 11008 -- and kept two copies of the digit planes: tools/diag.py mega_timeline.)
constexpr int MW = 16;                     // consumer warps
constexpr int MT = MW * 32;                // consumer threads
constexpr int M_PRODUCER = MW;             // warp 16
constexpr int M_THREADS = (MW + 2) * 32;   // 576
constexpr int M_MAX_STAGES = 12;
constexpr int HS = 128;                    // head size
constexpr int KV_ROWS = STAGE_BYTES / (HS * 2);   // 64 K (or V) rows per ring stage
constexpr int ATT_CHUNK = 128;             // keys per attention work item
constexpr long long SPIN_TIMEOUT_NS = 400LL * 1000 * 1000;

__host__ __device__ inline uint32_t plane_stride(int K) { return (uint32_t)K + ((K % 128 == 0) ? 64u : 0u); }

struct SmemLayout {
  uint32_t ring, xf, zero, scratch, red, bars, total;
};
__host__ __device__ inline SmemLayout smem_layout(int nst, int kmax, int ndig) {
  SmemLayout L;
  uint32_t o = 0;
  L.ring = o;    o += (uint32_t)nst * STAGE_BYTES;
  L.xf = o;      o += (uint32_t)ndig * plane_stride(kmax);
  L.zero = o;    o += 16;
  L.scratch = o; o += 2 * MW * MAX_HALVES * RB * 16;    // 16 KB: GEMV partials; attention: per-warp accumulators (8 KB + 128 B)
  L.red = o;     o += 320;                              // float[16] sumsq, float[16] max, int64[16] sum X, int sh, int last
  L.bars = o;    o += 2 * M_MAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

__device__ __forceinline__ uint32_t balanced_digits(int X) { return ((uint32_t)X + 0x00808080u) ^ 0x00808080u; }

// loads of data produced earlier in this launch by other CTAs: L2 (never a stale L1 line)
__device__ __forceinline__ uint4 ld_cg_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_cg_bf16(const __nv_bfloat16* p) {
  unsigned short v;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return __uint_as_float((uint32_t)v << 16);
}
__device__ __forceinline__ unsigned int ld_acquire(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release(unsigned int* p) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}

// bounded waits
__device__ __forceinline__ void flag_wait(const unsigned int* ctr, unsigned int target, unsigned int* err) {
  if (ld_acquire(ctr) >= target) return;
  const unsigned long long t0 = globaltimer_ns();
  for (;;) {
#pragma unroll 1
    for (int i = 0; i < 256; ++i)
      if (ld_acquire(ctr) >= target) return;
    if (*reinterpret_cast<volatile unsigned int*>(err) != 0u) return;
    if ((long long)(globaltimer_ns() - t0) > SPIN_TIMEOUT_NS) { atomicCAS(err, 0u, 1u); return; }
  }
}
__device__ __forceinline__ void mbar_wait_b(uint32_t a, uint32_t parity, unsigned int* err) {
  uint32_t ok;
  for (int i = 0; i < (1 << 22); ++i) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(a), "r"(parity)
        : "memory");
    if (ok) return;
  }
  atomicCAS(err, 0u, 2u);
}

// row-block range of this CTA for an op
__device__ __forceinline__ void op_range(const Op& op, int& rb_lo, int& rb_hi) {
  const int G = gridDim.x;
  int c = (int)blockIdx.x + op.rot;
  c -= (c >= G) ? G : 0;
  rb_lo = (int)(((long long)c * op.n_rb) / G);
  rb_hi = (int)(((long long)(c + 1) * op.n_rb) / G);
}
__device__ __forceinline__ int cta_eff(const Op& op) {
  int c = (int)blockIdx.x + op.rot;
  return c - ((c >= (int)gridDim.x) ? (int)gridDim.x : 0);
}

// IMMA on one 512-byte tile (16 rows x 64 k): two k32 chunks
__device__ __forceinline__ void tile_imma(int (&a0)[4], int (&a1)[4], const uint8_t* tile, const uint4& xb) {
  const uint4 wv = *reinterpret_cast<const uint4*>(tile);
  mma_u8s8_16832(a0, wv.x, wv.x & 0xf0f0f0f0u, wv.y, wv.y & 0xf0f0f0f0u, xb.x, xb.y);
  mma_u8s8_16832(a1, wv.z, wv.z & 0xf0f0f0f0u, wv.w, wv.w & 0xf0f0f0f0u, xb.z, xb.w);
}

__device__ __forceinline__ void bf16x8_to_f32(const uint4& u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

template <int MAXC, int NDIG>
__global__ void __launch_bounds__(M_THREADS, 1) decode_mega_kernel(const Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const SmemLayout L = smem_layout(p.nst, p.kmax, NDIG);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = gridDim.x;
  const uint32_t bar_full = sbase + L.bars, bar_empty = bar_full + M_MAX_STAGES * 8;
  const uint32_t PS = plane_stride(p.kmax);

  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) {
      mbar_init(bar_full + i * 8, 1);
      mbar_init(bar_empty + i * 8, MW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < 4) reinterpret_cast<uint32_t*>(smem + L.zero)[tid] = 0u;
  __syncthreads();

  // ---- inputs of the step (written by the host side before the launch)
  const long long pos = p.input_pos[0];
  const int S = p.S;
  const int w_slot = (int)(pos < S ? pos : (long long)S - 1);   // logical slot of the new token (model.py:211-218)
  const int Lk = w_slot + 1;                                     // valid logical slots 0 .. Lk-1
  const int n_active = (Lk + ATT_CHUNK - 1) / ATT_CHUNK;
  const int ring_old = *p.ring_start;
  const int ring = (pos >= (long long)S) ? (ring_old + 1) % S : ring_old;   // the roll branch as a ring advance
  long long tok = p.idx_is_i64 ? reinterpret_cast<const long long*>(p.idx)[0] : (long long)reinterpret_cast<const int*>(p.idx)[0];
  tok = tok < 0 ? 0 : (tok >= p.vocab ? p.vocab - 1 : tok);
  const __nv_bfloat16* emb = p.wte + (size_t)tok * p.C;          // transformer.wte(idx), model.py:102
  const int n_items = n_active * p.n_head;                       // attention work items of a layer

  if (warp == M_PRODUCER) {
    // ===================== producer: every op's bytes for this CTA, in op order, through one ring =====================
    if (lane == 0) {
      int slot = 0;
      uint32_t phase = 1;  // fresh barriers: waiting on parity 1 passes immediately
      const bool pdbg = (p.tl != nullptr && blockIdx.x == 0);
      for (int oi = 0; oi < p.n_ops; ++oi) {
        const Op& op = p.ops[oi];
        long long pw = 0;
        if (op.kind == OP_GEMV) {
          int rb_lo, rb_hi;
          op_range(op, rb_lo, rb_hi);
          const int n_kb = op.K / KB;
          for (int rb = rb_lo; rb < rb_hi; rb += 2) {
            const int halves = min(2, rb_hi - rb);
            const int per_stage = halves == 2 ? KBP_PER_STAGE : 2 * KBP_PER_STAGE;   // k-block positions per stage
            const uint8_t* src = op.qwt + (size_t)rb * n_kb * KB_BYTES;
            for (int kb0 = 0; kb0 < n_kb; kb0 += per_stage) {
              const int nkb = min(per_stage, n_kb - kb0);
              const uint32_t bytes = (uint32_t)nkb * KB_BYTES;
              const long long c0 = pdbg ? clock64() : 0;
              mbar_wait_b(bar_empty + slot * 8, phase, p.error);
              if (pdbg) pw += clock64() - c0;
              mbar_expect_tx(bar_full + slot * 8, bytes * halves);
              for (int h = 0; h < halves; ++h)
                tma_bulk_g2s(sbase + L.ring + slot * STAGE_BYTES + h * HALF_STAGE_BYTES,
                             src + ((size_t)h * n_kb + kb0) * KB_BYTES, bytes, bar_full + slot * 8);
              if (++slot == p.nst) { slot = 0; phase ^= 1; }
            }
          }
        } else {
          // attention: old K/V rows of this CTA's items, 64 rows per stage, K stage then V stage
          for (int w = cta_eff(op); w < n_items; w += G) {
            const int sp = w / p.n_head, h = w - sp * p.n_head;
            const int j0 = sp * ATT_CHUNK, j1 = min(Lk, j0 + ATT_CHUNK);
            const int n_old = min(j1, Lk - 1) - j0;
            const size_t head_base = (size_t)h * S * HS;
            for (int sub = 0; sub * KV_ROWS < n_old; ++sub) {
              const int cnt = min(KV_ROWS, n_old - sub * KV_ROWS);
              int phys0 = j0 + sub * KV_ROWS + ring; if (phys0 >= S) phys0 -= S;
              const int first = min(cnt, S - phys0);
#pragma unroll 1
              for (int kv = 0; kv < 2; ++kv) {
                const __nv_bfloat16* base = (kv == 0 ? op.k_cache : op.v_cache) + head_base;
                mbar_wait_b(bar_empty + slot * 8, phase, p.error);
                mbar_expect_tx(bar_full + slot * 8, (uint32_t)cnt * HS * 2);
                const uint32_t dst = sbase + L.ring + slot * STAGE_BYTES;
                tma_bulk_g2s(dst, base + (size_t)phys0 * HS, (uint32_t)first * HS * 2, bar_full + slot * 8);
                if (first < cnt) tma_bulk_g2s(dst + first * HS * 2, base, (uint32_t)(cnt - first) * HS * 2, bar_full + slot * 8);
                if (++slot == p.nst) { slot = 0; phase ^= 1; }
              }
            }
          }
        }
        if (pdbg) { p.tl[oi * 16 + 7] = (unsigned long long)pw; }
      }
    }
  } else if (warp < MW) {
    // ===================== consumer warps =====================
    constexpr int NT = MT;   // 512
    float* red = reinterpret_cast<float*>(smem + L.red);
    long long* red_sx = reinterpret_cast<long long*>(smem + L.red + 128);
    int* red_sh = reinterpret_cast<int*>(smem + L.red + 256);
    int* red_last = reinterpret_cast<int*>(smem + L.red + 260);
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    const int ncol = lane >> 2, t4 = lane & 3;
    const uint8_t* xf_lane = (ncol < NDIG) ? smem + L.xf + ncol * PS + t4 * 16 : smem + L.zero;
    const int xf_step = (ncol < NDIG) ? 64 : 0;
    int slot = 0;
    uint32_t phase = 0;

    for (int oi = 0; oi < p.n_ops; ++oi) {
      const Op& op = p.ops[oi];
      const bool dbg = (p.tl != nullptr && tid == 0);
      if (op.kind == OP_GEMV) {
        const bool norm = (op.prologue == B2L_PRO_RMSNORM);
        const int K = op.K;
        uint4 xv[MAXC], gv[MAXC];
        // the RMSNorm scale is a weight: fetch it before waiting for the producing op
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
          const int k = (c * NT + tid) * 8;
          gv[c] = make_uint4(0, 0, 0, 0);
          if (norm && k < K) gv[c] = *reinterpret_cast<const uint4*>(op.norm_scale + k);
        }
        // ---- dependency: the previous op is complete on every CTA
        if (oi > 0) {
          if (tid == 0) flag_wait(p.counters + oi - 1, (unsigned int)G, p.error);
          named_bar_sync(2, NT);
        }
        if (dbg) { atomicMin(p.tl + oi * 16 + 5, globaltimer_ns()); if (blockIdx.x == 0) p.tl[oi * 16 + 0] = globaltimer_ns(); }
        const __nv_bfloat16* xin = op.x_is_emb ? emb : op.x;
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
          const int k = (c * NT + tid) * 8;
          xv[c] = make_uint4(0, 0, 0, 0);
          if (k < K) xv[c] = ld_cg_u4(xin + k);
        }
        const int nchunk = (K + NT * 8 - 1) / (NT * 8);
        float ss = 0.f, mx = 0.f;
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
          if (c < nchunk) {
            const uint32_t w[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w};
            const uint32_t g[4] = {gv[c].x, gv[c].y, gv[c].z, gv[c].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float lo = __uint_as_float(w[q] << 16), hi = __uint_as_float(w[q] & 0xffff0000u);
              if (norm) {
                const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
                const __nv_bfloat162 sq = __hmul2(v, v);
                const uint32_t su = *reinterpret_cast<const uint32_t*>(&sq);
                ss += __uint_as_float(su << 16) + __uint_as_float(su & 0xffff0000u);
                const float glo = __uint_as_float(g[q] << 16), ghi = __uint_as_float(g[q] & 0xffff0000u);
                mx = fmaxf(mx, fmaxf(fabsf(lo * glo), fabsf(hi * ghi)));
              } else {
                mx = fmaxf(mx, fmaxf(fabsf(lo), fabsf(hi)));
              }
            }
          }
        }
        ss = warp_sum(ss);
        mx = warp_max(mx);
        if (lane == 0) { red[warp] = ss; red[MW + warp] = mx; }
        named_bar_sync(1, NT);
        ss = 0.f; mx = 0.f;
#pragma unroll
        for (int w = 0; w < MW; ++w) { ss += red[w]; mx = fmaxf(mx, red[MW + w]); }
        float rinv = 1.f;
        if (norm) {
          rinv = rms_rinv(ss, K, p.eps);
          mx = mx * rinv * 1.01f;
        }
        const int e = (int)((__float_as_uint(mx) >> 23) & 0xffu) - 127;
        int sh = (8 * NDIG - 3) - e;
        sh = max(-126, min(126, sh));
        const float scale = __uint_as_float((uint32_t)(sh + 127) << 23);
        const __nv_bfloat162 rinv2 = __float2bfloat162_rn(rinv);
        long long sx = 0;
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
          const int k = (c * NT + tid) * 8;
          if (c < nchunk && k < K) {
            uint32_t w[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w};
            if (norm) {
              const uint32_t g[4] = {gv[c].x, gv[c].y, gv[c].z, gv[c].w};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
                const __nv_bfloat162 gg = *reinterpret_cast<const __nv_bfloat162*>(&g[q]);
                const __nv_bfloat162 y2 = __hmul2(gg, __hmul2(v, rinv2));   // model.py:276-277
                w[q] = *reinterpret_cast<const uint32_t*>(&y2);
              }
            }
            uint32_t xd[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int X0 = __float2int_rn(__uint_as_float(w[q] << 16) * scale);
              const int X1 = __float2int_rn(__uint_as_float(w[q] & 0xffff0000u) * scale);
              sx += (long long)X0 + (long long)X1;
              xd[2 * q] = balanced_digits(X0);
              xd[2 * q + 1] = balanced_digits(X1);
            }
            uint32_t dj[2][4];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const uint32_t lo01 = __byte_perm(xd[4 * j], xd[4 * j + 1], 0x5140), hi01 = __byte_perm(xd[4 * j], xd[4 * j + 1], 0x7362);
              const uint32_t lo23 = __byte_perm(xd[4 * j + 2], xd[4 * j + 3], 0x5140), hi23 = __byte_perm(xd[4 * j + 2], xd[4 * j + 3], 0x7362);
              dj[j][0] = __byte_perm(lo01, lo23, 0x5410);
              dj[j][1] = __byte_perm(lo01, lo23, 0x7632);
              dj[j][2] = __byte_perm(hi01, hi23, 0x5410);
              dj[j][3] = __byte_perm(hi01, hi23, 0x7632);
            }
            uint8_t* dst = smem + L.xf + (k >> 6) * 64 + ((k >> 3) & 3) * 16 + ((k >> 5) & 1) * 8;
#pragma unroll
            for (int n = 0; n < NDIG; ++n) *reinterpret_cast<uint2*>(dst + n * PS) = make_uint2(dj[0][n], dj[1][n]);
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o);
        if (lane == 0) red_sx[warp] = sx;
        if (tid == 0) *red_sh = sh;
        named_bar_sync(3, NT + 32);   // digit planes, sum X and sh are ready (releases the epilogue warp too)
        if (dbg && blockIdx.x == 0) p.tl[oi * 16 + 1] = globaltimer_ns();

        // ---- weights: stage -> registers -> IMMA.  A stage holds 32 tiles of 512 B; warp w takes tiles w and w + 16.
        int rb_lo, rb_hi;
        op_range(op, rb_lo, rb_hi);
        const int n_kb = K / KB;
        int u = 0;
        long long cw = 0, bw = 0;
        const long long l0 = clock64();
        for (int rb = rb_lo; rb < rb_hi; rb += 2, ++u) {
          const int halves = min(2, rb_hi - rb);
          int acc[MAX_HALVES][2][4];
#pragma unroll
          for (int h = 0; h < MAX_HALVES; ++h)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
              for (int i = 0; i < 4; ++i) acc[h][c][i] = 0;
          const int per_stage = halves == 2 ? KBP_PER_STAGE : 2 * KBP_PER_STAGE;
          const int n_st = (n_kb + per_stage - 1) / per_stage;
          const int posB = halves == 2 ? warp : warp + MW;   // k-block position (inside a stage) of this warp's second tile
          // Two stages per round: both full-barrier waits, then 8 shared-memory loads, then 8 IMMAs, then both releases.
          // (One stage per round left each warp 4 IMMAs behind a ~250-cycle wait/load/arrive chain: measured 590
          // cycles per 16 KB stage per SM, barely above the HBM rate: tools/diag.py mega_timeline.)
          // A warp's tiles sit at the same addresses for one- and two-half units: tile w and tile 16 + w of the stage.
          for (int s0 = 0; s0 < n_st; s0 += 2) {
            const bool two = s0 + 1 < n_st;
            const int slot_a = slot;
            const uint32_t phase_a = phase;
            if (++slot == p.nst) { slot = 0; phase ^= 1; }
            const int slot_b = slot;
            const uint32_t phase_b = phase;
            if (two) { if (++slot == p.nst) { slot = 0; phase ^= 1; } }
            const long long c0 = (dbg && blockIdx.x == 0) ? clock64() : 0;
            mbar_wait_b(bar_full + slot_a * 8, phase_a, p.error);
            if (two) mbar_wait_b(bar_full + slot_b * 8, phase_b, p.error);
            if (dbg && blockIdx.x == 0) cw += clock64() - c0;
            const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
            const int kb_a = s0 * per_stage, kb_b = kb_a + per_stage;
            const int nkb_a = min(per_stage, n_kb - kb_a), nkb_b = two ? min(per_stage, n_kb - kb_b) : 0;
            const uint8_t* sta = smem + L.ring + slot_a * STAGE_BYTES + warp * KB_BYTES + lane * 16;
            const uint8_t* stb = smem + L.ring + slot_b * STAGE_BYTES + warp * KB_BYTES + lane * 16;
            const uint4 wa0 = *reinterpret_cast<const uint4*>(sta), wa1 = *reinterpret_cast<const uint4*>(sta + HALF_STAGE_BYTES);
            const uint4 xa0 = warp < nkb_a ? *reinterpret_cast<const uint4*>(xf_lane + (kb_a + warp) * xf_step) : zero4;
            const uint4 xa1 = posB < nkb_a ? *reinterpret_cast<const uint4*>(xf_lane + (kb_a + posB) * xf_step) : zero4;
            uint4 wb0 = zero4, wb1 = zero4, xb0 = zero4, xb1 = zero4;
            if (two) {
              wb0 = *reinterpret_cast<const uint4*>(stb); wb1 = *reinterpret_cast<const uint4*>(stb + HALF_STAGE_BYTES);
              if (warp < nkb_b) xb0 = *reinterpret_cast<const uint4*>(xf_lane + (kb_b + warp) * xf_step);
              if (posB < nkb_b) xb1 = *reinterpret_cast<const uint4*>(xf_lane + (kb_b + posB) * xf_step);
            }
            // a tile whose k-block position lies beyond the stage multiplies stale bytes by zero digits
            mma_u8s8_16832(acc[0][0], wa0.x, wa0.x & 0xf0f0f0f0u, wa0.y, wa0.y & 0xf0f0f0f0u, xa0.x, xa0.y);
            mma_u8s8_16832(acc[0][1], wa0.z, wa0.z & 0xf0f0f0f0u, wa0.w, wa0.w & 0xf0f0f0f0u, xa0.z, xa0.w);
            mma_u8s8_16832(acc[1][0], wa1.x, wa1.x & 0xf0f0f0f0u, wa1.y, wa1.y & 0xf0f0f0f0u, xa1.x, xa1.y);
            mma_u8s8_16832(acc[1][1], wa1.z, wa1.z & 0xf0f0f0f0u, wa1.w, wa1.w & 0xf0f0f0f0u, xa1.z, xa1.w);
            mma_u8s8_16832(acc[0][0], wb0.x, wb0.x & 0xf0f0f0f0u, wb0.y, wb0.y & 0xf0f0f0f0u, xb0.x, xb0.y);
            mma_u8s8_16832(acc[0][1], wb0.z, wb0.z & 0xf0f0f0f0u, wb0.w, wb0.w & 0xf0f0f0f0u, xb0.z, xb0.w);
            mma_u8s8_16832(acc[1][0], wb1.x, wb1.x & 0xf0f0f0f0u, wb1.y, wb1.y & 0xf0f0f0f0u, xb1.x, xb1.y);
            mma_u8s8_16832(acc[1][1], wb1.z, wb1.z & 0xf0f0f0f0u, wb1.w, wb1.w & 0xf0f0f0f0u, xb1.z, xb1.w);
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(bar_empty + slot_a * 8);
              if (two) mbar_arrive(bar_empty + slot_b * 8);
            }
          }
          // lane (g, t): rows g (c0, c1) and g + 8 (c2, c3), digits 2t, 2t + 1.  row g = D[g] - D[g+8], row g+8 = D[g+8] / 16
          const int buf = u & 1;
          const long long b0 = (dbg && blockIdx.x == 0) ? clock64() : 0;
          named_bar_sync(4 + buf, NT + 32);   // the epilogue warp has drained this scratch buffer
          if (dbg && blockIdx.x == 0) bw += clock64() - b0;
          if (t4 < 2) {
            if (halves == 2) {
#pragma unroll
              for (int h = 0; h < MAX_HALVES; ++h) {
                const int c0 = acc[h][0][0] + acc[h][1][0], c1 = acc[h][0][1] + acc[h][1][1];
                const int c2 = acc[h][0][2] + acc[h][1][2], c3 = acc[h][0][3] + acc[h][1][3];
                int* dst = scratch + (((buf * MW + warp) * MAX_HALVES + h) * RB + (lane >> 2)) * 4 + 2 * t4;
                *reinterpret_cast<int2*>(dst) = make_int2(c0 - c2, c1 - c3);
                *reinterpret_cast<int2*>(dst + 8 * 4) = make_int2(c2 >> 4, c3 >> 4);
              }
            } else {
              const int c0 = acc[0][0][0] + acc[0][1][0] + acc[1][0][0] + acc[1][1][0];
              const int c1 = acc[0][0][1] + acc[0][1][1] + acc[1][0][1] + acc[1][1][1];
              const int c2 = acc[0][0][2] + acc[0][1][2] + acc[1][0][2] + acc[1][1][2];
              const int c3 = acc[0][0][3] + acc[0][1][3] + acc[1][0][3] + acc[1][1][3];
              int* dst = scratch + (((buf * MW + warp) * MAX_HALVES + 0) * RB + (lane >> 2)) * 4 + 2 * t4;
              *reinterpret_cast<int2*>(dst) = make_int2(c0 - c2, c1 - c3);
              *reinterpret_cast<int2*>(dst + 8 * 4) = make_int2(c2 >> 4, c3 >> 4);
            }
          }
          __syncwarp();
          named_bar_arrive(6 + buf, NT + 32);
        }
        if (dbg) { atomicMax(p.tl + oi * 16 + 3, globaltimer_ns()); if (blockIdx.x == 0) { p.tl[oi * 16 + 2] = globaltimer_ns(); p.tl[oi * 16 + 6] = (unsigned long long)cw; p.tl[oi * 16 + 8] = (unsigned long long)bw; p.tl[oi * 16 + 9] = (unsigned long long)(clock64() - l0); p.tl[oi * 16 + 12] = (unsigned long long)u; } }
      } else {
        // ===================== attention work items =====================
        if (oi > 0) {
          if (tid == 0) flag_wait(p.counters + oi - 1, (unsigned int)G, p.error);
          named_bar_sync(2, NT);
        }
        if (dbg) { atomicMin(p.tl + oi * 16 + 5, globaltimer_ns()); if (blockIdx.x == 0) p.tl[oi * 16 + 0] = globaltimer_ns(); }
        float* sm_acc = reinterpret_cast<float*>(smem + L.scratch);     // [MW][HS]
        float* sm_m = sm_acc + MW * HS;                                 // [MW]
        float* sm_l = sm_m + MW;                                        // [MW]
        const int grp = lane >> 3, sub8 = lane & 7, d0 = sub8 * 16;
        const int C = p.C;
        for (int w = cta_eff(op); w < n_items; w += G) {
          const int sp = w / p.n_head, h = w - sp * p.n_head;
          const int j0 = sp * ATT_CHUNK, j1 = min(Lk, j0 + ATT_CHUNK);
          const int n_old = min(j1, Lk - 1) - j0;
          const bool has_new = (w_slot >= j0 && w_slot < j1);
          const size_t head_base = (size_t)h * S * HS;
          // rope row of this position (constant table) and q of this head, rotated (model.py:306-323) and scaled
          const long long prow = pos < p.block_size ? pos : (long long)p.block_size - 1;
          float cs[16];
          {
            const float4* rp = reinterpret_cast<const float4*>(p.rope + ((size_t)prow * (HS / 2) + d0 / 2) * 2);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float4 t = rp[i];
              cs[4 * i] = t.x; cs[4 * i + 1] = t.y; cs[4 * i + 2] = t.z; cs[4 * i + 3] = t.w;
            }
          }
          const __nv_bfloat16* qrow = p.qkv + h * HS + d0;
          float q[16];
          {
            float raw[16];
            bf16x8_to_f32(ld_cg_u4(qrow), raw);
            bf16x8_to_f32(ld_cg_u4(qrow + 8), raw + 8);
            const float scale = rsqrtf((float)HS);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float c = cs[2 * i], s_ = cs[2 * i + 1];
              const float e = rbf(__fsub_rn(__fmul_rn(raw[2 * i], c), __fmul_rn(raw[2 * i + 1], s_)));
              const float o = rbf(__fadd_rn(__fmul_rn(raw[2 * i + 1], c), __fmul_rn(raw[2 * i], s_)));
              q[2 * i] = e * scale;
              q[2 * i + 1] = o * scale;
            }
          }
          float m = -INFINITY, l = 0.f, acc[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) acc[i] = 0.f;
          // old rows: (K stage, V stage) pairs of up to 64 rows; warp w handles rows 4 w .. 4 w + 3 (8 lanes per key)
          for (int sub = 0; sub * KV_ROWS < n_old; ++sub) {
            const int cnt = min(KV_ROWS, n_old - sub * KV_ROWS);
            const int slot_k = slot;
            const uint32_t phase_k = phase;
            if (++slot == p.nst) { slot = 0; phase ^= 1; }
            const int slot_v = slot;
            const uint32_t phase_v = phase;
            if (++slot == p.nst) { slot = 0; phase ^= 1; }
            mbar_wait_b(bar_full + slot_k * 8, phase_k, p.error);
            const uint8_t* kst = smem + L.ring + slot_k * STAGE_BYTES;
            const uint8_t* vst = smem + L.ring + slot_v * STAGE_BYTES;
            const int r = warp * 4 + grp;
            float sc;
            {
              const int rc = r < cnt ? r : 0;
              const uint4* kr = reinterpret_cast<const uint4*>(kst + (size_t)rc * HS * 2 + d0 * 2);
              float kf[16];
              bf16x8_to_f32(kr[0], kf); bf16x8_to_f32(kr[1], kf + 8);
              float s_ = 0.f;
#pragma unroll
              for (int i = 0; i < 16; ++i) s_ = fmaf(q[i], kf[i], s_);
              s_ += __shfl_xor_sync(0xffffffffu, s_, 1);
              s_ += __shfl_xor_sync(0xffffffffu, s_, 2);
              s_ += __shfl_xor_sync(0xffffffffu, s_, 4);
              sc = s_;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + slot_k * 8);
            mbar_wait_b(bar_full + slot_v * 8, phase_v, p.error);
            if (r < cnt) {
              const uint4* vr = reinterpret_cast<const uint4*>(vst + (size_t)r * HS * 2 + d0 * 2);
              float vf[16];
              bf16x8_to_f32(vr[0], vf); bf16x8_to_f32(vr[1], vf + 8);
              const float mn = fmaxf(m, sc);
              const float corr = __expf(m - mn), pj = __expf(sc - mn);
              l = l * corr + pj;
#pragma unroll
              for (int i = 0; i < 16; ++i) acc[i] = fmaf(pj, vf[i], acc[i] * corr);
              m = mn;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + slot_v * 8);
          }
          // the new token's key/value: rotate k, append both to the cache, score from registers (warp 0, key group 0)
          if (has_new && warp == 0 && grp == 0) {
            int phys = w_slot + ring; if (phys >= S) phys -= S;
            float raw[16], kf[16], vf[16];
            bf16x8_to_f32(ld_cg_u4(qrow + C), raw);
            bf16x8_to_f32(ld_cg_u4(qrow + C + 8), raw + 8);
            uint32_t out[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float c = cs[2 * i], s_ = cs[2 * i + 1];
              kf[2 * i] = rbf(__fsub_rn(__fmul_rn(raw[2 * i], c), __fmul_rn(raw[2 * i + 1], s_)));
              kf[2 * i + 1] = rbf(__fadd_rn(__fmul_rn(raw[2 * i + 1], c), __fmul_rn(raw[2 * i], s_)));
              out[i] = (__float_as_uint(kf[2 * i]) >> 16) | (__float_as_uint(kf[2 * i + 1]) & 0xffff0000u);
            }
            const uint4 va = ld_cg_u4(qrow + 2 * C), vb = ld_cg_u4(qrow + 2 * C + 8);
            uint4* kd = reinterpret_cast<uint4*>(op.k_cache + head_base + (size_t)phys * HS + d0);
            uint4* vd = reinterpret_cast<uint4*>(op.v_cache + head_base + (size_t)phys * HS + d0);
            kd[0] = make_uint4(out[0], out[1], out[2], out[3]); kd[1] = make_uint4(out[4], out[5], out[6], out[7]);
            vd[0] = va; vd[1] = vb;
            bf16x8_to_f32(va, vf); bf16x8_to_f32(vb, vf + 8);
            float s_ = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) s_ = fmaf(q[i], kf[i], s_);
            s_ += __shfl_xor_sync(0x000000ffu, s_, 1);
            s_ += __shfl_xor_sync(0x000000ffu, s_, 2);
            s_ += __shfl_xor_sync(0x000000ffu, s_, 4);
            const float mn = fmaxf(m, s_);
            const float corr = __expf(m - mn), pj = __expf(s_ - mn);
            l = l * corr + pj;
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = fmaf(pj, vf[i], acc[i] * corr);
            m = mn;
          }
          __syncwarp();
          // merge the 4 key groups of the warp (lanes with the same sub8 hold the same dims)
#pragma unroll
          for (int off = 8; off <= 16; off <<= 1) {
            const float mo = __shfl_xor_sync(0xffffffffu, m, off);
            const float lo = __shfl_xor_sync(0xffffffffu, l, off);
            const float mn = fmaxf(m, mo);
            const float ca = (m == -INFINITY) ? 0.f : __expf(m - mn);
            const float cb = (mo == -INFINITY) ? 0.f : __expf(mo - mn);
            l = l * ca + lo * cb;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const float ao = __shfl_xor_sync(0xffffffffu, acc[i], off);
              acc[i] = acc[i] * ca + ao * cb;
            }
            m = mn;
          }
          if (lane == 0) { sm_m[warp] = m; sm_l[warp] = l; }
          if (grp == 0) {
#pragma unroll
            for (int i = 0; i < 16; ++i) sm_acc[warp * HS + d0 + i] = acc[i];
          }
          named_bar_sync(1, NT);
          float M = -INFINITY;
#pragma unroll
          for (int ww = 0; ww < MW; ++ww) M = fmaxf(M, sm_m[ww]);
          float Ls = 0.f, a = 0.f;
          const int d = tid & (HS - 1);
          const bool writer = tid < HS;
#pragma unroll
          for (int ww = 0; ww < MW; ++ww) {
            const float wg = (sm_m[ww] == -INFINITY) ? 0.f : __expf(sm_m[ww] - M);
            Ls += sm_l[ww] * wg;
            a += sm_acc[ww * HS + d] * wg;
          }
          if (n_active == 1) {
            if (writer) p.att[h * HS + d] = f2bf(a / Ls);
          } else {
            float* outp = p.attn_work + ((size_t)h * p.n_split + sp) * (HS + 2);
            if (tid == 0) { outp[0] = M; outp[1] = Ls; }
            if (writer) outp[2 + d] = a;
            named_bar_sync(1, NT);   // this CTA's partial is stored before the ticket (cumulative release below)
            if (tid == 0) {
              int t;
              asm volatile("atom.add.acq_rel.gpu.global.s32 %0, [%1], 1;" : "=r"(t) : "l"(p.tickets + h) : "memory");
              *red_last = (t == n_active - 1);
              if (t == n_active - 1) p.tickets[h] = 0;   // every contributor has arrived: re-arm for the next layer
            }
            named_bar_sync(1, NT);
            if (*red_last) {
              const float* base = p.attn_work + (size_t)h * p.n_split * (HS + 2);
              float MM = -INFINITY, LL = 0.f, aa = 0.f;
              for (int s0 = 0; s0 < n_active; s0 += 16) {
                float ms[16], ls[16], as[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                  const int s2 = s0 + i;
                  const bool ok = s2 < n_active;
                  const float* bp = base + (size_t)(ok ? s2 : s0) * (HS + 2);
                  ms[i] = ok ? __ldcg(bp) : -INFINITY;
                  ls[i] = ok ? __ldcg(bp + 1) : 0.f;
                  as[i] = ok ? __ldcg(bp + 2 + d) : 0.f;
                }
                float bm = MM;
#pragma unroll
                for (int i = 0; i < 16; ++i) bm = fmaxf(bm, ms[i]);
                const float c0 = (MM == -INFINITY) ? 0.f : __expf(MM - bm);
                LL *= c0; aa *= c0;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                  const float wg = (ms[i] == -INFINITY) ? 0.f : __expf(ms[i] - bm);
                  LL += ls[i] * wg;
                  aa += as[i] * wg;
                }
                MM = bm;
              }
              if (writer) p.att[h * HS + d] = f2bf(aa / LL);
            }
          }
          named_bar_sync(1, NT);   // sm_acc / red_last are reused by the next item; all stores of this item are issued
        }
        // every CTA arrives once per op: its items (and any merge it performed) are stored
        named_bar_sync(2, NT);
        if (tid == 0) {
          red_release(p.counters + oi);   // release: the barrier above orders every thread's stores before it
          if (dbg) { atomicMax(p.tl + oi * 16 + 4, globaltimer_ns()); }
        }
      }
    }
  } else {
    // ===================== epilogue warp: lane = row of the 32-row unit =====================
    const long long* red_sx = reinterpret_cast<const long long*>(smem + L.red + 128);
    const int* red_sh = reinterpret_cast<const int*>(smem + L.red + 256);
    const int* scratch = reinterpret_cast<const int*>(smem + L.scratch);
    constexpr int NB = MT + 32;
    const int half = lane >> 4, row = lane & 15;
    for (int oi = 0; oi < p.n_ops; ++oi) {
      const Op& op = p.ops[oi];
      if (op.kind != OP_GEMV) continue;
      int rb_lo, rb_hi;
      op_range(op, rb_lo, rb_hi);
      const int n_units = (rb_hi - rb_lo + 1) / 2;
      const __nv_bfloat16* resp = op.res_is_emb ? emb : op.res;
      // scale / zero / residual of a unit: weights, and a residual stream that was complete two ops ago -- fetched
      // BEFORE this op's dependency resolves (first unit) or while the consumers stream the unit (later ones)
      auto fetch = [&](int u, float& sc, float& zero, float& resv) {
        const int rb = rb_lo + 2 * u;
        const int orow = (rb + half) * RB + row;
        const int o = min(orow, op.N - 1);
        sc = load_sz(op.scales, p.szdt, o);
        zero = load_sz(op.zeros, p.szdt, o);
        resv = 0.f;
        if (op.epilogue == B2L_EPI_RESIDUAL && half < min(2, rb_hi - rb) && orow < op.N)
          resv = op.res_is_emb ? bf2f(resp[orow]) : ld_cg_bf16(resp + orow);
      };
      float sc = 0.f, zero = 0.f, resv = 0.f;
      if (n_units > 0) fetch(0, sc, zero, resv);
      named_bar_sync(3, NB);
      long long ew = 0;
      const long long et0 = clock64();
      long long sum_x = 0;
#pragma unroll
      for (int w = 0; w < MW; ++w) sum_x += red_sx[w];
      const double dsum_x = (double)sum_x;
      const int sh = *red_sh;
      const double inv_scale = __longlong_as_double((long long)(1023 - sh) << 52);
      if (n_units > 0) named_bar_arrive(4, NB);
      if (n_units > 1) named_bar_arrive(5, NB);
      for (int u = 0; u < n_units; ++u) {
        const int rb = rb_lo + 2 * u;
        const int halves = min(2, rb_hi - rb);
        const int buf = u & 1;
        const bool active = half < halves;
        const int orow = (rb + half) * RB + row;
        float sc_n = 0.f, zero_n = 0.f, resv_n = 0.f;
        if (u + 1 < n_units) fetch(u + 1, sc_n, zero_n, resv_n);
        const long long e0 = (p.tl != nullptr) ? clock64() : 0;
        named_bar_sync(6 + buf, NB);
        if (p.tl != nullptr) ew += clock64() - e0;
        int d0 = 0, d1 = 0, d2 = 0, d3 = 0;
        const int hsel = active ? half : 0;
#pragma unroll
        for (int w = 0; w < MW; ++w) {   // integer sums: exact, independent of the order
          const int4 v = *reinterpret_cast<const int4*>(scratch + (((buf * MW + w) * MAX_HALVES + hsel) * RB + row) * 4);
          d0 += v.x; d1 += v.y; d2 += v.z; d3 += v.w;
        }
        if (u + 2 < n_units) named_bar_arrive(4 + buf, NB);
        const long long tq = (long long)d0 + ((long long)d1 << 8) + ((long long)d2 << 16) + ((long long)d3 << 24);
        const float tf = (float)(((double)tq - (double)zero * dsum_x) * inv_scale);
        const float v = rbf(sc * tf);
        if (op.epilogue == B2L_EPI_SWIGLU) {
          const float b = __shfl_down_sync(0xffffffffu, v, 8);
          if (active && row < 8) {
            const float sl = rbf(v / (1.0f + expf(-v)));
            op.y[(rb + half) * 8 + row] = f2bf(sl * b);
          }
        } else if (active && orow < op.N) {
          op.y[orow] = f2bf(op.epilogue == B2L_EPI_RESIDUAL ? v + resv : v);
        }
        sc = sc_n; zero = zero_n; resv = resv_n;
      }
      // this CTA's rows of the op are stored: arrive (release; __syncwarp orders the other lanes' stores before it).
      // The last op's last arriver re-arms the step.
      __syncwarp();
      if (lane == 0) {
        if (oi + 1 < p.n_ops) {
          red_release(p.counters + oi);
        } else {
          unsigned int t;
          asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(t) : "l"(p.counters + oi) : "memory");
          if (t == (unsigned int)G - 1) {
            // every CTA has finished every op: reset the counters and commit the ring advance for the next token
            for (int i = 0; i < p.n_ops; ++i) p.counters[i] = 0u;
            *p.ring_start = ring;
            __threadfence();
          }
        }
        if (p.tl != nullptr) atomicMax(p.tl + oi * 16 + 4, globaltimer_ns());
        if (p.tl != nullptr && blockIdx.x == 0) { p.tl[oi * 16 + 10] = (unsigned long long)ew; p.tl[oi * 16 + 11] = (unsigned long long)(clock64() - et0); }
      }
    }
  }
}

}  // namespace mega
}  // namespace b2l

using namespace b2l;
using namespace b2l::q4mv;

namespace {

struct PlanHeader {   // head of the caller-owned device buffer `plan`
  unsigned int error;
  unsigned int n_ops;
  unsigned int pad[30];
};

inline size_t plan_ops_offset() { return sizeof(PlanHeader); }
inline size_t plan_counters_offset(int n_ops) { return plan_ops_offset() + (size_t)n_ops * sizeof(mega::Op); }
inline int plan_n_ops(const b2l_decode_args* d) { return 5 * d->n_layer + 1; }

bool mega_shape_ok(const b2l_decode_args* d) {
  if (d->B != 1 || d->n_embd % d->n_head != 0 || d->n_embd / d->n_head != mega::HS) return false;
  if (d->flags & B2L_F_W8) return false;   // the persistent kernel's GEMV reads int4 tilings only
  auto ok = [](const b2l_q4_weight& w) { return w.qw_mma != nullptr && w.K % KB == 0 && w.K <= 12288 && w.N > 0; };
  if (!ok(d->lm_head)) return false;
  for (int l = 0; l < d->n_layer; ++l) {
    const b2l_layer& L = d->layers[l];
    if (!ok(L.c_attn) || !ok(L.c_proj) || !ok(L.c_fc12) || !ok(L.mlp_proj)) return false;
    if (L.c_fc12.N % RB != 0) return false;
  }
  return d->n_embd % 8 == 0 && d->n_hidden % 8 == 0;
}

int mega_kmax(const b2l_decode_args* d) {
  int k = d->lm_head.K;
  for (int l = 0; l < d->n_layer; ++l) {
    const b2l_layer& L = d->layers[l];
    k = std::max(k, std::max(std::max(L.c_attn.K, L.c_proj.K), std::max(L.c_fc12.K, L.mlp_proj.K)));
  }
  return k;
}

}  // namespace

extern "C" size_t b2l_decode_plan_bytes(const b2l_decode_args* d) {
  if (!d || d->n_layer <= 0) return 0;
  const int n_ops = plan_n_ops(d);
  return plan_counters_offset(n_ops) + (size_t)(n_ops + 8) * sizeof(unsigned int);
}

extern "C" int b2l_decode_plan_build(const b2l_decode_args* d, b2l_stream_t stream) {
  B2L_CHECK_ARG(d != nullptr && d->layers != nullptr && d->plan != nullptr, "b2l_decode_plan_build: null args / plan");
  if (d->adapters != nullptr)
    for (int l = 0; l < d->n_layer; ++l)
      B2L_CHECK_SUPPORTED(d->adapters[l].len == 0, "b2l_decode_plan_build: LLaMA-Adapter layers (adapters[%d].len = %d) do not run in the persistent kernel", l, d->adapters[l].len);
  if (d->loras != nullptr)
    for (int l = 0; l < d->n_layer; ++l)
      B2L_CHECK_SUPPORTED(d->loras[l].r == 0, "b2l_decode_plan_build: LoRA layers (loras[%d].r = %d) do not run in the persistent kernel", l, d->loras[l].r);
  B2L_CHECK_SUPPORTED(d->affines == nullptr && d->lm_head_affine.scale == nullptr && d->lm_head_affine.bias == nullptr,
                      "b2l_decode_plan_build: LLaMA-Adapter v2 affines do not run in the persistent kernel");
  B2L_CHECK_SUPPORTED(mega_shape_ok(d), "b2l_decode_plan_build: the persistent kernel needs batch 1, head_size 128, int8-tiled per-row int4 weights, K %% 64 == 0, K <= 12288");
  const int n_ops = plan_n_ops(d);
  std::vector<mega::Op> ops((size_t)n_ops);
  const int C = d->n_embd;
  auto gemv = [&](const b2l_q4_weight& w, const void* x, void* y, int prologue, const void* norm_scale, int epilogue, const void* res, int rot) {
    mega::Op o{};
    o.kind = mega::OP_GEMV;
    o.N = w.N; o.K = w.K; o.n_rb = (w.N + RB - 1) / RB;
    o.prologue = prologue; o.epilogue = epilogue; o.rot = rot;
    o.qwt = (const uint8_t*)w.qw_mma; o.scales = w.scales; o.zeros = w.zeros;
    o.x = (const __nv_bfloat16*)x; o.y = (__nv_bfloat16*)y; o.res = (const __nv_bfloat16*)res;
    o.norm_scale = (const __nv_bfloat16*)norm_scale;
    return o;
  };
  const int G = sm_count();
  int oi = 0;
  for (int l = 0; l < d->n_layer; ++l) {
    const b2l_layer& L = d->layers[l];
    // rotations: spread the CTAs that get one row block more (or none) over the grid, op by op
    const int r0 = (l * 5 * 53) % G;
    ops[oi] = gemv(L.c_attn, d->x, d->qkv, B2L_PRO_RMSNORM, L.rms_1, B2L_EPI_STORE, nullptr, (r0 + 0) % G);
    if (l == 0) ops[oi].x_is_emb = 1;
    ++oi;
    mega::Op a{};
    a.kind = mega::OP_ATTN; a.rot = (r0 + 97) % G;
    a.k_cache = (__nv_bfloat16*)L.k_cache; a.v_cache = (__nv_bfloat16*)L.v_cache;
    ops[oi++] = a;
    ops[oi] = gemv(L.c_proj, d->att, d->x, B2L_PRO_NONE, nullptr, B2L_EPI_RESIDUAL, d->x, (r0 + 131) % G);
    if (l == 0) ops[oi].res_is_emb = 1;
    ++oi;
    ops[oi++] = gemv(L.c_fc12, d->x, d->hid, B2L_PRO_RMSNORM, L.rms_2, B2L_EPI_SWIGLU, nullptr, (r0 + 59) % G);
    ops[oi++] = gemv(L.mlp_proj, d->hid, d->x, B2L_PRO_NONE, nullptr, B2L_EPI_RESIDUAL, d->x, (r0 + 211) % G);
  }
  ops[oi++] = gemv(d->lm_head, d->x, d->logits, B2L_PRO_RMSNORM, d->ln_f, B2L_EPI_STORE, nullptr, 0);
  (void)C;
  cudaStream_t st = (cudaStream_t)stream;
  char* plan = (char*)d->plan;
  B2L_CUDA(cudaMemsetAsync(plan, 0, b2l_decode_plan_bytes(d), st));
  PlanHeader h{};
  h.n_ops = (unsigned int)n_ops;
  B2L_CUDA(cudaMemcpyAsync(plan, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  B2L_CUDA(cudaMemcpyAsync(plan + plan_ops_offset(), ops.data(), ops.size() * sizeof(mega::Op), cudaMemcpyHostToDevice, st));
  B2L_CUDA(cudaStreamSynchronize(st));   // `ops` is a host temporary
  return 0;
}

extern "C" int b2l_decode_plan_status(const void* plan, b2l_stream_t stream) {
  B2L_CHECK_ARG(plan != nullptr, "b2l_decode_plan_status: null plan");
  unsigned int e = 0;
  B2L_CUDA(cudaMemcpyAsync(&e, plan, sizeof(e), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  B2L_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  if (e != 0) {
    set_error("b2l_decode_step (persistent kernel): a bounded wait timed out (code %u: 1 = op counter, 2 = ring barrier)", e);
    return B2L_E_STATE;
  }
  return 0;
}

namespace b2l {

template <int MAXC, int NDIG>
static int launch_mega(const b2l_decode_args* d, mega::Params p, cudaStream_t st) {
  const uint32_t budget = 226u * 1024u;
  const uint32_t fixed = mega::smem_layout(0, p.kmax, NDIG).total;
  int nst = fixed + 2 * STAGE_BYTES <= budget ? (int)((budget - fixed) / STAGE_BYTES) : 0;
  if (nst > mega::M_MAX_STAGES) nst = mega::M_MAX_STAGES;
  static const int env_nst = [] { const char* e = getenv("B2L_MEGA_STAGES"); return e ? atoi(e) : 0; }();
  if (env_nst > 0 && nst > env_nst) nst = env_nst;
  if (nst < 2) {
    set_error("b2l_decode_step: K=%d leaves no room for the weight ring", p.kmax);
    return B2L_E_UNSUPPORTED;
  }
  p.nst = nst;
  const mega::SmemLayout L = mega::smem_layout(nst, p.kmax, NDIG);
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(mega::decode_mega_kernel<MAXC, NDIG>, L.total, smem_cache)) return rc;
  int occ = 0;
  B2L_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mega::decode_mega_kernel<MAXC, NDIG>, mega::M_THREADS, L.total));
  if (occ < 1) {
    set_error("b2l_decode_step: the persistent kernel does not fit an SM (occupancy %d)", occ);
    return B2L_E_UNSUPPORTED;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(sm_count());
  cfg.blockDim = dim3(mega::M_THREADS);
  cfg.dynamicSmemBytes = L.total;
  cfg.stream = st;
  // all CTAs must be co-resident (the op counters are grid-wide dependencies): one per SM by construction, and
  // declared to the driver as a cooperative launch (B2L_MEGA_COOP=0: plain launch)
  static const int env_coop = [] { const char* e = getenv("B2L_MEGA_COOP"); return e ? atoi(e) : 1; }();
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = env_coop ? 1 : 0;
  B2L_CUDA(cudaLaunchKernelEx(&cfg, mega::decode_mega_kernel<MAXC, NDIG>, p));
  return 0;
}

// called by b2l_decode_step when args->plan is set
int decode_step_persistent(const b2l_decode_args* d, b2l_stream_t stream) {
  B2L_CHECK_SUPPORTED(mega_shape_ok(d), "b2l_decode_step: the persistent kernel needs batch 1, head_size 128, int8-tiled per-row int4 weights");
  const int n_ops = plan_n_ops(d);
  char* plan = (char*)d->plan;
  mega::Params p{};
  p.ops = (const mega::Op*)(plan + plan_ops_offset());
  p.n_ops = n_ops;
  p.counters = (unsigned int*)(plan + plan_counters_offset(n_ops));
  p.error = (unsigned int*)plan;
  p.idx = d->idx; p.idx_is_i64 = d->idx_is_i64; p.wte = (const __nv_bfloat16*)d->wte; p.vocab = d->vocab;
  p.input_pos = d->input_pos; p.ring_start = d->ring_start;
  p.rope = (const float*)d->rope; p.block_size = d->block_size;
  p.C = d->n_embd; p.n_head = d->n_head; p.S = d->S;
  p.qkv = (const __nv_bfloat16*)d->qkv; p.att = (__nv_bfloat16*)d->att;
  p.attn_work = (float*)d->attn_work;
  p.n_split = (d->S + mega::ATT_CHUNK - 1) / mega::ATT_CHUNK;
  // tickets live behind the partials, exactly where b2l_attention keeps them (b2l_attn_workspace_bytes)
  p.tickets = reinterpret_cast<int*>(reinterpret_cast<char*>(d->attn_work) +
                                     (b2l_attn_workspace_bytes(1, d->n_head, mega::HS, 1, d->S) - (size_t)d->n_head * sizeof(int)));
  p.eps = d->eps; p.szdt = d->sz_dtype;
  p.kmax = mega_kmax(d);
  p.tl = (unsigned long long*)d->timeline;
  cudaStream_t st = (cudaStream_t)stream;
  // four digits (|X| < 2^30) up to K = 8192, three (|X| < 2^22, smaller planes, deeper ring) above
  if (p.kmax <= 8192) return launch_mega<2, 4>(d, p, st);
  return launch_mega<3, 3>(d, p, st);
}

}  // namespace b2l

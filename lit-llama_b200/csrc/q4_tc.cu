// Fused [RMSNorm ->] int4 weight-only linear [-> residual | SwiGLU] for M <= 16 rows
// (decode and short prefill) on the Hopper tensor cores (wgmma).
//
// Replaces, for gptq.int4 with one (scale, zero) per output row:
//   ColBlockQuantizedLinear.forward      lit_llama/quantization.py:413-423
//   linear_kernel_4bit_weight (Triton)   lit_llama/quantization.py:187-333
//   RMSNorm.forward                      lit_llama/model.py:270-277      (prologue)
//   x + h / silu(a) * b                  lit_llama/model.py:166-167, 252 (epilogue)
//
// Data flow per CTA (one 128-row output tile x one K range; the K ranges of a tile
// form a thread-block cluster and are reduced through distributed shared memory):
//
//   HBM --TMA bulk copy--> smem ring of packed slabs [128 rows][16 B = 32 nibbles]
//       --LDS.128, LOP3, HSUB2--> registers: bf16 pairs (level), exact, in the wgmma A-fragment order
//   x (bf16, RMSNorm'd on the fly) --> smem B operand (K-major core matrices)
//   wgmma.m64nNk16 (N = 8 or 16 token columns), one warpgroup per 64 output rows:
//       D (registers, fp32) += A (registers) * B (smem descriptor)
//   y[o] = scale[o] * (acc - zero[o] * sum_k x[k])
//
// The scale/zero are hoisted out of the K loop (exact algebra, fp32): the tensor core
// only ever sees the integers 0..15 and the bf16 activations.
//
// Weights do not depend on the previous kernel, so with programmatic dependent launch
// the TMA producer starts streaming before `griddepcontrol.wait`; only the x load waits.
#include "b2l_common.cuh"

namespace b2l {
namespace q4tc {

constexpr int TILE_N = 128;
constexpr int SLAB_K = 32;
constexpr int SLAB_BYTES = TILE_N * 16;  // 2048
constexpr int G = 2;                     // slabs per stage
constexpr int STAGE_BYTES = G * SLAB_BYTES;
constexpr int NCONV = 256;               // two MMA warpgroups (warps 0..7), 64 output rows each
constexpr int PRODUCER_WARP = NCONV / 32;      // warp 8: TMA producer
constexpr int NTHREADS = NCONV + 32;
constexpr int MAX_M = 16;
constexpr int MAX_STAGES = 16;
constexpr int SMEM_BUDGET = 74 * 1024;   // three CTAs per SM

struct Params {
  const __nv_bfloat16* x; int ldx;
  const uint8_t* qwt;
  const void* scales; const void* zeros; int szdt;
  __nv_bfloat16* y; int ldy;
  int M, N, K;
  int prologue; const __nv_bfloat16* norm_scale; float eps;
  int epilogue; const __nv_bfloat16* res; int ldres;
  int S;          // cluster size (split-K)
  int nst_ring;   // ring stages
  int kcb;        // bytes per 8-k core-matrix column of the B operand (256 for 16 token rows, 128 for 8)
  int kseg_max;   // max K elements of one rank
  unsigned long long* trace;  // debug: clock64 stamps of CTA 0 (nullptr = off)
};

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_dsmem_f32(uint32_t local_addr, uint32_t rank) {
  uint32_t ra;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(ra) : "memory");
  return v;
}
// the barrier id in a register (bar_sync_c, b2l_common.cuh, takes it as an immediate)
__device__ __forceinline__ void bar_sync_reg(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

template <int NR> __device__ __forceinline__ void reg_fence(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x NN] (fp32, registers) += A[64 x 16] (bf16, registers) * B[16 x NN] (bf16, smem, K-major)
template <int NN> struct Wgmma;
template <> struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1)
        : "memory");
  }
};
template <> struct Wgmma<8> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1)
        : "memory");
  }
};

// Nibble pair s of one word -> the bf16 pair (level[k], level[k+1]), k = 8 * word + 2 * s: 0x4300 is bf16 128.0
// whose ulp is 1, so OR-ing a 4-bit level into the mantissa gives 128 + level exactly, and subtracting 128 is exact.
// Feeding 128 + level would make the fp32 accumulator carry 128 x for every activation and round at that magnitude:
// an output whose level sits at its zero point on a massive channel (|x| ~ 1e4) would be off by several ulps.
__device__ __forceinline__ uint32_t unpack_pair(uint32_t w, int s) {
  uint32_t d;
  asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(((w >> (4 * s)) & 0x000f000fu) | 0x43004300u), "r"(0x43004300u));
  return d;
}

#define B2L_TRACE(slot)                                                      \
  do {                                                                       \
    if (p.trace != nullptr && blockIdx.x == 0) p.trace[(slot)] = clock64(); \
  } while (0)

// ---------------------------------------------------------------- shared memory map
struct SmemLayout {
  uint32_t ring, xb, part, xsum, red, bars, total;
};
__host__ __device__ inline SmemLayout smem_layout(int nst_ring, int kseg_max, int kcb, int M) {
  SmemLayout L;
  uint32_t o = 0;
  L.ring = o; o += (uint32_t)nst_ring * STAGE_BYTES;
  L.xb = o;   o += (uint32_t)(kseg_max / 8) * kcb;
  L.part = o; o += TILE_N * M * 4;  // [m][row] fp32 partials of this rank (DSMEM-read by rank 0)
  L.xsum = o; o += MAX_M * 4;
  L.red = o;  o += (NCONV / 32) * MAX_M * 4;  // per-warp partials
  o = (o + 7u) & ~7u;
  L.bars = o; o += 2 * MAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

template <int NN>
__global__ void __launch_bounds__(NTHREADS, 3) q4_linear_tc_kernel(const Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const SmemLayout L = smem_layout(p.nst_ring, p.kseg_max, p.kcb, p.M);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = p.S;
  const int nt = blockIdx.x / S;
  const int rank = (S > 1) ? (int)cluster_ctarank() : 0;

  // K range of this rank, in slabs
  const int slabs_total = p.K / SLAB_K;
  const int sl_base = slabs_total / S, sl_rem = slabs_total % S;
  const int nslab = sl_base + (rank < sl_rem ? 1 : 0);
  const int slab0 = rank * sl_base + min(rank, sl_rem);
  const int nstages = (nslab + G - 1) / G;
  const int k0 = slab0 * SLAB_K, kseg = nslab * SLAB_K;

  const uint32_t bar_w_full = sbase + L.bars;
  const uint32_t bar_w_empty = bar_w_full + MAX_STAGES * 8;

  if (tid == 0) B2L_TRACE(0);
  if (tid == 0) {
    for (int i = 0; i < p.nst_ring; ++i) {
      mbar_init(bar_w_full + i * 8, 1);
      mbar_init(bar_w_empty + i * 8, NCONV / 32);   // every MMA warp reads every slab
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ===================== TMA producer (warp 8, lane 0): stream the packed slabs of this rank ==========
    // The first ring-full of stages is requested before the dependent-launch trigger: the weights do not
    // depend on the previous kernel.
    if (lane == 0) {
      const uint8_t* w_src = p.qwt + ((size_t)nt * slabs_total + slab0) * SLAB_BYTES;
      const int n_first = min(nstages, p.nst_ring);
      for (int st = 0; st < n_first; ++st) {
        const int ns = min(G, nslab - st * G);
        const uint32_t bytes = (uint32_t)ns * SLAB_BYTES;
        mbar_expect_tx(bar_w_full + st * 8, bytes);
        tma_bulk_g2s(sbase + L.ring + st * STAGE_BYTES, w_src + (size_t)st * STAGE_BYTES, bytes, bar_w_full + st * 8);
        if (st < 20) B2L_TRACE(108 + st);
      }
      pdl_launch_dependents();  // the next kernel's CTAs may start prefetching their weights
      int slot = 0;
      uint32_t phase = 0;  // second use of slot 0 waits for its first release
      for (int st = n_first; st < nstages; ++st) {
        mbar_wait(bar_w_empty + slot * 8, phase);
        const int ns = min(G, nslab - st * G);
        const uint32_t bytes = (uint32_t)ns * SLAB_BYTES;
        mbar_expect_tx(bar_w_full + slot * 8, bytes);
        tma_bulk_g2s(sbase + L.ring + slot * STAGE_BYTES, w_src + (size_t)st * STAGE_BYTES, bytes, bar_w_full + slot * 8);
        if (st < 20) B2L_TRACE(108 + st);
        if (++slot == p.nst_ring) { slot = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  } else {
    // ===================== MMA warpgroups (warpgroup wg = output rows 64 wg .. 64 wg + 63 of the tile) =====
    // -- activations: wait for the producing kernel, normalise, lay out as the B operand
    pdl_wait();
    if (tid == 0) B2L_TRACE(2);
    float* xsum = reinterpret_cast<float*>(smem + L.xsum);
    float* red = reinterpret_cast<float*>(smem + L.red);  // [8 warps][MAX_M]
    {
      const int rows = (p.kcb == 256) ? 16 : 8;
      const int nkc = kseg / 8;
      if (p.M < rows) {
        for (int i = tid; i < nkc * rows; i += NCONV) {
          const int kc = i / rows, r = i % rows;
          if (r >= p.M)
            *reinterpret_cast<uint4*>(smem + L.xb + kc * p.kcb + (r >> 3) * 128 + (r & 7) * 16) = make_uint4(0, 0, 0, 0);
        }
      }
      for (int m = 0; m < p.M; ++m) {
        const __nv_bfloat16* xr = p.x + (size_t)m * p.ldx;
        const bool norm = (p.prologue == B2L_PRO_RMSNORM);
        // issue every global load of this row up front (one round trip): the whole row for the
        // sum of squares (4 chunks of 2048 elements in registers), this rank's segment, and the norm scale
        constexpr int MAXC = 4;
        uint4 full[MAXC];
        if (norm) {
#pragma unroll
          for (int c = 0; c < MAXC; ++c) {
            const int k = (c * NCONV + tid) * 8;
            full[c] = (k < p.K) ? *reinterpret_cast<const uint4*>(xr + k) : make_uint4(0, 0, 0, 0);
          }
        }
        // this rank's K segment: up to XC chunks of 8 elements per thread (kseg <= XC * NCONV * 8, host-checked)
        constexpr int XC = 2;
        uint4 u[XC], sc[XC];
#pragma unroll
        for (int c = 0; c < XC; ++c) {
          const int kk = (c * NCONV + tid) * 8;
          u[c] = make_uint4(0, 0, 0, 0);
          sc[c] = make_uint4(0, 0, 0, 0);
          if (kk < kseg) {
            u[c] = *reinterpret_cast<const uint4*>(xr + k0 + kk);
            if (norm) sc[c] = *reinterpret_cast<const uint4*>(p.norm_scale + k0 + kk);
          }
        }
        float rinv = 1.f;
        if (norm) {
          float ss = 0.f;
          if (p.K > MAXC * NCONV * 8) {  // very wide rows: remaining chunks the slow way
            for (int k = (MAXC * NCONV + tid) * 8; k < p.K; k += NCONV * 8) {
              uint4 t = *reinterpret_cast<const uint4*>(xr + k);
              const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                float a = __uint_as_float(w[q] << 16), b = __uint_as_float(w[q] & 0xffff0000u);
                ss += rbf(a * a) + rbf(b * b);
              }
            }
          }
#pragma unroll
          for (int c = 0; c < MAXC; ++c) {
            const uint32_t w[4] = {full[c].x, full[c].y, full[c].z, full[c].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float a = __uint_as_float(w[q] << 16), b = __uint_as_float(w[q] & 0xffff0000u);
              ss += rbf(a * a) + rbf(b * b);
            }
          }
          ss = warp_sum(ss);
          if (lane == 0) red[warp * MAX_M + m] = ss;
          bar_sync_reg(1, NCONV);
          ss = 0.f;
#pragma unroll
          for (int w = 0; w < NCONV / 32; ++w) ss += red[w * MAX_M + m];
          rinv = rms_rinv(ss, p.K, p.eps);
          bar_sync_reg(1, NCONV);
        }
        float sx = 0.f;
#pragma unroll
        for (int c = 0; c < XC; ++c) {
          const int kk = (c * NCONV + tid) * 8;
          if (kk < kseg) {
            uint32_t w[4] = {u[c].x, u[c].y, u[c].z, u[c].w};
            if (norm) {
              const uint32_t g[4] = {sc[c].x, sc[c].y, sc[c].z, sc[c].w};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                float a = rms_apply(__uint_as_float(w[q] << 16), rinv, __uint_as_float(g[q] << 16));
                float b = rms_apply(__uint_as_float(w[q] & 0xffff0000u), rinv, __uint_as_float(g[q] & 0xffff0000u));
                sx += a + b;
                w[q] = (__float_as_uint(a) >> 16) | (__float_as_uint(b) & 0xffff0000u);
              }
            } else {
#pragma unroll
              for (int q = 0; q < 4; ++q) sx += __uint_as_float(w[q] << 16) + __uint_as_float(w[q] & 0xffff0000u);
            }
            *reinterpret_cast<uint4*>(smem + L.xb + (kk / 8) * p.kcb + (m >> 3) * 128 + (m & 7) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
          }
        }
        sx = warp_sum(sx);
        if (lane == 0) red[warp * MAX_M + m] = sx;
        bar_sync_reg(1, NCONV);
        if (tid == 0) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < NCONV / 32; ++w) t += red[w * MAX_M + m];
          xsum[m] = t;
        }
      }
      fence_proxy_async_smem();  // B operand written with generic stores, read by the tensor core
      bar_sync_reg(1, NCONV);
      if (tid == 0) B2L_TRACE(3);
    }

    // -- weights: smem slab -> registers (A fragments) -> wgmma.  Thread (g = lane / 4, t = lane % 4) of warp wq of
    // warpgroup wg holds rows r0 = 64 wg + 16 wq + g and r0 + 8; within a slab, k16 step j reads words 2j (k 0..7)
    // and 2j + 1 (k 8..15) of those rows, nibble pair t = k 2t, 2t + 1 of each.
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2), tq = lane & 3;
    float acc[NN / 2];
#pragma unroll
    for (int i = 0; i < NN / 2; ++i) acc[i] = 0.f;
    const uint64_t bdesc0 = make_desc(sbase + L.xb, p.kcb, 128);
    const uint32_t kcb16 = (uint32_t)p.kcb >> 4;   // descriptor address units per 8-k column
    int slot = 0;
    uint32_t rphase = 0;
    for (int st = 0; st < nstages; ++st) {
      const int ns = min(G, nslab - st * G);
      mbar_wait(bar_w_full + slot * 8, rphase);
      if (tid == 0 && st < 20) B2L_TRACE(4 + st);
      uint32_t a[G][2][4];
#pragma unroll
      for (int s = 0; s < G; ++s) {
        if (s < ns) {
          const uint8_t* sl = smem + L.ring + slot * STAGE_BYTES + s * SLAB_BYTES;
          const uint4 lo = *reinterpret_cast<const uint4*>(sl + r0 * 16);
          const uint4 hi = *reinterpret_cast<const uint4*>(sl + (r0 + 8) * 16);
          a[s][0][0] = unpack_pair(lo.x, tq); a[s][0][1] = unpack_pair(hi.x, tq);
          a[s][0][2] = unpack_pair(lo.y, tq); a[s][0][3] = unpack_pair(hi.y, tq);
          a[s][1][0] = unpack_pair(lo.z, tq); a[s][1][1] = unpack_pair(hi.z, tq);
          a[s][1][2] = unpack_pair(lo.w, tq); a[s][1][3] = unpack_pair(hi.w, tq);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_w_empty + slot * 8);  // slab bytes are in registers: slot may be refilled
      wgmma_fence();
      reg_fence(acc);
#pragma unroll
      for (int s = 0; s < G; ++s) {
        if (s < ns) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint32_t kstep = (uint32_t)((st * G + s) * 2 + j);   // k16 step within this rank's segment
            Wgmma<NN>::mma(acc, a[s][j], bdesc0 + (uint64_t)(2 * kstep * kcb16));
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();   // the A registers are rewritten next stage
      reg_fence(acc);
      if (tid == 0 && st < 20) B2L_TRACE(44 + st);
      if (++slot == p.nst_ring) { slot = 0; rphase ^= 1; }
    }

    // -- epilogue part 1: accumulator -> scaled partial of this rank.  acc[4 c + e] = row r0 (+ 8 for e >= 2),
    // token column 8 c + 2 tq + (e & 1)
    float* part = reinterpret_cast<float*>(smem + L.part);
    if (tid == 0) B2L_TRACE(104);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      const int o = min(nt * TILE_N + row, p.N - 1);  // padded rows of the last tile are never stored
      const float sc = load_sz(p.scales, p.szdt, o);
      const float zz = load_sz(p.zeros, p.szdt, o);
#pragma unroll
      for (int c = 0; c < NN / 8; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 8 * c + 2 * tq + e;
          if (m < p.M) part[m * TILE_N + row] = sc * (acc[4 * c + 2 * h + e] - zz * xsum[m]);
        }
      }
    }
  }

  // ===================== cross-rank reduction + epilogue (rank 0, warps 0..3: thread = output row) ==========
  if (S > 1) cluster_sync_all(); else __syncthreads();
  if (tid == 0) B2L_TRACE(105);
  if (rank == 0 && warp < 4) {
    float tot[MAX_M];
    float* part = reinterpret_cast<float*>(smem + L.part);
    const uint32_t part_addr = sbase + L.part + tid * 4;
#pragma unroll
    for (int m = 0; m < MAX_M; ++m) {
      if (m < p.M) {
        float t = part[m * TILE_N + tid];
        for (int r = 1; r < S; ++r) t += ld_dsmem_f32(part_addr + m * TILE_N * 4, (uint32_t)r);  // fixed order
        tot[m] = t;
      }
    }
    const int o = nt * TILE_N + tid;
    if (p.epilogue == B2L_EPI_SWIGLU) {
      // rank 0's own partials were only read by the owning thread: reuse them for the exchange
      float* fin = part;
#pragma unroll
      for (int m = 0; m < MAX_M; ++m)
        if (m < p.M) fin[m * TILE_N + tid] = rbf(tot[m]);
      bar_sync_reg(2, 128);
      if (tid < 64) {
        const int oo = nt * 64 + tid;
#pragma unroll
        for (int m = 0; m < MAX_M; ++m) {
          if (m < p.M) {
            const float a = fin[m * TILE_N + tid], b = fin[m * TILE_N + tid + 64];
            const float sl = rbf(a / (1.0f + expf(-a)));
            p.y[(size_t)m * p.ldy + oo] = f2bf(sl * b);
          }
        }
      }
    } else {
#pragma unroll
      for (int m = 0; m < MAX_M; ++m) {
        if (m < p.M && o < p.N) {
          float v = rbf(tot[m]);
          if (p.epilogue == B2L_EPI_RESIDUAL) v = v + bf2f(p.res[(size_t)m * p.ldres + o]);
          p.y[(size_t)m * p.ldy + o] = f2bf(v);
        }
      }
    }
  }
  if (tid == 0) B2L_TRACE(106);
  if (S > 1) cluster_sync_all();   // peers keep their partials alive until rank 0 has read them
  if (tid == 0) B2L_TRACE(107);
}

// ---------------------------------------------------------------- re-tiling
// nibble position s of word i  <->  k = 32*slab + 8*i + (s < 4 ? 2*s : 2*(s-4)+1)
__global__ void q4_tile_kernel(const uint8_t* __restrict__ qw, uint32_t* __restrict__ out, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int KS = K / SLAB_K;
  const int ntiles = (N + TILE_N - 1) / TILE_N;
  const size_t total = (size_t)ntiles * KS * TILE_N * 4;
  if (idx >= total) return;
  const int i = idx & 3;
  const int r = (idx >> 2) & (TILE_N - 1);
  const size_t rest = idx >> 9;
  const int ks = (int)(rest % KS), nt = (int)(rest / KS);
  const int o = nt * TILE_N + r;
  uint32_t w = 0;
  if (o < N) {
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int k = ks * SLAB_K + 8 * i + (s < 4 ? 2 * s : 2 * (s - 4) + 1);
      const uint8_t b = qw[(size_t)(k >> 1) * N + o];
      w |= (uint32_t)((b >> ((k & 1) * 4)) & 0xF) << (4 * s);
    }
  }
  out[idx] = w;
}

__global__ void q4_untile_kernel(const uint32_t* __restrict__ tiled, uint8_t* __restrict__ qw, int N, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one packed byte [j][o]
  const size_t total = (size_t)(K / 2) * N;
  if (idx >= total) return;
  const int o = (int)(idx % N), j = (int)(idx / N);
  const int KS = K / SLAB_K;
  uint8_t b = 0;
#pragma unroll
  for (int nr = 0; nr < 2; ++nr) {
    const int k = 2 * j + nr;
    const int ks = k / SLAB_K, kl = k % SLAB_K, i = kl / 8, e = kl % 8;
    const int s = (e & 1) ? 4 + (e >> 1) : (e >> 1);
    const uint32_t w = tiled[(((size_t)(o / TILE_N) * KS + ks) * TILE_N + (o % TILE_N)) * 4 + i];
    b |= (uint8_t)(((w >> (4 * s)) & 0xF) << (4 * nr));
  }
  qw[idx] = b;
}

}  // namespace q4tc
}  // namespace b2l

using namespace b2l;
using namespace b2l::q4tc;

extern "C" size_t b2l_q4_tiled_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || K % SLAB_K != 0) return 0;
  return (size_t)((N + TILE_N - 1) / TILE_N) * (K / SLAB_K) * SLAB_BYTES;
}

extern "C" int b2l_q4_tile(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_q4_tile: bad argument");
  B2L_CHECK_SUPPORTED(K % SLAB_K == 0, "b2l_q4_tile: in_features %d must be a multiple of %d", K, SLAB_K);
  const size_t total = b2l_q4_tiled_bytes(N, K) / 4;
  q4_tile_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint8_t*)qw, (uint32_t*)qw_tiled, N, K);
  B2L_LAUNCH_CHECK("q4_tile_kernel");
  return 0;
}

extern "C" int b2l_q4_untile(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && qw_tiled && N > 0 && K > 0, "b2l_q4_untile: bad argument");
  B2L_CHECK_SUPPORTED(K % SLAB_K == 0, "b2l_q4_untile: in_features %d must be a multiple of %d", K, SLAB_K);
  const size_t total = (size_t)(K / 2) * N;
  q4_untile_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint32_t*)qw_tiled, (uint8_t*)qw, N, K);
  B2L_LAUNCH_CHECK("q4_untile_kernel");
  return 0;
}

namespace b2l {
// Split-K (cluster size) choice: one wave of at most 3 CTAs per SM if possible; cost model =
// waves x (slabs per CTA + a fixed per-CTA cost worth ~24 slabs of prologue/epilogue latency).
int q4_pick_split(int n_tiles, int slabs_total) {
  const int slots = 3 * sm_count();
  int best = 1;
  long best_cost = -1;
  for (int S = 1; S <= 8; ++S) {
    if (slabs_total / S < 2) break;
    const int per = (slabs_total + S - 1) / S;
    if (per * q4tc::SLAB_K > 2 * q4tc::NCONV * 8) continue;  // two activation chunks per convert thread
    const long waves = ((long)n_tiles * S + slots - 1) / slots;
    const long cost = waves * (per + 24);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = S; }
  }
  return best_cost < 0 ? 8 : best;
}

// b2l_q4_linear_tc's argument checks, split-K and shared-memory layout: 0, or B2L_E_* with a message
static int plan_linear_tc(const b2l_q4_linear_args* a, Params& p, SmemLayout& L) {
  B2L_CHECK_ARG(a != nullptr, "b2l_q4_linear_tc: null args");
  B2L_CHECK_ARG(a->x && a->qw_tiled && a->scales && a->zeros && a->y, "b2l_q4_linear_tc: null pointer");
  B2L_CHECK_SUPPORTED(a->out_affine.scale == nullptr && a->out_affine.bias == nullptr,
                      "b2l_q4_linear_tc: out_affine is not supported (apply b2l_linear_affine to y)");
  B2L_CHECK_SUPPORTED(a->M >= 1 && a->M <= MAX_M, "b2l_q4_linear_tc: M=%d outside 1..%d", a->M, MAX_M);
  B2L_CHECK_SUPPORTED(a->K > 0 && a->K % SLAB_K == 0, "b2l_q4_linear_tc: K=%d must be a multiple of %d", a->K, SLAB_K);
  B2L_CHECK_ARG(a->N > 0 && a->ldx >= a->K, "b2l_q4_linear_tc: bad N/ldx");
  B2L_CHECK_ARG(((uintptr_t)a->x % 16 == 0) && (a->ldx % 8 == 0) && ((uintptr_t)a->qw_tiled % 16 == 0),
                "b2l_q4_linear_tc: x / qw_tiled must be 16-byte aligned, ldx a multiple of 8");
  B2L_CHECK_ARG(a->sz_dtype == B2L_BF16 || a->sz_dtype == B2L_F32, "b2l_q4_linear_tc: bad sz_dtype");
  if (a->prologue == B2L_PRO_RMSNORM)
    B2L_CHECK_ARG(a->norm_scale && ((uintptr_t)a->norm_scale % 16 == 0), "b2l_q4_linear_tc: RMSNorm prologue needs a 16-byte aligned scale");
  else
    B2L_CHECK_ARG(a->prologue == B2L_PRO_NONE, "b2l_q4_linear_tc: bad prologue %d", a->prologue);
  if (a->epilogue == B2L_EPI_RESIDUAL) B2L_CHECK_ARG(a->res && a->ldres >= a->N, "b2l_q4_linear_tc: RESIDUAL epilogue needs res");
  else if (a->epilogue == B2L_EPI_SWIGLU) B2L_CHECK_SUPPORTED(a->N % TILE_N == 0, "b2l_q4_linear_tc: SWIGLU needs N %% 128 == 0");
  else B2L_CHECK_ARG(a->epilogue == B2L_EPI_STORE, "b2l_q4_linear_tc: bad epilogue %d", a->epilogue);

  const int n_tiles = (a->N + TILE_N - 1) / TILE_N;
  const int slabs_total = a->K / SLAB_K;
  int S = a->split_k > 0 ? a->split_k : q4_pick_split(n_tiles, slabs_total);
  B2L_CHECK_SUPPORTED(S >= 1 && S <= 8, "b2l_q4_linear_tc: split_k=%d must be in 1..8", S);
  while (S > 1 && slabs_total < 2 * S) --S;

  p.x = (const __nv_bfloat16*)a->x; p.ldx = a->ldx;
  p.qwt = (const uint8_t*)a->qw_tiled;
  p.scales = a->scales; p.zeros = a->zeros; p.szdt = a->sz_dtype;
  p.y = (__nv_bfloat16*)a->y; p.ldy = a->ldy;
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.prologue = a->prologue; p.norm_scale = (const __nv_bfloat16*)a->norm_scale; p.eps = a->eps;
  p.epilogue = a->epilogue; p.res = (const __nv_bfloat16*)a->res; p.ldres = a->ldres;
  p.S = S;
  p.trace = (unsigned long long*)a->trace;
  const int max_slabs = (slabs_total + S - 1) / S;
  p.kseg_max = max_slabs * SLAB_K;
  p.kcb = (!(a->flags & B2L_F_NO_ALIAS_N) && a->M <= 8) ? 128 : 256;  // 8 or 16 token rows in the B operand
  B2L_CHECK_SUPPORTED(p.kseg_max <= 2 * NCONV * 8, "b2l_q4_linear_tc: K/split_k = %d > %d: raise split_k (K=%d, split_k=%d)",
                      p.kseg_max, 2 * NCONV * 8, a->K, S);
  const int stages_needed = (max_slabs + G - 1) / G;
  // ring depth: the whole K range in flight when it fits the per-CTA budget (3 CTAs per SM), >= 4 stages
  const uint32_t fixed = smem_layout(0, p.kseg_max, p.kcb, p.M).total;
  int ring = fixed < (uint32_t)SMEM_BUDGET ? (int)((SMEM_BUDGET - fixed) / STAGE_BYTES) : 0;
  if (ring < 4) ring = 4;
  if (ring > MAX_STAGES) ring = MAX_STAGES;
  p.nst_ring = stages_needed < ring ? stages_needed : ring;
  if (p.nst_ring < 1) p.nst_ring = 1;
  L = smem_layout(p.nst_ring, p.kseg_max, p.kcb, p.M);
  B2L_CHECK_SUPPORTED(L.total <= 200 * 1024, "b2l_q4_linear_tc: shared memory %u B too large (K=%d, split_k=%d)", L.total, a->K, S);
  return 0;
}

int check_q4_linear_tc(const b2l_q4_linear_args* a) {
  Params p;
  SmemLayout L;
  return plan_linear_tc(a, p, L);
}
}  // namespace b2l

extern "C" int b2l_q4_linear_tc(const b2l_q4_linear_args* a, b2l_stream_t stream) {
  Params p;
  SmemLayout L;
  if (int rc = plan_linear_tc(a, p, L)) return rc;
  const int n_tiles = (a->N + TILE_N - 1) / TILE_N;
  static DynSmemCache smem_cache[2];
  LaunchCfg lc(dim3(n_tiles * p.S), dim3(NTHREADS), L.total, (cudaStream_t)stream, (a->flags & B2L_F_PDL) != 0, p.S);
  if (p.kcb == 256) {   // 16 token columns per MMA
    if (int rc = ensure_dyn_smem(q4_linear_tc_kernel<16>, L.total, smem_cache[1])) return rc;
    B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q4_linear_tc_kernel<16>, p));
  } else {              // at most 8 token rows: n8 MMAs on an 8-row B operand
    if (int rc = ensure_dyn_smem(q4_linear_tc_kernel<8>, L.total, smem_cache[0])) return rc;
    B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q4_linear_tc_kernel<8>, p));
  }
  return 0;
}

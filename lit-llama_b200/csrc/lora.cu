// LoRA (lit_llama/lora.py:308-326): the low-rank term of an UNMERGED MergedLinear, added in place to the output of
// its base linear.  A quantized base (gptq.int4 / gptq.int8 / llm.int8) cannot absorb s * B.A into its levels, so
// the term stays per-token work: one launch behind c_attn.
//
//   u_m  = bf16(A_g . xh_m)                      (F.linear(x, lora_A), :314; group g uses rows [g r, (g+1) r) of A)
//   d    = bf16(B_g . u_m)                       (grouped conv1d, :320-324; rows [g Ng, (g+1) Ng) of lora_B)
//   y    = bf16(y + bf16(d * scaling))           (zero_pad(d) * scaling added to the result, :325)
//
// xh_m is the linear's input row, or rms_1(x_m) recomputed from the residual stream with b2l_rmsnorm's rounding points
// when a norm scale is given (inside the whole-token step the normalised row only exists in c_attn's prologue).
// Accumulation is fp32 FMA: at M = 2048 the term is ~0.3 GFLOP next to ~200 GFLOP of c_attn GEMM.
//
// Grid: (enabled group, slice of that group's output rows) x (16-row tile of M).  Every CTA computes u for its tile
// and group (r x K of A, read from L2) and then its slice of rows, one row per thread.  The slice count aims at ~2
// CTAs per SM but never goes below 256 rows per slice: at M = 1 a 7B layer runs 2 x 16 CTAs, and a prompt does not
// recompute u more than it has to.
#include <algorithm>

#include "b2l_common.cuh"

namespace b2l {

constexpr int LORA_THREADS = 256;
constexpr int LORA_MT = 16;   // activation rows per CTA

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// x may have been written by the previous launch: a coherent ld.global (never ld.global.nc), as ld_coherent_u4, but
// without its memory clobber, so the compiler keeps several of a lane's K chunks in flight.  Every use of x follows
// griddepcontrol.wait (itself a memory-clobbering asm), so no load can be hoisted above it.
__device__ __forceinline__ uint4 ld_act(const __nv_bfloat16* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// The term of one CTA: mt rows of x / y (row m of the tile is row row_of(m) of the tensors), group G, whose lora_A /
// lora_B rows start at Ag / Bg, and that group's output rows [n_lo, n_hi).  lora_kernel and lora_rows_kernel differ
// only in which rows and which weights a CTA takes, so a row's arithmetic is the same in both.
template <class RowOf>
__device__ __forceinline__ void lora_tile(const __nv_bfloat16* __restrict__ Ag, const __nv_bfloat16* __restrict__ Bg,
                                          float scaling, int r, int G, int Ng, const __nv_bfloat16* x, int ldx,
                                          const __nv_bfloat16* __restrict__ norm, float eps, __nv_bfloat16* y, int ldy,
                                          int mt, int n_lo, int n_hi, int K, int warp, int lane, RowOf row_of) {
  __shared__ float U[LORA_MT][B2L_LORA_MAX_R];
  __shared__ float rinv[LORA_MT];

  // A and B are weights: ask the L2 for them before the activations exist.  x and y are not touched before the wait
  // (under PDL the previous launches may still be writing them).
  {
    const char* pa = (const char*)Ag;
    const size_t na = (size_t)r * K * 2;
    for (size_t o = (size_t)threadIdx.x * 128; o < na; o += (size_t)LORA_THREADS * 128) prefetch_l2(pa + o);
    if (n_hi > n_lo) {
      const char* pb = (const char*)(Bg + (size_t)n_lo * r);
      const size_t nb = (size_t)(n_hi - n_lo) * r * 2;
      for (size_t o = (size_t)threadIdx.x * 128; o < nb; o += (size_t)LORA_THREADS * 128) prefetch_l2(pb + o);
    }
  }
  pdl_launch_dependents();   // the next launch (attention) may start its own prefetch now
  pdl_wait();

  if (norm != nullptr) {   // rms_1 of the residual rows: ms = bf16(mean(bf16(x*x))) ... (elementwise.cu, rmsnorm_kernel)
    // every warp takes a share of every row's K, so a decode step (one row) is one round of loads, not one per chunk
    __shared__ float part[LORA_MT][LORA_THREADS / 32];
    for (int m = 0; m < mt; ++m) {
      const __nv_bfloat16* xr = x + (size_t)row_of(m) * ldx;
      float ss = 0.f;
#pragma unroll 4
      for (int k = threadIdx.x * 8; k < K; k += LORA_THREADS * 8) {
        const uint4 v = ld_act(xr + k);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) ss += rbf(bf_lo(w[q]) * bf_lo(w[q])) + rbf(bf_hi(w[q]) * bf_hi(w[q]));
      }
      ss = warp_sum(ss);
      if (lane == 0) part[m][warp] = ss;
    }
    __syncthreads();
    if (threadIdx.x < mt) {
      float ss = 0.f;
      for (int w = 0; w < LORA_THREADS / 32; ++w) ss += part[threadIdx.x][w];
      rinv[threadIdx.x] = rms_rinv(ss, K, eps);
    }
    __syncthreads();
  }

  // u[m][j] = bf16(sum_k xh[m][k] A_g[j][k]): one warp per (m, j), lanes along K
  for (int p = warp; p < mt * r; p += LORA_THREADS / 32) {
    const int m = p / r, j = p - m * r;
    const __nv_bfloat16* xr = x + (size_t)row_of(m) * ldx;
    const __nv_bfloat16* ar = Ag + (size_t)j * K;
    const float ri = norm != nullptr ? rinv[m] : 0.f;
    float acc = 0.f;
    for (int k0 = lane * 8; k0 < K; k0 += 4 * 256) {   // four 16-byte chunks of x, A (and the norm scale) in flight
      uint4 xv[4], av[4], sv[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int k = k0 + c * 256;
        if (k < K) {
          xv[c] = ld_act(xr + k);
          av[c] = __ldg(reinterpret_cast<const uint4*>(ar + k));
          if (norm != nullptr) sv[c] = __ldg(reinterpret_cast<const uint4*>(norm + k));
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (k0 + c * 256 >= K) break;
        const uint32_t xw[4] = {xv[c].x, xv[c].y, xv[c].z, xv[c].w}, aw[4] = {av[c].x, av[c].y, av[c].z, av[c].w};
        if (norm != nullptr) {
          const uint32_t sw[4] = {sv[c].x, sv[c].y, sv[c].z, sv[c].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            acc = fmaf(rms_apply(bf_lo(xw[q]), ri, bf_lo(sw[q])), bf_lo(aw[q]), acc);
            acc = fmaf(rms_apply(bf_hi(xw[q]), ri, bf_hi(sw[q])), bf_hi(aw[q]), acc);
          }
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            acc = fmaf(bf_lo(xw[q]), bf_lo(aw[q]), acc);
            acc = fmaf(bf_hi(xw[q]), bf_hi(aw[q]), acc);
          }
        }
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) U[m][j] = rbf(acc);
  }
  __syncthreads();

  // y[m][G Ng + n] = bf16(y + bf16(bf16(B_g[n] . u[m]) * scaling)): one thread per output row
  for (int n = n_lo + threadIdx.x; n < n_hi; n += LORA_THREADS) {
    const __nv_bfloat16* br = Bg + (size_t)n * r;
    if (r <= 8) {   // the common ranks (lit-llama finetunes with r = 8) keep the row in registers
      float b[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = j < r ? bf2f(br[j]) : 0.f;
      for (int m = 0; m < mt; ++m) {
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < r) d = fmaf(b[j], U[m][j], d);
        __nv_bfloat16* yp = y + (size_t)row_of(m) * ldy + (size_t)G * Ng + n;
        *yp = f2bf(bf2f(*yp) + rbf(rbf(d) * scaling));
      }
    } else {
      for (int m = 0; m < mt; ++m) {
        float d = 0.f;
        for (int j = 0; j < r; ++j) d = fmaf(bf2f(br[j]), U[m][j], d);
        __nv_bfloat16* yp = y + (size_t)row_of(m) * ldy + (size_t)G * Ng + n;
        *yp = f2bf(bf2f(*yp) + rbf(rbf(d) * scaling));
      }
    }
  }
}

__global__ void __launch_bounds__(LORA_THREADS) lora_kernel(const __nv_bfloat16* __restrict__ A,
                                                            const __nv_bfloat16* __restrict__ Bw, float scaling, int r,
                                                            int n_groups, unsigned enabled, const __nv_bfloat16* x,
                                                            int ldx, const __nv_bfloat16* __restrict__ norm, float eps,
                                                            __nv_bfloat16* y, int ldy, int M, int N, int K, int nslices) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bg = blockIdx.x / nslices, slice = blockIdx.x % nslices;
  int s = 0, G = -1;   // G: the bg-th enabled group
  while (s <= bg) {
    ++G;
    if ((enabled >> G) & 1u) ++s;
  }
  const int Ng = N / n_groups;
  const int per = (Ng + nslices - 1) / nslices;
  const int n_lo = slice * per, n_hi = min(Ng, n_lo + per);
  const int m0 = blockIdx.y * LORA_MT, mt = min(LORA_MT, M - m0);
  const __nv_bfloat16* Ag = A + (size_t)bg * r * K;
  const __nv_bfloat16* Bg = Bw + (size_t)bg * Ng * r;
  lora_tile(Ag, Bg, scaling, r, G, Ng, x, ldx, norm, eps, y, ldy, mt, n_lo, n_hi, K, warp, lane,
            [m0](int m) { return m0 + m; });
}

// The per-set fields of b2l_lora_apply_rows' terms, passed by value (a captured graph keeps its own copy).
struct LoraSets {
  const __nv_bfloat16* A[B2L_LORA_MAX_SETS];
  const __nv_bfloat16* B[B2L_LORA_MAX_SETS];
  float scaling[B2L_LORA_MAX_SETS];
  int r[B2L_LORA_MAX_SETS];   // 0: the set has no term here (a layer b2l_decode_step's lora_sets leave out)
  unsigned enabled[B2L_LORA_MAX_SETS];
};

// Grid: (enabled group of any set, slice) x (row slot m).  Slot m runs when row m is the first row of its set, and
// then takes every row of that set (at most M <= LORA_MT), so each set's lora_A / lora_B stream once per slice
// whatever the rows share.  row_set is read before griddepcontrol.wait: it must not be written by the launch this
// one overlaps (in the decode step it is copied in before the step begins).
__global__ void __launch_bounds__(LORA_THREADS) lora_rows_kernel(const __grid_constant__ LoraSets sets, int n_sets,
                                                                 const int32_t* row_set, int n_groups, unsigned any_on,
                                                                 const __nv_bfloat16* x, int ldx,
                                                                 const __nv_bfloat16* __restrict__ norm, float eps,
                                                                 __nv_bfloat16* y, int ldy, int M, int N, int nslices,
                                                                 int K) {
  __shared__ int rows[LORA_MT];
  const int bg = blockIdx.x / nslices, slice = blockIdx.x % nslices;
  int G = -1;   // the bg-th group enabled in some set
  for (int s = 0; s <= bg;) {
    ++G;
    if ((any_on >> G) & 1u) ++s;
  }
  auto set_of = [&](int m) {   // an entry outside -1..n_sets-1 is treated as -1
    const int s = row_set[m];
    return s >= 0 && s < n_sets ? s : -1;
  };
  const int slot = blockIdx.y, s = set_of(slot);
  if (s < 0 || sets.r[s] == 0 || !((sets.enabled[s] >> G) & 1u)) return;
  for (int m = 0; m < slot; ++m)
    if (set_of(m) == s) return;   // an earlier slot runs set s
  int mt = 0;
  for (int m = slot; m < M; ++m)
    if (set_of(m) == s) {
      if (threadIdx.x == 0) rows[mt] = m;
      ++mt;
    }
  __syncthreads();
  const int r = sets.r[s], Ng = N / n_groups;
  const int gi = __popc(sets.enabled[s] & ((1u << G) - 1u));   // G's place among the set's enabled groups
  const int per = (Ng + nslices - 1) / nslices;
  const int n_lo = slice * per, n_hi = min(Ng, n_lo + per);
  lora_tile(sets.A[s] + (size_t)gi * r * K, sets.B[s] + (size_t)gi * Ng * r, sets.scaling[s], r, G, Ng, x, ldx, norm,
            eps, y, ldy, mt, n_lo, n_hi, K, threadIdx.x >> 5, threadIdx.x & 31, [](int m) { return rows[m]; });
}

// Shape / pointer checks shared with b2l_decode_step (N, K: the linear's out / in features).
int check_lora(const b2l_lora* lo, int N, int K, const char* who) {
  B2L_CHECK_ARG(lo != nullptr && lo->A != nullptr && lo->B != nullptr, "%s: null LoRA weights", who);
  B2L_CHECK_SUPPORTED(lo->r >= 1 && lo->r <= B2L_LORA_MAX_R, "%s: LoRA rank %d unsupported (1..%d)", who, lo->r,
                      B2L_LORA_MAX_R);
  B2L_CHECK_SUPPORTED(lo->n_groups >= 1 && lo->n_groups <= 32 && N > 0 && N % lo->n_groups == 0,
                      "%s: LoRA n_groups %d must be 1..32 and divide N = %d", who, lo->n_groups, N);
  B2L_CHECK_SUPPORTED(lo->enabled != 0 && (lo->n_groups == 32 || (lo->enabled >> lo->n_groups) == 0),
                      "%s: LoRA enabled-group mask 0x%x invalid for %d groups", who, lo->enabled, lo->n_groups);
  B2L_CHECK_SUPPORTED(K >= 8 && K % 8 == 0, "%s: LoRA in_features %d must be a positive multiple of 8", who, K);
  B2L_CHECK_ARG(((uintptr_t)lo->A & 15) == 0, "%s: lora_A must be 16-byte aligned", who);
  B2L_CHECK_ARG(((uintptr_t)lo->B & 1) == 0, "%s: lora_B must be 2-byte aligned", who);
  B2L_CHECK_ARG(lo->scaling == lo->scaling && lo->scaling - lo->scaling == 0.f, "%s: LoRA scaling is not finite", who);
  return 0;
}

// The terms of a per-row call: set s is sets[s * stride] (b2l_decode_step's lora_sets hold one set per n_layer
// entries).  Every set with a term passes check_lora and all of them share n_groups; with empty_ok an entry with
// r == 0 stands for "no term" (a layer a decode-step set leaves out).  *any_on: the union of the enabled-group masks
// (0 when no set has a term); *n_groups: their shared group count.
int check_lora_sets(const b2l_lora* sets, size_t stride, int n_sets, int N, int K, bool empty_ok, unsigned* any_on,
                    int* n_groups, const char* who) {
  B2L_CHECK_ARG(sets != nullptr, "%s: null LoRA sets", who);
  B2L_CHECK_SUPPORTED(n_sets >= 1 && n_sets <= B2L_LORA_MAX_SETS, "%s: %d LoRA sets unsupported (1..%d)", who, n_sets,
                      B2L_LORA_MAX_SETS);
  unsigned on = 0;
  int ng = 0;
  for (int s = 0; s < n_sets; ++s) {
    const b2l_lora& lo = sets[(size_t)s * stride];
    if (empty_ok && lo.r == 0) continue;
    if (int rc = check_lora(&lo, N, K, who)) return rc;
    B2L_CHECK_ARG(ng == 0 || lo.n_groups == ng, "%s: LoRA set %d has %d groups, an earlier set %d (n_groups must match)",
                  who, s, lo.n_groups, ng);
    ng = lo.n_groups;
    on |= lo.enabled;
  }
  *any_on = on;
  *n_groups = ng;
  return 0;
}

// b2l_lora_apply_rows, and each LoRA layer of b2l_decode_step under lora_sets (empty_ok): checks, then one launch of
// lora_rows_kernel, or none when no set has a term.
int lora_rows(const b2l_lora* sets, size_t stride, int n_sets, bool empty_ok, const int32_t* row_set, const void* x,
              int ldx, const void* norm_scale, float eps, void* y, int ldy, int M, int N, int K, int flags,
              b2l_stream_t stream, const char* who) {
  B2L_CHECK_ARG(row_set != nullptr, "%s: null row_set", who);
  B2L_CHECK_SUPPORTED(M >= 1 && M <= LORA_MT, "%s: M = %d rows unsupported (1..%d)", who, M, LORA_MT);
  unsigned any_on = 0;
  int n_groups = 0;
  if (int rc = check_lora_sets(sets, stride, n_sets, N, K, empty_ok, &any_on, &n_groups, who)) return rc;
  B2L_CHECK_ARG(x != nullptr && y != nullptr, "%s: null x / y", who);
  B2L_CHECK_ARG(ldx >= K && ldx % 8 == 0 && ldy >= N, "%s: bad ldx / ldy (ldx=%d ldy=%d)", who, ldx, ldy);
  B2L_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)norm_scale & 15) == 0 && ((uintptr_t)y & 1) == 0,
                "%s: x and norm_scale must be 16-byte aligned", who);
  B2L_CHECK_ARG((flags & ~B2L_F_PDL) == 0, "%s: unknown flags 0x%x", who, flags);
  if (any_on == 0) return 0;
  LoraSets ls{};
  for (int s = 0; s < n_sets; ++s) {
    const b2l_lora& lo = sets[(size_t)s * stride];
    ls.A[s] = (const __nv_bfloat16*)lo.A;
    ls.B[s] = (const __nv_bfloat16*)lo.B;
    ls.scaling[s] = lo.scaling;
    ls.r[s] = lo.r;
    ls.enabled[s] = lo.enabled;
  }
  // b2l_lora_apply's slicing with one slot per set a row may use in place of its M tiles
  const int n_on = __builtin_popcount(any_on), slots = std::min(M, n_sets);
  const int Ng = N / n_groups;
  const int max_slices = (Ng + LORA_THREADS - 1) / LORA_THREADS;
  const int want = (2 * sm_count() + n_on * slots - 1) / (n_on * slots);
  const int nslices = std::max(1, std::min(max_slices, want));
  LaunchCfg lc(dim3((unsigned)(n_on * nslices), (unsigned)M), dim3(LORA_THREADS), 0, (cudaStream_t)stream,
               (flags & B2L_F_PDL) != 0);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, lora_rows_kernel, ls, n_sets, row_set, n_groups, any_on, (const __nv_bfloat16*)x,
                              ldx, (const __nv_bfloat16*)norm_scale, eps, (__nv_bfloat16*)y, ldy, M, N, nslices, K));
  return 0;
}

}  // namespace b2l

using namespace b2l;

extern "C" int b2l_lora_apply(const b2l_lora* lora, const void* x, int ldx, const void* norm_scale, float eps, void* y,
                              int ldy, int M, int N, int K, int flags, b2l_stream_t stream) {
  if (int rc = check_lora(lora, N, K, "b2l_lora_apply")) return rc;
  B2L_CHECK_ARG(x != nullptr && y != nullptr, "b2l_lora_apply: null x / y");
  B2L_CHECK_ARG(M >= 0 && ldx >= K && ldx % 8 == 0 && ldy >= N, "b2l_lora_apply: bad M / ldx / ldy (M=%d ldx=%d ldy=%d)",
                M, ldx, ldy);
  B2L_CHECK_ARG(((uintptr_t)x & 15) == 0 && ((uintptr_t)norm_scale & 15) == 0 && ((uintptr_t)y & 1) == 0,
                "b2l_lora_apply: x and norm_scale must be 16-byte aligned");
  B2L_CHECK_ARG((flags & ~B2L_F_PDL) == 0, "b2l_lora_apply: unknown flags 0x%x", flags);
  const int mtiles = (M + LORA_MT - 1) / LORA_MT;
  B2L_CHECK_SUPPORTED(mtiles <= 65535, "b2l_lora_apply: M = %d too large", M);
  if (M == 0) return 0;
  const int n_on = __builtin_popcount(lora->enabled);
  const int Ng = N / lora->n_groups;
  const int max_slices = (Ng + LORA_THREADS - 1) / LORA_THREADS;
  const int want = (2 * sm_count() + n_on * mtiles - 1) / (n_on * mtiles);
  const int nslices = std::max(1, std::min(max_slices, want));
  LaunchCfg lc(dim3((unsigned)(n_on * nslices), (unsigned)mtiles), dim3(LORA_THREADS), 0, (cudaStream_t)stream,
               (flags & B2L_F_PDL) != 0);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, lora_kernel, (const __nv_bfloat16*)lora->A, (const __nv_bfloat16*)lora->B,
                              lora->scaling, lora->r, lora->n_groups, lora->enabled, (const __nv_bfloat16*)x, ldx,
                              (const __nv_bfloat16*)norm_scale, eps, (__nv_bfloat16*)y, ldy, M, N, K, nslices));
  return 0;
}

extern "C" int b2l_lora_apply_rows(const b2l_lora* sets, int n_sets, const int32_t* row_set, const void* x, int ldx,
                                   const void* norm_scale, float eps, void* y, int ldy, int M, int N, int K, int flags,
                                   b2l_stream_t stream) {
  return lora_rows(sets, 1, n_sets, false, row_set, x, ldx, norm_scale, eps, y, ldy, M, N, K, flags, stream,
                   "b2l_lora_apply_rows");
}

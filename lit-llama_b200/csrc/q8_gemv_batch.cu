// LLM.int8() linear for 2..16 activation rows (batched decode on the whole-token step), fused with its neighbours of
// Block.forward as b2l_q8_linear is: [RMSNorm ->] Linear8bitLt [-> v2 affine] [-> residual | SwiGLU], reading CB / SCB
// in place.
//
// Replaces the module path at B >= 2: b2l_rmsnorm -> b2l_q8_gemm (b2l_q8_outlier_mask over all rows,
// q8_rowquant_kernel, q8_gemm_kernel) [-> b2l_linear_affine] [-> b2l_add | second b2l_q8_gemm + b2l_silu_mul].  Every
// output is bit-identical to it:
//   x^      = b2l_rmsnorm(x) with its 256-thread chunking and reduction order (the prologue of q8_gemv_kernel<.., true>)
//   mask    = one outlier mask for the batch: bit k set iff any row has |fp16(x^[m][k])| >= threshold
//   SCA[m]  = max over inlier columns of |fp16(x^[m])|, CA[m] = clamp(rint(fp16(x^) * (127 / SCA)), +-127), 0 on outliers
//   y       = q8_dequant(CA . CB[o], SCA, SCB) [+ the outlier columns' fp16 term, fmaf in ascending k] (q8_common.cuh)
//   then the module sequence's bf16 roundings: the store, the affine, then the residual add or silu(y1) * y2.
// The int32 contraction is exact, so its order does not matter.
//
// Two launches:
//   1. q8_batch_prep_kernel, one CTA per row, the M CTAs one thread-block cluster.  Each normalises its row into
//      shared memory and builds the row's outlier mask; the cluster ORs the M masks through distributed shared memory
//      (exact in any order), then each CTA writes its SCA, its CA in mma.m16n8k32 B-fragment order and its fp16 x^ on
//      the outlier columns, and rank 0 the ascending outlier column list.  Everything goes to a workspace that stays in
//      L2.  The conversion is done once here, not once per GEMV CTA.
//   2. q8_gemv_batch_kernel: q8_gemv_kernel's WS_CB skeleton -- persistent CTAs over 16-row blocks and the full K, one
//      bulk copy per CB row into the 1040-byte-pitch ring, ldmatrix.x4 A fragments -- with token n as column n of the
//      MMA: lane (g, t) feeds token g (group G: token 8 G + g), so M <= 8 costs one IMMA per 16 x 32 tile like batch 1
//      and M = 9..16 two.  Each stage's CA slice (8 k blocks x M tokens x 128 B) is streamed next to its weights with
//      one bulk copy.  The ring's weight copies are issued before griddepcontrol.wait, the CA copies after it.  Four
//      epilogue warps (thread = one row x tokens tg, tg + 8) compute the outlier term while the consumers contract the
//      unit, then dequantise, apply the affine and the residual / SwiGLU epilogue and store.
//
// Workspace (b2l_q8_linear_batch_workspace_bytes(K, M)): CA [K/128 k blocks][M tokens][4 t][32 B] | SCA fp32 [16] |
// n_outliers int32 (+ pad to 16 B) | outlier columns int32 [K] | fp16 x^ on the outlier columns [M][K].
#include <cooperative_groups.h>
#include <cuda_fp16.h>

#include "b2l_common.cuh"
#include "q8_common.cuh"

namespace cg = cooperative_groups;

namespace b2l {
namespace q8mb {

constexpr int MAXB = 16;
constexpr int RB = 16;
constexpr int KB = 128;                          // k per k block (4 IMMAs of k32)
constexpr int NCW = 8;                           // consumer warps, one k block each per stage
constexpr int KBP = NCW;                         // k blocks per stage
constexpr int ROW_PITCH = KBP * KB + 16;         // as q8_gemv_kernel WS_CB: conflict-free ldmatrix
constexpr uint32_t WSTAGE = RB * ROW_PITCH;      // weights of a stage (16 rows)
constexpr int PRODUCER_WARP = NCW;
constexpr int NEW = 4;                           // epilogue warps
constexpr int NTHREADS = (NCW + 1 + NEW) * 32;
constexpr int NBAR = (NCW + NEW) * 32;           // consumers + epilogue warps at the named barriers
constexpr int MAX_STAGES = 8;
constexpr int MAX_K = 32768;
constexpr int SST = MAXB + 1;                    // scratch ints per row (odd: no bank conflicts)
constexpr int PREP_THREADS = 256;                // b2l_rmsnorm's thread count: its chunking and reduction order

__host__ __device__ inline uint32_t ca_kb_bytes(int M) { return (uint32_t)M * 128; }   // one k block of CA
__host__ __device__ inline uint32_t stage_bytes(int M) { return WSTAGE + KBP * ca_kb_bytes(M); }
__host__ __device__ inline size_t ws_sca(int K, int M) { return (size_t)M * K; }
__host__ __device__ inline size_t ws_nout(int K, int M) { return ws_sca(K, M) + MAXB * 4; }
__host__ __device__ inline size_t ws_cols(int K, int M) { return ws_nout(K, M) + 16; }
__host__ __device__ inline size_t ws_xo(int K, int M) { return ws_cols(K, M) + (size_t)K * 4; }
__host__ __device__ inline size_t ws_bytes(int K, int M) { return ws_xo(K, M) + (size_t)M * K * 2; }

// coherent loads of what the prep launch wrote (PDL: griddepcontrol.wait orders coherent loads only)
__device__ __forceinline__ uint32_t ld_coherent_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_coherent_f16(const __half* p) {
  unsigned short v;
  asm volatile("ld.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return __half2float(__ushort_as_half(v));
}

// ---------------------------------------------------------------- step 1: rows -> CA, SCA and the outlier data
// Dynamic shared memory: fp16 x^ [K] | the row's mask [K/32] | the batch's mask [K/32].
__global__ void __launch_bounds__(PREP_THREADS) q8_batch_prep_kernel(const __nv_bfloat16* x, int M, int K,
                                                                     const __nv_bfloat16* __restrict__ norm_scale, float eps,
                                                                     float threshold, uint8_t* __restrict__ ws) {
  extern __shared__ __align__(16) uint8_t psmem[];
  __shared__ float red[NCW];
  __shared__ int wtot[NCW];
  cg::cluster_group cluster = cg::this_cluster();
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NT = PREP_THREADS;
  const int nwords = K / 32;
  __half* ah = reinterpret_cast<__half*>(psmem);
  uint32_t* rmask = reinterpret_cast<uint32_t*>(psmem + (size_t)K * 2);
  uint32_t* bmask = rmask + nwords;
  pdl_launch_dependents();   // the linear may start streaming its weights
  const __nv_bfloat16* xr = x + (size_t)n * K;
  // RMSNorm exactly as q8_gemv_kernel's FUSED prologue (b2l_rmsnorm's order): the scale staged in `ah` before the
  // dependency, each thread later overwriting exactly the chunks it staged
  if (norm_scale != nullptr)
    for (int k = tid * 8; k < K; k += NT * 8) *reinterpret_cast<uint4*>(ah + k) = *reinterpret_cast<const uint4*>(norm_scale + k);
  for (int i = tid; i < nwords; i += NT) rmask[i] = 0u;
  pdl_wait();
  float rinv = 0.f;
  if (norm_scale != nullptr) {
    float ss = 0.f;
    for (int k = tid * 8; k < K; k += NT * 8) {
      const uint4 v = ld_coherent_u4(xr + k);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float lo = __uint_as_float(w[q] << 16), hi = __uint_as_float(w[q] & 0xffff0000u);
        ss += rbf(lo * lo) + rbf(hi * hi);
      }
    }
    ss = warp_sum(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    ss = warp_sum(lane < NCW ? red[lane] : 0.f);
    rinv = rms_rinv(ss, K, eps);
  }
  __syncthreads();   // rmask cleared (and red read) before it is written below
  for (int k = tid * 8; k < K; k += NT * 8) {
    uint4 u = ld_coherent_u4(xr + k);
    if (norm_scale != nullptr) {
      const uint4 g = *reinterpret_cast<const uint4*>(ah + k);
      const uint32_t xw[4] = {u.x, u.y, u.z, u.w}, gw[4] = {g.x, g.y, g.z, g.w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        o[q] = pack_bf16x2(rms_apply(__uint_as_float(xw[q] << 16), rinv, __uint_as_float(gw[q] << 16)),
                           rms_apply(__uint_as_float(xw[q] & 0xffff0000u), rinv, __uint_as_float(gw[q] & 0xffff0000u)));
      u = make_uint4(o[0], o[1], o[2], o[3]);
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
      if (fabsf(__half2float(hv[e])) >= threshold) outl |= 1u << e;
    *reinterpret_cast<uint4*>(ah + k) = *reinterpret_cast<const uint4*>(hv);
    if (outl) atomicOr(&rmask[k >> 5], outl << (k & 31));
  }
  // the batch's mask: OR of the M row masks, read from every CTA of the cluster
  cluster.sync();
  for (int i = tid; i < nwords; i += NT) {
    uint32_t m = 0u;
    for (int r = 0; r < M; ++r) m |= *cluster.map_shared_rank(rmask + i, r);
    bmask[i] = m;
  }
  cluster.sync();   // no CTA leaves (or reuses rmask) while another still reads it
  // SCA and CA as q8_gemv_kernel / q8_rowquant_kernel
  float amax = 0.f;
  for (int k = tid * 8; k < K; k += NT * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(ah + k);
    const __half* hv = reinterpret_cast<const __half*>(&u);
    const uint32_t mb = (bmask[k >> 5] >> (k & 31)) & 0xFFu;
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (!((mb >> e) & 1u)) amax = fmaxf(amax, fabsf(__half2float(hv[e])));
  }
  amax = warp_max(amax);
  if (lane == 0) red[warp] = amax;
  __syncthreads();
  float sca = 0.f;
#pragma unroll
  for (int w = 0; w < NCW; ++w) sca = fmaxf(sca, red[w]);
  const float qs = sca > 0.f ? 127.0f / sca : 0.f;
  const uint32_t CAKB = ca_kb_bytes(M);
  for (int k = tid * 8; k < K; k += NT * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(ah + k);
    const __half* hv = reinterpret_cast<const __half*>(&u);
    const uint32_t mb = (bmask[k >> 5] >> (k & 31)) & 0xFFu;
    uint32_t pk[2] = {0u, 0u};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      int qv = ((mb >> e) & 1u) ? 0 : __float2int_rn(__half2float(hv[e]) * qs);
      qv = max(-127, min(127, qv));
      pk[e >> 2] |= (uint32_t)(qv & 0xFF) << (8 * (e & 3));
    }
    // k..k+3 -> lane t = (k % 16) / 4, half = (k % 32) / 16, chunk c32 = (k % 128) / 32; k+4..k+7 -> t + 1
    const int kb = k >> 7, c32 = (k >> 5) & 3, half = (k >> 4) & 1, t0 = (k >> 2) & 3;
    uint32_t* dst = reinterpret_cast<uint32_t*>(ws + (size_t)kb * CAKB + (size_t)n * 128);
    dst[t0 * 8 + c32 * 2 + half] = pk[0];
    dst[(t0 + 1) * 8 + c32 * 2 + half] = pk[1];
  }
  // outlier columns in ascending order: thread i owns mask words 4i .. 4i + 3; exclusive scan of their bit counts
  int cnt = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (tid * 4 + q < nwords) cnt += __popc(bmask[tid * 4 + q]);
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) wtot[warp] = incl;
  __syncthreads();
  int base = incl - cnt, total = 0;
#pragma unroll
  for (int w = 0; w < NCW; ++w) {
    if (w < warp) base += wtot[w];
    total += wtot[w];
  }
  int* cols = reinterpret_cast<int*>(ws + ws_cols(K, M));
  __half* xo = reinterpret_cast<__half*>(ws + ws_xo(K, M)) + (size_t)n * K;
  for (int q = 0; q < 4; ++q) {
    if (tid * 4 + q >= nwords) break;
    uint32_t mb = bmask[tid * 4 + q];
    while (mb) {
      const int k = (tid * 4 + q) * 32 + __ffs(mb) - 1;
      mb &= mb - 1;
      if (n == 0) cols[base] = k;
      xo[base] = ah[k];
      ++base;
    }
  }
  if (tid == 0) {
    reinterpret_cast<float*>(ws + ws_sca(K, M))[n] = sca;
    if (n == 0) *reinterpret_cast<int*>(ws + ws_nout(K, M)) = total;
  }
}

// ---------------------------------------------------------------- step 2: the streaming contraction
struct BParams {
  const int8_t* cb; const float* scb;
  const int8_t* cb2; const float* scb2;     // SWIGLU: rows 8..15 of every block
  const uint8_t* ca;                        // workspace
  const float* sca; const int* n_out; const int* cols; const __half* xo;
  __nv_bfloat16* y;                         // [M, N]
  const __nv_bfloat16* res;                 // RESIDUAL: [M, N]
  const __nv_bfloat16* aff_s; const __nv_bfloat16* aff_b;
  int M, N, K, n_rb, nst, epilogue;
};

struct BSmem {
  uint32_t ring, scratch, bars, total;
};
__host__ __device__ inline BSmem bsmem_layout(int nst, int M) {
  BSmem L;
  uint32_t o = 0;
  L.ring = o;    o += (uint32_t)nst * stage_bytes(M);
  L.scratch = o; o += (2u * RB * SST * 4 + 15u) & ~15u;   // [buf][16 rows][SST] int32 partials
  L.bars = o;    o += 2 * MAX_STAGES * 8;
  L.total = (o + 127u) & ~127u;
  return L;
}

// One output row of a 16-row block, as q8_gemv_kernel's FusedRow: SWIGLU rows 0..7 are outputs rb*8 .. rb*8+7 of cb,
// rows 8..15 the same outputs of cb2; the affine vectors are interleaved the same way (16 entries per block).
struct FusedRow {
  const int8_t* w;
  float scb, s, b;
  int col;
  bool valid;
};
__device__ __forceinline__ FusedRow fused_row(const BParams& p, int rb, int row) {
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

// NG = 1 (M <= 8) or 2 (M = 9..16) column groups of the MMA
template <int NG>
__global__ void __launch_bounds__(NTHREADS, 2) q8_gemv_batch_kernel(const BParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const BSmem L = bsmem_layout(p.nst, p.M);
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_kb = p.K / KB;
  const int spu = (n_kb + KBP - 1) / KBP;   // stages per unit
  const int rb_lo = (int)(((long long)blockIdx.x * p.n_rb) / gridDim.x);
  const int rb_hi = (int)(((long long)(blockIdx.x + 1) * p.n_rb) / gridDim.x);
  const int n_units = rb_hi - rb_lo;
  const int total_stages = n_units * spu;
  const uint32_t bar_full = sbase + L.bars, bar_empty = bar_full + MAX_STAGES * 8;
  const uint32_t SB = stage_bytes(p.M), CAKB = ca_kb_bytes(p.M);
  const bool glu = p.epilogue == B2L_EPI_SWIGLU;

  if (tid == 0) {
    for (int i = 0; i < p.nst; ++i) {
      mbar_init(bar_full + i * 8, 1);
      mbar_init(bar_empty + i * 8, NCW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // lanes 0..15: one bulk copy per weight row (SWIGLU: lanes 0..7 rows of cb, 8..15 the same rows of cb2); lane 0:
    // the barriers and the stage's CA slice
    const int per = glu ? 8 : RB, i = glu ? (lane & 7) : lane;
    const int pre = min(total_stages, p.nst);   // stages whose weights are requested before the dependency resolves
    for (int it = 0; it < total_stages; ++it) {
      const int u = it / spu, s = it - u * spu;
      const int slot = it % p.nst;
      const uint32_t phase = ((uint32_t)(it / p.nst) & 1u) ^ 1u;   // fresh barriers: parity 1 passes immediately
      const int row0 = (rb_lo + u) * per, nrows = min(per, p.N - row0);
      const int nkb = min(KBP, n_kb - s * KBP);
      const uint32_t row_bytes = (uint32_t)nkb * KB, xbytes = (uint32_t)nkb * CAKB;
      const uint32_t stage = sbase + L.ring + slot * SB;
      if (lane == 0) {
        mbar_wait(bar_empty + slot * 8, phase);
        mbar_expect_tx(bar_full + slot * 8, (uint32_t)(glu ? 2 : 1) * nrows * row_bytes + xbytes);
      }
      __syncwarp();
      if (lane < RB && i < nrows)
        tma_bulk_g2s(stage + lane * ROW_PITCH, ((glu && lane >= 8) ? p.cb2 : p.cb) + (size_t)(row0 + i) * p.K + (size_t)s * KBP * KB,
                     row_bytes, bar_full + slot * 8);
      if (lane == 0) {
        if (it >= pre) {
          tma_bulk_g2s(stage + WSTAGE, p.ca + (size_t)s * KBP * CAKB, xbytes, bar_full + slot * 8);
        } else if (it + 1 == pre) {
          // ring full of weights: let the next kernel in, wait for the prep launch, then request the CA slices of
          // every stage issued so far
          pdl_launch_dependents();
          pdl_wait();
          // CA was written with ordinary stores by the previous grid and is read by the async proxy
          asm volatile("fence.proxy.async;" ::: "memory");
          for (int j = 0; j < pre; ++j) {
            const int sj = j % spu;
            const int nkbj = min(KBP, n_kb - sj * KBP);
            tma_bulk_g2s(sbase + L.ring + (j % p.nst) * SB + WSTAGE, p.ca + (size_t)sj * KBP * CAKB, (uint32_t)nkbj * CAKB,
                         bar_full + (j % p.nst) * 8);
          }
        }
      }
    }
    if (total_stages == 0 && lane == 0) pdl_launch_dependents();
  } else if (warp < NCW) {
    // ===================== consumer warps: warp w takes k block w of every stage =====================
    const int g = lane >> 2, t4 = lane & 3;
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    // lane i addresses row i % 8 of ldmatrix matrix j = i / 8 (q8_gemv_kernel WS_CB)
    const uint32_t lm_row = (uint32_t)((lane & 7) + 8 * ((lane >> 3) & 1)) * ROW_PITCH;
    const uint32_t lm_unit = (uint32_t)(lane >> 4);
    int slot = 0;
    uint32_t phase = 0;
    for (int u = 0; u < n_units; ++u) {
      int acc[NG][2][4];
#pragma unroll
      for (int G = 0; G < NG; ++G)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[G][h][e] = 0;
      for (int s = 0; s < spu; ++s) {
        const int nkb = min(KBP, n_kb - s * KBP);
        mbar_wait(bar_full + slot * 8, phase);
        if (warp < nkb) {
          const uint8_t* xs = smem + L.ring + slot * SB + WSTAGE + warp * CAKB + t4 * 32;
          uint32_t bb[NG][8];
#pragma unroll
          for (int G = 0; G < NG; ++G) {
            uint4 xa = make_uint4(0, 0, 0, 0), xb = xa;
            if (8 * G + g < p.M) {   // token 8 G + g; zero columns past M
              xa = *reinterpret_cast<const uint4*>(xs + (8 * G + g) * 128);
              xb = *reinterpret_cast<const uint4*>(xs + (8 * G + g) * 128 + 16);
            }
            bb[G][0] = xa.x; bb[G][1] = xa.y; bb[G][2] = xa.z; bb[G][3] = xa.w;
            bb[G][4] = xb.x; bb[G][5] = xb.y; bb[G][6] = xb.z; bb[G][7] = xb.w;
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const uint4 a = ldmatrix_x4(sbase + L.ring + slot * SB + lm_row + warp * KB + (2 * c + lm_unit) * 16);
#pragma unroll
            for (int G = 0; G < NG; ++G) mma_s8s8_16832(acc[G][c & 1], a, bb[G][2 * c], bb[G][2 * c + 1]);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + slot * 8);
        if (++slot == p.nst) { slot = 0; phase ^= 1; }
      }
      // lane (g, t) holds rows g (e = 0, 1) and g + 8 (e = 2, 3) of tokens 8 G + 2 t (+1); exact integer atomics
      const int buf = u & 1;
      if (buf) bar_sync_c<5>(NBAR); else bar_sync_c<4>(NBAR);   // the epilogue has read and cleared this buffer
      int* sb = scratch + buf * RB * SST;
#pragma unroll
      for (int G = 0; G < NG; ++G) {
        const int col = 8 * G + 2 * t4;
        if (col < p.M) { atomicAdd(sb + g * SST + col, acc[G][0][0] + acc[G][1][0]); atomicAdd(sb + (g + 8) * SST + col, acc[G][0][2] + acc[G][1][2]); }
        if (col + 1 < p.M) { atomicAdd(sb + g * SST + col + 1, acc[G][0][1] + acc[G][1][1]); atomicAdd(sb + (g + 8) * SST + col + 1, acc[G][0][3] + acc[G][1][3]); }
      }
      __syncwarp();
      if (buf) bar_arrive_c<7>(NBAR); else bar_arrive_c<6>(NBAR);   // partials of this unit are in the buffer
    }
  } else {
    // ===================== epilogue warps: thread = row (e % 16) x tokens tg, tg + 8 (tg = e / 16) =====================
    const int e = tid - (NCW + 1) * 32;
    const int row = e & 15, tg = e >> 4;
    int* scratch = reinterpret_cast<int*>(smem + L.scratch);
    for (int i = e; i < 2 * RB * SST; i += NEW * 32) scratch[i] = 0;
    FusedRow fr{};
    if (n_units > 0) fr = fused_row(p, rb_lo, row);   // the first block's SCB and affine are weights: read before the dependency
    pdl_wait();
    const int M = p.M, K = p.K;
    const bool has1 = tg + 8 < M;
    const float sca0 = tg < M ? __uint_as_float(ld_coherent_u32(p.sca + tg)) : 0.f;
    const float sca1 = has1 ? __uint_as_float(ld_coherent_u32(p.sca + tg + 8)) : 0.f;
    const int n_out = (int)ld_coherent_u32(p.n_out);
    const __half* xo0 = p.xo + (size_t)min(tg, M - 1) * K;
    const __half* xo1 = p.xo + (size_t)(has1 ? tg + 8 : M - 1) * K;
    // both buffers start free (the clears above are ordered before the consumers' atomics by the barrier)
    if (n_units > 0) bar_arrive_c<4>(NBAR);
    if (n_units > 1) bar_arrive_c<5>(NBAR);
    for (int u = 0; u < n_units; ++u) {
      const int buf = u & 1;
      if (u > 0) fr = fused_row(p, rb_lo + u, row);
      // outlier term first (its loads overlap the consumers' work): fp16 weights, fp32 accumulate, k ascending
      float term0 = 0.f, term1 = 0.f;
      const float wsc = fr.scb / 127.0f;
#pragma unroll 4
      for (int j = 0; j < n_out; ++j) {
        const int k = (int)ld_coherent_u32(p.cols + j);
        const float wv = q8_outlier_weight(fr.w[k], wsc);
        term0 = fmaf(ld_coherent_f16(xo0 + j), wv, term0);
        if (has1) term1 = fmaf(ld_coherent_f16(xo1 + j), wv, term1);
      }
      if (buf) bar_sync_c<7>(NBAR); else bar_sync_c<6>(NBAR);
      int* sb = scratch + buf * RB * SST + row * SST;
      const int t0 = sb[tg], t1 = sb[tg + 8];
      sb[tg] = 0;
      sb[tg + 8] = 0;
      if (u + 2 < n_units) { if (buf) bar_arrive_c<5>(NBAR); else bar_arrive_c<4>(NBAR); }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int tok = tg + 8 * h;
        float v = q8_dequant(h ? t1 : t0, h ? sca1 : sca0, fr.scb);
        if (n_out > 0) v = q8_add_outliers(v, h ? term1 : term0);
        // the module path's bf16 output, then b2l_linear_affine, then b2l_add / b2l_silu_mul
        float yv = rbf(v);
        if (p.aff_s != nullptr) yv = rbf(affine1(yv, fr.s, fr.b));
        const bool ok = tok < M && fr.valid;
        __nv_bfloat16* yr = p.y + (size_t)min(tok, M - 1) * p.N;
        if (glu) {
          const float up = __shfl_down_sync(0xffffffffu, yv, 8);   // row r + 8: c_fc2's output of the same column
          if (row < 8 && ok) yr[fr.col] = f2bf(silu_mul1(yv, up));
        } else if (ok) {
          yr[fr.col] = f2bf(p.epilogue == B2L_EPI_RESIDUAL ? yv + ld_coherent_bf16(p.res + (size_t)tok * p.N + fr.col) : yv);
        }
      }
    }
  }
}

}  // namespace q8mb
}  // namespace b2l

using namespace b2l;
using namespace b2l::q8mb;

extern "C" size_t b2l_q8_linear_batch_workspace_bytes(int K, int M) {
  if (K <= 0 || K % KB != 0 || K > MAX_K || M < 2 || M > MAXB) return 0;
  return ws_bytes(K, M);
}

namespace {
template <int NG>
int launch_batch(BParams& p, bool pdl, cudaStream_t stream) {
  // two CTAs per SM (1 KB of each SM's 228 KB is reserved per CTA)
  const uint32_t budget = 110u * 1024u, fixed = bsmem_layout(0, p.M).total, sb = stage_bytes(p.M);
  int nst = (int)((budget - fixed) / sb);
  if (nst > MAX_STAGES) nst = MAX_STAGES;
  p.nst = nst;
  const BSmem L = bsmem_layout(nst, p.M);
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(q8_gemv_batch_kernel<NG>, L.total, smem_cache)) return rc;
  int grid = 2 * sm_count();
  if (grid > p.n_rb) grid = p.n_rb;
  LaunchCfg lc(dim3(grid), dim3(NTHREADS), L.total, stream, pdl, 1);
  B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q8_gemv_batch_kernel<NG>, p));
  return 0;
}
}  // namespace

namespace b2l {
int check_q8_disjoint(const b2l_q8_linear_args* a, int M, const char* who);   // q8_gemv.cu

// b2l_q8_linear_batch's argument checks: 0, or B2L_E_* with a message
int check_q8_linear_batch(const b2l_q8_linear_args* a, int M, const void* workspace, size_t workspace_bytes) {
  B2L_CHECK_ARG(a != nullptr && a->x && a->cb && a->scb && a->y, "b2l_q8_linear_batch: null pointer");
  B2L_CHECK_SUPPORTED(M >= 2 && M <= MAXB, "b2l_q8_linear_batch: M=%d (2..%d activation rows; use b2l_q8_linear for 1)", M, MAXB);
  const int N = a->N, K = a->K;
  B2L_CHECK_SUPPORTED(K > 0 && K % KB == 0 && K <= MAX_K, "b2l_q8_linear_batch: K=%d must be a multiple of %d and <= %d", K, KB, MAX_K);
  B2L_CHECK_ARG(N > 0, "b2l_q8_linear_batch: bad shape N=%d", N);
  B2L_CHECK_ARG(a->prologue == B2L_PRO_NONE || a->prologue == B2L_PRO_RMSNORM, "b2l_q8_linear_batch: bad prologue %d", a->prologue);
  B2L_CHECK_ARG(a->epilogue == B2L_EPI_STORE || a->epilogue == B2L_EPI_RESIDUAL || a->epilogue == B2L_EPI_SWIGLU,
                "b2l_q8_linear_batch: bad epilogue %d", a->epilogue);
  const bool norm = a->prologue == B2L_PRO_RMSNORM, glu = a->epilogue == B2L_EPI_SWIGLU;
  B2L_CHECK_ARG(!norm || a->norm_scale, "b2l_q8_linear_batch: RMSNORM needs norm_scale");
  B2L_CHECK_ARG(a->epilogue != B2L_EPI_RESIDUAL || a->res, "b2l_q8_linear_batch: RESIDUAL needs res");
  B2L_CHECK_ARG(!glu || (a->cb2 && a->scb2), "b2l_q8_linear_batch: SWIGLU needs cb2 and scb2");
  B2L_CHECK_ARG((a->out_affine.scale == nullptr) == (a->out_affine.bias == nullptr),
                "b2l_q8_linear_batch: out_affine needs both scale and bias (or neither)");
  B2L_CHECK_ARG(workspace != nullptr, "b2l_q8_linear_batch: null workspace (b2l_q8_linear_batch_workspace_bytes(K, M) bytes)");
  B2L_CHECK_ARG(((uintptr_t)a->x | (uintptr_t)a->cb | (uintptr_t)(glu ? a->cb2 : nullptr) |
                 (uintptr_t)(norm ? a->norm_scale : nullptr) | (uintptr_t)workspace) % 16 == 0,
                "b2l_q8_linear_batch: x / cb / cb2 / norm_scale / workspace must be 16-byte aligned");
  B2L_CHECK_ARG(workspace_bytes >= ws_bytes(K, M), "b2l_q8_linear_batch: workspace of %zu bytes is too small (%zu needed)",
                workspace_bytes, ws_bytes(K, M));
  B2L_CHECK_SUPPORTED((a->flags & ~B2L_F_PDL) == 0, "b2l_q8_linear_batch: unknown flags 0x%x (only B2L_F_PDL)", (unsigned)a->flags);
  return 0;
}
}  // namespace b2l

extern "C" int b2l_q8_linear_batch(const b2l_q8_linear_args* a, int M, void* workspace, size_t workspace_bytes, b2l_stream_t stream) {
  if (int rc = check_q8_linear_batch(a, M, workspace, workspace_bytes)) return rc;
  if (int rc = check_q8_disjoint(a, M, "b2l_q8_linear_batch")) return rc;
  const int N = a->N, K = a->K;
  const bool norm = a->prologue == B2L_PRO_RMSNORM, glu = a->epilogue == B2L_EPI_SWIGLU;
  const cudaStream_t st = (cudaStream_t)stream;
  const bool pdl = (a->flags & B2L_F_PDL) != 0;
  uint8_t* ws = (uint8_t*)workspace;
  {
    const size_t smem = (size_t)K * 2 + (size_t)K / 32 * 4 * 2;
    static DynSmemCache smem_cache;
    if (int rc = ensure_dyn_smem(q8_batch_prep_kernel, smem, smem_cache)) return rc;
    static bool non_portable = [] {   // clusters of up to 16 CTAs (sm_90 allows them on request)
      return cudaFuncSetAttribute(q8_batch_prep_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess;
    }();
    if (!non_portable) {
      set_error("b2l_q8_linear_batch: clusters of 16 CTAs are not available on this device");
      return B2L_E_STATE;
    }
    LaunchCfg lc(dim3(M), dim3(PREP_THREADS), smem, st, pdl, M);
    B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, q8_batch_prep_kernel, (const __nv_bfloat16*)a->x, M, K,
                                norm ? (const __nv_bfloat16*)a->norm_scale : (const __nv_bfloat16*)nullptr, a->eps, a->threshold, ws));
  }
  BParams p{};
  p.cb = (const int8_t*)a->cb; p.scb = (const float*)a->scb;
  p.cb2 = (const int8_t*)a->cb2; p.scb2 = (const float*)a->scb2;
  p.ca = ws;
  p.sca = (const float*)(ws + ws_sca(K, M)); p.n_out = (const int*)(ws + ws_nout(K, M));
  p.cols = (const int*)(ws + ws_cols(K, M)); p.xo = (const __half*)(ws + ws_xo(K, M));
  p.y = (__nv_bfloat16*)a->y; p.res = (const __nv_bfloat16*)a->res;
  p.aff_s = (const __nv_bfloat16*)a->out_affine.scale; p.aff_b = (const __nv_bfloat16*)a->out_affine.bias;
  p.M = M; p.N = N; p.K = K;
  p.n_rb = glu ? (N + 7) / 8 : (N + RB - 1) / RB;
  p.epilogue = a->epilogue;
  return M <= 8 ? launch_batch<1>(p, pdl, st) : launch_batch<2>(p, pdl, st);
}

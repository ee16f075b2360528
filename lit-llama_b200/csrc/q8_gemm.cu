// LLM.int8() linear for M >= 2 activation rows (batched decode, prompts, no-cache windows) on the Hopper int8
// tensor cores: y[M, N] = int8linear(x[M, K]) against CB[N, K], bit-identical per row to b2l_q8_gemv with the batch's
// shared outlier mask (the arithmetic of q8_gemv.cu, restated here element by element).
//
// Replaces Linear8bitLt.forward (lit_llama/quantization.py:38-77 + the bitsandbytes MatMul8bitLt it inherits).
//
// Three launches, all on the caller's stream, everything in a caller-provided workspace:
//   1. b2l_q8_outlier_mask (q8_gemv.cu): bit k set iff any row has |fp16(x[m][k])| >= threshold;
//   2. q8_rowquant_kernel, one CTA per row: SCA[m] = max |fp16(x)| over the inlier columns,
//      CA[m][k] = clamp(rint(fp16(x) * (127 / SCA)), +-127), 0 on outlier columns (and for SCA = 0);
//   3. q8_gemm_kernel: one CTA computes a (64 NWG weight rows) x (BT tokens) tile of y over the full K.
//        warpgroups 0 .. NWG-1: wgmma.mma_async.m64nBTk32.s32.s8.s8, A = CB rows (weights on the M side, 64 rows per
//            warpgroup), B = CA rows (tokens on the N side), both K-major in shared memory (no-swizzle canonical
//            core-matrix layout [k16 chunk][row][16 B]); int32 accumulators in registers, exact (127^2 * 32768 < 2^31);
//        the producer warp: per 128-wide k stage two tensor-map TMA copies (weights straight from CB, tokens from CA)
//            into an mbarrier ring; CA is padded with zero rows to a whole token tile, rows beyond N are zero-filled
//            by the TMA unit;
//        epilogue: v = fp16(t * (SCA * SCB * (1/127^2))), plus fp16(sum over outlier k of fp16(x) * fp16(CB * SCB/127))
//            (fmaf, ascending k) when the batch has outlier columns, stored as bf16.  No atomics: each output is
//            written once by the thread that holds its accumulator.
// Weights sit on the wgmma M side so that one kernel serves 2-row decode batches (BT = 16) and 4096-row prompts
// (BT = 128): the token count only picks the N of the instruction.
#include <cuda_fp16.h>

#include "b2l_common.cuh"
#include "q8_common.cuh"

namespace b2l {
namespace q8gm {

constexpr int BK = 128;                        // k (bytes) per stage
constexpr int MAX_K = 32768;

// Token tile of the GEMM for M rows, and the rows of CA padded up to it.  A TMA box that reaches past the end of the
// tensor is zero-filled, but measured on an H100 that path made the small-M GEMM ~1.5x slower than a box of
// real zero rows.
static int token_tile(int M) { return M <= 16 ? 16 : 128; }
static int padded_rows(int M) { const int t = token_tile(M); return (M + t - 1) / t * t; }

template <int BT, int NWG>
struct Cfg {
  static constexpr int ROWS = 64 * NWG;                      // weight rows of the tile
  static constexpr int A_BYTES = ROWS * BK;                  // [8 k16 chunks][ROWS][16 B]
  static constexpr int B_BYTES = BT * BK;                    // [8 k16 chunks][BT][16 B]
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int NSTAGE = BT <= 16 ? 8 : 4;
  static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + 2 * NSTAGE * 8;
  static constexpr int NMMA = 128 * NWG;
  static constexpr int NTHREADS = NMMA + 32;                 // + one producer warp
  static constexpr int LBO_A = ROWS * 16, LBO_B = BT * 16, SBO = 128;
};

struct Params {
  CUtensorMap wmap;        // CB[N, K] as (16 B | N rows, stride K | K/16 chunks, stride 16 B); first member (64-byte alignment)
  CUtensorMap amap;        // CA[M, K], same view
  const __nv_bfloat16* x; int ldx;
  const int8_t* cb;
  const float* scb;
  const float* sca;        // [M]
  const uint32_t* mask;    // [K/32]
  __nv_bfloat16* y; int ldy;
  int M, N, K;
};

// D[64 x BT] (int32, registers) += A[64 x 32] (smem) * B[32 x BT] (smem), both K-major int8
template <int BT> __device__ __forceinline__ void wgmma_s8(int (&d)[BT / 2], uint64_t adesc, uint64_t bdesc);
template <> __device__ __forceinline__ void wgmma_s8<16>(int (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1;"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
      : "l"(adesc), "l"(bdesc)
      : "memory");
}
template <> __device__ __forceinline__ void wgmma_s8<128>(int (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, 1;"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc)
      : "memory");
}
template <int N> __device__ __forceinline__ void reg_fence(int (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

__device__ __forceinline__ float fp16_of_bf16(__nv_bfloat16 v) { return __half2float(__float2half_rn(bf2f(v))); }

// ---- prologue: one CTA per row
constexpr int RQ_THREADS = 256;
__global__ void __launch_bounds__(RQ_THREADS) q8_rowquant_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int M, int K, const uint32_t* __restrict__ mask,
                                                                  int8_t* __restrict__ ca, float* __restrict__ sca) {
  __shared__ float red[RQ_THREADS / 32];
  const int m = blockIdx.x, tid = threadIdx.x;
  if (m >= M) {   // padding rows up to the token tile: zeros, so the GEMM's TMA box never leaves the tensor
    for (int k = tid * 16; k < K; k += RQ_THREADS * 16) *reinterpret_cast<uint4*>(ca + (size_t)m * K + k) = make_uint4(0, 0, 0, 0);
    return;
  }
  const __nv_bfloat16* xr = x + (size_t)m * ldx;
  float amax = 0.f;
  for (int k = tid * 8; k < K; k += RQ_THREADS * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(xr + k);
    const __nv_bfloat16* v = reinterpret_cast<const __nv_bfloat16*>(&u);
    const uint32_t mb = (mask[k >> 5] >> (k & 31)) & 0xFFu;
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (!((mb >> e) & 1u)) amax = fmaxf(amax, fabsf(fp16_of_bf16(v[e])));
  }
  amax = warp_max(amax);
  if ((tid & 31) == 0) red[tid >> 5] = amax;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < RQ_THREADS / 32; ++w) s = fmaxf(s, red[w]);
  const float qs = s > 0.f ? 127.0f / s : 0.f;
  for (int k = tid * 8; k < K; k += RQ_THREADS * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(xr + k);
    const __nv_bfloat16* v = reinterpret_cast<const __nv_bfloat16*>(&u);
    const uint32_t mb = (mask[k >> 5] >> (k & 31)) & 0xFFu;
    uint32_t pk[2] = {0u, 0u};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      int qv = ((mb >> e) & 1u) ? 0 : __float2int_rn(fp16_of_bf16(v[e]) * qs);
      qv = max(-127, min(127, qv));
      pk[e >> 2] |= (uint32_t)(qv & 0xFF) << (8 * (e & 3));
    }
    *reinterpret_cast<uint2*>(ca + (size_t)m * K + k) = make_uint2(pk[0], pk[1]);
  }
  if (tid == 0) sca[m] = s;
}

template <int BT, int NWG>
__global__ void __launch_bounds__(Cfg<BT, NWG>::NTHREADS, 1) q8_gemm_kernel(const __grid_constant__ Params p) {
  using C = Cfg<BT, NWG>;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar_full = sbase + C::NSTAGE * C::STAGE_BYTES, bar_empty = bar_full + C::NSTAGE * 8;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * C::ROWS, m0 = blockIdx.y * BT;
  const int n_kt = p.K / BK;

  if (tid == 0) {
    for (int i = 0; i < C::NSTAGE; ++i) {
      mbar_init(bar_full + i * 8, 1);                 // the producer's expect_tx
      mbar_init(bar_empty + i * 8, C::NMMA / 32);     // one arrival per MMA warp once its wgmma group has completed
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < C::NMMA / 32) {
    // ===================== MMA warpgroups =====================
    const int h = warp >> 2;                          // weight rows 64 h .. 64 h + 63 of the tile
    int acc[BT / 2];
#pragma unroll
    for (int i = 0; i < BT / 2; ++i) acc[i] = 0;
    for (int kt = 0; kt < n_kt; ++kt) {
      const int st = kt % C::NSTAGE;
      mbar_wait(bar_full + st * 8, (uint32_t)(kt / C::NSTAGE) & 1u);
      const uint32_t a_base = sbase + st * C::STAGE_BYTES, b_base = a_base + C::A_BYTES;
      wgmma_fence();
      reg_fence(acc);
#pragma unroll
      for (int j = 0; j < BK / 32; ++j)
        wgmma_s8<BT>(acc, make_desc(a_base + h * 64 * 16 + j * 2 * C::LBO_A, C::LBO_A, C::SBO), make_desc(b_base + j * 2 * C::LBO_B, C::LBO_B, C::SBO));
      wgmma_commit();
      wgmma_wait<1>();   // the group of stage kt - 1 has completed
      reg_fence(acc);
      if (kt > 0 && lane == 0) mbar_arrive(bar_empty + ((kt - 1) % C::NSTAGE) * 8);
    }
    wgmma_wait<0>();
    reg_fence(acc);

    // ===================== epilogue.  acc[4 c + e]: weight row 16 (warp % 4) + lane / 4 (+ 8 for e >= 2),
    // token 8 c + 2 (lane % 4) + (e & 1)
    const int nwords = p.K / 32;
    bool any = false;                                 // the batch has outlier columns
    for (int wi = 0; wi < nwords && !any; ++wi) any = p.mask[wi] != 0u;
    const int nr = n0 + h * 64 + (warp & 3) * 16 + (lane >> 2);
    const int mc = m0 + 2 * (lane & 3);
    float scb[2], wsc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int n = min(nr + 8 * r, p.N - 1);
      scb[r] = p.scb[n];
      wsc[r] = scb[r] / 127.0f;
    }
#pragma unroll
    for (int c = 0; c < BT / 8; ++c) {
      const int mt = mc + 8 * c;
      if (mt >= p.M) continue;
      float sca[2];
      sca[0] = p.sca[mt];
      sca[1] = mt + 1 < p.M ? p.sca[mt + 1] : 0.f;
      float term[4] = {0.f, 0.f, 0.f, 0.f};          // [r][token]
      if (any) {
        const int t1 = min(mt + 1, p.M - 1);
        const __nv_bfloat16* x0 = p.x + (size_t)mt * p.ldx;
        const __nv_bfloat16* x1 = p.x + (size_t)t1 * p.ldx;
        const int8_t* w0 = p.cb + (size_t)min(nr, p.N - 1) * p.K;
        const int8_t* w1 = p.cb + (size_t)min(nr + 8, p.N - 1) * p.K;
        for (int wi = 0; wi < nwords; ++wi) {
          uint32_t mb = p.mask[wi];
          while (mb) {
            const int k = wi * 32 + __ffs(mb) - 1;
            mb &= mb - 1;
            const float a0 = fp16_of_bf16(x0[k]), a1 = fp16_of_bf16(x1[k]);
            const float wv0 = q8_outlier_weight(w0[k], wsc[0]);
            const float wv1 = q8_outlier_weight(w1[k], wsc[1]);
            term[0] = fmaf(a0, wv0, term[0]);
            term[1] = fmaf(a1, wv0, term[1]);
            term[2] = fmaf(a0, wv1, term[2]);
            term[3] = fmaf(a1, wv1, term[3]);
          }
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1, t = e & 1;
        const int n = nr + 8 * r, m = mt + t;
        if (n >= p.N || m >= p.M) continue;
        float v = q8_dequant(acc[4 * c + e], sca[t], scb[r]);
        if (any) v = q8_add_outliers(v, term[2 * r + t]);
        p.y[(size_t)m * p.ldy + n] = f2bf(v);
      }
    }
  } else if (lane == 0) {
    // ===================== producer: weights and quantised tokens by tensor-map TMA =====================
    for (int kt = 0; kt < n_kt; ++kt) {
      const int st = kt % C::NSTAGE;
      if (kt >= C::NSTAGE) mbar_wait(bar_empty + st * 8, (uint32_t)(kt / C::NSTAGE - 1) & 1u);
      const uint32_t a_base = sbase + st * C::STAGE_BYTES;
      mbar_expect_tx(bar_full + st * 8, C::STAGE_BYTES);
      tma_load_3d(a_base, &p.wmap, 0, n0, kt * (BK / 16), bar_full + st * 8);
      tma_load_3d(a_base + C::A_BYTES, &p.amap, 0, m0, kt * (BK / 16), bar_full + st * 8);
    }
  }
}

// int8 [rows, K] row-major as (16 B | rows, stride K | K/16 chunks, stride 16 B): a box of 16 x box_rows x 8 lands in
// shared memory as [k16 chunk][row][16 B], the no-swizzle K-major core-matrix order wgmma reads
static int encode_rows(PFN_cuTensorMapEncodeTiled encode, CUtensorMap* map, const void* base, int rows, int K, int box_rows) {
  const cuuint64_t dims[3] = {16, (cuuint64_t)rows, (cuuint64_t)(K / 16)};
  const cuuint64_t strides[2] = {(cuuint64_t)K, 16};
  const cuuint32_t box[3] = {16, (cuuint32_t)box_rows, (cuuint32_t)(BK / 16)};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult cr = encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("b2l_q8_gemm: cuTensorMapEncodeTiled failed (%d) for rows=%d K=%d", (int)cr, rows, K);
    return B2L_E_ARG;
  }
  return 0;
}

template <int BT, int NWG>
static int launch_gemm(Params& p, PFN_cuTensorMapEncodeTiled encode, const void* cb, const void* ca, cudaStream_t stream) {
  using C = Cfg<BT, NWG>;
  if (int rc = encode_rows(encode, &p.wmap, cb, p.N, p.K, C::ROWS)) return rc;
  if (int rc = encode_rows(encode, &p.amap, ca, padded_rows(p.M), p.K, BT)) return rc;
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(q8_gemm_kernel<BT, NWG>, C::SMEM_BYTES, smem_cache)) return rc;
  dim3 grid((p.N + C::ROWS - 1) / C::ROWS, (p.M + BT - 1) / BT);
  q8_gemm_kernel<BT, NWG><<<grid, C::NTHREADS, C::SMEM_BYTES, stream>>>(p);
  B2L_LAUNCH_CHECK("q8_gemm_kernel");
  return 0;
}

// workspace: CA int8 [padded_rows(M)][K] | SCA fp32 [M] (16-byte aligned) | outlier mask uint32 [K/32] (16-byte aligned)
static size_t sca_offset(int M, int K) { return (size_t)padded_rows(M) * K; }
static size_t mask_offset(int M, int K) { return sca_offset(M, K) + (((size_t)M * 4 + 15) & ~(size_t)15); }

}  // namespace q8gm
}  // namespace b2l

using namespace b2l;
using namespace b2l::q8gm;

extern "C" size_t b2l_q8_gemm_workspace_bytes(int M, int K) {
  if (M <= 0 || K <= 0 || K % BK != 0 || K > MAX_K) return 0;
  return mask_offset(M, K) + (size_t)K / 8;
}

extern "C" int b2l_q8_gemm(const void* x, int ldx, const void* cb, const void* scb, void* workspace, size_t workspace_bytes, void* y,
                           int ldy, int M, int N, int K, float threshold, int flags, b2l_stream_t stream) {
  B2L_CHECK_ARG(x && cb && scb && workspace && y, "b2l_q8_gemm: null pointer");
  B2L_CHECK_ARG(M > 0 && N > 0, "b2l_q8_gemm: bad shape M=%d N=%d", M, N);
  B2L_CHECK_SUPPORTED(K > 0 && K % BK == 0 && K <= MAX_K, "b2l_q8_gemm: K=%d must be a multiple of %d and <= %d", K, BK, MAX_K);
  B2L_CHECK_ARG(ldx >= K && ldx % 8 == 0 && ldy >= N, "b2l_q8_gemm: bad leading dimension (ldx >= K, ldx %% 8 == 0, ldy >= N)");
  B2L_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)cb % 16 == 0) && ((uintptr_t)workspace % 16 == 0),
                "b2l_q8_gemm: x / cb / workspace must be 16-byte aligned");
  B2L_CHECK_ARG(workspace_bytes >= b2l_q8_gemm_workspace_bytes(M, K), "b2l_q8_gemm: workspace of %zu bytes is too small (%zu needed)",
                workspace_bytes, b2l_q8_gemm_workspace_bytes(M, K));
  B2L_CHECK_SUPPORTED(flags == 0, "b2l_q8_gemm: flags must be 0");
  const PFN_cuTensorMapEncodeTiled encode = tensor_map_encoder();
  if (encode == nullptr) {
    set_error("b2l_q8_gemm: cuTensorMapEncodeTiled is not available from this driver");
    return B2L_E_STATE;
  }
  uint8_t* ws = (uint8_t*)workspace;
  int8_t* ca = (int8_t*)ws;
  float* sca = (float*)(ws + sca_offset(M, K));
  uint32_t* mask = (uint32_t*)(ws + mask_offset(M, K));
  const cudaStream_t st = (cudaStream_t)stream;
  if (int rc = b2l_q8_outlier_mask(x, ldx, M, K, threshold, mask, stream)) return rc;
  q8_rowquant_kernel<<<padded_rows(M), RQ_THREADS, 0, st>>>((const __nv_bfloat16*)x, ldx, M, K, mask, ca, sca);
  B2L_LAUNCH_CHECK("q8_rowquant_kernel");
  Params p;
  p.x = (const __nv_bfloat16*)x; p.ldx = ldx;
  p.cb = (const int8_t*)cb; p.scb = (const float*)scb;
  p.sca = sca; p.mask = mask;
  p.y = (__nv_bfloat16*)y; p.ldy = ldy;
  p.M = M; p.N = N; p.K = K;
  if (token_tile(M) == 16) return launch_gemm<16, 1>(p, encode, cb, ca, st);
  return launch_gemm<128, 2>(p, encode, cb, ca, st);
}

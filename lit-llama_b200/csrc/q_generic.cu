// Generic ColBlockQuantizedLinear kernels: read the reference storage directly
// (quantization.py:350-369): uint8 [in/epb][out] row-major, scales/zeros [out][n_groups].
// Any bits in {4,8}, any tile_cols, any M.  This is the always-correct path; the
// wgmma kernel in q4_tc.cu is the fast path for bits=4 / one group per row.
#include "b2l_common.cuh"

namespace b2l {

// ----------------------------------------------------------------------------------
// get_weight(): dense [out][in] = (level - zero) * scale, evaluated in the output
// dtype exactly as quantization.py:392-411 does (level stored in dtype, `-=` zeros in
// dtype, `*=` scales in dtype).
// ----------------------------------------------------------------------------------
template <int BITS, typename OutT>
__global__ void dequant_kernel(const uint8_t* __restrict__ qw, const void* __restrict__ scales,
                               const void* __restrict__ zeros, int szdt, OutT* __restrict__ w, int N,
                               int K, int tile_cols, int n_groups) {
  constexpr int EPB = 8 / BITS;
  constexpr int MASK = (1 << BITS) - 1;
  // tile: 32 packed rows (j) x 32 outputs (o); read coalesced along o, write along k
  __shared__ uint8_t tile[32][33];
  const int o0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const int Kp = K / EPB;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int j = j0 + r, o = o0 + threadIdx.x;
    tile[r][threadIdx.x] = (j < Kp && o < N) ? qw[(size_t)j * N + o] : 0;
  }
  __syncthreads();
  // each thread writes EPB consecutive k of one row o
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int o = o0 + r;
    int j = j0 + threadIdx.x;
    if (o >= N || j >= Kp) continue;
    uint8_t b = tile[threadIdx.x][r];
#pragma unroll
    for (int nr = 0; nr < EPB; ++nr) {
      int k = j * EPB + nr;
      int g = k / tile_cols;
      float lv = (float)((b >> (nr * BITS)) & MASK);
      float z = load_sz(zeros, szdt, (size_t)o * n_groups + g);
      float s = load_sz(scales, szdt, (size_t)o * n_groups + g);
      float v;
      if constexpr (sizeof(OutT) == 2) {
        v = rbf(rbf(lv - z) * s);
        w[(size_t)o * K + k] = f2bf(v);
      } else {
        v = (lv - z) * s;
        w[(size_t)o * K + k] = v;
      }
    }
  }
}

// ----------------------------------------------------------------------------------
// forward(): y[m][o] = sum_k x[m][k] * ((level[o][k] - zero[o][g]) * scale[o][g]) (+bias)
// fp32 dequant and accumulate - the arithmetic of the reference GPU kernel
// (quantization.py:259-269) - output rounded once to bf16.
//
// Block = 8 warps over one tile of 32*VEC outputs; warp w takes packed rows w, w+8, ...
// (a 128-byte coalesced row segment per warp when VEC == 4); lane owns VEC outputs.
// ----------------------------------------------------------------------------------
template <int BITS, int VEC, int MT>
__global__ void __launch_bounds__(256)
    q_linear_kernel(const __nv_bfloat16* __restrict__ x, int ldx, const uint8_t* __restrict__ qw,
                    const void* __restrict__ scales, const void* __restrict__ zeros, int szdt,
                    const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int ldy, int M,
                    int N, int K, int tile_cols, int n_groups, int k_splits) {
  constexpr int EPB = 8 / BITS;
  constexpr int MASK = (1 << BITS) - 1;
  constexpr int NW = 8;
  __shared__ float red[NW][MT][32 * VEC + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int o_base = blockIdx.x * (32 * VEC) + lane * VEC;
  const int Kp = K / EPB;
  // blockIdx.y splits the packed rows; partial sums are combined with atomics only
  // when k_splits > 1 (not used by default: deterministic path has k_splits == 1).
  const int jp = (Kp + k_splits - 1) / k_splits;
  const int j_begin = blockIdx.y * jp, j_end = min(Kp, j_begin + jp);

  for (int m0 = 0; m0 < M; m0 += MT) {
    float acc[MT][VEC];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[m][v] = 0.f;

    int cur_g = -1;
    float s[VEC], z[VEC];
    for (int j = j_begin + warp; j < j_end; j += NW) {
      uint32_t packed = 0;
      if constexpr (VEC == 4) {
        if (o_base < N) packed = *reinterpret_cast<const uint32_t*>(qw + (size_t)j * N + o_base);
      } else {
        if (o_base < N) packed = qw[(size_t)j * N + o_base];
      }
      const int g = (j * EPB) / tile_cols;  // tile_cols is a multiple of EPB or >= K
      if (g != cur_g) {
        cur_g = g;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          int o = min(o_base + v, N - 1);
          s[v] = load_sz(scales, szdt, (size_t)o * n_groups + g);
          z[v] = load_sz(zeros, szdt, (size_t)o * n_groups + g);
        }
      }
#pragma unroll
      for (int nr = 0; nr < EPB; ++nr) {
        const int k = j * EPB + nr;
        float xv[MT];
#pragma unroll
        for (int m = 0; m < MT; ++m) xv[m] = (m0 + m < M) ? bf2f(x[(size_t)(m0 + m) * ldx + k]) : 0.f;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          float lv = (float)((packed >> (v * 8 + nr * BITS)) & MASK);
          float w = (lv - z[v]) * s[v];
#pragma unroll
          for (int m = 0; m < MT; ++m) acc[m][v] = fmaf(w, xv[m], acc[m][v]);
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int v = 0; v < VEC; ++v) red[warp][m][lane * VEC + v] = acc[m][v];
    __syncthreads();
    for (int i = threadIdx.x; i < MT * 32 * VEC; i += blockDim.x) {
      int m = i / (32 * VEC), c = i % (32 * VEC);
      int o = blockIdx.x * (32 * VEC) + c;
      if (m0 + m < M && o < N) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < NW; ++w) t += red[w][m][c];
        if (bias != nullptr) t += bf2f(bias[o]);
        y[(size_t)(m0 + m) * ldy + o] = f2bf(t);
      }
    }
  }
}

template <int BITS, int VEC>
static int launch_q_linear(const void* x, int ldx, const void* qw, const void* scales, const void* zeros,
                           int szdt, const void* bias, void* y, int ldy, int M, int N, int K, int tile_cols,
                           cudaStream_t stream) {
  const int n_groups = (K + tile_cols - 1) / tile_cols;
  dim3 grid((N + 32 * VEC - 1) / (32 * VEC), 1), block(256);
#define B2L_QL(MT)                                                                                         \
  q_linear_kernel<BITS, VEC, MT><<<grid, block, 0, stream>>>(                                              \
      (const __nv_bfloat16*)x, ldx, (const uint8_t*)qw, scales, zeros, szdt, (const __nv_bfloat16*)bias,   \
      (__nv_bfloat16*)y, ldy, M, N, K, tile_cols, n_groups, 1)
  if (M == 1) B2L_QL(1);
  else if (M == 2) B2L_QL(2);
  else B2L_QL(4);
#undef B2L_QL
  B2L_LAUNCH_CHECK("q_linear_kernel");
  return 0;
}

}  // namespace b2l

using namespace b2l;

extern "C" int b2l_q_dequant(const void* qw, const void* scales, const void* zeros, int sz_dtype, void* w_out,
                             int out_dtype, int out_features, int in_features, int bits, int tile_cols,
                             b2l_stream_t stream) {
  B2L_CHECK_ARG(qw && scales && zeros && w_out, "b2l_q_dequant: null pointer");
  B2L_CHECK_SUPPORTED(bits == 4 || bits == 8, "b2l_q_dequant: bits must be 4 or 8 (got %d)", bits);
  B2L_CHECK_ARG(out_features > 0 && in_features > 0 && in_features % (8 / bits) == 0,
                "b2l_q_dequant: bad shape (%d, %d)", out_features, in_features);
  if (tile_cols <= 0 || tile_cols > in_features) tile_cols = in_features;
  B2L_CHECK_SUPPORTED(tile_cols % (8 / bits) == 0, "b2l_q_dequant: tile_cols %d not a multiple of %d", tile_cols, 8 / bits);
  B2L_CHECK_ARG(sz_dtype == B2L_BF16 || sz_dtype == B2L_F32, "b2l_q_dequant: bad sz_dtype");
  const int n_groups = (in_features + tile_cols - 1) / tile_cols;
  const int Kp = in_features / (8 / bits);
  dim3 grid((out_features + 31) / 32, (Kp + 31) / 32), block(32, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (out_dtype == B2L_BF16) {
    if (bits == 4) dequant_kernel<4, __nv_bfloat16><<<grid, block, 0, st>>>((const uint8_t*)qw, scales, zeros, sz_dtype, (__nv_bfloat16*)w_out, out_features, in_features, tile_cols, n_groups);
    else dequant_kernel<8, __nv_bfloat16><<<grid, block, 0, st>>>((const uint8_t*)qw, scales, zeros, sz_dtype, (__nv_bfloat16*)w_out, out_features, in_features, tile_cols, n_groups);
  } else if (out_dtype == B2L_F32) {
    if (bits == 4) dequant_kernel<4, float><<<grid, block, 0, st>>>((const uint8_t*)qw, scales, zeros, sz_dtype, (float*)w_out, out_features, in_features, tile_cols, n_groups);
    else dequant_kernel<8, float><<<grid, block, 0, st>>>((const uint8_t*)qw, scales, zeros, sz_dtype, (float*)w_out, out_features, in_features, tile_cols, n_groups);
  } else {
    set_error("b2l_q_dequant: bad out_dtype %d", out_dtype);
    return B2L_E_ARG;
  }
  B2L_LAUNCH_CHECK("dequant_kernel");
  return 0;
}

extern "C" int b2l_q_linear(const void* x, int ldx, const void* qw, const void* scales, const void* zeros,
                            int sz_dtype, const void* bias, void* y, int ldy, int M, int N, int K, int bits,
                            int tile_cols, b2l_stream_t stream) {
  B2L_CHECK_ARG(x && qw && scales && zeros && y, "b2l_q_linear: null pointer");
  B2L_CHECK_SUPPORTED(bits == 4 || bits == 8, "b2l_q_linear: bits must be 4 or 8 (got %d)", bits);
  B2L_CHECK_ARG(M >= 0 && N > 0 && K > 0 && K % (8 / bits) == 0 && ldx >= K && ldy >= N,
                "b2l_q_linear: bad shape M=%d N=%d K=%d ldx=%d ldy=%d", M, N, K, ldx, ldy);
  B2L_CHECK_ARG(sz_dtype == B2L_BF16 || sz_dtype == B2L_F32, "b2l_q_linear: bad sz_dtype");
  if (M == 0) return 0;
  if (tile_cols <= 0 || tile_cols > K) tile_cols = K;
  B2L_CHECK_SUPPORTED(tile_cols % (8 / bits) == 0, "b2l_q_linear: tile_cols %d not a multiple of %d", tile_cols, 8 / bits);
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec4 = (N % 4 == 0) && ((uintptr_t)qw % 4 == 0);
  if (bits == 4)
    return vec4 ? launch_q_linear<4, 4>(x, ldx, qw, scales, zeros, sz_dtype, bias, y, ldy, M, N, K, tile_cols, st)
                : launch_q_linear<4, 1>(x, ldx, qw, scales, zeros, sz_dtype, bias, y, ldy, M, N, K, tile_cols, st);
  return vec4 ? launch_q_linear<8, 4>(x, ldx, qw, scales, zeros, sz_dtype, bias, y, ldy, M, N, K, tile_cols, st)
              : launch_q_linear<8, 1>(x, ldx, qw, scales, zeros, sz_dtype, bias, y, ldy, M, N, K, tile_cols, st);
}

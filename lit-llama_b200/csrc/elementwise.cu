// model.py element-wise pieces as stand-alone kernels (module-level drop-ins, prefill).
// In the decode step these are fused into the tensor-core linears' prologue/epilogue.
#include <algorithm>

#include "b2l_common.cuh"

namespace b2l {

// RMSNorm.forward, model.py:270-277, bf16 rounding points preserved.  One CTA per row.
__global__ void __launch_bounds__(256) rmsnorm_kernel(const __nv_bfloat16* __restrict__ x,
                                                      const __nv_bfloat16* __restrict__ scale,
                                                      __nv_bfloat16* __restrict__ y, int C, float eps) {
  __shared__ float red[32];
  const __nv_bfloat16* xr = x + (size_t)blockIdx.x * C;
  __nv_bfloat16* yr = y + (size_t)blockIdx.x * C;
  float ss = 0.f;
  const bool vec = (C % 8 == 0) && ((((uintptr_t)xr | (uintptr_t)yr | (uintptr_t)scale) & 15) == 0);
  if (vec) {
    for (int i = threadIdx.x; i < C / 8; i += blockDim.x) {
      const uint4 v = reinterpret_cast<const uint4*>(xr)[i];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float lo = __uint_as_float(w[q] << 16), hi = __uint_as_float(w[q] & 0xffff0000u);
        ss += rbf(lo * lo) + rbf(hi * hi);
      }
    }
  } else {
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      float v = bf2f(xr[i]);
      ss += rbf(v * v);
    }
  }
  ss = block_sum(ss, red);
  const float rinv = rms_rinv(ss, C, eps);
  if (vec) {
    for (int i = threadIdx.x; i < C / 8; i += blockDim.x) {
      const uint4 v = reinterpret_cast<const uint4*>(xr)[i], gsc = reinterpret_cast<const uint4*>(scale)[i];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w}, gw[4] = {gsc.x, gsc.y, gsc.z, gsc.w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const __nv_bfloat162 t = __floats2bfloat162_rn(rms_apply(__uint_as_float(w[q] << 16), rinv, __uint_as_float(gw[q] << 16)),
                                                       rms_apply(__uint_as_float(w[q] & 0xffff0000u), rinv, __uint_as_float(gw[q] & 0xffff0000u)));
        o[q] = *reinterpret_cast<const uint32_t*>(&t);
      }
      reinterpret_cast<uint4*>(yr)[i] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  } else {
    for (int i = threadIdx.x; i < C; i += blockDim.x) yr[i] = f2bf(rms_apply(bf2f(xr[i]), rinv, bf2f(scale[i])));
  }
}

template <typename IdxT>
__global__ void embedding_kernel(const IdxT* __restrict__ idx, const __nv_bfloat16* __restrict__ wte,
                                 __nv_bfloat16* __restrict__ out, int C, int vocab) {
  pdl_launch_dependents();  // the first c_attn of the step may start streaming its weights
  long long t = (long long)idx[blockIdx.x];
  if (t < 0 || t >= vocab) t = 0;  // torch would raise; keep the kernel memory-safe
  const __nv_bfloat16* src = wte + (size_t)t * C;
  __nv_bfloat16* dst = out + (size_t)blockIdx.x * C;
  for (int i = threadIdx.x; i < C; i += blockDim.x) dst[i] = src[i];
}

// silu_mul1 / pack_bf16x2 / affine1: b2l_common.cuh (the batch-1 llm.int8 linear fuses the same arithmetic).
// 8 elements (16 bytes) per thread when the pointers allow it (VEC), else one
template <bool VEC, bool SILU>
__global__ void __launch_bounds__(256) binary_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
                                                     __nv_bfloat16* __restrict__ y, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    if (i * 8 + 8 <= n) {
      const uint4 av = reinterpret_cast<const uint4*>(a)[i], bv = reinterpret_cast<const uint4*>(b)[i];
      const uint32_t aw[4] = {av.x, av.y, av.z, av.w}, bw[4] = {bv.x, bv.y, bv.z, bv.w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float a0 = __uint_as_float(aw[q] << 16), a1 = __uint_as_float(aw[q] & 0xffff0000u);
        const float b0 = __uint_as_float(bw[q] << 16), b1 = __uint_as_float(bw[q] & 0xffff0000u);
        o[q] = SILU ? pack_bf16x2(silu_mul1(a0, b0), silu_mul1(a1, b1)) : pack_bf16x2(a0 + b0, a1 + b1);
      }
      reinterpret_cast<uint4*>(y)[i] = make_uint4(o[0], o[1], o[2], o[3]);
    } else {
      for (size_t j = i * 8; j < n; ++j) y[j] = f2bf(SILU ? silu_mul1(bf2f(a[j]), bf2f(b[j])) : bf2f(a[j]) + bf2f(b[j]));
    }
  } else if (i < n) {
    y[i] = f2bf(SILU ? silu_mul1(bf2f(a[i]), bf2f(b[i])) : bf2f(a[i]) + bf2f(b[i]));
  }
}

template <bool SILU>
static int launch_binary(const void* a, const void* b, void* y, size_t n, cudaStream_t st) {
  const bool vec = (((uintptr_t)a | (uintptr_t)b | (uintptr_t)y) & 15) == 0;
  const __nv_bfloat16 *pa = (const __nv_bfloat16*)a, *pb = (const __nv_bfloat16*)b;
  if (vec) binary_kernel<true, SILU><<<(unsigned)(((n + 7) / 8 + 255) / 256), 256, 0, st>>>(pa, pb, (__nv_bfloat16*)y, n);
  else binary_kernel<false, SILU><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pa, pb, (__nv_bfloat16*)y, n);
  return 0;
}

// LLaMA-Adapter v2's affine of a linear's output, adapter_v2.py:30-33: y = bf16(s * bf16(y + b)) per column, in
// place.  VEC: 8 columns (16 bytes) per thread, N, ldy multiples of 8 and 16-byte aligned pointers.
template <bool VEC>
__global__ void __launch_bounds__(256) linear_affine_kernel(__nv_bfloat16* y, int ldy, int M, int N,
                                                            const __nv_bfloat16* __restrict__ scale,
                                                            const __nv_bfloat16* __restrict__ bias) {
  const int per = VEC ? 8 : 1;
  const int cols = N / per;
  const size_t total = (size_t)M * cols;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(i / cols), c = (int)(i - (size_t)m * cols) * per;
    __nv_bfloat16* row = y + (size_t)m * ldy + c;
    if (VEC) {
      const uint4 yv = *reinterpret_cast<const uint4*>(row);
      const uint4 sv = *reinterpret_cast<const uint4*>(scale + c), bv = *reinterpret_cast<const uint4*>(bias + c);
      const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w}, sw[4] = {sv.x, sv.y, sv.z, sv.w}, bw[4] = {bv.x, bv.y, bv.z, bv.w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        o[q] = pack_bf16x2(affine1(__uint_as_float(yw[q] << 16), __uint_as_float(sw[q] << 16), __uint_as_float(bw[q] << 16)),
                           affine1(__uint_as_float(yw[q] & 0xffff0000u), __uint_as_float(sw[q] & 0xffff0000u),
                                   __uint_as_float(bw[q] & 0xffff0000u)));
      *reinterpret_cast<uint4*>(row) = make_uint4(o[0], o[1], o[2], o[3]);
    } else {
      *row = f2bf(affine1(bf2f(*row), bf2f(scale[c]), bf2f(bias[c])));
    }
  }
}

}  // namespace b2l

using namespace b2l;

extern "C" int b2l_linear_affine(void* y, int ldy, int M, int N, const void* scale, const void* bias,
                                 b2l_stream_t stream) {
  B2L_CHECK_ARG(y && scale && bias, "b2l_linear_affine: null pointer");
  B2L_CHECK_ARG(M >= 0 && N > 0 && ldy >= N, "b2l_linear_affine: bad shape (M=%d, N=%d, ldy=%d)", M, N, ldy);
  B2L_CHECK_ARG((uintptr_t)y % 2 == 0 && (uintptr_t)scale % 2 == 0 && (uintptr_t)bias % 2 == 0,
                "b2l_linear_affine: y / scale / bias must be 2-byte aligned bf16");
  if (M == 0) return 0;
  const bool vec = N % 8 == 0 && ldy % 8 == 0 && (((uintptr_t)y | (uintptr_t)scale | (uintptr_t)bias) & 15) == 0;
  const size_t work = (size_t)M * (vec ? N / 8 : N);
  const unsigned grid = (unsigned)std::min<size_t>((work + 255) / 256, (size_t)sm_count() * 16);
  cudaStream_t st = (cudaStream_t)stream;
  const __nv_bfloat16 *s = (const __nv_bfloat16*)scale, *b = (const __nv_bfloat16*)bias;
  if (vec) linear_affine_kernel<true><<<grid, 256, 0, st>>>((__nv_bfloat16*)y, ldy, M, N, s, b);
  else linear_affine_kernel<false><<<grid, 256, 0, st>>>((__nv_bfloat16*)y, ldy, M, N, s, b);
  B2L_LAUNCH_CHECK("linear_affine_kernel");
  return 0;
}

extern "C" int b2l_rmsnorm(const void* x, const void* scale, void* y, int rows, int C, float eps,
                           b2l_stream_t stream) {
  B2L_CHECK_ARG(x && scale && y && rows >= 0 && C > 0, "b2l_rmsnorm: bad argument");
  if (rows == 0) return 0;
  rmsnorm_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)scale,
                                                         (__nv_bfloat16*)y, C, eps);
  B2L_LAUNCH_CHECK("rmsnorm_kernel");
  return 0;
}

extern "C" int b2l_embedding(const void* idx, int idx_is_i64, const void* wte, void* out, int n, int C, int vocab,
                             b2l_stream_t stream) {
  B2L_CHECK_ARG(idx && wte && out && n >= 0 && C > 0 && vocab > 0, "b2l_embedding: bad argument");
  if (n == 0) return 0;
  if (idx_is_i64)
    embedding_kernel<long long><<<n, 256, 0, (cudaStream_t)stream>>>((const long long*)idx, (const __nv_bfloat16*)wte, (__nv_bfloat16*)out, C, vocab);
  else
    embedding_kernel<int><<<n, 256, 0, (cudaStream_t)stream>>>((const int*)idx, (const __nv_bfloat16*)wte, (__nv_bfloat16*)out, C, vocab);
  B2L_LAUNCH_CHECK("embedding_kernel");
  return 0;
}

extern "C" int b2l_silu_mul(const void* a, const void* b, void* y, size_t n, b2l_stream_t stream) {
  B2L_CHECK_ARG(a && b && y, "b2l_silu_mul: null pointer");
  if (n == 0) return 0;
  launch_binary<true>(a, b, y, n, (cudaStream_t)stream);
  B2L_LAUNCH_CHECK("silu_mul kernel");
  return 0;
}

extern "C" int b2l_add(const void* a, const void* b, void* y, size_t n, b2l_stream_t stream) {
  B2L_CHECK_ARG(a && b && y, "b2l_add: null pointer");
  if (n == 0) return 0;
  launch_binary<false>(a, b, y, n, (cudaStream_t)stream);
  B2L_LAUNCH_CHECK("add kernel");
  return 0;
}

// CausalSelfAttention.forward between the two linears (model.py:197-232):
// RoPE (model.py:306-323), KV-cache append with the roll branch as a device-side ring
// (model.py:211-221), and masked softmax(q k^T / sqrt(hs)) v (model.py:230) as a
// split-S streaming kernel that only touches the valid slots 0..pos.
//
// All positions are read on the device; the host never synchronises (the reference
// does once per layer per token, model.py:214).
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <cstdlib>

#include "b2l_common.cuh"

namespace b2l {

// ---- fp8 KV cache (b2l_attention_kv8, B2L_F_KV_FP8): the number format of include/b2l.h ----
constexpr int KV8_E_MIN = -124;   // 2^-9 (smallest e4m3 subnormal) x 2^-124 = 2^-133, the smallest bf16 subnormal

// scale exponent e of a vector whose largest |element| has the fp32 bits a (finite): the smallest e with
// amax 2^-e <= 448, at least KV8_E_MIN; 0 for an all-zero vector
__device__ __forceinline__ int kv8_exponent(uint32_t a) {
  if (a == 0) return 0;
  if (a < 0x00800000u) return KV8_E_MIN;   // fp32 subnormal: far below 2^(KV8_E_MIN + 8)
  const int e = (int)(a >> 23) - 127 - 8 + ((a & 0x7fffffu) > 0x600000u);   // mantissa above 1.75: one binade up
  return e < KV8_E_MIN ? KV8_E_MIN : e;
}
__device__ __forceinline__ uint32_t abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }

// two values times inv = 2^-e as e4m3 codes (round to nearest even; |x inv| <= 448, so satfinite never clips), x in the
// low byte
__device__ __forceinline__ uint32_t kv8_code2(float a, float b, float inv) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(a * inv, b * inv), __NV_SATFINITE, __NV_E4M3);
}
// the values two codes (low byte first) stand for: float(code) x scale
__device__ __forceinline__ void kv8_value2(uint32_t c, float s, float& a, float& b) {
  const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(c & 0xffffu), __NV_E4M3);
  const float2 f = __half22float2(__half2(r));
  a = f.x * s;
  b = f.y * s;
}
__device__ __forceinline__ float kv8_value(uint8_t c, float s) {
  return __half2float(__half(__nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)c, __NV_E4M3))) * s;
}
// The value of one e4m3fn code (not NaN) from its bits, exact.  The new token's values are decoded this way from the
// code words kv8_quant16 returns, the words that are stored (kv8_decode16).
__device__ __forceinline__ float e4m3_value(uint32_t c) {
  const float mag = (c & 0x78u) ? __uint_as_float(((((c >> 3) & 15u) + 120u) << 23) | ((c & 7u) << 20))
                                : (float)(c & 7u) * 0.001953125f;   // subnormal: m 2^-9
  return (c & 0x80u) ? -mag : mag;
}
// 16 codes (16 consecutive dims) -> fp32 values
__device__ __forceinline__ void kv8_to_f32(const uint4& u, float s, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    kv8_value2(w[i], s, f[4 * i], f[4 * i + 1]);
    kv8_value2(w[i] >> 16, s, f[4 * i + 2], f[4 * i + 3]);
  }
}
// Quantizes 16 values of a vector whose largest |element| has the fp32 bits a: returns their codes and the vector's
// scale.  A non-finite element makes every code NaN (0x7f) and the scale NaN.
__device__ __forceinline__ uint4 kv8_quant16(const float* f, uint32_t a, float& scale) {
  if (a >= 0x7f800000u) {
    scale = __uint_as_float(0x7fc00000u);
    return make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);
  }
  const int e = kv8_exponent(a);
  scale = __uint_as_float((uint32_t)(127 + e) << 23);
  const float inv = __uint_as_float((uint32_t)(127 - e) << 23);
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    w[i] = (kv8_code2(f[4 * i], f[4 * i + 1], inv) & 0xffffu) | (kv8_code2(f[4 * i + 2], f[4 * i + 3], inv) << 16);
  return make_uint4(w[0], w[1], w[2], w[3]);
}
// The values 16 codes of kv8_quant16 stand for (NaN codes: NaN, since the scale is NaN then)
__device__ __forceinline__ void kv8_decode16(const uint4& u, float s, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 16; ++i) f[i] = e4m3_value((w[i >> 2] >> (8 * (i & 3))) & 0xffu) * s;
}

__global__ void ring_advance_kernel(const int64_t* __restrict__ input_pos, int T, int32_t* ring_start, int S) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (input_pos[T - 1] >= (int64_t)S) *ring_start = (*ring_start + 1) % S;
  }
}

// B2L_F_ROW_POS: row b's ring offset ring_start[b] follows its own position input_pos[b]
__global__ void ring_advance_rows_kernel(const int64_t* __restrict__ input_pos, int B, int32_t* ring_start, int S) {
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    if (input_pos[b] >= (int64_t)S) ring_start[b] = (ring_start[b] + 1) % S;
  }
}

// Sequence of packed token bt of a ragged launch (b2l_attention_ragged): its cache row and its position in the sequence
__device__ __forceinline__ void ragged_token(const b2l_ragged& rg, int bt, int& row, int& t) {
  int s = 0;
  while (s < rg.n_seq - 1 && bt >= rg.start[s] + rg.len[s]) ++s;
  row = rg.row[s];
  t = bt - rg.start[s];
}

// grid (B*T, n_head), block hs/2 threads (one per rotated pair).
// q is rotated in place inside qkv; k (rotated) and v go to the cache (or, without a
// cache, k is rotated in place as well).  pos_stride 1 (B2L_F_ROW_POS, T == 1): row b reads input_pos[b] and
// ring_start[b]; 0: every row reads the shared entries.  rotate_q 0 (B2L_F_STEPWISE on the fused path): qkv is left
// untouched and only the cache rows are written, since the fused kernel rotates q and its own key from qkv itself.
// RAGGED (b2l_attention_ragged): grid (N, n_head); packed token bt is token t of the sequence that `rg` places at
// [start, start + len), at position t in cache row `row`, whose ring offset restarts at 0 (the token-0 CTA of head 0
// stores it; nothing here reads it).  input_pos, T and pos_stride are unused.
template <bool RAGGED>
__global__ void rope_append_kernel(__nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ k_cache,
                                   __nv_bfloat16* __restrict__ v_cache, const float* __restrict__ rope,
                                   const int64_t* __restrict__ input_pos, const int32_t* __restrict__ ring_start,
                                   int T, int n_head, int hs, int S, int block_size, int rope_rows, int pos_stride,
                                   int rotate_q, const __grid_constant__ b2l_ragged rg) {
  const int bt = blockIdx.x, h = blockIdx.y;
  int b, t;
  if constexpr (RAGGED) {
    ragged_token(rg, bt, b, t);
    if (t == 0 && h == 0 && threadIdx.x == 0) const_cast<int32_t*>(ring_start)[b] = 0;   // never read by this kernel
  } else {
    b = bt / T;
    t = bt % T;
  }
  const int C = n_head * hs;
  long long p = (!RAGGED && input_pos) ? input_pos[b * pos_stride + t] : (long long)t;
  // rope_rows: `rope` already holds the T selected rows (reference call convention, model.py:93)
  const long long prow = rope_rows ? (long long)t : (p < block_size ? p : (long long)block_size - 1);
  __nv_bfloat16* q = qkv + (size_t)bt * 3 * C + h * hs;
  __nv_bfloat16* k = q + C;
  const __nv_bfloat16* v = q + 2 * C;
  __nv_bfloat16 *kd = k, *vd = nullptr;
  if (k_cache != nullptr) {
    const int w = (int)(p < S ? p : (long long)S - 1);
    const int phys = RAGGED ? w : (w + ring_start[b * pos_stride]) % S;
    const size_t off = (((size_t)b * n_head + h) * S + phys) * hs;
    kd = k_cache + off;
    vd = v_cache + off;
  }
  for (int i = threadIdx.x; i < hs / 2; i += blockDim.x) {
    const float c = rope[((size_t)prow * (hs / 2) + i) * 2 + 0];
    const float s = rope[((size_t)prow * (hs / 2) + i) * 2 + 1];
    const float q0 = bf2f(q[2 * i]), q1 = bf2f(q[2 * i + 1]);
    const float k0 = bf2f(k[2 * i]), k1 = bf2f(k[2 * i + 1]);
    // model.py:315-318 (separate multiplies and add/sub in fp32, then type_as(x))
    if (rotate_q) {
      q[2 * i] = f2bf(__fsub_rn(__fmul_rn(q0, c), __fmul_rn(q1, s)));
      q[2 * i + 1] = f2bf(__fadd_rn(__fmul_rn(q1, c), __fmul_rn(q0, s)));
    }
    kd[2 * i] = f2bf(__fsub_rn(__fmul_rn(k0, c), __fmul_rn(k1, s)));
    kd[2 * i + 1] = f2bf(__fadd_rn(__fmul_rn(k1, c), __fmul_rn(k0, s)));
    if (vd != nullptr) {
      vd[2 * i] = v[2 * i];
      vd[2 * i + 1] = v[2 * i + 1];
    }
  }
}

// Prefill of a prompt at positions 0..T-1 into an fp8 cache (b2l_attention_kv8, T > 1): grid (B*T, n_head), block 64
// (one thread per rotated pair).  q and k are rotated in place as rope_append_kernel does without a cache (the prompt
// then attends over its own bf16 rows), and the rotated k row and the v row are quantized into slot
// (t + ring_start[0]) % S of row b.
// RAGGED (b2l_attention_ragged_kv8): grid (N, n_head); packed token bt is token t of the sequence `rg` places at
// [start, start + len), quantized into slot t of cache row `row`, whose ring offset restarts at 0 (the token-0 CTA of
// head 0 stores it; nothing here reads it).  T is unused.
template <bool RAGGED>
__global__ void __launch_bounds__(64)
    rope_append_kv8_kernel(__nv_bfloat16* __restrict__ qkv, uint8_t* __restrict__ k_code, uint8_t* __restrict__ v_code,
                           float* __restrict__ k_scale, float* __restrict__ v_scale, const float* __restrict__ rope,
                           const int32_t* __restrict__ ring_start, int T, int n_head, int S,
                           const __grid_constant__ b2l_ragged rg) {
  constexpr int HS = 128;
  __shared__ uint32_t red[2][2];
  const int bt = blockIdx.x, h = blockIdx.y, i = threadIdx.x;
  int b, t;
  if constexpr (RAGGED) {
    ragged_token(rg, bt, b, t);
    if (t == 0 && h == 0 && i == 0) const_cast<int32_t*>(ring_start)[b] = 0;   // never read by this kernel
  } else {
    b = bt / T;
    t = bt % T;
  }
  const int C = n_head * HS;
  __nv_bfloat16* q = qkv + (size_t)bt * 3 * C + h * HS;
  __nv_bfloat16* k = q + C;
  const __nv_bfloat16* v = q + 2 * C;
  const float c = rope[((size_t)t * (HS / 2) + i) * 2 + 0];
  const float s = rope[((size_t)t * (HS / 2) + i) * 2 + 1];
  const float q0 = bf2f(q[2 * i]), q1 = bf2f(q[2 * i + 1]);
  const float k0 = bf2f(k[2 * i]), k1 = bf2f(k[2 * i + 1]);
  q[2 * i] = f2bf(__fsub_rn(__fmul_rn(q0, c), __fmul_rn(q1, s)));
  q[2 * i + 1] = f2bf(__fadd_rn(__fmul_rn(q1, c), __fmul_rn(q0, s)));
  const __nv_bfloat16 ke = f2bf(__fsub_rn(__fmul_rn(k0, c), __fmul_rn(k1, s)));
  const __nv_bfloat16 ko = f2bf(__fadd_rn(__fmul_rn(k1, c), __fmul_rn(k0, s)));
  k[2 * i] = ke;
  k[2 * i + 1] = ko;
  const float x[2][2] = {{bf2f(ke), bf2f(ko)}, {bf2f(v[2 * i]), bf2f(v[2 * i + 1])}};
  const int warp = i >> 5;
#pragma unroll
  for (int kv = 0; kv < 2; ++kv) {
    const uint32_t a = __reduce_max_sync(0xffffffffu, max(abs_bits(x[kv][0]), abs_bits(x[kv][1])));
    if ((i & 31) == 0) red[kv][warp] = a;
  }
  __syncthreads();
  const size_t slot = ((size_t)b * n_head + h) * S + (RAGGED ? t : (t + ring_start[0]) % S);
#pragma unroll
  for (int kv = 0; kv < 2; ++kv) {
    const uint32_t a = max(red[kv][0], red[kv][1]);
    uint32_t code;
    float scale;
    if (a >= 0x7f800000u) {   // a non-finite element: NaN codes and scale (kv8_quant16)
      code = 0x7f7fu;
      scale = __uint_as_float(0x7fc00000u);
    } else {
      const int e = kv8_exponent(a);
      scale = __uint_as_float((uint32_t)(127 + e) << 23);
      code = kv8_code2(x[kv][0], x[kv][1], __uint_as_float((uint32_t)(127 - e) << 23));
    }
    reinterpret_cast<uint16_t*>((kv ? v_code : k_code) + slot * HS)[i] = (uint16_t)code;
    if (i == 0) (kv ? v_scale : k_scale)[slot] = scale;
  }
}

struct KvView {
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  size_t b_stride, h_stride, s_stride;  // elements
  int S;                                // ring modulus (0 = no ring)
};

constexpr int ATT_WARPS = 4;
constexpr int ATT_MAX_EPL = 8;  // head_size <= 256

// grid (B*n_head, T, n_split).  Each CTA streams its chunk of the valid keys of query
// (b, t, h) with an online softmax per warp, merges its warps, and writes one partial
// (max, sum, acc[hs]) to `work`.
template <int EPL>  // elements per lane: head_size == 32*EPL when VEC, else generic
__global__ void __launch_bounds__(ATT_WARPS * 32)
    attn_partial_kernel(const __nv_bfloat16* __restrict__ qkv, KvView kv, const int64_t* __restrict__ input_pos,
                        const int32_t* __restrict__ ring_start, float* __restrict__ work, int T, int n_head,
                        int hs, int n_split, int chunk, int pos_stride) {
  const int bh = blockIdx.x, b = bh / n_head, h = bh % n_head, t = blockIdx.y, sp = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = n_head * hs;
  long long p = input_pos ? input_pos[b * pos_stride + t] : (long long)t;   // pos_stride as in rope_append_kernel
  const int cap = kv.S > 0 ? kv.S : T;
  const int L = (int)(p < cap ? p : (long long)cap - 1) + 1;  // valid logical slots 0..L-1
  const int ring = (kv.S > 0 && ring_start) ? ring_start[b * pos_stride] : 0;
  const int j0 = sp * chunk, j1 = min(L, j0 + chunk);
  float* out = work + (((size_t)bh * T + t) * n_split + sp) * (hs + 2);
  if (j0 >= j1) {  // empty split: neutral partial
    if (threadIdx.x == 0) { out[0] = -INFINITY; out[1] = 0.f; }
    for (int d = threadIdx.x; d < hs; d += blockDim.x) out[2 + d] = 0.f;
    return;
  }
  const float scale = rsqrtf((float)hs);
  float qv[ATT_MAX_EPL];
  const __nv_bfloat16* q = qkv + ((size_t)b * T + t) * 3 * C + h * hs;
#pragma unroll
  for (int e = 0; e < ATT_MAX_EPL; ++e) {
    int d = (EPL > 0) ? lane * EPL + e : lane + 32 * e;
    qv[e] = (e < (EPL > 0 ? EPL : ATT_MAX_EPL) && d < hs) ? bf2f(q[d]) * scale : 0.f;
  }
  float m = -INFINITY, l = 0.f, acc[ATT_MAX_EPL];
#pragma unroll
  for (int e = 0; e < ATT_MAX_EPL; ++e) acc[e] = 0.f;
  const __nv_bfloat16* kb = kv.k + b * kv.b_stride + h * kv.h_stride;
  const __nv_bfloat16* vb = kv.v + b * kv.b_stride + h * kv.h_stride;
  for (int j = j0 + warp; j < j1; j += ATT_WARPS) {
    int phys = j;
    if (kv.S > 0) { phys = j + ring; if (phys >= kv.S) phys -= kv.S; }
    const __nv_bfloat16* kr = kb + (size_t)phys * kv.s_stride;
    const __nv_bfloat16* vr = vb + (size_t)phys * kv.s_stride;
    float kx[ATT_MAX_EPL], vx[ATT_MAX_EPL];
    if constexpr (EPL == 4) {
      uint2 ku = *reinterpret_cast<const uint2*>(kr + lane * 4);
      uint2 vu = *reinterpret_cast<const uint2*>(vr + lane * 4);
      kx[0] = __uint_as_float(ku.x << 16); kx[1] = __uint_as_float(ku.x & 0xffff0000u);
      kx[2] = __uint_as_float(ku.y << 16); kx[3] = __uint_as_float(ku.y & 0xffff0000u);
      vx[0] = __uint_as_float(vu.x << 16); vx[1] = __uint_as_float(vu.x & 0xffff0000u);
      vx[2] = __uint_as_float(vu.y << 16); vx[3] = __uint_as_float(vu.y & 0xffff0000u);
    } else {
#pragma unroll
      for (int e = 0; e < ATT_MAX_EPL; ++e) {
        int d = lane + 32 * e;
        kx[e] = d < hs ? bf2f(kr[d]) : 0.f;
        vx[e] = d < hs ? bf2f(vr[d]) : 0.f;
      }
    }
    float sc = 0.f;
#pragma unroll
    for (int e = 0; e < (EPL > 0 ? EPL : ATT_MAX_EPL); ++e) sc = fmaf(qv[e], kx[e], sc);
    sc = warp_sum(sc);
    const float mn = fmaxf(m, sc);
    const float corr = __expf(m - mn), pj = __expf(sc - mn);
    l = l * corr + pj;
#pragma unroll
    for (int e = 0; e < (EPL > 0 ? EPL : ATT_MAX_EPL); ++e) acc[e] = fmaf(pj, vx[e], acc[e] * corr);
    m = mn;
  }
  // merge the warps
  __shared__ float sm_m[ATT_WARPS], sm_l[ATT_WARPS];
  __shared__ float sm_acc[ATT_WARPS][32 * ATT_MAX_EPL];
  if (lane == 0) { sm_m[warp] = m; sm_l[warp] = l; }
#pragma unroll
  for (int e = 0; e < (EPL > 0 ? EPL : ATT_MAX_EPL); ++e) {
    int d = (EPL > 0) ? lane * EPL + e : lane + 32 * e;
    sm_acc[warp][d] = acc[e];
  }
  __syncthreads();
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < ATT_WARPS; ++w) M = fmaxf(M, sm_m[w]);
  float Ls = 0.f;
  float wgt[ATT_WARPS];
#pragma unroll
  for (int w = 0; w < ATT_WARPS; ++w) {
    wgt[w] = (sm_m[w] == -INFINITY) ? 0.f : __expf(sm_m[w] - M);
    Ls += sm_l[w] * wgt[w];
  }
  if (threadIdx.x == 0) { out[0] = M; out[1] = Ls; }
  for (int d = threadIdx.x; d < hs; d += blockDim.x) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < ATT_WARPS; ++w) a += sm_acc[w][d] * wgt[w];
    out[2 + d] = a;
  }
}

// grid (B*n_head, T): merge the split partials and write y[b][t][h*hs + d] in bf16.
__global__ void attn_combine_kernel(const float* __restrict__ work, __nv_bfloat16* __restrict__ y, int T,
                                    int n_head, int hs, int n_split) {
  // the kernel after this one (attn.c_proj) may start streaming its weights now
  pdl_launch_dependents();
  const int bh = blockIdx.x, b = bh / n_head, h = bh % n_head, t = blockIdx.y;
  const float* base = work + ((size_t)bh * T + t) * n_split * (hs + 2);
  float M = -INFINITY;
  for (int s = 0; s < n_split; ++s) M = fmaxf(M, base[(size_t)s * (hs + 2)]);
  float Ls = 0.f;
  for (int s = 0; s < n_split; ++s) {
    float ms = base[(size_t)s * (hs + 2)];
    if (ms != -INFINITY) Ls += base[(size_t)s * (hs + 2) + 1] * __expf(ms - M);
  }
  const float inv = 1.0f / Ls;
  __nv_bfloat16* yr = y + ((size_t)b * T + t) * (n_head * hs) + h * hs;
  for (int d = threadIdx.x; d < hs; d += blockDim.x) {
    float a = 0.f;
    for (int s = 0; s < n_split; ++s) {
      float ms = base[(size_t)s * (hs + 2)];
      if (ms != -INFINITY) a += base[(size_t)s * (hs + 2) + 2 + d] * __expf(ms - M);
    }
    yr[d] = f2bf(a * inv);
  }
}

__global__ void kv_unroll_kernel(const __nv_bfloat16* __restrict__ cache, const int32_t* __restrict__ ring_start,
                                 __nv_bfloat16* __restrict__ out, int S, int hs, int n_head, int ring_stride) {
  // grid (B*n_head, S): logical slot blockIdx.y <- physical (slot + ring) % S; ring_stride 1: row b's own ring_start[b]
  const int ring = ring_start[(blockIdx.x / n_head) * ring_stride];
  const int phys = (blockIdx.y + ring) % S;
  const __nv_bfloat16* src = cache + ((size_t)blockIdx.x * S + phys) * hs;
  __nv_bfloat16* dst = out + ((size_t)blockIdx.x * S + blockIdx.y) * hs;
  for (int d = threadIdx.x; d < hs; d += blockDim.x) dst[d] = src[d];
}

// kv_unroll_kernel for an fp8 cache: the values read back, float(code) x scale, as bf16 (exact)
__global__ void kv8_unroll_kernel(const uint8_t* __restrict__ code, const float* __restrict__ scale,
                                  const int32_t* __restrict__ ring_start, __nv_bfloat16* __restrict__ out, int S, int hs,
                                  int n_head, int ring_stride) {
  const int ring = ring_start[(blockIdx.x / n_head) * ring_stride];
  const size_t phys = (size_t)blockIdx.x * S + (blockIdx.y + ring) % S;
  const float s = scale[phys];
  __nv_bfloat16* dst = out + ((size_t)blockIdx.x * S + blockIdx.y) * hs;
  for (int d = threadIdx.x; d < hs; d += blockDim.x) dst[d] = f2bf(kv8_value(code[phys * hs + d], s));
}

// ----------------------------------------------------------------------------------
// Fused single-token attention for head_size 128 (every LLaMA size): one kernel does
// RoPE(q), RoPE(k) + in-place KV append, split-S online-softmax attention over the valid
// slots, and the cross-split merge (last CTA of a head, atomic ticket).
//
// grid (B*n_head, ceil(S / 64)), 8 warps; CTAs beyond the position-dependent split count exit at once.  A CTA owns
// 64..256 keys of one head (chosen from the position and n_head so that ~400 CTAs work per batch row) and streams
// them as 64-key sub-tiles (K 16 KB + V 16 KB) through a two-deep shared-memory ring with TMA bulk copies: the first two
// sub-tiles are requested BEFORE griddepcontrol.wait (old cache rows do not depend on the current token), the
// next one as soon as a buffer has been consumed.  A warp handles 4 keys per round: 8 lanes per key, 16 head
// dims (32 B) per lane, a score needs 3 shuffles.  The new token's key / value never touch the tile: they are
// rotated, appended to the cache and scored from registers.
// Round 1 used one 128-key tile per CTA (64 KB, 3 CTAs per SM): at position 2047 its 512 CTAs needed a second
// wave and 16 partials per head had to be merged; 256 keys per CTA keep every position a single wave (<= 8 x n_head CTAs) with half the partials.
// ----------------------------------------------------------------------------------
constexpr int FD_CHUNK = 256;   // most keys per CTA
constexpr int FD_SUB = 64;      // keys per sub-tile = smallest number of keys per CTA
constexpr int FD_WARPS = 8;
constexpr int FD_CTAS_PER_SM = 3;   // resident CTAs per SM (shared memory): the working CTAs aimed at are one wave of them
constexpr int WS_CHUNK = FD_SUB;     // workspace sizing granularity (finest split of any kernel that uses it)

__device__ __forceinline__ void bf16x8_to_f32(const uint4& u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}

// Dynamic shared memory: 2 buffers x (K sub-tile 16 KB + V sub-tile 16 KB), merge scratch, 2 mbarriers.
constexpr int FD_SUB_BYTES = FD_SUB * 128 * 2;
constexpr int FD_SMEM_BYTES = 4 * FD_SUB_BYTES + FD_WARPS * 128 * 4 + 2 * FD_WARPS * 4 + 16;

// LLaMA-Adapter prefix term for one head of one query (adapter.py:164-167), called by every thread of a working CTA
// of the fused decode kernel.  sq: the rotated, 1/sqrt(hs)-scaled query [HS] (fp32, shared memory); ssc: score scratch
// [B2L_ADAPTER_MAX_LEN].  Warp w scores prefix keys w, w + 8, ... (4 dims per lane); thread d < HS then returns
// softmax(scores) . av[:, d] in fp32.
__device__ __forceinline__ float fd_adapter_prefix(const float* sq, float* ssc, const __nv_bfloat16* __restrict__ ak,
                                                   const __nv_bfloat16* __restrict__ av, int alen, int warp, int lane,
                                                   int d, bool writer) {
  constexpr int HS = 128;
  const float4 qv = reinterpret_cast<const float4*>(sq)[lane];
#pragma unroll 2
  for (int j = warp; j < alen; j += FD_WARPS) {
    const uint2 ku = __ldg(reinterpret_cast<const uint2*>(ak + (size_t)j * HS) + lane);
    float s = qv.x * __uint_as_float(ku.x << 16);
    s = fmaf(qv.y, __uint_as_float(ku.x & 0xffff0000u), s);
    s = fmaf(qv.z, __uint_as_float(ku.y << 16), s);
    s = fmaf(qv.w, __uint_as_float(ku.y & 0xffff0000u), s);
    s = warp_sum(s);
    if (lane == 0) ssc[j] = s;
  }
  __syncthreads();
  float ay = 0.f;
  if (writer) {
    float mx = -INFINITY;
    for (int j = 0; j < alen; ++j) mx = fmaxf(mx, ssc[j]);
    float l = 0.f;
    // 8 value loads in flight per round: this runs in the tail of the launch, where every L2 round trip is exposed
#pragma unroll 8
    for (int j = 0; j < alen; ++j) {
      const float p = __expf(ssc[j] - mx);
      l += p;
      ay = fmaf(p, bf2f(av[(size_t)j * HS + d]), ay);
    }
    ay /= l;
  }
  return ay;
}

// adapter.py:167 under bf16: y, the prefix attention and the gated term are each rounded, then their sum
__device__ __forceinline__ __nv_bfloat16 adapter_combine(float y, float ay, float gate) {
  return f2bf(rbf(y) + rbf(gate * rbf(ay)));
}

// ADAPTER: the LLaMA-Adapter variant.  Every working CTA asks the L2 for its head's prefix rows before
// griddepcontrol.wait (they do not depend on the current token) and computes the prefix attention as soon as its q
// is ready, while its first KV sub-tiles are still landing (q waits in the otherwise unused merge scratch).  The CTA
// that writes the head's output (the only one, or the last to arrive) adds the gated term before its store; the
// others drop it, so the term's two dependent L2 round trips overlap the KV stream instead of sitting in the tail of
// the writing CTA (DESIGN.md, LLaMA-Adapter, has the measurements of both placements).
// ROWS (B2L_F_ROW_POS): row b reads its own input_pos[b] and ring_start[b]; a template parameter, so the shared-position
// launch (batch 1 included) runs exactly the instructions it ran before per-row positions existed.
// STEP (B2L_F_STEPWISE): "row" b is query b of ONE sequence at input_pos[b]; every query reads batch row 0 of the cache,
// where a rope_append_kernel launch has already written all T new keys / values, so each query streams slots < its own
// as old rows, scores its own key from registers as the T == 1 launch does, and stores nothing to the cache (a second
// store of a slot would race the TMA reads of the later queries).
// KV8 (b2l_attention_kv8, B2L_F_KV_FP8): k_cache / v_cache hold e4m3 codes and k_scale / v_scale one fp32 scale per
// slot.  The ring carries 64-row sub-tiles of codes (8 KB of K, 8 KB of V); the CTA's old-row scales (<= 256 of each)
// are loaded once, before griddepcontrol.wait, into shared memory behind the barriers (a sub-tile's scales start at any
// slot of the ring, so they cannot always be a bulk copy's 16-byte aligned source).  Each lane turns its 16 codes into
// float(code) x scale; every FMA, shuffle, the split plan and the merge are those of the bf16 kernel.  The new key and
// value are quantized in registers (amax over the 8 lanes of the head), stored, and scored and accumulated as the
// values read back, so a step depends on the cache contents only.  Not with STEP.
template <bool ADAPTER, bool ROWS, bool STEP, bool KV8 = false>
__global__ void __launch_bounds__(FD_WARPS * 32, ADAPTER ? FD_CTAS_PER_SM : 0)
    attn_decode_fused_kernel(const __nv_bfloat16* qkv, __nv_bfloat16* __restrict__ k_cache,
                             __nv_bfloat16* __restrict__ v_cache, const float* __restrict__ rope,
                             const int64_t* __restrict__ input_pos, const int32_t* __restrict__ ring_start,
                             __nv_bfloat16* __restrict__ y, float* __restrict__ work, int* __restrict__ tickets,
                             int n_head, int S, int block_size, int n_split, unsigned long long* tl, int pre_tiles,
                             int smem_merge, int target_ctas, const __nv_bfloat16* __restrict__ pre_k,
                             const __nv_bfloat16* __restrict__ pre_v, const __nv_bfloat16* __restrict__ pre_gate,
                             int pre_len, float* k_scale, float* v_scale) {
  static_assert(!(KV8 && STEP), "the fp8 cache does not run the stepwise verify");
  constexpr int HS = 128;
  extern __shared__ __align__(128) uint8_t fsm[];
  float* sm_acc = reinterpret_cast<float*>(fsm + 4 * FD_SUB_BYTES);                // [FD_WARPS][HS]
  float* sm_m = sm_acc + FD_WARPS * HS;                                            // [FD_WARPS]
  float* sm_l = sm_m + FD_WARPS;                                                   // [FD_WARPS]
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(sm_l + FD_WARPS);  // 8-byte aligned by construction
  __shared__ int sm_last;

  if (threadIdx.x == 0) tl_min(tl, 0);
  const int bh = blockIdx.x, b = bh / n_head, h = bh % n_head, sp = blockIdx.y;
  // debug: raw stamps of CTA (0, 0) in slots 8.. (start, wait done, q ready, per sub-tile: data seen / done, merged, end)
  unsigned long long* tl0 = (tl != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) ? tl + 8 : nullptr;
  int tli = 0;
  auto stamp = [&]() { if (tl0 != nullptr && tli < 24) tl0[tli++] = globaltimer_ns(); };
  stamp();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = n_head * HS;
  const size_t head_base = ((size_t)(STEP ? 0 : b) * n_head + h) * S * HS;

  // input_pos and ring_start are inputs of the step (written by the host side long before), not
  // products of the previous kernel: they may be read before the dependency is resolved.  ROWS: row b is at its own
  // position input_pos[b] with its own ring offset ring_start[b], and everything below (write slot, key count, split
  // plan, ring wrap, merge) follows from that row's L.
  const long long p = input_pos[(ROWS || STEP) ? b : 0];
  const int w_slot = (int)(p < S ? p : (long long)S - 1);  // logical slot of the new token
  const int L = w_slot + 1;                                 // valid logical slots 0..L-1
  // keys per CTA: a multiple of 64 in [64, 256], chosen (identically by every CTA) so that at most target_ctas CTAs
  // per batch row have work: few long chunks would serialise sub-tiles inside a CTA, many short ones would need a
  // second wave (a sub-tile costs a CTA much less than the cross-CTA merge, tools/diag.py bench_ctx -- up to 256 keys
  // stay in ONE CTA per head, with no merge at all).  The plan is a function of (L, n_head, SM count) only, never of
  // B: it fixes the fp32 order of the online softmax and of the merge, so every row of a B-row launch equals the
  // B = 1 launch on that row's cache bit for bit (at B >= 2 and long context that is more than one wave of CTAs).
  const int want_splits = max(1, target_ctas / n_head);
  const int chunk = L <= FD_CHUNK ? FD_CHUNK
                                  : min(FD_CHUNK, max(FD_SUB, FD_SUB * ((L + FD_SUB * want_splits - 1) / (FD_SUB * want_splits))));
  const int n_active = (L + chunk - 1) / chunk;
  if (sp >= n_active) return;
  const int ring = ring_start[ROWS ? b : 0];
  const int j0 = sp * chunk, j1 = min(L, j0 + chunk);
  const int n_old = min(j1, L - 1) - j0;  // rows written by earlier steps (slot L-1 is written by this one)
  const int n_sub = (n_old + FD_SUB - 1) / FD_SUB;
  const bool has_new = (w_slot >= j0 && w_slot < j1);

  // sub-tile i -> buffer i & 1: old K rows then old V rows, each possibly in two pieces (the ring wraps)
  const uint32_t bar0 = smem_u32(bars);
  auto request = [&](int i) {
    const int buf = i & 1;
    const int cnt = min(FD_SUB, n_old - i * FD_SUB);
    int phys0 = j0 + i * FD_SUB + ring; if (phys0 >= S) phys0 -= S;
    const int first = min(cnt, S - phys0);  // rows before the ring wraps
    const uint32_t bar = bar0 + buf * 8;
    const uint32_t kd = smem_u32(fsm) + buf * 2 * FD_SUB_BYTES, vd = kd + FD_SUB_BYTES;
    if constexpr (KV8) {   // one byte per element
      const uint8_t* kc = reinterpret_cast<const uint8_t*>(k_cache) + head_base;
      const uint8_t* vc = reinterpret_cast<const uint8_t*>(v_cache) + head_base;
      mbar_expect_tx(bar, (uint32_t)cnt * HS * 2);
      tma_bulk_g2s(kd, kc + (size_t)phys0 * HS, (uint32_t)first * HS, bar);
      tma_bulk_g2s(vd, vc + (size_t)phys0 * HS, (uint32_t)first * HS, bar);
      if (first < cnt) {
        tma_bulk_g2s(kd + first * HS, kc, (uint32_t)(cnt - first) * HS, bar);
        tma_bulk_g2s(vd + first * HS, vc, (uint32_t)(cnt - first) * HS, bar);
      }
      return;
    }
    mbar_expect_tx(bar, (uint32_t)cnt * HS * 2 * 2);
    tma_bulk_g2s(kd, k_cache + head_base + (size_t)phys0 * HS, (uint32_t)first * HS * 2, bar);
    tma_bulk_g2s(vd, v_cache + head_base + (size_t)phys0 * HS, (uint32_t)first * HS * 2, bar);
    if (first < cnt) {  // wrapped part starts at physical row 0
      tma_bulk_g2s(kd + first * HS * 2, k_cache + head_base, (uint32_t)(cnt - first) * HS * 2, bar);
      tma_bulk_g2s(vd + first * HS * 2, v_cache + head_base, (uint32_t)(cnt - first) * HS * 2, bar);
    }
  };
  // ---- before the dependency: the first sub-tile (both when one CTA per head is all there is: nothing queues then)
  const int pre = (n_active == 1) ? 2 : pre_tiles;
  if (threadIdx.x == 0) {
    mbar_init_c<1>(bar0);
    mbar_init_c<1>(bar0 + 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (n_sub > 0) request(0);
    if (pre > 1 && n_sub > 1) request(1);
  }
  // KV8: the scales of old rows j0 .. j0 + n_old - 1 (thread j - j0 loads row j's)
  float* sks = reinterpret_cast<float*>(fsm + FD_SMEM_BYTES);
  float* svs = sks + FD_CHUNK;
  if constexpr (KV8) {
    if (threadIdx.x < n_old) {
      int ph = j0 + threadIdx.x + ring; if (ph >= S) ph -= S;
      const size_t si = head_base / HS + ph;
      sks[threadIdx.x] = k_scale[si];
      svs[threadIdx.x] = v_scale[si];
    }
  }
  if constexpr (ADAPTER) {
    if (threadIdx.x == 0) {   // the head's prefix rows
      const size_t off = (size_t)h * pre_len * HS;
      const uint32_t bytes = (uint32_t)pre_len * HS * 2;
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pre_k + off), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pre_v + off), "r"(bytes) : "memory");
    }
  }
  // the RoPE row of this position is a constant table entry: fetch it before the dependency too
  const long long prow = p < block_size ? p : (long long)block_size - 1;
  const int grp = lane >> 3, sub = lane & 7, d0 = sub * 16;
  float cs[16];
  {
    const float4* rp = reinterpret_cast<const float4*>(rope + ((size_t)prow * (HS / 2) + d0 / 2) * 2);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 t = rp[i];
      cs[4 * i] = t.x; cs[4 * i + 1] = t.y; cs[4 * i + 2] = t.z; cs[4 * i + 3] = t.w;
    }
  }
  __syncthreads();  // the barriers are initialised before anyone polls them
  pdl_wait();
  if (threadIdx.x == 0) tl_max(tl, 1);
  stamp();
  pdl_launch_dependents();  // attn.c_proj may start streaming its weights

  const __nv_bfloat16* qrow = qkv + (size_t)b * 3 * C + h * HS + d0;
  float q[16];
  {
    float raw[16];
    // qkv is the output of the kernel this one was launched behind (PDL): coherent loads only
    const uint4 qa = ld_coherent_u4(qrow), qb = ld_coherent_u4(qrow + 8);
    // The second sub-tile is requested BEHIND the q loads: a reply to this SM queues behind the bulk data already
    // on its way (measured, tools/diag.py timeline: with two 32 KB sub-tiles per CTA in flight the 32-byte q load
    // came back after 2.4 us at position 1033, 0.5 us with one), and q is what the first score needs.
    if (threadIdx.x == 0 && pre <= 1 && n_sub > 1) request(1);
    bf16x8_to_f32(qa, raw);
    bf16x8_to_f32(qb, raw + 8);
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
  float ay = 0.f;   // ADAPTER: the prefix attention of dim threadIdx.x (threads < HS), fp32
  if constexpr (ADAPTER) {
    if (warp == 0 && grp == 0) {   // lanes 0..7 hold the whole head
      float4* dq = reinterpret_cast<float4*>(sm_acc + d0);
#pragma unroll
      for (int i = 0; i < 4; ++i) dq[i] = make_float4(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]);
    }
    __syncthreads();
    ay = fd_adapter_prefix(sm_acc, sm_acc + HS, pre_k + (size_t)h * pre_len * HS, pre_v + (size_t)h * pre_len * HS,
                           pre_len, warp, lane, threadIdx.x & (HS - 1), threadIdx.x < HS);
  }

  float m = -INFINITY, l = 0.f, acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  if (tl0 != nullptr && q[0] != 12345.678f) stamp();   // q ready (the comparison keeps the stamp behind the loads)
  // ---- the new token FIRST (its k / v loads travel with the q loads, while the old tiles are still landing):
  // rotate k, append k and v to the cache, score from registers (warp 0, key group 0)
  if (has_new && warp == 0 && grp == 0) {
    int phys = w_slot + ring; if (phys >= S) phys -= S;
    float raw[16], kf[16], vf[16];
    bf16x8_to_f32(ld_coherent_u4(qrow + C), raw);
    bf16x8_to_f32(ld_coherent_u4(qrow + C + 8), raw + 8);
    uint32_t out[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float c = cs[2 * i], s_ = cs[2 * i + 1];
      kf[2 * i] = rbf(__fsub_rn(__fmul_rn(raw[2 * i], c), __fmul_rn(raw[2 * i + 1], s_)));
      kf[2 * i + 1] = rbf(__fadd_rn(__fmul_rn(raw[2 * i + 1], c), __fmul_rn(raw[2 * i], s_)));
      out[i] = (__float_as_uint(kf[2 * i]) >> 16) | (__float_as_uint(kf[2 * i + 1]) & 0xffff0000u);
    }
    const uint4 va = ld_coherent_u4(qrow + 2 * C), vb = ld_coherent_u4(qrow + 2 * C + 8);
    if constexpr (KV8) {   // quantize the head's key and value (lanes 0..7 hold it), store, go on with the values read back
      bf16x8_to_f32(va, vf); bf16x8_to_f32(vb, vf + 8);
      uint32_t ka = 0, vam = 0;
#pragma unroll
      for (int e = 0; e < 16; ++e) { ka = max(ka, abs_bits(kf[e])); vam = max(vam, abs_bits(vf[e])); }
#pragma unroll
      for (int o = 1; o <= 4; o <<= 1) {
        ka = max(ka, __shfl_xor_sync(0x000000ffu, ka, o));
        vam = max(vam, __shfl_xor_sync(0x000000ffu, vam, o));
      }
      float ksc, vsc;
      const uint4 kq = kv8_quant16(kf, ka, ksc), vq = kv8_quant16(vf, vam, vsc);
      kv8_decode16(kq, ksc, kf);
      kv8_decode16(vq, vsc, vf);
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(k_cache) + head_base + (size_t)phys * HS + d0) = kq;
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(v_cache) + head_base + (size_t)phys * HS + d0) = vq;
      if (lane == 0) {
        k_scale[head_base / HS + phys] = ksc;
        v_scale[head_base / HS + phys] = vsc;
      }
    } else {
    if constexpr (!STEP) {
      uint4* kd = reinterpret_cast<uint4*>(k_cache + head_base + (size_t)phys * HS + d0);
      uint4* vd = reinterpret_cast<uint4*>(v_cache + head_base + (size_t)phys * HS + d0);
      kd[0] = make_uint4(out[0], out[1], out[2], out[3]); kd[1] = make_uint4(out[4], out[5], out[6], out[7]);
      vd[0] = va; vd[1] = vb;
    }
    bf16x8_to_f32(va, vf); bf16x8_to_f32(vb, vf + 8);
    }
    float sc = 0.f;
#pragma unroll
    for (int e = 0; e < 16; ++e) sc = fmaf(q[e], kf[e], sc);
    sc += __shfl_xor_sync(0x000000ffu, sc, 1);
    sc += __shfl_xor_sync(0x000000ffu, sc, 2);
    sc += __shfl_xor_sync(0x000000ffu, sc, 4);
    const float mn = fmaxf(m, sc);
    const float corr = __expf(m - mn), pj = __expf(sc - mn);
    l = l * corr + pj;
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[e] = fmaf(pj, vf[e], acc[e] * corr);
    m = mn;
  }
  // ---- old rows, sub-tile by sub-tile: warp w takes rows 8 w .. 8 w + 7 (4 keys per round, 8 lanes per key)
  for (int i = 0; i < n_sub; ++i) {
    const int buf = i & 1;
    const int cnt = min(FD_SUB, n_old - i * FD_SUB);
    const uint32_t par = (uint32_t)(i >> 1) & 1u;
    mbar_wait(bar0 + buf * 8, par);
    const __nv_bfloat16* kt = reinterpret_cast<const __nv_bfloat16*>(fsm + buf * 2 * FD_SUB_BYTES);
    const __nv_bfloat16* vt = kt + FD_SUB * HS;
    stamp();
    // the warp's 8 keys of this sub-tile as two groups of 4 (8 lanes per key): both scores first (independent chains),
    // ONE running-max update, then both value rows -- half the dependent (m, l, acc) updates of a key-by-key loop
    float sc[2];
    bool valid[2];
    const uint4* vr[2];
    int rcs[2];   // KV8: the rows' index into the scales
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int r = warp * 8 + it * 4 + grp;
      valid[it] = r < cnt;
      const int rc = valid[it] ? r : 0;
      float kf[16];
      if constexpr (KV8) {
        const uint8_t* kt8 = fsm + buf * 2 * FD_SUB_BYTES;
        rcs[it] = i * FD_SUB + rc;
        vr[it] = reinterpret_cast<const uint4*>(kt8 + FD_SUB_BYTES + (size_t)rc * HS + d0);
        kv8_to_f32(*reinterpret_cast<const uint4*>(kt8 + (size_t)rc * HS + d0), sks[rcs[it]], kf);
      } else {
      const uint4* kr = reinterpret_cast<const uint4*>(kt + (size_t)rc * HS + d0);
      vr[it] = reinterpret_cast<const uint4*>(vt + (size_t)rc * HS + d0);
      bf16x8_to_f32(kr[0], kf); bf16x8_to_f32(kr[1], kf + 8);
      }
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { a0 = fmaf(q[e], kf[e], a0); a1 = fmaf(q[8 + e], kf[8 + e], a1); }
      sc[it] = a0 + a1;
    }
#pragma unroll
    for (int o = 1; o <= 4; o <<= 1) {
      sc[0] += __shfl_xor_sync(0xffffffffu, sc[0], o);
      sc[1] += __shfl_xor_sync(0xffffffffu, sc[1], o);
    }
    {
      const float s0 = valid[0] ? sc[0] : -INFINITY, s1 = valid[1] ? sc[1] : -INFINITY;
      const float mn = fmaxf(m, fmaxf(s0, s1));
      if (mn != -INFINITY) {   // at least one key so far in this lane group
        const float corr = __expf(m - mn), p0 = __expf(s0 - mn), p1 = __expf(s1 - mn);   // exp(-inf) = 0
        float v0[16], v1[16];
        if constexpr (KV8) {
          kv8_to_f32(vr[0][0], svs[rcs[0]], v0);
          kv8_to_f32(vr[1][0], svs[rcs[1]], v1);
        } else {
        bf16x8_to_f32(vr[0][0], v0); bf16x8_to_f32(vr[0][1], v0 + 8);
        bf16x8_to_f32(vr[1][0], v1); bf16x8_to_f32(vr[1][1], v1 + 8);
        }
        l = l * corr + p0 + p1;
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[e] = fmaf(p1, v1[e], fmaf(p0, v0[e], acc[e] * corr));
        m = mn;
      }
    }
    __syncthreads();   // every warp is done with this buffer
    stamp();
    if (threadIdx.x == 0 && i + 2 < n_sub) request(i + 2);
  }
  if (threadIdx.x == 0) tl_max(tl, 2);
  __syncwarp();
  if (threadIdx.x == 0) tl_max(tl, 3);
  // ---- merge the 32 (warp, key group) partials of the CTA.  smem_merge: every group leaves its row in shared memory (the
  // K / V ring is idle now: every requested sub-tile has been consumed behind a __syncthreads), one warp turns the 32
  // running maxima into weights, 128 threads add.  Otherwise: the 4 key groups of a warp merge with shuffles first
  // (36 per warp), then the 8 warps through shared memory -- the default: measured 1.1 % faster per token at position
  // 1030 on the same box (tools/env_sweep.sh "B2L_ATTN_SMEM_MERGE=0 B2L_ATTN_SMEM_MERGE=1").
  float* part = reinterpret_cast<float*>(fsm);                 // [32][HS]
  float* pm = part + 32 * HS;                                  // [32] running max, [32] sum, [32] weight, M, Ls
  float* pl = pm + 32, *pw = pl + 32;
  const int n_part = smem_merge ? 32 : FD_WARPS;
  if (smem_merge) {
    const int g = warp * 4 + grp;
    float4* dst = reinterpret_cast<float4*>(part + g * HS + d0);
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[i] = make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
    if (sub == 0) { pm[g] = m; pl[g] = l; }
  } else {
#pragma unroll
    for (int off = 8; off <= 16; off <<= 1) {   // lanes with the same `sub` hold the same dims
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
    if (lane == 0) { pm[warp] = m; pl[warp] = l; }
    if (grp == 0) {
      float4* dst = reinterpret_cast<float4*>(part + warp * HS + d0);
#pragma unroll
      for (int i = 0; i < 4; ++i) dst[i] = make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
  __syncthreads();
  if (warp == 0) {
    const float mi = lane < n_part ? pm[lane] : -INFINITY;
    const float Mx = warp_max(mi);
    const float wi = (mi == -INFINITY) ? 0.f : __expf(mi - Mx);
    const float Lx = warp_sum(lane < n_part ? pl[lane] * wi : 0.f);
    pw[lane] = wi;
    if (lane == 0) { pw[32] = Mx; pw[33] = Lx; }
  }
  __syncthreads();
  const float M = pw[32], Ls = pw[33];
  const int d = threadIdx.x & (HS - 1);
  const bool writer = threadIdx.x < HS;
  float a = 0.f;
  if (writer) {
#pragma unroll 8
    for (int g = 0; g < n_part; ++g) a = fmaf(part[g * HS + d], pw[g], a);
  }
  stamp();
  if (n_active == 1) {  // nothing to merge
    if constexpr (ADAPTER) {
      if (writer) y[(size_t)b * C + h * HS + d] = adapter_combine(a / Ls, ay, bf2f(pre_gate[h]));
    } else {
      if (writer) y[(size_t)b * C + h * HS + d] = f2bf(a / Ls);
    }
    if (threadIdx.x == 0) tl_max(tl, 4);
    stamp();
    return;
  }
  float* out = work + ((size_t)bh * n_split + sp) * (HS + 2);
  if (threadIdx.x == 0) { out[0] = M; out[1] = Ls; }
  if (writer) out[2 + d] = a;
  __syncthreads();  // all partial stores of this CTA are ordered before the ticket (cumulative release below)
  if (threadIdx.x == 0) {
    int t;
    asm volatile("atom.add.acq_rel.gpu.global.s32 %0, [%1], 1;" : "=r"(t) : "l"(tickets + bh) : "memory");
    sm_last = (t == n_active - 1);
    if (sm_last) tickets[bh] = 0;  // every contributor has arrived: safe to re-arm for the next step
  }
  __syncthreads();  // thread 0's acquire + this barrier order the other CTAs' partials before the loads below
  stamp();
  if (!sm_last) return;
  // merge: every load is issued before the first use (n_split <= 8 for S <= 2048; larger S loops in batches)
  const float* base = work + (size_t)bh * n_split * (HS + 2);
  float MM = -INFINITY, LL = 0.f, aa = 0.f;
  for (int s0 = 0; s0 < n_active; s0 += 8) {
    float ms[8], ls[8], as[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int s2 = s0 + i;
      const bool ok = s2 < n_active;
      const float* bp = base + (size_t)(ok ? s2 : s0) * (HS + 2);
      ms[i] = ok ? __ldcg(bp) : -INFINITY;
      ls[i] = ok ? __ldcg(bp + 1) : 0.f;
      as[i] = ok ? __ldcg(bp + 2 + d) : 0.f;
    }
    float bm = MM;
#pragma unroll
    for (int i = 0; i < 8; ++i) bm = fmaxf(bm, ms[i]);
    const float c0 = (MM == -INFINITY) ? 0.f : __expf(MM - bm);
    LL *= c0; aa *= c0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float wg = (ms[i] == -INFINITY) ? 0.f : __expf(ms[i] - bm);
      LL += ls[i] * wg;
      aa += as[i] * wg;
    }
    MM = bm;
  }
  if constexpr (ADAPTER) {
    if (writer) y[(size_t)b * C + h * HS + d] = adapter_combine(aa / LL, ay, bf2f(pre_gate[h]));
  } else {
    if (writer) y[(size_t)b * C + h * HS + d] = f2bf(aa / LL);
  }
  if (threadIdx.x == 0) tl_max(tl, 4);
}

// ----------------------------------------------------------------------------------
// LLaMA-Adapter prefix term for every attention shape the fused kernel above does not cover (T > 1, no cache, other
// head sizes, B2L_F_ATTN_UNFUSED): grid (B*T, n_head), 4 warps.  Reads the rotated q that rope_append_kernel left in
// qkv and adds the gated prefix attention into y in place (adapter.py:164-167, same rounding chain as the fused kernel).
// ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(ATT_WARPS * 32)
    attn_adapter_prefix_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ pk,
                               const __nv_bfloat16* __restrict__ pv, const __nv_bfloat16* __restrict__ gate,
                               __nv_bfloat16* __restrict__ y, int n_head, int hs, int alen) {
  pdl_launch_dependents();
  __shared__ float sq[32 * ATT_MAX_EPL];
  __shared__ float ssc[B2L_ADAPTER_MAX_LEN];
  const int bt = blockIdx.x, h = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = n_head * hs;
  const float scale = rsqrtf((float)hs);
  const __nv_bfloat16* q = qkv + (size_t)bt * 3 * C + h * hs;
  for (int d = threadIdx.x; d < hs; d += blockDim.x) sq[d] = bf2f(q[d]) * scale;
  __syncthreads();
  const __nv_bfloat16* kb = pk + (size_t)h * alen * hs;
  const __nv_bfloat16* vb = pv + (size_t)h * alen * hs;
  for (int j = warp; j < alen; j += ATT_WARPS) {
    float s = 0.f;
    for (int d = lane; d < hs; d += 32) s = fmaf(sq[d], bf2f(kb[(size_t)j * hs + d]), s);
    s = warp_sum(s);
    if (lane == 0) ssc[j] = s;
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = 0; j < alen; ++j) mx = fmaxf(mx, ssc[j]);
  float l = 0.f;
  for (int j = 0; j < alen; ++j) l += __expf(ssc[j] - mx);
  const float g = bf2f(gate[h]);
  __nv_bfloat16* yr = y + (size_t)bt * C + h * hs;
  for (int d = threadIdx.x; d < hs; d += blockDim.x) {
    float a = 0.f;
    for (int j = 0; j < alen; ++j) a = fmaf(__expf(ssc[j] - mx), bf2f(vb[(size_t)j * hs + d]), a);
    yr[d] = adapter_combine(bf2f(yr[d]), a / l, g);
  }
}

// ----------------------------------------------------------------------------------
// Prefill / no-cache attention for head_size 128 and T > 1 (model.py:200-230 over many query positions): a tiled
// online-softmax kernel on the tensor cores (mma.sync.m16n8k16 bf16, fp32 accumulate).  Round 1 gave every query row
// its own CTA that re-read all its keys from L2 (13B, 8 x 512 tokens: 153 ms of a 315 ms prefill); here a CTA owns
// 64 query rows of one head (4 warps x 16 rows), streams 64-key K / V tiles through a double-buffered shared-memory
// ring (cp.async, rows gathered through the cache ring), computes S = Q K^T and O += P V with ldmatrix-fed MMAs.
// Scores are scaled and exponentiated in fp32; P enters the second MMA as bf16 hi + lo parts (2^-17 relative), so the
// result matches an fp32 softmax(q k^T / sqrt(hs)) v to the final bf16 rounding.
// q is read from qkv (already rotated by rope_append_kernel); the mask is "slot <= position of the query"
// (model.py:94-96 through the tril rows selected by input_pos).
// ----------------------------------------------------------------------------------
constexpr int PF_Q = 64, PF_K = 64, PF_LD = 136;               // padded row: 128 + 8 elements (272 B) -> conflict-free ldmatrix
constexpr int PF_TILE_BYTES = PF_Q * PF_LD * 2;                 // 17408
constexpr int PF_SMEM_BYTES = 5 * PF_TILE_BYTES;                // Q + 2 x (K, V)

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr) : "memory");
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void pf_cp16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// bf16 hi / lo split of two fp32 values: hi = bf16(x), lo = bf16(x - hi)
__device__ __forceinline__ void split_bf16x2(float x, float y, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
  const __nv_bfloat162 l = __floats2bfloat162_rn(x - __low2float(h), y - __high2float(h));
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// RAGGED (b2l_attention_ragged): grid (n_head, sum over sequences of ceil(len / 64)); blockIdx.y walks the (sequence,
// 64-query tile) pairs in sequence order.  A CTA runs exactly what a B = 1, T = len launch runs for that tile: queries
// at positions t0..t0+63 of the sequence (rows past its end repeat its last one), keys from slot 0 of its cache row,
// no ring (the caller restarts the row's ring at 0).  input_pos and ring_start are unused; T is the sequence's length.
// SELF (with RAGGED, b2l_attention_ragged_kv8): the keys are the sequence's own rotated rows in qkv, not its cache row:
// `kv` views qkv (b_stride = s_stride = 3 C, S = 0) and its row index is the sequence's first packed token, so a CTA
// runs exactly what the B = 1, T = len no-cache launch (attn_prefill_kernel<false>) runs for that tile.
template <bool RAGGED, bool SELF = false>
__global__ void __launch_bounds__(128)
    attn_prefill_kernel(const __nv_bfloat16* __restrict__ qkv, KvView kv, const int64_t* __restrict__ input_pos,
                        const int32_t* __restrict__ ring_start, __nv_bfloat16* __restrict__ y, int T, int n_head,
                        const __grid_constant__ b2l_ragged rg) {
  static_assert(RAGGED || !SELF, "SELF walks the sequences of a ragged launch");
  constexpr int HS = 128;
  extern __shared__ __align__(128) uint8_t psm[];
  const uint32_t sq = smem_u32(psm), sk0 = sq + PF_TILE_BYTES;   // K tile of buffer b at sk0 + 2 b TILE, V tile right behind it
  int b, h, t0;
  size_t tok0 = 0;   // RAGGED: packed row of the sequence's token 0 in qkv and y
  if constexpr (RAGGED) {
    int s = 0, tile = blockIdx.y;
    for (; s < rg.n_seq - 1; ++s) {   // prefix sums over <= 16 sequences
      const int nt = (rg.len[s] + PF_Q - 1) / PF_Q;
      if (tile < nt) break;
      tile -= nt;
    }
    b = rg.row[s];
    h = blockIdx.x;
    t0 = tile * PF_Q;
    T = rg.len[s];
    tok0 = (size_t)rg.start[s];
  } else {
    const int bh = blockIdx.x;
    b = bh / n_head;
    h = bh % n_head;
    t0 = blockIdx.y * PF_Q;
  }
  // packed row of the CTA's query t in qkv and y
  auto tok = [&](int t) -> size_t { return RAGGED ? tok0 + t : (size_t)b * T + t; };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const int C = n_head * HS;
  const int cap = kv.S > 0 ? kv.S : T;
  const int ring = (!RAGGED && kv.S > 0 && ring_start) ? *ring_start : 0;
  const size_t kv_row = SELF ? tok0 : (size_t)b;
  const __nv_bfloat16* kb = kv.k + kv_row * kv.b_stride + (size_t)h * kv.h_stride;
  const __nv_bfloat16* vb = kv.v + kv_row * kv.b_stride + (size_t)h * kv.h_stride;

  // valid slots of this thread's two query rows (g and g + 8 of the warp's 16), and of the whole CTA
  int Lrow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int t = min(t0 + warp * 16 + g + 8 * i, T - 1);
    const long long p = (!RAGGED && input_pos) ? input_pos[t] : (long long)t;
    Lrow[i] = (int)(p < cap ? p : (long long)cap - 1) + 1;
  }
  __shared__ int s_lmax;
  if (tid == 0) s_lmax = 0;
  __syncthreads();
  atomicMax(&s_lmax, max(Lrow[0], Lrow[1]));
  // ---- Q tile (rows beyond T repeat row T - 1: never stored)
  for (int q = tid; q < PF_Q * 16; q += 128) {
    const int r = q >> 4, c = q & 15;
    const int t = min(t0 + r, T - 1);
    pf_cp16(sq + (r * PF_LD + c * 8) * 2, qkv + tok(t) * 3 * C + h * HS + c * 8);
  }
  __syncthreads();
  const int Lmax = s_lmax;
  const int n_kb = (Lmax + PF_K - 1) / PF_K;
  auto load_kv = [&](int kbi, int buf) {
    const uint32_t dk = sk0 + buf * 2 * PF_TILE_BYTES, dv = dk + PF_TILE_BYTES;
    for (int q = tid; q < PF_K * 16; q += 128) {
      const int r = q >> 4, c = q & 15;
      int j = min(kbi * PF_K + r, Lmax - 1);     // rows beyond the last valid slot repeat it (masked below)
      if (kv.S > 0) { j += ring; if (j >= kv.S) j -= kv.S; }
      pf_cp16(dk + (r * PF_LD + c * 8) * 2, kb + (size_t)j * kv.s_stride + c * 8);
      pf_cp16(dv + (r * PF_LD + c * 8) * 2, vb + (size_t)j * kv.s_stride + c * 8);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  load_kv(0, 0);   // group 0 also carries the Q tile
  uint32_t qf[8][4];
  float o[16][4];
#pragma unroll
  for (int n = 0; n < 16; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) o[n][i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const float scale = rsqrtf((float)HS);

  for (int kbi = 0; kbi < n_kb; ++kbi) {
    const int buf = kbi & 1;
    if (kbi + 1 < n_kb) {
      load_kv(kbi + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    if (kbi == 0) {   // Q fragments: 8 k-steps of 16 dims
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const int mi = lane >> 3;
        ldsm_x4(sq + ((warp * 16 + (mi & 1) * 8 + (lane & 7)) * PF_LD + ks * 16 + (mi >> 1) * 8) * 2, qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
      }
    }
    const uint32_t ksm = sk0 + buf * 2 * PF_TILE_BYTES, vsm = ksm + PF_TILE_BYTES;
    // ---- S = Q K^T for 64 keys: 8 n-tiles of 8 keys
    float sacc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int i = 0; i < 4; ++i) sacc[nt][i] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 8; ks += 2) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(ksm + ((nt * 8 + (lane & 7)) * PF_LD + ks * 16 + (lane >> 3) * 8) * 2, b0, b1, b2, b3);
        mma_bf16(sacc[nt], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b0, b1);
        mma_bf16(sacc[nt], qf[ks + 1][0], qf[ks + 1][1], qf[ks + 1][2], qf[ks + 1][3], b2, b3);
      }
    }
    // ---- scale, mask (slot < valid slots of the row), online softmax; lane (g, t4) holds rows g / g + 8, keys 8 nt + 2 t4 (+1)
    float mnew[2] = {mrow[0], mrow[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int key = kbi * PF_K + nt * 8 + 2 * t4 + (i & 1);
        const float v = (key < Lrow[i >> 1]) ? sacc[nt][i] * scale : -INFINITY;
        sacc[nt][i] = v;
        mnew[i >> 1] = fmaxf(mnew[i >> 1], v);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mnew[r] = fmaxf(mnew[r], __shfl_xor_sync(0xffffffffu, mnew[r], 1));
      mnew[r] = fmaxf(mnew[r], __shfl_xor_sync(0xffffffffu, mnew[r], 2));
    }
    float corr[2], psum[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) corr[r] = (mrow[r] == -INFINITY) ? 0.f : __expf(mrow[r] - mnew[r]);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float pj = (sacc[nt][i] == -INFINITY) ? 0.f : __expf(sacc[nt][i] - mnew[i >> 1]);
        sacc[nt][i] = pj;
        psum[i >> 1] += pj;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      lrow[r] = lrow[r] * corr[r] + psum[r];   // per-lane partial row sums; reduced across the quad at the end
      mrow[r] = mnew[r];
    }
#pragma unroll
    for (int n = 0; n < 16; ++n) {
      o[n][0] *= corr[0]; o[n][1] *= corr[0]; o[n][2] *= corr[1]; o[n][3] *= corr[1];
    }
    // ---- O += P V: 4 k-steps of 16 keys, 16 n-tiles of 8 dims; P as bf16 hi + lo
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t ah[4], al[4];
      split_bf16x2(sacc[2 * kk][0], sacc[2 * kk][1], ah[0], al[0]);          // row g,     keys 16 kk + 2 t4 (+1)
      split_bf16x2(sacc[2 * kk][2], sacc[2 * kk][3], ah[1], al[1]);          // row g + 8
      split_bf16x2(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1], ah[2], al[2]);  // row g,     keys 16 kk + 8 + 2 t4 (+1)
      split_bf16x2(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3], ah[3], al[3]);  // row g + 8
#pragma unroll
      for (int dn = 0; dn < 16; dn += 2) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(vsm + ((kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * PF_LD + dn * 8 + (lane >> 4) * 8) * 2, b0, b1, b2, b3);
        mma_bf16(o[dn], ah[0], ah[1], ah[2], ah[3], b0, b1);
        mma_bf16(o[dn], al[0], al[1], al[2], al[3], b0, b1);
        mma_bf16(o[dn + 1], ah[0], ah[1], ah[2], ah[3], b2, b3);
        mma_bf16(o[dn + 1], al[0], al[1], al[2], al[3], b2, b3);
      }
    }
    __syncthreads();   // this buffer is refilled two iterations later
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
    lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = t0 + warp * 16 + g + 8 * r;
    if (t < T) {
      const float inv = 1.0f / lrow[r];
      __nv_bfloat16* dst = y + tok(t) * C + h * HS + 2 * t4;
#pragma unroll
      for (int n = 0; n < 16; ++n)
        *reinterpret_cast<__nv_bfloat162*>(dst + n * 8) = __floats2bfloat162_rn(o[n][2 * r] * inv, o[n][2 * r + 1] * inv);
    }
  }
}

static inline void split_plan(int T, int S, int* n_split, int* chunk) {
  if (T > 1) { *n_split = 1; *chunk = S; return; }
  *chunk = 64;
  *n_split = (S + 63) / 64;
}

// stepwise (B2L_F_STEPWISE): each of the T queries takes the T == 1 split plan, so it merges its keys in the order a
// T == 1 launch at its position does
static int launch_attn(const __nv_bfloat16* qkv, KvView kv, const int64_t* input_pos, const int32_t* ring_start,
                       float* work, __nv_bfloat16* y, int B, int T, int n_head, int hs, int cap, int pos_stride,
                       bool stepwise, cudaStream_t st) {
  static const int env_pf = [] { const char* e = getenv("B2L_ATTN_PREFILL"); return e ? atoi(e) : 1; }();
  if (hs == 128 && T > 1 && env_pf && !stepwise) {   // tiled tensor-core kernel (B2L_ATTN_PREFILL=0: the per-query path below)
    static DynSmemCache smem_cache;
    if (int rc = ensure_dyn_smem(attn_prefill_kernel<false>, PF_SMEM_BYTES, smem_cache)) return rc;
    attn_prefill_kernel<false><<<dim3(B * n_head, (T + PF_Q - 1) / PF_Q), 128, PF_SMEM_BYTES, st>>>(qkv, kv, input_pos, ring_start, y, T,
                                                                                                    n_head, b2l_ragged{});
    B2L_LAUNCH_CHECK("attn_prefill_kernel");
    return 0;
  }
  int n_split, chunk;
  split_plan(stepwise ? 1 : T, cap, &n_split, &chunk);
  dim3 grid(B * n_head, T, n_split), block(ATT_WARPS * 32);
  if (hs == 128)
    attn_partial_kernel<4><<<grid, block, 0, st>>>(qkv, kv, input_pos, ring_start, work, T, n_head, hs, n_split, chunk,
                                                   pos_stride);
  else
    attn_partial_kernel<0><<<grid, block, 0, st>>>(qkv, kv, input_pos, ring_start, work, T, n_head, hs, n_split, chunk,
                                                   pos_stride);
  B2L_LAUNCH_CHECK("attn_partial_kernel");
  attn_combine_kernel<<<dim3(B * n_head, T), 128, 0, st>>>(work, y, T, n_head, hs, n_split);
  B2L_LAUNCH_CHECK("attn_combine_kernel");
  return 0;
}

// a LLaMA-Adapter prefix (b2l_adapter_prefix) before any launch: 0, or B2L_E_* with the message naming `who`
int check_adapter_prefix(const b2l_adapter_prefix* pre, const char* who) {
  B2L_CHECK_ARG(pre != nullptr && pre->k != nullptr && pre->v != nullptr && pre->gate != nullptr,
                "%s: null adapter prefix pointer", who);
  B2L_CHECK_SUPPORTED(pre->len > 0 && pre->len <= B2L_ADAPTER_MAX_LEN, "%s: adapter prefix length %d unsupported (1..%d)",
                      who, pre->len, B2L_ADAPTER_MAX_LEN);
  B2L_CHECK_ARG(((uintptr_t)pre->k & 15) == 0 && ((uintptr_t)pre->v & 15) == 0 && ((uintptr_t)pre->gate & 1) == 0,
                "%s: adapter prefix k / v must be 16-byte aligned, gate 2-byte aligned", who);
  return 0;
}

}  // namespace b2l

using namespace b2l;

static inline size_t ws_partials_bytes(int B, int n_head, int head_size, int T, int S) {
  int n_split, chunk;
  split_plan(T, S, &n_split, &chunk);
  size_t a = (size_t)B * n_head * T * n_split * (head_size + 2) * sizeof(float);
  size_t f = (size_t)B * n_head * ((S + WS_CHUNK - 1) / WS_CHUNK) * (head_size + 2) * sizeof(float);
  return ((a > f ? a : f) + 15) & ~(size_t)15;
}

// [partials | int32 tickets[B*n_head]].  The caller zero-fills the buffer once when it
// allocates it; the fused decode kernel re-arms its tickets itself.
extern "C" size_t b2l_attn_workspace_bytes(int B, int n_head, int head_size, int T, int S) {
  return ws_partials_bytes(B, n_head, head_size, T, S) + (size_t)B * n_head * sizeof(int);
}

extern "C" int b2l_ring_advance(const int64_t* input_pos, int T, int32_t* ring_start, int S, b2l_stream_t stream) {
  B2L_CHECK_ARG(input_pos && ring_start && T > 0 && S > 0, "b2l_ring_advance: bad argument");
  ring_advance_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(input_pos, T, ring_start, S);
  B2L_LAUNCH_CHECK("ring_advance_kernel");
  return 0;
}

extern "C" int b2l_ring_advance_rows(const int64_t* input_pos, int B, int32_t* ring_start, int S, b2l_stream_t stream) {
  B2L_CHECK_ARG(input_pos && ring_start, "b2l_ring_advance_rows: null pointer");
  B2L_CHECK_ARG(B > 0 && S > 0, "b2l_ring_advance_rows: bad shape (B=%d, S=%d)", B, S);
  ring_advance_rows_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(input_pos, B, ring_start, S);
  B2L_LAUNCH_CHECK("ring_advance_rows_kernel");
  return 0;
}

static int launch_adapter_prefix(const void* qkv, const b2l_adapter_prefix* pre, void* y, int B, int T, int n_head,
                                 int head_size, cudaStream_t st) {
  attn_adapter_prefix_kernel<<<dim3(B * T, n_head), ATT_WARPS * 32, 0, st>>>(
      (const __nv_bfloat16*)qkv, (const __nv_bfloat16*)pre->k, (const __nv_bfloat16*)pre->v,
      (const __nv_bfloat16*)pre->gate, (__nv_bfloat16*)y, n_head, head_size, pre->len);
  B2L_LAUNCH_CHECK("attn_adapter_prefix_kernel");
  return 0;
}

// B2L_F_ROW_POS (input_pos int64[B], ring_start int32[B]) is one query per row: T == 1, and the RoPE table (not
// B2L_F_ROPE_ROWS, whose T selected rows cannot serve B positions)
static int check_row_pos(int flags, int T, const char* who) {
  if (!(flags & B2L_F_ROW_POS)) return 0;
  B2L_CHECK_SUPPORTED(T == 1, "%s: B2L_F_ROW_POS runs one token per row (T == 1), got T=%d", who, T);
  B2L_CHECK_SUPPORTED(!(flags & B2L_F_ROPE_ROWS), "%s: B2L_F_ROW_POS does not combine with B2L_F_ROPE_ROWS", who);
  return 0;
}

// B2L_F_STEPWISE: T = 2..16 consecutive tokens of ONE sequence (B == 1), input_pos int64[T] from the RoPE table
static int check_stepwise(int flags, int B, int T, const char* who) {
  if (!(flags & B2L_F_STEPWISE)) return 0;
  B2L_CHECK_SUPPORTED(!(flags & B2L_F_ROW_POS), "%s: B2L_F_STEPWISE does not combine with B2L_F_ROW_POS", who);
  B2L_CHECK_SUPPORTED(!(flags & B2L_F_ROPE_ROWS), "%s: B2L_F_STEPWISE does not combine with B2L_F_ROPE_ROWS", who);
  B2L_CHECK_SUPPORTED(B == 1, "%s: B2L_F_STEPWISE runs the tokens of one sequence (B == 1), got B=%d", who, B);
  B2L_CHECK_SUPPORTED(T >= 2 && T <= 16, "%s: B2L_F_STEPWISE runs 2..16 tokens, got T=%d", who, T);
  return 0;
}

namespace b2l {
// b2l_attention's argument checks (`who` names the caller): 0, or B2L_E_* with a message
int check_attention(const void* qkv, const void* k_cache, const void* v_cache, const void* rope, const int64_t* input_pos,
                    const int32_t* ring_start, const void* y, const void* work, int B, int T, int n_head, int head_size,
                    int S, int block_size, int flags, const char* who) {
  B2L_CHECK_ARG(qkv && k_cache && v_cache && rope && input_pos && ring_start && y && work, "%s: null pointer", who);
  B2L_CHECK_ARG(B > 0 && T > 0 && n_head > 0 && S > 0 && T <= S && block_size > 0, "%s: bad shape", who);
  B2L_CHECK_SUPPORTED(head_size % 2 == 0 && head_size >= 2 && head_size <= 32 * ATT_MAX_EPL,
                      "%s: head_size %d unsupported (even, <= %d)", who, head_size, 32 * ATT_MAX_EPL);
  if (int rc = check_stepwise(flags, B, T, who)) return rc;
  return check_row_pos(flags, T, who);
}

// b2l_attention, b2l_attention_adapter and b2l_decode_step, after check_attention (and check_adapter_prefix when pre
// != nullptr); timeline: the fused kernel's debug stamps (uint64[64]), or nullptr
int attention_impl(void* qkv, void* k_cache, void* v_cache, const void* rope, const int64_t* input_pos,
                   const int32_t* ring_start, void* y, void* work, int B, int T, int n_head, int head_size, int S,
                   int block_size, int flags, const b2l_adapter_prefix* pre, void* timeline, cudaStream_t st) {
  const int pos_stride = (flags & B2L_F_ROW_POS) ? 1 : 0;
  const bool step = (flags & B2L_F_STEPWISE) != 0;
  if ((T == 1 || step) && head_size == 128 && !(flags & B2L_F_ROPE_ROWS) && !(flags & B2L_F_ATTN_UNFUSED)) {
    const int n_split = (S + FD_SUB - 1) / FD_SUB;
    // stepwise: the T queries are laid out as T rows of a T == 1 launch (partials and tickets of
    // b2l_attn_workspace_bytes(T, n_head, 128, 1, S))
    const int rows = step ? T : B;
    int* tickets = reinterpret_cast<int*>(reinterpret_cast<char*>(work) + ws_partials_bytes(rows, n_head, head_size, step ? 1 : T, S));
    if (step) {   // every new key / value row first, qkv untouched (the fused kernel rotates q and its own key itself)
      rope_append_kernel<false><<<dim3(T, n_head), 64, 0, st>>>((__nv_bfloat16*)qkv, (__nv_bfloat16*)k_cache, (__nv_bfloat16*)v_cache,
                                                        (const float*)rope, input_pos, ring_start, T, n_head, head_size, S,
                                                        block_size, 0, 0, 0, b2l_ragged{});
      B2L_LAUNCH_CHECK("rope_append_kernel");
    }
    // B2L_ATTN_PRE (read once): sub-tiles requested before griddepcontrol.wait, 1 (default) or 2
    static const int env_pre = [] { const char* e = getenv("B2L_ATTN_PRE"); return e ? atoi(e) : 1; }();
    // B2L_ATTN_SMEM_MERGE (read once): 1 = all 32 key groups merge through shared memory, 0 = shuffles inside a warp first
    // (default 0: the extra block barrier of 1 is not free)
    static const int env_smem_merge = [] { const char* e = getenv("B2L_ATTN_SMEM_MERGE"); return e ? atoi(e) : 0; }();
    // stepwise: no programmatic dependent launch, because the kernel requests old cache rows before
    // griddepcontrol.wait and the append launch in front of it writes some of them
    LaunchCfg lc(dim3(rows * n_head, n_split), dim3(FD_WARPS * 32), FD_SMEM_BYTES, st, (flags & B2L_F_PDL) != 0 && !step);
    static DynSmemCache smem_cache[2][3];   // [ADAPTER][shared position, ROWS, STEP]: the six instantiations share one function type
    auto launch = [&](auto kernel, const b2l_adapter_prefix* pf) -> int {
      if (int rc = ensure_dyn_smem(kernel, FD_SMEM_BYTES, smem_cache[pf != nullptr][step ? 2 : pos_stride])) return rc;
      B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, kernel, (const __nv_bfloat16*)qkv, (__nv_bfloat16*)k_cache,
                                  (__nv_bfloat16*)v_cache, (const float*)rope, input_pos, ring_start, (__nv_bfloat16*)y,
                                  (float*)work, tickets, n_head, S, block_size, n_split, (unsigned long long*)timeline, env_pre, env_smem_merge,
                                  FD_CTAS_PER_SM * sm_count(), (const __nv_bfloat16*)(pf ? pf->k : nullptr),
                                  (const __nv_bfloat16*)(pf ? pf->v : nullptr), (const __nv_bfloat16*)(pf ? pf->gate : nullptr),
                                  pf ? pf->len : 0, (float*)nullptr, (float*)nullptr));
      return 0;
    };
    if (step)
      return pre == nullptr ? launch(attn_decode_fused_kernel<false, false, true>, nullptr)
                            : launch(attn_decode_fused_kernel<true, false, true>, pre);
    if (pre == nullptr)
      return pos_stride ? launch(attn_decode_fused_kernel<false, true, false>, nullptr)
                        : launch(attn_decode_fused_kernel<false, false, false>, nullptr);
    return pos_stride ? launch(attn_decode_fused_kernel<true, true, false>, pre)
                      : launch(attn_decode_fused_kernel<true, false, false>, pre);
  }
  int rt = head_size / 2 < 32 ? 32 : head_size / 2;
  rope_append_kernel<false><<<dim3(B * T, n_head), rt, 0, st>>>((__nv_bfloat16*)qkv, (__nv_bfloat16*)k_cache,
                                                        (__nv_bfloat16*)v_cache, (const float*)rope, input_pos,
                                                        ring_start, T, n_head, head_size, S, block_size, (flags & B2L_F_ROPE_ROWS) ? 1 : 0,
                                                        pos_stride, 1, b2l_ragged{});
  B2L_LAUNCH_CHECK("rope_append_kernel");
  KvView kv{(const __nv_bfloat16*)k_cache, (const __nv_bfloat16*)v_cache, (size_t)n_head * S * head_size,
            (size_t)S * head_size, (size_t)head_size, S};
  if (int rc = launch_attn((const __nv_bfloat16*)qkv, kv, input_pos, ring_start, (float*)work, (__nv_bfloat16*)y, B, T,
                           n_head, head_size, S, pos_stride, step, st))
    return rc;
  return pre == nullptr ? 0 : launch_adapter_prefix(qkv, pre, y, B, T, n_head, head_size, st);
}

// the pointers of a non-null b2l_kv8_cache (`who` names the caller): 0, or B2L_E_ARG with a message
static int check_kv8_cache(const b2l_kv8_cache* kv, const char* who) {
  B2L_CHECK_ARG(kv->k && kv->v && kv->k_scale && kv->v_scale, "%s: null fp8 cache pointer (b2l_kv8_cache)", who);
  B2L_CHECK_ARG(((uintptr_t)kv->k & 15) == 0 && ((uintptr_t)kv->v & 15) == 0 && ((uintptr_t)kv->k_scale & 3) == 0 &&
                    ((uintptr_t)kv->v_scale & 3) == 0,
                "%s: fp8 cache codes must be 16-byte aligned, scales 4-byte aligned", who);
  return 0;
}

// b2l_attention_kv8's argument checks (`who` names the caller): 0, or B2L_E_* with a message
int check_attention_kv8(const void* qkv, const b2l_kv8_cache* kv, const void* rope, const int64_t* input_pos,
                        const int32_t* ring_start, const void* y, const void* work, int B, int T, int n_head,
                        int head_size, int S, int block_size, int flags, const char* who) {
  B2L_CHECK_ARG(qkv && kv && rope && ring_start && y && work, "%s: null pointer", who);
  if (int rc = check_kv8_cache(kv, who)) return rc;
  B2L_CHECK_ARG(B > 0 && T > 0 && n_head > 0 && S > 0 && T <= S && T <= block_size && block_size > 0, "%s: bad shape", who);
  B2L_CHECK_SUPPORTED(head_size == 128, "%s: the fp8 KV cache runs head_size 128 only (every LLaMA size), got %d", who,
                      head_size);
  B2L_CHECK_SUPPORTED(!(flags & B2L_F_STEPWISE), "%s: the fp8 KV cache does not run B2L_F_STEPWISE (speculative verify)", who);
  B2L_CHECK_SUPPORTED(!(flags & B2L_F_ATTN_UNFUSED), "%s: the fp8 KV cache runs the fused decode kernel only (not B2L_F_ATTN_UNFUSED)",
                      who);
  B2L_CHECK_SUPPORTED(!(flags & B2L_F_ROPE_ROWS), "%s: the fp8 KV cache reads the RoPE table (not B2L_F_ROPE_ROWS)", who);
  if (T > 1) {
    B2L_CHECK_SUPPORTED(input_pos == nullptr,
                        "%s: T > 1 is a prefill at positions 0..T-1 and takes input_pos == NULL (a prefill into an fp8 cache at a nonzero position is not supported)",
                        who);
    B2L_CHECK_SUPPORTED(!(flags & B2L_F_ROW_POS), "%s: B2L_F_ROW_POS runs one token per row (T == 1), got T=%d", who, T);
  } else {
    B2L_CHECK_ARG(input_pos != nullptr, "%s: T == 1 needs input_pos", who);
  }
  return 0;
}

// b2l_attention_kv8 and b2l_decode_step under B2L_F_KV_FP8, after check_attention_kv8 (and check_adapter_prefix when
// pre != nullptr); timeline as for attention_impl
int attention_kv8_impl(void* qkv, const b2l_kv8_cache* kv, const void* rope, const int64_t* input_pos,
                       const int32_t* ring_start, void* y, void* work, int B, int T, int n_head, int S, int flags,
                       int block_size, const b2l_adapter_prefix* pre, void* timeline, cudaStream_t st) {
  constexpr int HS = 128;
  if (T > 1) {   // prefill from position 0: quantize into the cache, attend over the prompt's own bf16 rows
    rope_append_kv8_kernel<false><<<dim3(B * T, n_head), HS / 2, 0, st>>>((__nv_bfloat16*)qkv, (uint8_t*)kv->k,
                                                                         (uint8_t*)kv->v, kv->k_scale, kv->v_scale,
                                                                         (const float*)rope, ring_start, T, n_head, S,
                                                                         b2l_ragged{});
    B2L_LAUNCH_CHECK("rope_append_kv8_kernel");
    const int C = n_head * HS;
    const __nv_bfloat16* base = (const __nv_bfloat16*)qkv;
    KvView kvv{base + C, base + 2 * C, (size_t)T * 3 * C, (size_t)HS, (size_t)3 * C, 0};
    if (int rc = launch_attn(base, kvv, nullptr, nullptr, (float*)work, (__nv_bfloat16*)y, B, T, n_head, HS, T, 0, false, st))
      return rc;
    return pre == nullptr ? 0 : launch_adapter_prefix(qkv, pre, y, B, T, n_head, HS, st);
  }
  const int n_split = (S + FD_SUB - 1) / FD_SUB;
  int* tickets = reinterpret_cast<int*>(reinterpret_cast<char*>(work) + ws_partials_bytes(B, n_head, HS, 1, S));
  static const int env_pre = [] { const char* e = getenv("B2L_ATTN_PRE"); return e ? atoi(e) : 1; }();
  static const int env_smem_merge = [] { const char* e = getenv("B2L_ATTN_SMEM_MERGE"); return e ? atoi(e) : 0; }();
  constexpr int smem = FD_SMEM_BYTES + 2 * FD_CHUNK * 4;   // + the CTA's old-row scales
  LaunchCfg lc(dim3(B * n_head, n_split), dim3(FD_WARPS * 32), smem, st, (flags & B2L_F_PDL) != 0);
  static DynSmemCache smem_cache[2][2];   // [ADAPTER][ROWS]
  const int rows = (flags & B2L_F_ROW_POS) ? 1 : 0;
  auto launch = [&](auto kernel) -> int {
    if (int rc = ensure_dyn_smem(kernel, smem, smem_cache[pre != nullptr][rows])) return rc;
    B2L_CUDA(cudaLaunchKernelEx(&lc.cfg, kernel, (const __nv_bfloat16*)qkv, (__nv_bfloat16*)kv->k, (__nv_bfloat16*)kv->v,
                                (const float*)rope, input_pos, ring_start, (__nv_bfloat16*)y, (float*)work, tickets, n_head,
                                S, block_size, n_split, (unsigned long long*)timeline, env_pre, env_smem_merge,
                                FD_CTAS_PER_SM * sm_count(), (const __nv_bfloat16*)(pre ? pre->k : nullptr),
                                (const __nv_bfloat16*)(pre ? pre->v : nullptr),
                                (const __nv_bfloat16*)(pre ? pre->gate : nullptr), pre ? pre->len : 0, kv->k_scale,
                                kv->v_scale));
    return 0;
  };
  if (pre == nullptr)
    return rows ? launch(attn_decode_fused_kernel<false, true, false, true>)
                : launch(attn_decode_fused_kernel<false, false, false, true>);
  return rows ? launch(attn_decode_fused_kernel<true, true, false, true>)
              : launch(attn_decode_fused_kernel<true, false, false, true>);
}
}  // namespace b2l

extern "C" int b2l_attention_kv8(void* qkv, const b2l_kv8_cache* kv, const void* rope, const int64_t* input_pos,
                                 const int32_t* ring_start, void* y, void* work, int B, int T, int n_head, int head_size,
                                 int S, int block_size, int flags, const b2l_adapter_prefix* prefix, b2l_stream_t stream) {
  if (int rc = check_attention_kv8(qkv, kv, rope, input_pos, ring_start, y, work, B, T, n_head, head_size, S, block_size,
                                   flags, "b2l_attention_kv8"))
    return rc;
  if (int rc = check_row_pos(flags, T, "b2l_attention_kv8")) return rc;
  if (prefix != nullptr) {
    if (int rc = check_adapter_prefix(prefix, "b2l_attention_kv8")) return rc;
  }
  return attention_kv8_impl(qkv, kv, rope, input_pos, ring_start, y, work, B, T, n_head, S, flags, block_size, prefix,
                            nullptr, (cudaStream_t)stream);
}

static int kv8_unroll(const void* code, const float* scale, const int32_t* ring_start, void* out, int B, int n_head, int S,
                      int head_size, int ring_stride, b2l_stream_t stream, const char* who) {
  B2L_CHECK_ARG(code && scale && ring_start && out, "%s: null pointer", who);
  B2L_CHECK_ARG(B > 0 && n_head > 0 && S > 0 && head_size > 0, "%s: bad shape", who);
  kv8_unroll_kernel<<<dim3(B * n_head, S), 64, 0, (cudaStream_t)stream>>>((const uint8_t*)code, scale, ring_start,
                                                                          (__nv_bfloat16*)out, S, head_size, n_head,
                                                                          ring_stride);
  B2L_LAUNCH_CHECK("kv8_unroll_kernel");
  return 0;
}

extern "C" int b2l_kv8_unroll(const void* code, const float* scale, const int32_t* ring_start, void* out, int B,
                              int n_head, int S, int head_size, b2l_stream_t stream) {
  return kv8_unroll(code, scale, ring_start, out, B, n_head, S, head_size, 0, stream, "b2l_kv8_unroll");
}

extern "C" int b2l_kv8_unroll_rows(const void* code, const float* scale, const int32_t* ring_start, void* out, int B,
                                   int n_head, int S, int head_size, b2l_stream_t stream) {
  return kv8_unroll(code, scale, ring_start, out, B, n_head, S, head_size, 1, stream, "b2l_kv8_unroll_rows");
}

extern "C" int b2l_attention(void* qkv, void* k_cache, void* v_cache, const void* rope, const int64_t* input_pos,
                             const int32_t* ring_start, void* y, void* work, int B, int T, int n_head,
                             int head_size, int S, int block_size, int flags, b2l_stream_t stream) {
  if (int rc = check_attention(qkv, k_cache, v_cache, rope, input_pos, ring_start, y, work, B, T, n_head, head_size, S,
                               block_size, flags, "b2l_attention"))
    return rc;
  return attention_impl(qkv, k_cache, v_cache, rope, input_pos, ring_start, y, work, B, T, n_head, head_size, S,
                        block_size, flags, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int b2l_attention_adapter(void* qkv, void* k_cache, void* v_cache, const void* rope,
                                     const int64_t* input_pos, const int32_t* ring_start, void* y, void* work, int B,
                                     int T, int n_head, int head_size, int S, int block_size, int flags,
                                     const b2l_adapter_prefix* prefix, b2l_stream_t stream) {
  if (int rc = check_attention(qkv, k_cache, v_cache, rope, input_pos, ring_start, y, work, B, T, n_head, head_size, S,
                               block_size, flags, "b2l_attention_adapter"))
    return rc;
  if (int rc = check_adapter_prefix(prefix, "b2l_attention_adapter")) return rc;
  return attention_impl(qkv, k_cache, v_cache, rope, input_pos, ring_start, y, work, B, T, n_head, head_size, S,
                        block_size, flags, prefix, nullptr, (cudaStream_t)stream);
}

static int attention_nocache_impl(void* qkv, const void* rope, void* y, void* work, int B, int T, int n_head,
                                  int head_size, int block_size, cudaStream_t st) {
  int rt = head_size / 2 < 32 ? 32 : head_size / 2;
  rope_append_kernel<false><<<dim3(B * T, n_head), rt, 0, st>>>((__nv_bfloat16*)qkv, nullptr, nullptr, (const float*)rope,
                                                        nullptr, nullptr, T, n_head, head_size, 0, block_size, 0, 0, 1, b2l_ragged{});
  B2L_LAUNCH_CHECK("rope_append_kernel");
  const int C = n_head * head_size;
  const __nv_bfloat16* base = (const __nv_bfloat16*)qkv;
  KvView kv{base + C, base + 2 * C, (size_t)T * 3 * C, (size_t)head_size, (size_t)3 * C, 0};
  return launch_attn(base, kv, nullptr, nullptr, (float*)work, (__nv_bfloat16*)y, B, T, n_head, head_size, T, 0, false, st);
}

extern "C" int b2l_attention_nocache(void* qkv, const void* rope, void* y, void* work, int B, int T, int n_head,
                                     int head_size, int block_size, b2l_stream_t stream) {
  B2L_CHECK_ARG(qkv && rope && y && work && B > 0 && T > 0 && n_head > 0 && T <= block_size,
                "b2l_attention_nocache: bad argument");
  B2L_CHECK_SUPPORTED(head_size % 2 == 0 && head_size >= 2 && head_size <= 32 * ATT_MAX_EPL,
                      "b2l_attention_nocache: head_size %d unsupported", head_size);
  return attention_nocache_impl(qkv, rope, y, work, B, T, n_head, head_size, block_size, (cudaStream_t)stream);
}

extern "C" int b2l_attention_nocache_adapter(void* qkv, const void* rope, void* y, void* work, int B, int T,
                                             int n_head, int head_size, int block_size,
                                             const b2l_adapter_prefix* prefix, b2l_stream_t stream) {
  B2L_CHECK_ARG(qkv && rope && y && work && B > 0 && T > 0 && n_head > 0 && T <= block_size,
                "b2l_attention_nocache_adapter: bad argument");
  B2L_CHECK_SUPPORTED(head_size % 2 == 0 && head_size >= 2 && head_size <= 32 * ATT_MAX_EPL,
                      "b2l_attention_nocache_adapter: head_size %d unsupported", head_size);
  if (int rc = check_adapter_prefix(prefix, "b2l_attention_nocache_adapter")) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = attention_nocache_impl(qkv, rope, y, work, B, T, n_head, head_size, block_size, st)) return rc;
  return launch_adapter_prefix(qkv, prefix, y, B, T, n_head, head_size, st);
}

// The checks b2l_attention_ragged and b2l_attention_ragged_kv8 share, after their own null-pointer checks (`who` names
// the caller; sequences are min_len..S tokens long): 0, or B2L_E_* with a message.  *tiles: the (sequence, 64-query
// tile) pairs of attn_prefill_kernel's grid.
static int check_ragged(const b2l_ragged& rg, int N, int B_rows, int n_head, int head_size, int S, int block_size,
                        int min_len, const b2l_adapter_prefix* prefix, const char* who, int* tiles) {
  B2L_CHECK_ARG(N > 0 && B_rows > 0 && n_head > 0 && S > 0 && block_size > 0,
                "%s: bad shape (N=%d, B_rows=%d, n_head=%d, S=%d, block_size=%d)", who, N, B_rows, n_head, S, block_size);
  B2L_CHECK_SUPPORTED(head_size == 128, "%s: head_size %d unsupported (128 only)", who, head_size);
  B2L_CHECK_ARG(rg.n_seq >= 1 && rg.n_seq <= B2L_RAGGED_MAX_SEQ, "%s: n_seq %d outside 1..%d", who, rg.n_seq,
                B2L_RAGGED_MAX_SEQ);
  int next = 0;
  *tiles = 0;
  for (int s = 0; s < rg.n_seq; ++s) {
    B2L_CHECK_ARG(rg.len[s] >= min_len && rg.len[s] <= S, "%s: sequence %d has length %d (%d..S=%d)", who, s, rg.len[s],
                  min_len, S);
    B2L_CHECK_ARG(rg.start[s] == next, "%s: sequence %d starts at %d, not %d (starts must tile [0, N))", who, s,
                  rg.start[s], next);
    B2L_CHECK_ARG(rg.row[s] >= 0 && rg.row[s] < B_rows, "%s: sequence %d names row %d of %d", who, s, rg.row[s], B_rows);
    for (int o = 0; o < s; ++o)
      B2L_CHECK_ARG(rg.row[o] != rg.row[s], "%s: sequences %d and %d both name row %d", who, o, s, rg.row[s]);
    next += rg.len[s];
    *tiles += (rg.len[s] + PF_Q - 1) / PF_Q;
  }
  B2L_CHECK_ARG(next == N, "%s: the sequences cover %d tokens, N=%d (starts must tile [0, N))", who, next, N);
  return prefix == nullptr ? 0 : check_adapter_prefix(prefix, who);
}

extern "C" int b2l_attention_ragged(void* qkv, void* k_cache, void* v_cache, const void* rope, const b2l_ragged* seqs,
                                    int32_t* ring_start, void* y, int N, int B_rows, int n_head, int head_size, int S,
                                    int block_size, const b2l_adapter_prefix* prefix, b2l_stream_t stream) {
  B2L_CHECK_ARG(qkv && k_cache && v_cache && rope && seqs && ring_start && y, "b2l_attention_ragged: null pointer");
  const b2l_ragged& rg = *seqs;
  int tiles;
  if (int rc = check_ragged(rg, N, B_rows, n_head, head_size, S, block_size, 1, prefix, "b2l_attention_ragged", &tiles))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rope_append_kernel<true><<<dim3(N, n_head), head_size / 2, 0, st>>>((__nv_bfloat16*)qkv, (__nv_bfloat16*)k_cache,
                                                                      (__nv_bfloat16*)v_cache, (const float*)rope, nullptr,
                                                                      ring_start, 0, n_head, head_size, S, block_size, 0,
                                                                      0, 1, rg);
  B2L_LAUNCH_CHECK("rope_append_kernel (ragged)");
  KvView kv{(const __nv_bfloat16*)k_cache, (const __nv_bfloat16*)v_cache, (size_t)n_head * S * head_size,
            (size_t)S * head_size, (size_t)head_size, S};
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(attn_prefill_kernel<true>, PF_SMEM_BYTES, smem_cache)) return rc;
  attn_prefill_kernel<true><<<dim3(n_head, tiles), 128, PF_SMEM_BYTES, st>>>((const __nv_bfloat16*)qkv, kv, nullptr,
                                                                             nullptr, (__nv_bfloat16*)y, 0, n_head, rg);
  B2L_LAUNCH_CHECK("attn_prefill_kernel (ragged)");
  return prefix == nullptr ? 0 : launch_adapter_prefix(qkv, prefix, y, 1, N, n_head, head_size, st);
}

extern "C" int b2l_attention_ragged_kv8(void* qkv, const b2l_kv8_cache* kv, const void* rope, const b2l_ragged* seqs,
                                        int32_t* ring_start, void* y, int N, int B_rows, int n_head, int head_size, int S,
                                        int block_size, const b2l_adapter_prefix* prefix, b2l_stream_t stream) {
  const char* who = "b2l_attention_ragged_kv8";
  B2L_CHECK_ARG(qkv && kv && rope && seqs && ring_start && y, "%s: null pointer", who);
  if (int rc = check_kv8_cache(kv, who)) return rc;
  const b2l_ragged& rg = *seqs;
  int tiles;
  // length 2 and up: a one-token prompt's batch-1 counterpart is the T == 1 decode kernel, which scores its token as
  // the value read back, not as its bf16 value
  if (int rc = check_ragged(rg, N, B_rows, n_head, head_size, S, block_size, 2, prefix, who, &tiles)) return rc;
  for (int s = 0; s < rg.n_seq; ++s)   // the batch-1 prefill reads RoPE rows 0..len-1 of the table (T <= block_size)
    B2L_CHECK_ARG(rg.len[s] <= block_size, "%s: sequence %d has length %d, past block_size=%d", who, s, rg.len[s],
                  block_size);
  constexpr int HS = 128;
  cudaStream_t st = (cudaStream_t)stream;
  rope_append_kv8_kernel<true><<<dim3(N, n_head), HS / 2, 0, st>>>((__nv_bfloat16*)qkv, (uint8_t*)kv->k, (uint8_t*)kv->v,
                                                                   kv->k_scale, kv->v_scale, (const float*)rope,
                                                                   ring_start, 0, n_head, S, rg);
  B2L_LAUNCH_CHECK("rope_append_kv8_kernel (ragged)");
  // each sequence attends over its own rotated bf16 rows in qkv, as the batch-1 fp8 prefill does
  const int C = n_head * HS;
  const __nv_bfloat16* base = (const __nv_bfloat16*)qkv;
  KvView kvv{base + C, base + 2 * C, (size_t)3 * C, (size_t)HS, (size_t)3 * C, 0};
  static DynSmemCache smem_cache;
  if (int rc = ensure_dyn_smem(attn_prefill_kernel<true, true>, PF_SMEM_BYTES, smem_cache)) return rc;
  attn_prefill_kernel<true, true><<<dim3(n_head, tiles), 128, PF_SMEM_BYTES, st>>>(base, kvv, nullptr, nullptr,
                                                                                   (__nv_bfloat16*)y, 0, n_head, rg);
  B2L_LAUNCH_CHECK("attn_prefill_kernel (ragged, fp8 cache)");
  return prefix == nullptr ? 0 : launch_adapter_prefix(qkv, prefix, y, 1, N, n_head, HS, st);
}

extern "C" int b2l_kv_unroll(const void* cache, const int32_t* ring_start, void* out, int B, int n_head, int S,
                             int head_size, b2l_stream_t stream) {
  B2L_CHECK_ARG(cache && ring_start && out && B > 0 && n_head > 0 && S > 0 && head_size > 0,
                "b2l_kv_unroll: bad argument");
  kv_unroll_kernel<<<dim3(B * n_head, S), 64, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)cache, ring_start,
                                                                         (__nv_bfloat16*)out, S, head_size, n_head, 0);
  B2L_LAUNCH_CHECK("kv_unroll_kernel");
  return 0;
}

extern "C" int b2l_kv_unroll_rows(const void* cache, const int32_t* ring_start, void* out, int B, int n_head, int S,
                                  int head_size, b2l_stream_t stream) {
  B2L_CHECK_ARG(cache && ring_start && out, "b2l_kv_unroll_rows: null pointer");
  B2L_CHECK_ARG(B > 0 && n_head > 0 && S > 0 && head_size > 0, "b2l_kv_unroll_rows: bad shape");
  kv_unroll_kernel<<<dim3(B * n_head, S), 64, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)cache, ring_start,
                                                                         (__nv_bfloat16*)out, S, head_size, n_head, 1);
  B2L_LAUNCH_CHECK("kv_unroll_kernel");
  return 0;
}

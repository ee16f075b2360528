// Shared device/host helpers for libb200llama (sm_90a only).
#pragma once
#include <cuda.h>           // CUtensorMap and its enums only: tensor_map_encoder() fetches the encoder (no libcuda link)
#include <cudaTypedefs.h>   // PFN_cuTensorMapEncodeTiled
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>

#include "../../include/b2l.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libb200llama is written for sm_90a (H100) only"
#endif

namespace b2l {

// ---- error state (thread-local message, returned through b2l_last_error) ----
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);  // records + returns (int)e

#define B2L_CHECK_ARG(cond, ...)                  \
  do {                                            \
    if (!(cond)) {                                \
      b2l::set_error(__VA_ARGS__);                \
      return B2L_E_ARG;                           \
    }                                             \
  } while (0)
#define B2L_CHECK_SUPPORTED(cond, ...)            \
  do {                                            \
    if (!(cond)) {                                \
      b2l::set_error(__VA_ARGS__);                \
      return B2L_E_UNSUPPORTED;                   \
    }                                             \
  } while (0)
#define B2L_CUDA(call)                                          \
  do {                                                          \
    cudaError_t e_ = (call);                                    \
    if (e_ != cudaSuccess) return b2l::cuda_fail(e_, #call);    \
  } while (0)
#define B2L_LAUNCH_CHECK(name)                                       \
  do {                                                               \
    cudaError_t e_ = cudaGetLastError();                             \
    if (e_ != cudaSuccess) return b2l::cuda_fail(e_, "launch " name); \
  } while (0)

int sm_count();  // of the current device, cached per device

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device setting: remember per device what a kernel was given.
constexpr int B2L_MAX_DEVICES = 64;
struct DynSmemCache {
  size_t bytes[B2L_MAX_DEVICES] = {};
};
template <typename Kernel>
inline int ensure_dyn_smem(Kernel kernel, size_t bytes, DynSmemCache& cache) {
  int dev = 0;
  B2L_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= B2L_MAX_DEVICES) {
    B2L_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return 0;
  }
  if (bytes > cache.bytes[dev]) {
    B2L_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    cache.bytes[dev] = bytes;
  }
  return 0;
}

// cuTensorMapEncodeTiled through the runtime, resolved once; nullptr when the driver does not provide it
inline PFN_cuTensorMapEncodeTiled tensor_map_encoder() {
  static const PFN_cuTensorMapEncodeTiled encode = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) fn = nullptr;
    return (PFN_cuTensorMapEncodeTiled)fn;
  }();
  return encode;
}

// ---- small device helpers ----
__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ __nv_bfloat16 f2bf(float v) { return __float2bfloat16_rn(v); }
// round a float through bf16 (the reference keeps every intermediate in bf16)
__device__ __forceinline__ float rbf(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__device__ __forceinline__ float load_sz(const void* p, int dtype, size_t i) {
  return dtype == B2L_BF16 ? bf2f(reinterpret_cast<const __nv_bfloat16*>(p)[i])
                           : reinterpret_cast<const float*>(p)[i];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum for blockDim.x <= 1024 (multiple of 32); `red` is >= 32 floats of smem.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : 0.f;
  return warp_sum(t);
}

// Debug timeline (tools/diag.py `timeline`): per-launch uint64[8] of %globaltimer nanoseconds,
// slot 0 = min over CTAs (start), slots 1.. = max over CTAs.  nullptr = off.
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void tl_min(unsigned long long* tr, int slot) {
  if (tr != nullptr) atomicMin(tr + slot, globaltimer_ns());
}
__device__ __forceinline__ void tl_max(unsigned long long* tr, int slot) {
  if (tr != nullptr) atomicMax(tr + slot, globaltimer_ns());
}

// Programmatic dependent launch (PDL) device side.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// Coherent 16-byte global load (ld.global, never ld.global.nc).  Mandatory for data written by the PREVIOUS kernel
// when this kernel runs under programmatic dependent launch: griddepcontrol.wait orders coherent loads only, and a
// `const __restrict__` pointer lets the compiler pick the non-coherent path (LDG.E.CONSTANT).
__device__ __forceinline__ uint4 ld_coherent_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_coherent_bf16(const __nv_bfloat16* p) {
  unsigned short v;
  asm volatile("ld.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return __uint_as_float((uint32_t)v << 16);
}

// ---- sm_90 wrappers: mbarriers, TMA, named barriers, ldmatrix, int8 mma.sync, wgmma ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t a, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
}
// the arrival count as an immediate (a different instruction from mbar_init's register operand)
template <int COUNT> __device__ __forceinline__ void mbar_init_c(uint32_t a) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "n"(COUNT) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t a) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(a) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t a, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t a, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(a), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(mbar)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t mbar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
               "l"(map), "r"(mbar), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// named barriers with an immediate id, so that ptxas reserves only the barriers a kernel uses
template <int ID> __device__ __forceinline__ void bar_sync_c(int n) { asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(n) : "memory"); }
template <int ID> __device__ __forceinline__ void bar_arrive_c(int n) { asm volatile("bar.arrive %0, %1;" ::"n"(ID), "r"(n) : "memory"); }

__device__ __forceinline__ uint4 ldmatrix_x4(uint32_t addr) {
  uint4 r;
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr) : "memory");
  return r;
}

// IMMA.16832: D (16 x 8, s32) += A (16 x 32, s8 or u8, row) * B (32 x 8, s8, col)
__device__ __forceinline__ void mma_s8s8_16832(int (&d)[4], const uint4& a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_u8s8_16832(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// K-major, no-swizzle shared-memory matrix descriptor (sm_90 wgmma format):
//   core matrix = 8 rows x 16 bytes, contiguous (128 B)
//   LBO = byte distance between the two K halves of one K=16 MMA (next 8-k column)
//   SBO = byte distance between 8-row groups along N
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;                // layout_type = 0 (no swizzle), base_offset = 0
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups are pending
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// RMSNorm with the reference's bf16 rounding points (model.py:270-277, no upcast):
//   ms = bf16(mean(bf16(x*x)));  r = bf16(rsqrt(bf16(ms + eps)));  y = bf16(scale * bf16(x * r))
// `sumsq` is the fp32 sum over the row of bf16-rounded squares.
__device__ __forceinline__ float rms_rinv(float sumsq, int C, float eps) {
  float ms = rbf(sumsq / (float)C);
  float t = rbf(ms + eps);
  return rbf(1.0f / sqrtf(t));
}
__device__ __forceinline__ float rms_apply(float x, float rinv, float scale) {
  return rbf(scale * rbf(x * rinv));
}

// silu(a) * b, model.py:252: silu rounds to bf16, then the product rounds to bf16 (at the caller's store).
__device__ __forceinline__ float silu_mul1(float av, float bv) { return rbf(av / (1.0f + expf(-av))) * bv; }
// LLaMA-Adapter v2's affine of one output feature, adapter_v2.py:30-33: bf16(s * bf16(y + b)) (rounded at the store).
__device__ __forceinline__ float affine1(float y, float s, float b) { return s * rbf(y + b); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  const __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&t);
}

// Launch helper: optional PDL attribute and cluster dimension.
struct LaunchCfg {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attrs[2];
  LaunchCfg(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, int cluster_x = 1) {
    cfg = cudaLaunchConfig_t{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    int n = 0;
    if (pdl) {
      attrs[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attrs[n].val.programmaticStreamSerializationAllowed = 1;
      ++n;
    }
    if (cluster_x > 1) {
      attrs[n].id = cudaLaunchAttributeClusterDimension;
      attrs[n].val.clusterDim.x = cluster_x;
      attrs[n].val.clusterDim.y = 1;
      attrs[n].val.clusterDim.z = 1;
      ++n;
    }
    cfg.attrs = attrs;
    cfg.numAttrs = n;
  }
};

}  // namespace b2l

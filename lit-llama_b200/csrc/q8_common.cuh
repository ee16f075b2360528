// The per-output arithmetic of LLM.int8() (q8_gemv.cu, q8_gemm.cu, q8_gemv_batch.cu): one statement of each
// rounding, so every llm.int8 kernel computes the same value for the same inputs.  The activation quantisation
// CA_k = clamp(rint(fp16(x_k) * (127 / SCA)), +-127) (0 on outlier columns) stays restated in each kernel: as a
// function its fp16 argument is converted on outlier columns too, which changes the existing kernels' SASS.
#pragma once
#include <cuda_fp16.h>

namespace b2l {

// fp16(CB[o][k] * SCB[o] / 127): an outlier column's weight as the fp16 matmul sees it; wsc = SCB[o] / 127
__device__ __forceinline__ float q8_outlier_weight(int8_t w, float wsc) { return __half2float(__float2half_rn((float)w * wsc)); }
// fp16(t * (SCA * SCB / 127^2)): the int32 contraction dequantised
__device__ __forceinline__ float q8_dequant(int t, float sca, float scb) {
  return __half2float(__float2half_rn((float)t * (sca * scb * (1.0f / (127.0f * 127.0f)))));
}
// fp16(v + fp16(term)): the outlier columns' fp16 matmul added to the dequantised part
__device__ __forceinline__ float q8_add_outliers(float v, float term) { return __half2float(__float2half_rn(v + __half2float(__float2half_rn(term)))); }

}  // namespace b2l

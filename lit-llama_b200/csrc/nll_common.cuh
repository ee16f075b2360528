// Next-token NLL from bf16 logits, shared by the standalone kernel (nll.cu) and the NLL epilogue of q4_gemm_kernel
// (q4_gemm.cu).  Both reduce a row's 128 columns of a tile with the same lane layout and the same operation order, and
// merge the tiles with the same combine kernel, so the two paths give bit-identical results:
//   nll[m] = logsumexp_n(float(L[m, n])) - float(L[m, t_m]),  n over all N columns, L = bf16 logits
// The four lanes of a quad hold one row of a tile: lane q holds columns 8 c + 2 q + e (c = 0..15, e = 0, 1) in
// v[2 c + e], -inf past N.
#pragma once
#include "b2l_common.cuh"

namespace b2l {
namespace nll {

constexpr int TILE = 128;

// Workspace: partials [n_tiles][M] (max, sum of exp) | target logits [M].  Both 16-byte aligned.
__host__ __device__ inline size_t part_bytes(int M, int N) {
  return (((size_t)((N + TILE - 1) / TILE) * (size_t)M * sizeof(float2)) + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t workspace_bytes(int M, int N) {
  return part_bytes(M, N) + ((((size_t)M * sizeof(float)) + 15) & ~(size_t)15);
}

__device__ __forceinline__ long long load_target(const void* t, int i64, int m) {
  return i64 ? reinterpret_cast<const long long*>(t)[m] : (long long)reinterpret_cast<const int*>(t)[m];
}

// (max, sum of expf(v - max)) of one row's tile; every lane of the quad returns the same pair.  A tile whose columns
// are all -inf gives (-inf, 0), which adds nothing in the combine (0 * expf(-inf - mx) = 0); expf(-inf - -inf) would
// make it NaN.
__device__ __forceinline__ float2 quad_partial(const float (&v)[32]) {
  float mx = v[0];
#pragma unroll
  for (int i = 1; i < 32; ++i) mx = fmaxf(mx, v[i]);
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  const float base = mx == -INFINITY ? 0.f : mx;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) s += expf(v[i] - base);
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  return make_float2(mx, s);
}

// Row m (m < M) of tile `tile`, held by a quad (all 32 lanes must call): lane q == 0 writes the partial, and the lane
// holding the row's target column, if it lies in this tile, writes the target logit.  nc = first column of the lane.
__device__ __forceinline__ void tile_row(const float (&v)[32], int m, int M, int tile, int nc, int N, const void* targets,
                                         int tgt_i64, float2* part, float* tl) {
  const float2 pr = quad_partial(v);
  if (m >= M) return;
  if ((threadIdx.x & 3) == 0) part[(size_t)tile * M + m] = pr;
  const long long t = load_target(targets, tgt_i64, m);
  if (t < nc || t >= nc + 8 * 15 + 2 || t >= N) return;
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    if (t == nc + 8 * c) tl[m] = v[2 * c];
    if (t == nc + 8 * c + 1) tl[m] = v[2 * c + 1];
  }
}

// Validates a b2l_nll_args block for M rows (0, or B2L_E_ARG with a message).
int check_args(const b2l_nll_args* a, int M, const char* fn);

// Merges the partials into nll[M] and the window sum *nll_sum (fp64, fixed order); enqueued behind the tile kernel.
int launch_combine(const void* targets, int tgt_i64, int M, int N, const void* workspace, float* nll, double* nll_sum,
                   cudaStream_t stream);

}  // namespace nll
}  // namespace b2l

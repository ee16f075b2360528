// Next-token negative log-likelihood of a window (the loss of evaluate/*.py: cross_entropy(logits[:-1], inp[1:])),
// from bf16 logits.  Two launches:
//   logits_nll_tile_kernel: one CTA per (32 rows, 128 columns); each quad of lanes reduces one row of the tile to
//       (max, sum of exp) with the lane layout and order of q4_gemm_kernel's NLL epilogue (nll_common.cuh), and the
//       lane holding the row's target column records its logit.  q4_gemm_kernel<*, true> writes the same workspace
//       straight from its accumulators, so the logits never reach memory there;
//   nll_combine_kernel: one CTA; row m merges its tile partials in ascending tile order,
//       nll[m] = (mx + log(sum_j s_j exp(mx_j - mx))) - L[m, t_m], then the fp64 window sum in a fixed order.
#include <math.h>

#include "nll_common.cuh"

namespace b2l {
namespace nll {

constexpr int ROWS = 32;            // rows per CTA of the tile kernel: 4 warps x 8 quads
constexpr int COMBINE_THREADS = 1024;

__global__ void __launch_bounds__(128) logits_nll_tile_kernel(const __nv_bfloat16* __restrict__ L, int ldl, int M, int N,
                                                              bool vec, const void* targets, int tgt_i64, float2* part,
                                                              float* tl) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tile = blockIdx.x;
  const int m = blockIdx.y * ROWS + warp * 8 + (lane >> 2);
  const int nc = tile * TILE + 2 * (lane & 3);
  const bool row = m < M;
  const __nv_bfloat16* src = L + (size_t)(row ? m : 0) * ldl;
  float v[32];
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const int n = nc + 8 * c;
    if (!row) {   // the quad still takes part in the shuffles; nothing is written for it
      v[2 * c] = v[2 * c + 1] = 0.f;
    } else if (vec && n + 1 < N) {
      const __nv_bfloat162 p = *reinterpret_cast<const __nv_bfloat162*>(src + n);
      v[2 * c] = __low2float(p);
      v[2 * c + 1] = __high2float(p);
    } else {
      v[2 * c] = n < N ? bf2f(src[n]) : -INFINITY;
      v[2 * c + 1] = n + 1 < N ? bf2f(src[n + 1]) : -INFINITY;
    }
  }
  tile_row(v, m, M, tile, nc, N, targets, tgt_i64, part, tl);
}

__global__ void __launch_bounds__(COMBINE_THREADS) nll_combine_kernel(const void* targets, int tgt_i64, int M, int N,
                                                                      const float2* part, const float* tl, float* nll,
                                                                      double* nll_sum) {
  __shared__ double red[COMBINE_THREADS];
  const int n_tiles = (N + TILE - 1) / TILE;
  double acc = 0.0;
  for (int m = threadIdx.x; m < M; m += COMBINE_THREADS) {
    const long long t = load_target(targets, tgt_i64, m);
    float r;
    if (t < 0 || t >= N) {
      r = __int_as_float(0x7fc00000);   // NaN: no such class
    } else {
      float mx = -INFINITY;
#pragma unroll 8
      for (int j = 0; j < n_tiles; ++j) mx = fmaxf(mx, part[(size_t)j * M + m].x);
      float s = 0.f;
#pragma unroll 8
      for (int j = 0; j < n_tiles; ++j) {
        const float2 p = part[(size_t)j * M + m];
        s += p.y * expf(p.x - mx);
      }
      r = (mx + logf(s)) - tl[m];
    }
    nll[m] = r;
    acc += (double)r;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int w = COMBINE_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *nll_sum = red[0];
}

int launch_combine(const void* targets, int tgt_i64, int M, int N, const void* workspace, float* nll, double* nll_sum,
                   cudaStream_t stream) {
  const uint8_t* ws = (const uint8_t*)workspace;
  nll_combine_kernel<<<1, COMBINE_THREADS, 0, stream>>>(targets, tgt_i64, M, N, (const float2*)ws,
                                                       (const float*)(ws + part_bytes(M, N)), nll, nll_sum);
  B2L_LAUNCH_CHECK("nll_combine_kernel");
  return 0;
}

int check_args(const b2l_nll_args* a, int M, const char* fn) {
  B2L_CHECK_ARG(a != nullptr, "%s: null nll args", fn);
  B2L_CHECK_ARG(a->nll_sum != nullptr, "%s: null nll_sum", fn);
  B2L_CHECK_ARG(M == 0 || (a->targets && a->nll && a->workspace), "%s: null targets / nll / workspace", fn);
  B2L_CHECK_ARG((uintptr_t)a->workspace % 16 == 0, "%s: workspace must be 16-byte aligned", fn);
  B2L_CHECK_ARG((uintptr_t)a->nll_sum % 8 == 0 && (uintptr_t)a->nll % 4 == 0, "%s: misaligned nll / nll_sum", fn);
  B2L_CHECK_ARG((uintptr_t)a->targets % (a->targets_i64 ? 8 : 4) == 0, "%s: misaligned targets", fn);
  return 0;
}

}  // namespace nll
}  // namespace b2l

using namespace b2l;

extern "C" size_t b2l_nll_workspace_bytes(int M, int N) {
  return (M > 0 && N > 0) ? nll::workspace_bytes(M, N) : 0;
}

extern "C" int b2l_logits_nll(const void* logits, int ldl, int M, int N, const b2l_nll_args* a, b2l_stream_t stream) {
  if (int rc = nll::check_args(a, M, "b2l_logits_nll")) return rc;
  B2L_CHECK_ARG(M >= 0 && N > 0 && ldl >= N, "b2l_logits_nll: bad shape (M=%d, N=%d, ldl=%d)", M, N, ldl);
  B2L_CHECK_ARG(M == 0 || logits != nullptr, "b2l_logits_nll: null logits");
  B2L_CHECK_ARG((uintptr_t)logits % 2 == 0, "b2l_logits_nll: logits must be 2-byte aligned bf16");
  B2L_CHECK_SUPPORTED((M + nll::ROWS - 1) / nll::ROWS <= 65535, "b2l_logits_nll: M=%d is too large", M);
  cudaStream_t st = (cudaStream_t)stream;
  if (M > 0) {
    uint8_t* ws = (uint8_t*)a->workspace;
    const bool vec = ldl % 2 == 0 && (uintptr_t)logits % 4 == 0;
    dim3 grid((N + nll::TILE - 1) / nll::TILE, (M + nll::ROWS - 1) / nll::ROWS);
    nll::logits_nll_tile_kernel<<<grid, 128, 0, st>>>((const __nv_bfloat16*)logits, ldl, M, N, vec, a->targets,
                                                      a->targets_i64, (float2*)ws, (float*)(ws + nll::part_bytes(M, N)));
    B2L_LAUNCH_CHECK("logits_nll_tile_kernel");
  }
  return nll::launch_combine(a->targets, a->targets_i64, M, N, a->workspace, a->nll, a->nll_sum, st);
}

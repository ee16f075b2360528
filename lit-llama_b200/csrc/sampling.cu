// The sampling tail of generate() (generate.py:68-75) up to the probabilities:
//   logits / temperature -> top-k threshold -> where(logits < thr, -inf, logits) -> softmax
// as ONE kernel with one CTA per logits row (the reference spends ~10 launches per row, including a
// radix sort for topk), optionally followed in the same kernel by the draw itself:
// torch.multinomial(probs, 1) is argmax(probs / q) per row with q ~ Exp(1)
// (ATen/native/Distributions.cpp); the caller draws q [B, V] with torch (`empty_like(probs).exponential_(1)`,
// the same RNG consumption as multinomial) so each row's token equals the reference's for the same
// generator state, without multinomial's ~12 launches.  B rows (generate_batch's parallel samples) run
// as B CTAs of the same launch; row b reads logits + b * ld (ld == 0: every row draws from the same
// logits, the prefill's last position), noise + b * V, and writes probs + b * V and token[b].
//
// Rounding points follow the reference as it runs on the GPU in bf16:
//   * logits / temperature is a bf16 tensor: ATen multiplies by the fp32 reciprocal of the
//     scalar and rounds to bf16;
//   * the threshold is the k-th largest of those bf16 values; ties at the threshold are kept
//     (`logits < thr` is false for them), exactly like torch.where.  -0 is stored as +0, so keys, ranks and the
//     threshold follow IEEE equality (-0 == +0) and a -0 at a +0 threshold is kept; exp(±0 - max) is the same;
//   * softmax is evaluated in fp32 (exp(x - max) / sum) and rounded to bf16;
//   * the draw is argmax(bf16(p / q)) with torch.argmax's rule: the lowest index among equal maxima, and NaN (a NaN
//     logit, or scaled logits that overflow to inf) ranks above every number, so the token is always in 0..V-1.
#include "b2l_common.cuh"

namespace b2l {

constexpr int SAMP_THREADS = 1024;

__device__ __forceinline__ uint32_t bf16_key(uint16_t b) {  // monotone map: larger float -> larger key
  return (b & 0x8000u) ? (uint32_t)(uint16_t)~b : (uint32_t)(b | 0x8000u);
}

// warp-aggregated shared-memory histogram increment: lanes that hit the same bin elect one to add their count
// (after scaling, most logits share a few exponent bins -- plain atomics would serialise 32-way)
__device__ __forceinline__ void hist_add(int* hist, uint32_t bin, bool valid) {
  const uint32_t key = valid ? bin : 0xFFFFFFFFu;
  const uint32_t peers = __match_any_sync(0xffffffffu, key);
  if (valid && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
}

// warp 0: which of the 256 bins holds the `want`-th largest element (counting from bin 255 down), and the
// rank of that element inside the bin
__device__ __forceinline__ void find_bin(const int* hist, int want, int* sel_bin, int* sel_rank) {
  const int lane = threadIdx.x & 31;
  int c[8], s = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) { c[j] = hist[lane * 8 + j]; s += c[j]; }
  int incl = s;  // sum over lanes >= lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += t;
  }
  const int above = incl - s;
  if (above < want && want <= above + s) {
    int cum = above;
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      if (cum + c[j] >= want) { *sel_bin = lane * 8 + j; *sel_rank = want - cum; break; }
      cum += c[j];
    }
  }
}

__device__ __forceinline__ float bits_f(uint32_t bits16) { return __uint_as_float(bits16 << 16); }

// bf16 bits of a scaled logit as stored in `sv`: -0 becomes +0
__device__ __forceinline__ uint32_t canon_zero(uint32_t bits16) { return bits16 == 0x8000u ? 0u : bits16; }

// the draw's order, torch.argmax(p / q): a larger r wins, equal r go to the lower index.  r = bf16(p / q) is +0..+inf
// or the canonical NaN of the bf16 rounding (0x7fff), so its bits order it as a number, with NaN above +inf.
__device__ __forceinline__ bool draw_beats(uint32_t r, int i, uint32_t best, int best_i) {
  return r > best || (r == best && i < best_i);
}

// elements 8i..8i+7 of a bf16 row: one 16-byte load, or eight 2-byte loads for a row that does not start on 16 bytes
// (V or ld not a multiple of 8)
__device__ __forceinline__ uint4 load8(const __nv_bfloat16* p, int i, bool vec) {
  if (vec) return reinterpret_cast<const uint4*>(p)[i];
  const uint16_t* s = reinterpret_cast<const uint16_t*>(p) + 8 * i;
  return make_uint4(s[0] | ((uint32_t)s[1] << 16), s[2] | ((uint32_t)s[3] << 16), s[4] | ((uint32_t)s[5] << 16),
                    s[6] | ((uint32_t)s[7] << 16));
}

// One row of the sampling tail, by every thread of a SAMP_THREADS CTA; ssm: dynamic shared memory of launch_topk's size.
// probs may be the scaled-logit buffer itself (ssm, as b2l_spec_accept uses it): every 16-byte vector of it is read and
// then written by the same thread.
__device__ __forceinline__ void topk_softmax_row(const __nv_bfloat16* __restrict__ logits, float inv_temperature, int top_k,
                                                 __nv_bfloat16* probs, const __nv_bfloat16* __restrict__ noise,
                                                 long long* __restrict__ token, int V, uint8_t* ssm) {
  const bool vec = ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(noise)) & 15) == 0;
  const int Vp = (V + 7) & ~7;
  uint16_t* sv = reinterpret_cast<uint16_t*>(ssm);  // scaled logits as bf16 bits [Vp]
  uint16_t* sq = sv + Vp;                            // Exp(1) noise as bf16 bits [Vp] (only with `noise`)
  __shared__ int hist[256];
  __shared__ int sel_hi, sel_rank, sel_lo;
  __shared__ float red[32];
  __shared__ uint32_t red_b[32];
  __shared__ int red_i[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool select = top_k > 0 && top_k < V;
  const int nvec = V / 8;  // 16-byte vectors; the (V % 8) tail is handled element-wise by the first threads
  constexpr int PRE = 4;   // rounds whose global loads are issued up front (covers V <= 32768)

  // 0. every global load of the first PRE rounds is in flight before anything waits
  uint4 lpre[PRE], npre[PRE];
#pragma unroll
  for (int r = 0; r < PRE; ++r) {
    const int i = r * SAMP_THREADS + tid;
    lpre[r] = make_uint4(0, 0, 0, 0);
    npre[r] = make_uint4(0, 0, 0, 0);
    if (i < nvec) {
      lpre[r] = load8(logits, i, vec);
      if (noise != nullptr) npre[r] = load8(noise, i, vec);
    }
  }

  // 1. scale (bf16 result) and histogram of the high byte of the sortable key
  if (tid < 256) hist[tid] = 0;
  __syncthreads();
  float lmax = -INFINITY;
  const int rounds = (nvec + SAMP_THREADS - 1) / SAMP_THREADS;
#pragma unroll 1
  for (int r0 = 0; r0 < rounds; r0 += PRE) {
#pragma unroll
    for (int rr = 0; rr < PRE; ++rr) {
      const int r = r0 + rr;
      if (r >= rounds) break;   // block-uniform
      const int i = r * SAMP_THREADS + tid;
      const bool valid = i < nvec;
      uint4 v = lpre[rr];
      if (r0 > 0) { v = make_uint4(0, 0, 0, 0); if (valid) v = load8(logits, i, vec); }
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float a = rbf(__uint_as_float(w[q] << 16) * inv_temperature);
        const float b = rbf(__uint_as_float(w[q] & 0xffff0000u) * inv_temperature);
        const uint32_t ab = canon_zero(__float_as_uint(a) >> 16), bb = canon_zero(__float_as_uint(b) >> 16);
        o[q] = ab | (bb << 16);
        if (valid) lmax = fmaxf(lmax, fmaxf(a, b));
        if (select) {
          hist_add(hist, bf16_key((uint16_t)ab) >> 8, valid);
          hist_add(hist, bf16_key((uint16_t)bb) >> 8, valid);
        }
      }
      if (valid) {
        reinterpret_cast<uint4*>(sv)[i] = make_uint4(o[0], o[1], o[2], o[3]);
        if (noise != nullptr) {
          uint4 n = npre[rr];
          if (r0 > 0) n = load8(noise, i, vec);
          reinterpret_cast<uint4*>(sq)[i] = n;
        }
      }
    }
  }
  {
    const int i = nvec * 8 + tid;   // tail (fewer than 8 elements) and zero padding up to Vp
    const bool valid = i < V;
    uint16_t bits = 0xff80;         // padding: -inf, below every threshold
    if (valid) {
      const float sc = rbf(bf2f(logits[i]) * inv_temperature);
      bits = (uint16_t)canon_zero(__float_as_uint(sc) >> 16);
      lmax = fmaxf(lmax, sc);
    }
    if (i < Vp) {
      sv[i] = bits;
      if (noise != nullptr) sq[i] = valid ? *reinterpret_cast<const uint16_t*>(noise + i) : (uint16_t)0x3f80;
    }
    if (select) hist_add(hist, bf16_key(bits) >> 8, valid);
  }
  lmax = warp_max(lmax);
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  float gmax = red[lane];
  gmax = warp_max(gmax);   // every warp reduces the 32 partials itself

  const int nvp = Vp / 8;
  uint32_t thr_key = 0;  // keep everything
  if (select) {
    // 2. bin of the k-th largest (from the top), then its rank inside the bin
    if (warp == 0) find_bin(hist, top_k, &sel_hi, &sel_rank);
    __syncthreads();
    const int hi = sel_hi, rank = sel_rank;
    __syncthreads();
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int base = 0; base < nvp; base += SAMP_THREADS) {
      const int i = base + tid;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (i < nvp) v = reinterpret_cast<const uint4*>(sv)[i];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint32_t key = bf16_key((uint16_t)(hf ? (w[q] >> 16) : (w[q] & 0xffffu)));
          const bool hit = i < nvp && (int)(key >> 8) == hi && (8 * i + 2 * q + hf) < V;
          if (__any_sync(0xffffffffu, hit)) hist_add(hist, key & 0xFF, hit);
        }
      }
    }
    __syncthreads();
    if (warp == 0) { int dummy; find_bin(hist, rank, &sel_lo, &dummy); }
    __syncthreads();
    thr_key = ((uint32_t)hi << 8) | (uint32_t)sel_lo;
  }

  // 3. softmax over the kept entries: e = exp(l - max) is kept in registers for the first PRE rounds
  float sum = 0.f;
  for (int base = 0; base < nvp; base += SAMP_THREADS) {
    const int i = base + tid;
    if (i < nvp) {
      const uint4 v = reinterpret_cast<const uint4*>(sv)[i];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      bool any = false;  // with top-k, 99 % of the vectors hold no kept entry: skip their exponentials
#pragma unroll
      for (int q = 0; q < 4; ++q)
        any = any || bf16_key((uint16_t)(w[q] & 0xffffu)) >= thr_key || bf16_key((uint16_t)(w[q] >> 16)) >= thr_key;
      if (any) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t lo = w[q] & 0xffffu, hi2 = w[q] >> 16;
          if (bf16_key((uint16_t)lo) >= thr_key && lo != 0xff80u) sum += expf(bits_f(lo) - gmax);
          if (bf16_key((uint16_t)hi2) >= thr_key && hi2 != 0xff80u) sum += expf(bits_f(hi2) - gmax);
        }
      }
    }
  }
  sum = warp_sum(sum);
  __syncthreads();
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  float total = red[lane];
  total = warp_sum(total);

  // 4. probabilities (bf16) and, with `noise` (q ~ Exp(1) drawn by torch), the sample argmax(p / q) --
  // torch.multinomial's own algorithm for one draw (ATen/native/Distributions.cpp), ties to the lower index
  uint32_t best = 0;   // the bits of +0: every entry ties or beats it, at a lower index
  int best_i = 0x7fffffff;
  for (int base = 0; base < nvp; base += SAMP_THREADS) {
    const int i = base + tid;
    if (i < nvp) {
      const uint4 v = reinterpret_cast<const uint4*>(sv)[i];
      uint4 n = make_uint4(0, 0, 0, 0);
      if (noise != nullptr) n = reinterpret_cast<const uint4*>(sq)[i];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      const uint32_t nw[4] = {n.x, n.y, n.z, n.w};
      uint32_t o[4] = {0u, 0u, 0u, 0u};
      bool any = false;  // a vector without kept entries has probability 0 everywhere and cannot win the argmax
#pragma unroll
      for (int q = 0; q < 4; ++q)
        any = any || bf16_key((uint16_t)(w[q] & 0xffffu)) >= thr_key || bf16_key((uint16_t)(w[q] >> 16)) >= thr_key;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!any) break;
        uint32_t pb2[2];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint32_t bits = hf ? (w[q] >> 16) : (w[q] & 0xffffu);
          const bool kept = bf16_key((uint16_t)bits) >= thr_key && bits != 0xff80u;
          const float pv = kept ? expf(bits_f(bits) - gmax) / total : 0.f;
          const float pr = rbf(pv);
          pb2[hf] = __float_as_uint(pr) >> 16;
          if (noise != nullptr) {
            const int idx = 8 * i + 2 * q + hf;
            const uint32_t r = __float_as_uint(rbf(pr / bits_f(hf ? (nw[q] >> 16) : (nw[q] & 0xffffu))));
            if (idx < V && draw_beats(r, idx, best, best_i)) { best = r; best_i = idx; }
          }
        }
        o[q] = pb2[0] | (pb2[1] << 16);
      }
      if (probs != nullptr) {
        if (8 * i + 8 <= V && (reinterpret_cast<uintptr_t>(probs) & 15) == 0) {
          reinterpret_cast<uint4*>(probs)[i] = make_uint4(o[0], o[1], o[2], o[3]);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (8 * i + e < V) reinterpret_cast<uint16_t*>(probs)[8 * i + e] = (uint16_t)(o[e >> 1] >> (16 * (e & 1)));
        }
      }
    }
  }
  if (noise != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint32_t ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (draw_beats(ob, oi, best, best_i)) { best = ob; best_i = oi; }
    }
    __syncthreads();
    if (lane == 0) { red_b[warp] = best; red_i[warp] = best_i; }
    __syncthreads();
    if (warp == 0) {
      best = red_b[lane]; best_i = red_i[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const uint32_t ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
        if (draw_beats(ob, oi, best, best_i)) { best = ob; best_i = oi; }
      }
      if (lane == 0) *token = (long long)best_i;
    }
  }
}

__global__ void __launch_bounds__(SAMP_THREADS)
    topk_softmax_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, float inv_temperature, int top_k,
                        __nv_bfloat16* __restrict__ probs, const __nv_bfloat16* __restrict__ noise,
                        long long* __restrict__ token, int V) {
  extern __shared__ __align__(16) uint8_t ssm[];
  {  // this CTA's row
    const size_t row = blockIdx.x;
    logits += row * (size_t)ld;
    if (noise != nullptr) noise += row * (size_t)V;
    if (probs != nullptr) probs += row * (size_t)V;
    if (token != nullptr) token += row;
  }
  topk_softmax_row(logits, inv_temperature, top_k, probs, noise, token, V, ssm);
}

// bf16 bits of the draw's key bf16(a / n) for a >= 0 (see draw_beats)
__device__ __forceinline__ uint32_t draw_key(float a, float n) { return __float_as_uint(rbf(a / n)); }

// The block-wide argmax of draw_key(w(i), noise[i]) over i < V, ties to the lower index (every thread gets it).
template <class W>
__device__ __forceinline__ int block_draw(W w, const __nv_bfloat16* __restrict__ noise, int V, uint32_t* red_b, int* red_i) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t best = 0;
  int best_i = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += SAMP_THREADS) {
    const uint32_t r = draw_key(w(i), bf2f(noise[i]));
    if (draw_beats(r, i, best, best_i)) { best = r; best_i = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (draw_beats(ob, oi, best, best_i)) { best = ob; best_i = oi; }
  }
  __syncthreads();
  if (lane == 0) { red_b[warp] = best; red_i[warp] = best_i; }
  __syncthreads();
  best = red_b[lane]; best_i = red_i[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (draw_beats(ob, oi, best, best_i)) { best = ob; best_i = oi; }
  }
  return best_i;
}

// b2l_spec_accept: ONE CTA walks the T = k + 1 target rows in order.  Row t's probabilities p_t are computed by
// topk_softmax_row into shared memory (the bits b2l_topk_softmax_rows writes); the draft token of row t < k is then
// accepted or the residual is drawn and the kernel ends.  A rejection at row j never computes the rows after it.
__global__ void __launch_bounds__(SAMP_THREADS)
    spec_accept_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, float inv_temperature, int top_k,
                       const __nv_bfloat16* __restrict__ draft_probs, const long long* __restrict__ draft_tokens,
                       const float* __restrict__ u, const __nv_bfloat16* __restrict__ noise, int* __restrict__ n_accepted,
                       long long* __restrict__ token, int T, int V) {
  extern __shared__ __align__(16) uint8_t ssm[];
  __shared__ uint32_t red_b[32];
  __shared__ int red_i[32];
  const uint16_t* p = reinterpret_cast<const uint16_t*>(ssm);   // p_t as bf16 bits, after topk_softmax_row
  const int k = T - 1;
  for (int t = 0; t < T; ++t) {
    __syncthreads();   // every thread is done with the previous row's p
    topk_softmax_row(logits + (size_t)t * ld, inv_temperature, top_k, reinterpret_cast<__nv_bfloat16*>(ssm), nullptr, nullptr,
                     V, ssm);
    __syncthreads();
    if (t == k) {   // every draft token accepted: draw from the last row
      const int tok = block_draw([&](int i) { return bits_f(p[i]); }, noise, V, red_b, red_i);
      if (threadIdx.x == 0) { *n_accepted = k; *token = tok; }
      return;
    }
    const long long x = draft_tokens[t];
    const __nv_bfloat16* q = draft_probs + (size_t)t * V;
    const bool in = x >= 0 && x < V;
    if (in && u[t] * bf2f(q[x]) < bits_f(p[in ? x : 0])) continue;   // accepted (block-uniform)
    // rejected: draw from max(0, p - q); when that is zero everywhere (bf16 rounding), from p
    auto resid = [&](int i) { return fmaxf(bits_f(p[i]) - bf2f(q[i]), 0.f); };
    int any = 0;
    for (int i = threadIdx.x; i < V; i += SAMP_THREADS) any |= resid(i) > 0.f;
    int tok;
    if (__syncthreads_or(any))
      tok = block_draw(resid, noise, V, red_b, red_i);
    else
      tok = block_draw([&](int i) { return bits_f(p[i]); }, noise, V, red_b, red_i);
    if (threadIdx.x == 0) { *n_accepted = t; *token = tok; }
    return;
  }
}

constexpr int NGRAM_THREADS = 1024;

// b2l_ngram_propose: ONE CTA.  For each g from max_ngram down, the threads test the candidate starts of one chunk of
// NGRAM_THREADS at a time, from the end of the history backwards (thread t tests start hi - t), so the first chunk with
// a match holds the most recent occurrence: the match of the lowest thread.  Most lookups end in the first chunk.
__global__ void __launch_bounds__(NGRAM_THREADS)
    ngram_propose_kernel(const long long* __restrict__ history, int base_len, const int* __restrict__ n_accepted,
                         int min_ngram, int max_ngram, int k, long long* __restrict__ tokens, __nv_bfloat16* __restrict__ probs,
                         int* __restrict__ count, int V) {
  __shared__ long long pat[16];
  __shared__ int first;   // the lowest thread of the current chunk whose start matches
  const int tid = threadIdx.x;
  const long long n = base_len + (n_accepted != nullptr ? (long long)*n_accepted + 1 : 0);
  long long start = -1;
  int g = max_ngram;
  for (; g >= min_ngram; --g) {
    if (g > n - 1) continue;   // block-uniform
    // the previous g's last __syncthreads_or came after its every read of pat and first
    if (tid < g) pat[tid] = history[n - g + tid];
    if (tid == 0) first = NGRAM_THREADS;
    __syncthreads();
    for (long long hi = n - 1 - g; hi >= 0; hi -= NGRAM_THREADS) {
      const long long i = hi - tid;
      bool hit = i >= 0;
      for (int j = g - 1; hit && j >= 0; --j) hit = history[i + j] == pat[j];
      if (hit) atomicMin(&first, tid);
      if (__syncthreads_or(hit)) { start = hi - first; break; }
    }
    if (start >= 0) break;   // block-uniform
  }
  const int c = start < 0 ? 0 : (int)min((long long)k, n - (start + g));
  if (tid < c) tokens[tid] = history[start + g + tid];
  if (tid == 0) *count = c;
  if (probs == nullptr) return;
  // every element of the k rows is zeroed, then each proposed token's element set to 1.0; the barrier orders the two
  // stores to that element
  const size_t total = (size_t)k * V, nvec = total / 8;
  for (size_t v = tid; v < nvec; v += NGRAM_THREADS) reinterpret_cast<uint4*>(probs)[v] = make_uint4(0, 0, 0, 0);
  for (size_t e = nvec * 8 + tid; e < total; e += NGRAM_THREADS) reinterpret_cast<uint16_t*>(probs)[e] = 0;
  __syncthreads();
  if (tid < c) {
    const long long x = history[start + g + tid];
    if (x >= 0 && x < V) reinterpret_cast<uint16_t*>(probs)[(size_t)tid * V + x] = 0x3f80;   // bf16 1.0
  }
}

}  // namespace b2l

using namespace b2l;

static int launch_topk(const void* logits, long long ld, float temperature, int top_k, void* probs, const void* noise, void* token,
                       int B, int V, b2l_stream_t stream, const char* who) {
  B2L_CHECK_ARG(logits && V > 0 && temperature > 0.f && top_k >= 0, "%s: bad argument", who);
  B2L_CHECK_ARG(ld == 0 || ld >= V, "%s: ld = %lld: 0 (every row reads the same logits) or at least V = %d", who, ld, V);
  B2L_CHECK_ARG(((uintptr_t)logits % 16) == 0, "%s: logits must be 16-byte aligned", who);
  B2L_CHECK_ARG(noise == nullptr || ((uintptr_t)noise % 16) == 0, "%s: noise must be 16-byte aligned", who);
  const size_t Vp = ((size_t)V + 7) & ~(size_t)7;
  const size_t smem = Vp * 2 * (noise != nullptr ? 2 : 1);
  B2L_CHECK_SUPPORTED(smem <= 200 * 1024, "%s: vocabulary %d too large for one CTA", who, V);
  static DynSmemCache smem_cache;
  if (smem > 48 * 1024)
    if (int rc = ensure_dyn_smem(topk_softmax_kernel, smem, smem_cache)) return rc;
  topk_softmax_kernel<<<B, SAMP_THREADS, smem, (cudaStream_t)stream>>>((const __nv_bfloat16*)logits, ld, 1.0f / temperature, top_k,
                                                                      (__nv_bfloat16*)probs, (const __nv_bfloat16*)noise,
                                                                      (long long*)token, V);
  B2L_LAUNCH_CHECK("topk_softmax_kernel");
  return 0;
}

extern "C" int b2l_topk_softmax(const void* logits, float temperature, int top_k, void* probs, int V, b2l_stream_t stream) {
  B2L_CHECK_ARG(probs != nullptr, "b2l_topk_softmax: null probs");
  return launch_topk(logits, V, temperature, top_k, probs, nullptr, nullptr, 1, V, stream, "b2l_topk_softmax");
}

extern "C" int b2l_topk_softmax_sample(const void* logits, float temperature, int top_k, const void* noise, void* probs,
                                       int64_t* token, int V, b2l_stream_t stream) {
  B2L_CHECK_ARG(noise != nullptr && token != nullptr, "b2l_topk_softmax_sample: null noise / token");
  return launch_topk(logits, V, temperature, top_k, probs, noise, token, 1, V, stream, "b2l_topk_softmax_sample");
}

// the checks every row entry point makes before launch_topk's, each naming its argument
static int check_rows(const void* logits, int B, int V, float temperature, int top_k, const char* who) {
  B2L_CHECK_ARG(logits != nullptr, "%s: null logits", who);
  B2L_CHECK_ARG(B >= 1, "%s: B = %d rows, at least 1", who, B);
  B2L_CHECK_ARG(V > 0, "%s: V = %d, at least 1", who, V);
  B2L_CHECK_ARG(temperature > 0.f, "%s: temperature %g, must be positive", who, (double)temperature);
  B2L_CHECK_ARG(top_k >= 0, "%s: top_k = %d, 0 (no filter) or positive", who, top_k);
  return 0;
}

extern "C" int b2l_topk_softmax_rows(const void* logits, int64_t ld, float temperature, int top_k, void* probs, int B, int V,
                                     b2l_stream_t stream) {
  const char* who = "b2l_topk_softmax_rows";
  if (int rc = check_rows(logits, B, V, temperature, top_k, who)) return rc;
  B2L_CHECK_ARG(probs != nullptr, "%s: null probs", who);
  return launch_topk(logits, ld, temperature, top_k, probs, nullptr, nullptr, B, V, stream, who);
}

extern "C" int b2l_spec_accept(const void* target_logits, int64_t ld, float temperature, int top_k, const void* draft_probs,
                               const int64_t* draft_tokens, const float* u, const void* noise, int32_t* n_accepted,
                               int64_t* token, int T, int V, b2l_stream_t stream) {
  const char* who = "b2l_spec_accept";
  if (int rc = check_rows(target_logits, T, V, temperature, top_k, who)) return rc;
  B2L_CHECK_SUPPORTED(T >= 2 && T <= 16, "%s: T = %d target rows; 2..16 (k = T - 1 = 1..15 draft tokens)", who, T);
  B2L_CHECK_ARG(ld >= V, "%s: ld = %lld, at least V = %d", who, (long long)ld, V);
  B2L_CHECK_ARG(draft_probs != nullptr, "%s: null draft_probs", who);
  B2L_CHECK_ARG(draft_tokens != nullptr, "%s: null draft_tokens", who);
  B2L_CHECK_ARG(u != nullptr, "%s: null u", who);
  B2L_CHECK_ARG(noise != nullptr, "%s: null noise", who);
  B2L_CHECK_ARG(n_accepted != nullptr && token != nullptr, "%s: null n_accepted / token", who);
  B2L_CHECK_ARG(((uintptr_t)target_logits % 16) == 0, "%s: target_logits must be 16-byte aligned", who);
  B2L_CHECK_ARG(((uintptr_t)draft_probs % 16) == 0 && ((uintptr_t)noise % 16) == 0,
                "%s: draft_probs and noise must be 16-byte aligned", who);
  const size_t smem = (((size_t)V + 7) & ~(size_t)7) * 2;   // p as bf16 (topk_softmax_row without noise)
  B2L_CHECK_SUPPORTED(smem <= 200 * 1024, "%s: vocabulary %d too large for one CTA", who, V);
  static DynSmemCache smem_cache;
  if (smem > 48 * 1024)
    if (int rc = ensure_dyn_smem(spec_accept_kernel, smem, smem_cache)) return rc;
  spec_accept_kernel<<<1, SAMP_THREADS, smem, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)target_logits, (long long)ld, 1.0f / temperature, top_k, (const __nv_bfloat16*)draft_probs,
      (const long long*)draft_tokens, u, (const __nv_bfloat16*)noise, n_accepted, (long long*)token, T, V);
  B2L_LAUNCH_CHECK("spec_accept_kernel");
  return 0;
}

extern "C" int b2l_ngram_propose(const int64_t* history, int base_len, const int32_t* n_accepted, int min_ngram,
                                 int max_ngram, int k, int64_t* tokens, void* probs, int32_t* count, int V,
                                 b2l_stream_t stream) {
  const char* who = "b2l_ngram_propose";
  B2L_CHECK_ARG(history != nullptr, "%s: null history", who);
  B2L_CHECK_ARG(tokens != nullptr, "%s: null tokens", who);
  B2L_CHECK_ARG(count != nullptr, "%s: null count", who);
  B2L_CHECK_ARG(((uintptr_t)history % 8) == 0, "%s: history must be 8-byte aligned", who);
  B2L_CHECK_ARG(((uintptr_t)tokens % 8) == 0, "%s: tokens must be 8-byte aligned", who);
  B2L_CHECK_ARG(((uintptr_t)n_accepted % 4) == 0, "%s: n_accepted must be 4-byte aligned", who);
  B2L_CHECK_ARG(((uintptr_t)count % 4) == 0, "%s: count must be 4-byte aligned", who);
  B2L_CHECK_ARG(((uintptr_t)probs % 16) == 0, "%s: probs must be 16-byte aligned", who);
  B2L_CHECK_ARG(base_len >= 1, "%s: base_len = %d, at least 1", who, base_len);
  B2L_CHECK_ARG(min_ngram >= 1 && min_ngram <= max_ngram && max_ngram <= 16,
                "%s: min_ngram = %d, max_ngram = %d; 1 <= min_ngram <= max_ngram <= 16", who, min_ngram, max_ngram);
  B2L_CHECK_ARG(k >= 1 && k <= 15, "%s: k = %d; 1..15 (the verify step runs 2..16 tokens)", who, k);
  B2L_CHECK_ARG(V >= 1, "%s: V = %d, at least 1", who, V);
  ngram_propose_kernel<<<1, NGRAM_THREADS, 0, (cudaStream_t)stream>>>(
      (const long long*)history, base_len, n_accepted, min_ngram, max_ngram, k, (long long*)tokens,
      (__nv_bfloat16*)probs, count, V);
  B2L_LAUNCH_CHECK("ngram_propose_kernel");
  return 0;
}

extern "C" int b2l_topk_softmax_sample_rows(const void* logits, int64_t ld, float temperature, int top_k, const void* noise,
                                            void* probs, int64_t* tokens, int B, int V, b2l_stream_t stream) {
  const char* who = "b2l_topk_softmax_sample_rows";
  if (int rc = check_rows(logits, B, V, temperature, top_k, who)) return rc;
  B2L_CHECK_ARG(noise != nullptr, "%s: null noise", who);
  B2L_CHECK_ARG(tokens != nullptr, "%s: null tokens", who);
  return launch_topk(logits, ld, temperature, top_k, probs, noise, tokens, B, V, stream, who);
}

/*
 * b2l.h - C ABI of libb200llama.so: the H100 (sm_90a) quantized-decode path for
 * Lightning-AI/lit-llama.
 *
 * The reference has no native boundary of its own: its "operator API" for this path
 * is a set of Python nn.Module classes that lit_llama/utils.py:141-162 swaps in for
 * torch.nn.Linear, plus the model-level modules of lit_llama/model.py.  Each entry
 * point below states the reference forward it replaces (file:line relative to the
 * reference checkout).  INTEGRATION.md shows the ctypes binding a maintainer adds.
 *
 * Conventions
 *  - Every pointer is a DEVICE pointer owned by the caller (PyTorch).  The library
 *    never allocates or frees device memory on the call path and never synchronises;
 *    every call only enqueues work on `stream` and is CUDA-graph capturable.
 *  - Return value: 0 = ok, <0 = bad argument / unsupported shape (B2L_E_*),
 *    >0 = a cudaError_t.  b2l_last_error() returns a thread-local message.
 *  - There is no CPU fallback.
 *  - Activations are bf16 (B2L_BF16).  Scales/zeros may be bf16 or f32 (the
 *    reference creates them in the default dtype, quantization.py:360-369).
 */
#ifndef B2L_H_
#define B2L_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* b2l_stream_t; /* == cudaStream_t */

enum { B2L_BF16 = 0, B2L_F32 = 1 };

enum {
  B2L_E_ARG = -1,         /* null pointer / negative size / misaligned pointer      */
  B2L_E_UNSUPPORTED = -2, /* shape or mode outside what the kernels implement        */
  B2L_E_STATE = -3        /* call sequence error (e.g. model not finalised)          */
};

int b2l_version(void);
const char* b2l_last_error(void);
/* Device facts the host side sizes grids with (SM count etc.).  0 on success. */
int b2l_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------
 * ColBlockQuantizedLinear  (lit_llama/quantization.py:340-423)
 *
 * Reference storage (quantization.py:350-369, 386-390): quant_weight is uint8, logical
 * (out, in/epb) with strides (1, out) - i.e. memory is row-major (in/epb, out) - and
 * entry nr of byte [o, j] holds column epb*j+nr at bit nr*bits.  scales/zeros are
 * (out, n_groups) row-major, n_groups = ceil(in / tile_cols).
 * ---------------------------------------------------------------------------- */

/* get_weight(): dense (out, in) row-major weight, (level - zero) * scale evaluated in
 * out_dtype like quantization.py:392-411 (bit-exact with the reference). */
int b2l_q_dequant(const void* qw, const void* scales, const void* zeros, int sz_dtype,
                  void* w_out, int out_dtype, int out_features, int in_features, int bits,
                  int tile_cols, b2l_stream_t stream);

/* forward(): y[M,N] = x[M,K] @ dequant(W)^T (+ bias).  Generic kernel: any bits in
 * {4,8}, any tile_cols, any M; reads the reference layout directly.  Replaces both
 * branches of quantization.py:413-423 (the Triton kernel :187-333 and the dense
 * fallback).  x, y bf16 row-major with leading dimensions ldx, ldy (elements). */
int b2l_q_linear(const void* x, int ldx, const void* qw, const void* scales, const void* zeros,
                 int sz_dtype, const void* bias, void* y, int ldy, int M, int N, int K, int bits,
                 int tile_cols, b2l_stream_t stream);

/* One-time (load-time) re-tiling of a 4-bit, one-group-per-row weight for the
 * wgmma kernels: [N/128 tiles][K/32 slabs][128 rows][16 B].  N is padded up to a
 * multiple of 128 with zero levels.  Pure permutation of nibbles (bit-exact,
 * invertible: b2l_q4_untile).  Precedent for load-time transforms in the
 * reference: Linear8bitLt._load_from_state_dict, quantization.py:52-67. */
size_t b2l_q4_tiled_bytes(int N, int K);
int b2l_q4_tile(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream);
int b2l_q4_untile(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream);

/* Prologue / epilogue selectors of the fused linears. */
enum { B2L_PRO_NONE = 0, B2L_PRO_RMSNORM = 1 };
enum {
  B2L_EPI_STORE = 0,    /* y = bf16(acc)                                              */
  B2L_EPI_RESIDUAL = 1, /* y = bf16(bf16(acc) + res)            model.py:166-167       */
  B2L_EPI_SWIGLU = 2    /* rows interleaved [64 of c_fc1 | 64 of c_fc2] per tile:
                           y = bf16(bf16(silu(bf16(a))) * bf16(b))   model.py:252     */
};

/* LLaMA-Adapter v2's per-output-feature affine of a linear (lit_llama/adapter_v2.py:30-47):
 *   y = bf16(scale * bf16(linear(x) + bias))
 * scale, bias bf16 [N] in the row order of the weight layout in use (for B2L_EPI_SWIGLU: interleaved like the
 * weight rows).  Both NULL = off; exactly one NULL is B2L_E_ARG. */
typedef struct b2l_out_affine {
  const void* scale;
  const void* bias;
} b2l_out_affine;

#define B2L_PF_SEGMENTS 4
typedef struct b2l_q4_linear_args {
  const void* x;        /* bf16 [M, K], leading dim ldx                               */
  int ldx;
  const void* qw_tiled; /* from b2l_q4_tile                                           */
  const void* scales;   /* [N] per-row                                                */
  const void* zeros;    /* [N]                                                        */
  int sz_dtype;
  void* y;              /* bf16 [M, N_out], leading dim ldy (N_out = N/2 for SWIGLU)  */
  int ldy;
  int M, N, K;          /* M <= 16; N % 128 == 0 after padding; K % 32 == 0           */
  int prologue;         /* B2L_PRO_*                                                  */
  const void* norm_scale; /* bf16 [K] RMSNorm scale when prologue == RMSNORM          */
  float eps;
  int epilogue;         /* B2L_EPI_*                                                  */
  const void* res;      /* bf16 [M, N] residual (leading dim ldres) for RESIDUAL      */
  int ldres;
  int split_k;          /* cluster size along K: 1..8 (0 = library picks)             */
  int flags;            /* B2L_F_*                                                    */
  void* trace;          /* debug: device uint64[256] receiving clock64() stamps of CTA 0
                           (NULL = off); see tools/diag.py `trace`                     */
  void* workspace;      /* b2l_q4_gemv_batch only: b2l_q4_gemv_batch_workspace_bytes(K) bytes of device
                           scratch, 16-byte aligned (activation fragments; may be shared by all
                           launches of one stream)                                       */
  /* unused (no kernel reads them): they keep the layout of the block                           */
  const void* pf_ptr[B2L_PF_SEGMENTS];
  unsigned long long pf_bytes[B2L_PF_SEGMENTS];
  const void* pf_kv[2];
  const long long* pf_rows;
  int pf_rows_max, pf_nseg, pf_row_bytes;
  unsigned long long pf_seg_stride;
  b2l_out_affine out_affine; /* b2l_q4_gemv / b2l_w8_gemv only: the affine above, applied to the linear's bf16
                           output before the STORE / RESIDUAL / SWIGLU epilogue.  b2l_q4_linear_tc, b2l_q4_gemm,
                           b2l_w8_gemm and b2l_q4_gemv_batch return B2L_E_UNSUPPORTED when it is set (their
                           callers apply b2l_linear_affine to the output instead)                        */
} b2l_q4_linear_args;

enum {
  B2L_F_PDL = 1,        /* launch with programmatic dependent launch                   */
  B2L_F_NO_ALIAS_N = 2, /* debug: b2l_q4_linear_tc uses 16-column MMAs even for M <= 8  */
  B2L_F_ROPE_ROWS = 4,  /* b2l_attention: `rope` holds the T rows already selected by
                           input_pos (the reference's call convention, model.py:93)    */
  B2L_F_ATTN_UNFUSED = 8, /* debug: force the three-kernel attention path for T == 1   */
  B2L_F_DEBUG_NOCOMPUTE = 16, /* debug: b2l_q4_gemv streams the weights but skips the math */
  B2L_F_W8 = 32,        /* b2l_decode_step: every linear is gptq.int8, qw_mma from b2l_w8_tile_i8
                           (b2l_w8_gemv); B == 1 (2..16 with B2L_F_W8_BATCH)        */
  B2L_F_Q8 = 64,        /* b2l_decode_step: every linear is llm.int8 (b2l_decode_args::q8_layers / q8_lm_head,
                           b2l_q8_linear); B == 1, not with B2L_F_W8                   */
  B2L_F_W8_BATCH = 128, /* b2l_decode_step with B2L_F_W8 at B in 2..16: every linear runs b2l_w8_gemv_batch on
                           the b2l_w8_tile_i8 tilings in qw_mma; batch_work must hold
                           b2l_w8_gemv_batch_workspace_bytes(max K, B) bytes; no affines */
  B2L_F_Q4_BATCH_I8 = 256, /* b2l_decode_step (gptq.int4) at B in 2..16: every linear runs b2l_q4_gemv_batch_i8 on
                           the b2l_q4_tile_i8 tilings in qw_mma; batch_work must hold
                           b2l_w8_gemv_batch_workspace_bytes(max K, B) bytes; not with B2L_F_W8, B2L_F_Q8 or
                           B2L_F_W8_BATCH; no affines */
  B2L_F_Q8_BATCH = 512, /* b2l_decode_step with B2L_F_Q8 at B in 2..16: every linear runs b2l_q8_linear_batch on
                           CB / SCB in place; batch_work must hold b2l_q8_linear_batch_workspace_bytes(max K, B)
                           bytes; v2 affines allowed; not with B2L_F_W8, B2L_F_W8_BATCH or B2L_F_Q4_BATCH_I8 */
  B2L_F_ROW_POS = 1024, /* b2l_attention(_adapter) at T == 1 and b2l_decode_step: one position per row.
                           input_pos is int64[B] (row b's token is at input_pos[b]) and ring_start int32[B] (row b's
                           own ring offset); not with B2L_F_ROPE_ROWS.  The step advances each
                           row's ring on its own (b2l_ring_advance_rows) */
  B2L_F_STEPWISE = 2048, /* b2l_attention(_adapter) at B == 1, T = 2..16, and b2l_decode_step with B = 2..16: the rows
                           are consecutive tokens of ONE sequence (the verify step of speculative decoding), each
                           computed exactly as a T == 1 launch / a batch-1 step at its position would compute it.
                           See b2l_attention and b2l_decode_step; not with B2L_F_ROW_POS or B2L_F_ROPE_ROWS */
  B2L_F_GEMM_I8 = 4096, /* b2l_q4_gemm(_nll) / b2l_w8_gemm(_nll): qw_tiled is the batch-1 tiling of the layer,
                           b2l_q4_tile_i8 / b2l_w8_tile_i8 of its N rows (see b2l_q4_gemm) */
  B2L_F_GEMM_I8_LO = 8192,  /* with B2L_F_GEMM_I8: qw_tiled is a 2N-row interleaved b2l_*_tile_i8 tiling and the layer
                           is rows 0..7 of its every 16-row block (c_fc1 of the fc1|fc2 tiling); N % 8 == 0 */
  B2L_F_GEMM_I8_HI = 16384, /* the same, rows 8..15 of every 16-row block (c_fc2) */
  B2L_F_KV_FP8 = 1 << 15    /* b2l_decode_step: every layer's KV cache is fp8 (b2l_decode_args::kv8, b2l_attention_kv8);
                               on every route, not with B2L_F_STEPWISE or B2L_F_ATTN_UNFUSED; head_size 128 */
};

/* Fused [RMSNorm ->] int4 linear [-> residual | SwiGLU] on wgmma (M <= 16).  Replaces
 * RMSNorm.forward (model.py:270-277) + ColBlockQuantizedLinear.forward
 * (quantization.py:413-423) + the residual add / silu*mul of Block/MLP.forward
 * (model.py:166-167, 252). */
int b2l_q4_linear_tc(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* Prefill-shaped linear (any M; meant for M > 16): y[M, N] = x[M, K] . dequant(W)^T on wgmma (csrc/q4_gemm.cu):
 * 128 x 128 output tile per CTA, both operands from shared memory (producer warps dequantise the packed levels with
 * the reference's own bf16 roundings, so the tensor core multiplies exactly get_weight()'s matrix), fp32 accumulators
 * in registers.  Same argument block as b2l_q4_linear_tc; qw_tiled from b2l_q4_tile; prologue / epilogue must be
 * NONE / STORE; K % 64 == 0; ldx % 8 == 0.  Replaces quantization.py:187-333 (Triton tile kernel) / :413-423.
 * flags (the same for b2l_w8_gemm, b2l_q4_gemm_nll and b2l_w8_gemm_nll), any other bit is rejected:
 *   0                   qw_tiled from b2l_q4_tile (b2l_w8_gemm: quant_weight in the reference layout);
 *   B2L_F_GEMM_I8       qw_tiled from b2l_q4_tile_i8 (b2l_w8_gemm: b2l_w8_tile_i8) of the layer's N rows, the resident
 *                       copy the batch-1 kernels read; rows at or beyond N rounded up to 16 are never read;
 *   B2L_F_GEMM_I8 | B2L_F_GEMM_I8_LO / _HI
 *                       qw_tiled is that tiling of 2N interleaved rows (layer row o at 16 (o / 8) + o % 8, + 8 for _HI:
 *                       the fc1|fc2 tiling of b2l_decode_step's c_fc12), N % 8 == 0; each launch reads all 2N rows'
 *                       bytes.  Both halves together, or a half without B2L_F_GEMM_I8, are rejected.
 * Every source gives bit-identical results: the producers write the same bf16 values to the same shared memory. */
int b2l_q4_gemm(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* Batch-1 decode variant of the fused linear (M == 1): TMA-staged packed weights, PDL prefetch, persistent CTAs
 * that own 16-row blocks over the full K (no cross-CTA reduction), and an EXACT integer contraction on the legacy
 * tensor pipe: the activation row is scaled by a power of two and split into balanced base-256 digits, digit plane j
 * is column j of mma.sync.m16n8k32 (u8 x s8 -> s32), a packed byte feeds two weight rows (csrc/q4_gemv.cu).
 * Same argument block as b2l_q4_linear_tc (ldx/ldy/ldres unused; split_k > 0 overrides the grid size);
 * qw_tiled must come from b2l_q4_tile_i8: [N/16 row blocks][K/64 k blocks][32 lanes][16 B], byte = level of row g
 * (low nibble) and of row g + 8 (high nibble).  For B2L_EPI_SWIGLU the rows of a 16-row block are
 * [8 of c_fc1 | 8 of c_fc2].  K % 64 == 0, K <= 24576. */
size_t b2l_q4_tiled_i8_bytes(int N, int K);
int b2l_q4_tile_i8(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream);
int b2l_q4_untile_i8(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream);
int b2l_q4_gemv(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* gptq.int8 (8-bit levels, one (scale, zero) per row, no bias): the batch-1 kernel above with 8-bit weights.  Same
 * argument block, prologues, epilogues, B2L_F_PDL and split_k grid override as b2l_q4_gemv; flags other than
 * B2L_F_PDL / B2L_F_DEBUG_NOCOMPUTE are rejected.  qw_tiled from b2l_w8_tile_i8: [N/16 row blocks][K/64 k blocks]
 * [2 chunks][32 lanes][16 B]; in chunk c lane (g, t) holds rows g, g + 8, g, g + 8 at k = k0 .. k0+3, k0 .. k0+3,
 * k0+4 .. k0+7, k0+4 .. k0+7 (k0 = 64 kb + 32 c + 8 t), rows beyond N zero.  For B2L_EPI_SWIGLU the rows of a 16-row
 * block are [8 of c_fc1 | 8 of c_fc2].  K % 64 == 0, K <= 24576.  qw for (un)tiling: quant_weight in the reference
 * layout, uint8 [K][N]. */
size_t b2l_w8_tiled_i8_bytes(int N, int K);
int b2l_w8_tile_i8(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream);
int b2l_w8_untile_i8(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream);
int b2l_w8_gemv(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* gptq.int8 for 2..16 activation rows (batched decode) on the same resident tiling (qw_tiled from b2l_w8_tile_i8)
 * and in the same exact integer form as b2l_w8_gemv: every row is scaled, rounded and split into three base-256
 * digit planes as b2l_w8_gemv does it, and the 3 M planes are the columns of mma.m16n8k32.  Row n of y is
 * bit-identical to b2l_w8_gemv on row n alone (csrc/w8_gemv_batch.cu).  Same argument block, prologues, epilogues
 * and split_k grid override as b2l_w8_gemv, plus: x [M, K] with leading dimension ldx (ldx >= K, ldx % 8 == 0), y
 * and res with ldy / ldres, and `workspace`, b2l_w8_gemv_batch_workspace_bytes(K, M) bytes of 16-byte aligned device
 * scratch (may be shared by all launches of one stream).  M in 2..16, K % 64 == 0, K <= 24576, flags 0 or B2L_F_PDL,
 * out_affine must be unset.  Two launches: the rows' digit planes are built once (w8_batch_prep_kernel), then
 * streamed stage by stage next to the weights (w8_gemv_batch_kernel). */
size_t b2l_w8_gemv_batch_workspace_bytes(int K, int M);
int b2l_w8_gemv_batch(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* gptq.int4 for 2..16 activation rows (batched decode) on the resident batch-1 tiling (qw_tiled from b2l_q4_tile_i8)
 * and in b2l_q4_gemv's exact integer form: the kernel above with 4-bit levels, each packed byte fed to the MMA as
 * b2l_q4_gemv does (unmasked for row g, high nibble for row g + 8) and the row pair recovered from the two results.
 * Row n of y is bit-identical to b2l_q4_gemv on row n alone.  Same argument block, checks, prologues, epilogues and
 * split_k grid override as b2l_w8_gemv_batch; the digit planes are the same, so `workspace` is
 * b2l_w8_gemv_batch_workspace_bytes(K, M) bytes.  M in 2..16, K % 64 == 0, K <= 24576, flags 0 or B2L_F_PDL,
 * out_affine must be unset.  Two launches (w8_batch_prep_kernel, then w8_gemv_batch_kernel<.., false>). */
int b2l_q4_gemv_batch_i8(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* gptq.int8 for M >= 1 rows (meant for M >= 2: prompts, batched decode) on the wgmma GEMM of b2l_q4_gemm: the
 * producers dequantise the 8-bit levels with get_weight's roundings, so the tensor core multiplies exactly
 * get_weight()'s bf16 matrix.  qw_tiled is quant_weight itself in the reference layout (uint8 [K][N], no
 * re-tiled copy), or with B2L_F_GEMM_I8 (| _LO / _HI) the resident b2l_w8_tile_i8 tiling as for b2l_q4_gemm; other
 * requirements as b2l_q4_gemm (K % 64 == 0, ldx % 8 == 0, 16-byte aligned x and weights, NONE / STORE). */
int b2l_w8_gemm(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * Perplexity (evaluate/full.py:120-129 and its lora / adapter / adapter_v2 twins): the next-token NLL of one
 * window, cross_entropy(logits[:-1], inp[1:]), from the bf16 logits L of M = T - 1 rows and N columns:
 *   nll[m] = logsumexp_n(float(L[m, n])) - float(L[m, targets[m]])      (fp32, maximum-subtracted expf)
 *   *nll_sum = sum_m nll[m]                                             (fp64, fixed order)
 * Rows are reduced per 128-column tile to (max, sum of exp) in a fixed order and the tiles merged in ascending
 * order (csrc/nll.cu).  A target < 0 or >= N gives NaN for that row (and the sum).
 *   targets    int32 (targets_i64 == 0) or int64 [M], device
 *   nll        fp32 [M], device; nll_sum: one fp64, device (written, not accumulated)
 *   workspace  b2l_nll_workspace_bytes(M, N) bytes of device scratch, 16-byte aligned
 * Every call only enqueues work.
 * ---------------------------------------------------------------------------- */
typedef struct b2l_nll_args {
  const void* targets;
  int targets_i64;
  float* nll;
  double* nll_sum;
  void* workspace;
} b2l_nll_args;
size_t b2l_nll_workspace_bytes(int M, int N);
/* b2l_q4_gemm / b2l_w8_gemm with the loss in the epilogue: the fp32 accumulators are rounded to bf16 exactly as the
 * STORE epilogue would write them and reduced per tile; nothing is stored to y (y / ldy are ignored).  Same
 * requirements as b2l_q4_gemm / b2l_w8_gemm.  The result is bit-identical to b2l_logits_nll on the logits the plain
 * GEMM writes. */
int b2l_q4_gemm_nll(const b2l_q4_linear_args* args, const b2l_nll_args* nll, b2l_stream_t stream);
int b2l_w8_gemm_nll(const b2l_q4_linear_args* args, const b2l_nll_args* nll, b2l_stream_t stream);
/* The same from a bf16 logits matrix [M, N] with leading dimension ldl >= N (any N, M >= 0): for lm_heads the
 * fused form does not cover (dense, llm.int8, gptq.int4 at M <= 16, LLaMA-Adapter v2's affine). */
int b2l_logits_nll(const void* logits, int ldl, int M, int N, const b2l_nll_args* nll, b2l_stream_t stream);

/* The same fused linear for 1..8 activation rows (batched decode) on mma.sync.m16n8k16 (f16), weight tiling
 * b2l_q4_tile_mma ([N/16 row blocks][K/64 k blocks][32 lanes][16 B] in m16n8k16 A-fragment order), argument block of
 * b2l_q4_gemv plus `workspace`; x [M, K] with leading dimension ldx (ldx % 8 == 0), y / res
 * with ldy / ldres.  An mma.m16n8k16 tile has 8 columns: activation row n is column n, so 8 rows cost the MMAs
 * of one.  Two launches: the rows are normalised and converted to MMA fragment order once
 * (q4_batch_prep_kernel), then streamed stage by stage next to the weights (q4_gemv_batch_kernel).
 * Replaces the same reference code as b2l_q4_gemv for B > 1 (model.py:76-122 accepts any batch). */
size_t b2l_q4_gemv_batch_workspace_bytes(int K);
size_t b2l_q4_tiled_mma_bytes(int N, int K);
int b2l_q4_tile_mma(const void* qw, void* qw_tiled, int N, int K, b2l_stream_t stream);
int b2l_q4_untile_mma(const void* qw_tiled, void* qw, int N, int K, b2l_stream_t stream);
int b2l_q4_gemv_batch(const b2l_q4_linear_args* args, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * model.py element-wise pieces (used by the module-level drop-ins and by prefill)
 * ---------------------------------------------------------------------------- */

/* RMSNorm.forward, model.py:270-277, evaluated with the reference's bf16 rounding
 * points.  x, y bf16 [rows, C]. */
int b2l_rmsnorm(const void* x, const void* scale, void* y, int rows, int C, float eps,
                b2l_stream_t stream);

/* transformer.wte(idx), model.py:102.  idx int32 or int64 [n]; out bf16 [n, C]. */
int b2l_embedding(const void* idx, int idx_is_i64, const void* wte, void* out, int n, int C,
                  int vocab, b2l_stream_t stream);

/* silu(a) * b with the reference's bf16 rounding points, model.py:252. */
int b2l_silu_mul(const void* a, const void* b, void* y, size_t n, b2l_stream_t stream);

/* x + h, model.py:166-167. */
int b2l_add(const void* a, const void* b, void* y, size_t n, b2l_stream_t stream);

/* LLaMA-Adapter v2's linear affine (adapter_v2.py:30-33) in place on a linear's output:
 * y[m, n] = bf16(scale[n] * bf16(y[m, n] + bias[n])) for M rows of N columns, leading dimension ldy >= N.
 * y, scale, bias bf16.  Bad arguments are rejected before any launch. */
int b2l_linear_affine(void* y, int ldy, int M, int N, const void* scale, const void* bias,
                      b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * Linear8bitLt  (lit_llama/quantization.py:38-77; forward inherited from bitsandbytes:
 * LLM.int8() with has_fp16_weights=False, threshold=6.0).  CB int8 (out, in) row-major,
 * SCB fp32 (out) as produced by quantization.py:69-77.
 * ---------------------------------------------------------------------------- */
/* load-time re-tiling of CB into mma.m16n8k32 fragment order: [N/16][K/128][4][32 lanes][16 B] */
size_t b2l_q8_tiled_bytes(int N, int K);
int b2l_q8_tile(const void* cb, void* tiled, int N, int K, b2l_stream_t stream);
/* y[N] (bf16) for ONE activation row x[K] (bf16): fp16 cast, outlier columns (|a| >= threshold)
 * in fp16 against CB*SCB/127, the rest row-absmax-quantised to int8 and contracted on the tensor
 * cores, dequantised by SCA*SCB/127^2.  outlier_mask: optional K-bit mask shared by a batch
 * (b2l_q8_outlier_mask); NULL = derive it from this row. */
int b2l_q8_gemv(const void* x, const void* w_tiled, const void* cb, const void* scb,
                const void* outlier_mask, void* y, int N, int K, float threshold, int flags,
                b2l_stream_t stream);
/* b2l_q8_gemv reading CB itself (reference layout, int8 (N, K) row-major) with one bulk copy per weight row, so
 * no re-tiled copy has to exist: every output is bit-identical to b2l_q8_gemv on b2l_q8_tile(cb).
 * K a multiple of 128 up to 32768, N > 0; x and cb 16-byte aligned; flags 0 or B2L_F_PDL.
 * Bad arguments are rejected before the device is touched. */
int b2l_q8_gemv_cb(const void* x, const void* cb, const void* scb, const void* outlier_mask,
                   void* y, int N, int K, float threshold, int flags, b2l_stream_t stream);
int b2l_q8_outlier_mask(const void* x, int ldx, int M, int K, float threshold, void* mask,
                        b2l_stream_t stream);
/* The batch-1 linear above fused with its neighbours of Block.forward, for the whole-token step (B2L_F_Q8):
 *   x^ = RMSNorm(x) (prologue RMSNORM, b2l_rmsnorm's rounding points and order; NONE: x^ = x)
 *   y  = Linear8bitLt.forward(x^) exactly as b2l_q8_gemv_cb computes it (outliers, SCA and CA from x^)
 *   then out_affine (LLaMA-Adapter v2, as b2l_linear_affine), then the epilogue:
 *     STORE     out = y                     (bf16 [N])
 *     RESIDUAL  out = bf16(y + res)         (as b2l_add; res may alias out)
 *     SWIGLU    out = silu(y1) * y2         (as b2l_silu_mul on the bf16 outputs y1 of cb / scb and y2 of cb2 /
 *               scb2, both [N, K]: each 16-row block streams 8 rows of each, so no interleaved copy exists)
 * Every output is bit-identical to the module sequence b2l_rmsnorm -> b2l_q8_gemv_cb [-> b2l_linear_affine]
 * [-> b2l_add | second b2l_q8_gemv_cb + b2l_silu_mul].  For SWIGLU, out_affine's vectors hold 16 entries per 8
 * outputs: 8 of c_fc1 | 8 of c_fc2 (the layout of b2l_layer_affine::c_fc12).  K a multiple of 128 up to 32768, any
 * N > 0; x, cb, cb2 and norm_scale 16-byte aligned; out must not overlap x.  flags 0 or B2L_F_PDL: the weight ring
 * fills and norm_scale, SCB and the affine are read before griddepcontrol.wait, x and res after it.  Bad arguments
 * are rejected before the device is touched. */
typedef struct b2l_q8_linear_args {
  const void* x;            /* bf16 [K]                                                   */
  const void* cb;           /* int8 [N, K] row-major (weight.CB)                          */
  const void* scb;          /* fp32 [N]   (weight.SCB)                                    */
  const void* cb2;          /* SWIGLU only: the second linear's CB / SCB                  */
  const void* scb2;
  void* y;                  /* bf16 [N]                                                   */
  int N, K;
  float threshold;          /* outlier threshold (Linear8bitLt.threshold)                 */
  int prologue;             /* B2L_PRO_NONE / B2L_PRO_RMSNORM                             */
  const void* norm_scale;   /* bf16 [K] when prologue == RMSNORM                          */
  float eps;
  int epilogue;             /* B2L_EPI_STORE / RESIDUAL / SWIGLU                          */
  const void* res;          /* bf16 [N] for RESIDUAL                                      */
  b2l_out_affine out_affine;
  int flags;                /* 0 or B2L_F_PDL                                             */
} b2l_q8_linear_args;
int b2l_q8_linear(const b2l_q8_linear_args* args, b2l_stream_t stream);
/* b2l_q8_linear for M = 2..16 activation rows (batched decode on the whole-token step, B2L_F_Q8_BATCH): the same
 * argument block, prologues, epilogues and affine, with x [M, K] and y / res [M, N], all contiguous.  Every output is
 * bit-identical to the module sequence at M rows: b2l_rmsnorm -> b2l_q8_gemm (one outlier mask for the whole batch:
 * bit k set iff any row has |fp16(x^[m][k])| >= threshold) [-> b2l_linear_affine] [-> b2l_add | second b2l_q8_gemm +
 * b2l_silu_mul].  A row's outputs therefore depend on its batch-mates through that mask.  workspace: at least
 * b2l_q8_linear_batch_workspace_bytes(K, M) bytes of 16-byte aligned device memory (may be shared by all launches of
 * one stream).  Two launches: q8_batch_prep_kernel (one cluster of M CTAs: RMSNorm, the batch mask, SCA, CA and the
 * outlier data, into the workspace), then q8_gemv_batch_kernel, which streams CB as b2l_q8_linear does and contracts
 * all M rows per weight tile (csrc/q8_gemv_batch.cu).  K a multiple of 128 up to 32768, N > 0; x, cb, cb2,
 * norm_scale and workspace 16-byte aligned; y must not overlap x; flags 0 or B2L_F_PDL.  Bad arguments are rejected
 * before the device is touched. */
size_t b2l_q8_linear_batch_workspace_bytes(int K, int M);
int b2l_q8_linear_batch(const b2l_q8_linear_args* args, int M, void* workspace, size_t workspace_bytes,
                        b2l_stream_t stream);
/* y[M, N] (bf16, leading dimension ldy) for M activation rows x[M, K] (bf16, leading dimension
 * ldx, a multiple of 8) on the int8 wgmma tensor cores: every row bit-identical to b2l_q8_gemv
 * on that row with the batch's outlier mask (b2l_q8_outlier_mask over all M rows).  cb is CB
 * itself (reference layout, int8 (N, K) row-major); no re-tiled copy is read.  K a multiple of
 * 128 up to 32768; x, cb and workspace 16-byte aligned; flags must be 0.  workspace (at least
 * b2l_q8_gemm_workspace_bytes(M, K) bytes, device memory) receives the quantised rows CA, SCA
 * and the outlier mask; the library allocates nothing. */
size_t b2l_q8_gemm_workspace_bytes(int M, int K);
int b2l_q8_gemm(const void* x, int ldx, const void* cb, const void* scb, void* workspace,
                size_t workspace_bytes, void* y, int ldy, int M, int N, int K, float threshold,
                int flags, b2l_stream_t stream);

/* generate.py:68-75 up to the probabilities: probs = softmax(where(l < kth, -inf, l)) with
 * l = logits / temperature (bf16, rounded like ATen does on the GPU) and kth the top_k-th
 * largest l (top_k == 0: no filtering).  logits, probs bf16 [V].  One launch; the caller draws
 * with torch.multinomial so the RNG stream is the reference's. */
int b2l_topk_softmax(const void* logits, float temperature, int top_k, void* probs, int V,
                     b2l_stream_t stream);

/* generate.py:68-76 in one launch: the probabilities above AND the draw of generate.py:76
 * (torch.multinomial(probs, num_samples=1)).  For one draw ATen computes argmax(probs / q), q ~ Exp(1)
 * (ATen/native/Distributions.cpp, ties to the lower index); `noise` is that q, bf16 [V], drawn by the caller with
 * torch (`torch.empty_like(probs).exponential_(1)`: the RNG consumption of multinomial), so `*token` (device
 * int64) equals the reference's sample for the same generator state.  probs may be NULL. */
int b2l_topk_softmax_sample(const void* logits, float temperature, int top_k, const void* noise, void* probs,
                            int64_t* token, int V, b2l_stream_t stream);

/* The two entry points above over B rows in one launch (one CTA per row): parallel samples of one prompt,
 * generate.py:68-76 for every row of a batched decode step (lit_llama_b200.generate_batch).  Row b reads
 * logits + b * ld (bf16; ld == 0: every row reads the same V logits, e.g. the prefill's last position when all
 * samples share a prompt) and noise + b * V (bf16 [B, V], q ~ Exp(1) drawn by the caller as
 * `torch.empty_like(probs).exponential_(1)` on probs [B, V]), and writes probs + b * V (bf16 [B, V], may be NULL
 * for the _sample_ form) and tokens[b] (device int64 [B]).  Row b equals the B = 1 call on that row: probs bit for
 * bit, and tokens[b] == torch.multinomial(probs, 1)[b] for the same generator state (argmax(probs / q) per row, ties
 * to the lower index).  logits and noise 16-byte aligned; rows that do not start on 16 bytes (V or ld not a multiple
 * of 8) are read element-wise.  Null pointers, B < 1, 0 < ld < V (or ld < 0) and misaligned logits / noise are
 * B2L_E_ARG, with a message naming the argument, before the device is touched.  b2l_topk_softmax and
 * b2l_topk_softmax_sample are the B = 1, ld = V case. */
int b2l_topk_softmax_rows(const void* logits, int64_t ld, float temperature, int top_k, void* probs, int B, int V,
                          b2l_stream_t stream);
int b2l_topk_softmax_sample_rows(const void* logits, int64_t ld, float temperature, int top_k, const void* noise,
                                 void* probs, int64_t* tokens, int B, int V, b2l_stream_t stream);

/* Speculative sampling (accept / resample) of one verify step in one launch.  The target's T = k + 1 logits rows
 * (target_logits + t * ld, bf16, ld >= V) give p_t exactly as b2l_topk_softmax_rows computes it (bit for bit); the
 * draft proposed tokens x_0..x_{k-1} (draft_tokens int64 [k]) with probability rows q_t (draft_probs bf16 [k, V]).
 *   x_t is accepted iff u_t * q_t(x_t) < p_t(x_t) in fp32 (u fp32 [k], uniform [0, 1)); strict, so u = 0 never
 *   accepts a token the target gives probability 0.  A draft token outside 0..V-1 is rejected.
 *   j = the first rejected t:   *token = argmax_i bf16(max(0, p_j(i) - q_j(i)) / noise[i])  (the residual
 *                               distribution's draw, unnormalised); when that residual is zero everywhere (bf16
 *                               rounding only): argmax_i bf16(p_j(i) / noise[i]), a draw from p_j
 *   every x_t accepted:         *token = argmax_i bf16(p_k(i) / noise[i])
 * noise bf16 [V] is q ~ Exp(1) drawn by the caller (as for b2l_topk_softmax_sample); argmax ties go to the lower
 * index.  *n_accepted (device int32) = j, or k when every draft token is accepted; *token is device int64.
 * With top_k == 1 this is "accept while x_t == argmax p_t, then emit the target's argmax".  T in 2..16; target_logits,
 * draft_probs and noise 16-byte aligned.  Bad arguments are B2L_E_ARG / B2L_E_UNSUPPORTED with a message naming
 * the argument, before the device is touched.  One CTA walks the rows in order and stops at the first rejection. */
int b2l_spec_accept(const void* target_logits, int64_t ld, float temperature, int top_k, const void* draft_probs,
                    const int64_t* draft_tokens, const float* u, const void* noise, int32_t* n_accepted, int64_t* token,
                    int T, int V, b2l_stream_t stream);

/* Prompt-lookup proposal: draft tokens taken from the sequence itself, for b2l_spec_accept without a draft model.
 * history (device int64) holds the sequence's n tokens, n = base_len + (n_accepted ? *n_accepted + 1 : 0), read on
 * the device (n_accepted: b2l_spec_accept's device int32, so the host need not learn how many tokens the last verify
 * step emitted).  The rule, deterministic:
 *   for g = max_ngram down to min_ngram, skipping g > n - 1: the pattern is history[n-g .. n); i is the largest start
 *   with i + g <= n - 1 and history[i .. i+g) == pattern (the most recent earlier occurrence; it may overlap the
 *   pattern).  The first g with a match proposes history[i+g .. min(i+g+k, n)) into tokens[0 .. *count); tokens past
 *   *count are not written.  No match: *count = 0.
 * probs (bf16 [k, V], 16-byte aligned, may be NULL) receives the deterministic draft's rows: row t < *count is 1.0 at
 * tokens[t] and 0 elsewhere; a token outside 0..V-1 and every row t >= *count are all zero.  Fed to b2l_spec_accept,
 * x_t is then accepted iff u_t < p_t(x_t), and the residual at a rejection is p_j with x_j removed: speculative
 * sampling with a deterministic draft.  *count is device int32.  1 <= min_ngram <= max_ngram <= 16, k in 1..15,
 * base_len >= 1, V >= 1; null history / tokens / count and misaligned pointers are B2L_E_ARG with a message naming
 * the argument, before the device is touched.  One CTA. */
int b2l_ngram_propose(const int64_t* history, int base_len, const int32_t* n_accepted, int min_ngram, int max_ngram,
                      int k, int64_t* tokens, void* probs, int32_t* count, int V, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * CausalSelfAttention.forward without the two linears, model.py:197-232:
 * split qkv, apply_rope(q), apply_rope(k) (model.py:306-323), append k,v to the
 * cache at input_pos (roll-when-full branch model.py:214-218 handled on the device
 * with a ring offset), causal softmax(q k^T / sqrt(hs)) v.
 *
 * qkv   bf16 [B, T, 3*C]   (q | k | v thirds, each [nh, hs])
 * k/v cache bf16 [B, nh, S, hs]; physical slot = (logical slot + *ring_start) % S
 * rope  f32 [block_size, hs/2, 2] (cos, sin) - build_rope_cache, model.py:280-303
 * input_pos int64 [T] on the device (never read by the host).  Query t writes its
 *            k,v at logical slot min(input_pos[t], S-1) and attends slots <= that.
 * ring_start int32 [1] on the device, read-only here; b2l_ring_advance moves it
 * With B2L_F_ROW_POS (T == 1): input_pos int64 [B] and ring_start int32 [B], row b at
 *            its own position and ring offset (b2l_ring_advance_rows moves them).  Each
 *            row's y and cache rows equal a B = 1 launch on that row bit for bit.
 * With B2L_F_STEPWISE (B == 1, T = 2..16): input_pos int64 [T] holds consecutive positions
 *            p..p+T-1, all < S (no roll).  Query t's y row and its appended k / v row equal,
 *            bit for bit, a T == 1 launch at position p+t on the cache holding the tokens
 *            before it.  head_size 128: one launch appends every rotated k row and v row,
 *            then the fused kernel runs one CTA group per (t, head), without programmatic
 *            dependent launch; B2L_F_ATTN_UNFUSED and other head sizes: the three-kernel
 *            path with the T == 1 split plan per query.  work: b2l_attn_workspace_bytes(T,
 *            n_head, head_size, 1, S) bytes (T rows at T == 1).
 * y     bf16 [B, T, C]
 * work  scratch of b2l_attn_workspace_bytes(...) bytes (split-S partials + tickets);
 *       the caller zero-fills it ONCE after allocating it
 * ---------------------------------------------------------------------------- */
size_t b2l_attn_workspace_bytes(int B, int n_head, int head_size, int T, int S);
int b2l_attention(void* qkv, void* k_cache, void* v_cache, const void* rope,
                  const int64_t* input_pos, const int32_t* ring_start, void* y, void* work, int B,
                  int T, int n_head, int head_size, int S, int block_size, int flags,
                  b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * Tensor-parallel decode (new capability: every reference script is Fabric(devices=1); the split dims are the ones
 * scripts/convert_checkpoint.py:56-64 records).  One-shot all-reduce (sum, fp32 accumulation in rank order, one
 * rounding) of a bf16 row of n elements over the GPUs of one node, through peer memory: every rank pushes
 * {2 values, epoch} words into its slot of every peer's exchange buffer (NVLink stores) and polls its own buffer
 * (csrc/tp_allreduce.cu).  `out` may alias `partial`.  All ranks must issue the same sequence of calls.
 * peer_buf[r]: rank r's buffer of b2l_tp_buffer_bytes(world, max_elems) bytes as mapped into this process
 * (peer_buf[rank] = the local one), zero-filled once before the first call; epoch: 16 local device words, status:
 * one, zero-filled once.  status becomes 1 if a bounded wait timed out (the result is then undefined).
 * ---------------------------------------------------------------------------- */
typedef struct b2l_tp_comm {
  void* peer_buf[8];
  int rank, world;
  int max_elems;
  unsigned int* epoch;
  int* status;
} b2l_tp_comm;
size_t b2l_tp_buffer_bytes(int world, int max_elems);
int b2l_tp_allreduce(const b2l_tp_comm* comm, const void* partial, void* out, int n, int flags,
                     b2l_stream_t stream);

/* The roll branch of model.py:214-218 as a ring: if input_pos[T-1] >= S the ring start
 * advances by one slot (the oldest entry is dropped, exactly what torch.roll(-1) +
 * overwrite of slot S-1 does).  Call once per forward, before the layers. */
int b2l_ring_advance(const int64_t* input_pos, int T, int32_t* ring_start, int S,
                     b2l_stream_t stream);
/* The same for B rows at their own positions (B2L_F_ROW_POS): input_pos int64 [B], ring_start
 * int32 [B]; row b's ring advances when input_pos[b] >= S. */
int b2l_ring_advance_rows(const int64_t* input_pos, int B, int32_t* ring_start, int S,
                          b2l_stream_t stream);

/* Same without a cache (input_pos is None, model.py:104-106): positions 0..T-1.
 * qkv is rotated in place; work as for b2l_attention with S = T. */
int b2l_attention_nocache(void* qkv, const void* rope, void* y, void* work, int B, int T,
                          int n_head, int head_size, int block_size, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * LLaMA-Adapter (lit_llama/adapter.py:88-174): the attention above plus the gated
 * attention over a learned prefix, adapter.py:151-167:
 *   y = bf16(bf16(y) + bf16(gate[h] * bf16(softmax(q ak^T / sqrt(hs)) av)))
 * with q the rotated query, no mask and no RoPE on the prefix, and a softmax of its
 * own (not joint with the cache keys).  The prefix keys / values are the k and v
 * thirds of c_attn(adapter_wte.weight), computed once by the caller.
 *   k, v  bf16 [n_head][len][head_size], 16-byte aligned (shared by every sequence of the batch)
 *   gate  bf16 [n_head] (gating_factor)
 *   len   1..64 (adapter_prompt_length)
 * Bad arguments are rejected before any launch.  T == 1 at head_size 128 runs the
 * fused decode kernel's adapter variant (the same single launch); every other shape
 * adds one small kernel behind the attention.
 * ---------------------------------------------------------------------------- */
typedef struct b2l_adapter_prefix {
  const void* k;
  const void* v;
  const void* gate;
  int len;
} b2l_adapter_prefix;
#define B2L_ADAPTER_MAX_LEN 64
int b2l_attention_adapter(void* qkv, void* k_cache, void* v_cache, const void* rope,
                          const int64_t* input_pos, const int32_t* ring_start, void* y, void* work,
                          int B, int T, int n_head, int head_size, int S, int block_size, int flags,
                          const b2l_adapter_prefix* prefix, b2l_stream_t stream);
int b2l_attention_nocache_adapter(void* qkv, const void* rope, void* y, void* work, int B, int T,
                                  int n_head, int head_size, int block_size,
                                  const b2l_adapter_prefix* prefix, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * Ragged prefill (continuous batching): n_seq prompts packed back to back into one qkv,
 * each prefilled into its own row of a B_rows-row cache, in one launch per kernel.
 *   qkv   bf16 [N, 3*C]: sequence s is tokens [start[s], start[s] + len[s]), at positions
 *         0..len[s]-1; q is rotated in place
 *   k/v cache bf16 [B_rows, nh, S, hs]: sequence s writes slots 0..len[s]-1 of row row[s]
 *   ring_start int32 [B_rows]: ring_start[row[s]] is set to 0
 *   y     bf16 [N, C]: causal attention within each sequence (plus the LLaMA-Adapter
 *         prefix term when `prefix` is given, the same prefix for every query)
 * Rows and ring offsets no sequence names are not touched.  Each sequence's y rows and
 * cache rows equal, bit for bit, b2l_attention(_adapter) with B = 1, T = len[s], input_pos
 * 0..len[s]-1 and ring offset 0 on a cache holding only that row: every 64-query tile
 * starts at its sequence's first token, so it has the same queries, key bound and key
 * order as in that launch.  `seqs` is read on the host and passed by value to the kernels
 * (no device table, no copy: the call can be captured in a CUDA graph).
 * head_size 128 only (else B2L_E_UNSUPPORTED).  B2L_E_ARG before any launch for null
 * pointers, n_seq outside 1..16, a length outside 1..S, starts that do not tile [0, N) in
 * order, a row outside 0..B_rows-1, or two sequences naming the same row.
 * ---------------------------------------------------------------------------- */
#define B2L_RAGGED_MAX_SEQ 16
typedef struct b2l_ragged {
  int n_seq;
  int row[B2L_RAGGED_MAX_SEQ];
  int start[B2L_RAGGED_MAX_SEQ];
  int len[B2L_RAGGED_MAX_SEQ];
} b2l_ragged;
int b2l_attention_ragged(void* qkv, void* k_cache, void* v_cache, const void* rope, const b2l_ragged* seqs,
                         int32_t* ring_start, void* y, int N, int B_rows, int n_head, int head_size, int S,
                         int block_size, const b2l_adapter_prefix* prefix, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * LoRA (lit_llama/lora.py:92-326): the low-rank term of an UNMERGED MergedLinear,
 * added in place to the output y of its base linear (lora.py:308-326):
 *   u_m = bf16(A_g . xh_m)   d = bf16(B_g . u_m)   y = bf16(y + bf16(d * scaling))
 * for every enabled group g (zero_pad, lora.py:205-241), fp32 accumulation.  A quantized
 * base (gptq.int4 / gptq.int8 / llm.int8) cannot absorb the merge of lora.py:243-280,
 * so this term runs per token.
 *   A        bf16 lora_A [r * n_on][K], 16-byte aligned (n_on = enabled groups)
 *   B        bf16 lora_B [N / n_groups * n_on][r]
 *   scaling  lora_alpha / r (lora.py:171)
 *   r        1..64
 *   n_groups len(enable_lora), 1..32, divides N;  enabled: bit g = enable_lora[g]
 * ---------------------------------------------------------------------------- */
typedef struct b2l_lora {
  const void* A;
  const void* B;
  float scaling;
  int r;
  int n_groups;
  unsigned enabled;
} b2l_lora;
#define B2L_LORA_MAX_R 64
/* y[M, N] (leading dim ldy) += the term for M rows of x[M, K] (leading dim ldx, a multiple
 * of 8, 16-byte aligned; K a multiple of 8).  norm_scale != NULL: xh = RMSNorm(x) with
 * norm_scale / eps and b2l_rmsnorm's rounding points (x is then the residual stream, as in
 * the whole-token step); NULL: xh = x.  flags 0 or B2L_F_PDL (lora_A / lora_B are requested
 * from L2 before griddepcontrol.wait; x and y are read only after it).  Any M.  Bad
 * arguments are rejected before any launch. */
int b2l_lora_apply(const b2l_lora* lora, const void* x, int ldx, const void* norm_scale, float eps,
                   void* y, int ldy, int M, int N, int K, int flags, b2l_stream_t stream);
/* Multi-LoRA: each of M = 1..16 rows adds its own term of one linear.  sets: HOST array of
 * n_sets (1..B2L_LORA_MAX_SETS) terms; they may differ in r, scaling and enabled mask but
 * share n_groups.  row_set: device int32 [M]; row m adds the term of sets[row_set[m]], -1 adds
 * nothing and leaves row m of y unwritten.  An entry outside -1..n_sets-1 is a caller error;
 * the kernel treats it as -1 and never reads out of bounds.  The host never reads row_set,
 * so a captured graph stays valid when rows change sets; the kernel reads it before
 * griddepcontrol.wait, so under B2L_F_PDL it must not be written by the previous launch.
 * Row m of y equals, bit for bit, b2l_lora_apply(&sets[row_set[m]], ...) on that row alone;
 * each set's lora_A / lora_B are read once per output slice whatever rows share it.
 * x, norm_scale, eps, ldx, ldy, flags as b2l_lora_apply.  Bad arguments (every set through
 * b2l_lora_apply's checks, a null row_set, M, n_sets, differing n_groups) are rejected
 * before any launch. */
#define B2L_LORA_MAX_SETS 64
int b2l_lora_apply_rows(const b2l_lora* sets, int n_sets, const int32_t* row_set, const void* x, int ldx,
                        const void* norm_scale, float eps, void* y, int ldy, int M, int N, int K, int flags,
                        b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * fp8 KV cache (opt-in): e4m3 keys and values with one power-of-two scale per (row, head, slot),
 * half the bytes of the bf16 cache.  Number format, for each cached vector x[0..127] (the bf16
 * value the bf16 cache would hold there: the rotated key bf16(rot(k)), or the value):
 *   amax = max |x_i|;  e = 0 when amax == 0, else the smallest integer with amax 2^-e <= 448,
 *                      raised to -124 when smaller (so the smallest bf16 subnormal, 2^-133, maps to
 *                      the smallest e4m3 subnormal, 2^-9, and nothing nonzero rounds to zero)
 *   code_i = e4m3fn(x_i 2^-e), round to nearest even (cvt.rn.satfinite.e4m3x2.f32; torch.float8_e4m3fn
 *            agrees: every scaled input is at most 448)
 *   scale  = 2^e (fp32)
 * The value read back is float(code_i) * scale in fp32: a bf16 number, exact, except that a code
 * of 256 or more at e = 120 (|x_i| >= 1.9375 2^127, the top of the bf16 range) reads back as +-inf.
 * A vector with a non-finite element (NaN, +-inf) is stored as NaN codes (0x7f) and a NaN scale,
 * so every value read back from it is NaN.
 *   k, v              e4m3 codes [B, nh, S, hs], 16-byte aligned, in the slot / ring order of the bf16 cache
 *   k_scale, v_scale  fp32 [B, nh, S]
 * ---------------------------------------------------------------------------- */
typedef struct b2l_kv8_cache {
  void* k;
  void* v;
  float* k_scale;
  float* v_scale;
} b2l_kv8_cache;
/* b2l_attention (b2l_attention_adapter when prefix != NULL) on an fp8 cache, head_size 128:
 *  - T == 1: the fused decode kernel.  It quantizes the new key / value into the cache and scores
 *    and accumulates them as the values read back; every old value is float(code) * scale, and
 *    every FMA, the split plan and the merge are those of the bf16 kernel.  So the result equals
 *    b2l_attention on a bf16 cache holding the values read back, and each row of a B-row launch
 *    equals the B = 1 launch on that row.  B2L_F_ROW_POS and B2L_F_PDL as for b2l_attention.
 *  - T > 1: a prefill at positions 0..T-1 (input_pos must be NULL): q and k are rotated in place,
 *    the rotated keys and the values are quantized into slots (t + ring_start[0]) % S, and the
 *    prompt attends over its own bf16 rows as b2l_attention_nocache(_adapter) does.
 * Refused before any launch: head_size != 128, B2L_F_STEPWISE, B2L_F_ATTN_UNFUSED, B2L_F_ROPE_ROWS
 * (B2L_E_UNSUPPORTED), and T > 1 with an input_pos (B2L_E_UNSUPPORTED: no prefill at a nonzero
 * position).  work as for b2l_attention. */
int b2l_attention_kv8(void* qkv, const b2l_kv8_cache* kv, const void* rope, const int64_t* input_pos,
                      const int32_t* ring_start, void* y, void* work, int B, int T, int n_head, int head_size,
                      int S, int block_size, int flags, const b2l_adapter_prefix* prefix, b2l_stream_t stream);
/* b2l_attention_ragged into an fp8 cache: n_seq prompts packed back to back, each prefilled
 * into its own row of a B_rows-row fp8 cache, in one launch per kernel.
 *   qkv   bf16 [N, 3*C]: sequence s is tokens [start[s], start[s] + len[s]), at positions
 *         0..len[s]-1; q and k are rotated in place
 *   kv    codes and scales [B_rows, ...]: sequence s writes slots 0..len[s]-1 of row row[s]
 *   ring_start int32 [B_rows]: ring_start[row[s]] is set to 0
 *   y     bf16 [N, C]: each sequence's causal attention over its own rotated bf16 rows in qkv
 *         (plus the LLaMA-Adapter prefix term when `prefix` is given)
 * Each sequence's y rows, its rotated q / k rows in qkv, and its row's codes and scales at
 * slots 0..len[s]-1 equal, bit for bit, one b2l_attention_kv8 launch with B = 1, T = len[s],
 * input_pos NULL and ring offset 0 on a cache holding only that row: the same quantizer per
 * (token, head), and every 64-query tile starts at its sequence's first token with the same
 * queries, keys and key order as that launch's.  Slots >= len[s] of a named row are left as
 * that launch leaves them (untouched).  Rows and ring offsets no sequence names are not
 * touched.  The cache is never read, so stale or NaN contents cannot leak in.  `seqs` is read
 * on the host and passed by value (the call can be captured in a CUDA graph).
 * head_size 128 only (else B2L_E_UNSUPPORTED).  B2L_E_ARG before any launch for what
 * b2l_attention_ragged refuses, for a null or misaligned b2l_kv8_cache pointer, and for a
 * length outside 2..S or above block_size: a one-token prompt's batch-1 counterpart is the
 * T == 1 decode kernel, which scores its token as the value read back, not as its bf16 value. */
int b2l_attention_ragged_kv8(void* qkv, const b2l_kv8_cache* kv, const void* rope, const b2l_ragged* seqs,
                             int32_t* ring_start, void* y, int N, int B_rows, int n_head, int head_size, int S,
                             int block_size, const b2l_adapter_prefix* prefix, b2l_stream_t stream);
/* b2l_kv_unroll / b2l_kv_unroll_rows for one fp8 cache tensor (codes and their scales): `out` bf16
 * [B, nh, S, hs] holds the values read back, in logical slot order. */
int b2l_kv8_unroll(const void* code, const float* scale, const int32_t* ring_start, void* out, int B,
                   int n_head, int S, int head_size, b2l_stream_t stream);
int b2l_kv8_unroll_rows(const void* code, const float* scale, const int32_t* ring_start, void* out, int B,
                        int n_head, int S, int head_size, b2l_stream_t stream);

/* kv_caches as the reference would hold them (logical order): un-rotates the ring
 * into `out` [B, nh, S, hs]. */
int b2l_kv_unroll(const void* cache, const int32_t* ring_start, void* out, int B, int n_head,
                  int S, int head_size, b2l_stream_t stream);
/* The same with one ring offset per row (B2L_F_ROW_POS): ring_start int32 [B]. */
int b2l_kv_unroll_rows(const void* cache, const int32_t* ring_start, void* out, int B, int n_head,
                       int S, int head_size, b2l_stream_t stream);

/* ------------------------------------------------------------------------------
 * Whole decode step: LLaMA.forward for T == 1 with a KV cache (model.py:76-122),
 * every kernel of the step enqueued by one call.
 * ---------------------------------------------------------------------------- */
typedef struct b2l_q4_weight {
  const void* qw_tiled;   /* b2l_q4_tile layout (wgmma kernel), used when B > 1; may be NULL if B == 1 */
  const void* qw_mma;     /* mma.sync kernels: b2l_q4_tile_i8 layout when B == 1 (b2l_q4_gemv), b2l_q4_tile_mma
                             layout when B in 2..8 (b2l_q4_gemv_batch); may be NULL if B > 8.  B2L_F_W8:
                             b2l_w8_tile_i8 layout at B == 1 and, with B2L_F_W8_BATCH, at B = 2..16.
                             B2L_F_Q4_BATCH_I8: b2l_q4_tile_i8 layout at B = 2..16 too */
  const void* scales;
  const void* zeros;
  int N, K;
} b2l_q4_weight;

typedef struct b2l_layer {
  const void* rms_1;       /* bf16 [C] */
  const void* rms_2;       /* bf16 [C] */
  b2l_q4_weight c_attn;    /* [3C, C]                                                */
  b2l_q4_weight c_proj;    /* [C, C]                                                 */
  b2l_q4_weight c_fc12;    /* [2*n_hidden, C]; qw_tiled rows interleaved 64/64 per 128-row tile,
                              qw_mma rows interleaved 8/8 per 16-row block (scales/zeros in the
                              order of the layout in use)                               */
  b2l_q4_weight mlp_proj;  /* [C, n_hidden]                                          */
  void* k_cache;           /* bf16 [B, nh, S, hs]                                    */
  void* v_cache;
} b2l_layer;

/* LLaMA-Adapter v2: the affine of each of a Block's linears (adapter_v2.py:30-47); c_fc12's vectors are
 * [2*n_hidden] in the row order of c_fc12.qw_mma (8 of c_fc1 | 8 of c_fc2 per 16 rows). */
typedef struct b2l_layer_affine {
  b2l_out_affine c_attn, c_proj, c_fc12, mlp_proj;
} b2l_layer_affine;

/* llm.int8 weights of the step (B2L_F_Q8): Linear8bitLt's weight.CB (int8 [N, K] row-major) and weight.SCB (fp32 [N])
 * themselves, read in place. */
typedef struct b2l_q8_weight {
  const void* cb;
  const void* scb;
  int N, K;
} b2l_q8_weight;
typedef struct b2l_q8_layer {
  b2l_q8_weight c_attn, c_proj, c_fc1, c_fc2, mlp_proj;
} b2l_q8_layer;

typedef struct b2l_decode_args {
  int n_layer, n_head, n_embd, n_hidden, vocab; /* vocab = padded_vocab_size          */
  int B, S;                                     /* batch, max_seq_length              */
  int sz_dtype;
  float eps;
  const b2l_layer* layers;   /* HOST array [n_layer]                                  */
  const void* wte;           /* bf16 [vocab, C]                                       */
  const void* ln_f;          /* bf16 [C]                                              */
  b2l_q4_weight lm_head;     /* [vocab, C]                                            */
  const void* rope;          /* f32 [block_size, hs/2, 2]                             */
  const void* idx;           /* int32/int64 [B] tokens of this step                   */
  int idx_is_i64;
  const int64_t* input_pos;  /* int64 [1]; [B] under B2L_F_ROW_POS or B2L_F_STEPWISE   */
  int32_t* ring_start;       /* int32 [1] ([B] under B2L_F_ROW_POS); advanced by the step when the cache is full */
  int block_size;            /* rows of the rope table                                */
  void* x;                   /* bf16 [B, C]   residual stream scratch                 */
  void* qkv;                 /* bf16 [B, 3C]                                          */
  void* att;                 /* bf16 [B, C]                                           */
  void* hid;                 /* bf16 [B, n_hidden]                                    */
  void* attn_work;           /* f32, b2l_attn_workspace_bytes                         */
  void* logits;              /* bf16 [B, vocab]                                       */
  int flags;                 /* B2L_F_*                                               */
  void* timeline;            /* debug: device uint64[(5*n_layer+1)*64] of %globaltimer stamps per
                                launch (NULL = off); tools/diag.py `timeline`               */
  void* batch_work;          /* B in 2..8: scratch of b2l_q4_gemv_batch_workspace_bytes(max K) bytes; the
                                linears then run on the mma.sync batch kernel (weights need qw_mma).
                                NULL: wgmma kernel (weights need qw_tiled).
                                B2L_F_W8 | B2L_F_W8_BATCH and B2L_F_Q4_BATCH_I8:
                                b2l_w8_gemv_batch_workspace_bytes(max K, B) bytes (required).
                                B2L_F_Q8 | B2L_F_Q8_BATCH: b2l_q8_linear_batch_workspace_bytes(max K, B) bytes
                                (required) */
  const b2l_adapter_prefix* adapters; /* HOST array [n_layer] of LLaMA-Adapter prefixes (b2l_attention_adapter);
                                NULL = no adapter anywhere, an entry with len == 0 = none in that layer. */
  const b2l_lora* loras;     /* HOST array [n_layer] of c_attn LoRA terms (lora.py:405-446; b2l_lora_apply with
                                rms_1 as the norm, enqueued between c_attn and the attention, without timeline
                                stamps).  NULL = no LoRA anywhere, an entry with r == 0 = none in that layer. */
  const b2l_layer_affine* affines; /* HOST array [n_layer] of LLaMA-Adapter v2 affines, applied inside each linear's
                                launch (b2l_q4_linear_args::out_affine), so the launch count does not change.
                                NULL = none.  Only at B == 1 on the batch-1 kernels (every weight needs qw_mma);
                                not with `loras`.                                         */
  b2l_out_affine lm_head_affine; /* the same for lm_head (both NULL = none)                 */
  const b2l_q8_layer* q8_layers; /* B2L_F_Q8: HOST array [n_layer] of llm.int8 weights; the b2l_q4_weight members of
                                layers[] and lm_head are then unused (layers[] still supplies the norms and the
                                KV cache).  Every linear runs b2l_q8_linear, the same 5*n_layer + 3 launches
                                (+1 per LoRA layer); affines are applied inside them (c_fc12's interleaved
                                8 / 8 as documented above).  With B2L_F_Q8_BATCH at B = 2..16 every linear
                                runs b2l_q8_linear_batch instead: two launches per linear. */
  b2l_q8_weight q8_lm_head;
  float q8_threshold;        /* B2L_F_Q8: Linear8bitLt.threshold of every linear          */
  const b2l_lora* lora_sets; /* Multi-LoRA: HOST [n_lora_sets][n_layer] c_attn terms; r == 0 = that set has no
                                term in that layer.  Each layer where some set has a term runs
                                b2l_lora_apply_rows (rms_1 as the norm) where `loras` would run b2l_lora_apply:
                                row b adds set lora_row_set[b]'s term.  NULL = off.  Not with `loras`,
                                `affines` / `lm_head_affine` or B2L_F_STEPWISE (B2L_E_UNSUPPORTED). */
  int n_lora_sets;           /* 1..B2L_LORA_MAX_SETS                                      */
  const int32_t* lora_row_set; /* device int32 [B]: row b's set, -1 = none (read by the kernels only) */
  const b2l_kv8_cache* kv8;  /* B2L_F_KV_FP8: HOST array [n_layer] of fp8 caches, [B, nh, S, hs] each; every layer's
                                attention runs b2l_attention_kv8 (layers[].k_cache / v_cache are then unused).
                                The launch count does not change.                       */
} b2l_decode_args;

/* Every linear of a step runs the same kernel.  B2L_F_W8 / B2L_F_Q8 and the batch flags select it; otherwise B == 1
 * runs the batch-1 GEMV when lm_head has qw_mma and the wgmma kernel (qw_tiled) when it does not, B = 2..8 with
 * batch_work the mma.sync batch kernel (qw_mma), and every other B the wgmma kernel.  A weight without the tiling its
 * kernel reads is B2L_E_STATE; at B == 1 a weight whose tiling would pick the other kernel is B2L_E_UNSUPPORTED.  Every
 * argument is checked before the first launch. */
/* With B2L_F_STEPWISE the B = 2..16 rows are consecutive tokens of ONE sequence: idx [B], input_pos int64 [B] holding
 * p..p+B-1 (all < S), layers[].k_cache / v_cache the batch-1 caches [1, nh, S, hs], attn_work
 * b2l_attn_workspace_bytes(B, nh, hs, 1, S) bytes.  Row t's logits equal the batch-1 step's at position p+t on the cache
 * holding the tokens before it, bit for bit, and the cache ends as B batch-1 steps leave it.  Only with the row-exact
 * linears: B2L_F_Q4_BATCH_I8, or B2L_F_W8 | B2L_F_W8_BATCH; not with B2L_F_Q8, B2L_F_ROW_POS or `affines`.
 * Adapters and LoRA run as in the batched step; each layer's attention is one launch more (b2l_attention). */
int b2l_decode_step(const b2l_decode_args* args, b2l_stream_t stream);
/* Number of kernels one b2l_decode_step enqueues (for bench.py's gpu_launches). */
int b2l_decode_step_launches(const b2l_decode_args* args);

#ifdef __cplusplus
}
#endif
#endif /* B2L_H_ */

// Error state, device facts and the whole-token entry point of libb200llama.
#include <mutex>

#include "b2l_common.cuh"

namespace b2l {

extern void* g_attn_timeline;
int decode_step_persistent(const b2l_decode_args* d, b2l_stream_t stream);   // decode_mega.cu
int check_adapter_prefix(const b2l_adapter_prefix* pre, const char* who);     // attention.cu
int check_lora(const b2l_lora* lo, int N, int K, const char* who);            // lora.cu
int check_lora_sets(const b2l_lora* sets, size_t stride, int n_sets, int N, int K, bool empty_ok, unsigned* any_on,
                    int* n_groups, const char* who);
int lora_rows(const b2l_lora* sets, size_t stride, int n_sets, bool empty_ok, const int32_t* row_set, const void* x,
              int ldx, const void* norm_scale, float eps, void* y, int ldy, int M, int N, int K, int flags,
              b2l_stream_t stream, const char* who);

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
  (void)cudaGetLastError();  // clear the sticky-less error so the next call starts clean
  return (int)e;
}

int sm_count() {
  static int n[B2L_MAX_DEVICES] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= B2L_MAX_DEVICES) return 132;
  if (n[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev] = v;
  }
  return n[dev];
}

}  // namespace b2l

using namespace b2l;

extern "C" int b2l_version(void) { return 100; }

extern "C" const char* b2l_last_error(void) { return g_err; }

extern "C" int b2l_device_info(int* sm, int* cc_major, int* cc_minor) {
  int dev = 0;
  B2L_CUDA(cudaGetDevice(&dev));
  int a = 0, b = 0, c = 0;
  B2L_CUDA(cudaDeviceGetAttribute(&a, cudaDevAttrMultiProcessorCount, dev));
  B2L_CUDA(cudaDeviceGetAttribute(&b, cudaDevAttrComputeCapabilityMajor, dev));
  B2L_CUDA(cudaDeviceGetAttribute(&c, cudaDevAttrComputeCapabilityMinor, dev));
  if (sm) *sm = a;
  if (cc_major) *cc_major = b;
  if (cc_minor) *cc_minor = c;
  return 0;
}

// ---------------------------------------------------------------------------------
// LLaMA.forward for one new token per sequence (model.py:76-122 with T == 1):
//   wte -> n_layer x Block (model.py:156-168) -> ln_f -> lm_head
// Per Block: [rms_1 + c_attn] -> rope/append/attention -> [c_proj + residual]
//            -> [rms_2 + c_fc1|c_fc2 + silu*mul] -> [mlp.c_proj + residual]
// ---------------------------------------------------------------------------------
static int q4_call(const b2l_q4_weight& w, const void* x, int ldx, void* y, int ldy, int M, int sz_dtype, int prologue,
                   const void* norm_scale, float eps, int epilogue, const void* res, int ldres, int flags,
                   b2l_stream_t stream, void* trace = nullptr, void* batch_work = nullptr, const b2l_out_affine* aff = nullptr) {
  b2l_q4_linear_args a{};
  if (aff != nullptr) a.out_affine = *aff;   // batch-1 kernels only (b2l_decode_step checks B == 1 and qw_mma)
  a.x = x; a.ldx = ldx;
  const bool gemv = (M == 1 && w.qw_mma != nullptr);
  const bool batch = (!gemv && M <= 8 && w.qw_mma != nullptr && batch_work != nullptr);
  a.qw_tiled = (gemv || batch) ? w.qw_mma : w.qw_tiled; a.scales = w.scales; a.zeros = w.zeros; a.sz_dtype = sz_dtype;
  a.y = y; a.ldy = ldy;
  a.M = M; a.N = w.N; a.K = w.K;
  a.prologue = prologue; a.norm_scale = norm_scale; a.eps = eps;
  a.epilogue = epilogue; a.res = res; a.ldres = ldres;
  a.split_k = 0;
  a.flags = flags;
  a.trace = gemv ? trace : nullptr;
  if ((flags & B2L_F_Q4_BATCH_I8) && M > 1) {   // gptq.int4 at 2..16 rows on the batch-1 b2l_q4_tile_i8 tiling
    a.qw_tiled = w.qw_mma; a.trace = nullptr; a.workspace = batch_work;
    a.flags = flags & B2L_F_PDL;
    return b2l_q4_gemv_batch_i8(&a, stream);
  }
  if (flags & B2L_F_W8) {   // gptq.int8: batch 1, or 2..16 under B2L_F_W8_BATCH (checked by b2l_decode_step)
    if (M > 1) {            // the batch kernel on the same b2l_w8_tile_i8 tiling
      a.qw_tiled = w.qw_mma; a.trace = nullptr; a.workspace = batch_work;
      a.flags = flags & B2L_F_PDL;
      return b2l_w8_gemv_batch(&a, stream);
    }
    a.flags = flags & (B2L_F_PDL | B2L_F_DEBUG_NOCOMPUTE);   // only the kernel's own flags pass
    return b2l_w8_gemv(&a, stream);
  }
  if (gemv) return b2l_q4_gemv(&a, stream);
  if (batch) {
    a.workspace = batch_work;
    return b2l_q4_gemv_batch(&a, stream);
  }
  if (a.qw_tiled == nullptr) {
    set_error("b2l_decode_step: weight has no tiling for batch %d", M);
    return B2L_E_STATE;
  }
  return b2l_q4_linear_tc(&a, stream);
}

// llm.int8 (B2L_F_Q8): one b2l_q8_linear launch per linear, or at B = 2..16 under B2L_F_Q8_BATCH b2l_q8_linear_batch
// (checked by b2l_decode_step); w2 = c_fc2 for the SwiGLU pair
static int q8_call(const b2l_decode_args* d, const b2l_q8_weight& w, const b2l_q8_weight* w2, const void* x, void* y,
                   const void* norm_scale, int epilogue, const void* res, const b2l_out_affine* aff, b2l_stream_t stream) {
  b2l_q8_linear_args a{};
  a.x = x; a.cb = w.cb; a.scb = w.scb;
  if (w2 != nullptr) { a.cb2 = w2->cb; a.scb2 = w2->scb; }
  a.y = y; a.N = w.N; a.K = w.K; a.threshold = d->q8_threshold;
  a.prologue = norm_scale != nullptr ? B2L_PRO_RMSNORM : B2L_PRO_NONE; a.norm_scale = norm_scale; a.eps = d->eps;
  a.epilogue = epilogue; a.res = res;
  if (aff != nullptr) a.out_affine = *aff;
  a.flags = d->flags & B2L_F_PDL;
  if (d->flags & B2L_F_Q8_BATCH)
    return b2l_q8_linear_batch(&a, d->B, d->batch_work, b2l_q8_linear_batch_workspace_bytes(w.K, d->B), stream);
  return b2l_q8_linear(&a, stream);
}

// every llm.int8 weight of the step has the shape its place in the Block implies and one the kernel runs
static int check_q8_weight(const b2l_q8_weight& w, int N, int K, const char* what, int l) {
  B2L_CHECK_ARG(w.cb != nullptr && w.scb != nullptr, "b2l_decode_step: B2L_F_Q8 %s of layer %d has no CB / SCB", what, l);
  B2L_CHECK_ARG(w.N == N && w.K == K, "b2l_decode_step: B2L_F_Q8 %s of layer %d is [%d, %d], expected [%d, %d]", what, l,
                w.N, w.K, N, K);
  B2L_CHECK_SUPPORTED(K % 128 == 0 && K <= 32768, "b2l_decode_step: B2L_F_Q8 %s: in_features %d must be a multiple of 128 and <= 32768",
                      what, K);
  B2L_CHECK_ARG((uintptr_t)w.cb % 16 == 0, "b2l_decode_step: B2L_F_Q8 %s of layer %d: CB must be 16-byte aligned", what, l);
  return 0;
}

static int check_q8(const b2l_decode_args* d) {
  B2L_CHECK_SUPPORTED(!(d->flags & B2L_F_W8), "b2l_decode_step: B2L_F_Q8 (llm.int8) and B2L_F_W8 (gptq.int8) exclude each other");
  if (d->flags & B2L_F_Q8_BATCH) {
    B2L_CHECK_SUPPORTED(!(d->flags & (B2L_F_W8_BATCH | B2L_F_Q4_BATCH_I8)),
                        "b2l_decode_step: B2L_F_Q8_BATCH (llm.int8) does not combine with B2L_F_W8_BATCH or B2L_F_Q4_BATCH_I8");
    B2L_CHECK_SUPPORTED(d->B >= 2 && d->B <= 16, "b2l_decode_step: B2L_F_Q8_BATCH runs batches of 2..16, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: B2L_F_Q8_BATCH does not run in the persistent kernel (plan must be NULL)");
    B2L_CHECK_ARG(d->batch_work != nullptr,
                  "b2l_decode_step: B2L_F_Q8_BATCH needs batch_work (b2l_q8_linear_batch_workspace_bytes(max K, B) bytes)");
  } else {
    B2L_CHECK_SUPPORTED(d->B == 1, "b2l_decode_step: B2L_F_Q8 (llm.int8) runs batch 1 only, got B=%d", d->B);
  }
  B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: B2L_F_Q8 (llm.int8) does not run in the persistent kernel (plan must be NULL)");
  B2L_CHECK_ARG(d->q8_layers != nullptr, "b2l_decode_step: B2L_F_Q8 needs q8_layers");
  const int C = d->n_embd, H = d->n_hidden;
  for (int l = 0; l < d->n_layer; ++l) {
    const b2l_q8_layer& q = d->q8_layers[l];
    int rc;
    if ((rc = check_q8_weight(q.c_attn, 3 * C, C, "c_attn", l)) || (rc = check_q8_weight(q.c_proj, C, C, "c_proj", l)) ||
        (rc = check_q8_weight(q.c_fc1, H, C, "c_fc1", l)) || (rc = check_q8_weight(q.c_fc2, H, C, "c_fc2", l)) ||
        (rc = check_q8_weight(q.mlp_proj, C, H, "mlp.c_proj", l)))
      return rc;
  }
  return check_q8_weight(d->q8_lm_head, d->vocab, C, "lm_head", -1);
}

extern "C" int b2l_decode_step_launches(const b2l_decode_args* d) {
  if (!d) return 0;
  if (d->plan != nullptr) return 1;   // the persistent kernel
  // fused single-token attention for head_size 128 (B2L_F_ATTN_UNFUSED: the three-kernel path)
  const bool fused = d->n_embd / d->n_head == 128 && !(d->flags & B2L_F_ATTN_UNFUSED);
  // B2L_F_STEPWISE: the fused kernel runs behind one launch that appends every token's key / value rows
  const int attn = fused ? ((d->flags & B2L_F_STEPWISE) ? 2 : 1) : 3;
  // the batch kernels (int4 at 2..8 rows, gptq.int8, llm.int8 under B2L_F_Q8_BATCH and, under B2L_F_Q4_BATCH_I8,
  // int4 at 2..16) are two launches per linear
  const bool b16 = (d->flags & (B2L_F_W8_BATCH | B2L_F_Q4_BATCH_I8 | B2L_F_Q8_BATCH)) && d->B > 1 && d->B <= 16 && d->batch_work;
  const int lin = (b16 || (d->B > 1 && d->B <= 8 && d->batch_work)) ? 2 : 1;
  int n = 2 + d->n_layer * (4 * lin + attn) + lin;  // ring advance + embedding, per Block 4 linears + attention, ln_f+lm_head
  // an adapter layer adds the prefix kernel behind the three-kernel attention (the fused kernel does it in-launch)
  if (!fused && d->adapters != nullptr)
    for (int l = 0; l < d->n_layer; ++l) n += d->adapters[l].len != 0;
  // a LoRA layer adds its low-rank term's launch behind c_attn
  if (d->loras != nullptr)
    for (int l = 0; l < d->n_layer; ++l) n += d->loras[l].r != 0;
  // per-row LoRA: one launch in each layer where some set has a term
  if (d->lora_sets != nullptr && d->n_lora_sets >= 1 && d->n_lora_sets <= B2L_LORA_MAX_SETS)
    for (int l = 0; l < d->n_layer; ++l) {
      bool any = false;
      for (int s = 0; s < d->n_lora_sets; ++s) any |= d->lora_sets[(size_t)s * d->n_layer + l].r != 0;
      n += any;
    }
  return n;
}

extern "C" int b2l_decode_step(const b2l_decode_args* d, b2l_stream_t stream) {
  B2L_CHECK_ARG(d != nullptr && d->layers != nullptr, "b2l_decode_step: null args");
  B2L_CHECK_ARG(d->n_layer > 0 && d->n_head > 0 && d->n_embd % d->n_head == 0 && d->B >= 1 && d->S >= 1,
                "b2l_decode_step: bad model shape");
  B2L_CHECK_SUPPORTED(d->B <= 16, "b2l_decode_step: batch %d > 16", d->B);
  B2L_CHECK_ARG(d->wte && d->ln_f && d->rope && d->idx && d->input_pos && d->ring_start && d->x && d->qkv && d->att &&
                    d->hid && d->attn_work && d->logits,
                "b2l_decode_step: null pointer");
  const bool row_pos = (d->flags & B2L_F_ROW_POS) != 0;   // input_pos / ring_start hold one entry per row
  // B2L_F_STEPWISE: the B rows are consecutive tokens of ONE sequence (input_pos int64[B], batch-1 caches); every row
  // must equal the batch-1 step at its position, so only the row-exact linears may run it
  const bool stepwise = (d->flags & B2L_F_STEPWISE) != 0;
  if (stepwise) {
    B2L_CHECK_SUPPORTED(!row_pos, "b2l_decode_step: B2L_F_STEPWISE does not combine with B2L_F_ROW_POS");
    B2L_CHECK_SUPPORTED(!(d->flags & B2L_F_Q8),
                        "b2l_decode_step: B2L_F_STEPWISE does not run llm.int8 (B2L_F_Q8): its rows interact through the batch outlier mask");
    B2L_CHECK_SUPPORTED((d->flags & B2L_F_Q4_BATCH_I8) || ((d->flags & B2L_F_W8) && (d->flags & B2L_F_W8_BATCH)),
                        "b2l_decode_step: B2L_F_STEPWISE needs the row-exact linears (B2L_F_Q4_BATCH_I8, or B2L_F_W8 | B2L_F_W8_BATCH)");
    B2L_CHECK_SUPPORTED(d->B >= 2 && d->B <= 16, "b2l_decode_step: B2L_F_STEPWISE runs 2..16 tokens, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: B2L_F_STEPWISE does not run in the persistent kernel (plan must be NULL)");
    B2L_CHECK_SUPPORTED(d->affines == nullptr && d->lm_head_affine.scale == nullptr && d->lm_head_affine.bias == nullptr,
                        "b2l_decode_step: B2L_F_STEPWISE does not apply LLaMA-Adapter v2 affines");
  }
  B2L_CHECK_SUPPORTED(!row_pos || d->plan == nullptr,
                      "b2l_decode_step: B2L_F_ROW_POS does not run in the persistent kernel (plan must be NULL)");
  B2L_CHECK_SUPPORTED(!row_pos || !(d->flags & B2L_F_ROPE_ROWS), "b2l_decode_step: B2L_F_ROW_POS does not combine with B2L_F_ROPE_ROWS");
  if (d->flags & B2L_F_Q4_BATCH_I8) {
    B2L_CHECK_SUPPORTED(!(d->flags & (B2L_F_W8 | B2L_F_Q8 | B2L_F_W8_BATCH)),
                        "b2l_decode_step: B2L_F_Q4_BATCH_I8 (gptq.int4) does not combine with B2L_F_W8, B2L_F_Q8 or B2L_F_W8_BATCH");
    B2L_CHECK_SUPPORTED(d->B >= 2 && d->B <= 16, "b2l_decode_step: B2L_F_Q4_BATCH_I8 runs batches of 2..16, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: B2L_F_Q4_BATCH_I8 does not run in the persistent kernel (plan must be NULL)");
    B2L_CHECK_SUPPORTED(d->affines == nullptr && d->lm_head_affine.scale == nullptr && d->lm_head_affine.bias == nullptr,
                        "b2l_decode_step: B2L_F_Q4_BATCH_I8 does not apply LLaMA-Adapter v2 affines (batch 1 only)");
    B2L_CHECK_ARG(d->batch_work != nullptr, "b2l_decode_step: B2L_F_Q4_BATCH_I8 needs batch_work (b2l_w8_gemv_batch_workspace_bytes(max K, B) bytes)");
  }
  const bool q8 = (d->flags & B2L_F_Q8) != 0;
  B2L_CHECK_SUPPORTED(q8 || !(d->flags & B2L_F_Q8_BATCH), "b2l_decode_step: B2L_F_Q8_BATCH needs B2L_F_Q8 (llm.int8)");
  if (q8)
    if (int rc = check_q8(d)) return rc;
  if (d->flags & B2L_F_W8_BATCH) {
    B2L_CHECK_SUPPORTED(d->flags & B2L_F_W8, "b2l_decode_step: B2L_F_W8_BATCH needs B2L_F_W8 (gptq.int8)");
    B2L_CHECK_SUPPORTED(d->B >= 2 && d->B <= 16, "b2l_decode_step: B2L_F_W8_BATCH runs batches of 2..16, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: B2L_F_W8_BATCH does not run in the persistent kernel (plan must be NULL)");
    B2L_CHECK_SUPPORTED(d->affines == nullptr && d->lm_head_affine.scale == nullptr && d->lm_head_affine.bias == nullptr,
                        "b2l_decode_step: B2L_F_W8_BATCH does not apply LLaMA-Adapter v2 affines (batch 1 only)");
    B2L_CHECK_ARG(d->batch_work != nullptr, "b2l_decode_step: B2L_F_W8_BATCH needs batch_work (b2l_w8_gemv_batch_workspace_bytes(max K, B) bytes)");
  } else if (d->flags & B2L_F_W8) {
    B2L_CHECK_SUPPORTED(d->B == 1, "b2l_decode_step: B2L_F_W8 (gptq.int8) runs batch 1 only, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: B2L_F_W8 (gptq.int8) does not run in the persistent kernel (plan must be NULL)");
  }
  if (d->adapters != nullptr) {
    for (int l = 0; l < d->n_layer; ++l) {
      if (d->adapters[l].len == 0) continue;   // no adapter in this layer
      B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: adapters do not run in the persistent kernel (plan must be NULL)");
      if (int rc = check_adapter_prefix(&d->adapters[l], "b2l_decode_step")) return rc;
    }
  }
  if (d->loras != nullptr) {
    for (int l = 0; l < d->n_layer; ++l) {
      if (d->loras[l].r == 0) continue;   // no LoRA in this layer
      B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: LoRA layers do not run in the persistent kernel (plan must be NULL)");
      if (int rc = check_lora(&d->loras[l], 3 * d->n_embd, d->n_embd, "b2l_decode_step")) return rc;
    }
  }
  if (d->lora_sets != nullptr) {   // per-row LoRA: every layer's sets checked here, before any launch
    B2L_CHECK_SUPPORTED(d->loras == nullptr, "b2l_decode_step: lora_sets and loras do not combine");
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: lora_sets do not run in the persistent kernel (plan must be NULL)");
    B2L_CHECK_SUPPORTED(d->affines == nullptr && d->lm_head_affine.scale == nullptr && d->lm_head_affine.bias == nullptr,
                        "b2l_decode_step: lora_sets and LLaMA-Adapter v2 affines do not combine");
    B2L_CHECK_SUPPORTED(!stepwise, "b2l_decode_step: lora_sets do not run under B2L_F_STEPWISE (one sequence, one adapter: use loras)");
    B2L_CHECK_ARG(d->lora_row_set != nullptr, "b2l_decode_step: lora_sets need lora_row_set");
    for (int l = 0; l < d->n_layer; ++l) {
      unsigned any_on = 0;
      int n_groups = 0;
      if (int rc = check_lora_sets(d->lora_sets + l, (size_t)d->n_layer, d->n_lora_sets, 3 * d->n_embd, d->n_embd, true,
                                   &any_on, &n_groups, "b2l_decode_step"))
        return rc;
    }
  }
  // LLaMA-Adapter v2: every linear's affine runs in its own batch-1 launch (b2l_q4_linear_args::out_affine)
  const bool any_affine = d->affines != nullptr || d->lm_head_affine.scale != nullptr || d->lm_head_affine.bias != nullptr;
  if (any_affine) {
    // llm.int8's batch kernel applies them in its epilogue too
    B2L_CHECK_SUPPORTED(d->B == 1 || (d->flags & B2L_F_Q8_BATCH),
                        "b2l_decode_step: LLaMA-Adapter v2 affines run at batch 1 only, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->plan == nullptr, "b2l_decode_step: LLaMA-Adapter v2 affines do not run in the persistent kernel (plan must be NULL)");
    B2L_CHECK_SUPPORTED(d->loras == nullptr, "b2l_decode_step: LLaMA-Adapter v2 affines and LoRA do not combine");
    auto ok = [](const b2l_out_affine& f) { return (f.scale == nullptr) == (f.bias == nullptr); };
    B2L_CHECK_ARG(ok(d->lm_head_affine), "b2l_decode_step: lm_head_affine needs both scale and bias (or neither)");
    B2L_CHECK_SUPPORTED(q8 || d->lm_head.qw_mma != nullptr, "b2l_decode_step: affines need the batch-1 tiling (qw_mma) of every weight");
    for (int l = 0; d->affines != nullptr && l < d->n_layer; ++l) {
      const b2l_layer_affine& f = d->affines[l];
      B2L_CHECK_ARG(ok(f.c_attn) && ok(f.c_proj) && ok(f.c_fc12) && ok(f.mlp_proj),
                    "b2l_decode_step: affines[%d] needs both scale and bias (or neither) per linear", l);
      const b2l_layer& L = d->layers[l];
      B2L_CHECK_SUPPORTED(q8 || (L.c_attn.qw_mma && L.c_proj.qw_mma && L.c_fc12.qw_mma && L.mlp_proj.qw_mma),
                          "b2l_decode_step: affines need the batch-1 tiling (qw_mma) of every weight");
    }
  }
  if (d->plan != nullptr) return decode_step_persistent(d, stream);   // one persistent kernel per token (decode_mega.cu)
  const int C = d->n_embd, hs = C / d->n_head, B = d->B;
  const int fl = d->flags & ~(B2L_F_ROW_POS | B2L_F_STEPWISE);   // the linears' flags (q4_call routes B2L_F_W8 to b2l_w8_gemv)
  const int afl = d->flags & ~(B2L_F_W8 | B2L_F_Q8 | B2L_F_W8_BATCH | B2L_F_Q4_BATCH_I8 | B2L_F_Q8_BATCH);   // the attention's
  int rc;
  // debug timeline: launch i of the step writes uint64[64] at timeline + 512*i (order: per Block c_attn,
  // attention, c_proj, fc12, mlp_proj; then lm_head)
  char* tlb = (char*)d->timeline;
  int li = 0;
  auto tl = [&]() -> void* { void* r = tlb ? (void*)(tlb + 512 * li) : nullptr; ++li; return r; };
  if ((rc = row_pos ? b2l_ring_advance_rows(d->input_pos, B, d->ring_start, d->S, stream)
                    : b2l_ring_advance(d->input_pos, stepwise ? B : 1, d->ring_start, d->S, stream)))
    return rc;
  // the attention's view: B sequences of one token, or (stepwise) one sequence of B tokens
  const int aB = stepwise ? 1 : B, aT = stepwise ? B : 1;
  if ((rc = b2l_embedding(d->idx, d->idx_is_i64, d->wte, d->x, B, C, d->vocab, stream))) return rc;
  for (int l = 0; l < d->n_layer; ++l) {
    const b2l_layer& L = d->layers[l];
    const b2l_layer_affine* af = d->affines != nullptr ? &d->affines[l] : nullptr;
    const b2l_q8_layer* Q = q8 ? &d->q8_layers[l] : nullptr;   // llm.int8: b2l_q8_linear (no timeline stamps)
    void* t = tl();
    if ((rc = Q ? q8_call(d, Q->c_attn, nullptr, d->x, d->qkv, L.rms_1, B2L_EPI_STORE, nullptr, af ? &af->c_attn : nullptr, stream)
                : q4_call(L.c_attn, d->x, C, d->qkv, 3 * C, B, d->sz_dtype, B2L_PRO_RMSNORM, L.rms_1, d->eps, B2L_EPI_STORE,
                          nullptr, 0, fl, stream, t, d->batch_work, af ? &af->c_attn : nullptr)))
      return rc;
    // LoRA on c_attn (lora.py:308-326): the low-rank term from rms_1(x), added into qkv in place
    if (d->loras != nullptr && d->loras[l].r != 0 &&
        (rc = b2l_lora_apply(&d->loras[l], d->x, C, L.rms_1, d->eps, d->qkv, 3 * C, B, 3 * C, C, fl & B2L_F_PDL, stream)))
      return rc;
    // per-row LoRA: row b adds set lora_row_set[b]'s term (no launch in a layer where no set has one)
    if (d->lora_sets != nullptr &&
        (rc = lora_rows(d->lora_sets + l, (size_t)d->n_layer, d->n_lora_sets, true, d->lora_row_set, d->x, C, L.rms_1,
                        d->eps, d->qkv, 3 * C, B, 3 * C, C, fl & B2L_F_PDL, stream, "b2l_decode_step")))
      return rc;
    g_attn_timeline = tl();
    const b2l_adapter_prefix* pre = (d->adapters != nullptr && d->adapters[l].len != 0) ? &d->adapters[l] : nullptr;
    if ((rc = pre != nullptr
                  ? b2l_attention_adapter(d->qkv, L.k_cache, L.v_cache, d->rope, d->input_pos, d->ring_start, d->att,
                                          d->attn_work, aB, aT, d->n_head, hs, d->S, d->block_size, afl, pre, stream)
                  : b2l_attention(d->qkv, L.k_cache, L.v_cache, d->rope, d->input_pos, d->ring_start, d->att,
                                  d->attn_work, aB, aT, d->n_head, hs, d->S, d->block_size, afl, stream))) {
      g_attn_timeline = nullptr;
      return rc;
    }
    g_attn_timeline = nullptr;
    t = tl();
    if ((rc = Q ? q8_call(d, Q->c_proj, nullptr, d->att, d->x, nullptr, B2L_EPI_RESIDUAL, d->x, af ? &af->c_proj : nullptr, stream)
                : q4_call(L.c_proj, d->att, C, d->x, C, B, d->sz_dtype, B2L_PRO_NONE, nullptr, 0.f, B2L_EPI_RESIDUAL, d->x, C,
                          fl, stream, t, d->batch_work, af ? &af->c_proj : nullptr)))
      return rc;
    t = tl();
    if ((rc = Q ? q8_call(d, Q->c_fc1, &Q->c_fc2, d->x, d->hid, L.rms_2, B2L_EPI_SWIGLU, nullptr, af ? &af->c_fc12 : nullptr, stream)
                : q4_call(L.c_fc12, d->x, C, d->hid, d->n_hidden, B, d->sz_dtype, B2L_PRO_RMSNORM, L.rms_2, d->eps,
                          B2L_EPI_SWIGLU, nullptr, 0, fl, stream, t, d->batch_work, af ? &af->c_fc12 : nullptr)))
      return rc;
    t = tl();
    if ((rc = Q ? q8_call(d, Q->mlp_proj, nullptr, d->hid, d->x, nullptr, B2L_EPI_RESIDUAL, d->x, af ? &af->mlp_proj : nullptr, stream)
                : q4_call(L.mlp_proj, d->hid, d->n_hidden, d->x, C, B, d->sz_dtype, B2L_PRO_NONE, nullptr, 0.f,
                          B2L_EPI_RESIDUAL, d->x, C, fl, stream, t, d->batch_work, af ? &af->mlp_proj : nullptr)))
      return rc;
  }
  if (q8) return q8_call(d, d->q8_lm_head, nullptr, d->x, d->logits, d->ln_f, B2L_EPI_STORE, nullptr, &d->lm_head_affine, stream);
  return q4_call(d->lm_head, d->x, C, d->logits, d->vocab, B, d->sz_dtype, B2L_PRO_RMSNORM, d->ln_f, d->eps,
                 B2L_EPI_STORE, nullptr, 0, fl, stream, tl(), d->batch_work, &d->lm_head_affine);
}

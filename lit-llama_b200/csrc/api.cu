// Error state, device facts and the whole-token entry point of libb200llama.
#include <mutex>

#include "b2l_common.cuh"

namespace b2l {

int check_adapter_prefix(const b2l_adapter_prefix* pre, const char* who);     // attention.cu
int check_attention(const void* qkv, const void* k_cache, const void* v_cache, const void* rope, const int64_t* input_pos,
                    const int32_t* ring_start, const void* y, const void* work, int B, int T, int n_head, int head_size,
                    int S, int block_size, int flags, const char* who);
int attention_impl(void* qkv, void* k_cache, void* v_cache, const void* rope, const int64_t* input_pos,
                   const int32_t* ring_start, void* y, void* work, int B, int T, int n_head, int head_size, int S,
                   int block_size, int flags, const b2l_adapter_prefix* pre, void* timeline, cudaStream_t st);
int check_attention_kv8(const void* qkv, const b2l_kv8_cache* kv, const void* rope, const int64_t* input_pos,
                        const int32_t* ring_start, const void* y, const void* work, int B, int T, int n_head,
                        int head_size, int S, int block_size, int flags, const char* who);
int attention_kv8_impl(void* qkv, const b2l_kv8_cache* kv, const void* rope, const int64_t* input_pos,
                       const int32_t* ring_start, void* y, void* work, int B, int T, int n_head, int S, int flags,
                       int block_size, const b2l_adapter_prefix* pre, void* timeline, cudaStream_t st);
int check_gemv(const b2l_q4_linear_args* a, bool w8);                         // q4_gemv.cu
int check_q4_gemv_batch(const b2l_q4_linear_args* a);                         // q4_gemv_batch.cu
int check_gemv_batch_i8(const b2l_q4_linear_args* a, bool w8);                // w8_gemv_batch.cu
int check_q4_linear_tc(const b2l_q4_linear_args* a);                          // q4_tc.cu
int check_q8_linear(const b2l_q8_linear_args* a);                             // q8_gemv.cu
int check_q8_disjoint(const b2l_q8_linear_args* a, int M, const char* who);
int check_q8_linear_batch(const b2l_q8_linear_args* a, int M, const void* workspace, size_t workspace_bytes);  // q8_gemv_batch.cu
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

// Every linear of one step runs on one route: a kernel and the tiling it reads.  resolve_route picks it from the flags,
// B, batch_work and lm_head's tiling; the step's checks, its dispatch (linear) and b2l_decode_step_launches read it
// from this table.  LoRA, adapters, B2L_F_ROW_POS and B2L_F_KV_FP8 run on every route.
enum RouteId { Q4_GEMV, Q4_BATCH, Q4_TC, Q4_BATCH_I8, W8_GEMV, W8_BATCH, Q8, Q8_BATCH };
enum Tiling { MMA, TILED, CB };   // b2l_q4_weight::qw_mma, b2l_q4_weight::qw_tiled, llm.int8's CB / SCB
struct Route {
  const char* flag;   // the flag that selects the route, in messages (nullptr: B, batch_work and the tiling do)
  int b_min, b_max;   // batch range
  int launches;       // per linear
  Tiling tiling;
  int kernel_flags;   // the step's flags its kernel takes
  bool batch_work;    // needs b2l_decode_args::batch_work
  bool timeline;      // writes the debug timeline
  bool affines;       // applies LLaMA-Adapter v2 affines in its epilogue
  bool stepwise;      // row-exact (each row equals the batch-1 step), so it may run B2L_F_STEPWISE
};
constexpr int Q4_FLAGS = ~(B2L_F_ROW_POS | B2L_F_STEPWISE | B2L_F_KV_FP8);
// flag, B range, launches, tiling, kernel flags, batch_work, timeline, affines, stepwise
static const Route kRoutes[] = {
    /* Q4_GEMV: b2l_q4_gemv */ {nullptr, 1, 1, 1, MMA, Q4_FLAGS, false, true, true, false},
    /* Q4_BATCH: b2l_q4_gemv_batch */ {nullptr, 2, 8, 2, MMA, Q4_FLAGS, true, false, false, false},
    /* Q4_TC: b2l_q4_linear_tc */ {nullptr, 1, 16, 1, TILED, Q4_FLAGS, false, false, false, false},
    /* Q4_BATCH_I8: b2l_q4_gemv_batch_i8 */ {"B2L_F_Q4_BATCH_I8", 2, 16, 2, MMA, B2L_F_PDL, true, false, false, true},
    /* W8_GEMV: b2l_w8_gemv */ {"B2L_F_W8 (gptq.int8)", 1, 1, 1, MMA, B2L_F_PDL | B2L_F_DEBUG_NOCOMPUTE, false, true, true, false},
    /* W8_BATCH: b2l_w8_gemv_batch */ {"B2L_F_W8_BATCH", 2, 16, 2, MMA, B2L_F_PDL, true, false, false, true},
    /* Q8: b2l_q8_linear */ {"B2L_F_Q8 (llm.int8)", 1, 1, 1, CB, B2L_F_PDL, false, false, true, false},
    /* Q8_BATCH: b2l_q8_linear_batch */ {"B2L_F_Q8_BATCH", 2, 16, 2, CB, B2L_F_PDL, true, false, true, false},
};

// The route the flags select; the flag combinations no route takes are refused here.
static int resolve_route(const b2l_decode_args* d, RouteId* r) {
  const int f = d->flags;
  B2L_CHECK_SUPPORTED(!(f & B2L_F_Q8_BATCH) || (f & B2L_F_Q8), "b2l_decode_step: B2L_F_Q8_BATCH needs B2L_F_Q8 (llm.int8)");
  if (f & B2L_F_Q4_BATCH_I8) {
    B2L_CHECK_SUPPORTED(!(f & (B2L_F_W8 | B2L_F_Q8 | B2L_F_W8_BATCH)),
                        "b2l_decode_step: B2L_F_Q4_BATCH_I8 (gptq.int4) does not combine with B2L_F_W8, B2L_F_Q8 or B2L_F_W8_BATCH");
    *r = Q4_BATCH_I8;
  } else if (f & B2L_F_Q8) {
    B2L_CHECK_SUPPORTED(!(f & B2L_F_W8), "b2l_decode_step: B2L_F_Q8 (llm.int8) and B2L_F_W8 (gptq.int8) exclude each other");
    B2L_CHECK_SUPPORTED(!(f & B2L_F_Q8_BATCH) || !(f & B2L_F_W8_BATCH),
                        "b2l_decode_step: B2L_F_Q8_BATCH (llm.int8) does not combine with B2L_F_W8_BATCH or B2L_F_Q4_BATCH_I8");
    B2L_CHECK_SUPPORTED(!(f & B2L_F_W8_BATCH), "b2l_decode_step: B2L_F_W8_BATCH needs B2L_F_W8 (gptq.int8)");
    *r = (f & B2L_F_Q8_BATCH) ? Q8_BATCH : Q8;
  } else {
    B2L_CHECK_SUPPORTED(!(f & B2L_F_W8_BATCH) || (f & B2L_F_W8), "b2l_decode_step: B2L_F_W8_BATCH needs B2L_F_W8 (gptq.int8)");
    if (f & B2L_F_W8) *r = (f & B2L_F_W8_BATCH) ? W8_BATCH : W8_GEMV;
    else if (d->B == 1) *r = d->lm_head.qw_mma != nullptr ? Q4_GEMV : Q4_TC;
    else *r = (d->B <= kRoutes[Q4_BATCH].b_max && d->batch_work != nullptr) ? Q4_BATCH : Q4_TC;
  }
  return 0;
}

// One linear of the step (layer == n_layer: lm_head), as its kernel sees it
struct Linear {
  const char* name;
  int layer;
  const b2l_q4_weight* w;                   // gptq routes
  const b2l_q8_weight *q8, *q8_up;          // llm.int8 (q8_up: c_fc2 of the SwiGLU pair)
  const void* x;
  int ldx;                                  // = K
  void* y;
  int ldy;                                  // = N (SwiGLU: N / 2)
  int prologue;
  const void* norm;                         // the RMSNorm prologue's scale
  int epilogue;
  const b2l_out_affine* aff;                // or nullptr
};

// linear k (0..3: c_attn, c_proj, c_fc12, mlp.c_proj) of layer l, or lm_head (l == n_layer)
static Linear linear_of(const b2l_decode_args* d, int l, int k) {
  const int C = d->n_embd, H = d->n_hidden;
  if (l == d->n_layer)
    return {"lm_head", l, &d->lm_head, &d->q8_lm_head, nullptr, d->x, C, d->logits, d->vocab, B2L_PRO_RMSNORM, d->ln_f,
            B2L_EPI_STORE, &d->lm_head_affine};
  const b2l_layer& L = d->layers[l];
  const b2l_layer_affine* af = d->affines != nullptr ? &d->affines[l] : nullptr;
  const b2l_q8_layer* Q = (d->flags & B2L_F_Q8) && d->q8_layers != nullptr ? &d->q8_layers[l] : nullptr;
  switch (k) {
    case 0: return {"c_attn", l, &L.c_attn, Q ? &Q->c_attn : nullptr, nullptr, d->x, C, d->qkv, 3 * C, B2L_PRO_RMSNORM,
                    L.rms_1, B2L_EPI_STORE, af ? &af->c_attn : nullptr};
    case 1: return {"c_proj", l, &L.c_proj, Q ? &Q->c_proj : nullptr, nullptr, d->att, C, d->x, C, B2L_PRO_NONE,
                    nullptr, B2L_EPI_RESIDUAL, af ? &af->c_proj : nullptr};
    case 2: return {"c_fc12", l, &L.c_fc12, Q ? &Q->c_fc1 : nullptr, Q ? &Q->c_fc2 : nullptr, d->x, C, d->hid, H,
                    B2L_PRO_RMSNORM, L.rms_2, B2L_EPI_SWIGLU, af ? &af->c_fc12 : nullptr};
    default: return {"mlp.c_proj", l, &L.mlp_proj, Q ? &Q->mlp_proj : nullptr, nullptr, d->hid, H, d->x, C, B2L_PRO_NONE,
                     nullptr, B2L_EPI_RESIDUAL, af ? &af->mlp_proj : nullptr};
  }
}

// "c_attn of layer 3" / "lm_head", for messages
static const char* where(const b2l_decode_args* d, const Linear& li, const char* name, char (&buf)[64]) {
  if (li.layer == d->n_layer) return name;
  snprintf(buf, sizeof(buf), "%s of layer %d", name, li.layer);
  return buf;
}

// The weight carries the tiling its route reads (B2L_E_STATE when it does not).  At batch 1 the gptq.int4 route follows
// lm_head's tiling, and a weight that would have run the other kernel disagrees with lm_head (B2L_E_UNSUPPORTED).
// llm.int8 weights also have the shape their place in the Block implies.
static int check_tiling(RouteId r, const b2l_decode_args* d, const Linear& li) {
  char buf[64];
  if (kRoutes[r].tiling == CB) {
    for (const b2l_q8_weight* w : {li.q8, li.q8_up}) {
      if (w == nullptr) continue;
      const char* at = where(d, li, w == li.q8_up ? "c_fc2" : li.q8_up ? "c_fc1" : li.name, buf);
      B2L_CHECK_ARG(w->cb != nullptr && w->scb != nullptr, "b2l_decode_step: B2L_F_Q8 %s has no CB / SCB", at);
      B2L_CHECK_ARG(w->N == li.ldy && w->K == li.ldx, "b2l_decode_step: B2L_F_Q8 %s is [%d, %d], expected [%d, %d]", at,
                    w->N, w->K, li.ldy, li.ldx);
    }
    return 0;
  }
  const bool mma = kRoutes[r].tiling == MMA;
  const char* at = where(d, li, li.name, buf);
  if (kRoutes[r].flag == nullptr && d->B == 1) {   // a weight with qw_mma would run the GEMV, one with only qw_tiled not
    const bool gemv = li.w->qw_mma != nullptr, tc = li.w->qw_tiled != nullptr;
    B2L_CHECK_SUPPORTED(mma ? gemv || !tc : !gemv,
                        "b2l_decode_step: %s has %s, lm_head %s (at batch 1 every weight runs the kernel lm_head's tiling picks)",
                        at, mma ? "qw_tiled but no qw_mma" : "qw_mma", mma ? "has qw_mma" : "has no qw_mma");
  }
  if ((mma ? li.w->qw_mma : li.w->qw_tiled) != nullptr) return 0;
  set_error("b2l_decode_step: %s has no tiling for batch %d (%s)", at, d->B, mma ? "qw_mma" : "qw_tiled");
  return B2L_E_STATE;
}

// Checks (launch == false) or launches (launch == true) one linear on route r, from the same argument block.
static int linear(RouteId r, const b2l_decode_args* d, const Linear& li, void* trace, bool launch, b2l_stream_t stream) {
  const Route& R = kRoutes[r];
  if (R.tiling == CB) {
    b2l_q8_linear_args a{};
    a.x = li.x; a.cb = li.q8->cb; a.scb = li.q8->scb;
    if (li.q8_up != nullptr) { a.cb2 = li.q8_up->cb; a.scb2 = li.q8_up->scb; }
    a.y = li.y; a.N = li.q8->N; a.K = li.q8->K; a.threshold = d->q8_threshold;
    a.prologue = li.prologue; a.norm_scale = li.norm; a.eps = d->eps;
    a.epilogue = li.epilogue; a.res = li.epilogue == B2L_EPI_RESIDUAL ? d->x : nullptr;
    if (li.aff != nullptr) a.out_affine = *li.aff;
    a.flags = d->flags & R.kernel_flags;
    if (r == Q8) return launch ? b2l_q8_linear(&a, stream) : check_q8_linear(&a);
    const size_t bytes = b2l_q8_linear_batch_workspace_bytes(a.K, d->B);
    return launch ? b2l_q8_linear_batch(&a, d->B, d->batch_work, bytes, stream)
                  : check_q8_linear_batch(&a, d->B, d->batch_work, bytes);
  }
  b2l_q4_linear_args a{};
  const b2l_q4_weight& w = *li.w;
  a.x = li.x; a.ldx = li.ldx;
  a.qw_tiled = R.tiling == MMA ? w.qw_mma : w.qw_tiled; a.scales = w.scales; a.zeros = w.zeros; a.sz_dtype = d->sz_dtype;
  a.y = li.y; a.ldy = li.ldy;
  a.M = d->B; a.N = w.N; a.K = w.K;
  a.prologue = li.prologue; a.norm_scale = li.norm; a.eps = li.prologue == B2L_PRO_RMSNORM ? d->eps : 0.f;
  a.epilogue = li.epilogue;
  if (li.epilogue == B2L_EPI_RESIDUAL) { a.res = d->x; a.ldres = d->n_embd; }
  if (li.aff != nullptr) a.out_affine = *li.aff;
  a.flags = d->flags & R.kernel_flags;
  a.trace = R.timeline ? trace : nullptr;
  if (R.batch_work) a.workspace = d->batch_work;
  switch (r) {
    case Q4_GEMV: return launch ? b2l_q4_gemv(&a, stream) : check_gemv(&a, false);
    case W8_GEMV: return launch ? b2l_w8_gemv(&a, stream) : check_gemv(&a, true);
    case Q4_BATCH: return launch ? b2l_q4_gemv_batch(&a, stream) : check_q4_gemv_batch(&a);
    case Q4_BATCH_I8: return launch ? b2l_q4_gemv_batch_i8(&a, stream) : check_gemv_batch_i8(&a, false);
    case W8_BATCH: return launch ? b2l_w8_gemv_batch(&a, stream) : check_gemv_batch_i8(&a, true);
    default: return launch ? b2l_q4_linear_tc(&a, stream) : check_q4_linear_tc(&a);
  }
}

// a refusal of one linear's kernel check names the step and the linear in front of the kernel's own message
static int in_step(int rc, const b2l_decode_args* d, const Linear& li) {
  if (rc == 0) return 0;
  char buf[64], msg[512];
  snprintf(msg, sizeof(msg), "%s", b2l_last_error());
  set_error("b2l_decode_step: %s: %s", where(d, li, li.q8_up != nullptr ? "c_fc1" : li.name, buf), msg);
  return rc;
}

extern "C" int b2l_decode_step_launches(const b2l_decode_args* d) {
  if (!d) return 0;
  RouteId r;
  if (resolve_route(d, &r) != 0) return 0;
  // fused single-token attention for head_size 128 (B2L_F_ATTN_UNFUSED: the three-kernel path)
  const bool fused = d->n_embd / d->n_head == 128 && !(d->flags & B2L_F_ATTN_UNFUSED);
  // B2L_F_STEPWISE: the fused kernel runs behind one launch that appends every token's key / value rows
  const int attn = fused ? ((d->flags & B2L_F_STEPWISE) ? 2 : 1) : 3;
  const int lin = kRoutes[r].launches;
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
  B2L_CHECK_ARG(d->n_layer > 0 && d->n_head > 0 && d->n_embd > 0 && d->n_embd % d->n_head == 0 && d->vocab > 0 &&
                    d->B >= 1 && d->S >= 1,
                "b2l_decode_step: bad model shape");
  B2L_CHECK_SUPPORTED(d->B <= 16, "b2l_decode_step: batch %d > 16", d->B);
  B2L_CHECK_ARG(d->wte && d->ln_f && d->rope && d->idx && d->input_pos && d->ring_start && d->x && d->qkv && d->att &&
                    d->hid && d->attn_work && d->logits,
                "b2l_decode_step: null pointer");
  RouteId r;
  if (int rc = resolve_route(d, &r)) return rc;
  const Route& R = kRoutes[r];
  const bool any_affine = d->affines != nullptr || d->lm_head_affine.scale != nullptr || d->lm_head_affine.bias != nullptr;
  const bool row_pos = (d->flags & B2L_F_ROW_POS) != 0;   // input_pos / ring_start hold one entry per row
  // B2L_F_STEPWISE: the B rows are consecutive tokens of ONE sequence (input_pos int64[B], batch-1 caches); every row
  // must equal the batch-1 step at its position, so only the row-exact linears may run it
  const bool stepwise = (d->flags & B2L_F_STEPWISE) != 0;
  if (stepwise) {
    B2L_CHECK_SUPPORTED(!row_pos, "b2l_decode_step: B2L_F_STEPWISE does not combine with B2L_F_ROW_POS");
    B2L_CHECK_SUPPORTED(R.tiling != CB,
                        "b2l_decode_step: B2L_F_STEPWISE does not run llm.int8 (B2L_F_Q8): its rows interact through the batch outlier mask");
    B2L_CHECK_SUPPORTED(R.stepwise,
                        "b2l_decode_step: B2L_F_STEPWISE needs the row-exact linears (B2L_F_Q4_BATCH_I8, or B2L_F_W8 | B2L_F_W8_BATCH)");
    B2L_CHECK_SUPPORTED(d->B >= 2 && d->B <= 16, "b2l_decode_step: B2L_F_STEPWISE runs 2..16 tokens, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(!any_affine, "b2l_decode_step: B2L_F_STEPWISE does not apply LLaMA-Adapter v2 affines");
  }
  // B2L_F_KV_FP8: every layer's attention on its fp8 cache (kv8), whatever route the linears take
  const bool kv8 = (d->flags & B2L_F_KV_FP8) != 0;
  if (kv8) {
    B2L_CHECK_SUPPORTED(!stepwise, "b2l_decode_step: B2L_F_KV_FP8 does not run B2L_F_STEPWISE (speculative verify)");
    B2L_CHECK_SUPPORTED(!(d->flags & B2L_F_ATTN_UNFUSED),
                        "b2l_decode_step: B2L_F_KV_FP8 runs the fused decode kernel only (not B2L_F_ATTN_UNFUSED)");
    B2L_CHECK_SUPPORTED(d->n_embd / d->n_head == 128,
                        "b2l_decode_step: B2L_F_KV_FP8 runs head_size 128 only (every LLaMA size), got %d", d->n_embd / d->n_head);
    B2L_CHECK_ARG(d->kv8 != nullptr, "b2l_decode_step: B2L_F_KV_FP8 needs kv8 (one b2l_kv8_cache per layer)");
  }
  B2L_CHECK_SUPPORTED(!row_pos || !(d->flags & B2L_F_ROPE_ROWS), "b2l_decode_step: B2L_F_ROW_POS does not combine with B2L_F_ROPE_ROWS");
  if (R.flag != nullptr) {   // a route a flag selects: its batch range and its workspace
    if (R.b_min == R.b_max)
      B2L_CHECK_SUPPORTED(d->B == R.b_min, "b2l_decode_step: %s runs batch 1 only, got B=%d", R.flag, d->B);
    else
      B2L_CHECK_SUPPORTED(d->B >= R.b_min && d->B <= R.b_max, "b2l_decode_step: %s runs batches of %d..%d, got B=%d",
                          R.flag, R.b_min, R.b_max, d->B);
    B2L_CHECK_SUPPORTED(R.affines || !any_affine, "b2l_decode_step: %s does not apply LLaMA-Adapter v2 affines (batch 1 only)",
                        R.flag);
    B2L_CHECK_ARG(!R.batch_work || d->batch_work != nullptr, "b2l_decode_step: %s needs batch_work (%s(max K, B) bytes)",
                  R.flag, R.tiling == CB ? "b2l_q8_linear_batch_workspace_bytes" : "b2l_w8_gemv_batch_workspace_bytes");
  }
  if (R.tiling == CB) B2L_CHECK_ARG(d->q8_layers != nullptr, "b2l_decode_step: B2L_F_Q8 needs q8_layers");
  if (d->adapters != nullptr) {
    for (int l = 0; l < d->n_layer; ++l) {
      if (d->adapters[l].len == 0) continue;   // no adapter in this layer
      if (int rc = check_adapter_prefix(&d->adapters[l], "b2l_decode_step")) return rc;
    }
  }
  if (d->loras != nullptr) {
    for (int l = 0; l < d->n_layer; ++l) {
      if (d->loras[l].r == 0) continue;   // no LoRA in this layer
      if (int rc = check_lora(&d->loras[l], 3 * d->n_embd, d->n_embd, "b2l_decode_step")) return rc;
    }
  }
  if (d->lora_sets != nullptr) {   // per-row LoRA: every layer's sets checked here, before any launch
    B2L_CHECK_SUPPORTED(d->loras == nullptr, "b2l_decode_step: lora_sets and loras do not combine");
    B2L_CHECK_SUPPORTED(!any_affine, "b2l_decode_step: lora_sets and LLaMA-Adapter v2 affines do not combine");
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
  // LLaMA-Adapter v2: every linear's affine runs in its own launch (b2l_q4_linear_args::out_affine)
  if (any_affine) {
    B2L_CHECK_SUPPORTED(R.affines || d->B == 1, "b2l_decode_step: LLaMA-Adapter v2 affines run at batch 1 only, got B=%d", d->B);
    B2L_CHECK_SUPPORTED(d->loras == nullptr, "b2l_decode_step: LLaMA-Adapter v2 affines and LoRA do not combine");
    auto ok = [](const b2l_out_affine& f) { return (f.scale == nullptr) == (f.bias == nullptr); };
    B2L_CHECK_ARG(ok(d->lm_head_affine), "b2l_decode_step: lm_head_affine needs both scale and bias (or neither)");
    B2L_CHECK_SUPPORTED(R.affines, "b2l_decode_step: affines need the batch-1 tiling (qw_mma) of every weight");
    for (int l = 0; d->affines != nullptr && l < d->n_layer; ++l) {
      const b2l_layer_affine& f = d->affines[l];
      B2L_CHECK_ARG(ok(f.c_attn) && ok(f.c_proj) && ok(f.c_fc12) && ok(f.mlp_proj),
                    "b2l_decode_step: affines[%d] needs both scale and bias (or neither) per linear", l);
      const b2l_layer& L = d->layers[l];
      B2L_CHECK_SUPPORTED(R.tiling == CB || (L.c_attn.qw_mma && L.c_proj.qw_mma && L.c_fc12.qw_mma && L.mlp_proj.qw_mma),
                          "b2l_decode_step: affines need the batch-1 tiling (qw_mma) of every weight");
    }
  }
  const int C = d->n_embd, hs = C / d->n_head, B = d->B;
  const int afl = d->flags & ~(B2L_F_W8 | B2L_F_Q8 | B2L_F_W8_BATCH | B2L_F_Q4_BATCH_I8 | B2L_F_Q8_BATCH);   // the attention's
  // the attention's view: B sequences of one token, or (stepwise) one sequence of B tokens
  const int aB = stepwise ? 1 : B, aT = stepwise ? B : 1;
  // every weight's tiling (lm_head's first: at batch 1 it picks the route), then every launch's own checks, so that
  // nothing is enqueued for a step that cannot run
  if (int rc = check_tiling(r, d, linear_of(d, d->n_layer, 0))) return rc;
  for (int l = 0; l < d->n_layer; ++l)
    for (int k = 0; k < 4; ++k)
      if (int rc = check_tiling(r, d, linear_of(d, l, k))) return rc;
  for (int l = 0; l <= d->n_layer; ++l) {
    for (int k = 0; k < (l < d->n_layer ? 4 : 1); ++k) {
      const Linear li = linear_of(d, l, k);
      if (int rc = in_step(linear(r, d, li, nullptr, false, stream), d, li)) return rc;
    }
    if (l < d->n_layer && kv8) {
      if (int rc = check_attention_kv8(d->qkv, &d->kv8[l], d->rope, d->input_pos, d->ring_start, d->att, d->attn_work, aB,
                                       aT, d->n_head, hs, d->S, d->block_size, afl, "b2l_decode_step"))
        return rc;
    } else if (l < d->n_layer) {
      const b2l_layer& L = d->layers[l];
      if (int rc = check_attention(d->qkv, L.k_cache, L.v_cache, d->rope, d->input_pos, d->ring_start, d->att,
                                   d->attn_work, aB, aT, d->n_head, hs, d->S, d->block_size, afl, "b2l_decode_step"))
        return rc;
    }
  }
  if (R.tiling == CB)   // llm.int8's kernels read x after they start writing y
    for (int l = 0; l <= d->n_layer; ++l)
      for (int k = 0; k < (l < d->n_layer ? 4 : 1); ++k) {
        const Linear li = linear_of(d, l, k);
        b2l_q8_linear_args a{};
        a.x = li.x; a.y = li.y; a.N = li.ldy; a.K = li.ldx;
        if (int rc = in_step(check_q8_disjoint(&a, B, r == Q8 ? "b2l_q8_linear" : "b2l_q8_linear_batch"), d, li)) return rc;
      }

  // Launches: from here on the only errors come from the device (a CUDA error, or b2l_q8_linear_batch finding no
  // 16-CTA clusters).
  // debug timeline: launch i of the step writes uint64[64] at timeline + 512*i (order: per Block c_attn,
  // attention, c_proj, fc12, mlp_proj; then lm_head)
  char* tlb = (char*)d->timeline;
  auto tl = [&](int i) -> void* { return tlb ? (void*)(tlb + 512 * i) : nullptr; };
  int rc;
  if ((rc = row_pos ? b2l_ring_advance_rows(d->input_pos, B, d->ring_start, d->S, stream)
                    : b2l_ring_advance(d->input_pos, stepwise ? B : 1, d->ring_start, d->S, stream)))
    return rc;
  if ((rc = b2l_embedding(d->idx, d->idx_is_i64, d->wte, d->x, B, C, d->vocab, stream))) return rc;
  const int pdl = d->flags & B2L_F_PDL;
  for (int l = 0; l < d->n_layer; ++l) {
    const b2l_layer& L = d->layers[l];
    if ((rc = linear(r, d, linear_of(d, l, 0), tl(5 * l), true, stream))) return rc;
    // LoRA on c_attn (lora.py:308-326): the low-rank term from rms_1(x), added into qkv in place
    if (d->loras != nullptr && d->loras[l].r != 0 &&
        (rc = b2l_lora_apply(&d->loras[l], d->x, C, L.rms_1, d->eps, d->qkv, 3 * C, B, 3 * C, C, pdl, stream)))
      return rc;
    // per-row LoRA: row b adds set lora_row_set[b]'s term (no launch in a layer where no set has one)
    if (d->lora_sets != nullptr &&
        (rc = lora_rows(d->lora_sets + l, (size_t)d->n_layer, d->n_lora_sets, true, d->lora_row_set, d->x, C, L.rms_1,
                        d->eps, d->qkv, 3 * C, B, 3 * C, C, pdl, stream, "b2l_decode_step")))
      return rc;
    const b2l_adapter_prefix* pre = (d->adapters != nullptr && d->adapters[l].len != 0) ? &d->adapters[l] : nullptr;
    if ((rc = kv8 ? attention_kv8_impl(d->qkv, &d->kv8[l], d->rope, d->input_pos, d->ring_start, d->att, d->attn_work, B,
                                       1, d->n_head, d->S, afl, d->block_size, pre, tl(5 * l + 1), (cudaStream_t)stream)
                  : attention_impl(d->qkv, L.k_cache, L.v_cache, d->rope, d->input_pos, d->ring_start, d->att, d->attn_work,
                                   aB, aT, d->n_head, hs, d->S, d->block_size, afl, pre, tl(5 * l + 1), (cudaStream_t)stream)))
      return rc;
    for (int k = 1; k < 4; ++k)
      if ((rc = linear(r, d, linear_of(d, l, k), tl(5 * l + k + 1), true, stream))) return rc;
  }
  return linear(r, d, linear_of(d, d->n_layer, 0), tl(5 * d->n_layer), true, stream);
}

"""-m gpu: llm.int8 on the whole-token decode step.  b2l_q8_linear (the batch-1 LLM.int8() linear with the RMSNorm
prologue and the affine / residual / SwiGLU epilogue) against the module ops it replaces, and the B2L_F_Q8 step
(LLaMA.int8_step) against the module path, bit for bit."""
import ctypes as C
from contextlib import nullcontext

import pytest
import torch

pytestmark = pytest.mark.gpu

import lit_llama_b200 as P  # noqa: E402
from lit_llama_b200 import _lib as L  # noqa: E402
from lit_llama_b200 import adapter as PA  # noqa: E402
from lit_llama_b200 import adapter_v2 as PV  # noqa: E402
from lit_llama_b200 import lora as PL  # noqa: E402
from lit_llama_b200.int8 import quantize_rows_int8  # noqa: E402
from lit_llama_b200.utils import quantization  # noqa: E402

THR = 6.0
EPS = 1e-5


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


# ----------------------------------------------------------------------------------------------- the kernel
def _weight(N, K, dev):
    cb, scb = quantize_rows_int8(torch.randn(N, K, device=dev) * 0.05)
    return cb, scb


def _row(kind, K, dev, norm):
    """(x, norm scale): `none` keeps every |x^| < 6; `several` puts a few columns of x^ over the threshold; `late`
    (RMSNorm only) has every |x| far below it and one column that crosses it only after the scale."""
    x = torch.randn(K, device=dev)
    g = torch.rand(K, device=dev) * 0.5 + 0.5
    if kind == "several":
        idx = torch.randperm(K, device=dev)[:7]
        if norm:
            g[idx] = 25.0
        else:
            x[idx] = torch.tensor([9.0, -7.5, 12.0, -30.0, 6.5, 8.0, -11.0], device=dev)
    elif kind == "late":
        x = x * 0.01
        x[K // 3] = 0.04
        g[K // 3] = 3.0
    else:
        x = x * (0.3 if not norm else 1.0)
    x, g = x.bfloat16(), g.bfloat16()
    if kind == "late":
        assert float(x.float().abs().max()) < THR
    return x, g


def _module_gemv(x, cb, scb):
    y = torch.empty(cb.shape[0], device=x.device, dtype=torch.bfloat16)
    L.check(L.lib().b2l_q8_gemv_cb(x.data_ptr(), cb.data_ptr(), scb.data_ptr(), None, y.data_ptr(), cb.shape[0],
                                   cb.shape[1], THR, 0, L.stream_ptr()), "b2l_q8_gemv_cb")
    return y


def _module(x, g, w, w2, epi, res, aff):
    """The module path: b2l_rmsnorm -> b2l_q8_gemv_cb [-> b2l_linear_affine] [-> b2l_add | b2l_silu_mul]."""
    lib = L.lib()
    if g is not None:
        xh = torch.empty_like(x)
        L.check(lib.b2l_rmsnorm(x.data_ptr(), g.data_ptr(), xh.data_ptr(), 1, x.numel(), EPS, L.stream_ptr()), "b2l_rmsnorm")
    else:
        xh = x
    outs = []
    for i, (cb, scb) in enumerate([w] + ([w2] if w2 is not None else [])):
        y = _module_gemv(xh, cb, scb)
        if aff is not None:
            N = y.numel()
            s, b = aff
            if w2 is not None:   # the kernel's vectors are interleaved 8 / 8; the module's are per linear
                s, b = (t.view(-1, 2, 8)[:, i].reshape(-1)[:N].contiguous() for t in (s, b))
            L.check(lib.b2l_linear_affine(y.data_ptr(), N, 1, N, s.data_ptr(), b.data_ptr(), L.stream_ptr()), "b2l_linear_affine")
        outs.append(y)
    if epi == L.EPI_RESIDUAL:
        out = torch.empty_like(outs[0])
        L.check(lib.b2l_add(res.data_ptr(), outs[0].data_ptr(), out.data_ptr(), out.numel(), L.stream_ptr()), "b2l_add")
        return out
    if epi == L.EPI_SWIGLU:
        out = torch.empty_like(outs[0])
        L.check(lib.b2l_silu_mul(outs[0].data_ptr(), outs[1].data_ptr(), out.data_ptr(), out.numel(), L.stream_ptr()), "b2l_silu_mul")
        return out
    return outs[0]


def _fused(x, g, w, w2, epi, res, aff, flags, y=None):
    cb, scb = w
    N, K = cb.shape
    y = torch.full((N,), float("nan"), device=x.device, dtype=torch.bfloat16) if y is None else y
    a = L.Q8LinearArgs(x=x.data_ptr(), cb=cb.data_ptr(), scb=scb.data_ptr(), y=y.data_ptr(), N=N, K=K, threshold=THR,
                       prologue=L.PRO_RMSNORM if g is not None else L.PRO_NONE,
                       norm_scale=None if g is None else g.data_ptr(), eps=EPS, epilogue=epi,
                       res=None if res is None else res.data_ptr(), flags=flags)
    if w2 is not None:
        a.cb2, a.scb2 = w2[0].data_ptr(), w2[1].data_ptr()
    if aff is not None:
        a.out_affine = L.OutAffine(aff[0].data_ptr(), aff[1].data_ptr())
    L.check(L.lib().b2l_q8_linear(C.byref(a), L.stream_ptr()), "b2l_q8_linear")
    return y


# (N, K): 7B c_attn / c_fc / mlp.c_proj, 13B c_proj, 65B c_fc / mlp.c_proj, K = 32768, N not a multiple of 16
SHAPES = [(12288, 4096), (11008, 4096), (4096, 11008), (5120, 5120), (22016, 8192), (8192, 22016), (1000, 32768),
          (4100, 4096), (1003, 512)]


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("kind", ["none", "several", "late"])
@pytest.mark.parametrize("pdl", [0, 1])
def test_q8_linear_equals_module_ops(dev, N, K, kind, pdl):
    w, w2 = _weight(N, K, dev), _weight(N, K, dev)
    res = (torch.randn(N, device=dev) * 2).bfloat16()
    n_aff = 16 * ((N + 7) // 8)
    aff = ((torch.rand(N, device=dev) + 0.5).bfloat16(), (torch.randn(N, device=dev) * 0.1).bfloat16())
    aff_glu = ((torch.rand(n_aff, device=dev) + 0.5).bfloat16(), (torch.randn(n_aff, device=dev) * 0.1).bfloat16())
    for norm in (True, False):
        x, g = _row(kind, K, dev, norm)
        if kind == "late" and norm:   # the mask of the un-normalised row misses the column that x^ puts over 6
            xh = torch.empty_like(x)
            L.check(L.lib().b2l_rmsnorm(x.data_ptr(), g.data_ptr(), xh.data_ptr(), 1, K, EPS, L.stream_ptr()), "b2l_rmsnorm")
            assert float(xh.float().half().float().abs().max()) >= THR
        elif kind == "late":
            continue
        g = g if norm else None
        cases = [(L.EPI_STORE, None, None, None), (L.EPI_STORE, None, None, aff), (L.EPI_SWIGLU, w2, None, None),
                 (L.EPI_SWIGLU, w2, None, aff_glu), (L.EPI_RESIDUAL, None, res, None), (L.EPI_RESIDUAL, None, res, aff)]
        for epi, second, r, af in cases:
            want = _module(x, g, w, second, epi, r, af)
            got = _fused(x, g, w, second, epi, r, af, pdl)
            assert torch.equal(got, want), (norm, epi, af is not None, int((got != want).sum()))


def test_q8_linear_residual_in_place_and_pdl_chain(dev):
    """The step's pattern: h = W1 rms(x), then x = x + W2 h written in place over the residual stream, as back-to-back
    PDL launches that each read what the one before wrote."""
    K = N = 4096
    w1, w2 = _weight(N, K, dev), _weight(N, K, dev)
    x0 = torch.randn(K, device=dev).bfloat16()
    g = (torch.rand(K, device=dev) + 0.5).bfloat16()
    want = x0.clone()
    for _ in range(4):
        h = _module(want, g, w1, None, L.EPI_STORE, None, None)
        want = _module(h, None, w2, None, L.EPI_RESIDUAL, want, None)
    got, h = x0.clone(), torch.empty_like(x0)
    for _ in range(4):
        _fused(got, g, w1, None, L.EPI_STORE, None, None, L.F_PDL, y=h)
        _fused(h, None, w2, None, L.EPI_RESIDUAL, got, None, L.F_PDL, y=got)
    assert torch.equal(got, want)


# ----------------------------------------------------------------------------------------------- the model
CFG = dict(block_size=64, vocab_size=256, n_layer=2, n_head=4, n_embd=512)
PROMPT = torch.tensor([5, 100, 3, 7, 200, 9, 31])
TOKS = [77, 12, 9, 150, 42, 3, 8, 199, 61, 20]


def _build(dev, kind, cfg=CFG, seed=1234):
    from oracle import adapter_oracle as A
    from oracle import adapter_v2_oracle as A2
    from oracle import llama_oracle as O
    from oracle import lora_oracle as LO

    n_layer, n_head, n_embd, vocab = cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"]
    ada = dict(adapter_prompt_length=10, adapter_start_layer=1)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("llm.int8"), (PL.lora(r=8, alpha=16, dropout=0.05) if kind == "lora" else nullcontext()):
            if kind in ("adapter", "adapter_v2"):
                model = PA.LLaMA(PA.LLaMAConfig(**cfg, **ada))
                if kind == "adapter_v2":
                    PV.add_adapter_v2_parameters_to_linear_layers(model)
            else:
                model = P.LLaMA(P.LLaMAConfig(**cfg))
    finally:
        torch.set_default_dtype(prev)
    if kind == "adapter":
        sd = A.adapter_state_dict(n_layer, n_head, n_embd, vocab, None, 10, 1, seed=seed, adapter_seed=4321)
    elif kind == "adapter_v2":
        sd = A2.adapter_v2_state_dict(n_layer, n_head, n_embd, vocab, None, 10, 1, v2_seed=2468)
    else:
        sd = O.synth_state_dict(n_layer, n_head, n_embd, vocab, None, dtype=torch.bfloat16, seed=seed)
        if kind == "lora":
            sd = dict(sd, **LO.lora_weights(n_layer, n_embd, seed=4321))
    model.load_state_dict(sd, strict=False)
    if kind == "lora":
        assert all(bool(blk.attn.c_attn.lora_B.abs().sum() > 0) for blk in model.transformer.h)
    return model.eval()


def _run(model, dev, S, toks=TOKS, reload=None):
    """Prefill + one decode per token; logits of every call and the logical KV caches at the end.  reload: (step,
    fn) calls fn() before that decode step."""
    T = PROMPT.numel()
    model.reset_cache()
    with torch.no_grad():
        out = [model(PROMPT.view(1, -1).to(dev), S, torch.arange(T, device=dev)).clone()]
        for i, t in enumerate(toks):
            if reload is not None and reload[0] == i:
                reload[1]()
            out.append(model(torch.tensor([[t]], device=dev), S, torch.tensor([T + i], device=dev)).clone())
        kv = model.logical_kv_caches()
    torch.cuda.synchronize()
    return out, kv


def _both(model, dev, S, **kw):
    model.int8_step = True
    fast = _run(model, dev, S, **kw)
    st = model._decode
    assert st is not None and st.args.flags & L.F_Q8 and st.graph is not None
    assert L.lib().b2l_decode_step_launches(C.byref(st.args)) == \
        5 * model.config.n_layer + 3 + (model.config.n_layer if st.args.loras else 0)
    model.int8_step = False
    slow = _run(model, dev, S, **kw)
    assert model._decode is None
    return fast, slow


def _assert_equal(fast, slow):
    for a, b in zip(fast[0], slow[0]):
        assert torch.equal(a, b), float((a.float() - b.float()).abs().max())
    for (ka, va), (kb, vb) in zip(fast[1], slow[1]):
        assert torch.equal(ka, kb) and torch.equal(va, vb)


@pytest.mark.parametrize("kind", ["plain", "adapter", "adapter_v2", "lora"])
@pytest.mark.parametrize("S", [32, 12])   # S = 12: the cache fills after 5 decode steps and the roll branch runs
def test_step_equals_module_path(dev, kind, S):
    model = _build(dev, kind)
    assert model._fast_decode_ok() == "q8"
    model.graph_after = 2   # eager steps, then graph replay
    _assert_equal(*_both(model, dev, S))


def test_default_keeps_the_module_path(dev):
    model = _build(dev, "plain")
    assert not P.LLaMA.int8_step
    _run(model, dev, 32, toks=TOKS[:3])
    assert model._decode is None and model._module_graph is not None
    with pytest.raises(RuntimeError, match="compact"):
        model.compact()


@pytest.mark.parametrize("widths", ["13B", "65B"])
def test_step_equals_module_path_wide(dev, widths):
    """Two Blocks at the 13B / 65B widths (head_size 128; 65B's n_hidden 22016 is mlp.c_proj's K)."""
    C_, nh = (5120, 40) if widths == "13B" else (8192, 64)
    cfg = dict(block_size=64, vocab_size=256, n_layer=2, n_head=nh, n_embd=C_)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("llm.int8"):
            model = P.LLaMA(P.LLaMAConfig(**cfg))
    finally:
        torch.set_default_dtype(prev)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, P.RMSNorm):
                m.scale.copy_(torch.rand_like(m.scale) + 0.5)
    model = model.eval()
    model.graph_after = 2
    fast, slow = _both(model, dev, 16, toks=TOKS[:8])
    _assert_equal(fast, slow)
    if widths == "13B":   # building the step makes no copy of any weight
        model.int8_step = True
        model.graph_after = 0
        with torch.no_grad():
            model.reset_cache()
            model(PROMPT.view(1, -1).to(dev), 16, torch.arange(7, device=dev))
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated(dev)
            model(torch.tensor([[3]], device=dev), 16, torch.tensor([7], device=dev))
            torch.cuda.synchronize()
            grown = torch.cuda.memory_allocated(dev) - before
        assert model._decode is not None
        smallest = C_ * C_   # c_proj's CB
        assert grown < smallest // 4, grown


def test_reload_between_tokens(dev):
    """Re-quantising one layer's weight between two tokens: the next token uses the new weights, on the step as on
    the module path (captured graph included)."""
    model = _build(dev, "plain")
    model.graph_after = 2
    lin = model.transformer.h[1].mlp.c_fc2
    orig = {"weight": lin.weight.data.clone(), "SCB": lin.weight.SCB.clone()}
    new = {"weight": torch.randn(lin.out_features, lin.in_features, device=dev, dtype=torch.bfloat16) * 0.05}
    reload = (5, lambda: lin.load_state_dict(new))
    model.int8_step = True
    fast = _run(model, dev, 32, reload=reload)
    assert model._decode is not None and model._decode.graph is not None
    lin.load_state_dict(orig)
    model.int8_step = False
    slow = _run(model, dev, 32, reload=reload)
    _assert_equal(fast, slow)
    lin.load_state_dict(orig)
    model.int8_step = True
    unchanged = _run(model, dev, 32)
    assert not torch.equal(unchanged[0][-1], fast[0][-1])
    assert all(torch.equal(a, b) for a, b in zip(unchanged[0][:6], fast[0][:6]))

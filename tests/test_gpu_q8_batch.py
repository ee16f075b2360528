"""-m gpu: llm.int8 at 2..16 rows on the whole-token step.  b2l_q8_linear_batch against the module ops it replaces
(b2l_rmsnorm -> b2l_q8_gemm -> b2l_linear_affine -> b2l_add / b2l_silu_mul) and, row by row, against b2l_q8_gemv_cb
with the batch's outlier mask; the B2L_F_Q8 | B2L_F_Q8_BATCH step (LLaMA.int8_step at B >= 2) against the module
path.  Every comparison is torch.equal.  Never against the B = 1 step: the outlier mask belongs to the batch."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

import lit_llama_b200 as P  # noqa: E402
from lit_llama_b200 import _lib as L  # noqa: E402
from lit_llama_b200.int8 import quantize_rows_int8  # noqa: E402
from lit_llama_b200.utils import quantization  # noqa: E402

from test_gpu_int8_step import PROMPT, TOKS, _build  # noqa: E402

THR = 6.0
EPS = 1e-5


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _weight(N, K, dev):
    return quantize_rows_int8(torch.randn(N, K, device=dev) * 0.05)


def _rows(kind, M, K, dev, norm):
    """(x [M, K], norm scale).  none: every |x^| < 6; one: a single row has an outlier; late: (RMSNorm) one column
    crosses 6 only after the scale; many: dozens of outlier columns; zero: an all-zero row (SCA = 0); all: a row
    whose every column is an outlier."""
    x = torch.randn(M, K, device=dev) * (1.0 if norm else 0.3)
    g = torch.rand(K, device=dev) * 0.5 + 0.5
    if kind == "one":
        if norm:
            x[M - 1, K // 5] = 0.0
            x[M - 1] *= 0.05
            x[M - 1, K // 5] = 40.0
        else:
            x[M - 1, K // 5] = -9.0
    elif kind == "late":
        x = x * 0.01
        x[:, K // 3] = 0.04
        g[K // 3] = 3.0
    elif kind == "many":
        idx = torch.randperm(K, device=dev)[:48]
        if norm:
            g[idx] = 25.0
        else:
            x[torch.arange(48, device=dev) % M, idx] = 8.0
    elif kind == "zero":
        x[0] = 0.0
        x[M - 1, 7] = 10.0 if not norm else x[M - 1, 7]
    elif kind == "all":
        x[M // 2] = 7.0 * torch.sign(torch.randn(K, device=dev))
        if norm:
            g[:] = 8.0
    return x.bfloat16(), g.bfloat16()


def _mask(xh):
    M, K = xh.shape
    m = torch.empty(K // 32, dtype=torch.int32, device=xh.device)
    L.check(L.lib().b2l_q8_outlier_mask(xh.data_ptr(), K, M, K, THR, m.data_ptr(), L.stream_ptr()), "b2l_q8_outlier_mask")
    return m


def _module(x, g, w, w2, epi, res, aff):
    """The module path at M rows: b2l_rmsnorm -> b2l_q8_gemm [-> b2l_linear_affine] [-> b2l_add | b2l_silu_mul];
    also returns x^ (for the per-row check)."""
    lib = L.lib()
    M, K = x.shape
    if g is not None:
        xh = torch.empty_like(x)
        L.check(lib.b2l_rmsnorm(x.data_ptr(), g.data_ptr(), xh.data_ptr(), M, K, EPS, L.stream_ptr()), "b2l_rmsnorm")
    else:
        xh = x
    outs = []
    for i, (cb, scb) in enumerate([w] + ([w2] if w2 is not None else [])):
        N = cb.shape[0]
        y = torch.empty((M, N), device=x.device, dtype=torch.bfloat16)
        nb = lib.b2l_q8_gemm_workspace_bytes(M, K)
        work = torch.empty(nb, dtype=torch.uint8, device=x.device)
        L.check(lib.b2l_q8_gemm(xh.data_ptr(), K, cb.data_ptr(), scb.data_ptr(), work.data_ptr(), nb, y.data_ptr(), N, M, N, K,
                                THR, 0, L.stream_ptr()), "b2l_q8_gemm")
        if aff is not None:
            s, b = aff
            if w2 is not None:   # the kernel's vectors are interleaved 8 / 8; the module's are per linear
                s, b = (t.view(-1, 2, 8)[:, i].reshape(-1)[:N].contiguous() for t in (s, b))
            L.check(lib.b2l_linear_affine(y.data_ptr(), N, M, N, s.data_ptr(), b.data_ptr(), L.stream_ptr()), "b2l_linear_affine")
        outs.append(y)
    if epi == L.EPI_RESIDUAL:
        out = torch.empty_like(outs[0])
        L.check(lib.b2l_add(res.data_ptr(), outs[0].data_ptr(), out.data_ptr(), out.numel(), L.stream_ptr()), "b2l_add")
        return out, xh
    if epi == L.EPI_SWIGLU:
        out = torch.empty_like(outs[0])
        L.check(lib.b2l_silu_mul(outs[0].data_ptr(), outs[1].data_ptr(), out.data_ptr(), out.numel(), L.stream_ptr()), "b2l_silu_mul")
        return out, xh
    return outs[0], xh


def _batch(x, g, w, w2, epi, res, aff, flags, y=None):
    cb, scb = w
    M, K = x.shape
    N = cb.shape[0]
    y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16) if y is None else y
    a = L.Q8LinearArgs(x=x.data_ptr(), cb=cb.data_ptr(), scb=scb.data_ptr(), y=y.data_ptr(), N=N, K=K, threshold=THR,
                       prologue=L.PRO_RMSNORM if g is not None else L.PRO_NONE,
                       norm_scale=None if g is None else g.data_ptr(), eps=EPS, epilogue=epi,
                       res=None if res is None else res.data_ptr(), flags=flags)
    if w2 is not None:
        a.cb2, a.scb2 = w2[0].data_ptr(), w2[1].data_ptr()
    if aff is not None:
        a.out_affine = L.OutAffine(aff[0].data_ptr(), aff[1].data_ptr())
    lib = L.lib()
    nb = lib.b2l_q8_linear_batch_workspace_bytes(K, M)
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    L.check(lib.b2l_q8_linear_batch(C.byref(a), M, ws.data_ptr(), nb, L.stream_ptr()), "b2l_q8_linear_batch")
    return y


def _cases(N, dev):
    res = None
    aff = ((torch.rand(N, device=dev) + 0.5).bfloat16(), (torch.randn(N, device=dev) * 0.1).bfloat16())
    n_aff = 16 * ((N + 7) // 8)
    aff_glu = ((torch.rand(n_aff, device=dev) + 0.5).bfloat16(), (torch.randn(n_aff, device=dev) * 0.1).bfloat16())
    return [(L.EPI_STORE, False, res, None), (L.EPI_STORE, False, res, aff), (L.EPI_SWIGLU, True, res, None),
            (L.EPI_SWIGLU, True, res, aff_glu), (L.EPI_RESIDUAL, False, "res", None), (L.EPI_RESIDUAL, False, "res", aff)]


def _check(dev, M, N, K, kind, pdl, norms=(True, False), per_row=False):
    w, w2 = _weight(N, K, dev), _weight(N, K, dev)
    res = (torch.randn(M, N, device=dev) * 2).bfloat16()
    for norm in norms:
        x, g = _rows(kind, M, K, dev, norm)
        g = g if norm else None
        for epi, glu, r, af in _cases(N, dev):
            want, xh = _module(x, g, w, w2 if glu else None, epi, res if r else None, af)
            got = _batch(x, g, w, w2 if glu else None, epi, res if r else None, af, pdl)
            assert torch.equal(got, want), (M, N, K, kind, norm, epi, af is not None, int((got != want).sum()))
        if per_row:   # each row against the batch-1 kernel with the batch's mask
            mask = _mask(xh)
            y = _batch(x, g, w, None, L.EPI_STORE, None, None, pdl)
            for m in range(M):
                ym = torch.empty(N, device=dev, dtype=torch.bfloat16)
                L.check(L.lib().b2l_q8_gemv_cb(xh[m].contiguous().data_ptr(), w[0].data_ptr(), w[1].data_ptr(), mask.data_ptr(),
                                               ym.data_ptr(), N, K, THR, 0, L.stream_ptr()), "b2l_q8_gemv_cb")
                assert torch.equal(y[m], ym), (M, m)


# (N, K): 7B c_attn / c_proj / c_fc / mlp.c_proj, 65B mlp.c_proj, K = 32768, a 32000-row lm_head, ragged N
SHAPES = [(12288, 4096), (4096, 4096), (11008, 4096), (4096, 11008), (8192, 22016), (1000, 32768), (32000, 4096),
          (1003, 512), (4100, 1024)]


@pytest.mark.parametrize("M", [2, 3, 5, 8, 9, 12, 16])
@pytest.mark.parametrize("N,K", SHAPES)
def test_kernel_equals_module_ops(dev, M, N, K):
    _check(dev, M, N, K, "many" if M % 2 else "none", pdl=M % 2, per_row=(N, K) in ((4096, 11008), (1003, 512)))


@pytest.mark.parametrize("kind", ["none", "one", "late", "many", "zero", "all"])
@pytest.mark.parametrize("M", [2, 9, 16])
@pytest.mark.parametrize("pdl", [0, 1])
def test_outlier_cases(dev, kind, M, pdl):
    norms = (True,) if kind == "late" else (True, False)
    _check(dev, M, 4096, 4096, kind, pdl, norms=norms, per_row=True)
    if kind == "one":   # the row's outlier is an outlier column of every row
        x, g = _rows(kind, M, 4096, dev, False)
        m = _mask(x)
        assert int(m.ne(0).sum()) >= 1


def test_pdl_chain_in_place(dev):
    """h = W1 rms(x), then x = x + W2 h in place over the residual stream, as back-to-back PDL launches."""
    M, K = 8, 4096
    w1, w2 = _weight(K, K, dev), _weight(K, K, dev)
    x0 = torch.randn(M, K, device=dev).bfloat16()
    g = (torch.rand(K, device=dev) + 0.5).bfloat16()
    want = x0.clone()
    for _ in range(4):
        h, _ = _module(want, g, w1, None, L.EPI_STORE, None, None)
        want, _ = _module(h, None, w2, None, L.EPI_RESIDUAL, want, None)
    got, h = x0.clone(), torch.empty_like(x0)
    for _ in range(4):
        _batch(got, g, w1, None, L.EPI_STORE, None, None, L.F_PDL, y=h)
        _batch(h, None, w2, None, L.EPI_RESIDUAL, got, None, L.F_PDL, y=got)
    assert torch.equal(got, want)


# ----------------------------------------------------------------------------------------------- the step
def _run(model, dev, S, B, toks=TOKS, reload=None):
    """A different prompt per row (prefill at B rows), then one decode per step with a different token per row."""
    T = PROMPT.numel()
    g = torch.Generator().manual_seed(B)
    prompts = torch.stack([PROMPT.roll(b) for b in range(B)]).to(dev)
    model.reset_cache()
    with torch.no_grad():
        out = [model(prompts, S, torch.arange(T, device=dev)).clone()]
        for i, t in enumerate(toks):
            if reload is not None and reload[0] == i:
                reload[1]()
            idx = ((torch.randperm(256, generator=g)[:B] + t) % 256).view(B, 1).to(dev)
            out.append(model(idx, S, torch.tensor([T + i], device=dev)).clone())
        kv = model.logical_kv_caches()
    torch.cuda.synchronize()
    return out, kv


def _both(model, dev, S, B, **kw):
    model.int8_step = True
    fast = _run(model, dev, S, B, **kw)
    st = model._decode
    assert st is not None and st.args.flags & L.F_Q8 and st.args.flags & L.F_Q8_BATCH and st.graph is not None
    n = model.config.n_layer
    assert L.lib().b2l_decode_step_launches(C.byref(st.args)) == 2 + n * (4 * 2 + 1) + 2 + (n if st.args.loras else 0)
    model.int8_step = False
    slow = _run(model, dev, S, B, **kw)
    assert model._decode is None
    return fast, slow


def _assert_equal(fast, slow):
    for a, b in zip(fast[0], slow[0]):
        assert torch.equal(a, b), float((a.float() - b.float()).abs().max())
    for (ka, va), (kb, vb) in zip(fast[1], slow[1]):
        assert torch.equal(ka, kb) and torch.equal(va, vb)


@pytest.mark.parametrize("kind", ["plain", "adapter", "adapter_v2", "lora"])
@pytest.mark.parametrize("B", [2, 4, 8, 16])
@pytest.mark.parametrize("S", [32, 12])   # S = 12: the roll branch runs
def test_step_equals_module_path(dev, kind, B, S):
    model = _build(dev, kind)
    model.graph_after = 2   # eager steps, then graph replay
    _assert_equal(*_both(model, dev, S, B))


@pytest.mark.parametrize("widths", ["13B", "65B"])
def test_step_equals_module_path_wide(dev, widths):
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
    _assert_equal(*_both(model, dev, 16, 4, toks=TOKS[:6]))
    if widths == "13B":   # building the batched step makes no copy of any weight
        model.int8_step = True
        model.graph_after = 0
        with torch.no_grad():
            model.reset_cache()
            model(PROMPT.view(1, -1).repeat(4, 1).to(dev), 16, torch.arange(7, device=dev))
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated(dev)
            model(torch.tensor([[3], [4], [5], [6]], device=dev), 16, torch.tensor([7], device=dev))
            torch.cuda.synchronize()
            grown = torch.cuda.memory_allocated(dev) - before
        assert model._decode is not None and model._decode.args.flags & L.F_Q8_BATCH
        assert grown < C_ * C_ // 4, grown


def test_reload_between_tokens(dev):
    model = _build(dev, "plain")
    model.graph_after = 2
    lin = model.transformer.h[1].mlp.c_fc2
    orig = {"weight": lin.weight.data.clone(), "SCB": lin.weight.SCB.clone()}
    new = {"weight": torch.randn(lin.out_features, lin.in_features, device=dev, dtype=torch.bfloat16) * 0.05}
    reload = (5, lambda: lin.load_state_dict(new))
    model.int8_step = True
    fast = _run(model, dev, 32, 4, reload=reload)
    assert model._decode is not None and model._decode.graph is not None
    lin.load_state_dict(orig)
    model.int8_step = False
    slow = _run(model, dev, 32, 4, reload=reload)
    _assert_equal(fast, slow)
    lin.load_state_dict(orig)
    model.int8_step = True
    unchanged = _run(model, dev, 32, 4)
    assert not torch.equal(unchanged[0][-1], fast[0][-1])


def test_batch_1_and_17_keep_their_paths(dev):
    model = _build(dev, "plain")
    model.int8_step = True
    _run(model, dev, 32, 1, toks=TOKS[:3])
    st = model._decode
    assert st is not None and st.args.flags & L.F_Q8 and not st.args.flags & L.F_Q8_BATCH and st.batch_ws is None
    model._decode = None
    _run(model, dev, 32, 17, toks=TOKS[:3])
    assert model._decode is None and model._module_graph is not None and model._module_graph["key"][0] == 17

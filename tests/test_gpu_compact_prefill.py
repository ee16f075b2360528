"""-m gpu: the prefill GEMM on the resident batch-1 tilings (B2L_F_GEMM_I8), so a compacted gptq.int4 / gptq.int8 model
prefills, refills and evaluates without rebuilding any weight layout.

1. Kernel: b2l_q4_gemm / b2l_w8_gemm (and the _nll forms) reading b2l_q4_tile_i8 / b2l_w8_tile_i8, or one half of an
   interleaved fc1|fc2 tiling, equal the same calls on today's sources (b2l_q4_tile, quant_weight) bit for bit.
2. Model: after compact(), with every untile / re-tile path made to raise, prefill, a packed refill_rows, window_nll
   and LoRA / LLaMA-Adapter v2 models over the compacted base equal the uncompacted model bit for bit.
3. Memory: a compacted prefill holds no transient weight copy."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _levels(dev, g, N, K, bits):
    """Random packed levels in the reference layout (uint8 [K/epb][N], viewed (N, K/epb))."""
    return torch.randint(0, 256, (K // (8 // bits), N), dtype=torch.uint8, device=dev, generator=g).t()


def _sz(dev, g, N, bits, dtype):
    sc = (torch.rand(N, 1, device=dev, generator=g) * 0.01 + 0.002).to(dtype)
    z = torch.randint(0, 2**bits, (N, 1), device=dev, generator=g).to(dtype)
    return sc, z


def _tile_i8(qw, N, K, bits):
    from lit_llama_b200.quantization import tile_i8

    return tile_i8(qw, N, K, bits)


def _own(qw, N, K, bits):
    """Today's source: b2l_q4_tile's tiling at 4 bits, quant_weight itself at 8."""
    if bits == 8:
        return qw
    L = _L()
    t = torch.empty(L.lib().b2l_q4_tiled_bytes(N, K), dtype=torch.uint8, device=qw.device)
    L.check(L.lib().b2l_q4_tile(qw.data_ptr(), t.data_ptr(), N, K, L.stream_ptr()), "b2l_q4_tile")
    return t


def _gemm(bits, x, wt, sc, z, N, flags=0, targets=None):
    L = _L()
    M, K = x.shape
    y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16)
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=wt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                       sz_dtype=L.sz_dtype_of(sc), y=y.data_ptr(), ldy=N, M=M, N=N, K=K, prologue=L.PRO_NONE, norm_scale=None,
                       eps=0.0, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=flags)
    kind = "w8" if bits == 8 else "q4"
    if targets is None:
        L.check(getattr(L.lib(), f"b2l_{kind}_gemm")(C.byref(a), L.stream_ptr()), f"b2l_{kind}_gemm")
        return y
    from lit_llama_b200.evaluate import _nll_args

    a.M = targets.numel()
    nl, (nll, s, _ws) = _nll_args(targets, targets.numel(), N)
    L.check(getattr(L.lib(), f"b2l_{kind}_gemm_nll")(C.byref(a), C.byref(nl), L.stream_ptr()), f"b2l_{kind}_gemm_nll")
    torch.cuda.synchronize()
    return nll, s


# --------------------------------------------------------------------------------------------- 1. kernel
# (N, K): 200 is a multiple of neither 16 nor 128; 7B / 65B-vocab widths; 13B c_attn (15360 x 5120)
SHAPES = [(200, 64), (200, 4096), (4096, 4096), (4096, 11008), (11008, 4096), (12288, 4096), (32000, 4096),
          (4096, 64), (15360, 5120)]


@pytest.mark.parametrize("sz", ["bf16", "fp32"])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K", SHAPES)
def test_i8_source_equals_todays_source(dev, N, K, bits, sz):
    L = _L()
    if sz == "fp32" and (N, K) not in ((200, 64), (200, 4096), (12288, 4096)):
        pytest.skip("fp32 scales / zeros: three shapes are enough")
    g = torch.Generator(device=dev).manual_seed(N * 7 + K + bits)
    qw = _levels(dev, g, N, K, bits)
    sc, z = _sz(dev, g, N, bits, torch.bfloat16 if sz == "bf16" else torch.float32)
    own, i8 = _own(qw, N, K, bits), _tile_i8(qw, N, K, bits)
    for M in ((2,) if bits == 8 else ()) + (17, 128, 129, 600):
        x = torch.randn(M, K, device=dev, generator=g).bfloat16()
        want = _gemm(bits, x, own, sc, z, N)
        got = _gemm(bits, x, i8, sc, z, N, flags=L.F_GEMM_I8)
        assert not torch.isnan(want).any()
        assert torch.equal(got, want), (N, K, M)


# nh: a multiple of 8 but not of 16 (200), of 16 but not of 128 (1040), the 7B hidden width
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("nh,K", [(200, 64), (1040, 4096), (11008, 4096)])
def test_half_of_an_interleaved_tiling_equals_the_layer(dev, nh, K, bits):
    """c_fc1 / c_fc2 read as rows 0..7 / 8..15 of every 16-row block of the fc1|fc2 tiling LLaMA._fc12(i, "i8") builds."""
    L = _L()
    g = torch.Generator(device=dev).manual_seed(nh + K + bits)
    q1, q2 = _levels(dev, g, nh, K, bits), _levels(dev, g, nh, K, bits)
    (s1, z1), (s2, z2) = _sz(dev, g, nh, bits, torch.bfloat16), _sz(dev, g, nh, bits, torch.bfloat16)
    kb = K // (8 // bits)
    both = torch.stack((q1.reshape(nh // 8, 8, kb), q2.reshape(nh // 8, 8, kb)), dim=1).reshape(2 * nh, kb)
    fc12 = _tile_i8(both.t().contiguous().t(), 2 * nh, K, bits)
    for M in ((2,) if bits == 8 else ()) + (17, 129, 600):
        x = torch.randn(M, K, device=dev, generator=g).bfloat16()
        for q, s, z, half in ((q1, s1, z1, L.F_GEMM_I8_LO), (q2, s2, z2, L.F_GEMM_I8_HI)):
            want = _gemm(bits, x, _own(q, nh, K, bits), s, z, nh)
            got = _gemm(bits, x, fc12, s, z, nh, flags=L.F_GEMM_I8 | half)
            assert torch.equal(got, want), (nh, K, M, half)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K", [(200, 4096), (32000, 4096)])
def test_nll_epilogue_on_the_i8_source(dev, N, K, bits):
    L = _L()
    g = torch.Generator(device=dev).manual_seed(N + bits)
    qw = _levels(dev, g, N, K, bits)
    sc, z = _sz(dev, g, N, bits, torch.bfloat16)
    own, i8 = _own(qw, N, K, bits), _tile_i8(qw, N, K, bits)
    for T in (18, 130, 600):
        x = torch.randn(T, K, device=dev, generator=g).bfloat16()
        t = torch.randint(0, N, (T - 1,), device=dev, generator=g)
        nll0, s0 = _gemm(bits, x, own, sc, z, N, targets=t)
        nll1, s1 = _gemm(bits, x, i8, sc, z, N, flags=L.F_GEMM_I8, targets=t)
        assert torch.isfinite(s0) and torch.equal(nll1, nll0) and torch.equal(s1, s0), (N, T)


# --------------------------------------------------------------------------------------------- 2. model
CFG128 = dict(block_size=512, vocab_size=256, n_layer=2, n_head=4, n_embd=512)   # head_size 128


def _no_rebuild(monkeypatch):
    """Every path that rebuilds a weight layout from a compacted model's resident copy raises."""
    from lit_llama_b200.model import LLaMA
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    def boom(*a, **k):
        raise AssertionError("a compacted prefill must read only the resident tiling")

    monkeypatch.setattr(ColBlockQuantizedLinear, "reference_quant_weight", boom)
    monkeypatch.setattr(ColBlockQuantizedLinear, "tiled", boom)
    monkeypatch.setattr(LLaMA, "_fc_from_fc12", boom)
    for name in ("b2l_q4_untile_i8", "b2l_w8_untile_i8", "b2l_q4_tile"):
        monkeypatch.setattr(_L().lib(), name, boom)


def _prompts(dev, V, lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, V, (n,), generator=g).to(torch.int32).to(dev) for n in lengths]


def _model_outputs(model, dev, prompts, S):
    """Prefill logits of each prompt alone, a packed prefill_rows of the first three, window_nll of the last."""
    from lit_llama_b200.evaluate import window_nll

    out = []
    with torch.no_grad():
        for p in prompts:
            model.reset_cache()
            out.append(model(p.view(1, -1), S, torch.arange(p.numel(), device=dev)).float().cpu())
        model.reset_cache()
        out.append(model.prefill_rows(prompts[:3], S).float().cpu())
        nll, s = window_nll(model, prompts[-1].view(1, -1))
        out += [nll.cpu(), s.cpu()]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_compacted_prefill_refill_and_eval_read_only_the_resident_copy(dev, mode, monkeypatch):
    from gpu_util import build_tiny

    lengths = (17, 64, 300) if mode == "gptq.int4" else (2, 17, 64, 300)
    model, _, _ = build_tiny(dev, CFG128, mode=mode, seed=31)
    prompts = _prompts(dev, CFG128["vocab_size"], lengths, seed=3)
    assert model._pack_plan([p.numel() for p in prompts[:3]]) == [0, 1, 2]
    before = _model_outputs(model, dev, prompts, 320)
    model.reset_cache()
    model.compact()
    _no_rebuild(monkeypatch)
    after = _model_outputs(model, dev, prompts, 320)
    for i, (a, b) in enumerate(zip(before, after)):
        assert torch.equal(a, b), i


@pytest.mark.parametrize("kind", ["lora", "adapter_v2"])
@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_lora_and_adapter_v2_over_a_compacted_base(dev, kind, mode, monkeypatch):
    if kind == "lora":
        import test_gpu_lora as T

        build = lambda: T.build(dev, mode)[0]   # noqa: E731
    else:
        import test_gpu_adapter_v2 as T

        # a 20-token adapter prefix: its keys and values go through c_attn at M = 20, on the prefill GEMM (10 rows
        # would take gptq.int4's 9..16-row kernel, which still rebuilds its layout)
        build = lambda: T.build(dev, dict(T.CFG128, adapter_prompt_length=20), mode)[0]   # noqa: E731
    ref = build()
    prompts = _prompts(dev, 256, (20, 45), seed=9)

    def outs(model):
        res = []
        with torch.no_grad():
            for p in prompts:
                model.reset_cache()
                res.append(model(p.view(1, -1), 48, torch.arange(p.numel(), device=dev)).float().cpu())
        torch.cuda.synchronize()
        return res

    want = outs(ref)
    cm = build()
    cm.compact()
    _no_rebuild(monkeypatch)
    for a, b in zip(want, outs(cm)):
        assert torch.equal(a, b)


# --------------------------------------------------------------------------------------------- 3. memory
@pytest.mark.parametrize("bits", [4, 8])
def test_compacted_prefill_holds_no_weight_copy(dev, bits):
    """7B widths, two blocks, vocab 32000: a T = 64 prefill raises the peak above the resident level by less than the
    weights of the smallest linear (attn.c_proj); rebuilding any one layout would hold at least that much."""
    import gpu_util  # noqa: F401  (puts tools/ on sys.path)
    from diag import _random_w8_model

    model = _random_w8_model("7B", dev, seed=7, n_layer=2, bits=bits).compact()
    idx = torch.randint(0, 32000, (1, 64), device=dev, dtype=torch.int32)
    with torch.no_grad():
        model(idx, 64, torch.arange(64, device=dev))   # the KV cache and RoPE table exist from here on
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        y = model(idx, 64, torch.arange(64, device=dev))
        torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    smallest = 4096 * 4096 * bits // 8
    assert y.shape == (1, 64, 32000)
    assert peak < smallest, (peak, smallest)
    del model, y
    torch.cuda.empty_cache()

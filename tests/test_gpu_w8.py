"""-m gpu: gptq.int8 on its own kernels -- the batch-1 kernel with 8-bit weights (b2l_w8_gemv, tiling b2l_w8_tile_i8),
the wgmma GEMM with 8-bit weights (b2l_w8_gemm), the fused decode step under B2L_F_W8 and one resident weight copy."""
import ctypes as C

import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

from oracle import llama_oracle as O  # noqa: E402

CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _tile(qw, N, K):
    from lit_llama_b200.quantization import tile_i8

    return tile_i8(qw, N, K, 8)


def _gemv(x, qt, sc, z, N, K, *, y=None, prologue=0, norm_scale=None, epilogue=0, res=None, grid=0, flags=0, n_out=None):
    L = _L()
    n_out = n_out or N
    y = torch.zeros((1, n_out), device=x.device, dtype=torch.bfloat16) if y is None else y
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                       sz_dtype=L.sz_dtype_of(sc), y=y.data_ptr(), ldy=n_out, M=1, N=N, K=K, prologue=prologue,
                       norm_scale=None if norm_scale is None else norm_scale.data_ptr(), eps=1e-5, epilogue=epilogue,
                       res=None if res is None else res.data_ptr(), ldres=N, split_k=grid, flags=flags)
    L.check(L.lib().b2l_w8_gemv(C.byref(a), L.stream_ptr()), "b2l_w8_gemv")
    return y


def _lin(lv, qw, sc, z, dev):
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    N, K = lv.shape
    lin = ColBlockQuantizedLinear(K, N, False, bits=8, tile_cols=-1).to(dev)
    lin.load_state_dict({"quant_weight": qw, "scales": sc, "zeros": z})
    lin.scales, lin.zeros = lin.scales.to(sc.dtype), lin.zeros.to(z.dtype)
    return lin


@pytest.mark.parametrize("N,K", [(16, 64), (130, 256), (4096, 4096), (22016, 4096)])
def test_tile_roundtrip_bit_exact(dev, N, K):
    from gpu_util import rand_q4

    L = _L()
    lv, qw, _, _ = rand_q4(N, K, dev, seed=N + K, bits=8)
    qt = _tile(qw, N, K)
    back = torch.empty_like(qw)
    L.check(L.lib().b2l_w8_untile_i8(qt.data_ptr(), back.data_ptr(), N, K, L.stream_ptr()), "untile")
    assert torch.equal(back, qw)
    # the documented layout, decoded on the host: [N/16][K/64][2 chunks][32 lanes][4 words]
    w = qt.view(torch.int32).reshape((N + 15) // 16, K // 64, 2, 32, 4).cpu()
    lvc = lv.cpu()
    for rb, kb, c, lane, wd in [(0, 0, 0, 0, 0), (0, K // 64 - 1, 1, 31, 3), ((N - 1) // 16, 0, 1, 13, 2), (0, 0, 0, 6, 1)]:
        word = int(w[rb, kb, c, lane, wd]) & 0xFFFFFFFF
        row = 16 * rb + lane // 4 + 8 * (wd & 1)
        for i in range(4):
            k = 64 * kb + 32 * c + 8 * (lane % 4) + 4 * (wd >> 1) + i
            assert ((word >> (8 * i)) & 0xFF) == (int(lvc[row, k]) if row < N else 0)


@pytest.mark.parametrize("N", [16, 48, 130, 4096, 32000])
@pytest.mark.parametrize("K", [64, 192, 4096, 11008, 22016])
def test_gemv_vs_exact_any_grid_and_pdl(dev, N, K):
    from gpu_util import assert_q4_linear_close, rand_q4

    if N * K > 4096 * 22016:
        pytest.skip("covered by the smaller shapes")
    lv, qw, sc, z = rand_q4(N, K, dev, seed=3 * N + K, bits=8)
    qt = _tile(qw, N, K)
    x = (torch.randn(1, K, generator=torch.Generator().manual_seed(K)) * 2).bfloat16().to(dev)
    y = _gemv(x, qt, sc, z, N, K)
    assert_q4_linear_close(y, x, lv, sc, z, min_equal=0.995)
    for grid, flags in [(1, 0), (3, 1), (0, 1), (7, 0)]:   # forced tiny grids, with and without PDL: same integers
        assert torch.equal(_gemv(x, qt, sc, z, N, K, grid=grid, flags=flags), y), (grid, flags)


def test_gemv_f32_scales(dev):
    from gpu_util import assert_q4_linear_close, rand_q4

    N, K = 256, 1024
    lv, qw, sc, z = rand_q4(N, K, dev, seed=5, bits=8, sz_dtype=torch.float32)
    x = torch.randn(1, K, generator=torch.Generator().manual_seed(5)).bfloat16().to(dev)
    assert_q4_linear_close(_gemv(x, _tile(qw, N, K), sc, z, N, K), x, lv, sc, z, min_equal=0.995)


def test_gemv_fused_prologue_and_epilogues_match_module_ops(dev):
    import lit_llama_b200 as P
    from gpu_util import rand_q4

    L = _L()
    g = torch.Generator().manual_seed(11)
    N, K = 1024, 2048
    lv, qw, sc, z = rand_q4(N, K, dev, seed=11, bits=8)
    lin, qt = _lin(lv, qw, sc, z, dev), _tile(qw, N, K)
    x = torch.randn(1, K, generator=g).bfloat16().to(dev)
    # RMSNorm prologue == RMSNorm module, then the linear
    norm = P.RMSNorm(K).to(dev).bfloat16()
    norm.scale.data = (1 + 0.1 * torch.randn(K, generator=g)).bfloat16().to(dev)
    with torch.no_grad():
        want = lin(norm(x))
    got = _gemv(x, qt, sc, z, N, K, prologue=L.PRO_RMSNORM, norm_scale=norm.scale.data)
    assert float((got == want).float().mean()) >= 0.99
    torch.testing.assert_close(got.float(), want.float(), rtol=2 ** -7, atol=1e-3)
    # residual epilogue == linear, then x + h
    xs = torch.randn(1, N, generator=g).bfloat16().to(dev)
    xk = torch.randn(1, N, generator=g).bfloat16().to(dev)
    lv2, qw2, sc2, z2 = rand_q4(N, N, dev, seed=12, bits=8)
    lin2 = _lin(lv2, qw2, sc2, z2, dev)
    with torch.no_grad():
        want = lin2(xk).float() + xs.float()
    got = _gemv(xk, _tile(qw2, N, N), sc2, z2, N, N, epilogue=L.EPI_RESIDUAL, res=xs)
    assert torch.equal(got, want.bfloat16())
    # SwiGLU epilogue on the 8 / 8 interleave == silu(fc1(x)) * fc2(x)
    nh = N // 2
    inter = torch.stack((lv[:nh].reshape(nh // 8, 8, K), lv[nh:].reshape(nh // 8, 8, K)), 1).reshape(N, K)
    qwi = inter.t().contiguous().t()
    sci = torch.stack((sc[:nh].reshape(nh // 8, 8, 1), sc[nh:].reshape(nh // 8, 8, 1)), 1).reshape(N, 1).contiguous()
    zi = torch.stack((z[:nh].reshape(nh // 8, 8, 1), z[nh:].reshape(nh // 8, 8, 1)), 1).reshape(N, 1).contiguous()
    a = _lin(lv[:nh], qw[:nh].t().contiguous().t(), sc[:nh].contiguous(), z[:nh].contiguous(), dev)
    b = _lin(lv[nh:], qw[nh:].t().contiguous().t(), sc[nh:].contiguous(), z[nh:].contiguous(), dev)
    with torch.no_grad():
        ya, yb = a(x), b(x)
    h = torch.empty_like(ya)
    L.check(L.lib().b2l_silu_mul(ya.data_ptr(), yb.data_ptr(), h.data_ptr(), ya.numel(), L.stream_ptr()), "silu_mul")
    got = _gemv(x, _tile(qwi, N, K), sci, zi, N, K, epilogue=L.EPI_SWIGLU, n_out=nh)
    assert float((got == h).float().mean()) >= 0.99
    torch.testing.assert_close(got.float(), h.float(), rtol=2 ** -7, atol=1e-3)


@pytest.mark.parametrize("N,K", [(130, 256), (4096, 4096), (11008, 4096), (5120, 13824)])
@pytest.mark.parametrize("M", [2, 8, 17, 300, 4096])
def test_gemm_vs_dense_and_exact(dev, N, K, M):
    from gpu_util import rand_q4, ref_linear, relerr

    if N * K * M > 4096 * 11008 * 4096:
        pytest.skip("covered by the smaller shapes")
    lv, qw, sc, z = rand_q4(N, K, dev, seed=N + 7 * K + M, bits=8)
    lin = _lin(lv, qw, sc, z, dev)
    x = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).bfloat16().to(dev)
    with torch.no_grad():
        y = lin(x)
    W = lin.get_weight(torch.bfloat16).float()
    want = x.float() @ W.t()
    mag = x.float().abs() @ W.abs().t()
    err = (y.float() - want).abs()
    assert bool((err <= want.abs() * 2.0 ** -8 + mag * 2.0 ** -16 + 1e-30).all()), float(err.max())
    assert relerr(y, ref_linear(x, lv, sc, z)) < 1e-3 + 2.0 ** -9


@pytest.mark.parametrize("N,K", [(130, 256), (4096, 4096)])
def test_gemm_multiplies_get_weight_bit_for_bit(dev, N, K):
    """x = the K x K identity: every output is one exact product, so y must be get_weight(bf16).T bit for bit."""
    from gpu_util import rand_q4

    lv, qw, sc, z = rand_q4(N, K, dev, seed=N, bits=8)
    lin = _lin(lv, qw, sc, z, dev)
    x = torch.eye(K, device=dev, dtype=torch.bfloat16)
    with torch.no_grad():
        y = lin(x)
    assert torch.equal(y, lin.get_weight(torch.bfloat16).t())


def test_golden_cases_per_row_8bit(dev):
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    cases = [c for c in load_golden("quant_cases.pt") if c["bits"] == 8 and c["groupsize"] == -1]
    assert cases
    for c in cases:
        out_f, in_f = c["w"].shape
        lin = ColBlockQuantizedLinear(in_f, out_f, False, bits=8, tile_cols=-1).to(dev)
        lin.load_state_dict({"quant_weight": c["quant_weight"], "scales": c["scales"].bfloat16(), "zeros": c["zeros"].bfloat16()})
        lin.scales, lin.zeros = lin.scales.bfloat16(), lin.zeros.bfloat16()
        assert lin.w8_gemv_capable
        x = c["x"].bfloat16().to(dev)
        exact = O.qlinear_exact(x.cpu().float(), c["quant_weight"], c["scales"].bfloat16(), c["zeros"].bfloat16(), 8, in_f)
        with torch.no_grad():
            rows = torch.cat([lin(x[i : i + 1]) for i in range(x.shape[0])]).float().cpu()   # M = 1: b2l_w8_gemv
            full = lin(x).float().cpu()                                                      # M > 1: b2l_w8_gemm
        for y in (rows, full):
            torch.testing.assert_close(y, c["y_bf16"].float(), rtol=2.0 ** -7, atol=5e-3)
            assert (y - exact).norm() / exact.norm() < 1e-3 + 2.0 ** -9


def _close(a, b, bar=1e-2):
    a, b = a.float().cpu(), b.float().cpu()
    r = float((a - b).norm() / b.norm())
    assert r < bar, r


def test_tiny_model_vs_oracle(dev):
    """Prefill, eager and graph-replayed decode on the fused step, the roll branch and no-cache, against the oracle."""
    from gpu_util import build_tiny

    model, oracle, _ = build_tiny(dev, CFG, mode="gptq.int8", seed=8)
    assert model._fast_decode_ok() == "w8"
    prompt = torch.tensor([[3, 17, 40, 41, 2, 77, 5]])
    for S in (16, 8):   # S = 8: the cache fills and the roll branch runs
        model.reset_cache()
        oracle.reset_cache()
        with torch.no_grad():
            _close(model(prompt.to(dev), S, torch.arange(7, device=dev)), oracle.forward(prompt, S, torch.arange(7)))
            for i, t in enumerate([9, 60, 3, 77, 12, 45]):   # > graph_after steps: the later ones replay the graph
                got = model(torch.tensor([[t]], device=dev), S, torch.tensor([7 + i], device=dev))
                _close(got, oracle.forward(torch.tensor([[t]]), S, torch.tensor([7 + i])))
        assert model._decode is not None and model._decode.graph is not None
    model.reset_cache()
    with torch.no_grad():
        _close(model(prompt.to(dev)), oracle.forward(prompt))


def test_generate_greedy_matches_oracle(dev):
    import lit_llama_b200 as P
    from gpu_util import build_tiny

    model, oracle, _ = build_tiny(dev, CFG, mode="gptq.int8", seed=9)
    prompt = torch.tensor([3, 17, 40, 41, 2, 77, 5], dtype=torch.int32)
    y = P.generate(model, prompt.to(dev), 12, top_k=1)
    want = O.generate(oracle, prompt, 12, top_k=1)
    assert float((y.cpu() == want).float().mean()) >= 0.9, (y.tolist(), want.tolist())


def _run(m, dev, B=1, steps=(9, 11, 60, 2)):
    prompt = torch.tensor([[3, 17, 40, 41, 2, 77, 5]], device=dev)
    m.reset_cache()
    out = [m(prompt.repeat(B, 1), 16, torch.arange(7, device=dev))]
    for i, t in enumerate(steps):
        out.append(m(torch.full((B, 1), t, device=dev), 16, torch.tensor([7 + i], device=dev)).clone())
    return out


def test_fused_step_equals_module_path(dev):
    """The fused step (RMSNorm / SwiGLU / residual inside the linears) against the module path: same kernels, the
    norm's sum of squares in another order."""
    from gpu_util import build_tiny

    model, _, _ = build_tiny(dev, CFG, mode="gptq.int8", seed=10)
    with torch.no_grad():
        fast = _run(model, dev)
        assert model._decode is not None
        model._fast_ok = False
        slow = _run(model, dev)
        assert model._decode is None
    assert torch.equal(fast[0], slow[0])
    for a, b in zip(fast, slow):
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-3, atol=5e-3)


def test_batch2_runs_the_module_path_on_the_gemm(dev):
    from gpu_util import build_tiny

    model, _, _ = build_tiny(dev, CFG, mode="gptq.int8", seed=10)
    with torch.no_grad():
        two = _run(model, dev, B=2)
        assert model._decode is None and model._module_graph is not None
        one = _run(model, dev, B=1)
    # rows of a batch are independent; batch 2 decodes on the GEMM (fp32 sums of bf16 products), batch 1 on the exact
    # integer GEMV
    assert torch.equal(two[0][0:1], one[0])
    for a, b in zip(two, one):
        assert torch.equal(a[0:1], a[1:2])
        _close(a[0:1], b, 1e-2)


def test_compact_keeps_one_copy_and_changes_nothing(dev):
    from gpu_util import build_tiny

    model, _, sd = build_tiny(dev, CFG, mode="gptq.int8", seed=77)
    with torch.no_grad():
        before = _run(model, dev)
        before2 = _run(model, dev, B=2)
        before_sd = {k: v.clone() for k, v in model.state_dict().items()}
        model.reset_cache()
        torch.cuda.synchronize()
        model.compact()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        levels = sum(v.numel() for k, v in before_sd.items() if k.endswith("quant_weight"))
        after = _run(model, dev)
        after2 = _run(model, dev, B=2)
        live = torch.cuda.memory_allocated()
    for a, b in zip(before + before2, after + after2):
        assert torch.equal(a, b)
    # one level copy: the compacted tilings are the levels (N padded to 16); everything else is small for this model
    lin = model.transformer.h[0].attn.c_attn
    assert lin.quant_weight.numel() == 0 and model.transformer.h[1].mlp.c_fc1._tiled_i8 is None
    held = sum(m._tiled_i8.numel() for m in model.modules() if getattr(m, "_tiled_i8", None) is not None)
    held += sum(v[1][0].numel() for k, v in model._fc12_cache.items())
    assert held == levels
    kv = model._kv_store.numel() * 2
    assert live - base <= 0.05 * (levels + kv) + kv + (8 << 20), (live - base, levels, kv)
    got_sd = model.state_dict()
    assert got_sd.keys() == before_sd.keys()
    for k, v in before_sd.items():
        assert torch.equal(got_sd[k], v), k
        if k.endswith("quant_weight"):
            assert got_sd[k].stride() == v.stride(), k
    other, _, sd2 = build_tiny(dev, CFG, mode="gptq.int8", seed=78)
    with torch.no_grad():
        model.load_state_dict(sd2)
        for a, b in zip(_run(model, dev), _run(other, dev)):
            assert torch.equal(a, b)
    assert lin.quant_weight.numel() > 0


def test_mixed_bit_widths_do_not_compact(dev):
    from gpu_util import build_tiny
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    model, _, _ = build_tiny(dev, CFG, mode="gptq.int8", seed=3)
    four, _, _ = build_tiny(dev, CFG, mode="gptq.int4", seed=3)
    model.transformer.h[1].attn.c_proj = four.transformer.h[1].attn.c_proj
    assert isinstance(model.transformer.h[1].attn.c_proj, ColBlockQuantizedLinear)
    with pytest.raises(RuntimeError, match="one bit width"):
        model.compact()


def _random_w8_model(dev, name, n_layer=None, seed=0):
    """A gptq.int8 LLaMA at `name`'s widths with random levels, scales and zeros (per row, bf16)."""
    import lit_llama_b200 as P
    from lit_llama_b200.quantization import ColBlockQuantizedLinear, weights_changed
    from lit_llama_b200.utils import quantization

    cfg = P.LLaMAConfig.from_name(name)
    if n_layer is not None:
        cfg.n_layer = n_layer
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("gptq.int8"):
            model = P.LLaMA(cfg)
    finally:
        torch.set_default_dtype(prev)
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, ColBlockQuantizedLinear):
                m.quant_weight.copy_(torch.randint(0, 256, m.quant_weight.shape, generator=g, device=dev, dtype=torch.uint8))
                m.scales.copy_(torch.rand(m.scales.shape, generator=g, device=dev) * 2e-3 / (m.in_features ** 0.5) * 64 + 1e-4)
                m.zeros.copy_(torch.randint(96, 160, m.zeros.shape, generator=g, device=dev))
            elif isinstance(m, P.RMSNorm):
                m.scale.fill_(1)
        model.transformer.wte.weight.normal_(0, 1, generator=g)
    weights_changed()
    return model.eval()


def test_65b_widths_two_blocks_fused_equals_module_path(dev):
    model = _random_w8_model(dev, "65B", n_layer=2, seed=65)
    V = model.config.padded_vocab_size
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(0, V, (1, 12), generator=g)
    toks = torch.randint(0, V, (5,), generator=g).tolist()

    def run():
        model.reset_cache()
        out = [model(prompt.to(dev), 64, torch.arange(12, device=dev))]
        for i, t in enumerate(toks):
            out.append(model(torch.tensor([[t]], device=dev), 64, torch.tensor([12 + i], device=dev)).clone())
        return out

    with torch.no_grad():
        assert model._fast_decode_ok() == "w8"
        fast = run()
        model._fast_ok = False
        slow = run()
        model._fast_ok = None
        model.compact()
        compact = run()
    for a, b in zip(fast, slow):
        _close(a, b, 1e-2)
    for a, b in zip(fast, compact):
        assert torch.equal(a, b)
    del model
    torch.cuda.empty_cache()


def test_65b_fits_one_gpu(dev):
    """Full-size LLaMA-65B gptq.int8 (random levels), compacted: a 512-token prompt and graph-replayed batch-1 decode
    steps at max_seq_length 2048, with peak memory under 80 GB."""
    import lit_llama_b200 as P

    c = P.LLaMAConfig.from_name("65B")
    C_, H, V = c.n_embd, P.find_multiple(int(2 * 4 * c.n_embd / 3), 256), c.padded_vocab_size
    levels = c.n_layer * (4 * C_ * C_ + 3 * C_ * H) + V * C_
    kv = 2 * c.n_layer * 2 * c.n_head * 2048 * (C_ // c.n_head)
    need = levels + 2 * V * C_ + kv + (2 << 30)
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{free / 2**30:.1f} GiB free; LLaMA-65B gptq.int8 needs {need / 2**30:.1f} GiB")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    model = _random_w8_model(dev, "65B", seed=650)
    try:
        model.compact()
        g = torch.Generator().manual_seed(2)
        with torch.no_grad():
            out = [model(torch.randint(0, V, (1, 512), generator=g).to(dev), 2048, torch.arange(512, device=dev))]
            for i in range(6):
                out.append(model(torch.randint(0, V, (1, 1), generator=g).to(dev), 2048, torch.tensor([512 + i], device=dev)).clone())
        torch.cuda.synchronize()
        assert model._decode is not None and model._decode.graph is not None
        assert all(bool(torch.isfinite(o.float()).all()) for o in out)
        peak = torch.cuda.max_memory_allocated() - base
        assert peak < 80e9, peak / 2**30
        assert peak <= need, (peak / 2**30, need / 2**30)
    finally:
        del model
        torch.cuda.empty_cache()

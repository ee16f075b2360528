"""-m gpu: gptq.int4 at 2..16 activation rows on b2l_q4_gemv_batch_i8 (the resident b2l_q4_tile_i8 tiling, exact
integer contraction) -- every row bit-identical to b2l_q4_gemv on that row alone -- and the whole-token step at
B = 2..16 (B2L_F_Q4_BATCH_I8, `LLaMA.q4_batch_step`)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _tile(qw, N, K):
    from lit_llama_b200.quantization import tile_i8

    return tile_i8(qw, N, K, 4)


def _args(x, qt, sc, z, N, K, y, *, prologue, norm_scale, epilogue, res, grid, flags, ws=None):
    L = _L()
    return L.Q4LinearArgs(x=x.data_ptr(), ldx=x.stride(0), qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                          sz_dtype=L.sz_dtype_of(sc), y=y.data_ptr(), ldy=y.stride(0), M=x.shape[0], N=N, K=K,
                          prologue=prologue, norm_scale=None if norm_scale is None else norm_scale.data_ptr(), eps=1e-5,
                          epilogue=epilogue, res=None if res is None else res.data_ptr(),
                          ldres=0 if res is None else res.stride(0), split_k=grid, flags=flags,
                          workspace=None if ws is None else ws.data_ptr())


def _one(x, qt, sc, z, N, K, *, prologue=0, norm_scale=None, epilogue=0, res=None, grid=0, flags=0):
    """b2l_q4_gemv on each row of x separately."""
    L = _L()
    n_out = N // 2 if epilogue == L.EPI_SWIGLU else N
    rows = []
    for n in range(x.shape[0]):
        y = torch.zeros((1, n_out), device=x.device, dtype=torch.bfloat16)
        a = _args(x[n:n + 1], qt, sc, z, N, K, y, prologue=prologue, norm_scale=norm_scale, epilogue=epilogue,
                  res=None if res is None else res[n:n + 1], grid=grid, flags=flags)
        L.check(L.lib().b2l_q4_gemv(C.byref(a), L.stream_ptr()), "b2l_q4_gemv")
        rows.append(y)
    return torch.cat(rows)


def _batch(x, qt, sc, z, N, K, *, prologue=0, norm_scale=None, epilogue=0, res=None, grid=0, flags=0):
    L = _L()
    M = x.shape[0]
    n_out = N // 2 if epilogue == L.EPI_SWIGLU else N
    y = torch.full((M, n_out), float("nan"), device=x.device, dtype=torch.bfloat16)
    ws = torch.full((L.lib().b2l_w8_gemv_batch_workspace_bytes(K, M),), 0xA5, dtype=torch.uint8, device=x.device)
    a = _args(x, qt, sc, z, N, K, y, prologue=prologue, norm_scale=norm_scale, epilogue=epilogue, res=res, grid=grid,
              flags=flags, ws=ws)
    L.check(L.lib().b2l_q4_gemv_batch_i8(C.byref(a), L.stream_ptr()), "b2l_q4_gemv_batch_i8")
    return y


def _rows(M, K, seed):
    """M activation rows of very different magnitudes: row 0 scaled by 1e-3, row 1 one large outlier, row 2 all zero."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g) * 2
    x[0] *= 1e-3
    x[1, K // 3] = 300.0
    if M > 2:
        x[2] = 0
    return x.bfloat16()


SHAPES = [(48, 256), (130, 192), (12288, 4096), (4096, 4096), (15360, 5120), (5120, 13824), (8192, 22016), (32000, 4096)]


@pytest.mark.parametrize("M", [2, 3, 5, 8, 9, 13, 16])
@pytest.mark.parametrize("N,K", SHAPES)
def test_rows_bit_identical_to_batch1_and_exact(dev, M, N, K):
    from gpu_util import assert_q4_linear_close, rand_q4

    if N * K >= 5120 * 13824 and M not in (2, 9, 16):
        pytest.skip("covered by the other batch sizes")
    lv, qw, sc, z = rand_q4(N, K, dev, seed=N + K + M)
    qt = _tile(qw, N, K)
    x = _rows(M, K, M * K).to(dev)
    y = _batch(x, qt, sc, z, N, K)
    assert torch.equal(y, _one(x, qt, sc, z, N, K))
    assert_q4_linear_close(y, x, lv, sc, z, min_equal=0.995)
    # a larger leading dimension for x: the same rows
    xw = torch.zeros(M, K + 64, device=dev, dtype=torch.bfloat16)
    xw[:, :K] = x
    assert torch.equal(_batch(xw[:, :K], qt, sc, z, N, K), y)


@pytest.mark.parametrize("M", [2, 5, 9, 16])
def test_f32_scales(dev, M):
    from gpu_util import assert_q4_linear_close, rand_q4

    N, K = 256, 1024
    lv, qw, sc, z = rand_q4(N, K, dev, seed=5 + M, sz_dtype=torch.float32)
    qt = _tile(qw, N, K)
    x = _rows(M, K, 5).to(dev)
    y = _batch(x, qt, sc, z, N, K)
    assert torch.equal(y, _one(x, qt, sc, z, N, K))
    assert_q4_linear_close(y, x, lv, sc, z, min_equal=0.995)


@pytest.mark.parametrize("M", [2, 3, 8, 13, 16])
@pytest.mark.parametrize("N,K", [(1024, 2048), (4096, 11008)])
def test_prologue_epilogues_pdl_and_grids_bit_identical(dev, M, N, K):
    from gpu_util import rand_q4

    L = _L()
    g = torch.Generator().manual_seed(M + N)
    lv, qw, sc, z = rand_q4(N, K, dev, seed=11 + M)
    qt = _tile(qw, N, K)
    x = _rows(M, K, 3 * M).to(dev)
    ns = (1 + 0.1 * torch.randn(K, generator=g)).bfloat16().to(dev)
    xr = _rows(M, N, 7 * M).to(dev)    # residual rows (and the input of the N x N residual linear)
    lv2, qw2, sc2, z2 = rand_q4(N, N, dev, seed=12 + M)
    qt2 = _tile(qw2, N, N)
    res = torch.randn(M, N, generator=g).bfloat16().to(dev)
    cases = [
        dict(x=x, qt=qt, sc=sc, z=z, N=N, K=K),
        dict(x=x, qt=qt, sc=sc, z=z, N=N, K=K, prologue=L.PRO_RMSNORM, norm_scale=ns),
        dict(x=xr, qt=qt2, sc=sc2, z=z2, N=N, K=N, epilogue=L.EPI_RESIDUAL, res=res),
        dict(x=x, qt=qt, sc=sc, z=z, N=N, K=K, prologue=L.PRO_RMSNORM, norm_scale=ns, epilogue=L.EPI_SWIGLU),
        dict(x=x, qt=qt, sc=sc, z=z, N=N, K=K, prologue=L.PRO_RMSNORM, norm_scale=ns, epilogue=L.EPI_RESIDUAL,
             res=torch.randn(M, N, generator=g).bfloat16().to(dev)),
    ]
    for c in cases:
        c = dict(c)
        xx, qq, ss, zz, n, k = (c.pop(a) for a in ("x", "qt", "sc", "z", "N", "K"))
        want = _one(xx, qq, ss, zz, n, k, **c)
        for grid, flags in [(0, 0), (0, 1), (1, 1), (3, 0), (7, 1)]:
            got = _batch(xx, qq, ss, zz, n, k, grid=grid, flags=flags, **c)
            assert torch.equal(got, want), (c.get("prologue"), c.get("epilogue"), grid, flags)


@pytest.mark.parametrize("M", [2, 9, 16])
@pytest.mark.parametrize("N,K", [(256, 1024), (1024, 22016)])
def test_extreme_levels_full_range_rows(dev, M, N, K):
    """Rows of all-15 and all-0 levels in every combination of a packed byte's two rows (bytes 0xff, 0x0f, 0xf0, 0x00)
    against activations at the full digit range: the row-pair recovery at its extremes."""
    from gpu_util import assert_q4_linear_close

    lv = torch.zeros(N, K, dtype=torch.uint8)
    r = torch.arange(N)
    blk = (r // 16) % 4                       # which of the four byte patterns this 16-row block carries
    lo, hi = (r % 16) < 8, (r % 16) >= 8
    lv[(lo & ((blk == 0) | (blk == 1))) | (hi & ((blk == 0) | (blk == 2)))] = 15
    qw = (lv[:, 0::2] | (lv[:, 1::2] << 4)).t().contiguous().t().to(dev)
    sc = torch.full((N, 1), 0.0078125, dtype=torch.bfloat16, device=dev)
    z = torch.tensor([0.0, 15.0, 8.0], dtype=torch.bfloat16).repeat(N // 3 + 1)[:N].view(N, 1).to(dev)
    g = torch.Generator().manual_seed(N + M)
    x = (torch.rand(M, K, generator=g) * 2 - 1) * 448.0   # every digit value, |X| up to the top of the range (2^22)
    x[:, 0] = 448.0
    x[1] = 448.0                                        # rows at the largest sums of either sign
    x[-1] = -448.0
    x = x.bfloat16().to(dev)
    qt = _tile(qw, N, K)
    y = _batch(x, qt, sc, z, N, K)
    assert torch.equal(y, _one(x, qt, sc, z, N, K))
    assert_q4_linear_close(y, x, lv.to(dev), sc, z, min_equal=0.995)


def test_swiglu_matches_the_module_ops(dev):
    """SwiGLU on the 8 / 8 interleave of c_fc1 | c_fc2 (the resident "i8" copy) == silu(fc1(x)) * fc2(x) per row."""
    from gpu_util import rand_q4

    L = _L()
    N, K, M = 1024, 2048, 4
    lv, qw, sc, z = rand_q4(N, K, dev, seed=21)
    nh = N // 2
    inter = lambda t: torch.stack((t[:nh].reshape(nh // 8, 8, *t.shape[1:]), t[nh:].reshape(nh // 8, 8, *t.shape[1:])), 1).reshape(N, *t.shape[1:])  # noqa: E731
    qwi = inter(qw).t().contiguous().t()
    x = _rows(M, K, 21).to(dev)
    got = _batch(x, _tile(qwi, N, K), inter(sc).contiguous(), inter(z).contiguous(), N, K, epilogue=L.EPI_SWIGLU)
    a = _batch(x, _tile(qw[:nh].t().contiguous().t(), nh, K), sc[:nh].contiguous(), z[:nh].contiguous(), nh, K)
    b = _batch(x, _tile(qw[nh:].t().contiguous().t(), nh, K), sc[nh:].contiguous(), z[nh:].contiguous(), nh, K)
    h = torch.empty_like(a)
    L.check(L.lib().b2l_silu_mul(a.data_ptr(), b.data_ptr(), h.data_ptr(), a.numel(), L.stream_ptr()), "silu_mul")
    assert torch.equal(got, h)


# ---------------------------------------------------------------- the whole-token step at B = 2..16
# Prompts are 17 tokens: prefill then runs every batch size, B = 1 included, on the same GEMM (b2l_q4_gemm, M > 16),
# whose rows do not depend on M, so the step's rows can be compared bit for bit with the B = 1 step.
T_PROMPT = 17


def _close(a, b, bar=1e-2):
    """Each row of the [B, vocab] logits a within `bar` (normwise) of the same row of b."""
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape
    for n in range(a.shape[0]):
        r = float((a[n] - b[n]).norm() / b[n].norm())
        assert r < bar, (n, r)


def _seqs(B, T, steps, V, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, V, (B, T), generator=g), torch.randint(0, V, (steps, B), generator=g)


def _run(model, dev, prompts, toks, S):
    model.reset_cache()
    T = prompts.shape[1]
    with torch.no_grad():
        out = [model(prompts.to(dev), S, torch.arange(T, device=dev))[:, -1].float().cpu()]
        for i in range(toks.shape[0]):
            out.append(model(toks[i].view(-1, 1).to(dev), S, torch.tensor([T + i], device=dev))[:, -1].float().cpu())
    torch.cuda.synchronize()
    return out


def _oracle(oracle, prompts, toks, S):
    T = prompts.shape[1]
    oracle.reset_cache()
    out = [oracle.forward(prompts.long(), S, torch.arange(T))[:, -1].float()]
    for i in range(toks.shape[0]):
        out.append(oracle.forward(toks[i].view(-1, 1).long(), S, torch.tensor([T + i]))[:, -1].float())
    return out


@pytest.mark.parametrize("B", [2, 4, 8, 16])
def test_tiny_model_step_vs_todays_step_batch1_and_oracle(dev, B):
    from gpu_util import build_tiny

    L = _L()
    model, oracle, _ = build_tiny(dev, CFG, mode="gptq.int4", seed=30 + B, exact_linears=True)
    model.q4_batch_step = True
    prompts, toks = _seqs(B, T_PROMPT, 6, CFG["vocab_size"], B)
    step = _run(model, dev, prompts, toks, 32)
    st = model._decode
    assert st is not None and st.B == B and st.graph is not None and st.args.flags & L.F_Q4_BATCH_I8
    assert L.lib().b2l_decode_step_launches(C.byref(st.args)) == 2 + CFG["n_layer"] * (4 * 2 + 3) + 2
    model.q4_batch_step = False
    today = _run(model, dev, prompts, toks, 32)
    assert model._decode is not None and not model._decode.args.flags & L.F_Q4_BATCH_I8
    for a, b in zip(step, today):
        _close(a, b)
    want = _oracle(oracle, prompts, toks, 32)
    for a, b in zip(step, want):
        _close(a, b)
    model.q4_batch_step = True
    for r in range(0, B, max(1, B // 4)):   # a few rows alone on the batch-1 step
        one = _run(model, dev, prompts[r:r + 1], toks[:, r:r + 1], 32)
        assert model._decode is not None and model._decode.B == 1
        for a, b in zip(step, one):
            assert torch.equal(a[r:r + 1], b)


def test_roll_branch_at_batch4(dev):
    from gpu_util import build_tiny

    model, oracle, _ = build_tiny(dev, CFG, mode="gptq.int4", seed=44, exact_linears=True)
    model.q4_batch_step = True
    prompts, toks = _seqs(4, 7, 6, CFG["vocab_size"], 44)
    step = _run(model, dev, prompts, toks, 8)   # S = 8: positions past max_seq_length roll the cache
    assert model._decode is not None and model._decode.B == 4 and model._decode.args.flags & _L().F_Q4_BATCH_I8
    model.q4_batch_step = False
    today = _run(model, dev, prompts, toks, 8)
    want = _oracle(oracle, prompts, toks, 8)
    for a, b, c in zip(step, today, want):
        _close(a, b)
        _close(a, c)


def test_flag_off_keeps_the_tiled_mma_state_at_batch2(dev):
    from gpu_util import build_tiny

    L = _L()
    model, _, _ = build_tiny(dev, CFG, mode="gptq.int4", seed=10)
    model.q4_batch_step = False
    prompts, toks = _seqs(2, 7, 4, CFG["vocab_size"], 10)
    _run(model, dev, prompts, toks, 16)
    st = model._decode
    assert st is not None and st.B == 2 and not st.args.flags & L.F_Q4_BATCH_I8
    c_attn = model.transformer.h[0].attn.c_attn
    assert st.layers[0].c_attn.qw_mma == c_attn.tiled_mma().data_ptr()
    model.q4_batch_step = True
    _run(model, dev, prompts, toks, 16)
    st = model._decode
    assert st.args.flags & L.F_Q4_BATCH_I8 and st.layers[0].c_attn.qw_mma == c_attn.tiled_i8().data_ptr()


@pytest.mark.parametrize("name", ["13B", "65B"])
def test_wide_two_block_models_batch8_bit_identical_to_batch1(dev, name):
    """Every row of the B = 8 step equals the B = 1 step on that row alone.  Today's batched step (b2l_q4_gemv_batch:
    activations rounded to fp16) is held to 2e-2 per row: at 65B widths it differs from the batch-1 step by up to
    1.1e-2 on these random-level logits (H100)."""
    import gpu_util  # noqa: F401  (puts tools/ on sys.path)
    from diag import _random_w8_model

    model = _random_w8_model(name, dev, seed=66, n_layer=2, bits=4)   # gptq.int4, gain about one per linear
    model.q4_batch_step = True
    V = model.config.padded_vocab_size
    prompts, toks = _seqs(8, T_PROMPT, 4, V, 66)
    try:
        step = _run(model, dev, prompts, toks, 64)
        assert model._decode is not None and model._decode.B == 8
        for r in range(8):
            one = _run(model, dev, prompts[r:r + 1], toks[:, r:r + 1], 64)
            assert model._decode.B == 1
            for a, b in zip(step, one):
                assert torch.equal(a[r:r + 1], b), r
        model.q4_batch_step = False
        today = _run(model, dev, prompts, toks, 64)
        for a, b in zip(step, today):
            _close(a, b, 2e-2)
    finally:
        del model
        torch.cuda.empty_cache()


def test_lora_over_gptq_int4_batch4_on_the_step(dev):
    import test_gpu_lora as TL

    model, _, _ = TL.build(dev, "gptq.int4")
    model.q4_batch_step = True
    prompts, toks = _seqs(4, 7, 5, TL.CFG["vocab_size"], 4)
    step = _run(model, dev, prompts, toks, 32)
    st = model._decode
    assert st is not None and st.args.loras and st.B == 4 and st.args.flags & _L().F_Q4_BATCH_I8
    n = TL.CFG["n_layer"]   # head_size 128: one attention launch; one LoRA launch per layer
    assert _L().lib().b2l_decode_step_launches(C.byref(st.args)) == 2 + n * (4 * 2 + 1) + 2 + n
    model.q4_batch_step = False
    today = _run(model, dev, prompts, toks, 32)
    assert model._decode is not None and model._decode.args.loras
    for a, b in zip(step, today):
        _close(a, b)


def test_adapter_v1_gptq_int4_batch4_on_the_step(dev):
    import test_gpu_adapter as TA

    model, _, _ = TA.build(dev, TA.CFG128, "gptq.int4")
    model.q4_batch_step = True
    prompts, toks = _seqs(4, 7, 5, TA.CFG128["vocab_size"], 5)
    step = _run(model, dev, prompts, toks, 32)
    st = model._decode
    assert st is not None and st.args.adapters and st.B == 4 and st.args.flags & _L().F_Q4_BATCH_I8
    model.q4_batch_step = False
    today = _run(model, dev, prompts, toks, 32)
    assert model._decode is not None and model._decode.args.adapters
    for a, b in zip(step, today):
        _close(a, b)


def test_compacted_batch8_bit_identical_and_reads_only_the_resident_copy(dev, monkeypatch):
    from gpu_util import build_tiny
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    cfg = dict(block_size=64, vocab_size=256, n_layer=2, n_head=4, n_embd=512)
    model, _, _ = build_tiny(dev, cfg, mode="gptq.int4", seed=88)
    model.q4_batch_step = True
    prompts, toks = _seqs(8, 7, 5, cfg["vocab_size"], 88)
    before = _run(model, dev, prompts, toks, 16)
    model.reset_cache()
    model.compact()
    T = prompts.shape[1]
    with torch.no_grad():
        after = [model(prompts.to(dev), 16, torch.arange(T, device=dev))[:, -1].float().cpu()]   # prefill: module path
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()

        def boom(*a, **k):
            raise AssertionError("the batched step must read only the resident tiling")

        monkeypatch.setattr(ColBlockQuantizedLinear, "reference_quant_weight", boom)
        for name in ("b2l_q4_untile_i8", "b2l_q4_tile_mma", "b2l_q4_tile"):
            monkeypatch.setattr(_L().lib(), name, boom)
        for i in range(toks.shape[0]):
            after.append(model(toks[i].view(-1, 1).to(dev), 16, torch.tensor([T + i], device=dev))[:, -1].float().cpu())
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    st = model._decode
    assert st is not None and st.B == 8 and st.graph is not None and st.args.flags & _L().F_Q4_BATCH_I8
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    state = sum(t.numel() * t.element_size() for t in (st.batch_ws, st.x, st.qkv, st.att, st.hid, st.logits, st.work,
                                                       st.idx, st.pos))
    assert peak <= state + (1 << 20), (peak, state)

"""-m gpu: different prompts decoded together (`generate_prompts`), and the per-row positions under it (B2L_F_ROW_POS).

Kernel level: a B-row launch with one position and one ring offset per row equals, bit for bit, B = 1 launches on each
row (output and appended K / V rows), on the fused head_size-128 kernel, its LLaMA-Adapter variant and the three-kernel
path; b2l_ring_advance_rows and b2l_kv_unroll_rows equal their torch restatements.  Model level: on the exact 2..16-row
steps (gptq.int4 `q4_batch_step`, gptq.int8 `w8_batch_step`) every row's logits equal the batch-1 model's on that row's
own sequence (teacher-forced after `reset_cache()`), in and past the roll branch; the other batched paths are held to
the bars of their existing B >= 2 tests; greedy rows match the reference's tokens (tests/golden/tiny_prompts_int4_bf16.pt,
oracle/make_golden_prompts.py)."""
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)       # the golden tiny model (head_size 32)
CFG128 = dict(block_size=64, vocab_size=256, n_layer=3, n_head=4, n_embd=512)   # head_size 128
LENGTHS = (3, 16, 40, 7)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _P():
    import lit_llama_b200 as P

    return P


def _L():
    from lit_llama_b200 import _lib as L

    return L


# --------------------------------------------------------------------------------------------- 1. kernels
def _rows_launch(qkv, kc, vc, pos, ring, nh, flags, prefix=None):
    import test_gpu_attention as TA

    return TA._launch(qkv, kc, vc, pos, ring, nh, flags=flags, prefix=prefix)


KERNEL_CASES = {
    # positions {5, 200, 300, 1030} of S = 2048: at 32 / 40 heads the 1030 row's keys split over several CTAs, the 5 row
    # stays in one
    "inside": ([5, 200, 300, 1030], [0, 0, 0, 0]),
    # rows past S (the roll branch) with a different ring offset per row, one wrapping inside a sub-tile
    "rolled": ([5, 2048, 300, 3000], [3, 777, 1500, 2047]),
}


@pytest.mark.parametrize("case", list(KERNEL_CASES))
@pytest.mark.parametrize("variant", ["fused", "adapter", "unfused", "hs32"])
@pytest.mark.parametrize("nh", [32, 40])
def test_row_positions_equal_batch1_launches(dev, nh, variant, case):
    import test_gpu_attention as TA

    L = _L()
    S, B = 2048, 4
    hs = 32 if variant == "hs32" else 128
    positions, rings = KERNEL_CASES[case]
    qkv, kl, vl = TA._flat(dev, B, nh, hs, S, seed=nh + hs)
    prefix = TA._prefix(dev, nh, 10, hs, seed=nh) if variant == "adapter" else None
    flags = TA.F_UNFUSED if variant == "unfused" else 0
    kp = torch.stack([TA._phys(kl[b:b + 1], rings[b])[0] for b in range(B)])
    vp = torch.stack([TA._phys(vl[b:b + 1], rings[b])[0] for b in range(B)])
    pos = torch.tensor(positions, dtype=torch.int64, device=dev)
    ring = torch.tensor(rings, dtype=torch.int32, device=dev)
    kb, vb = kp.clone(), vp.clone()
    y = _rows_launch(qkv.clone(), kb, vb, pos, ring, nh, flags | L.F_ROW_POS, prefix)
    for b in range(B):
        k1, v1 = kp[b:b + 1].clone(), vp[b:b + 1].clone()
        y1 = _rows_launch(qkv[b:b + 1].clone(), k1, v1, positions[b], rings[b], nh, flags, prefix)
        assert torch.equal(y[b], y1[0]), (b, positions[b], int((y[b] != y1[0]).sum()))
        assert torch.equal(kb[b], k1[0]) and torch.equal(vb[b], v1[0]), b
    assert not torch.isnan(y).any()


def test_ring_advance_and_kv_unroll_rows(dev):
    L = _L()
    lib = L.lib()
    S, B, nh, hs = 48, 5, 3, 32
    g = torch.Generator(device=dev).manual_seed(3)
    pos = torch.tensor([0, 47, 48, 100, 5], dtype=torch.int64, device=dev)
    ring = torch.tensor([0, 9, 47, 30, 12], dtype=torch.int32, device=dev)
    want = torch.where(pos >= S, (ring + 1) % S, ring)
    L.check(lib.b2l_ring_advance_rows(pos.data_ptr(), B, ring.data_ptr(), S, L.stream_ptr()), "b2l_ring_advance_rows")
    assert torch.equal(ring, want)
    cache = torch.randn(B, nh, S, hs, device=dev, generator=g).bfloat16()
    out = torch.full_like(cache, float("nan"))
    L.check(lib.b2l_kv_unroll_rows(cache.data_ptr(), ring.data_ptr(), out.data_ptr(), B, nh, S, hs, L.stream_ptr()),
            "b2l_kv_unroll_rows")
    for b in range(B):
        assert torch.equal(out[b], torch.roll(cache[b], -int(ring[b]), dims=1)), b


# --------------------------------------------------------------------------------------------- helpers
def _record(model):
    """Wraps model.prefill_rows and model.forward: the prefill's (B, V) logits and every per-row step's last-position
    logits are appended to the returned list."""
    logs = []
    fwd, pre = model.forward, model.prefill_rows

    def rec(idx, max_seq_length=None, input_pos=None):
        out = fwd(idx, max_seq_length, input_pos)
        if input_pos is not None and input_pos.dim() == 2:
            logs.append(out[:, -1].clone())
        return out

    def rec_pre(prompts, max_seq_length):
        out = pre(prompts, max_seq_length)
        logs.append(out.clone())
        return out

    model.forward, model.prefill_rows = rec, rec_pre
    return logs


def _unrecord(model):
    del model.forward
    del model.prefill_rows


def _prompts(dev, V, lengths=LENGTHS, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, V, (n,), generator=g).to(torch.int32).to(dev) for n in lengths]


def _sampled(model, prompts, steps, S, seed, temperature=1.0, top_k=None, eos_id=None):
    """generate_prompts with every step's (B, V) logits recorded, and the Exp(1) noise each step drew (regenerated from
    the same seed: the model calls draw nothing)."""
    P = _P()
    model.reset_cache()
    logs = _record(model)
    try:
        torch.manual_seed(seed)
        ys = P.generate_prompts(model, prompts, steps, max_seq_length=S, temperature=temperature, top_k=top_k, eos_id=eos_id)
        torch.cuda.synchronize()
    finally:
        _unrecord(model)
    B, V = len(prompts), logs[0].shape[-1]
    torch.manual_seed(seed)
    qs = [torch.empty((B, V), dtype=torch.bfloat16, device=prompts[0].device).exponential_(1) for _ in logs]
    return ys, logs, qs


def _check_draws(ys, logs, qs, prompts, temperature=1.0, top_k=None):
    """Every drawn token is argmax(probs / q) of its row (ties to the lower index), probs from the recorded logits."""
    P = _P()
    for i, (lg, q) in enumerate(zip(logs, qs)):
        want = torch.argmax(P.sample_probs(lg, temperature, top_k) / q, dim=-1)
        got = torch.stack([y[p.numel() + i] for y, p in zip(ys, prompts)]).to(torch.int64)
        assert torch.equal(got, want), i


def _teacher_forced(model, prompt, y, S):
    """The batch-1 model's last-position logits at every step of the sequence y (prompt + sampled tokens)."""
    T = prompt.numel()
    model.reset_cache()
    with torch.no_grad():
        out = [model(prompt.view(1, -1), S, torch.arange(T, device=prompt.device))[:, -1].clone()]
        for i in range(1, y.numel() - T):
            out.append(model(y[T + i - 1].view(1, 1), S, torch.tensor([T + i - 1], device=prompt.device))[:, -1].clone())
    torch.cuda.synchronize()
    assert model._kv_store.shape[2] == 1
    return out


def _rows_vs_batch1(model, prompts, ys, logs, S, bar=None, caches=None):
    """Each row's recorded logits against the batch-1 model on that row's own sequence: bit for bit (bar None), or each
    step within `bar` normwise.  `caches`: the B-row model's logical KV caches after the run, compared with the batch-1
    model's (bit for bit).  Returns whether every row was bit-identical, and the largest normwise distance."""
    same, worst = True, 0.0
    for b, (p, y) in enumerate(zip(prompts, ys)):
        one = _teacher_forced(model, p, y, S)
        assert len(one) == len(logs)
        for i, (lg, o) in enumerate(zip(logs, one)):
            eq = torch.equal(lg[b], o[0])
            same = same and eq
            r = float((lg[b].float() - o[0].float()).norm() / o[0].float().norm())
            worst = max(worst, r)
            if bar is None:
                assert eq, (b, i, r)
            else:
                assert r < bar, (b, i, r)
        if caches is not None:
            for (k, v), (k1, v1) in zip(caches, model.logical_kv_caches()):
                assert torch.equal(k[b], k1[0]) and torch.equal(v[b], v1[0]), b
    return same, worst


def _exact_model(dev, kind):
    import gpu_util  # noqa: F401  (puts tools/ on sys.path)
    from diag import _random_w8_model
    from gpu_util import build_tiny

    if kind == "hs128-q4":
        model, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=21)
    elif kind == "hs128-w8":
        model, _, _ = build_tiny(dev, CFG128, mode="gptq.int8", seed=22)
    else:   # 13B widths, two blocks, gain about one per linear
        model = _random_w8_model("13B", dev, seed=66, n_layer=2, bits=4 if kind == "13B-q4" else 8)
    if "q4" in kind:
        model.q4_batch_step = True
    else:
        model.w8_batch_step = True
    return model


# --------------------------------------------------------------------------------------------- 2. / 3. exact steps
@pytest.mark.parametrize("kind", ["hs128-q4", "hs128-w8", "13B-q4", "13B-w8"])
def test_rows_bit_identical_to_batch1(dev, kind):
    L = _L()
    model = _exact_model(dev, kind)
    try:
        prompts = _prompts(dev, model.config.vocab_size, seed=4)
        S = max(LENGTHS) + 10
        ys, logs, qs = _sampled(model, prompts, 10, S=S, seed=40)
        st = model._decode
        flag = L.F_Q4_BATCH_I8 if "q4" in kind else L.F_W8_BATCH
        assert st is not None and st.B == 4 and st.args.flags & flag and st.args.flags & L.F_ROW_POS
        assert st.row_pos and st.graph is not None and model._ring.numel() == 4
        assert [y.numel() for y in ys] == [n + 10 for n in LENGTHS]
        assert all(torch.equal(y[:p.numel()], p) for y, p in zip(ys, prompts))
        _check_draws(ys, logs, qs, prompts)
        _rows_vs_batch1(model, prompts, ys, logs, S)
    finally:
        del model
        torch.cuda.empty_cache()


@pytest.mark.parametrize("kind", ["hs128-q4", "hs128-w8"])
def test_roll_per_row_bit_identical_to_batch1(dev, kind):
    """S = 44 with prompts of 3, 38, 40 and 7 tokens and 12 new tokens: the 40- and 38-token rows roll their rings (at
    different steps), the others never do.  Logits and the logical KV caches equal batch 1 on each row."""
    L = _L()
    model = _exact_model(dev, kind)
    lengths, S = (3, 38, 40, 7), 44
    prompts = _prompts(dev, CFG128["vocab_size"], lengths, seed=5)
    ys, logs, qs = _sampled(model, prompts, 12, S=S, seed=50, temperature=1.3)
    assert model._decode.B == 4 and model._decode.args.flags & L.F_ROW_POS
    rings = model._ring.tolist()
    assert rings == [0, 38 + 10 - S + 1, 40 + 10 - S + 1, 0], rings   # the last step ran at position T + 10
    caches = [(k.clone(), v.clone()) for k, v in model.logical_kv_caches()]
    _check_draws(ys, logs, qs, prompts, temperature=1.3)
    _rows_vs_batch1(model, prompts, ys, logs, S, caches=caches)


# --------------------------------------------------------------------------------------------- 4. golden
@pytest.mark.parametrize("path", ["module", "step"])
def test_greedy_rows_match_reference_and_generate(dev, path):
    from gpu_util import build_tiny

    P, L = _P(), _L()
    gd = load_golden("tiny_prompts_int4_bf16.pt")
    model, _, _ = build_tiny(dev, CFG)
    if path == "module":
        model._fast_ok = False   # module by module (head_size 32: the three-kernel attention)
    else:
        model.q4_batch_step = True
    prompts = [p.to(torch.int32).to(dev) for p in gd["prompts"]]
    n = gd["max_new_tokens"]
    rows = P.generate_prompts(model, prompts, n, top_k=1)
    if path == "module":
        assert model._decode is None and model._module_graph is not None and model._module_graph["key"][-1]
    else:
        st = model._decode
        assert st is not None and st.B == 4 and st.args.flags & L.F_Q4_BATCH_I8 and st.args.flags & L.F_ROW_POS
    for y, p, want in zip(rows, prompts, gd["gen_greedy"]):
        model.reset_cache()
        one = P.generate(model, p, n, top_k=1)
        assert torch.equal(y, one), (y.tolist(), one.tolist())
        # as test_gpu_model.py::test_generate_matches_reference_tokens requires of generate()
        assert y.shape == want.shape and (y.cpu() == want).float().mean() >= 0.9, (y.tolist(), want.tolist())


# --------------------------------------------------------------------------------------------- 5. other routes
@pytest.mark.parametrize("kind", ["adapter", "lora", "llm.int8", "adapter_v2", "q4-default"])
def test_other_routes_within_their_bars(dev, kind):
    """LLaMA-Adapter v1 and LoRA over gptq.int4 on `q4_batch_step` (1e-2 per row, as their B = 4 step tests), llm.int8
    on its 2..16-row step (rows interact through the batch outlier mask: 6e-2), v2 on the module path and gptq.int4 on
    its default batched kernels (2e-2); whether the rows came out bit-identical to batch 1 is printed."""
    from gpu_util import build_tiny

    L = _L()
    if kind == "adapter":
        import test_gpu_adapter as TA

        model, _, _ = TA.build(dev, TA.CFG128, "gptq.int4")
        model.q4_batch_step = True
        bar = 1e-2
    elif kind == "lora":
        import test_gpu_lora as TL

        model, _, _ = TL.build(dev, "gptq.int4")
        model.q4_batch_step = True
        bar = 1e-2
    elif kind == "adapter_v2":
        import test_gpu_adapter_v2 as TV

        model, _, _ = TV.build(dev, TV.CFG128, "gptq.int4")
        bar = 2e-2
    elif kind == "llm.int8":
        model, _, _ = build_tiny(dev, CFG128, mode="llm.int8", seed=31)
        model.int8_step = True
        bar = 6e-2
    else:
        model, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=32)
        bar = 2e-2
    lengths = (3, 16, 20, 7)
    prompts = _prompts(dev, 256, lengths, seed=8)
    ys, logs, qs = _sampled(model, prompts, 8, S=32, seed=70)
    st = model._decode
    if kind == "adapter_v2":
        assert st is None and model._module_graph is not None and model._module_graph["key"][-1]
    else:
        assert st is not None and st.B == 4 and st.args.flags & L.F_ROW_POS
        want = {"adapter": L.F_Q4_BATCH_I8, "lora": L.F_Q4_BATCH_I8, "llm.int8": L.F_Q8_BATCH}.get(kind)
        assert (st.args.flags & want) if want else not st.args.flags & L.F_Q4_BATCH_I8
    if kind == "adapter":   # the prefix store does not depend on B; its views follow the cache
        caches = [c for c in model.adapter_kv_caches if c is not None]
        assert caches and all(k.shape[0] == 4 and v.shape[0] == 4 for k, v in caches)
    _check_draws(ys, logs, qs, prompts)
    same, worst = _rows_vs_batch1(model, prompts, ys, logs, 32, bar=bar)
    print(f"{kind}, 4 prompts: rows bit-identical to batch 1: {same} (max normwise {worst:.3g})")


# --------------------------------------------------------------------------------------------- 6. rows and state
def test_eos_per_row(dev):
    """A row that draws eos ends there, eos included; the tokens before it are the eos-free run's (eos changes no draw),
    and rows without it run to the end."""
    from gpu_util import build_tiny

    P = _P()
    model, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=9)
    model.q4_batch_step = True
    prompts = _prompts(dev, 256, seed=7)
    steps = 12
    torch.manual_seed(5)
    free = P.generate_prompts(model, prompts, steps, temperature=1.5, top_k=3)
    new = [y[p.numel():].cpu() for y, p in zip(free, prompts)]
    eos = int(new[0][2])
    model.reset_cache()
    torch.manual_seed(5)
    out = P.generate_prompts(model, prompts, steps, temperature=1.5, top_k=3, eos_id=eos)
    for y, y_free, nw, p in zip(out, free, new, prompts):
        hits = (nw == eos).nonzero()
        n = int(hits[0]) + 1 if hits.numel() else steps
        assert torch.equal(y, y_free[:p.numel() + n]), (y.tolist(), y_free.tolist())
    assert out[0].numel() <= prompts[0].numel() + 3 and int(out[0][-1]) == eos


def test_one_prompt_equals_generate_and_reset(dev):
    """generate_prompts with one prompt is generate() for the same seed; after a 4-row run, reset_cache() gives batch-1
    generate() its old tokens back, with one shared ring offset."""
    from gpu_util import build_tiny

    P = _P()
    model, _, _ = build_tiny(dev, CFG, seed=11)
    model.q4_batch_step = True
    prompts = _prompts(dev, CFG["vocab_size"], (3, 16, 12, 7), seed=9)
    for S in (None, 20):   # 20: the 16-token prompt rolls
        model.reset_cache()
        torch.manual_seed(11)
        want = P.generate(model, prompts[1], 12, max_seq_length=S, temperature=0.8, top_k=20)
        model.reset_cache()
        torch.manual_seed(11)
        got = P.generate_prompts(model, [prompts[1]], 12, max_seq_length=S, temperature=0.8, top_k=20)
        assert len(got) == 1 and got[0].dtype == want.dtype and torch.equal(got[0], want), (got[0].tolist(), want.tolist())
        P.generate_prompts(model, prompts, 12, max_seq_length=S, temperature=0.8, top_k=20)
        assert model._ring.numel() == 4
        model.reset_cache()
        assert model._ring.numel() == 1 and model._decode is None and model.kv_caches == []
        torch.manual_seed(11)
        again = P.generate(model, prompts[1], 12, max_seq_length=S, temperature=0.8, top_k=20)
        assert torch.equal(again, want)

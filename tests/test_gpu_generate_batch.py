"""-m gpu: parallel samples of one prompt (`generate_batch`) on the batched decode step, and the row sampling launch
under it (b2l_topk_softmax_rows / b2l_topk_softmax_sample_rows).

The draw of every row is torch.multinomial's on the step's [B, V] probabilities for the same generator state.  On the
exact 2..16-row steps (gptq.int4 `q4_batch_step`, gptq.int8 `w8_batch_step`) every row's logits equal, bit for bit, the
batch-1 model's on that row's tokens (teacher-forced after `reset_cache()`); the other batched paths are held to the
bars of their existing B >= 2 tests."""
import importlib

import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)       # the golden tiny model (head_size 32)
CFG128 = dict(block_size=64, vocab_size=256, n_layer=3, n_head=4, n_embd=512)   # head_size 128


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


# --------------------------------------------------------------------------------------------- 1. row sampling
@pytest.mark.parametrize("V", [32000, 32001, 128])
@pytest.mark.parametrize("ld", ["V", "V+8", "V+3", "0"])
def test_rows_draw_equals_torch_multinomial(dev, V, ld):
    """Row b's token is torch.multinomial(probs, 1)[b] on the [B, V] probabilities for the same generator state, the
    generator ends in the same state, and probs equal the single-row kernel's on each row bit for bit.  Rows ld apart
    (ld = V + 3, and V = 32001: rows that do not start on 16 bytes) or all reading one row (ld = 0)."""
    P, L = _P(), _L()
    G = importlib.import_module("lit_llama_b200.generate")
    g = torch.Generator(device=dev).manual_seed(V * 7 + len(ld))
    extra = {"V": 0, "V+8": 8, "V+3": 3, "0": 0}[ld]
    seed = 0
    for B in (1, 2, 5, 16):
        for top_k in (None, 1, 50, 200, V):
            for temp in (0.7, 1.0, 1.7):
                seed += 1
                base = (torch.randn(B, V + extra, device=dev, generator=g) * (1 + seed % 4)).bfloat16()
                base[:, 5] = base[:, 9]   # a tie
                rows = base[:, :V] if ld != "0" else base[0, :V].expand(B, V)
                if ld == "V":
                    rows = rows.contiguous()
                want_ld = {"V": V, "V+8": V + 8, "V+3": V + 3, "0": 0}[ld] if B > 1 else V
                x, got_ld = G._rows(rows)
                assert got_ld == want_ld and x.data_ptr() == rows.data_ptr()   # read in place
                probs = P.sample_probs(rows, temp, top_k)
                assert probs.shape == (B, V)
                for b in range(B):
                    assert torch.equal(probs[b], P.sample_probs(rows[b], temp, top_k)), (B, top_k, temp, b)
                torch.manual_seed(seed)
                want = torch.multinomial(probs, num_samples=1).view(B)
                state = torch.cuda.get_rng_state()
                torch.manual_seed(seed)
                got = P.sample_token(rows, temp, top_k)
                assert torch.equal(torch.cuda.get_rng_state(), state)   # multinomial's RNG consumption
                assert got.shape == (B,) and got.dtype == torch.int64
                assert torch.equal(got, want), (B, top_k, temp, got.tolist(), want.tolist())
                # the sampling entry point with probs written too
                torch.manual_seed(seed)
                q = torch.empty((B, V), dtype=torch.bfloat16, device=dev).exponential_(1)
                pr = torch.full((B, V), 7.0, dtype=torch.bfloat16, device=dev)
                tok = torch.full((B,), -1, dtype=torch.int64, device=dev)
                k = 0 if top_k is None else min(top_k, V)
                L.check(L.lib().b2l_topk_softmax_sample_rows(x.data_ptr(), got_ld, temp, k, q.data_ptr(), pr.data_ptr(),
                                                             tok.data_ptr(), B, V, L.stream_ptr()), "sample_rows")
                assert torch.equal(pr, probs) and torch.equal(tok, want)


# --------------------------------------------------------------------------------------------- helpers
def _record(model):
    """Wraps model.forward: every call's last-position logits are appended to the returned list."""
    logs = []
    fwd = model.forward

    def rec(*a, **k):
        out = fwd(*a, **k)
        logs.append(out[:, -1].clone())
        return out

    model.forward = rec
    return logs


def _unrecord(model):
    del model.forward


def _sampled(model, prompt, n, steps, S, seed, temperature=1.0, top_k=None, eos_id=None):
    """generate_batch with every step's batched logits recorded, and the Exp(1) noise each step drew (regenerated from
    the same seed: the model calls draw nothing)."""
    P = _P()
    model.reset_cache()
    logs = _record(model)
    try:
        torch.manual_seed(seed)
        ys = P.generate_batch(model, prompt, n, steps, max_seq_length=S, temperature=temperature, top_k=top_k, eos_id=eos_id)
        torch.cuda.synchronize()
    finally:
        _unrecord(model)
    V = logs[0].shape[-1]
    torch.manual_seed(seed)
    qs = [torch.empty((n, V), dtype=torch.bfloat16, device=prompt.device).exponential_(1) for _ in logs]
    return ys, logs, qs


def _check_draws(ys, logs, qs, T, temperature=1.0, top_k=None):
    """Every drawn token is argmax(probs / q) of its row (ties to the lower index), probs from the recorded logits."""
    P = _P()
    n = len(ys)
    for i, (lg, q) in enumerate(zip(logs, qs)):
        rows = lg.expand(n, -1) if i == 0 else lg
        assert rows.shape[0] == n
        want = torch.argmax(P.sample_probs(rows, temperature, top_k) / q, dim=-1)
        got = torch.stack([y[T + i] for y in ys]).to(torch.int64)
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


def _rows_vs_batch1(model, prompt, ys, logs, S, bar=None):
    """Each row's recorded logits against the batch-1 model on that row: bit for bit (bar None), or each step within
    `bar` normwise.  Returns whether every row was bit-identical, and the largest normwise distance."""
    same, worst = True, 0.0
    for b, y in enumerate(ys):
        one = _teacher_forced(model, prompt, y, S)
        assert len(one) == len(logs)
        for i, (lg, o) in enumerate(zip(logs, one)):
            a = lg[0] if i == 0 else lg[b]
            eq = torch.equal(a, o[0])
            same = same and eq
            r = float((a.float() - o[0].float()).norm() / o[0].float().norm())
            worst = max(worst, r)
            if bar is None:
                assert eq, (b, i, r)
            else:
                assert r < bar, (b, i, r)
    return same, worst


def _prompt(dev, V, T=16, seed=3):
    return torch.randint(0, V, (T,), generator=torch.Generator().manual_seed(seed)).to(torch.int32).to(dev)


# --------------------------------------------------------------------------------------------- 2. / 3. tiny golden model
def test_one_sample_equals_generate(dev):
    from gpu_util import build_tiny

    P = _P()
    gd = load_golden("tiny_int4_bf16.pt")
    model, _, _ = build_tiny(dev, CFG)
    prompt = gd["prompt"].to(torch.int32).to(dev)
    for S in (None, 10):   # S = 10: the roll branch
        model.reset_cache()
        torch.manual_seed(11)
        want = P.generate(model, prompt, 20, max_seq_length=S, temperature=0.8, top_k=200)
        model.reset_cache()
        torch.manual_seed(11)
        got = P.generate_batch(model, prompt, 1, 20, max_seq_length=S, temperature=0.8, top_k=200)
        assert isinstance(got, list) and len(got) == 1
        assert got[0].dtype == want.dtype and torch.equal(got[0], want), (got[0].tolist(), want.tolist())
    # torch.multinomial replaced (the reference's tests/test_generate.py patches it): called on the [B, V] probabilities,
    # and it draws what the fused launch draws for the same seed
    from unittest import mock

    model.reset_cache()
    torch.manual_seed(12)
    fused = P.generate_batch(model, prompt, 4, 20, max_seq_length=10, temperature=0.8, top_k=4)
    draws = []
    orig = torch.multinomial

    def spy(*a, **k):
        out = orig(*a, **k)
        draws.append(out)
        return out

    model.reset_cache()
    torch.manual_seed(12)
    with mock.patch("torch.multinomial", spy):
        out = P.generate_batch(model, prompt, 4, 20, max_seq_length=10, temperature=0.8, top_k=4)
    assert len(draws) == 20 and all(d.shape == (4, 1) for d in draws)
    for b in range(4):
        assert out[b].numel() == 7 + 20
        assert torch.equal(out[b], torch.cat((prompt, torch.cat([d[b] for d in draws]).to(torch.int32))))
        assert torch.equal(out[b], fused[b])


def test_greedy_rows_equal_generate_and_golden(dev):
    from gpu_util import build_tiny

    P, L = _P(), _L()
    gd = load_golden("tiny_int4_bf16.pt")
    model, _, _ = build_tiny(dev, CFG)
    model.q4_batch_step = True
    prompt = gd["prompt"].to(torch.int32).to(dev)
    want = P.generate(model, prompt, 12, top_k=1)
    model.reset_cache()
    rows = P.generate_batch(model, prompt, 8, 12, top_k=1)
    st = model._decode
    assert st is not None and st.B == 8 and st.args.flags & L.F_Q4_BATCH_I8
    model.reset_cache()
    for y in rows:
        assert torch.equal(y, want)
        # as test_gpu_model.py::test_generate_matches_reference_tokens requires of generate()
        assert (y.cpu() == gd["gen_greedy"]).float().mean() >= 0.9


# --------------------------------------------------------------------------------------------- 4. / 5. exactness
def _exact_model(dev, kind):
    import gpu_util  # noqa: F401  (puts tools/ on sys.path)
    from diag import _random_w8_model
    from gpu_util import build_tiny

    if kind == "hs128-q4":
        model, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=21)
    elif kind == "hs128-w8":
        model, _, _ = build_tiny(dev, CFG128, mode="gptq.int8", seed=22)
    else:   # 13B widths, two blocks, gain about one per linear (as test_wide_two_block_models_batch8_bit_identical_to_batch1)
        model = _random_w8_model("13B", dev, seed=66, n_layer=2, bits=4 if kind == "13B-q4" else 8)
    if "q4" in kind:
        model.q4_batch_step = True
    else:
        model.w8_batch_step = True
    return model


@pytest.mark.parametrize("kind", ["hs128-q4", "hs128-w8", "13B-q4", "13B-w8"])
def test_rows_bit_identical_to_batch1_on_the_digit_kernels(dev, kind):
    L = _L()
    model = _exact_model(dev, kind)
    try:
        V = model.config.vocab_size
        prompt = _prompt(dev, V, T=16, seed=4)
        ys, logs, qs = _sampled(model, prompt, 4, 10, S=32, seed=40)
        st = model._decode
        flag = L.F_Q4_BATCH_I8 if "q4" in kind else L.F_W8_BATCH
        assert st is not None and st.B == 4 and st.args.flags & flag and st.graph is not None
        assert len(ys) == 4 and all(y.numel() == 16 + 10 for y in ys)
        assert len({tuple(y.tolist()) for y in ys}) > 1   # the samples differ
        _check_draws(ys, logs, qs, 16)
        _rows_vs_batch1(model, prompt, ys, logs, 32)
    finally:
        del model
        torch.cuda.empty_cache()


def test_roll_branch_at_batch4_bit_identical_to_batch1(dev):
    L = _L()
    model = _exact_model(dev, "hs128-q4")
    prompt = _prompt(dev, CFG128["vocab_size"], T=7, seed=5)
    ys, logs, qs = _sampled(model, prompt, 4, 12, S=8, seed=50, temperature=1.3)   # positions 8..17 roll the cache
    assert model._decode.B == 4 and model._decode.args.flags & L.F_Q4_BATCH_I8
    assert all(y.numel() == 7 + 12 for y in ys)
    _check_draws(ys, logs, qs, 7, temperature=1.3)
    _rows_vs_batch1(model, prompt, ys, logs, 8)


@pytest.mark.parametrize("kind", ["adapter", "lora"])
def test_adapter_v1_and_lora_rows_on_the_q4_batched_step(dev, kind):
    """Held to the bar of their existing B = 4 step tests (_close, 1e-2 per row); whether the rows came out bit-identical
    to batch 1 is printed."""
    L = _L()
    if kind == "adapter":
        import test_gpu_adapter as TA

        model, _, _ = TA.build(dev, TA.CFG128, "gptq.int4")
    else:
        import test_gpu_lora as TL

        model, _, _ = TL.build(dev, "gptq.int4")
    model.q4_batch_step = True
    prompt = _prompt(dev, 256, T=7, seed=6)
    ys, logs, qs = _sampled(model, prompt, 4, 8, S=32, seed=60)
    st = model._decode
    assert st is not None and st.B == 4 and st.args.flags & L.F_Q4_BATCH_I8
    assert (st.args.adapters if kind == "adapter" else st.args.loras)
    if kind == "adapter":   # the prefix store does not depend on B; its views follow the cache
        caches = [c for c in model.adapter_kv_caches if c is not None]
        assert caches and all(k.shape[0] == 4 and v.shape[0] == 4 for k, v in caches)
    _check_draws(ys, logs, qs, 7)
    same, worst = _rows_vs_batch1(model, prompt, ys, logs, 32, bar=1e-2)
    print(f"{kind} over gptq.int4, q4_batch_step, B = 4: rows bit-identical to batch 1: {same} (max normwise {worst:.3g})")


# --------------------------------------------------------------------------------------------- 6. eos
def test_eos_rows_stop_at_their_first_eos(dev):
    from gpu_util import build_tiny

    P = _P()
    model, _, _ = build_tiny(dev, CFG, seed=9)
    model.q4_batch_step = True
    prompt = _prompt(dev, CFG["vocab_size"], T=7, seed=7)
    n, steps, T = 4, 16, 7
    cases = {}
    for seed in range(40):
        model.reset_cache()
        torch.manual_seed(seed)
        free = P.generate_batch(model, prompt, n, steps, temperature=1.5, top_k=3)
        new = torch.stack(free)[:, T:].cpu()
        for eos in sorted(set(new[:, :-1].flatten().tolist())):
            firsts = [int((r == eos).nonzero()[0]) if bool((r == eos).any()) else None for r in new]
            hit = [f for f in firsts if f is not None]
            if len(hit) == n and len(set(hit)) > 1 and max(hit) < steps - 1:
                cases.setdefault("all", (seed, eos, free, firsts))
            elif 0 < len(hit) < n:
                cases.setdefault("some", (seed, eos, free, firsts))
        if len(cases) == 2:
            break
    assert "all" in cases, "no seed gave every row an eos at different steps"
    for name, (seed, eos, free, firsts) in cases.items():
        model.reset_cache()
        logs = _record(model)
        try:
            torch.manual_seed(seed)
            out = P.generate_batch(model, prompt, n, steps, temperature=1.5, top_k=3, eos_id=eos)
        finally:
            _unrecord(model)
        for y, f, y_free in zip(out, firsts, free):
            if f is None:
                assert torch.equal(y, y_free)
            else:   # ends at its first eos, which is included; the tokens before it are the eos-free run's
                assert y.numel() == T + f + 1 and int(y[-1]) == eos and torch.equal(y, y_free[:T + f + 1])
        # the loop ends once every row has finished: one model call per token up to the last row's eos
        want_calls = max(firsts) + 1 if name == "all" else steps
        assert len(logs) == want_calls, (name, len(logs), firsts)


# --------------------------------------------------------------------------------------------- 7. other batched paths
@pytest.mark.parametrize("kind", ["adapter_v2", "llm.int8", "q4-default"])
def test_other_batched_paths_within_their_bars(dev, kind):
    """A v2 model samples on the module path at B >= 2, llm.int8 on its 2..16-row step (rows interact only through the
    batch outlier mask, as in bitsandbytes), gptq.int4 by default on b2l_q4_gemv_batch; each row's logits within the bar
    of that path's existing B >= 2 tests of the batch-1 / oracle logits."""
    from gpu_util import build_tiny

    L = _L()
    if kind == "adapter_v2":
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
    prompt = _prompt(dev, 256, T=7, seed=8)
    ys, logs, qs = _sampled(model, prompt, 4, 8, S=32, seed=70)
    st = model._decode
    if kind == "adapter_v2":
        assert st is None and model._module_graph is not None
    elif kind == "llm.int8":
        assert st is not None and st.B == 4 and st.args.flags & L.F_Q8_BATCH
    else:
        assert st is not None and st.B == 4 and not st.args.flags & L.F_Q4_BATCH_I8
    _check_draws(ys, logs, qs, 7)
    same, worst = _rows_vs_batch1(model, prompt, ys, logs, 32, bar=bar)
    print(f"{kind}, B = 4: rows bit-identical to batch 1: {same} (max normwise {worst:.3g})")


# --------------------------------------------------------------------------------------------- 8. expand_cache
def test_expand_cache_then_reset(dev):
    from gpu_util import build_tiny

    model, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=33)
    model.q4_batch_step = True
    prompt = _prompt(dev, 256, T=9, seed=9).view(1, -1)
    S = 24

    def batch1():
        model.reset_cache()
        with torch.no_grad():
            a = model(prompt, S, torch.arange(9, device=dev)).clone()
            b = model(torch.tensor([[17]], device=dev), S, torch.tensor([9], device=dev)).clone()
        return a, b

    fresh = batch1()
    model.reset_cache()
    with torch.no_grad():
        model(prompt, S, torch.arange(9, device=dev))
        one = [(k.clone(), v.clone()) for k, v in model.logical_kv_caches()]
        model(torch.tensor([[17]], device=dev), S, torch.tensor([9], device=dev))   # a batch-1 step state exists
        model.reset_cache()
        model(prompt, S, torch.arange(9, device=dev))
        model.expand_cache(5)
        assert model._decode is None and model._module_graph is None
        assert model._kv_store.shape[2] == 5
        for i, (k, v) in enumerate(model.kv_caches):
            assert k.data_ptr() == model._kv_store[i, 0].data_ptr() and v.data_ptr() == model._kv_store[i, 1].data_ptr()
        for (k, v), (k1, v1) in zip(model.logical_kv_caches(), one):
            assert k.shape[0] == 5 and all(torch.equal(k[b], k1[0]) and torch.equal(v[b], v1[0]) for b in range(5))
        step = model(torch.full((5, 1), 17, device=dev), S, torch.tensor([9], device=dev)).clone()
        assert model._decode is not None and model._decode.B == 5
        assert all(torch.equal(step[b], fresh[1][0]) for b in range(5))   # the exact batched step
    model.reset_cache()
    assert model._kv_store is None and model._decode is None and model._module_graph is None and model.kv_caches == []
    again = batch1()
    assert model._decode is not None and model._decode.B == 1
    assert torch.equal(again[0], fresh[0]) and torch.equal(again[1], fresh[1])

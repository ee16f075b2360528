"""-m gpu: speculative decoding.  The stepwise attention (B2L_F_STEPWISE) against T successive T == 1 launches, bit for
bit in output and cache rows; `LLaMA.decode_tokens` rows against the teacher-forced batch-1 step, bit for bit;
`b2l_spec_accept` against its torch restatement and, by a chi-square test, its first emitted token against the target's
distribution; and `generate_speculative(top_k=1)` against `generate(top_k=1)` token for token."""
import ctypes as C
import importlib

import pytest
import torch

from test_speculative_cpu import spec_accept_ref

pytestmark = pytest.mark.gpu

CFG128 = dict(block_size=512, vocab_size=256, n_layer=3, n_head=4, n_embd=512)   # head_size 128


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _P():
    import lit_llama_b200 as P

    return P


# --------------------------------------------------------------------------------------------- 1. attention
ATTN_KINDS = ["fused", "fused-adapter", "unfused128", "unfused128-adapter", "hs32", "hs64"]


@pytest.mark.parametrize("kind", ATTN_KINDS)
@pytest.mark.parametrize("n_head", [32, 40])
def test_stepwise_attention_equals_successive_single_token_launches(dev, kind, n_head):
    """Query t of one stepwise launch and the cache rows it appends equal a T == 1 launch at position p + t on the
    cache holding the tokens before it, for T in {2, 5, 16} and p in {0, 250 (straddles 256), 1020, S - T}."""
    L = _L()
    lib = L.lib()
    P = _P()
    hs = 32 if kind == "hs32" else 64 if kind == "hs64" else 128
    adapter = kind.endswith("adapter")
    flags = L.F_PDL | (8 if kind.startswith("unfused") else 0)   # 8: B2L_F_ATTN_UNFUSED
    S, Cn = 1040, n_head * hs
    rope = P.model.build_rope_cache(2048, hs, torch.int64, dev).float().contiguous()
    g = torch.Generator(device=dev).manual_seed(n_head * 7 + len(kind))
    pre = None
    if adapter:
        ak = (torch.randn(n_head, 10, hs, device=dev, generator=g)).bfloat16()
        av = (torch.randn(n_head, 10, hs, device=dev, generator=g)).bfloat16()
        gate = (torch.randn(n_head, device=dev, generator=g) * 0.5).bfloat16()
        pre = L.AdapterPrefix(ak.data_ptr(), av.data_ptr(), gate.data_ptr(), 10)
    ring = torch.zeros(1, dtype=torch.int32, device=dev)
    st = L.stream_ptr()

    def attn(qkv, kc, vc, pos, y, work, T, fl):
        args = (qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), rope.data_ptr(), pos.data_ptr(), ring.data_ptr(), y.data_ptr(),
                work.data_ptr(), 1, T, n_head, hs, S, 2048, fl)
        if pre is None:
            L.check(lib.b2l_attention(*args, st), "b2l_attention")
        else:
            L.check(lib.b2l_attention_adapter(*args, C.byref(pre), st), "b2l_attention_adapter")

    w1 = torch.zeros(lib.b2l_attn_workspace_bytes(1, n_head, hs, 1, S) // 4 + 1, device=dev)
    for T in (2, 5, 16):
        wT = torch.zeros(lib.b2l_attn_workspace_bytes(T, n_head, hs, 1, S) // 4 + 1, device=dev)
        for p in (0, 250, 1020, S - T):
            kc = torch.zeros(1, n_head, S, hs, device=dev, dtype=torch.bfloat16)
            vc = torch.zeros_like(kc)
            kc[:, :, :p] = torch.randn(1, n_head, p, hs, device=dev, generator=g).bfloat16()
            vc[:, :, :p] = torch.randn(1, n_head, p, hs, device=dev, generator=g).bfloat16()
            kc2, vc2 = kc.clone(), vc.clone()
            qkv = (torch.randn(1, T, 3 * Cn, device=dev, generator=g) * 2).bfloat16()
            pos = torch.arange(p, p + T, device=dev)
            y = torch.empty(1, T, Cn, device=dev, dtype=torch.bfloat16)
            attn(qkv.clone(), kc, vc, pos, y, wT, T, flags | L.F_STEPWISE)
            for t in range(T):
                y1 = torch.empty(1, 1, Cn, device=dev, dtype=torch.bfloat16)
                attn(qkv[:, t:t + 1].clone(), kc2, vc2, pos[t:t + 1], y1, w1, 1, flags)
                assert torch.equal(y[0, t], y1[0, 0]), (T, p, t)
            assert torch.equal(kc, kc2) and torch.equal(vc, vc2), (T, p)
            if kind == "fused" and p == 250:   # qkv is left untouched by the fused stepwise path
                q0 = qkv.clone()
                attn(q0, kc.clone(), vc.clone(), pos, y, wT, T, flags | L.F_STEPWISE)
                assert torch.equal(q0, qkv)
    torch.cuda.synchronize()


# --------------------------------------------------------------------------------------------- 2. the model
def _model(dev, kind):
    import gpu_util  # noqa: F401  (puts tools/ on sys.path)
    from diag import _random_w8_model
    from gpu_util import build_tiny

    if kind.startswith("hs128-q4"):
        m, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=21)
    elif kind.startswith("hs128-w8"):
        m, _, _ = build_tiny(dev, CFG128, mode="gptq.int8", seed=22)
    elif kind.startswith("13B"):
        m = _random_w8_model("13B", dev, seed=66, n_layer=2, bits=4 if "q4" in kind else 8)
    elif kind == "adapter-q4":
        import test_gpu_adapter as TA

        m, _, _ = TA.build(dev, dict(TA.CFG128, block_size=512), "gptq.int4")
    elif kind == "lora-q4":
        import test_gpu_lora as TL

        m, _, _ = TL.build(dev, "gptq.int4", cfg=dict(TL.CFG, block_size=512))
    else:
        raise ValueError(kind)
    if kind.endswith("-compact"):
        m.compact()
    return m


def _batch1_logits(model, prompt, toks, S):
    """The batch-1 step's logits for tokens toks[i] at positions len(prompt) + i, after the prompt's prefill."""
    T0 = prompt.numel()
    model.reset_cache()
    model(prompt.view(1, -1), S, torch.arange(T0, device=prompt.device))
    out = []
    for i in range(toks.numel()):
        out.append(model(toks[i].view(1, 1), S, torch.tensor([T0 + i], device=prompt.device))[0, -1].clone())
    return torch.stack(out)


@pytest.mark.parametrize("kind", ["hs128-q4", "hs128-q4-compact", "hs128-w8", "hs128-w8-compact", "13B-q4", "13B-w8",
                                  "adapter-q4", "lora-q4"])
def test_decode_tokens_rows_equal_the_batch1_step(dev, kind):
    """Rows of decode_tokens over chunks of 2..16 tokens (positions 250..300, past 256) equal the teacher-forced batch-1
    step bit for bit, on the CUDA-graph replay too, and the cache ends where the batch-1 steps leave it."""
    L = _L()
    model = _model(dev, kind)
    try:
        V = model.config.vocab_size
        S = 320
        g = torch.Generator().manual_seed(8)
        prompt = torch.randint(0, V, (250,), generator=g).to(dev)
        chunks = [2, 5, 16, 2, 2, 3, 5, 16, 2]
        toks = torch.randint(0, V, (sum(chunks),), generator=g).to(dev)
        want = _batch1_logits(model, prompt, toks, S)
        kv1 = model._kv_store.clone()
        model.reset_cache()
        model(prompt.view(1, -1), S, torch.arange(250, device=dev))
        i = 0
        for T in chunks:
            got = model.decode_tokens(toks[i:i + T].view(1, T), S, torch.arange(250 + i, 250 + i + T, device=dev))
            assert got.shape == (T, model.config.padded_vocab_size)
            for t in range(T):
                assert torch.equal(got[t], want[i + t]), (kind, T, i + t)
            i += T
        assert torch.equal(model._kv_store, kv1)
        st = model._verify[2]
        assert st.graph is not None and st.args.flags & L.F_STEPWISE
        assert st.args.flags & (L.F_Q4_BATCH_I8 if "q4" in kind else L.F_W8_BATCH)
    finally:
        del model
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- 3. b2l_spec_accept
def _accept(L, logits, temp, top_k, q, x, u, noise):
    T, V = logits.shape
    n = torch.full((1,), -1, dtype=torch.int32, device=logits.device)
    tok = torch.full((1,), -1, dtype=torch.int64, device=logits.device)
    L.check(L.lib().b2l_spec_accept(logits.data_ptr(), V, float(temp), top_k, q.data_ptr(), x.data_ptr(), u.data_ptr(),
                                    noise.data_ptr(), n.data_ptr(), tok.data_ptr(), T, V, L.stream_ptr()), "b2l_spec_accept")
    return int(n), int(tok)


@pytest.mark.parametrize("V", [256, 32000])
def test_spec_accept_equals_torch_restatement(dev, V):
    """On random logits at several temperature / top_k settings, with draft tokens drawn from q, from the target's
    argmax, and out of range, every (n_accepted, token) equals spec_accept_ref on the probabilities
    b2l_topk_softmax_rows computes."""
    L, P = _L(), _P()
    g = torch.Generator(device=dev).manual_seed(V)
    seen = set()
    for temp, top_k in ((1.0, None), (0.7, 50), (1.3, 1), (0.9, 4)):
        for k in (1, 3, 15):
            for trial in range(6):
                scale = 1 + trial % 3
                lt = (torch.randn(k + 1, V, device=dev, generator=g) * scale).bfloat16()
                ld = (lt[:k].float() + torch.randn(k, V, device=dev, generator=g) * 0.5 * trial).bfloat16()
                p = P.sample_probs(lt, temp, top_k)
                q = P.sample_probs(ld.contiguous(), temp, top_k)
                if trial % 3 == 0:
                    x = torch.multinomial(q.float(), 1, generator=g).view(k)
                elif trial % 3 == 1:
                    x = p[:k].float().argmax(-1)
                else:
                    x = torch.multinomial(q.float(), 1, generator=g).view(k)
                    x[k // 2] = V + 3
                u = torch.rand(k, device=dev, generator=g)
                noise = torch.empty(V, dtype=torch.bfloat16, device=dev).exponential_(1, generator=g)
                got = _accept(L, lt, temp, 0 if top_k is None else top_k, q, x, u, noise)
                want = spec_accept_ref(p, q, x, u, noise)
                assert got == want, (temp, top_k, k, trial, got, want)
                seen.add(got[0] == k)
    assert seen == {True, False}   # both all-accepted rounds and rejections were exercised


def test_spec_accept_first_token_is_distributed_as_the_target(dev):
    """k = 2 rounds with the draft token drawn from q: the first emitted token (x_0 when accepted, else the residual
    draw) of 20 000 rounds follows the target's p_0 (chi-square, fixed seed)."""
    from scipy.stats import chisquare

    L, P = _L(), _P()
    V, k, N = 32, 2, 20000
    g = torch.Generator(device=dev).manual_seed(123)
    lt = (torch.randn(k + 1, V, device=dev, generator=g) * 1.5).bfloat16()
    ld = (torch.randn(k, V, device=dev, generator=g) * 1.5).bfloat16()
    p = P.sample_probs(lt, 1.0, None)
    q = P.sample_probs(ld, 1.0, None)
    xs = torch.stack([torch.multinomial(q[t].float(), N, replacement=True, generator=g) for t in range(k)], dim=1).contiguous()
    us = torch.rand(N, k, device=dev, generator=g)
    noises = torch.empty(N, V, dtype=torch.bfloat16, device=dev).exponential_(1, generator=g)
    ns = torch.empty(N, dtype=torch.int32, device=dev)
    toks = torch.empty(N, dtype=torch.int64, device=dev)
    lib, st = L.lib(), L.stream_ptr()
    for i in range(N):
        x = xs[i]
        L.check(lib.b2l_spec_accept(lt.data_ptr(), V, 1.0, 0, q.data_ptr(), x.data_ptr(), us[i].data_ptr(),
                                    noises[i].data_ptr(), ns[i:].data_ptr(), toks[i:].data_ptr(), k + 1, V, st),
                "b2l_spec_accept")
    first = torch.where(ns > 0, xs[:, 0], toks).cpu()
    counts = torch.bincount(first, minlength=V).double()
    exp = p[0].double().cpu()
    exp = exp / exp.sum() * N
    keep = exp >= 5
    obs = torch.cat((counts[keep], counts[~keep].sum().view(1)))
    ex = torch.cat((exp[keep], exp[~keep].sum().view(1)))
    if float(ex[-1]) < 5:   # fold a small remainder into the largest bin
        obs, ex = obs[:-1].clone(), ex[:-1].clone()
        obs[ex.argmax()] += counts[~keep].sum()
        ex[ex.argmax()] += exp[~keep].sum()
    ex = ex * obs.sum() / ex.sum()
    stat, pval = chisquare(obs.numpy(), ex.numpy())
    assert 0 < int((ns == 0).sum()) < N   # rejections happen
    assert pval > 1e-3, (stat, pval)


# --------------------------------------------------------------------------------------------- 4. end to end
def _greedy_ties(model, prompt, y, S):
    """Whether any step of the greedy sequence y had a tie for the top logit (teacher-forced batch-1 logits)."""
    T0 = prompt.numel()
    lg = [None]
    model.reset_cache()
    lg = [model(prompt.view(1, -1), S, torch.arange(T0, device=prompt.device))[0, -1].clone()]
    for i in range(T0, y.numel() - 1):
        lg.append(model(y[i].view(1, 1), S, torch.tensor([i], device=prompt.device))[0, -1].clone())
    model.reset_cache()
    top2 = torch.stack(lg).float().topk(2, dim=-1).values
    return bool((top2[:, 0] == top2[:, 1]).any())


@pytest.fixture(scope="module")
def models(dev):
    from gpu_util import build_tiny

    target, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=21)
    same, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=21)     # the target's weights: every token accepted
    other, _, _ = build_tiny(dev, CFG128, mode="gptq.int4", seed=77)    # another model: rejections
    return target, same, other


def _prompt_without_ties(P, target, dev, n_new, S):
    for seed in range(8):
        prompt = torch.randint(0, 256, (9,), generator=torch.Generator().manual_seed(seed)).to(torch.int32).to(dev)
        target.reset_cache()
        want = P.generate(target, prompt, n_new, max_seq_length=S, top_k=1)
        if not _greedy_ties(target, prompt, want, S if S is not None else min(prompt.numel() + n_new, 512)):
            return prompt, want
    raise AssertionError("every candidate prompt had a top-1 tie")


@pytest.mark.parametrize("num_draft", [1, 3, 15])
@pytest.mark.parametrize("which", ["other", "same"])
def test_greedy_speculative_equals_generate(dev, models, num_draft, which):
    P = _P()
    target, same, other = models
    draft = same if which == "same" else other
    prompt, want = _prompt_without_ties(P, target, dev, 40, None)
    target.reset_cache()
    draft.reset_cache()
    stats = {}
    got = P.generate_speculative(target, draft, prompt, 40, num_draft=num_draft, top_k=1, stats=stats)
    target.reset_cache()
    draft.reset_cache()
    assert got.dtype == want.dtype and torch.equal(got, want), (got.tolist(), want.tolist())
    assert stats["rounds"] == len(stats["accepted"]) and stats["rounds"] > 0
    assert 1 + sum(a + 1 for a in stats["accepted"]) + stats["tail_steps"] == 40
    if which == "same":
        assert stats["accepted"] == stats["proposed"]
    else:
        assert sum(stats["accepted"]) < sum(stats["proposed"])   # rejections happened


def test_greedy_speculative_eos_and_tight_cache(dev, models):
    P = _P()
    target, same, other = models
    # eos in the middle of a round: the output ends at its first occurrence, eos included
    prompt, want = _prompt_without_ties(P, target, dev, 40, None)
    eos = int(want[9 + 17])
    first = int((want[9:] == eos).nonzero()[0]) + 9
    for draft in (same, other):
        target.reset_cache()
        draft.reset_cache()
        got = P.generate_speculative(target, draft, prompt, 40, num_draft=5, top_k=1, eos_id=eos)
        assert torch.equal(got, want[:first + 1]), (got.tolist(), want[:first + 1].tolist())
    # max_seq_length = 19 for 9 + 24 tokens: k shrinks as the cache fills, and the tail rolls like generate()'s
    prompt, want = _prompt_without_ties(P, target, dev, 24, 19)
    for draft in (same, other):
        target.reset_cache()
        draft.reset_cache()
        stats = {}
        got = P.generate_speculative(target, draft, prompt, 24, num_draft=4, top_k=1, max_seq_length=19, stats=stats)
        assert torch.equal(got, want), (got.tolist(), want.tolist())
        # the last verified position is 18 = S - 1, so at most 10 + 1 tokens come out of rounds
        assert stats["tail_steps"] >= 24 - (19 - 9) - 1
        assert max(stats["proposed"]) <= 4 and min(stats["proposed"]) >= 1
    target.reset_cache()
    same.reset_cache()
    other.reset_cache()


def test_sampled_speculative_runs(dev, models):
    """Sampling at temperature 0.8 / top_k 50: the tokens are in range and the statistics add up."""
    P = _P()
    target, _, other = models
    prompt = torch.randint(0, 256, (9,), generator=torch.Generator().manual_seed(1)).to(torch.int32).to(dev)
    target.reset_cache()
    other.reset_cache()
    torch.manual_seed(3)
    stats = {}
    y = P.generate_speculative(target, other, prompt, 30, num_draft=4, temperature=0.8, top_k=50, stats=stats)
    assert y.numel() == 39 and torch.equal(y[:9], prompt) and int(y.min()) >= 0 and int(y.max()) < 256
    assert 1 + sum(a + 1 for a in stats["accepted"]) + stats["tail_steps"] == 30
    target.reset_cache()
    other.reset_cache()

"""-m gpu: continuous batching (`generate_stream`), the rows it refills (`LLaMA.refill_rows`) and the ragged prefill
attention under it (`b2l_attention_ragged`).

1. Kernel: sequences packed into one qkv, each sent into its own row of a cache holding stale data with nonzero ring
   offsets, equal per-sequence B = 1 launches bit for bit (y, rotated q, written rows); untouched rows and their ring
   offsets stay byte for byte; refilled rings are 0.
2. Premise: the row-exact kernels (b2l_q4_gemm, b2l_w8_gemm, b2l_lora_apply, b2l_linear_affine) give a row the same bits
   at any M and at any offset inside a 128-row tile.
3. refill_rows: logits and logical KV caches equal a reset_cache() batch-1 prefill, packed and alone routes alike; other
   rows are untouched; the B-row decode state and its CUDA graph are the same objects after a refill.
4. / 5. generate_stream: greedy output equals generate(top_k=1) per prompt (refills, rolled rows, eos); sampled draws are
   argmax(probs / q) of their rows; with <= B prompts it is generate_prompts.
6. Other routes (LLaMA-Adapter v1 / v2, LoRA, llm.int8, dense, the golden head_size-32 model): refill logits are bit
   for bit batch 1 (packed or alone), and decoded rows are held to the bars of test_gpu_generate_prompts."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

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


def _ragged(L, lengths, rows):
    sq = L.Ragged()
    sq.n_seq = len(lengths)
    at = 0
    for s, (n, r) in enumerate(zip(lengths, rows)):
        sq.row[s], sq.start[s], sq.len[s] = r, at, n
        at += n
    return sq


# --------------------------------------------------------------------------------------------- 1. kernel
@pytest.mark.parametrize("adapter", [False, True])
@pytest.mark.parametrize("nh", [32, 40])
def test_ragged_equals_batch1_launches(dev, nh, adapter):
    import test_gpu_attention as TA

    L = _L()
    lib = L.lib()
    hs, S, B_rows = 128, 256, 8
    lengths = [1, 63, 64, 65, 130, S]
    rows = [5, 0, 7, 2, 6, 3]            # rows 1 and 4 are not named
    N = sum(lengths)
    g = torch.Generator(device=dev).manual_seed(nh + adapter)
    qkv = torch.randn(1, N, 3 * nh * hs, device=dev, generator=g).bfloat16()
    kc = (torch.randn(B_rows, nh, S, hs, device=dev, generator=g) * 0.5).bfloat16()   # stale contents
    vc = (torch.randn(B_rows, nh, S, hs, device=dev, generator=g) * 0.5).bfloat16()
    ring = torch.randint(1, S, (B_rows,), device=dev, generator=g).to(torch.int32)
    prefix = TA._prefix(dev, nh, 10, hs, seed=nh) if adapter else None
    rope = TA._rope(hs, dev)[1]
    q2, k2, v2, r2 = qkv.clone(), kc.clone(), vc.clone(), ring.clone()
    y = torch.full((1, N, nh * hs), float("nan"), device=dev, dtype=torch.bfloat16)
    sq = _ragged(L, lengths, rows)
    rc = lib.b2l_attention_ragged(q2.data_ptr(), k2.data_ptr(), v2.data_ptr(), rope.data_ptr(), C.byref(sq),
                                  r2.data_ptr(), y.data_ptr(), N, B_rows, nh, hs, S, rope.shape[0],
                                  None if prefix is None else C.byref(prefix[0]), L.stream_ptr())
    L.check(rc, "b2l_attention_ragged")
    at = 0
    for n, r in zip(lengths, rows):
        q1 = qkv[:, at:at + n].clone()
        k1, v1 = kc[r:r + 1].clone(), vc[r:r + 1].clone()
        y1 = TA._launch(q1, k1, v1, 0, 0, nh, prefix=prefix, rope=rope)
        assert torch.equal(y[:, at:at + n], y1), (n, r)
        assert torch.equal(q2[:, at:at + n], q1), (n, r)   # q rotated in place, k / v thirds untouched, as at B = 1
        assert torch.equal(k2[r], k1[0]) and torch.equal(v2[r], v1[0]), (n, r)
        assert int(r2[r]) == 0
        at += n
    for r in (1, 4):
        assert torch.equal(k2[r], kc[r]) and torch.equal(v2[r], vc[r]) and int(r2[r]) == int(ring[r]), r
    assert not torch.isnan(y).any()


# --------------------------------------------------------------------------------------------- 2. premise
def _rows_any_m(fn, x, what):
    """fn(rows of x) at M = 300 against the same rows at M = T, at offsets that put them elsewhere in a 128-row tile."""
    full = fn(x)
    for off, T in ((0, 17), (17, 40), (100, 130), (130, 1), (255, 45), (299, 1)):
        part = fn(x[off:off + T].contiguous())
        assert torch.equal(part, full[off:off + T]), (what, off, T)


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_gemm_rows_independent_of_m(dev, mode):
    from gpu_util import build_tiny

    model, _, _ = build_tiny(dev, CFG128, mode=mode, seed=5)
    kern = "q4_gemm" if mode == "gptq.int4" else "w8_gemm"
    g = torch.Generator(device=dev).manual_seed(1)
    for lin in (model.transformer.h[0].attn.c_attn, model.transformer.h[1].mlp.c_proj, model.lm_head):
        x = torch.randn(300, lin.in_features, device=dev, generator=g).bfloat16()
        _rows_any_m(lambda t: lin.run(t, kern), x, kern)


def test_lora_and_affine_rows_independent_of_m(dev):
    import test_gpu_lora as TL
    from lit_llama_b200.adapter_v2 import linear_affine

    model, _, _ = TL.build(dev, "gptq.int4")
    lin = model.transformer.h[0].attn.c_attn
    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(300, lin.in_features, device=dev, generator=g).bfloat16()
    y0 = torch.randn(300, lin.out_features, device=dev, generator=g).bfloat16()
    full = lin._add_lora(x, y0.clone())
    for off, T in ((0, 17), (17, 40), (100, 130), (130, 1), (255, 45)):
        part = lin._add_lora(x[off:off + T].contiguous(), y0[off:off + T].clone())
        assert torch.equal(part, full[off:off + T]), ("lora", off, T)
    N = 384
    scale = (torch.rand(N, device=dev, generator=g) + 0.5).bfloat16()
    bias = torch.randn(N, device=dev, generator=g).bfloat16()
    z = torch.randn(300, N, device=dev, generator=g).bfloat16()
    _rows_any_m(lambda t: linear_affine(t.clone(), scale, bias), z, "affine")


# --------------------------------------------------------------------------------------------- 3. refill_rows
LENGTHS = (1, 3, 16, 17, 40, 130)   # the tiny head_size-128 models (block_size 64) take 60 for 130


def _exact_model(dev, kind, compact):
    import test_gpu_generate_prompts as TG

    model = TG._exact_model(dev, kind)
    if compact:
        model.compact()
    return model


def _prompts(dev, V, lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, V, (n,), generator=g).to(torch.int32).to(dev) for n in lengths]


def _batch1(model, prompts, S):
    """The batch-1 prefill of each prompt after reset_cache(): (last-position logits, logical KV caches [layer](k, v))."""
    out = []
    for p in prompts:
        model.reset_cache()
        lg = model(p.view(1, -1), S, torch.arange(p.numel(), device=p.device))[0, -1].clone()
        out.append((lg, [(k[0].clone(), v[0].clone()) for k, v in model.logical_kv_caches()]))
    model.reset_cache()
    return out


def _check_rows(model, got, refs, rows, prompts):
    caches = model.logical_kv_caches()
    for lg, (lg1, kv1), r, p in zip(got, refs, rows, prompts):
        n = p.numel()
        assert torch.equal(lg, lg1), (r, n)
        for (k, v), (k1, v1) in zip(caches, kv1):
            assert torch.equal(k[r][:, :n], k1[:, :n]) and torch.equal(v[r][:, :n], v1[:, :n]), (r, n)
        assert int(model._ring[r]) == 0


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("kind", ["hs128-q4", "hs128-w8", "13B-q4", "13B-w8"])
def test_refill_rows_bit_identical_to_batch1(dev, kind, compact):
    model = _exact_model(dev, kind, compact)
    try:
        S = min(160, model.config.block_size)
        prompts = _prompts(dev, model.config.vocab_size, [min(n, S - 4) for n in LENGTHS], seed=12)
        refs = _batch1(model, prompts, S)
        # four rows: 17, 3, 130 (60), 40 (three packed, one alone at gptq.int4; all four packed at gptq.int8)
        first = [3, 1, 5, 4]
        got = model.prefill_rows([prompts[i] for i in first], S)
        _check_rows(model, got, [refs[i] for i in first], range(4), [prompts[i] for i in first])
        pos = torch.tensor([prompts[i].numel() for i in first], device=dev).view(4, 1)
        x = torch.randint(0, 50, (4, 1), device=dev, dtype=torch.int32)
        for _ in range(3):   # eager, eager, captured: the B-row state and its graph exist
            model(x, S, pos)
            pos = pos + 1
        st = model._decode
        assert st is not None and st.B == 4 and st.graph is not None
        graph = st.graph
        for rows, ids in (([2, 0], [0, 2]), ([3, 1, 0], [5, 0, 4])):   # 1- and 16-token prompts, then 130, 1, 40
            keep = [r for r in range(4) if r not in rows]
            store, ring = model._kv_store.clone(), model._ring.clone()
            want_packed = model._pack_plan([prompts[i].numel() for i in ids])
            got = model.refill_rows([prompts[i] for i in ids], rows, S)
            _check_rows(model, got, [refs[i] for i in ids], rows, [prompts[i] for i in ids])
            for r in keep:
                assert torch.equal(model._kv_store[:, :, r], store[:, :, r]) and int(model._ring[r]) == int(ring[r]), r
            assert model._decode is st and st.graph is graph, "the B-row decode state was rebuilt"
            assert model._ring.numel() == 4 and model._kv_store.shape[2] == 4
            print(f"{kind} compact={compact}: refill of {[prompts[i].numel() for i in ids]}, packed {want_packed}")
        model(x, S, pos)   # the same graph replays on the refilled cache
        assert model._decode is st and st.graph is graph
    finally:
        del model
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- 4. greedy
STREAM_LENGTHS = (1, 3, 16, 17, 40, 5, 20, 33, 2, 18, 44, 9)
STREAM_NEW = (10, 30, 5, 25, 14, 40, 8, 3, 22, 15, 6, 35)


def _first_argmax(probs, num_samples):
    """torch.multinomial's stand-in for greedy decoding with ties broken to the lowest token id: bf16 logits over a small
    vocabulary tie often, top_k=1 keeps every tied token, and the draw among them would depend on the RNG stream."""
    return probs.argmax(dim=-1, keepdim=True)


@pytest.mark.parametrize("with_eos", [False, True])
@pytest.mark.parametrize("kind", ["hs128-q4", "hs128-w8"])
def test_greedy_stream_equals_generate(dev, kind, with_eos, monkeypatch):
    """12 prompts on 4 rows, S = 48: the 40- and 44-token prompts roll before their rows are refilled.  generate() ends
    before an eos it draws (`idx[:input_pos]`, as the reference's generate.py does); generate_stream keeps it, as
    generate_prompts does."""
    P = _P()
    monkeypatch.setattr(torch, "multinomial", _first_argmax)   # generate() and generate_stream() both call it
    model = _exact_model(dev, kind, compact=False)
    S = 48
    prompts = _prompts(dev, CFG128["vocab_size"], STREAM_LENGTHS, seed=21)
    eos = None
    if with_eos:
        model.reset_cache()
        free = P.generate_stream(model, prompts, list(STREAM_NEW), batch_size=4, max_seq_length=S, top_k=1)
        eos = int(free[5][prompts[5].numel() + 3])   # a token the 5th prompt draws early on
    model.reset_cache()
    stats = {}
    ys = P.generate_stream(model, prompts, list(STREAM_NEW), batch_size=4, max_seq_length=S, top_k=1, eos_id=eos,
                           stats=stats)
    assert model._decode.B == 4 and stats["refills"] == 8 and stats["packed"] + stats["alone"] == 12, stats
    for p, m, y in zip(prompts, STREAM_NEW, ys):
        model.reset_cache()
        want = P.generate(model, p, m, max_seq_length=S, top_k=1, eos_id=eos)
        if want.numel() < p.numel() + m:   # generate() drew eos
            want = torch.cat((want, torch.tensor([eos], dtype=want.dtype, device=dev)))
        assert torch.equal(y, want), (p.numel(), m, y.tolist(), want.tolist())
    if with_eos:
        assert any(y.numel() < p.numel() + m for y, p, m in zip(ys, prompts, STREAM_NEW))
    print(f"{kind} eos={eos}: {stats}")


# --------------------------------------------------------------------------------------------- 5. sampling
def _recorded(monkeypatch, model, fn, seed):
    """Runs fn() with every sampling launch's (B, V) logits and tokens recorded; returns (fn's result, logits, tokens,
    the Exp(1) noise of each launch regenerated from `seed`)."""
    import importlib

    G = importlib.import_module("lit_llama_b200.generate")
    logs, toks = [], []
    orig = G.sample_token

    def rec(rows, temperature=1.0, top_k=None):
        logs.append(rows.clone())
        t = orig(rows, temperature, top_k)
        toks.append(t.clone())
        return t

    monkeypatch.setattr(G, "sample_token", rec)
    model.reset_cache()
    torch.manual_seed(seed)
    out = fn()
    torch.cuda.synchronize()
    monkeypatch.setattr(G, "sample_token", orig)
    torch.manual_seed(seed)
    qs = [torch.empty_like(lg).exponential_(1) for lg in logs]
    return out, logs, toks, qs


def test_sampled_draws_and_generate_prompts(dev, monkeypatch):
    P = _P()
    model = _exact_model(dev, "hs128-q4", compact=False)
    prompts = _prompts(dev, CFG128["vocab_size"], STREAM_LENGTHS, seed=22)
    kw = dict(temperature=1.3, top_k=20)
    ys, logs, toks, qs = _recorded(monkeypatch, model, lambda: P.generate_stream(
        model, prompts, list(STREAM_NEW), batch_size=4, max_seq_length=48, **kw), seed=31)
    for lg, t, q in zip(logs, toks, qs):
        assert torch.equal(t, torch.argmax(P.sample_probs(lg, **kw) / q, dim=-1))
    assert all(y.numel() == p.numel() + m for y, p, m in zip(ys, prompts, STREAM_NEW))
    # <= B prompts and one max_new_tokens: no refill, and generate_prompts' output for the same seed
    few = prompts[2:6]
    model.reset_cache()
    torch.manual_seed(7)
    a = P.generate_stream(model, few, 12, batch_size=8, **kw)
    model.reset_cache()
    torch.manual_seed(7)
    b = P.generate_prompts(model, few, 12, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


# --------------------------------------------------------------------------------------------- 6. other routes
def _schedule(n, B, news):
    """generate_stream's FIFO admission without eos: (row, step of the first token) of every prompt."""
    out = {i: (i, 0) for i in range(B)}
    rows = [(news[i], i) for i in range(B)]   # (step the row takes its next prompt, row): lower rows first on a tie
    for i in range(B, n):
        rows.sort()
        t, r = rows.pop(0)
        out[i] = (r, t)
        rows.append((t + news[i], r))
    return out


@pytest.mark.parametrize("kind", ["adapter", "adapter_v2", "lora", "llm.int8", "dense", "hs32"])
def test_other_routes(dev, kind, monkeypatch):
    """Refill logits equal batch 1 bit for bit (packed where the model packs, alone where it does not); every draw is
    argmax(probs / q); each prompt's decoded logits are within the bar of its route's B >= 2 test against the batch-1
    model teacher-forced on its output (test_gpu_generate_prompts.test_other_routes_within_their_bars; the golden
    head_size-32 model and the dense model as its "q4-default" and module routes)."""
    import test_gpu_generate_prompts as TG
    from gpu_util import build_tiny

    P = _P()
    packs = kind in ("adapter", "adapter_v2", "lora")
    if kind == "adapter":
        import test_gpu_adapter as TA

        model, _, _ = TA.build(dev, TA.CFG128, "gptq.int4")
        model.q4_batch_step = True
        bar = 1e-2
    elif kind == "adapter_v2":
        import test_gpu_adapter_v2 as TV

        model, _, _ = TV.build(dev, TV.CFG128, "gptq.int4")
        bar = 2e-2
    elif kind == "lora":
        import test_gpu_lora as TL

        model, _, _ = TL.build(dev, "gptq.int4")
        model.q4_batch_step = True
        bar = 1e-2
    elif kind == "llm.int8":
        model, _, _ = build_tiny(dev, CFG128, mode="llm.int8", seed=31)
        model.int8_step = True
        bar = 6e-2
    elif kind == "dense":
        model, _, _ = build_tiny(dev, CFG128, mode=None, seed=33)
        bar = 2e-2
    else:
        model, _, _ = build_tiny(dev, TG.CFG, seed=34)
        model.q4_batch_step = True
        bar = 2e-2
    V = model.config.vocab_size
    lengths, news, S = (3, 20, 17, 7, 40, 1), (6, 3, 5, 4, 6, 5), 48
    prompts = _prompts(dev, V, lengths, seed=9)
    plan = model._pack_plan(list(lengths))
    assert (plan == [1, 2, 4]) if packs else plan == [], plan
    refs = _batch1(model, prompts, S)
    got = model.prefill_rows(prompts[:3], S)
    got2 = model.refill_rows(prompts[3:], [2, 0, 1], S)
    for lg, (lg1, _) in zip(list(got) + list(got2), refs):
        assert torch.equal(lg, lg1)
    ys, logs, toks, qs = _recorded(monkeypatch, model, lambda: P.generate_stream(
        model, prompts, list(news), batch_size=3, max_seq_length=S), seed=41)
    for lg, t, q in zip(logs, toks, qs):
        assert torch.equal(t, torch.argmax(P.sample_probs(lg) / q, dim=-1))
    same, worst = True, 0.0
    for i, (row, s0) in _schedule(len(prompts), 3, news).items():
        one = TG._teacher_forced(model, prompts[i], ys[i], S)
        assert len(one) == news[i]
        for j, o in enumerate(one):
            lg = logs[s0 + j][row]
            r = float((lg.float() - o[0].float()).norm() / o[0].float().norm())
            same, worst = same and torch.equal(lg, o[0]), max(worst, r)
            assert r < bar, (kind, i, j, r)
    print(f"{kind}: packed {plan}; decoded rows bit-identical to batch 1: {same} (max normwise {worst:.3g})")

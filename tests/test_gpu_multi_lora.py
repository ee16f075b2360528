"""GPU: multi-LoRA.  b2l_lora_apply_rows row by row against b2l_lora_apply on that row alone (bit for bit); the
batched decode step with one adapter per row against separate batch-1 models that carry only that row's adapter,
eager, graph-replayed and after rows change adapters; generate_stream / generate_prompts with adapters against
generate(); the module path within its batched bars; and the memory an adapter adds."""
import ctypes as C
import functools
from contextlib import nullcontext

import pytest
import torch

import lit_llama_b200 as P
from lit_llama_b200 import _lib as L
from lit_llama_b200 import lora as PL
from lit_llama_b200.utils import quantization
from oracle import llama_oracle as O
from oracle import lora_oracle as LO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    return torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------------ 1. the kernel
def _one(spec, x, y, norm):
    M, K = x.shape
    N = y.shape[1]
    L.check(L.lib().b2l_lora_apply(C.byref(spec), x.data_ptr(), K, None if norm is None else norm.data_ptr(), 1e-5,
                                   y.data_ptr(), N, M, N, K, 0, L.stream_ptr()), "b2l_lora_apply")


def _rows(specs, row_set, x, y, norm, flags=0):
    M, K = x.shape
    N = y.shape[1]
    arr = (L.LoRA * len(specs))(*specs)
    L.check(L.lib().b2l_lora_apply_rows(arr, len(specs), row_set.data_ptr(), x.data_ptr(), K,
                                        None if norm is None else norm.data_ptr(), 1e-5, y.data_ptr(), N, M, N, K, flags,
                                        L.stream_ptr()), "b2l_lora_apply_rows")


def _check_rows(dev, K, N, n_groups, terms, patterns, seed):
    """terms: (r, mask) per set.  Every row of b2l_lora_apply_rows equals b2l_lora_apply of its set on that row alone;
    -1 rows (and out-of-range entries) are untouched."""
    g = torch.Generator(device=dev).manual_seed(seed)
    keep, specs = [], []
    for j, (r, mask) in enumerate(terms):
        n_on = bin(mask).count("1")
        A = ((torch.rand(r * n_on, K, device=dev, generator=g) * 2 - 1) / K ** 0.5).bfloat16()
        B = (torch.randn(N // n_groups * n_on, r, device=dev, generator=g) * 0.05).bfloat16()
        keep += [A, B]
        specs.append(L.LoRA(A.data_ptr(), B.data_ptr(), 16.0 / r * (1 + j / 8), r, n_groups, mask))
    sc = (0.25 + 1.5 * torch.rand(K, device=dev, generator=g)).bfloat16()
    for sets in patterns:
        M = len(sets)
        x = (torch.randn(M, K, device=dev, generator=g) * 8).bfloat16()
        y0 = (torch.randn(M, N, device=dev, generator=g) * 0.5).bfloat16()
        row_set = torch.tensor(sets, dtype=torch.int32, device=dev)
        for norm in (None, sc):
            for flags in (0, L.F_PDL):
                got = y0.clone()
                _rows(specs, row_set, x, got, norm, flags)
                for m, s in enumerate(sets):
                    want = y0[m:m + 1].clone()
                    if 0 <= s < len(specs):
                        _one(specs[s], x[m:m + 1].contiguous(), want, norm)
                        assert not torch.equal(want, y0[m:m + 1])
                    assert torch.equal(got[m:m + 1], want), (M, sets, m, norm is not None)
    torch.cuda.synchronize()


@pytest.mark.parametrize("C_", [4096, 5120, 8192])
def test_rows_kernel_bit_identical_to_one_row(dev, C_):
    """c_attn of 7B / 13B / 65B (q and v), ranks 1 / 8 / 64 mixed across sets, M = 1..16: every row the same set,
    every row its own, and a mix with -1 rows and an out-of-range entry (treated as -1)."""
    terms = [(8, 0b101), (1, 0b101), (64, 0b101), (8, 0b101)] * 4
    pats = []
    for M in (1, 2, 3, 5, 8, 13, 16):
        pats += [[2] * M, [(m * 5) % 16 for m in range(M)], [[-1, 1, 3, 16, 1, 0][m % 6] if m % 4 else -1 for m in range(M)]]
    _check_rows(dev, C_, 3 * C_, 3, terms, pats, C_)


@pytest.mark.parametrize("enable", [[True, True, True], [False, True, False], [True, False, False, True],
                                    [False, False, True, True, False, False, True, False]])
def test_rows_kernel_group_masks(dev, enable):
    """The group patterns of test_lora_kernel_group_patterns, and sets whose masks differ (same n_groups)."""
    n = len(enable)
    mask = sum(1 << i for i, e in enumerate(enable) if e)
    other = ((1 << n) - 1) ^ mask or 1
    terms = [(4, mask), (8, other), (2, (1 << n) - 1)]
    pats = [[0, 1, 2, -1, 2, 0, 1], [1] * 5, [0], [-1, -1, 2]]
    _check_rows(dev, 512, 1024 if n != 3 else 1536, n, terms, pats, n * 17 + sum(enable))


# ------------------------------------------------------------------------------------------------ 2. models
TINY = dict(block_size=64, vocab_size=256, n_layer=2, n_head=4, n_embd=512)
W13B = dict(block_size=64, vocab_size=256, n_layer=2, n_head=40, n_embd=5120)


@functools.lru_cache(maxsize=4)
def _base_sd(mode, key):
    cfg = dict(key)
    return O.synth_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"],
                              None if mode == "llm.int8" else mode)


def _lw(cfg, k):
    """Adapter k's LoRA state dict (ranks differ between adapters)."""
    return LO.lora_weights(cfg["n_layer"], cfg["n_embd"], r=(8, 4, 16, 8)[k % 4], seed=1000 + 7 * k)


def _model(dev, mode, cfg, lw=None, compact=False):
    """Built and loaded the reference way: the base checkpoint, then (if given) one LoRA state dict."""
    sd = _base_sd(mode, tuple(sorted(cfg.items())))
    r = next(v.shape[0] // 2 for k, v in lw.items() if k.endswith("lora_A")) if lw else 0
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization(mode), (PL.lora(r=r, alpha=16, dropout=0.0) if lw else nullcontext()):
            m = P.LLaMA(P.LLaMAConfig(**cfg))
    finally:
        torch.set_default_dtype(prev)
    m.load_state_dict(sd, strict=lw is None)
    if lw:
        m.load_state_dict(lw, strict=False)
    m.eval()
    if compact:
        m.compact()
    return m


def _multi(dev, mode, cfg, n_added, compact=False):
    """Adapter 0 loaded as generate/lora.py does, adapters 1..n_added registered."""
    m = _model(dev, mode, cfg, _lw(cfg, 0), compact)
    for k in range(1, n_added + 1):
        assert PL.add_lora_adapter(m, _lw(cfg, k), alpha=16) == k
    if mode == "gptq.int4":
        m.q4_batch_step = True
    elif mode == "gptq.int8":
        m.w8_batch_step = True
    else:
        m.int8_step = True
    return m


def _batch1(dev, mode, cfg, adapter, prompt, toks, S, compact=False):
    m = _model(dev, mode, cfg, None if adapter < 0 else _lw(cfg, adapter), compact)
    T = prompt.numel()
    with torch.no_grad():
        out = [m(prompt.view(1, -1), S, torch.arange(T, device=dev))[0, -1].clone()]
        for i, t in enumerate(toks):
            out.append(m(torch.tensor([[t]], device=dev), S, torch.tensor([T + i], device=dev))[0, -1].clone())
    torch.cuda.synchronize()
    return out


def _prompts(dev, n, seed, V=256):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, V, (int(torch.randint(1, 20, (1,), generator=g)),), generator=g).to(torch.int32).to(dev)
            for _ in range(n)]


@pytest.mark.parametrize("mode,cfg,compact,ads", [
    ("gptq.int4", TINY, False, [0, 1, -1, 2, 1, 0, 3, 2, 1, -1, 3, 0, 2, 2, 1, 0]),
    ("gptq.int4", TINY, True, [3, -1, 1]),
    ("gptq.int4", W13B, True, [1, 0, -1, 2, 3]),
    ("gptq.int8", TINY, False, [2, 0, -1, 1, 3, 1, 2]),
    ("gptq.int8", W13B, False, [0, 2]),
    ("llm.int8", TINY, False, [1, -1, 0, 2]),
])
def test_step_rows_equal_batch1_models(dev, mode, cfg, compact, ads):
    """The fused step under B2L_F_ROW_POS with a different adapter per row (and -1 rows): each row's prefill and
    decode logits equal a batch-1 model carrying only that adapter, bit for bit, eager and graph-replayed; then one
    row is refilled with another adapter between replays (the graph stays) and follows that adapter's model."""
    B, S = len(ads), 48
    prompts = _prompts(dev, B, seed=B + len(cfg))
    toks = [77, 12, 9, 150, 42, 5]
    new_a = (ads[0] + 2) % 4 if ads[0] >= 0 else 1
    p = _prompts(dev, 1, seed=99)[0]
    # the batch-1 references first: loading a model bumps the weight generation, which rebuilds every decode state
    check = [b for b, a in enumerate(ads) if b <= 4 or a not in ads[:b] or mode == "llm.int8"]
    wants = {b: _batch1(dev, mode, cfg, ads[b], prompts[b], toks, S, compact) for b in check}
    want_refill = _batch1(dev, mode, cfg, new_a, p, toks[:3], S, compact)
    m = _multi(dev, mode, cfg, 3, compact)
    with torch.no_grad():
        got = [m.prefill_rows(prompts, S, ads)]
        pos = torch.tensor([p.numel() for p in prompts], device=dev).view(B, 1)
        for i, t in enumerate(toks):
            got.append(m(torch.full((B, 1), t, device=dev), S, pos + i)[:, -1])
    torch.cuda.synchronize()
    st = m._decode
    assert st is not None and st.lora_rows is not None and st.graph is not None and st.args.n_lora_sets == 4
    assert not st.args.loras
    bar = 6e-2 if mode == "llm.int8" else 0   # llm.int8's batched rows share the outlier mask (its B >= 2 bar)
    for b in check:   # every row up to 4, then one per adapter
        a = ads[b]
        for step, (g, w) in enumerate(zip(got, wants[b])):
            if bar == 0:
                assert torch.equal(g[b], w), (b, a, step)
            else:
                assert float((g[b].float() - w.float()).norm() / w.float().norm()) < bar, (b, a, step)
    # row 0 takes a new prompt and adapter between two replays
    with torch.no_grad():
        first = m.refill_rows([p], [0], S, [new_a])[0]
        pos[0, 0] = p.numel() - len(toks)
        more = [m(torch.full((B, 1), t, device=dev), S, pos + len(toks) + i)[0, -1] for i, t in enumerate(toks[:3])]
    assert m._decode is st and st.graph is not None
    for step, (g, w) in enumerate(zip([first] + more, want_refill)):
        if bar == 0:
            assert torch.equal(g, w), ("refill", step)
        else:
            assert float((g.float() - w.float()).norm() / w.float().norm()) < bar


def test_stream_and_prompts_equal_generate(dev):
    """generate_stream on 3 rows over 8 prompts and 4 adapters (-1 included), refills in packed passes and alone,
    top_k=1: each prompt's tokens equal generate() on the batch-1 model carrying its adapter; generate_prompts the
    same for the first prompts."""
    m = _multi(dev, "gptq.int4", TINY, 2)
    lengths = (3, 17, 1, 9, 40, 2, 16, 5)
    g = torch.Generator().manual_seed(8)
    prompts = [torch.randint(0, 256, (n,), generator=g).to(torch.int32).to(dev) for n in lengths]
    ads = [0, 1, -1, 2, 1, -1, 0, 2]
    news = [6, 3, 7, 4, 5, 6, 3, 4]
    st = {}
    ys = P.generate_stream(m, prompts, news, batch_size=3, top_k=1, max_seq_length=48, adapters=ads, stats=st)
    assert st["refills"] == 5 and st["packed"] > 0
    m.reset_cache()
    ref = {}
    for i, (p, a) in enumerate(zip(prompts, ads)):
        if a not in ref:
            ref[a] = _model(dev, "gptq.int4", TINY, None if a < 0 else _lw(TINY, a))
        ref[a].reset_cache()
        want = P.generate(ref[a], p, news[i], max_seq_length=48, top_k=1)
        assert torch.equal(ys[i], want), (i, a)
    ys2 = P.generate_prompts(m, prompts[:5], 4, top_k=1, max_seq_length=48, adapters=ads[:5])
    for i in range(5):
        ref[ads[i]].reset_cache()
        assert torch.equal(ys2[i], P.generate(ref[ads[i]], prompts[i], 4, max_seq_length=48, top_k=1)), i
    m.reset_cache()
    assert m._lora_route is None


@pytest.mark.parametrize("mode", ["gptq.int8", "llm.int8"])
def test_module_route_within_its_bar(dev, mode):
    """gptq.int8 without w8_batch_step and llm.int8 without int8_step decode module by module: c_attn adds each row's
    adapter with b2l_lora_apply_rows.  Rows within the bars those routes' B >= 2 tests hold against batch 1."""
    m = _multi(dev, mode, TINY, 2)
    m.w8_batch_step = m.int8_step = False
    ads = [2, -1, 0, 1]
    B, S = len(ads), 48
    prompts = _prompts(dev, B, seed=5)
    toks = [7, 99, 31, 4]
    with torch.no_grad():
        got = [m.prefill_rows(prompts, S, ads)]
        pos = torch.tensor([p.numel() for p in prompts], device=dev).view(B, 1)
        for i, t in enumerate(toks):
            got.append(m(torch.full((B, 1), t, device=dev), S, pos + i)[:, -1])
    assert m._decode is None and m._module_graph is not None and m._module_graph["graph"] is not None
    bar = 6e-2 if mode == "llm.int8" else 2e-2
    for b, a in enumerate(ads):
        want = _batch1(dev, mode, TINY, a, prompts[b], toks, S)
        assert torch.equal(got[0][b], want[0]) or mode == "llm.int8"   # the prefill is batch 1 on both sides
        for g, w in zip(got, want):
            assert float((g[b].float() - w.float()).norm() / w.float().norm()) < bar


def test_memory_is_the_adapters_bytes(dev):
    """Adding n adapters grows the allocated memory by their lora_A + lora_B bytes only (the caching allocator's
    512-byte granules aside): no second base copy, and decoding with one adapter per row copies no weight."""
    m = _multi(dev, "gptq.int4", W13B, 0, compact=True)
    torch.cuda.synchronize()
    a0 = torch.cuda.memory_allocated()
    want = 0
    for k in range(1, 5):
        lw = _lw(W13B, k)
        PL.add_lora_adapter(m, lw)
        want += sum(-(-v.numel() * 2 // 512) * 512 for v in lw.values())
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - a0 == want
    prompts = _prompts(dev, 5, seed=3)
    with torch.no_grad():
        m.prefill_rows(prompts, 48, [0, 1, 2, 3, 4])
        pos = torch.tensor([p.numel() for p in prompts], device=dev).view(5, 1)
        for i in range(3):   # two eager steps, then the graph is captured
            m(torch.full((5, 1), 3, device=dev), 48, pos + i)
        torch.cuda.synchronize()
        a1 = torch.cuda.memory_allocated()
        for i in range(3, 6):
            m(torch.full((5, 1), 3, device=dev), 48, pos + i)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == a1   # steady decode allocates nothing per step
    c = m.transformer.h[0].attn.c_attn
    A, B_, _, _ = c._adapters[0]
    spec = m._decode.args.lora_sets[1 * W13B["n_layer"] + 0]
    assert spec.A == A.data_ptr() and spec.B == B_.data_ptr()   # the step reads the registered tensors in place

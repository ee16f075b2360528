"""GPU: LoRA inference (lit_llama_b200.lora).  b2l_lora_apply against the oracle's restatement of the reference's
unmerged branch; gptq.int4 / gptq.int8 / llm.int8 LoRA models against the oracle on every decode path (fused step,
module path, CUDA graphs); zero lora_B = the plain model bit for bit; compact(); reloading LoRA weights after graph
capture; and the dense model through patch_reference() against the unmodified reference's fixture."""
import ctypes as C
import json
import os
import sys
import types
from contextlib import nullcontext

import pytest
import torch

from conftest import load_golden

import lit_llama_b200 as P
from lit_llama_b200 import _lib as L
from lit_llama_b200 import lora as PL
from lit_llama_b200.utils import quantization
from oracle import llama_oracle as O
from oracle import lora_oracle as LO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    return torch.device("cuda", 0)


def _apply(dev, y, x, A, B, scaling, n_groups, mask, norm=None, flags=0):
    r = A.shape[0] // bin(mask).count("1")
    spec = L.LoRA(A.data_ptr(), B.data_ptr(), scaling, r, n_groups, mask)
    M, K = x.shape
    N = y.shape[1]
    rc = L.lib().b2l_lora_apply(C.byref(spec), x.data_ptr(), K, None if norm is None else norm.data_ptr(), 1e-5,
                                y.data_ptr(), N, M, N, K, flags, L.stream_ptr())
    L.check(rc, "b2l_lora_apply")
    torch.cuda.synchronize()
    return y


def _ulp(v: torch.Tensor) -> torch.Tensor:
    """bf16 spacing at |v| (8 significant bits), taken one step up so a value that rounds across a power of two is
    covered; a tiny floor for zeros."""
    a = (v.float().abs() * (1 + 2 ** -7)).clamp_min(2 ** -120)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _pad(t: torch.Tensor, enable) -> torch.Tensor:
    n_g = t.shape[-1] // sum(enable)
    out = t.new_zeros((*t.shape[:-1], n_g * len(enable)))
    ind = torch.tensor(enable).repeat_interleave(n_g)
    out[..., ind] = t
    return out


def _want_and_bound(xh, y0, A, B, s, enable):
    """The oracle's output (the reference's unmerged branch, lora.py:313-325) and the most a rounding-boundary flip can
    move each element.  The kernel and the CPU accumulate u = A.xh in fp32 in different orders, so where the exact sum
    lies on a bf16 rounding boundary u_j may come out one bf16 ulp apart.  That moves the exact d_n = sum_j B_nj u_j by
    at most D_n = sum_j |B_nj| ulp(u_j); its bf16 rounding by at most one more ulp(d_n); the term bf16(d * s) by at
    most s (D_n + ulp(d_n)) + ulp(term_n); and the output bf16(y + term) by that plus ulp(y_out).  A 2^-16 share of
    s sum_j |B_nj u_j| covers the two fp32 accumulation orders of d.  Elements of disabled groups get no allowance: they
    must be untouched."""
    n_on = sum(enable)
    want = LO.lora_branch(xh, y0, A, B, s, enable)
    u = torch.nn.functional.linear(xh, A)
    d = torch.nn.functional.conv1d(u.transpose(-2, -1), B.unsqueeze(-1), groups=n_on).transpose(-2, -1)
    term = d * s

    def conv_abs(v):
        return torch.nn.functional.conv1d(v.transpose(-2, -1), B.float().abs().unsqueeze(-1), groups=n_on).transpose(-2, -1)

    flip = s * (conv_abs(_ulp(u)) + _ulp(d)) + _ulp(term) + 2 ** -16 * s * conv_abs(u.float().abs())
    on = _pad(torch.ones_like(term, dtype=torch.float32), enable)
    return want, _pad(flip, enable) + on * _ulp(want)


def _check_rows(got, y0, candidates):
    """Every row of `got` within the flip bound of one candidate (want, bound), and the term not vacuous."""
    got = got.float().cpu()
    ok = torch.zeros(got.shape[0], dtype=torch.bool)
    for want, bound in candidates:
        ok |= ((got - want.float()).abs() <= bound).all(dim=-1)
    assert ok.all(), f"rows outside the rounding-flip bound: {(~ok).nonzero().flatten().tolist()[:8]}"
    assert not torch.equal(got, y0.float())   # the term is not vacuous


def _rms_candidates(x, sc, eps=1e-5):
    """rms_1(x) as model.py:270-277 evaluates it in bf16 (O.rmsnorm), and the same with the row's bf16 rinv one ulp up
    or down: rinv = bf16(rsqrt(bf16(mean(bf16(x x)) + eps))) is itself a rounded fp32 reduction, so the kernel's sum
    order may land it on the neighbouring value, which rescales the whole row."""
    rinv = torch.rsqrt(torch.mean(x * x, dim=-1, keepdim=True) + eps)
    assert torch.equal(sc * (x * rinv), O.rmsnorm(x, sc))
    bits = rinv.view(torch.int16)
    return [sc * (x * r) for r in (rinv, (bits + 1).view(torch.bfloat16), (bits - 1).view(torch.bfloat16))]


@pytest.mark.parametrize("C_", [4096, 5120, 8192])
@pytest.mark.parametrize("r", [1, 8, 64])
@pytest.mark.parametrize("M", [1, 2, 5, 16, 512])
def test_lora_kernel_vs_oracle(dev, C_, r, M):
    """7B / 13B / 65B c_attn widths, q and v: with and without the RMSNorm prologue, with and without PDL.  The
    residual rows have an RMS of about 8 and the norm scale spans 0.25..1.75, so rms_1(x) is far from x; every output
    must sit within the rounding-flip bound of _want_and_bound."""
    g = torch.Generator().manual_seed(C_ * 131 + r * 7 + M)
    N = 3 * C_
    x = (torch.randn(M, C_, generator=g) * 8).to(torch.bfloat16)
    y0 = (torch.randn(M, N, generator=g) * 0.5).to(torch.bfloat16)
    A = ((torch.rand(2 * r, C_, generator=g) * 2 - 1) / C_ ** 0.5).to(torch.bfloat16)
    B = (torch.randn(2 * C_, r, generator=g) * 0.05).to(torch.bfloat16)
    sc = (0.25 + 1.5 * torch.rand(C_, generator=g)).to(torch.bfloat16)
    s = 16 / r
    for norm in (False, True):
        xhs = _rms_candidates(x, sc) if norm else [x]
        cands = [_want_and_bound(xh, y0, A, B, s, LO.QV) for xh in xhs]
        for flags in (0, 1):
            got = _apply(dev, y0.to(dev), x.to(dev), A.to(dev), B.to(dev), s, 3, 0b101,
                         norm=sc.to(dev) if norm else None, flags=flags)
            _check_rows(got, y0, cands)


@pytest.mark.parametrize("enable", [[True, True, True], [False, True, False], [True, False, False, True],
                                    [False, False, True, True, False, False, True, False]])
def test_lora_kernel_group_patterns(dev, enable):
    g = torch.Generator().manual_seed(len(enable) * 17 + sum(enable))
    K, N, r, M = 512, 1024 if len(enable) != 3 else 1536, 4, 7
    n_on = sum(enable)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    y0 = (torch.randn(M, N, generator=g) * 0.5).to(torch.bfloat16)
    A = ((torch.rand(r * n_on, K, generator=g) * 2 - 1) / K ** 0.5).to(torch.bfloat16)
    B = (torch.randn(N // len(enable) * n_on, r, generator=g) * 0.05).to(torch.bfloat16)
    mask = sum(1 << i for i, e in enumerate(enable) if e)
    got = _apply(dev, y0.to(dev), x.to(dev), A.to(dev), B.to(dev), 1.5, len(enable), mask)
    _check_rows(got, y0, [_want_and_bound(x, y0, A, B, 1.5, enable)])
    # the disabled groups are not touched (their bound is 0 too)
    off = torch.tensor(enable).repeat_interleave(N // len(enable)).logical_not()
    assert torch.equal(got.cpu()[:, off], y0[:, off])


CFG = dict(block_size=64, vocab_size=256, n_layer=3, n_head=4, n_embd=512)
PROMPT = torch.tensor([5, 100, 3, 7, 200, 9, 31])
TOKS = [77, 12, 9, 150, 42]


def build(dev, mode, cfg=CFG, zero_b=False, lora_seed=4321, plain=False, exact_linears=True):
    sd = O.synth_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"],
                            None if mode == "llm.int8" else mode)
    lw = LO.lora_weights(cfg["n_layer"], cfg["n_embd"], seed=lora_seed, zero_b=zero_b)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization(mode), (nullcontext() if plain else PL.lora(r=8, alpha=16, dropout=0.05)):
            model = P.LLaMA(P.LLaMAConfig(**cfg))
    finally:
        torch.set_default_dtype(prev)
    full = sd if plain else dict(sd, **lw)
    res = model.load_state_dict(full)
    assert not res.missing_keys and not res.unexpected_keys
    oracle = LO.from_state_dict(full, cfg["n_layer"], cfg["n_head"], cfg["block_size"], mode, exact_linears=exact_linears)
    return model.eval(), oracle, lw


def run(model, dev, B=1, S=32, prompt=PROMPT, toks=TOKS):
    T = prompt.numel()
    with torch.no_grad():
        out = [model(prompt.view(1, -1).repeat(B, 1).to(dev), S, torch.arange(T, device=dev))]
        for i, t in enumerate(toks):
            out.append(model(torch.full((B, 1), t, device=dev), S, torch.tensor([T + i], device=dev)))
    torch.cuda.synchronize()
    return out


def want_of(oracle, B=1, S=32, prompt=PROMPT, toks=TOKS):
    T = prompt.numel()
    oracle.reset_cache()
    out = [oracle.forward(prompt.view(1, -1).repeat(B, 1), S, torch.arange(T))]
    for i, t in enumerate(toks):
        out.append(oracle.forward(torch.full((B, 1), t), S, torch.tensor([T + i])))
    return out


def close(got, want, bar=2e-2):
    for a, b in zip(got, want):
        a, b = a.float().cpu(), b.float().cpu()
        assert float((a - b).norm() / b.norm()) < bar


def test_tiny_gptq_int4_lora_model_vs_oracle(dev):
    """The tiny model of the existing tests (head_size 32) under gptq.int4 with LoRA in every layer, at their bars
    (rtol 1e-3, atol 5e-3 against the oracle's reference arithmetic): prefill, eager and graph-replayed decode on the
    fused step, the roll branch, the no-cache forward and greedy tokens."""
    cfg = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)
    prompt, toks = torch.tensor([3, 17, 40, 41, 2, 77, 5]), [11, 5, 90, 33]
    for graph_after in (0, 2):
        model, oracle, _ = build(dev, "gptq.int4", cfg, exact_linears=False)
        model.graph_after = graph_after
        got = run(model, dev, S=16, prompt=prompt, toks=toks)
        assert model._decode is not None and model._decode.args.loras
        assert (model._decode.graph is not None) == (graph_after > 0)
        for a, b in zip(got, want_of(oracle, S=16, prompt=prompt, toks=toks)):
            torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    roll = [x[:, -1] for x in run(model, dev, S=8, prompt=prompt, toks=[3, 17, 40, 41, 2, 77])]
    want = [x[:, -1] for x in want_of(oracle, S=8, prompt=prompt, toks=[3, 17, 40, 41, 2, 77])]
    for a, b in zip(roll, want):
        torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    oracle.reset_cache()
    with torch.no_grad():
        nc = model(prompt.view(1, -1).to(dev))
    torch.testing.assert_close(nc.float().cpu(), oracle.forward(prompt.view(1, -1)).float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    oracle.reset_cache()
    oracle.block_size = cfg["block_size"]
    greedy = P.generate(model, prompt.to(torch.int32).to(dev), 12, top_k=1).cpu()
    assert (greedy == O.generate(oracle, prompt.to(torch.int32), 12, top_k=1)).float().mean() >= 0.9


@pytest.mark.parametrize("mode,B,fused", [("gptq.int4", 1, True), ("gptq.int4", 4, True), ("gptq.int8", 1, True),
                                          ("gptq.int8", 2, False), ("llm.int8", 2, False), ("llm.int8", 1, False)])
def test_lora_model_paths_vs_oracle_and_zero_b(dev, mode, B, fused):
    """head_size 128: the fused step (LoRA launch between c_attn and the attention) or the module path, under the
    graph, against the oracle; the fused step against the module path on the same model; zero lora_B (the
    reference's initial state) gives the plain model's logits bit for bit."""
    model, oracle, _ = build(dev, mode)
    model.graph_after = 2
    got = run(model, dev, B)
    assert (model._decode is not None) == fused
    if fused:
        assert L.lib().b2l_decode_step_launches(C.byref(model._decode.args)) == 5 * CFG["n_layer"] + 3 + CFG["n_layer"] + \
            (CFG["n_layer"] * 4 + 1 if 1 < B <= 8 else 0)   # the 2..8-row kernel is two launches per linear
    # llm.int8: the bar of the existing llm.int8 model tests (its restatement is parity-unpinned, DESIGN.md Numerics)
    bar = 6e-2 if mode == "llm.int8" else 2e-2
    close(got, want_of(oracle, B), bar)
    if fused:   # the module path on the same model (no fused step) gives the same numbers up to rounding
        model.reset_cache()
        model._fast_ok = False
        mod = run(model, dev, B)
        assert model._decode is None
        close(got, mod, 5e-3)
    plain, _, _ = build(dev, mode, plain=True)
    plain.graph_after = 2
    want = run(plain, dev, B)
    assert not torch.equal(got[-1], want[-1])
    zero, _, _ = build(dev, mode, zero_b=True)
    zero.graph_after = 2
    for a, b in zip(run(zero, dev, B), want):
        assert torch.equal(a, b)
    with torch.no_grad():
        model.reset_cache()
        nc = model(PROMPT.view(1, -1).to(dev))
        zero.reset_cache()
        plain.reset_cache()
        assert torch.equal(zero(PROMPT.view(1, -1).to(dev)), plain(PROMPT.view(1, -1).to(dev)))
    oracle.reset_cache()
    close([nc], [oracle.forward(PROMPT.view(1, -1))], bar)


def test_lora_reload_after_graph_and_compact(dev):
    """Loading new LoRA weights after the decode graph was captured takes effect at the next step; compact() changes
    no output and no state_dict entry."""
    model, oracle, _ = build(dev, "gptq.int4")
    model.graph_after = 2
    run(model, dev)
    assert model._decode.graph is not None
    before = model(torch.tensor([[88]], device=dev), 32, torch.tensor([7 + len(TOKS)], device=dev)).clone()
    model.reset_cache()
    run(model, dev)
    _, o2, lw2 = build(dev, "gptq.int4", lora_seed=999)
    model.load_state_dict(lw2, strict=False)
    with torch.no_grad():
        got = model(torch.tensor([[88]], device=dev), 32, torch.tensor([7 + len(TOKS)], device=dev))
    assert not torch.equal(got, before)
    want_of(oracle)   # the history with the old LoRA weights, then the new ones
    for lay, lay2 in zip(oracle.layers, o2.layers):
        lay["c_attn"] = lay2["c_attn"]
    want = oracle.forward(torch.tensor([[88]]), 32, torch.tensor([7 + len(TOKS)]))
    close([got], [want])
    ref, _, _ = build(dev, "gptq.int4")
    ref.graph_after = 2
    a = run(ref, dev)
    sd0 = {k: v.clone() for k, v in ref.state_dict().items()}
    cm, _, _ = build(dev, "gptq.int4")
    cm.graph_after = 2
    cm.compact()
    assert cm.transformer.h[0].attn.c_attn._released
    for x, y in zip(a, run(cm, dev)):
        assert torch.equal(x, y)
    sd1 = cm.state_dict()
    assert set(sd1) == set(sd0) and all(torch.equal(sd1[k], sd0[k]) for k in sd0)
    # LoRA-only reload into the compacted, graph-captured model: the base keeps its only copy, the step follows
    cm.reset_cache()
    run(cm, dev)
    cm.load_state_dict(lw2, strict=False)
    assert cm.transformer.h[0].attn.c_attn._released
    with torch.no_grad():
        got_c = cm(torch.tensor([[88]], device=dev), 32, torch.tensor([7 + len(TOKS)], device=dev))
    assert torch.equal(got_c, got)


def test_dense_lora_through_patch_reference_matches_reference(dev):
    """generate/lora.py's flow on a dense base through patch_reference(): lora() (the name the script bound) builds
    LoRA layers, base then LoRA checkpoint (strict=False), eval() merges; the tiny model against the unmodified
    reference's logits and tokens at the existing dense tests' bars.  The unmerged dense forward (train mode, the
    LoRA kernel) matches the reference's stand-alone MergedLinear."""
    g = load_golden("tiny_lora_bf16.pt")
    gd = os.path.join(ROOT, "tests", "golden")
    surface = json.load(open(os.path.join(gd, "reference_surface.json")))["modules"]
    surface.update(json.load(open(os.path.join(gd, "reference_lora_surface.json")))["modules"])
    pkg = "lit_llama_lora_gpu"
    names = {"pkg": pkg, "model": pkg + ".model", "quant": pkg + ".quantization", "utils": pkg + ".utils",
             "generate": pkg + "_generate", "lora": pkg + ".lora", "generate_lora": pkg + "_generate_lora"}
    mods = {key: types.ModuleType(name) for key, name in names.items()}
    objs = {}
    for key, ns in surface.items():
        for name, origin in ns.items():
            setattr(mods[key], name, objs.setdefault(origin, type(name, (), {})))
    sys.modules.update({mod.__name__: mod for mod in mods.values()})
    try:
        P.patch_reference(mods["pkg"])
        script = mods["generate_lora"]
        c = g["cfg"]
        sd = O.synth_state_dict(c["n_layer"], c["n_head"], c["n_embd"], c["vocab_size"], None, seed=g["seed"])
        lw = LO.lora_weights(c["n_layer"], c["n_embd"], r=g["lora"]["r"], seed=g["lora_seed"])
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.bfloat16)
        try:
            with torch.device(dev), script.lora(r=8, alpha=16, dropout=0.05, enabled=True):
                model = script.LLaMA(P.LLaMAConfig(**c))
        finally:
            torch.set_default_dtype(prev)
        model.load_state_dict(sd, strict=False)
        assert not model.load_state_dict(lw, strict=False).unexpected_keys
        model.eval()
    finally:
        for mod in mods.values():
            sys.modules.pop(mod.__name__, None)
    for blk, w in zip(model.transformer.h, g["merged_c_attn"]):
        assert blk.attn.c_attn.merged
        assert torch.equal(blk.attn.c_attn.weight.cpu(), w) or \
            float((blk.attn.c_attn.weight.float().cpu() - w.float()).abs().max()) <= 2 ** -8 * float(w.float().abs().max())
    p = g["prompt"]
    got = run(model, dev, S=16, prompt=p, toks=g["steps_tokens"])
    for a, b in zip(got, g["steps_logits"]):
        torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    greedy = P.generate(model, p.to(torch.int32).to(dev), 12, top_k=1).cpu()
    assert (greedy == g["gen_greedy"]).float().mean() >= 0.9
    # the unmerged dense forward: base linear + the LoRA kernel, against the reference's MergedLinear
    for case in g["merged_linear_cases"]:
        lin = PL.MergedLinear(case["in_features"], case["out_features"], r=case["r"], lora_alpha=case["alpha"],
                              lora_dropout=0.0, enable_lora=case["enable_lora"], bias=False).to(dev, torch.bfloat16)
        with torch.no_grad():
            lin.weight.copy_(case["weight"])
            lin.lora_A.copy_(case["lora_A"])
            lin.lora_B.copy_(case["lora_B"])
            out = lin(case["x"].to(dev))
        assert not lin.merged
        torch.testing.assert_close(out.float().cpu(), case["y"].float(), rtol=2 ** -7, atol=2e-2)

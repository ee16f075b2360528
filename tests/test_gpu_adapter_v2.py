"""GPU: LLaMA-Adapter v2 inference (lit_llama_b200.adapter_v2) - b2l_linear_affine against torch, the batch-1 kernels'
out_affine epilogue against the plain kernel plus the stand-alone ops, the tiny model against the unmodified
reference's fixture, every mode and path against the v2 oracle, the fused step against the module path, identity
affines against the v1-adapter model bit for bit, compact() and reloading after graph capture."""
import ctypes as C
import json
import os
import sys
import types

import pytest
import torch

from conftest import load_golden

import lit_llama_b200 as P
from lit_llama_b200 import _lib as L
from lit_llama_b200 import adapter as PA
from lit_llama_b200 import adapter_v2 as PV
from lit_llama_b200.utils import quantization
from oracle import adapter_v2_oracle as A2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    return torch.device("cuda", 0)


def _rand_affine(N, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    s = ((torch.rand(N, generator=g, device=dev) + 0.5) * torch.where(torch.rand(N, generator=g, device=dev) < 0.5, -1.0, 1.0))
    b = torch.randn(N, generator=g, device=dev) * 0.5
    return s.to(torch.bfloat16), b.to(torch.bfloat16)


@pytest.mark.parametrize("M", [1, 7, 512])
@pytest.mark.parametrize("N,pad", [(4096, 0), (11008, 8), (32000, 0), (100, 0), (96, 3)])
def test_linear_affine_matches_torch(dev, M, N, pad):
    g = torch.Generator(device=dev).manual_seed(M * 31 + N)
    ld = N + pad
    buf = (torch.randn(M, ld, generator=g, device=dev) * 2).to(torch.bfloat16)
    s, b = _rand_affine(N, dev, N + M)
    want = buf.clone()
    want[:, :N] = s * (buf[:, :N] + b)
    got = buf.clone()
    L.check(L.lib().b2l_linear_affine(got.data_ptr(), ld, M, N, s.data_ptr(), b.data_ptr(), L.stream_ptr()), "affine")
    torch.cuda.synchronize()
    assert torch.equal(got, want)   # the padding columns are untouched too


def _gemv(bits, x, qt, sc, z, N, K, *, epilogue=0, res=None, aff=None, n_out=None):
    n_out = n_out or N
    y = torch.zeros((1, n_out), device=x.device, dtype=torch.bfloat16)
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                       sz_dtype=L.sz_dtype_of(sc), y=y.data_ptr(), ldy=n_out, M=1, N=N, K=K, prologue=0, eps=1e-5,
                       epilogue=epilogue, res=None if res is None else res.data_ptr(), ldres=N, split_k=0, flags=0)
    if aff is not None:
        a.out_affine = L.OutAffine(aff[0].data_ptr(), aff[1].data_ptr())
    fn = "b2l_w8_gemv" if bits == 8 else "b2l_q4_gemv"
    L.check(getattr(L.lib(), fn)(C.byref(a), L.stream_ptr()), fn)
    return y


def _affine(y, aff):
    y = y.clone()
    L.check(L.lib().b2l_linear_affine(y.data_ptr(), y.shape[-1], 1, y.shape[-1], aff[0].data_ptr(), aff[1].data_ptr(),
                                      L.stream_ptr()), "affine")
    return y


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K", [(12288, 4096), (4096, 11008), (32000, 4096), (27648, 5120), (8192, 22016), (16384, 8192)])
def test_gemv_out_affine_epilogues(dev, bits, N, K):
    """7B / 13B / 65B shapes (lm_head, K > 12288): STORE = plain kernel + b2l_linear_affine; RESIDUAL = that + b2l_add;
    SWIGLU = STORE-with-affine on the interleaved weight, de-interleaved, + b2l_silu_mul.  All bit for bit."""
    from lit_llama_b200.quantization import tile_i8

    g = torch.Generator(device=dev).manual_seed(N + K + bits)
    epb = 8 // bits
    qw = torch.randint(0, 256, (K // epb, N), generator=g, device=dev, dtype=torch.uint8).t()
    qt = tile_i8(qw, N, K, bits)
    lv = 2 ** bits
    sc = ((torch.rand(N, 1, generator=g, device=dev) + 0.5) / (0.3 * lv * K ** 0.5)).to(torch.bfloat16)
    z = torch.randint(lv // 2 - lv // 8, lv // 2 + lv // 8, (N, 1), generator=g, device=dev).to(torch.bfloat16)
    x = torch.randn(1, K, generator=g, device=dev).to(torch.bfloat16)
    aff = _rand_affine(N, dev, N * 3 + K)
    plain = _gemv(bits, x, qt, sc, z, N, K)
    want = _affine(plain, aff)
    got = _gemv(bits, x, qt, sc, z, N, K, aff=aff)
    torch.cuda.synchronize()
    assert torch.equal(got, want) and not torch.equal(got, plain)
    res = torch.randn(1, N, generator=g, device=dev).to(torch.bfloat16)
    want_r = torch.empty_like(res)
    L.check(L.lib().b2l_add(want.data_ptr(), res.data_ptr(), want_r.data_ptr(), N, L.stream_ptr()), "add")
    got_r = _gemv(bits, x, qt, sc, z, N, K, epilogue=1, res=res, aff=aff)
    torch.cuda.synchronize()
    assert torch.equal(got_r, want_r)
    # SWIGLU: rows of a 16-row block are [8 of a | 8 of b]; the vectors are interleaved the same way
    ab = want.view(N // 16, 2, 8)
    a_, b_ = ab[:, 0].reshape(1, N // 2).contiguous(), ab[:, 1].reshape(1, N // 2).contiguous()
    want_s = torch.empty_like(a_)
    L.check(L.lib().b2l_silu_mul(a_.data_ptr(), b_.data_ptr(), want_s.data_ptr(), N // 2, L.stream_ptr()), "silu_mul")
    got_s = _gemv(bits, x, qt, sc, z, N, K, epilogue=2, aff=aff, n_out=N // 2)
    torch.cuda.synchronize()
    assert torch.equal(got_s, want_s)


# ------------------------------------------------------------------ models
CFG128 = dict(block_size=64, vocab_size=256, n_layer=3, n_head=4, n_embd=512, adapter_prompt_length=10, adapter_start_layer=1)
PROMPT = torch.tensor([5, 100, 3, 7, 200, 9, 31])
TOKS = [77, 12, 9, 150, 42]


def build(dev, cfg, mode, *, identity=False, v2=True, v2_seed=2468, exact_linears=True):
    """generate/adapter_v2.py's construction sequence: adapter.LLaMA and add_adapter_v2_parameters_to_linear_layers
    under quantization(mode), then the base checkpoint and the adapter checkpoint, both strict=False.  v2=False: the
    v1-adapter model on the same weights (without the affines)."""
    sd = A2.adapter_v2_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"],
                                  None if mode == "llm.int8" else mode, cfg["adapter_prompt_length"],
                                  cfg["adapter_start_layer"], v2_seed=v2_seed, identity=identity)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization(mode):
            model = PA.LLaMA(PA.LLaMAConfig(**cfg))
            if v2:
                PV.add_adapter_v2_parameters_to_linear_layers(model)
    finally:
        torch.set_default_dtype(prev)
    if not v2:
        sd = {k: v for k, v in sd.items() if ".adapter_scale" not in k and ".adapter_bias" not in k}
    ada = PV.adapter_v2_state_from_state_dict(sd)
    assert not model.load_state_dict({k: v for k, v in sd.items() if k not in ada}, strict=False).unexpected_keys
    res = model.load_state_dict(ada, strict=False)
    assert not res.unexpected_keys
    oracle = A2.OracleAdapterV2LLaMA.from_state_dict(sd, cfg["n_layer"], cfg["n_head"], cfg["block_size"], mode,
                                                     exact_linears=exact_linears)
    return model.eval(), oracle, sd


def run(model, dev, B=1, S=32, prompt=PROMPT, toks=TOKS):
    with torch.no_grad():
        idx = prompt.view(1, -1).repeat(B, 1).to(dev)
        out = [model(idx, S, torch.arange(prompt.numel(), device=dev))]
        for i, t in enumerate(toks):
            out.append(model(torch.full((B, 1), t, device=dev), S, torch.tensor([prompt.numel() + i], device=dev)))
    torch.cuda.synchronize()
    return out


def want_of(oracle, B=1, S=32):
    oracle.reset_cache()
    idx = PROMPT.view(1, -1).repeat(B, 1)
    want = [oracle.forward(idx, S, torch.arange(7))]
    for i, t in enumerate(TOKS):
        want.append(oracle.forward(torch.full((B, 1), t), S, torch.tensor([7 + i])))
    return want


def close(got, want, bar=2e-2):
    for a, b in zip(got, want):
        a, b = a.float().cpu(), b.float()
        assert float((a - b).norm() / b.norm()) < bar


def rel(got, want):
    return max(float((a.float() - b.float()).norm() / b.float().norm()) for a, b in zip(got, want))


@pytest.mark.parametrize("base,graph_after", [("gptq.int4", 0), ("gptq.int4", 2), ("dense", 0), ("dense", 2)])
def test_tiny_adapter_v2_model_matches_reference(dev, base, graph_after):
    """The reference's construction sequence through patch_reference() (the names generate/adapter_v2.py bound)
    against the unmodified reference's logits and tokens."""
    g = load_golden("tiny_adapter_v2_bf16.pt")
    c, want = g["cfg"], g["bases"][base]
    mode = None if base == "dense" else base
    gd = os.path.join(ROOT, "tests", "golden")
    surface = json.load(open(os.path.join(gd, "reference_surface.json")))["modules"]
    for f in ("reference_adapter_surface.json", "reference_adapter_v2_surface.json"):
        surface.update(json.load(open(os.path.join(gd, f)))["modules"])
    pkg = "lit_llama_adapter_v2_gpu"
    names = {"pkg": pkg, "model": pkg + ".model", "quant": pkg + ".quantization", "utils": pkg + ".utils",
             "generate": pkg + "_generate", "adapter": pkg + ".adapter", "generate_adapter": pkg + "_generate_adapter",
             "adapter_v2": pkg + ".adapter_v2", "generate_adapter_v2": pkg + "_generate_adapter_v2"}
    mods = {key: types.ModuleType(name) for key, name in names.items()}
    objs = {}
    for key, ns in surface.items():
        for name, origin in ns.items():
            setattr(mods[key], name, objs.setdefault(origin, type(name, (), {})))
    sys.modules.update({mod.__name__: mod for mod in mods.values()})
    try:
        P.patch_reference(mods["pkg"])
        script = mods["generate_adapter_v2"]
        sd = A2.adapter_v2_state_dict(c["n_layer"], c["n_head"], c["n_embd"], c["vocab_size"], mode,
                                      c["adapter_prompt_length"], c["adapter_start_layer"], seed=g["seed"],
                                      adapter_seed=g["adapter_seed"], v2_seed=g["v2_seed"])
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.bfloat16)
        try:
            with torch.device(dev), script.quantization(mode):
                model = script.LLaMA(mods["adapter"].LLaMAConfig(**c))
                script.add_adapter_v2_parameters_to_linear_layers(model)
        finally:
            torch.set_default_dtype(prev)
        ada = mods["adapter_v2"].adapter_v2_state_from_state_dict(sd)
        model.load_state_dict({k: v for k, v in sd.items() if k not in ada}, strict=False)
        assert not model.load_state_dict(ada, strict=False).unexpected_keys
        model.eval()
    finally:
        for mod in mods.values():
            sys.modules.pop(mod.__name__, None)
    model.graph_after = graph_after
    p = want["prompt"]
    got = run(model, dev, S=16, prompt=p, toks=want["steps_tokens"])
    assert (model._decode is not None) == (base == "gptq.int4")
    for a, b in zip(got, want["steps_logits"]):
        torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    with torch.no_grad():
        nc = model(p.view(1, -1).to(dev))
    torch.testing.assert_close(nc.float().cpu(), want["nocache_logits"].float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    roll = [x[:, -1] for x in run(model, dev, S=8, prompt=p, toks=want["roll_tokens"])]
    # a dense base runs its linears on torch's GEMM, which accumulates in another order than the reference's CPU run:
    # a one-ulp flip early in the 13 positions of the roll, carried through every linear's scale (|s| up to 1.5), was
    # measured at 3 bf16 ulps in one of 96 logits (0.0059 at 0.34), so the roll there gets twice the absolute bar
    atol = 1e-2 if base == "dense" else 5e-3
    for a, b in zip(roll, want["roll_logits"]):
        torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=atol)
    model.reset_cache()
    greedy = P.generate(model, p.to(torch.int32).to(dev), 12, top_k=1).cpu()
    assert (greedy == want["gen_greedy"]).float().mean() >= 0.9


@pytest.mark.parametrize("mode,B,fused", [("gptq.int4", 1, True), ("gptq.int4", 4, False), ("gptq.int8", 1, True),
                                          ("gptq.int8", 2, False), ("llm.int8", 1, False), (None, 1, False)])
def test_adapter_v2_paths_vs_oracle_and_identity(dev, mode, B, fused):
    """head_size 128, under the graph: the fused step (B = 1) or the module path against the v2 oracle, the prefill and
    the no-cache forward included; at B = 1 the fused step against the module path, no farther apart than the plain
    model's two paths; identity affines (scale 1, bias 0) give the v1-adapter model's logits bit for bit."""
    model, oracle, _ = build(dev, CFG128, mode)
    model.graph_after = 2
    got = run(model, dev, B)
    assert (model._decode is not None) == fused
    if fused:
        assert L.lib().b2l_decode_step_launches(C.byref(model._decode.args)) == 5 * CFG128["n_layer"] + 3
        assert model._decode.args.affines and model._decode.args.lm_head_affine.scale
    bar = 6e-2 if mode == "llm.int8" else 2e-2
    close(got, want_of(oracle, B), bar)
    v1, _, _ = build(dev, CFG128, mode, v2=False)
    v1.graph_after = 2
    want_v1 = run(v1, dev, B)
    assert not torch.equal(got[-1], want_v1[-1])
    if fused:   # the module path on the same models
        model.reset_cache()
        model._fast_ok = False
        mod = run(model, dev, B)
        assert model._decode is None
        v1.reset_cache()
        v1._fast_ok = False
        v1_mod = run(v1, dev, B)
        d_v2, d_v1 = rel(got, mod), rel(want_v1, v1_mod)
        assert d_v2 <= max(d_v1 * 1.5, 1e-3) or all(torch.equal(a, b) for a, b in zip(got, mod)), (d_v2, d_v1)
        if all(torch.equal(a, b) for a, b in zip(want_v1, v1_mod)):
            assert all(torch.equal(a, b) for a, b in zip(got, mod))
        v1._fast_ok = None
        v1.reset_cache()
        want_v1 = run(v1, dev, B)
    elif v1._decode is not None:   # B >= 2: the v2 model decodes module by module, so compare on that path
        v1.reset_cache()
        v1._fast_ok = False
        want_v1 = run(v1, dev, B)
        assert v1._decode is None
    ident, _, _ = build(dev, CFG128, mode, identity=True)
    ident.graph_after = 2
    for a, b in zip(run(ident, dev, B), want_v1):
        assert torch.equal(a, b)
    with torch.no_grad():
        model.reset_cache()
        nc = model(PROMPT.view(1, -1).to(dev))
        ident.reset_cache()
        v1.reset_cache()
        assert torch.equal(ident(PROMPT.view(1, -1).to(dev)), v1(PROMPT.view(1, -1).to(dev)))
    oracle.reset_cache()
    close([nc], [oracle.forward(PROMPT.view(1, -1))], bar)


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_adapter_v2_compact_and_reload_after_graph(dev, mode):
    """compact(): the same logits and state_dict, one resident copy; loading a second v2 checkpoint (scales, biases,
    norm scales, prefix, gates) into a graph-captured model: the next token equals a freshly built model's."""
    ref, _, _ = build(dev, CFG128, mode)
    ref.graph_after = 2
    a = run(ref, dev)
    sd0 = {k: v.clone() for k, v in ref.state_dict().items()}
    cm, _, _ = build(dev, CFG128, mode)
    cm.graph_after = 2
    cm.compact()
    assert all(lin._released for blk in cm.transformer.h for lin in (blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_proj))
    for x, y in zip(a, run(cm, dev)):
        assert torch.equal(x, y)
    sd1 = cm.state_dict()
    assert set(sd1) == set(sd0) and all(torch.equal(sd1[k], sd0[k]) for k in sd0)
    # a second v2 checkpoint on the same base, loaded after graph capture into the compacted model
    assert cm._decode is not None and cm._decode.graph is not None
    _, _, sd2 = build(dev, CFG128, mode, v2_seed=999)
    sd2 = dict(sd2)
    g = torch.Generator().manual_seed(5)
    for k in [k for k in sd2 if "adapter_wte" in k or "gating_factor" in k]:
        sd2[k] = (sd2[k].float() + 0.25 * torch.randn(sd2[k].shape, generator=g)).to(sd2[k].dtype)
    new = PV.adapter_v2_state_from_state_dict(sd2)
    cm.load_state_dict(new, strict=False)
    assert cm.transformer.h[0].attn.c_attn._released
    # a model that never captured a graph, with the same history, then the same new weights
    fresh, _, _ = build(dev, CFG128, mode)
    fresh.graph_after = 0
    run(fresh, dev)
    fresh.load_state_dict(new, strict=False)
    nxt = (torch.tensor([[88]], device=dev), 32, torch.tensor([7 + len(TOKS)], device=dev))
    with torch.no_grad():
        got, want, old = cm(*nxt), fresh(*nxt), ref(*nxt)
    assert torch.equal(got, want) and not torch.equal(got, old)
    assert cm._decode is not None

"""GPU: LLaMA-Adapter inference (lit_llama_b200.adapter) against the unmodified reference's fixture and the oracle,
the fused decode attention's adapter variant against the three-kernel path plus the prefix kernel, and the
exactness properties (zero gates / no adapter layer = the plain model, bit for bit)."""
import ctypes as C

import pytest
import torch

from conftest import load_golden

import lit_llama_b200 as P
from lit_llama_b200 import _lib as L
from lit_llama_b200 import adapter as PA
from lit_llama_b200.utils import quantization
from oracle import adapter_oracle as A

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    return torch.device("cuda", 0)


def build(dev, cfg, mode, seed=1234, adapter_seed=4321, zero_gates=False, exact_linears=True, cls=None):
    sd = A.adapter_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"],
                              None if mode == "llm.int8" else mode, cfg.get("adapter_prompt_length", 10),
                              cfg.get("adapter_start_layer", 2), seed=seed, adapter_seed=adapter_seed, zero_gates=zero_gates)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization(mode):
            if cls is None:
                model = PA.LLaMA(PA.LLaMAConfig(**cfg))
            else:   # the plain model on the same base weights
                model = cls(P.LLaMAConfig(**{k: v for k, v in cfg.items() if not k.startswith("adapter_")}))
    finally:
        torch.set_default_dtype(prev)
    if cls is not None:
        sd = {k: v for k, v in sd.items() if "adapter_wte" not in k and "gating_factor" not in k}
    res = model.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    oracle = A.OracleAdapterLLaMA.from_state_dict(sd, cfg["n_layer"], cfg["n_head"], cfg["block_size"], mode,
                                                   exact_linears=exact_linears)
    return model.eval(), oracle, sd


def run_steps(model, dev, prompt, S, toks):
    with torch.no_grad():
        out = [model(prompt.view(1, -1).to(dev), S, torch.arange(prompt.numel(), device=dev))]
        for i, t in enumerate(toks):
            out.append(model(torch.tensor([[t]], device=dev), S, torch.tensor([prompt.numel() + i], device=dev)))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("graph_after", [0, 2])
def test_tiny_adapter_model_matches_reference(dev, graph_after):
    g = load_golden("tiny_adapter_int4_bf16.pt")
    c = g["cfg"]
    model, _, _ = build(dev, c, "gptq.int4", seed=g["seed"], adapter_seed=g["adapter_seed"])
    model.graph_after = graph_after
    p = g["prompt"]
    for a, b in zip(run_steps(model, dev, p, 16, g["steps_tokens"]), g["steps_logits"]):
        torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    with torch.no_grad():
        nc = model(p.view(1, -1).to(dev))
    torch.testing.assert_close(nc.float().cpu(), g["nocache_logits"].float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    roll = [x[:, -1] for x in run_steps(model, dev, p, 8, g["roll_tokens"])]
    for a, b in zip(roll, g["roll_logits"]):
        torch.testing.assert_close(a.float().cpu(), b.float(), rtol=1e-3, atol=5e-3)
    model.reset_cache()
    greedy = P.generate(model, p.to(torch.int32).to(dev), 12, top_k=1).cpu()
    assert (greedy == g["gen_greedy"]).float().mean() >= 0.9


def _rand_attention_inputs(dev, B, nh, S, pos, aT, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    hs = 128
    bf = dict(device=dev, dtype=torch.bfloat16)
    r = lambda *s: torch.randn(*s, generator=gen, device=dev).to(torch.bfloat16)  # noqa: E731
    return dict(qkv=r(B, 3 * nh * hs), kc=r(B, nh, S, hs), vc=r(B, nh, S, hs), pk=r(nh, aT, hs), pv=r(nh, aT, hs),
                gate=(torch.rand(nh, generator=gen, device=dev) + 0.5).to(torch.bfloat16),
                rope=P.build_rope_cache(S, hs, torch.int64, dev).float().contiguous(),
                pos=torch.tensor([pos], dtype=torch.int64, device=dev), ring=torch.zeros(1, dtype=torch.int32, device=dev),
                work=torch.zeros(L.lib().b2l_attn_workspace_bytes(B, nh, hs, 1, S) // 4 + 1, device=dev, dtype=torch.float32),
                zero=torch.zeros(nh, **bf))


def _attend(x, B, nh, S, flags, gate=None, adapter=True):
    lib = L.lib()
    qkv, kc, vc = x["qkv"].clone(), x["kc"].clone(), x["vc"].clone()
    y = torch.empty(B, nh * 128, device=qkv.device, dtype=torch.bfloat16)
    args = (qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), x["rope"].data_ptr(), x["pos"].data_ptr(), x["ring"].data_ptr(),
            y.data_ptr(), x["work"].data_ptr(), B, 1, nh, 128, S, S, flags)
    if adapter:
        g = x["gate"] if gate is None else gate
        pre = L.AdapterPrefix(x["pk"].data_ptr(), x["pv"].data_ptr(), g.data_ptr(), x["pk"].shape[1])
        L.check(lib.b2l_attention_adapter(*args, C.byref(pre), L.stream_ptr()), "b2l_attention_adapter")
    else:
        L.check(lib.b2l_attention(*args, L.stream_ptr()), "b2l_attention")
    torch.cuda.synchronize()
    return y, qkv, kc, vc


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("pos,aT", [(37, 10), (200, 64), (1500, 10), (2047, 1)])
def test_fused_adapter_attention(dev, B, pos, aT):
    """head_size 128, T = 1: the fused kernel's adapter variant (one CTA per head at short positions, a cross-CTA merge
    at long ones) against exact softmax arithmetic and against B2L_F_ATTN_UNFUSED + the prefix kernel."""
    nh, S = 4, 2048
    x = _rand_attention_inputs(dev, B, nh, S, pos, aT, seed=pos * 7 + B)
    yf, _, kf, _ = _attend(x, B, nh, S, 0)
    yu, qu, ku, vu = _attend(x, B, nh, S, 8)
    assert torch.equal(kf, ku)
    # exact arithmetic from the rotated bf16 q the unfused path leaves in qkv
    q = qu[:, : nh * 128].view(B, nh, 1, 128).double()
    k, v = ku[:, :, : pos + 1].double(), vu[:, :, : pos + 1].double()
    y = torch.softmax(q @ k.transpose(-1, -2) / 128 ** 0.5, -1) @ v
    ak, av = x["pk"].double().unsqueeze(0), x["pv"].double().unsqueeze(0)
    ay = torch.softmax(q @ ak.transpose(-1, -2) / 128 ** 0.5, -1) @ av
    g = x["gate"].view(1, nh, 1, 1)
    want = (y.bfloat16() + (g * ay.bfloat16()).bfloat16()).bfloat16().view(B, nh * 128).float()
    for got in (yf, yu):
        torch.testing.assert_close(got.float(), want, rtol=2 ** -7, atol=2e-2)
        assert (got.float() == want).float().mean() > 0.9
    assert (yf == yu).float().mean() > 0.9
    # zero gates: bit-identical to the plain kernel
    y0, _, _, _ = _attend(x, B, nh, S, 0, gate=x["zero"])
    yp, _, _, _ = _attend(x, B, nh, S, 0, adapter=False)
    assert torch.equal(y0, yp)


CFG128 = dict(block_size=64, vocab_size=256, n_layer=3, n_head=4, n_embd=512, adapter_prompt_length=10, adapter_start_layer=1)
PROMPT = torch.tensor([5, 100, 3, 7, 200, 9, 31])
TOKS = [77, 12, 9, 150, 42]


def _close_to_oracle(got, oracle, S=32):
    want = [oracle.forward(PROMPT.view(1, -1), S, torch.arange(7))]
    for i, t in enumerate(TOKS):
        want.append(oracle.forward(torch.tensor([[t]]), S, torch.tensor([7 + i])))
    for a, b in zip(got, want):
        a, b = a.float().cpu(), b.float()
        assert float((a - b).norm() / b.norm()) < 2e-2


@pytest.mark.parametrize("mode,fused", [("gptq.int4", True), ("gptq.int8", True), ("llm.int8", False)])
def test_adapter_model_vs_oracle_and_exactness(dev, mode, fused):
    """head_size 128: gptq.int4 / gptq.int8 decode on the fused step (adapter attention in the fused kernel, launch
    count unchanged), llm.int8 module by module; zero gates and adapter_start_layer >= n_layer give the plain
    model's logits bit for bit."""
    model, oracle, _ = build(dev, CFG128, mode)
    model.graph_after = 2
    got = run_steps(model, dev, PROMPT, 32, TOKS)
    assert (model._decode is not None) == fused
    if fused:
        plain_launches = 5 * CFG128["n_layer"] + 3
        assert L.lib().b2l_decode_step_launches(C.byref(model._decode.args)) == plain_launches
        assert model._decode.args.adapters
    _close_to_oracle(got, oracle)
    plain, _, _ = build(dev, CFG128, mode, cls=P.LLaMA)
    plain.graph_after = 2
    want = run_steps(plain, dev, PROMPT, 32, TOKS)
    assert not torch.equal(got[-1], want[-1])
    for kw in (dict(zero_gates=True), dict(cfg=dict(CFG128, adapter_start_layer=CFG128["n_layer"]))):
        cfg = kw.pop("cfg", CFG128)
        m0, _, _ = build(dev, cfg, mode, **kw)
        m0.graph_after = 2
        for a, b in zip(run_steps(m0, dev, PROMPT, 32, TOKS), want):
            assert torch.equal(a, b)
    with torch.no_grad():
        model.reset_cache()
        nc = model(PROMPT.view(1, -1).to(dev))
    oracle.reset_cache()
    want_nc = oracle.forward(PROMPT.view(1, -1))
    assert float((nc.float().cpu() - want_nc.float()).norm() / want_nc.float().norm()) < 2e-2


def test_adapter_reload_after_graph_and_compact(dev):
    """Loading new adapter weights after the decode graph was captured takes effect at the next step; compact()
    changes no output."""
    model, oracle, _ = build(dev, CFG128, "gptq.int4")
    model.graph_after = 2
    run_steps(model, dev, PROMPT, 32, TOKS)
    assert model._decode.graph is not None
    _, _, sd2 = build(dev, CFG128, "gptq.int4", adapter_seed=999)
    new = PA.adapter_state_from_state_dict(sd2)
    model.load_state_dict(new, strict=False)
    with torch.no_grad():
        got = model(torch.tensor([[88]], device=dev), 32, torch.tensor([7 + len(TOKS)], device=dev))
    # the oracle with the same history, then the new adapter weights (prefix recomputed from them)
    for i, t in enumerate([None] + TOKS):
        if t is None:
            oracle.forward(PROMPT.view(1, -1), 32, torch.arange(7))
        else:
            oracle.forward(torch.tensor([[t]]), 32, torch.tensor([7 + i - 1]))
    o2 = A.OracleAdapterLLaMA.from_state_dict(sd2, CFG128["n_layer"], CFG128["n_head"], CFG128["block_size"], "gptq.int4",
                                              exact_linears=True)
    oracle.adapters, oracle.akv = o2.adapters, {}
    want = oracle.forward(torch.tensor([[88]]), 32, torch.tensor([7 + len(TOKS)]))
    assert float((got.float().cpu() - want.float()).norm() / want.float().norm()) < 2e-2
    # compact(): the same logits bit for bit, prefill and graph-replayed decode
    ref, _, _ = build(dev, CFG128, "gptq.int4")
    ref.graph_after = 2
    a = run_steps(ref, dev, PROMPT, 32, TOKS)
    cm, _, _ = build(dev, CFG128, "gptq.int4")
    cm.graph_after = 2
    cm.compact()
    for x, y in zip(a, run_steps(cm, dev, PROMPT, 32, TOKS)):
        assert torch.equal(x, y)
    # adapter-only reload (strict=False) into a COMPACTED model after graph capture: the compacted layers keep their
    # only weight copy, and the next step follows the new adapter weights
    cm.load_state_dict(new, strict=False)
    for blk in cm.transformer.h:
        for lin in (blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_fc1, blk.mlp.c_fc2, blk.mlp.c_proj):
            assert lin._released
    with torch.no_grad():
        got_c = cm(torch.tensor([[88]], device=dev), 32, torch.tensor([7 + len(TOKS)], device=dev))
    assert torch.equal(got_c, got)   # same history, same new adapter: the uncompacted model's step, bit for bit
    assert float((got_c.float().cpu() - want.float()).norm() / want.float().norm()) < 2e-2
    with torch.no_grad():   # and a base-model reload after that still brings the reference buffers back
        cm.load_state_dict({k: v for k, v in sd2.items() if "adapter" not in k and "gating" not in k}, strict=False)
    assert not cm.transformer.h[0].attn.c_attn._released

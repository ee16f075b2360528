"""CPU: LLaMA-Adapter (lit_llama/adapter.py) - the oracle against the unmodified reference's fixture, the module
contract of lit_llama_b200.adapter, patch_reference() on the adapter surface, and the C entry points' argument
checks, struct layout, launch count and refusals (all decided before any launch)."""
import ctypes as C
import json
import os
import subprocess
import sys
import types

import pytest
import torch

from conftest import load_golden

import __graft_entry__ as entry
import lit_llama_b200 as P
from lit_llama_b200 import adapter as PA
from lit_llama_b200.utils import quantization
from oracle import adapter_oracle as A
from oracle import llama_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden():
    return load_golden("tiny_adapter_int4_bf16.pt")


def golden_sd(g, **kw):
    c = g["cfg"]
    return A.adapter_state_dict(c["n_layer"], c["n_head"], c["n_embd"], c["vocab_size"], "gptq.int4",
                                c["adapter_prompt_length"], c["adapter_start_layer"], seed=g["seed"],
                                adapter_seed=g["adapter_seed"], **kw)


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_adapter_oracle_matches_reference_fixture():
    g = golden()
    c = g["cfg"]
    o = A.OracleAdapterLLaMA.from_state_dict(golden_sd(g), c["n_layer"], c["n_head"], c["block_size"], "gptq.int4")
    p = g["prompt"]
    got = [o.forward(p.view(1, -1), 16, torch.arange(7))]
    for i, t in enumerate(g["steps_tokens"]):
        got.append(o.forward(torch.tensor([[t]]), 16, torch.tensor([7 + i])))
    for a, b in zip(got, g["steps_logits"]):
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-3, atol=5e-3)
    o.reset_cache()
    torch.testing.assert_close(o.forward(p.view(1, -1)).float(), g["nocache_logits"].float(), rtol=1e-3, atol=5e-3)
    o.reset_cache()
    roll = [o.forward(p.view(1, -1), 8, torch.arange(7))[:, -1]]
    for i, t in enumerate(g["roll_tokens"]):
        roll.append(o.forward(torch.tensor([[t]]), 8, torch.tensor([7 + i]))[:, -1])
    for a, b in zip(roll, g["roll_logits"]):
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-3, atol=5e-3)
    o.reset_cache()
    o.block_size = c["block_size"]
    greedy = O.generate(o, p.to(torch.int32), 12, top_k=1)
    assert (greedy == g["gen_greedy"]).float().mean() >= 0.9
    # the gates are not vacuous: with them zeroed the logits move far beyond the tolerance
    o0 = A.OracleAdapterLLaMA.from_state_dict(golden_sd(g, zero_gates=True), c["n_layer"], c["n_head"], c["block_size"], "gptq.int4")
    assert (o0.forward(p.view(1, -1)).float() - g["nocache_logits"].float()).abs().max() > 0.02


def test_adapter_module_contract():
    g = golden()
    c = g["cfg"]
    with quantization("gptq.int4"):
        m = PA.LLaMA(PA.LLaMAConfig(**c))
    assert sorted(m.state_dict().keys()) == g["state_dict_keys"]
    for i, blk in enumerate(m.transformer.h):
        has = i >= c["adapter_start_layer"]
        assert hasattr(blk.attn, "adapter_wte") == has and hasattr(blk.attn, "gating_factor") == has
        assert blk.attn.block_idx == i and isinstance(blk, P.Block) and isinstance(blk.attn, P.CausalSelfAttention)
        if has:
            assert blk.attn.adapter_wte.weight.shape == (c["adapter_prompt_length"], c["n_embd"])
            assert blk.attn.gating_factor.shape == (1, c["n_head"], 1, 1)
            assert torch.count_nonzero(blk.attn.gating_factor) == 0   # zero-init (adapter.py:79)
    assert m.transformer.wte.weight.shape[0] == c["vocab_size"] and m.lm_head.out_features == c["vocab_size"]
    assert isinstance(m, P.LLaMA) and m.adapter_kv_caches == []
    sd = golden_sd(g)
    res = m.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    # base checkpoint then adapter checkpoint, both strict=False (generate/adapter.py:70-73)
    base = {k: v for k, v in sd.items() if "adapter_wte" not in k and "gating_factor" not in k}
    ada = PA.adapter_state_from_state_dict(sd)
    assert set(ada) == set(sd) - set(base)
    with quantization("gptq.int4"):
        m2 = PA.LLaMA(PA.LLaMAConfig(**c))
    m2.load_state_dict(base, strict=False)
    m2.load_state_dict(ada, strict=False)
    for k, v in m2.state_dict().items():
        assert torch.equal(v.to(sd[k].dtype), sd[k]), k
    # legacy checkpoints: one gating value for all heads (adapter.py:184-186)
    m2.load_state_dict({"transformer.h.2.attn.gating_factor": torch.tensor(0.25)}, strict=False)
    assert torch.equal(m2.transformer.h[2].attn.gating_factor.data, torch.full((1, c["n_head"], 1, 1), 0.25))
    # loading adapter weights invalidates baked decode states
    from lit_llama_b200.quantization import WEIGHTS_GENERATION

    g0 = WEIGHTS_GENERATION[0]
    m2.load_state_dict(ada, strict=False)
    assert WEIGHTS_GENERATION[0] > g0
    assert PA.LLaMAConfig.from_name("7B").adapter_start_layer == 2 and isinstance(PA.LLaMA.from_name, object)


def test_patch_reference_rewires_the_adapter_surface():
    """patch_reference() against the recorded surface of the unmodified reference (reference_surface.json for the
    package, reference_adapter_surface.json for lit_llama.adapter and generate/adapter.py)."""
    gd = os.path.join(ROOT, "tests", "golden")
    surface = json.load(open(os.path.join(gd, "reference_surface.json")))["modules"]
    surface.update(json.load(open(os.path.join(gd, "reference_adapter_surface.json")))["modules"])
    objs = {}

    def stand_in(origin):
        return objs.setdefault(origin, type(origin.rsplit(".", 1)[-1], (), {"origin": origin}))

    pkg = "lit_llama_adapter_surface"
    names = {"pkg": pkg, "model": pkg + ".model", "quant": pkg + ".quantization", "utils": pkg + ".utils",
             "generate": pkg + "_generate", "adapter": pkg + ".adapter", "generate_adapter": pkg + "_generate_adapter"}
    mods = {key: types.ModuleType(name) for key, name in names.items()}
    for key, ns in surface.items():
        for name, origin in ns.items():
            setattr(mods[key], name, stand_in(origin))
    ref = {key: dict(vars(mod)) for key, mod in mods.items()}
    sys.modules.update({mod.__name__: mod for mod in mods.values()})
    try:
        saved = P.patch_reference(mods["pkg"])
        for name in ("LLaMA", "LLaMAConfig", "Block", "CausalSelfAttention"):
            assert getattr(mods["adapter"], name) is getattr(PA, name)
            assert saved[("adapter", name)] is ref["adapter"][name]
        assert mods["model"].LLaMA is P.LLaMA   # the base model keeps its own drop-in
        assert mods["generate_adapter"].LLaMA is PA.LLaMA   # `from lit_llama.adapter import LLaMA` follows
        assert mods["generate_adapter"].quantization is P.utils.quantization
        assert mods["adapter"].mark_only_adapter_as_trainable is ref["adapter"]["mark_only_adapter_as_trainable"]
        with mods["generate_adapter"].quantization("gptq.int4"):
            m = mods["generate_adapter"].LLaMA(mods["adapter"].LLaMAConfig(block_size=16, vocab_size=64, n_layer=3, n_head=2, n_embd=64))
        assert isinstance(m, PA.LLaMA) and isinstance(m.lm_head, P.ColBlockQuantizedLinear)
        assert hasattr(m.transformer.h[2].attn, "gating_factor") and not hasattr(m.transformer.h[1].attn, "gating_factor")
    finally:
        for mod in mods.values():
            sys.modules.pop(mod.__name__, None)


def test_adapter_entry_points_reject_bad_arguments(L):
    lib = L.lib()
    p = C.c_void_p(256)
    ok = L.AdapterPrefix(256, 512, 256, 10)

    def att(pre):
        return lib.b2l_attention_adapter(p, p, p, p, p, p, p, p, 1, 1, 4, 128, 16, 64, 0, pre, None)

    def noc(pre):
        return lib.b2l_attention_nocache_adapter(p, p, p, p, 1, 4, 4, 128, 64, pre, None)

    for fn in (att, noc):
        assert fn(None) == -1 and b"null adapter prefix" in lib.b2l_last_error()
        for bad in (L.AdapterPrefix(None, 512, 256, 10), L.AdapterPrefix(256, None, 256, 10), L.AdapterPrefix(256, 512, None, 10)):
            assert fn(C.byref(bad)) == -1 and b"null adapter prefix" in lib.b2l_last_error()
        for n in (0, -1, 65):
            assert fn(C.byref(L.AdapterPrefix(256, 512, 256, n))) == -2 and b"prefix length" in lib.b2l_last_error()
        for bad in (L.AdapterPrefix(264, 512, 256, 10), L.AdapterPrefix(256, 520, 256, 10), L.AdapterPrefix(256, 512, 257, 10)):
            assert fn(C.byref(bad)) == -1 and b"aligned" in lib.b2l_last_error()
    assert lib.b2l_attention_adapter(None, p, p, p, p, p, p, p, 1, 1, 4, 128, 16, 64, 0, C.byref(ok), None) == -1
    assert lib.b2l_attention_nocache_adapter(p, p, p, p, 1, 4, 4, 130 * 2, 64, C.byref(ok), None) == -2


def test_adapter_struct_layout_matches_c_compiler(L, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "int main(void){\n"
        'printf("%zu %zu %zu %zu %zu\\n", sizeof(b2l_adapter_prefix), offsetof(b2l_adapter_prefix, len), '
        "sizeof(b2l_decode_args), offsetof(b2l_decode_args, batch_work), offsetof(b2l_decode_args, adapters));\n"
        "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    got = [C.sizeof(L.AdapterPrefix), L.AdapterPrefix.len.offset, C.sizeof(L.DecodeArgs), L.DecodeArgs.batch_work.offset,
           L.DecodeArgs.adapters.offset]
    assert [int(v) for v in out] == got


def _decode_args(L, n_layer, n_head, n_embd, adapters):
    layers = (L.Layer * n_layer)()
    d = L.DecodeArgs(n_layer=n_layer, n_head=n_head, n_embd=n_embd, n_hidden=4 * n_embd, vocab=128, B=1, S=64,
                     layers=layers, wte=16, ln_f=16, rope=16, idx=16, input_pos=16, ring_start=16, block_size=64, x=16,
                     qkv=16, att=16, hid=16, attn_work=16, logits=16)
    keep = [layers]
    if adapters is not None:
        arr = (L.AdapterPrefix * n_layer)(*adapters)
        keep.append(arr)
        d.adapters = C.cast(arr, C.POINTER(L.AdapterPrefix))
    return d, keep


def test_decode_step_launch_count_and_refusals(L):
    lib = L.lib()
    pre = L.AdapterPrefix(256, 512, 256, 10)
    none = L.AdapterPrefix(None, None, None, 0)
    # head_size 128: the prefix term runs inside the fused attention launch, so the count stays 5 n_layer + 3
    d, keep = _decode_args(L, 4, 4, 512, [none, none, pre, pre])
    d0, keep0 = _decode_args(L, 4, 4, 512, None)
    assert lib.b2l_decode_step_launches(C.byref(d)) == lib.b2l_decode_step_launches(C.byref(d0)) == 5 * 4 + 3
    # other head sizes: one prefix kernel per adapter layer behind the three-kernel attention
    d, keep = _decode_args(L, 4, 4, 256, [none, none, pre, pre])
    d0, keep0 = _decode_args(L, 4, 4, 256, None)
    assert lib.b2l_decode_step_launches(C.byref(d)) == lib.b2l_decode_step_launches(C.byref(d0)) + 2
    # B2L_F_ATTN_UNFUSED at head_size 128: three attention kernels plus the prefix kernel per adapter layer
    d, keep = _decode_args(L, 4, 4, 512, [none, none, pre, pre])
    d.flags = 8
    assert lib.b2l_decode_step_launches(C.byref(d)) == 2 + 4 * (4 + 3) + 1 + 2
    # bad prefixes are rejected before any launch
    d, keep = _decode_args(L, 4, 4, 512, [none, none, pre, L.AdapterPrefix(256, 512, 256, 65)])
    assert lib.b2l_decode_step(C.byref(d), None) == -2 and b"prefix length" in lib.b2l_last_error()
    d, keep = _decode_args(L, 4, 4, 512, [none, none, pre, L.AdapterPrefix(256, None, 256, 10)])
    assert lib.b2l_decode_step(C.byref(d), None) == -1 and b"null adapter prefix" in lib.b2l_last_error()

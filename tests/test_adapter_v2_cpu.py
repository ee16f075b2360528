"""CPU: LLaMA-Adapter v2 (lit_llama/adapter_v2.py) - the oracle against the unmodified reference's fixture on a dense
and a gptq.int4 base, the module contract of lit_llama_b200.adapter_v2 under every quantization mode, patch_reference()
on the v2 surface, and the C entry points' argument checks, struct layout, launch count and refusals (all decided
before any launch)."""
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
from lit_llama_b200 import adapter_v2 as PV
from lit_llama_b200.quantization import WEIGHTS_GENERATION
from lit_llama_b200.utils import quantization
from oracle import adapter_v2_oracle as A2
from oracle import llama_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASES = {"dense": None, "gptq.int4": "gptq.int4"}
TINY = dict(block_size=16, vocab_size=64, n_layer=2, n_head=2, n_embd=64, adapter_prompt_length=4, adapter_start_layer=1)


def golden():
    return load_golden("tiny_adapter_v2_bf16.pt")


def golden_sd(g, mode, **kw):
    c = g["cfg"]
    return A2.adapter_v2_state_dict(c["n_layer"], c["n_head"], c["n_embd"], c["vocab_size"], mode,
                                    c["adapter_prompt_length"], c["adapter_start_layer"], seed=g["seed"],
                                    adapter_seed=g["adapter_seed"], v2_seed=g["v2_seed"], **kw)


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


@pytest.mark.parametrize("base", list(BASES))
def test_adapter_v2_oracle_matches_reference_fixture(base):
    g = golden()
    c, want = g["cfg"], g["bases"][base]
    mode = BASES[base]
    o = A2.OracleAdapterV2LLaMA.from_state_dict(golden_sd(g, mode), c["n_layer"], c["n_head"], c["block_size"], mode)
    p = want["prompt"]
    got = [o.forward(p.view(1, -1), 16, torch.arange(7))]
    for i, t in enumerate(want["steps_tokens"]):
        got.append(o.forward(torch.tensor([[t]]), 16, torch.tensor([7 + i])))
    for a, b in zip(got, want["steps_logits"]):
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-3, atol=5e-3)
    o.reset_cache()
    nc = o.forward(p.view(1, -1))
    torch.testing.assert_close(nc.float(), want["nocache_logits"].float(), rtol=1e-3, atol=5e-3)
    o.reset_cache()
    roll = [o.forward(p.view(1, -1), 8, torch.arange(7))[:, -1]]
    for i, t in enumerate(want["roll_tokens"]):
        roll.append(o.forward(torch.tensor([[t]]), 8, torch.tensor([7 + i]))[:, -1])
    for a, b in zip(roll, want["roll_logits"]):
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-3, atol=5e-3)
    o.reset_cache()
    o.block_size = c["block_size"]
    greedy = O.generate(o, p.to(torch.int32), 12, top_k=1)
    assert (greedy == want["gen_greedy"]).float().mean() >= 0.9
    # the affine is not vacuous: with scale 1 and bias 0 the logits move far beyond the tolerance
    o1 = A2.OracleAdapterV2LLaMA.from_state_dict(golden_sd(g, mode, identity=True), c["n_layer"], c["n_head"],
                                                 c["block_size"], mode)
    assert (o1.forward(p.view(1, -1)).float() - want["nocache_logits"].float()).abs().max() > 0.1


def _v2_model(cfg, mode):
    with quantization(mode):
        m = PA.LLaMA(PA.LLaMAConfig(**cfg))
        PV.add_adapter_v2_parameters_to_linear_layers(m)
    return m


@pytest.mark.parametrize("base", list(BASES))
def test_adapter_v2_module_contract(base):
    g = golden()
    c = g["cfg"]
    m = _v2_model(c, BASES[base])
    keys = sorted(m.state_dict().keys())
    assert keys == g["bases"][base]["state_dict_keys"]
    adapter_keys = [k for k in keys if ".adapter_" in k]
    assert len(adapter_keys) == 34   # 2 per linear (5 per Block + lm_head) + adapter_wte of layers 1, 2
    for p in A2.linear_prefixes(c["n_layer"]):
        lin = m.get_submodule(p)
        assert torch.equal(lin.adapter_scale.data, torch.ones(lin.out_features))
        assert torch.equal(lin.adapter_bias.data, torch.zeros(lin.out_features))
        assert lin.adapter_scale.dtype == torch.get_default_dtype() and lin.adapter_scale.requires_grad
    sd = golden_sd(g, BASES[base])
    res = m.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    # base checkpoint then adapter checkpoint, both strict=False (generate/adapter_v2.py:72-75)
    ada = PV.adapter_v2_state_from_state_dict(sd)
    subs = PV.get_adapter_substrings()
    assert set(ada) == {k for k in sd if any(s in k for s in subs)}
    m2 = _v2_model(c, BASES[base])
    m2.load_state_dict({k: v for k, v in sd.items() if k not in ada}, strict=False)
    g0 = WEIGHTS_GENERATION[0]
    res = m2.load_state_dict(ada, strict=False)
    assert not res.unexpected_keys and WEIGHTS_GENERATION[0] > g0
    for k, v in m2.state_dict().items():
        assert torch.equal(v.to(sd[k].dtype), sd[k]), k
    # a load that touches only one linear's affine, or one RMSNorm scale, also bumps the generation
    for mod, key in ((m2.lm_head, "adapter_bias"), (m2.transformer.h[0].rms_1, "scale")):
        g0 = WEIGHTS_GENERATION[0]
        mod.load_state_dict({key: getattr(mod, key).detach().clone()}, strict=False)
        assert WEIGHTS_GENERATION[0] > g0
    PV.mark_only_adapter_v2_as_trainable(m2)
    trainable = {n for n, p in m2.named_parameters() if p.requires_grad}
    assert trainable == {n for n, _ in m2.named_parameters() if any(s in n for s in subs)}
    assert any("rms_1" in n for n in trainable) and any("adapter_scale" in n for n in trainable)


def test_adapter_v2_refuses_lora_layers():
    from lit_llama_b200 import lora as PL

    with PL.lora(r=4, alpha=8, dropout=0.0):
        m = P.LLaMA(P.LLaMAConfig(**{k: v for k, v in TINY.items() if not k.startswith("adapter_")}))
    with pytest.raises(ValueError, match="LoRA"):
        PV.add_adapter_v2_parameters_to_linear_layers(m)


def test_patch_reference_rewires_the_adapter_v2_surface():
    """patch_reference() against the recorded surface of the unmodified reference, then generate/adapter_v2.py's
    construction sequence (adapter.LLaMA, add_adapter_v2_parameters_to_linear_layers, base then adapter checkpoint with
    strict=False) under every --quantize value."""
    gd = os.path.join(ROOT, "tests", "golden")
    surface = json.load(open(os.path.join(gd, "reference_surface.json")))["modules"]
    surface.update(json.load(open(os.path.join(gd, "reference_adapter_surface.json")))["modules"])
    surface.update(json.load(open(os.path.join(gd, "reference_adapter_v2_surface.json")))["modules"])
    objs = {}

    def stand_in(origin):
        return objs.setdefault(origin, type(origin.rsplit(".", 1)[-1], (), {"origin": origin}))

    pkg = "lit_llama_adapter_v2_surface"
    names = {"pkg": pkg, "model": pkg + ".model", "quant": pkg + ".quantization", "utils": pkg + ".utils",
             "generate": pkg + "_generate", "adapter": pkg + ".adapter", "generate_adapter": pkg + "_generate_adapter",
             "adapter_v2": pkg + ".adapter_v2", "generate_adapter_v2": pkg + "_generate_adapter_v2"}
    mods = {key: types.ModuleType(name) for key, name in names.items()}
    for key, ns in surface.items():
        for name, origin in ns.items():
            setattr(mods[key], name, stand_in(origin))
    ref = {key: dict(vars(mod)) for key, mod in mods.items()}
    sys.modules.update({mod.__name__: mod for mod in mods.values()})
    try:
        saved = P.patch_reference(mods["pkg"])
        for name in ("get_adapter_substrings", "mark_only_adapter_v2_as_trainable", "adapter_v2_state_from_state_dict",
                     "adapter_v2_new_forward", "adapter_v2_linear_with_bias_and_scale",
                     "add_adapter_v2_parameters_to_linear_layers"):
            assert getattr(mods["adapter_v2"], name) is getattr(PV, name)
            assert saved[("adapter_v2", name)] is ref["adapter_v2"][name]
        gen = mods["generate_adapter_v2"]
        assert gen.add_adapter_v2_parameters_to_linear_layers is PV.add_adapter_v2_parameters_to_linear_layers
        assert gen.LLaMA is PA.LLaMA and mods["adapter_v2"].LLaMA is PA.LLaMA
        assert gen.quantization is P.utils.quantization
        lin_kind = {None: torch.nn.modules.linear.Linear, "gptq.int4": P.ColBlockQuantizedLinear,
                    "gptq.int8": P.ColBlockQuantizedLinear, "llm.int8": P.Linear8bitLt}
        for q, kind in lin_kind.items():
            with gen.quantization(q):
                m = gen.LLaMA(mods["adapter"].LLaMAConfig(**TINY))
                gen.add_adapter_v2_parameters_to_linear_layers(m)
            assert isinstance(m, PA.LLaMA) and isinstance(m.lm_head, kind)
            want = sorted(k for k in m.state_dict() if ".adapter_" in k)
            assert want == sorted([p + ".adapter_bias" for p in A2.linear_prefixes(TINY["n_layer"])] +
                                  [p + ".adapter_scale" for p in A2.linear_prefixes(TINY["n_layer"])] +
                                  ["transformer.h.1.attn.adapter_wte.weight"])
            sd = A2.adapter_v2_state_dict(TINY["n_layer"], TINY["n_head"], TINY["n_embd"], TINY["vocab_size"],
                                          None if q == "llm.int8" else q, TINY["adapter_prompt_length"],
                                          TINY["adapter_start_layer"], dtype=torch.float32)
            ada = PV.adapter_v2_state_from_state_dict(sd)
            res = m.load_state_dict({k: v for k, v in sd.items() if k not in ada}, strict=False)
            assert not res.unexpected_keys, q
            res = m.load_state_dict(ada, strict=False)
            assert not res.unexpected_keys, q   # no v2 key dropped
            got = m.state_dict()
            for k, v in ada.items():
                assert torch.equal(got[k].float(), v.float()), (q, k)
    finally:
        for mod in mods.values():
            sys.modules.pop(mod.__name__, None)


def test_adapter_v2_struct_layout_matches_c_compiler(L, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "int main(void){\n"
        'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b2l_out_affine), offsetof(b2l_out_affine, bias), '
        "sizeof(b2l_layer_affine), offsetof(b2l_layer_affine, c_fc12), offsetof(b2l_layer_affine, mlp_proj), "
        "sizeof(b2l_q4_linear_args), offsetof(b2l_q4_linear_args, pf_seg_stride), offsetof(b2l_q4_linear_args, out_affine), "
        "sizeof(b2l_decode_args), offsetof(b2l_decode_args, affines), offsetof(b2l_decode_args, lm_head_affine));\n"
        "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    got = [C.sizeof(L.OutAffine), L.OutAffine.bias.offset, C.sizeof(L.LayerAffine), L.LayerAffine.c_fc12.offset,
           L.LayerAffine.mlp_proj.offset, C.sizeof(L.Q4LinearArgs), L.Q4LinearArgs.pf_seg_stride.offset,
           L.Q4LinearArgs.out_affine.offset, C.sizeof(L.DecodeArgs), L.DecodeArgs.affines.offset,
           L.DecodeArgs.lm_head_affine.offset]
    assert [int(v) for v in out] == got
    # existing fields keep their offsets: out_affine and the decode step's two fields are appended at the end
    assert L.Q4LinearArgs.out_affine.offset == L.Q4LinearArgs.pf_seg_stride.offset + 8
    assert L.DecodeArgs.affines.offset == L.DecodeArgs.loras.offset + 8


def test_linear_affine_rejects_bad_arguments(L):
    lib = L.lib()

    def call(y=256, ldy=64, M=4, N=64, s=512, b=768):
        return lib.b2l_linear_affine(y, ldy, M, N, s, b, None)

    for kw in (dict(y=None), dict(s=None), dict(b=None)):
        assert call(**kw) == -1 and b"null pointer" in lib.b2l_last_error()
    for kw in (dict(M=-1), dict(N=0), dict(N=-3), dict(ldy=63)):
        assert call(**kw) == -1 and b"bad shape" in lib.b2l_last_error()
    for kw in (dict(y=257), dict(s=513), dict(b=769)):
        assert call(**kw) == -1 and b"aligned" in lib.b2l_last_error()
    assert call(M=0) == 0   # nothing to do: no launch


def test_out_affine_rejected_where_unsupported(L):
    lib = L.lib()

    def args(scale, bias, **kw):
        a = dict(x=256, ldx=64, qw_tiled=256, scales=256, zeros=256, sz_dtype=0, y=256, ldy=16, M=1, N=16, K=64,
                 prologue=0, epilogue=0, workspace=256)
        a.update(kw)
        a = L.Q4LinearArgs(**a)
        a.out_affine = L.OutAffine(scale, bias)
        return a

    for fn in ("b2l_q4_linear_tc", "b2l_q4_gemm", "b2l_w8_gemm", "b2l_q4_gemv_batch"):
        for s, b in ((512, 768), (512, None), (None, 768)):
            assert getattr(lib, fn)(C.byref(args(s, b)), None) == -2, fn
            assert b"out_affine" in lib.b2l_last_error()
    # the batch-1 kernels take it, but only as a pair
    for fn in ("b2l_q4_gemv", "b2l_w8_gemv"):
        for s, b in ((512, None), (None, 768)):
            assert getattr(lib, fn)(C.byref(args(s, b)), None) == -1, fn
            assert b"out_affine" in lib.b2l_last_error()


def _decode_args(L, n_layer, n_head, n_embd, affines, B=1):
    layers = (L.Layer * n_layer)()
    w = L.Q4Weight(None, 256, 256, 256, 16, 64)
    for i in range(n_layer):
        layers[i] = L.Layer(rms_1=16, rms_2=16, c_attn=w, c_proj=w, c_fc12=w, mlp_proj=w, k_cache=16, v_cache=16)
    d = L.DecodeArgs(n_layer=n_layer, n_head=n_head, n_embd=n_embd, n_hidden=4 * n_embd, vocab=128, B=B, S=64,
                     layers=layers, wte=16, ln_f=16, lm_head=w, rope=16, idx=16, input_pos=16, ring_start=16,
                     block_size=64, x=16, qkv=16, att=16, hid=16, attn_work=16, logits=16)
    keep = [layers]
    if affines is not None:
        arr = (L.LayerAffine * n_layer)(*affines)
        keep.append(arr)
        d.affines = C.cast(arr, C.POINTER(L.LayerAffine))
        d.lm_head_affine = L.OutAffine(512, 768)
    return d, keep


def test_decode_step_launch_count_and_refusals(L):
    lib = L.lib()
    f = L.OutAffine(512, 768)
    lay = L.LayerAffine(f, f, f, f)
    # the affine runs inside each linear's launch: 5 n_layer + 3 with or without it (7B: 163)
    d, keep = _decode_args(L, 32, 32, 4096, [lay] * 32)
    d0, keep0 = _decode_args(L, 32, 32, 4096, None)
    assert lib.b2l_decode_step_launches(C.byref(d)) == lib.b2l_decode_step_launches(C.byref(d0)) == 163
    d.flags = d0.flags = 8   # B2L_F_ATTN_UNFUSED: the same count as the plain step
    assert lib.b2l_decode_step_launches(C.byref(d)) == lib.b2l_decode_step_launches(C.byref(d0))
    # batch 1 only
    for B in (2, 4, 16):
        d, keep = _decode_args(L, 4, 4, 512, [lay] * 4, B=B)
        assert lib.b2l_decode_step(C.byref(d), None) == -2 and b"batch 1" in lib.b2l_last_error()
    d, keep = _decode_args(L, 4, 4, 512, None, B=2)   # lm_head's affine alone counts too
    d.lm_head_affine = f
    assert lib.b2l_decode_step(C.byref(d), None) == -2 and b"batch 1" in lib.b2l_last_error()
    # not with LoRA
    d, keep = _decode_args(L, 4, 4, 512, [lay] * 4)
    loras = (L.LoRA * 4)()
    keep.append(loras)
    d.loras = C.cast(loras, C.POINTER(L.LoRA))
    assert lib.b2l_decode_step(C.byref(d), None) == -2 and b"LoRA" in lib.b2l_last_error()
    # half-set pairs are bad arguments
    half = L.OutAffine(512, None)
    d, keep = _decode_args(L, 4, 4, 512, [lay, lay, L.LayerAffine(f, f, half, f), lay])
    assert lib.b2l_decode_step(C.byref(d), None) == -1 and b"affines[2]" in lib.b2l_last_error()
    d, keep = _decode_args(L, 4, 4, 512, [lay] * 4)
    d.lm_head_affine = L.OutAffine(None, 768)
    assert lib.b2l_decode_step(C.byref(d), None) == -1 and b"lm_head_affine" in lib.b2l_last_error()
    # every weight needs the batch-1 tiling
    d, keep = _decode_args(L, 4, 4, 512, [lay] * 4)
    keep[0][1].c_proj.qw_mma = None
    assert lib.b2l_decode_step(C.byref(d), None) == -2 and b"qw_mma" in lib.b2l_last_error()

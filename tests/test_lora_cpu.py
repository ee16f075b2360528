"""CPU: LoRA (lit_llama/lora.py) - the oracle's unmerged branch against the unmodified reference's fixture, the module
contract of lit_llama_b200.lora (dense merge bit for bit, quantized bases never merged), patch_reference() on the LoRA
surface (the silent drop of every lora_A / lora_B key it fixes), and b2l_lora_apply's / the step's argument checks,
struct layout, launch count and refusals (all decided before any launch)."""
import ctypes as C
import inspect
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
from lit_llama_b200 import lora as PL
from lit_llama_b200.utils import quantization
from oracle import llama_oracle as O
from oracle import lora_oracle as LO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden():
    return load_golden("tiny_lora_bf16.pt")


def golden_sd(g):
    c = g["cfg"]
    sd = O.synth_state_dict(c["n_layer"], c["n_head"], c["n_embd"], c["vocab_size"], None, seed=g["seed"])
    sd.update(LO.lora_weights(c["n_layer"], c["n_embd"], r=g["lora"]["r"], seed=g["lora_seed"]))
    return sd


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_oracle_branch_matches_reference_merged_linear_bit_for_bit():
    for case in golden()["merged_linear_cases"]:
        x = case["x"]
        base = torch.nn.functional.linear(x, case["weight"])
        got = LO.lora_branch(x, base, case["lora_A"], case["lora_B"], case["alpha"] / case["r"], case["enable_lora"])
        assert torch.equal(got, case["y"])
        # the 2-D form (which the reference's zero_pad cannot take) gives the same rows
        got2 = LO.lora_branch(x[0], base[0], case["lora_A"], case["lora_B"], case["alpha"] / case["r"], case["enable_lora"])
        assert torch.equal(got2, case["y"][0])
        # the branch is not vacuous
        assert not torch.equal(base, case["y"])


def _dense_model(g, **lora_kw):
    c = g["cfg"]
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with PL.lora(**(lora_kw or g["lora"])):
            m = P.LLaMA(P.LLaMAConfig(**c))
    finally:
        torch.set_default_dtype(prev)
    return m


def test_dense_merge_is_the_reference_merge_bit_for_bit():
    g = golden()
    m = _dense_model(g)
    assert sorted(m.state_dict().keys()) == g["state_dict_keys"]
    sd = golden_sd(g)
    res = m.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    assert not m.transformer.h[0].attn.c_attn.merged
    m.eval()
    for blk, want in zip(m.transformer.h, g["merged_c_attn"]):
        assert blk.attn.c_attn.merged and torch.equal(blk.attn.c_attn.weight.data, want)
    m.train()   # unmerge: back to (nearly) the loaded weight, the reference's arithmetic
    assert not m.transformer.h[0].attn.c_attn.merged
    w0 = sd["transformer.h.0.attn.c_attn.weight"]
    assert (m.transformer.h[0].attn.c_attn.weight.data.float() - w0.float()).abs().max() < 1e-2


def test_module_contract():
    g = golden()
    m = _dense_model(g)
    c = m.transformer.h[0].attn.c_attn
    assert isinstance(m.transformer.h[0].attn, PL.CausalSelfAttention) and isinstance(c, PL.MergedLinear)
    assert isinstance(c, PL.LoRALayer) and isinstance(c, torch.nn.Linear)
    assert c.lora_A.shape == (16, 128) and c.lora_B.shape == (256, 8) and c.scaling == 2.0 and c.enable_lora == [True, False, True]
    assert torch.count_nonzero(c.lora_B) == 0   # zero-init (lora.py:203)
    assert isinstance(c.lora_dropout, torch.nn.Dropout) and c.lora_dropout.p == 0.05
    assert P.model.CausalSelfAttention is not PL.CausalSelfAttention   # lora() restored the plain class
    assert PL.CausalSelfAttention.lora_config is None
    for name in ("LoRALayer", "MergedLinear", "LoRAConfig", "CausalSelfAttention", "lora", "mark_only_lora_as_trainable",
                 "lora_state_dict"):
        assert hasattr(PL, name)
    assert list(inspect.signature(PL.lora).parameters) == ["r", "alpha", "dropout", "enabled"]
    assert list(inspect.signature(PL.MergedLinear.__init__).parameters)[:9] == [
        "self", "in_features", "out_features", "r", "lora_alpha", "lora_dropout", "enable_lora", "fan_in_fan_out",
        "merge_weights"]
    assert PL.LoRAConfig() == PL.LoRAConfig(r=0.0, alpha=1.0, dropout=0.0)
    PL.mark_only_lora_as_trainable(m)
    assert {n for n, p in m.named_parameters() if p.requires_grad} == {
        f"transformer.h.{i}.attn.c_attn.lora_{x}" for i in range(2) for x in "AB"}
    assert set(PL.lora_state_dict(m)) == {f"transformer.h.{i}.attn.c_attn.lora_{x}" for i in range(2) for x in "AB"}
    with PL.lora(r=8, alpha=16, dropout=0.0, enabled=False):
        plain = P.LLaMA(P.LLaMAConfig(**g["cfg"]))
    assert type(plain.transformer.h[0].attn) is P.CausalSelfAttention


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8", "llm.int8"])
def test_quantized_base_keys_and_no_merge(mode):
    """Under quantization(mode) c_attn is a LoRA layer over the quantized class: the base's buffers plus lora_A /
    lora_B; a base checkpoint then a LoRA checkpoint (both strict=False) leave nothing unexpected; eval() never
    merges; loading LoRA weights bumps the weight generation."""
    cfg = dict(block_size=16, vocab_size=64, n_layer=2, n_head=2, n_embd=128)
    with quantization(mode), PL.lora(r=8, alpha=16, dropout=0.05):
        m = P.LLaMA(P.LLaMAConfig(**cfg))
    c = m.transformer.h[1].attn.c_attn
    base = P.Linear8bitLt if mode == "llm.int8" else P.ColBlockQuantizedLinear
    assert isinstance(c, base) and isinstance(c, PL.LoRALayer) and c.lora_A.shape == (16, 128) and c.lora_B.shape == (256, 8)
    if mode != "llm.int8":
        assert c.bits == (4 if mode == "gptq.int4" else 8)
    keys = set(m.state_dict())
    p = "transformer.h.1.attn.c_attn."
    assert {p + "lora_A", p + "lora_B"} <= keys and (p + "weight" in keys) == (mode == "llm.int8")
    sd = O.synth_state_dict(2, 2, 128, 64, None if mode == "llm.int8" else mode)
    lw = LO.lora_weights(2, 128)
    r1 = m.load_state_dict(sd, strict=False)
    assert not r1.unexpected_keys and set(r1.missing_keys) == set(lw)
    from lit_llama_b200.quantization import WEIGHTS_GENERATION

    g0 = WEIGHTS_GENERATION[0]
    r2 = m.load_state_dict(lw, strict=False)
    assert not r2.unexpected_keys and WEIGHTS_GENERATION[0] > g0
    assert torch.equal(c.lora_B.data, lw[p + "lora_B"].to(c.lora_B.dtype))
    m.eval()
    assert not c.merged
    full = dict(sd, **lw)
    r3 = m.load_state_dict(full)
    assert not r3.missing_keys and not r3.unexpected_keys


def test_patch_reference_gives_lora_layers_and_loads_every_lora_key():
    """The silent drop: without the rewiring, `lora()` of the reference swaps lit_llama.model.CausalSelfAttention,
    which the patched LLaMA never reads, so c_attn stays a plain linear and a LoRA checkpoint loaded strict=False
    drops every lora_A / lora_B key as unexpected.  After patch_reference(), lora() (also the name generate/lora.py
    bound) builds LoRA layers and the checkpoint loads with no unexpected key."""
    gd = os.path.join(ROOT, "tests", "golden")
    surface = json.load(open(os.path.join(gd, "reference_surface.json")))["modules"]
    surface.update(json.load(open(os.path.join(gd, "reference_lora_surface.json")))["modules"])
    objs = {}

    def stand_in(origin):
        return objs.setdefault(origin, type(origin.rsplit(".", 1)[-1], (), {"origin": origin}))

    pkg = "lit_llama_lora_surface"
    names = {"pkg": pkg, "model": pkg + ".model", "quant": pkg + ".quantization", "utils": pkg + ".utils",
             "generate": pkg + "_generate", "lora": pkg + ".lora", "generate_lora": pkg + "_generate_lora"}
    mods = {key: types.ModuleType(name) for key, name in names.items()}
    for key, ns in surface.items():
        for name, origin in ns.items():
            setattr(mods[key], name, stand_in(origin))
    ref = {key: dict(vars(mod)) for key, mod in mods.items()}
    sys.modules.update({mod.__name__: mod for mod in mods.values()})
    try:
        saved = P.patch_reference(mods["pkg"])
        for name in ("LoRALayer", "MergedLinear", "LoRAConfig", "CausalSelfAttention", "lora", "mark_only_lora_as_trainable",
                     "lora_state_dict"):
            assert getattr(mods["lora"], name) is getattr(PL, name)
            assert saved[("lora", name)] is ref["lora"][name]
        assert mods["generate_lora"].lora is PL.lora   # `from lit_llama.lora import lora` follows
        assert mods["generate_lora"].LLaMA is P.LLaMA
        cfg = dict(block_size=16, vocab_size=64, n_layer=2, n_head=2, n_embd=64)
        with mods["generate_lora"].lora(r=8, alpha=16, dropout=0.05, enabled=True):
            m = mods["generate_lora"].LLaMA(P.LLaMAConfig(**cfg))
        assert all(isinstance(b.attn.c_attn, PL.MergedLinear) for b in m.transformer.h)
        lw = LO.lora_weights(2, 64, dtype=torch.float32)
        res = m.load_state_dict(lw, strict=False)
        assert not res.unexpected_keys
        assert torch.equal(m.transformer.h[1].attn.c_attn.lora_B.data, lw["transformer.h.1.attn.c_attn.lora_B"])
    finally:
        for mod in mods.values():
            sys.modules.pop(mod.__name__, None)


def test_lora_apply_rejects_bad_arguments(L):
    lib = L.lib()
    p = C.c_void_p(256)

    def call(lo, x=256, ldx=128, norm=None, y=512, ldy=384, M=2, N=384, K=128, flags=0):
        return lib.b2l_lora_apply(lo if lo is None else C.byref(lo), x, ldx, norm, 1e-5, y, ldy, M, N, K, flags, None)

    ok = L.LoRA(256, 512, 2.0, 8, 3, 0b101)
    assert call(None) == -1 and b"null LoRA" in lib.b2l_last_error()
    assert call(L.LoRA(None, 512, 2.0, 8, 3, 5)) == -1 and b"null LoRA" in lib.b2l_last_error()
    assert call(L.LoRA(256, None, 2.0, 8, 3, 5)) == -1
    for r in (0, -1, 65):
        assert call(L.LoRA(256, 512, 2.0, r, 3, 5)) == -2 and b"rank" in lib.b2l_last_error()
    for ng in (0, 33, 5):   # 5 does not divide 384
        assert call(L.LoRA(256, 512, 2.0, 8, ng, 1)) == -2 and b"n_groups" in lib.b2l_last_error()
    for mask in (0, 0b1000):
        assert call(L.LoRA(256, 512, 2.0, 8, 3, mask)) == -2 and b"mask" in lib.b2l_last_error()
    assert call(ok, K=100, ldx=128) == -2 and b"in_features" in lib.b2l_last_error()
    assert call(L.LoRA(264, 512, 2.0, 8, 3, 5)) == -1 and b"aligned" in lib.b2l_last_error()
    assert call(L.LoRA(256, 512, float("nan"), 8, 3, 5)) == -1 and b"scaling" in lib.b2l_last_error()
    assert call(L.LoRA(256, 512, float("inf"), 8, 3, 5)) == -1 and b"scaling" in lib.b2l_last_error()
    assert call(ok, x=None) == -1 and b"null x" in lib.b2l_last_error()
    assert call(ok, x=264) == -1 and b"aligned" in lib.b2l_last_error()
    assert call(ok, norm=264) == -1 and b"aligned" in lib.b2l_last_error()
    assert call(ok, ldx=120) == -1 and call(ok, ldx=132) == -1 and call(ok, ldy=380) == -1 and call(ok, M=-1) == -1
    assert call(ok, flags=8) == -1 and b"flags" in lib.b2l_last_error()
    assert call(ok, M=0) == 0   # nothing to do: no launch
    # every enabled-group pattern of 3 groups and every rank 1..64 passes the checks (M = 0: nothing launched)
    for mask in range(1, 8):
        for r in (1, 7, 8, 64):
            assert call(L.LoRA(256, 512, 2.0, r, 3, mask), M=0) == 0


def test_lora_struct_layout_matches_c_compiler(L, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "int main(void){\n"
        'printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b2l_lora), offsetof(b2l_lora, scaling), '
        "offsetof(b2l_lora, r), offsetof(b2l_lora, n_groups), offsetof(b2l_lora, enabled), "
        "sizeof(b2l_decode_args), offsetof(b2l_decode_args, adapters), offsetof(b2l_decode_args, loras));\n"
        "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    got = [C.sizeof(L.LoRA), L.LoRA.scaling.offset, L.LoRA.r.offset, L.LoRA.n_groups.offset, L.LoRA.enabled.offset,
           C.sizeof(L.DecodeArgs), L.DecodeArgs.adapters.offset, L.DecodeArgs.loras.offset]
    assert [int(v) for v in out] == got


def _decode_args(L, n_layer, n_head, n_embd, loras):
    layers = (L.Layer * n_layer)()
    d = L.DecodeArgs(n_layer=n_layer, n_head=n_head, n_embd=n_embd, n_hidden=4 * n_embd, vocab=128, B=1, S=64,
                     layers=layers, wte=16, ln_f=16, rope=16, idx=16, input_pos=16, ring_start=16, block_size=64, x=16,
                     qkv=16, att=16, hid=16, attn_work=16, logits=16)
    keep = [layers]
    if loras is not None:
        arr = (L.LoRA * n_layer)(*loras)
        keep.append(arr)
        d.loras = C.cast(arr, C.POINTER(L.LoRA))
    return d, keep


def test_decode_step_launch_count_and_refusals(L):
    lib = L.lib()
    lo = L.LoRA(256, 512, 2.0, 8, 3, 0b101)
    none = L.LoRA(None, None, 0.0, 0, 0, 0)
    # 7B: 5 n_layer + 3 launches, plus one per LoRA layer (195 with LoRA in all 32 layers)
    d, keep = _decode_args(L, 32, 32, 4096, [lo] * 32)
    d0, keep0 = _decode_args(L, 32, 32, 4096, None)
    assert lib.b2l_decode_step_launches(C.byref(d0)) == 163 and lib.b2l_decode_step_launches(C.byref(d)) == 195
    d, keep = _decode_args(L, 4, 4, 512, [none, lo, none, lo])
    assert lib.b2l_decode_step_launches(C.byref(d)) == 5 * 4 + 3 + 2
    d.flags = 8   # B2L_F_ATTN_UNFUSED: three attention kernels, the LoRA launch count unchanged
    assert lib.b2l_decode_step_launches(C.byref(d)) == 2 + 4 * (4 + 3) + 1 + 2
    d, keep = _decode_args(L, 4, 4, 512, [none] * 4)
    assert lib.b2l_decode_step_launches(C.byref(d)) == 5 * 4 + 3
    # bad terms are rejected before any launch
    d, keep = _decode_args(L, 4, 4, 512, [none, lo, none, L.LoRA(256, 512, 2.0, 65, 3, 5)])
    assert lib.b2l_decode_step(C.byref(d), None) == -2 and b"rank" in lib.b2l_last_error()
    d, keep = _decode_args(L, 4, 4, 512, [none, L.LoRA(256, None, 2.0, 8, 3, 5), none, none])
    assert lib.b2l_decode_step(C.byref(d), None) == -1 and b"null LoRA" in lib.b2l_last_error()

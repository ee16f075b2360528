"""CPU: multi-LoRA.  b2l_lora_apply_rows and b2l_decode_args::lora_sets against the header (ctypes binding, struct
layout), their refusals before any launch, the step's launch count, and add_lora_adapter's validation."""
import ctypes as C
import os
import subprocess

import pytest
import torch

import __graft_entry__ as entry
import lit_llama_b200 as P
from lit_llama_b200 import lora as PL
from lit_llama_b200.quantization import WEIGHTS_GENERATION
from lit_llama_b200.utils import quantization
from oracle import lora_oracle as LO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_binding_and_layout_match_the_header(L, tmp_path):
    """The new decode-args fields sit at the end: every old offset is what it was, and the C compiler agrees on the
    new ones; the binding of b2l_lora_apply_rows is the header's prototype."""
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "typedef int (*fn_t)(const b2l_lora*, int, const int32_t*, const void*, int, const void*, float, void*, int, int,"
        " int, int, int, b2l_stream_t);\n"
        "int main(void){ fn_t f = b2l_lora_apply_rows; (void)f;\n"
        'printf("%zu %zu %zu %zu %zu %zu %d\\n", sizeof(b2l_decode_args), offsetof(b2l_decode_args, q8_threshold), '
        "offsetof(b2l_decode_args, lora_sets), offsetof(b2l_decode_args, n_lora_sets), "
        "offsetof(b2l_decode_args, lora_row_set), offsetof(b2l_decode_args, loras), B2L_LORA_MAX_SETS);\n"
        "return 0;}\n")
    exe = tmp_path / "layout"
    # -Werror: a prototype that differs from fn_t fails the compile
    subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(prog), "-o", str(exe) + ".o"],
                   check=True)
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe), "-Wl,--unresolved-symbols=ignore-all"],
                   check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    D = L.DecodeArgs
    assert out == [C.sizeof(D), D.q8_threshold.offset, D.lora_sets.offset, D.n_lora_sets.offset, D.lora_row_set.offset,
                   D.loras.offset, L.LORA_MAX_SETS]
    assert D.lora_sets.offset >= D.q8_threshold.offset + 4   # appended after every existing field
    fn = L._SIGS["b2l_lora_apply_rows"]
    assert fn[0] is C.c_int and len(fn[1]) == 14 and fn[1][0] is C.POINTER(L.LoRA) and fn[1][6] is C.c_float


P16 = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its checks or launches nothing


def _sets(L, *terms):
    return (L.LoRA * len(terms))(*terms)


def test_apply_rows_refuses_before_any_launch(L):
    lib = L.lib()
    ok = L.LoRA(P16, P16 + 4096, 2.0, 8, 3, 0b101)
    ok2 = L.LoRA(P16 + 8192, P16 + 12288, 0.5, 64, 3, 0b010)   # another rank, scaling and mask: accepted together

    def call(sets, n=None, row_set=P16, x=P16, ldx=128, norm=None, y=P16, ldy=384, M=4, N=384, K=128, flags=0):
        n = len(sets) if n is None and sets is not None else n
        rc = lib.b2l_lora_apply_rows(sets, n, row_set, x, ldx, norm, 1e-5, y, ldy, M, N, K, flags, None)
        return rc, lib.b2l_last_error().decode()

    rc, msg = call(_sets(L, ok, ok2), row_set=None)
    assert rc == -1 and "null row_set" in msg, msg
    for M in (0, 17, -1):
        rc, msg = call(_sets(L, ok, ok2), M=M)
        assert rc == -2 and f"M = {M}" in msg and "1..16" in msg, msg
    for n in (0, 65):
        rc, msg = call(_sets(L, *([ok] * 65)), n=n)
        assert rc == -2 and "LoRA sets" in msg and "1..64" in msg, msg
    rc, msg = call(None, n=2)
    assert rc == -1 and "null LoRA sets" in msg, msg
    rc, msg = call(_sets(L, ok, L.LoRA(P16, P16, 2.0, 8, 6, 0b1)))
    assert rc == -1 and "n_groups must match" in msg, msg
    # every set goes through b2l_lora_apply's checks; r == 0 is not "no term" here
    for bad, code, word in [(L.LoRA(P16, P16, 2.0, 0, 3, 5), -2, "rank"), (L.LoRA(None, P16, 2.0, 8, 3, 5), -1, "null LoRA"),
                            (L.LoRA(P16 + 8, P16, 2.0, 8, 3, 5), -1, "aligned"), (L.LoRA(P16, P16, 2.0, 8, 3, 0b1000), -2, "mask"),
                            (L.LoRA(P16, P16, float("nan"), 8, 3, 5), -1, "scaling")]:
        rc, msg = call(_sets(L, ok, bad))
        assert rc == code and word in msg and "b2l_lora_apply_rows" in msg, (bad, msg)
    rc, msg = call(_sets(L, ok), x=None)
    assert rc == -1 and "null x" in msg, msg
    rc, msg = call(_sets(L, ok), x=P16 + 8)
    assert rc == -1 and "aligned" in msg, msg
    rc, msg = call(_sets(L, ok), ldx=120)
    assert rc == -1 and "ldx" in msg, msg
    rc, msg = call(_sets(L, ok), flags=8)
    assert rc == -1 and "flags" in msg, msg


def _decode(L, n_layer=4, B=4, **kw):
    layers = (L.Layer * n_layer)()
    d = L.DecodeArgs(n_layer=n_layer, n_head=4, n_embd=512, n_hidden=2048, vocab=128, B=B, S=64, layers=layers, wte=16,
                     ln_f=16, rope=16, idx=16, input_pos=16, ring_start=16, block_size=64, x=16, qkv=16, att=16, hid=16,
                     attn_work=16, logits=16, flags=L.F_PDL | L.F_ROW_POS)
    keep = [layers]
    for k, v in kw.items():
        if k == "lora_sets":   # [n_sets][n_layer] terms
            arr = (L.LoRA * len(v))(*v)
            keep.append(arr)
            v = C.cast(arr, C.POINTER(L.LoRA))
        elif k == "loras":
            arr = (L.LoRA * n_layer)(*v)
            keep.append(arr)
            v = C.cast(arr, C.POINTER(L.LoRA))
        setattr(d, k, v)
    d._keep = keep
    return d


def test_decode_step_refusals_and_launch_count(L):
    lib = L.lib()
    lo = L.LoRA(P16, P16 + 4096, 2.0, 8, 3, 0b101)
    lo2 = L.LoRA(P16, P16 + 4096, 1.0, 4, 3, 0b001)
    none = L.LoRA(None, None, 0.0, 0, 0, 0)
    # 3 sets over 4 layers: layer 0 in every set, layer 1 in set 2 only, layers 2 and 3 in none
    sets = [lo, none, none, none,  lo2, none, none, none,  lo, lo2, none, none]
    base = lib.b2l_decode_step_launches(C.byref(_decode(L)))
    assert base == 2 + 4 * (4 + 1) + 1
    d = _decode(L, lora_sets=sets, n_lora_sets=3, lora_row_set=P16)
    assert lib.b2l_decode_step_launches(C.byref(d)) == base + 2
    assert lib.b2l_decode_step_launches(C.byref(_decode(L, lora_sets=[none] * 8, n_lora_sets=2, lora_row_set=P16))) == base
    # the same count as `loras` with the same layers
    assert lib.b2l_decode_step_launches(C.byref(_decode(L, loras=[lo, lo2, none, none]))) == base + 2

    def refused(code, *words, **kw):
        a = dict(lora_sets=sets, n_lora_sets=3, lora_row_set=P16)
        a.update(kw)
        rc = lib.b2l_decode_step(C.byref(_decode(L, **a)), None)
        msg = lib.b2l_last_error().decode()
        assert rc == code and all(w in msg for w in words), (kw.keys(), rc, msg)

    refused(-2, "lora_sets and loras", loras=[lo, none, none, none])
    refused(-2, "affines", affines=C.cast((L.LayerAffine * 4)(), C.POINTER(L.LayerAffine)))
    refused(-2, "affines", lm_head_affine=L.OutAffine(P16, P16))
    refused(-2, "B2L_F_STEPWISE", flags=L.F_PDL | L.F_STEPWISE | L.F_Q4_BATCH_I8, batch_work=P16)
    refused(-1, "lora_row_set", lora_row_set=None)
    refused(-2, "LoRA sets", "1..64", n_lora_sets=0)
    refused(-2, "LoRA sets", "1..64", n_lora_sets=65)
    refused(-2, "rank", lora_sets=[lo, none, none, L.LoRA(P16, P16, 2.0, 65, 3, 5)], n_lora_sets=1)
    refused(-1, "n_groups must match", lora_sets=[lo, none, none, none, L.LoRA(P16, P16, 2.0, 8, 6, 1), none, none, none],
            n_lora_sets=2)


CFG = dict(block_size=16, vocab_size=64, n_layer=2, n_head=2, n_embd=128)


def _model(mode="gptq.int4", lora=True):
    with quantization(mode), (PL.lora(r=8, alpha=16, dropout=0.0) if lora else PL.lora(0, 1, 0, enabled=False)):
        return P.LLaMA(P.LLaMAConfig(**CFG))


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8", "llm.int8"])
def test_add_lora_adapter(mode):
    """Adapters 1, 2, ... with their own rank and scaling; state_dict() unchanged; the weight generation bumped;
    refusals for a dense base, a model without LoRA, missing / extra keys, a wrong shape and a 64th set."""
    m = _model(mode)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    g0 = WEIGHTS_GENERATION[0]
    assert PL.add_lora_adapter(m, LO.lora_weights(2, 128, r=4, seed=1), alpha=8) == 1
    assert WEIGHTS_GENERATION[0] > g0
    assert PL.add_lora_adapter(m, LO.lora_weights(2, 128, r=64, seed=2)) == 2
    c = m.transformer.h[1].attn.c_attn
    A, B, scaling, r = c._adapters[0]
    assert (A.dtype, tuple(A.shape), tuple(B.shape), scaling, r) == (torch.bfloat16, (8, 128), (256, 4), 2.0, 4)
    assert c._adapters[1][2:] == (0.25, 64)
    spec, _ = c.lora_set(2)
    assert (spec.r, spec.n_groups, spec.enabled, spec.scaling) == (64, 3, 0b101, 0.25)
    sd1 = m.state_dict()

    def same(a, b):   # bit for bit (the model was never loaded: its buffers may hold NaN)
        return a.shape == b.shape and torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))

    assert set(sd1) == set(sd0) and all(same(sd1[k], sd0[k]) for k in sd0)

    lw = LO.lora_weights(2, 128, seed=3)
    with pytest.raises(ValueError, match="missing"):
        PL.add_lora_adapter(m, {k: v for k, v in lw.items() if "h.1." not in k})
    with pytest.raises(ValueError, match="unexpected"):
        PL.add_lora_adapter(m, dict(lw, **{"transformer.h.0.attn.c_proj.lora_A": lw["transformer.h.0.attn.c_attn.lora_A"]}))
    bad = dict(lw)
    bad["transformer.h.0.attn.c_attn.lora_B"] = torch.zeros(128, 4)   # r = 8 from lora_A
    with pytest.raises(ValueError, match="do not fit"):
        PL.add_lora_adapter(m, bad)
    bad = dict(lw)
    bad["transformer.h.0.attn.c_attn.lora_A"] = torch.zeros(16, 64)   # in_features 128
    with pytest.raises(ValueError, match="do not fit"):
        PL.add_lora_adapter(m, bad)
    assert len(c._adapters) == 2   # nothing was registered by a refused call
    while len(c._adapters) < 63:
        PL.add_lora_adapter(m, lw)
    with pytest.raises(ValueError, match="63 adapters"):
        PL.add_lora_adapter(m, lw)

    with pytest.raises(ValueError, match="no LoRA layers"):
        PL.add_lora_adapter(_model(mode, lora=False), lw)
    with PL.lora(r=8, alpha=16, dropout=0.0):
        dense = P.LLaMA(P.LLaMAConfig(**CFG))
    with pytest.raises(ValueError, match="dense base"):
        PL.add_lora_adapter(dense, lw)


def test_adapter_ids_are_checked():
    m = _model()
    PL.add_lora_adapter(m, LO.lora_weights(2, 128, seed=1))
    assert m._check_adapters([-1, 0, 1], 3, "t") == [-1, 0, 1]
    for ids in ([2], [-2], [0, 0]):
        with pytest.raises(ValueError, match=r"ids in -1\.\.1"):
            m._check_adapters(ids, 1, "t")
    with pytest.raises(ValueError, match="LoRA model"):
        _model(lora=False)._check_adapters([0], 1, "t")

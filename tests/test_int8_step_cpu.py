"""CPU: the C ABI of llm.int8 on the whole-token step -- b2l_q8_linear_args / b2l_q8_weight / b2l_q8_layer and the
appended b2l_decode_args members laid out as a C compiler lays them out, the launch count of a B2L_F_Q8 step, and
every refusal of b2l_q8_linear and of b2l_decode_step under B2L_F_Q8 (all before the device is touched)."""
import ctypes as C
import os
import subprocess

import pytest

import __graft_entry__ as entry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20   # a 16-byte aligned non-NULL address: every call below is refused before it is dereferenced


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_struct_layout_matches_c_compiler(L, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "int main(void){\n"
        'printf("%zu %zu %zu %zu\\n", sizeof(b2l_q8_linear_args), sizeof(b2l_q8_weight), sizeof(b2l_q8_layer), sizeof(b2l_decode_args));\n'
        'printf("%zu %zu %zu %zu %zu\\n", offsetof(b2l_q8_linear_args, threshold), offsetof(b2l_q8_linear_args, out_affine), '
        "offsetof(b2l_q8_linear_args, flags), offsetof(b2l_q8_layer, mlp_proj), offsetof(b2l_decode_args, lm_head_affine));\n"
        'printf("%zu %zu %zu\\n", offsetof(b2l_decode_args, q8_layers), offsetof(b2l_decode_args, q8_lm_head), '
        "offsetof(b2l_decode_args, q8_threshold));\n"
        "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    got = [C.sizeof(L.Q8LinearArgs), C.sizeof(L.Q8Weight), C.sizeof(L.Q8Layer), C.sizeof(L.DecodeArgs),
           L.Q8LinearArgs.threshold.offset, L.Q8LinearArgs.out_affine.offset, L.Q8LinearArgs.flags.offset,
           L.Q8Layer.mlp_proj.offset, L.DecodeArgs.lm_head_affine.offset,
           L.DecodeArgs.q8_layers.offset, L.DecodeArgs.q8_lm_head.offset, L.DecodeArgs.q8_threshold.offset]
    assert out == got
    assert L.F_Q8 == 64


# ------------------------------------------------------------------------------------------- b2l_q8_linear
def _args(L, **kw):
    a = L.Q8LinearArgs(x=FAKE, cb=FAKE * 2, scb=FAKE * 3, y=FAKE * 4, N=4096, K=4096, threshold=6.0,
                       prologue=L.PRO_RMSNORM, norm_scale=FAKE * 5, eps=1e-5, epilogue=L.EPI_STORE)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(x=None), -1, b"null pointer"),
    (dict(cb=None), -1, b"null pointer"),
    (dict(scb=None), -1, b"null pointer"),
    (dict(y=None), -1, b"null pointer"),
    (dict(K=4000), -2, b"multiple of 128"),
    (dict(K=32768 + 128), -2, b"<= 32768"),
    (dict(K=0), -2, b"multiple of 128"),
    (dict(N=0), -1, b"bad shape"),
    (dict(prologue=2), -1, b"bad prologue"),
    (dict(epilogue=3), -1, b"bad epilogue"),
    (dict(norm_scale=None), -1, b"norm_scale"),
    (dict(epilogue=1), -1, b"RESIDUAL needs res"),
    (dict(epilogue=2), -1, b"SWIGLU needs cb2"),
    (dict(epilogue=2, cb2=FAKE * 6), -1, b"SWIGLU needs cb2"),
    (dict(x=FAKE + 8), -1, b"16-byte aligned"),
    (dict(cb=FAKE * 2 + 4), -1, b"16-byte aligned"),
    (dict(norm_scale=FAKE * 5 + 2), -1, b"16-byte aligned"),
    (dict(epilogue=2, cb2=FAKE * 6 + 8, scb2=FAKE * 7), -1, b"16-byte aligned"),
    (dict(y=FAKE + 4096), -1, b"overlaps"),
    (dict(flags=2), -2, b"unknown flags"),
])
def test_q8_linear_refusals(L, kw, rc, msg):
    a = _args(L, **kw)
    assert L.lib().b2l_q8_linear(C.byref(a), None) == rc
    assert msg in L.lib().b2l_last_error()


def test_q8_linear_refuses_half_an_affine_and_null_args(L):
    a = _args(L)
    a.out_affine = L.OutAffine(FAKE * 8, None)
    assert L.lib().b2l_q8_linear(C.byref(a), None) == -1 and b"both scale and bias" in L.lib().b2l_last_error()
    assert L.lib().b2l_q8_linear(None, None) == -1


# ------------------------------------------------------------------------------------------- b2l_decode_step
def _decode(L, n_layer=2, C_=512, H=1536, vocab=256, **kw):
    keep = []
    layers = (L.Layer * n_layer)()
    q8 = (L.Q8Layer * n_layer)()
    w = lambda N, K: L.Q8Weight(FAKE, FAKE, N, K)  # noqa: E731
    for i in range(n_layer):
        layers[i] = L.Layer(rms_1=FAKE, rms_2=FAKE, k_cache=FAKE, v_cache=FAKE)
        q8[i] = L.Q8Layer(w(3 * C_, C_), w(C_, C_), w(H, C_), w(H, C_), w(C_, H))
    keep += [layers, q8]
    d = L.DecodeArgs(n_layer=n_layer, n_head=C_ // 128, n_embd=C_, n_hidden=H, vocab=vocab, B=1, S=64, eps=1e-5,
                     layers=C.cast(layers, C.POINTER(L.Layer)), wte=FAKE, ln_f=FAKE, rope=FAKE, idx=FAKE, input_pos=FAKE,
                     ring_start=FAKE, block_size=64, x=FAKE, qkv=FAKE, att=FAKE, hid=FAKE, attn_work=FAKE, logits=FAKE,
                     flags=L.F_PDL | L.F_Q8, q8_layers=C.cast(q8, C.POINTER(L.Q8Layer)), q8_lm_head=w(vocab, C_),
                     q8_threshold=6.0)
    for k, v in kw.items():
        setattr(d, k, v)
    d._keep = keep
    return d, q8


def test_launch_count(L):
    d, _ = _decode(L, n_layer=3)
    assert L.lib().b2l_decode_step_launches(C.byref(d)) == 5 * 3 + 3
    loras = (L.LoRA * 3)()
    for i in range(3):
        loras[i] = L.LoRA(FAKE, FAKE, 2.0, 8, 3, 5)
    d.loras = C.cast(loras, C.POINTER(L.LoRA))
    assert L.lib().b2l_decode_step_launches(C.byref(d)) == 5 * 3 + 3 + 3


def _refused(L, d, rc, msg):
    assert L.lib().b2l_decode_step(C.byref(d), None) == rc
    assert msg in L.lib().b2l_last_error(), L.lib().b2l_last_error()


def test_step_refusals(L):
    d, q8 = _decode(L)
    d.flags |= L.F_W8
    _refused(L, d, -2, b"exclude each other")
    d, q8 = _decode(L, B=2)
    _refused(L, d, -2, b"batch 1 only")
    d, q8 = _decode(L)
    d.q8_layers = None
    _refused(L, d, -1, b"needs q8_layers")
    d, q8 = _decode(L)
    q8[1].c_fc2.cb = None
    _refused(L, d, -1, b"c_fc2 of layer 1 has no CB")
    d, q8 = _decode(L)
    q8[0].mlp_proj.K = 1024
    _refused(L, d, -1, b"mlp.c_proj of layer 0 is [512, 1024]")
    d, q8 = _decode(L)
    d.q8_lm_head.cb = FAKE + 8
    _refused(L, d, -1, b"16-byte aligned")
    d, q8 = _decode(L, C_=512, H=1000)   # in_features of mlp.c_proj not a multiple of 128
    _refused(L, d, -2, b"multiple of 128")
    d, q8 = _decode(L, C_=512, H=33024)
    _refused(L, d, -2, b"<= 32768")

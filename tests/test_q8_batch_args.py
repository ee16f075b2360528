"""CPU: b2l_q8_linear_batch (llm.int8 at 2..16 rows) and B2L_F_Q8_BATCH in b2l_decode_step -- the header and the
ctypes binding agree, every refusal comes with a message before the device is touched, and the launch counts."""
import ctypes as C
import os
import re

import pytest

import __graft_entry__ as entry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20   # a 16-byte aligned non-NULL address: every call below is refused before it is dereferenced


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_header_and_binding_agree(L):
    h = open(os.path.join(ROOT, "include", "b2l.h")).read()
    assert re.search(r"B2L_F_Q8_BATCH = 512\b", h) and L.F_Q8_BATCH == 512
    assert "size_t b2l_q8_linear_batch_workspace_bytes(int K, int M);" in h
    assert re.search(r"int b2l_q8_linear_batch\(const b2l_q8_linear_args\* args, int M, void\* workspace, size_t workspace_bytes,"
                     r"\s+b2l_stream_t stream\);", h)
    lib = L.lib()
    assert lib.b2l_q8_linear_batch.argtypes == [C.POINTER(L.Q8LinearArgs), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    assert lib.b2l_q8_linear_batch_workspace_bytes.restype == C.c_size_t


def test_workspace_bytes(L):
    ws = L.lib().b2l_q8_linear_batch_workspace_bytes
    # CA (M K) + SCA / count (80 B) + outlier columns (4 K) + fp16 x^ on them (2 M K)
    assert ws(32768, 16) == 16 * 32768 * 3 + 80 + 4 * 32768
    assert ws(4096, 2) == 2 * 4096 * 3 + 80 + 4 * 4096
    for K, M in ((4096, 8), (11008, 5), (22016, 16)):
        assert ws(K, M) >= ws(K - 128, M) and ws(K, M) >= ws(K, M - 1)
    for K, M in ((4000, 4), (0, 4), (32768 + 128, 4), (4096, 1), (4096, 17)):
        assert ws(K, M) == 0, (K, M)


# ------------------------------------------------------------------------------------------- b2l_q8_linear_batch
def _args(L, **kw):
    a = L.Q8LinearArgs(x=FAKE, cb=FAKE * 2, scb=FAKE * 3, y=FAKE * 4, N=4096, K=4096, threshold=6.0,
                       prologue=L.PRO_RMSNORM, norm_scale=FAKE * 5, eps=1e-5, epilogue=L.EPI_STORE)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


WS = FAKE * 16


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(x=None), -1, b"null pointer"),
    (dict(cb=None), -1, b"null pointer"),
    (dict(scb=None), -1, b"null pointer"),
    (dict(y=None), -1, b"null pointer"),
    (dict(M=1), -2, b"M=1 (2..16"),
    (dict(M=17), -2, b"M=17 (2..16"),
    (dict(M=0), -2, b"M=0 (2..16"),
    (dict(K=4000), -2, b"multiple of 128"),
    (dict(K=32768 + 128), -2, b"<= 32768"),
    (dict(N=0), -1, b"bad shape"),
    (dict(prologue=2), -1, b"bad prologue"),
    (dict(epilogue=3), -1, b"bad epilogue"),
    (dict(norm_scale=None), -1, b"norm_scale"),
    (dict(epilogue=1), -1, b"RESIDUAL needs res"),
    (dict(epilogue=2), -1, b"SWIGLU needs cb2"),
    (dict(epilogue=2, cb2=FAKE * 6), -1, b"SWIGLU needs cb2"),
    (dict(ws=None), -1, b"null workspace"),
    (dict(x=FAKE + 8), -1, b"16-byte aligned"),
    (dict(cb=FAKE * 2 + 4), -1, b"16-byte aligned"),
    (dict(norm_scale=FAKE * 5 + 2), -1, b"16-byte aligned"),
    (dict(epilogue=2, cb2=FAKE * 6 + 8, scb2=FAKE * 7), -1, b"16-byte aligned"),
    (dict(ws=WS + 8), -1, b"16-byte aligned"),
    (dict(nbytes=-1), -1, b"too small"),
    (dict(y=FAKE + 4 * 4096 * 2 - 16), -1, b"overlaps"),   # x spans M rows: 4 x 4096 x 2 bytes
    (dict(y=FAKE - 4 * 4096 * 2 + 2), -1, b"overlaps"),
    (dict(flags=2), -2, b"unknown flags"),
    (dict(flags=512), -2, b"unknown flags"),
])
def test_linear_batch_refusals(L, kw, rc, msg):
    kw = dict(kw)
    M = kw.pop("M", 4)
    ws = kw.pop("ws", WS)
    nbytes = L.lib().b2l_q8_linear_batch_workspace_bytes(4096, max(2, min(M, 16))) + kw.pop("nbytes", 0)
    a = _args(L, **kw)
    assert L.lib().b2l_q8_linear_batch(C.byref(a), M, ws, nbytes, None) == rc
    assert msg in L.lib().b2l_last_error(), L.lib().b2l_last_error()


def test_linear_batch_refuses_half_an_affine_and_null_args(L):
    a = _args(L)
    a.out_affine = L.OutAffine(FAKE * 8, None)
    nb = L.lib().b2l_q8_linear_batch_workspace_bytes(4096, 4)
    assert L.lib().b2l_q8_linear_batch(C.byref(a), 4, WS, nb, None) == -1
    assert b"both scale and bias" in L.lib().b2l_last_error()
    assert L.lib().b2l_q8_linear_batch(None, 4, WS, nb, None) == -1


# ------------------------------------------------------------------------------------------- b2l_decode_step
def _decode(L, n_layer=2, C_=512, H=1536, vocab=256, B=4, **kw):
    keep = []
    layers = (L.Layer * n_layer)()
    q8 = (L.Q8Layer * n_layer)()
    w = lambda N, K: L.Q8Weight(FAKE, FAKE, N, K)  # noqa: E731
    for i in range(n_layer):
        layers[i] = L.Layer(rms_1=FAKE, rms_2=FAKE, k_cache=FAKE, v_cache=FAKE)
        q8[i] = L.Q8Layer(w(3 * C_, C_), w(C_, C_), w(H, C_), w(H, C_), w(C_, H))
    keep += [layers, q8]
    d = L.DecodeArgs(n_layer=n_layer, n_head=C_ // 128, n_embd=C_, n_hidden=H, vocab=vocab, B=B, S=64, eps=1e-5,
                     layers=C.cast(layers, C.POINTER(L.Layer)), wte=FAKE, ln_f=FAKE, rope=FAKE, idx=FAKE, input_pos=FAKE,
                     ring_start=FAKE, block_size=64, x=FAKE, qkv=FAKE, att=FAKE, hid=FAKE, attn_work=FAKE, logits=FAKE,
                     flags=L.F_PDL | L.F_Q8 | L.F_Q8_BATCH, q8_layers=C.cast(q8, C.POINTER(L.Q8Layer)),
                     q8_lm_head=w(vocab, C_), q8_threshold=6.0, batch_work=FAKE)
    for k, v in kw.items():
        setattr(d, k, v)
    d._keep = keep
    return d, q8


def _refused(L, d, rc, *words):
    assert L.lib().b2l_decode_step(C.byref(d), None) == rc
    msg = L.lib().b2l_last_error().decode()
    assert all(w in msg for w in words), msg


def test_step_refuses_the_flag_outside_its_combinations(L):
    d, _ = _decode(L, flags=L.F_PDL | L.F_Q8_BATCH)
    _refused(L, d, -2, "B2L_F_Q8_BATCH needs B2L_F_Q8")
    for other in (L.F_W8, L.F_W8 | L.F_W8_BATCH):
        d, _ = _decode(L, flags=L.F_PDL | L.F_Q8 | L.F_Q8_BATCH | other)
        _refused(L, d, -2, "exclude each other")
    d, _ = _decode(L, flags=L.F_PDL | L.F_Q8 | L.F_Q8_BATCH | L.F_W8_BATCH)
    _refused(L, d, -2, "B2L_F_Q8_BATCH", "does not combine")
    d, _ = _decode(L, flags=L.F_PDL | L.F_Q8 | L.F_Q8_BATCH | L.F_Q4_BATCH_I8)
    _refused(L, d, -2, "does not combine")
    d, _ = _decode(L, B=1)
    _refused(L, d, -2, "B2L_F_Q8_BATCH", "2..16", "B=1")
    d, _ = _decode(L, B=17)
    _refused(L, d, -2, "batch 17 > 16")
    d, _ = _decode(L, batch_work=None)
    _refused(L, d, -1, "B2L_F_Q8_BATCH", "batch_work")
    d, q8 = _decode(L)
    q8[1].c_fc2.cb = None
    _refused(L, d, -1, "c_fc2 of layer 1 has no CB")


def test_q8_at_batch_two_without_the_flag_stays_batch_1_only(L):
    d, _ = _decode(L, B=2, flags=L.F_PDL | L.F_Q8)
    _refused(L, d, -2, "batch 1 only")


def test_v2_affines_at_batch_two_only_under_the_flag(L):
    layer_aff = (L.LayerAffine * 2)()
    aff = dict(affines=C.cast(layer_aff, C.POINTER(L.LayerAffine)))
    # without the flag: refused for the batch (B2L_F_Q8 at B = 2) or for the affines (any other route)
    d, _ = _decode(L, B=2, flags=L.F_PDL | L.F_Q8, **aff)
    _refused(L, d, -2, "batch 1 only")
    d, _ = _decode(L, B=2, flags=L.F_PDL, **aff)
    _refused(L, d, -2, "affines run at batch 1 only")
    # half an affine is still a bad argument under the flag: the affine checks run, and accept whole ones
    d, _ = _decode(L, B=2, lm_head_affine=L.OutAffine(FAKE, None), **aff)
    _refused(L, d, -1, "lm_head_affine needs both")
    lo = (L.LoRA * 2)()
    d, _ = _decode(L, B=2, lm_head_affine=L.OutAffine(FAKE, FAKE), loras=C.cast(lo, C.POINTER(L.LoRA)), **aff)
    _refused(L, d, -2, "affines and LoRA do not combine")


def test_launch_counts(L):
    lib = L.lib()
    for B in (2, 8, 9, 16):
        d, _ = _decode(L, n_layer=3, B=B)
        # ring advance + embedding, per Block 4 linears (2 launches each) + attention, ln_f + lm_head (2 launches)
        assert lib.b2l_decode_step_launches(C.byref(d)) == 2 + 3 * (4 * 2 + 1) + 2, B
    loras = (L.LoRA * 3)()
    for i in range(3):
        loras[i] = L.LoRA(FAKE, FAKE, 2.0, 8, 3, 5)
    d, _ = _decode(L, n_layer=3, B=12, loras=C.cast(loras, C.POINTER(L.LoRA)))
    assert lib.b2l_decode_step_launches(C.byref(d)) == 2 + 3 * (4 * 2 + 1) + 2 + 3
    # batch 1 under B2L_F_Q8: one launch per linear, as before
    d, _ = _decode(L, n_layer=3, B=1, flags=L.F_PDL | L.F_Q8, batch_work=None)
    assert lib.b2l_decode_step_launches(C.byref(d)) == 5 * 3 + 3

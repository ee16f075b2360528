"""CPU: b2l_w8_gemv_batch (gptq.int8 at 2..16 rows) and B2L_F_W8 | B2L_F_W8_BATCH in b2l_decode_step reject bad
arguments with a message before they touch the device; workspace sizes and launch counts."""
import ctypes as C

import pytest

import __graft_entry__ as entry


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


P = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first


def _args(L, **kw):
    a = dict(x=P, ldx=1024, qw_tiled=P, scales=P, zeros=P, sz_dtype=L.B2L_BF16, y=P, ldy=256, M=4, N=256, K=1024,
             prologue=L.PRO_NONE, norm_scale=None, eps=1e-5, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=0,
             workspace=P)
    a.update(kw)
    return L.Q4LinearArgs(**a)


def test_gemv_batch_rejects_bad_arguments_with_a_message(L):
    lib = L.lib()

    def call(**kw):
        return lib.b2l_w8_gemv_batch(C.byref(_args(L, **kw)), None), lib.b2l_last_error().decode()

    assert lib.b2l_w8_gemv_batch(None, None) == -1 and "null args" in lib.b2l_last_error().decode()
    for kw in ("x", "qw_tiled", "scales", "zeros", "y"):
        rc, msg = call(**{kw: None})
        assert rc == -1 and "b2l_w8_gemv_batch" in msg and "null pointer" in msg, (kw, msg)
    rc, msg = call(workspace=None)
    assert rc == -1 and "workspace" in msg, msg
    rc, msg = call(out_affine=L.OutAffine(P, P))
    assert rc == -2 and "out_affine" in msg, msg
    rc, msg = call(out_affine=L.OutAffine(P, None))
    assert rc == -2 and "out_affine" in msg, msg
    for m in (0, 1, 17):
        rc, msg = call(M=m)
        assert rc == -2 and f"M={m}" in msg and "2..16" in msg, (m, msg)
    for k in (1000, 96):
        rc, msg = call(K=k, ldx=1024)
        assert rc == -2 and "multiple of 64" in msg, msg
    rc, msg = call(K=24576 + 64, ldx=24576 + 64)
    assert rc == -2 and "<= 24576" in msg, msg
    rc, msg = call(ldx=1028)
    assert rc == -1 and "ldx" in msg, msg
    rc, msg = call(ldx=512)
    assert rc == -1 and "ldx" in msg, msg
    for kw in ("x", "qw_tiled", "workspace"):
        rc, msg = call(**{kw: P + 8})
        assert rc == -1 and "16-byte aligned" in msg, (kw, msg)
    for flags in (2, 4, 16, 32, 128, 1 << 20):
        rc, msg = call(flags=flags)
        assert rc == -2 and "unknown flags" in msg, (flags, msg)
    rc, msg = call(epilogue=L.EPI_RESIDUAL)
    assert rc == -1 and "needs res" in msg, msg
    rc, msg = call(epilogue=L.EPI_SWIGLU, N=264, ldy=132)
    assert rc == -2 and "N % 16" in msg, msg
    rc, msg = call(prologue=L.PRO_RMSNORM)
    assert rc == -1 and "RMSNorm" in msg, msg
    rc, msg = call(sz_dtype=7)
    assert rc == -1 and "sz_dtype" in msg, msg


def test_batch1_kernel_still_refuses_two_rows(L):
    lib = L.lib()
    assert lib.b2l_w8_gemv(C.byref(_args(L, M=2)), None) == -2
    msg = lib.b2l_last_error().decode()
    assert "b2l_w8_gemv: M=2" in msg and "batch-1" in msg, msg


def test_workspace_bytes(L):
    lib = L.lib()
    # [K/64][3 M planes][64 B] digits, then int64 sum X [16] and int sh [16]
    for K, M in [(64, 2), (4096, 2), (4096, 8), (11008, 16), (22016, 16), (24576, 16)]:
        assert lib.b2l_w8_gemv_batch_workspace_bytes(K, M) == 3 * M * K + 16 * 12
    for K, M in [(96, 4), (0, 4), (4096, 1), (4096, 17), (-64, 4)]:
        assert lib.b2l_w8_gemv_batch_workspace_bytes(K, M) == 0


def _decode(L, **kw):
    layers = (L.Layer * 1)()
    base = dict(n_layer=1, n_head=4, n_embd=512, n_hidden=1536, vocab=128, B=4, S=16, sz_dtype=L.B2L_BF16, eps=1e-5,
                layers=layers, wte=P, ln_f=P, rope=P, idx=P, idx_is_i64=1, input_pos=P, ring_start=P, block_size=16,
                x=P, qkv=P, att=P, hid=P, attn_work=P, logits=P, flags=L.F_PDL | L.F_W8 | L.F_W8_BATCH, batch_work=P)
    base.update(kw)
    a = L.DecodeArgs(**base)
    a._layers = layers
    return a


def test_decode_step_accepts_the_batch_flag_only_in_its_combinations(L):
    lib = L.lib()

    def refused(rc_want, *words, **kw):
        rc = lib.b2l_decode_step(C.byref(_decode(L, **kw)), None)
        msg = lib.b2l_last_error().decode()
        assert rc == rc_want and all(w in msg for w in words), (kw, rc, msg)

    refused(-2, "B2L_F_W8_BATCH needs B2L_F_W8", flags=L.F_PDL | L.F_W8_BATCH)
    refused(-2, "exclude each other", flags=L.F_PDL | L.F_W8 | L.F_W8_BATCH | L.F_Q8)
    layer_aff = (L.LayerAffine * 1)()
    refused(-2, "affines", affines=C.cast(layer_aff, C.POINTER(L.LayerAffine)))
    refused(-2, "affines", lm_head_affine=L.OutAffine(P, P))
    refused(-2, "2..16", "B=1", B=1)
    refused(-2, "batch 17 > 16", B=17)   # the step's own bound comes first
    refused(-1, "batch_work", batch_work=None)
    # without the new flag, B2L_F_W8 at B >= 2 is refused as before
    refused(-2, "B2L_F_W8", "batch 1", flags=L.F_PDL | L.F_W8)


def test_decode_step_launches(L):
    lib = L.lib()
    # head_size 128: ring advance + embedding, per Block 4 linears (2 launches each) + 1 attention, lm_head (2 launches)
    for B in (2, 9, 16):
        a = _decode(L, B=B)
        assert lib.b2l_decode_step_launches(C.byref(a)) == 2 + (4 * 2 + 1) + 2
    # a LoRA layer adds one launch
    loras = (L.LoRA * 1)()
    loras[0].r = 8
    a = _decode(L, B=8, loras=C.cast(loras, C.POINTER(L.LoRA)))
    assert lib.b2l_decode_step_launches(C.byref(a)) == 2 + (4 * 2 + 1) + 2 + 1
    # batch 1 on B2L_F_W8 alone: unchanged
    a = _decode(L, B=1, flags=L.F_PDL | L.F_W8, batch_work=None)
    assert lib.b2l_decode_step_launches(C.byref(a)) == 2 + 5 + 1

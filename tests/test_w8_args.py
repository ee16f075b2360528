"""CPU: the gptq.int8 entry points (b2l_w8_gemv, b2l_w8_gemm, the b2l_w8_tile_i8 tiling and B2L_F_W8 in
b2l_decode_step) reject bad arguments with a message before they touch the device."""
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
    a = dict(x=P, ldx=1024, qw_tiled=P, scales=P, zeros=P, sz_dtype=L.B2L_BF16, y=P, ldy=256, M=1, N=256, K=1024,
             prologue=L.PRO_NONE, norm_scale=None, eps=1e-5, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=0)
    a.update(kw)
    return L.Q4LinearArgs(**a)


@pytest.mark.parametrize("fn", ["b2l_w8_gemv", "b2l_w8_gemm"])
def test_bad_arguments_are_rejected_with_a_message(L, fn):
    lib = L.lib()

    def call(**kw):
        return getattr(lib, fn)(C.byref(_args(L, **kw)), None), lib.b2l_last_error().decode()

    assert getattr(lib, fn)(None, None) == -1 and "null args" in lib.b2l_last_error().decode()
    for kw in ("x", "qw_tiled", "scales", "zeros", "y"):
        rc, msg = call(**{kw: None})
        assert rc == -1 and fn in msg and "null pointer" in msg, (kw, msg)
    for k in (1000, 96):
        rc, msg = call(K=k, ldx=1024)
        assert rc == -2 and "multiple of 64" in msg, msg
    rc, msg = call(x=P + 8)
    assert rc == -1 and "16-byte aligned" in msg, msg
    rc, msg = call(qw_tiled=P + 4)
    assert rc == -1 and "16-byte aligned" in msg, msg
    for flags in (2, 4, 64, 1 << 20):
        rc, msg = call(flags=flags)
        assert rc == -2 and "unknown flags" in msg, (flags, msg)
    if fn == "b2l_w8_gemm":
        rc, msg = call(flags=1)
        assert rc == -2 and "unknown flags" in msg, msg
        rc, msg = call(M=8, ldx=1001)
        assert rc == -1 and "leading dimension" in msg, msg
        rc, msg = call(prologue=L.PRO_RMSNORM, norm_scale=P)
        assert rc == -2 and "plain linear only" in msg, msg
    else:
        rc, msg = call(K=24576 + 64, ldx=24576 + 64)
        assert rc == -2 and "<= 24576" in msg, msg
        rc, msg = call(M=2)
        assert rc == -2 and "batch-1" in msg, msg
        rc, msg = call(epilogue=L.EPI_RESIDUAL)
        assert rc == -1 and "needs res" in msg, msg


def test_tile_arguments_and_sizes(L):
    lib = L.lib()
    # [ceil(N/16) row blocks][K/64 k blocks][1024 B]: N is padded to a multiple of 16
    assert lib.b2l_w8_tiled_i8_bytes(16, 64) == 1024
    assert lib.b2l_w8_tiled_i8_bytes(17, 64) == 2048
    assert lib.b2l_w8_tiled_i8_bytes(130, 256) == 9 * 4 * 1024
    assert lib.b2l_w8_tiled_i8_bytes(4096, 4096) == 4096 * 4096
    assert lib.b2l_w8_tiled_i8_bytes(22016, 8192) == 22016 * 8192
    assert lib.b2l_w8_tiled_i8_bytes(16, 96) == 0 and lib.b2l_w8_tiled_i8_bytes(0, 64) == 0
    assert lib.b2l_w8_tile_i8(None, P, 16, 64, None) == -1 and b"bad argument" in lib.b2l_last_error()
    assert lib.b2l_w8_untile_i8(P, P, 16, 96, None) == -2 and b"multiple of 64" in lib.b2l_last_error()


def test_decode_step_rejects_w8_with_a_batch(L):
    lib = L.lib()
    layers = (L.Layer * 1)()
    base = dict(n_layer=1, n_head=4, n_embd=512, n_hidden=1536, vocab=128, B=1, S=16, sz_dtype=L.B2L_BF16, eps=1e-5,
                layers=layers, wte=P, ln_f=P, rope=P, idx=P, idx_is_i64=1, input_pos=P, ring_start=P, block_size=16,
                x=P, qkv=P, att=P, hid=P, attn_work=P, logits=P, flags=L.F_PDL | L.F_W8)
    a = L.DecodeArgs(**dict(base, B=2))
    assert lib.b2l_decode_step(C.byref(a), None) == -2
    assert "B2L_F_W8" in lib.b2l_last_error().decode() and "batch 1" in lib.b2l_last_error().decode()
    # the flag leaves the launch count alone (head_size 128: ring advance, embedding, 4 linears + 1 attention, lm_head)
    a = L.DecodeArgs(**base)
    b = L.DecodeArgs(**dict(base, flags=L.F_PDL))
    assert lib.b2l_decode_step_launches(C.byref(a)) == lib.b2l_decode_step_launches(C.byref(b)) == 2 + 5 + 1

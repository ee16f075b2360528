"""CPU: b2l_decode_step resolves one route for its linears and runs every check of every launch before the first one,
so a step that cannot run is refused with a B2L_E_* code and a message without touching the device (here, where there
is no device, a negative code is the proof that nothing was launched).  Launch counts per route."""
import ctypes as C

import pytest

import __graft_entry__ as entry

P = 1 << 20   # a 16-byte aligned non-NULL address: every call below is refused before it is dereferenced


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


# (flags without B2L_F_PDL, B, batch_work, the tiling the route reads) of every gptq route
def _routes(L):
    return {
        "q4 gemv": (0, 1, None, "qw_mma"),
        "q4 batch": (0, 4, P, "qw_mma"),
        "q4 wgmma": (0, 12, None, "qw_tiled"),
        "q4 wgmma at batch 1": (0, 1, None, "qw_tiled"),
        "q4 row-exact batch": (L.F_Q4_BATCH_I8, 4, P, "qw_mma"),
        "w8 gemv": (L.F_W8, 1, None, "qw_mma"),
        "w8 batch": (L.F_W8 | L.F_W8_BATCH, 4, P, "qw_mma"),
    }


def _weight(L, tiling, N, K):
    return L.Q4Weight(P if tiling == "qw_tiled" else None, P if tiling == "qw_mma" else None, P, P, N, K)


def _decode(L, flags, B, batch_work, tiling, n_layer=2, n_head=4, C_=512, H=1536, vocab=256):
    """A step whose every argument passes every check: a test breaks one of them."""
    layers = (L.Layer * n_layer)()
    for i in range(n_layer):
        layers[i] = L.Layer(rms_1=P, rms_2=P, c_attn=_weight(L, tiling, 3 * C_, C_), c_proj=_weight(L, tiling, C_, C_),
                            c_fc12=_weight(L, tiling, 2 * H, C_), mlp_proj=_weight(L, tiling, C_, H), k_cache=P, v_cache=P)
    d = L.DecodeArgs(n_layer=n_layer, n_head=n_head, n_embd=C_, n_hidden=H, vocab=vocab, B=B, S=16, sz_dtype=L.B2L_BF16,
                     eps=1e-5, layers=C.cast(layers, C.POINTER(L.Layer)), wte=P, ln_f=P, lm_head=_weight(L, tiling, vocab, C_),
                     rope=P, idx=P, idx_is_i64=1, input_pos=P, ring_start=P, block_size=16, x=P, qkv=P, att=P, hid=P,
                     attn_work=P, logits=P, flags=L.F_PDL | flags, batch_work=batch_work)
    d._keep = layers
    return d, layers


def _step(L, d):
    return L.lib().b2l_decode_step(C.byref(d), None), L.lib().b2l_last_error().decode()


def test_each_route_refuses_k_outside_its_kernel(L):
    for name, (flags, B, bw, tiling) in _routes(L).items():
        d, layers = _decode(L, flags, B, bw, tiling)
        layers[1].mlp_proj.K = 1000
        rc, msg = _step(L, d)
        assert rc == -2 and msg.startswith("b2l_decode_step: mlp.c_proj of layer 1: ") and "K=1000 must be a multiple of" in msg, \
            (name, rc, msg)
        if tiling == "qw_tiled":   # the wgmma kernel has no K bound of its own
            continue
        d, layers = _decode(L, flags, B, bw, tiling)
        layers[0].c_proj.K = 24576 + 64
        rc, msg = _step(L, d)
        assert rc == -2 and "c_proj of layer 0" in msg and "<= 24576" in msg, (name, rc, msg)


def _q8_decode(L, B, H=1536, C_=512, vocab=256, n_layer=2):
    layers = (L.Layer * n_layer)()
    q8 = (L.Q8Layer * n_layer)()
    w = lambda N, K: L.Q8Weight(P, P, N, K)  # noqa: E731
    for i in range(n_layer):
        layers[i] = L.Layer(rms_1=P, rms_2=P, k_cache=P, v_cache=P)
        q8[i] = L.Q8Layer(w(3 * C_, C_), w(C_, C_), w(H, C_), w(H, C_), w(C_, H))
    # disjoint activations: llm.int8's kernels refuse a y that overlaps x
    x, qkv, att, hid, logits = (P * k for k in (2, 3, 4, 5, 6))
    flags = L.F_PDL | L.F_Q8 | (L.F_Q8_BATCH if B > 1 else 0)
    d = L.DecodeArgs(n_layer=n_layer, n_head=C_ // 128, n_embd=C_, n_hidden=H, vocab=vocab, B=B, S=64, eps=1e-5,
                     layers=C.cast(layers, C.POINTER(L.Layer)), wte=P, ln_f=P, rope=P, idx=P, input_pos=P, ring_start=P,
                     block_size=64, x=x, qkv=qkv, att=att, hid=hid, attn_work=P, logits=logits, flags=flags,
                     q8_layers=C.cast(q8, C.POINTER(L.Q8Layer)), q8_lm_head=w(vocab, C_), q8_threshold=6.0,
                     batch_work=P if B > 1 else None)
    d._keep = (layers, q8)
    return d


@pytest.mark.parametrize("B", [1, 4])
def test_q8_routes_refuse_k_outside_their_kernel(L, B):
    rc, msg = _step(L, _q8_decode(L, B, H=1000))
    assert rc == -2 and "mlp.c_proj" in msg and "multiple of 128" in msg, msg
    rc, msg = _step(L, _q8_decode(L, B, H=33024))
    assert rc == -2 and "<= 32768" in msg, msg


@pytest.mark.parametrize("B", [1, 4])
def test_q8_routes_refuse_overlapping_activations(L, B):
    d = _q8_decode(L, B)
    d.hid = d.x
    rc, msg = _step(L, d)
    assert rc == -1 and "b2l_decode_step: c_fc1 of layer 0: " in msg and "y overlaps x" in msg, msg


def test_misaligned_tiling_or_batch_work(L):
    for name, (flags, B, bw, tiling) in _routes(L).items():
        d, layers = _decode(L, flags, B, bw, tiling)
        setattr(layers[1].c_fc12, tiling, P + 8)
        rc, msg = _step(L, d)
        assert rc == -1 and "c_fc12 of layer 1" in msg and "16-byte aligned" in msg, (name, rc, msg)
        if bw is None:
            continue
        d, layers = _decode(L, flags, B, P + 8, tiling)
        rc, msg = _step(L, d)
        assert rc == -1 and "c_attn of layer 0" in msg and "workspace must be 16-byte aligned" in msg, (name, rc, msg)
    d = _q8_decode(L, 4)
    d.batch_work = P + 8
    rc, msg = _step(L, d)
    assert rc == -1 and "16-byte aligned" in msg, msg


def test_a_weight_without_the_tiling_its_route_reads(L):
    for name, (flags, B, bw, tiling) in _routes(L).items():
        other = "qw_tiled" if tiling == "qw_mma" else "qw_mma"
        d, layers = _decode(L, flags, B, bw, tiling)
        d.lm_head = _weight(L, other, 256, 512)
        rc, msg = _step(L, d)
        if B == 1 and not flags:   # at batch 1 the route follows lm_head's tiling: the layers then disagree with it
            assert rc == -2 and "c_attn of layer 0 has" in msg and "lm_head's tiling picks" in msg, (name, rc, msg)
        else:
            assert rc == -3 and f"lm_head has no tiling for batch {B}" in msg, (name, rc, msg)
        d, layers = _decode(L, flags, B, bw, tiling)
        layers[1].c_proj = _weight(L, None, 512, 512)
        rc, msg = _step(L, d)
        assert rc == -3 and f"c_proj of layer 1 has no tiling for batch {B} ({tiling})" in msg, (name, rc, msg)
    # lm_head with no tiling at all
    d, layers = _decode(L, 0, 1, None, "qw_mma")
    d.lm_head = _weight(L, None, 256, 512)
    rc, msg = _step(L, d)
    assert rc == -3 and "lm_head has no tiling for batch 1" in msg, msg


def test_weights_that_disagree_on_their_tiling(L):
    # batch 1: lm_head's tiling picks the batch-1 GEMV or the wgmma kernel; a layer with the other one would mix them
    d, layers = _decode(L, 0, 1, None, "qw_mma")
    layers[1].mlp_proj = _weight(L, "qw_tiled", 512, 1536)
    rc, msg = _step(L, d)
    assert rc == -2 and "mlp.c_proj of layer 1 has qw_tiled but no qw_mma, lm_head has qw_mma" in msg, msg
    d, layers = _decode(L, 0, 1, None, "qw_tiled")
    layers[0].c_attn = _weight(L, "qw_mma", 1536, 512)
    rc, msg = _step(L, d)
    assert rc == -2 and "c_attn of layer 0 has qw_mma, lm_head has no qw_mma" in msg, msg
    # a layer with both tilings would run the batch-1 GEMV, lm_head with only qw_tiled the wgmma kernel
    d, layers = _decode(L, 0, 1, None, "qw_tiled")
    layers[1].c_proj.qw_mma = P
    rc, msg = _step(L, d)
    assert rc == -2 and "c_proj of layer 1 has qw_mma, lm_head has no qw_mma" in msg, msg
    # 2..8 rows with batch_work: the mma.sync batch kernel reads qw_mma of every weight
    d, layers = _decode(L, 0, 4, P, "qw_mma")
    layers[0].c_fc12 = _weight(L, "qw_tiled", 3072, 512)
    rc, msg = _step(L, d)
    assert rc == -3 and "c_fc12 of layer 0 has no tiling for batch 4 (qw_mma)" in msg, msg


def test_a_missing_rmsnorm_scale(L):
    for name, (flags, B, bw, tiling) in _routes(L).items():
        for field in ("rms_1", "rms_2"):
            d, layers = _decode(L, flags, B, bw, tiling)
            setattr(layers[1], field, None)
            rc, msg = _step(L, d)
            where = "c_attn" if field == "rms_1" else "c_fc12"
            assert rc == -1 and f"{where} of layer 1: " in msg and "RMSNorm prologue needs" in msg, (name, rc, msg)
    for B in (1, 4):
        d = _q8_decode(L, B)
        d._keep[0][0].rms_2 = None
        rc, msg = _step(L, d)
        assert rc == -1 and "c_fc1 of layer 0: " in msg and "RMSNORM needs norm_scale" in msg, msg


def test_q8_batch_flag_needs_q8(L):
    d, _ = _decode(L, L.F_Q4_BATCH_I8 | L.F_Q8_BATCH, 4, P, "qw_mma")
    rc, msg = _step(L, d)
    assert rc == -2 and "B2L_F_Q8_BATCH needs B2L_F_Q8" in msg, msg


def test_unsupported_head_size(L):
    d, layers = _decode(L, 0, 1, None, "qw_mma", n_head=2, C_=640)
    rc, msg = _step(L, d)
    assert rc == -2 and msg == "b2l_decode_step: head_size 320 unsupported (even, <= 256)", msg


def test_launch_counts(L):
    lib = L.lib()
    n_layer = 3
    # (flags, B values, batch_work, launches per linear)
    cases = [
        (0, [1], None, 1), (0, [1], P, 1),
        (0, [2, 5, 8], P, 2), (0, [2, 5, 8], None, 1),
        (0, [9, 12, 16], P, 1), (0, [9, 12, 16], None, 1),
        (L.F_W8, [1], None, 1),
        (L.F_W8 | L.F_W8_BATCH, [2, 8, 9, 16], P, 2),
        (L.F_Q4_BATCH_I8, [2, 8, 9, 16], P, 2),
        (L.F_Q8, [1], None, 1),
        (L.F_Q8 | L.F_Q8_BATCH, [2, 8, 9, 16], P, 2),
    ]
    for flags, Bs, bw, lin in cases:
        for B in Bs:
            d, _ = _decode(L, flags, B, bw, "qw_mma", n_layer=n_layer)
            # ring advance + embedding, per Block 4 linears + the fused attention, lm_head
            assert lib.b2l_decode_step_launches(C.byref(d)) == 2 + n_layer * (4 * lin + 1) + lin, (flags, B, bw)

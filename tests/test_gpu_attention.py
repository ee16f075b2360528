"""-m gpu: the attention entry points called directly, against themselves and against exact arithmetic.

Paths: the fused single-token kernel (head_size 128), the three-kernel split-S path (B2L_F_ATTN_UNFUSED at head_size
128, the generic path at any other head size), the tensor-core prefill kernel (T > 1, head_size 128), the per-query
kernel (T > 1, other head sizes), no-cache attention, the LLaMA-Adapter prefix on the fused, unfused, prefill and
no-cache paths, B2L_F_ROPE_ROWS, b2l_ring_advance and b2l_kv_unroll.

1. Exact invariances, bit for bit, no tolerance: every row of a B-row launch equals the B = 1 launch on that row's
   cache; the same logical cache at any ring offset gives the same output and appends at (slot + ring) % S; permuting
   heads and rows permutes the output; repeated launches and CUDA-graph replays give the same bits; y(2^e V) = 2^e y(V);
   slots a launch may not read can hold NaN.
2. Against float64 attention with one final bf16 rounding, under the per-element bar derived in `_exact`, for flat,
   attention-sink, massive-channel, equal-key, zero-query and cancelling-value inputs.
3. b2l_kv_unroll is an exact logical copy.
4. The model-level promise: on the exact 2..16-row decode steps every sampled row's logits equal the batch-1 model's
   bit for bit past position 256, where the fused kernel splits a head across CTAs.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu

F_ROPE_ROWS, F_UNFUSED = 4, 8   # B2L_F_ROPE_ROWS, B2L_F_ATTN_UNFUSED
BLK = 8192                      # RoPE table rows: every position used here has its own row
U = 2.0 ** -24                  # fp32 unit roundoff
NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


_ROPE = {}


def _rope(hs, dev):
    """(host table, device table) of BLK rows for head size hs."""
    if hs not in _ROPE:
        t = O.rope_table(BLK, hs)
        _ROPE[hs] = (t, t.to(torch.device("cuda", 0)))
    return _ROPE[hs]


def _work(B, nh, hs, T, S, dev):
    """A zero-filled attention workspace (its tickets start at zero; the fused kernel re-arms them itself)."""
    return torch.zeros(_L().lib().b2l_attn_workspace_bytes(B, nh, hs, T, S) // 4 + 1, device=dev, dtype=torch.float32)


def _prefix(dev, nh, alen, hs, seed):
    """A LLaMA-Adapter prefix: (b2l_adapter_prefix, k, v, gate); the tensors stay alive with the tuple."""
    g = torch.Generator(device=dev).manual_seed(seed)
    k = torch.randn(nh, alen, hs, device=dev, generator=g).bfloat16()
    v = (torch.randn(nh, alen, hs, device=dev, generator=g) * 0.5).bfloat16()
    gate = (torch.rand(nh, device=dev, generator=g) + 0.25).bfloat16()
    return (_L().AdapterPrefix(k.data_ptr(), v.data_ptr(), gate.data_ptr(), alen), k, v, gate)


def _launch(qkv, kc, vc, p0, ring, nh, *, flags=0, prefix=None, work=None, y=None, rope=None):
    """b2l_attention(_adapter) for T = qkv.shape[1] queries at positions p0..p0+T-1 with the ring offset `ring` (an int,
    or a device int32 tensor).  qkv, kc and vc change in place as the kernels change them; y is NaN-filled before the
    launch, so an output the kernels never write shows up.  `rope`: the T selected RoPE rows for B2L_F_ROPE_ROWS
    (default: the whole table)."""
    L = _L()
    lib, dev = L.lib(), qkv.device
    B, T, C3 = qkv.shape
    hs, S = C3 // (3 * nh), kc.shape[2]
    pos = p0 if torch.is_tensor(p0) else torch.arange(p0, p0 + T, dtype=torch.int64, device=dev)
    r = ring if torch.is_tensor(ring) else torch.tensor([ring], dtype=torch.int32, device=dev)
    work = _work(B, nh, hs, T, S, dev) if work is None else work
    y = torch.full((B, T, nh * hs), NAN, device=dev, dtype=torch.bfloat16) if y is None else y.fill_(NAN)
    rope = _rope(hs, dev)[1] if rope is None else rope
    args = (qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), rope.data_ptr(), pos.data_ptr(), r.data_ptr(),
            y.data_ptr(), work.data_ptr(), B, T, nh, hs, S, rope.shape[0], flags)
    if prefix is None:
        L.check(lib.b2l_attention(*args, L.stream_ptr()), "b2l_attention")
    else:
        L.check(lib.b2l_attention_adapter(*args, C.byref(prefix[0]), L.stream_ptr()), "b2l_attention_adapter")
    return y


def _nocache(qkv, nh, prefix=None):
    L = _L()
    lib, dev = L.lib(), qkv.device
    B, T, C3 = qkv.shape
    hs = C3 // (3 * nh)
    work = _work(B, nh, hs, T, T, dev)
    y = torch.full((B, T, nh * hs), NAN, device=dev, dtype=torch.bfloat16)
    rope = _rope(hs, dev)[1]
    if prefix is None:
        rc = lib.b2l_attention_nocache(qkv.data_ptr(), rope.data_ptr(), y.data_ptr(), work.data_ptr(), B, T, nh, hs, BLK,
                                       L.stream_ptr())
    else:
        rc = lib.b2l_attention_nocache_adapter(qkv.data_ptr(), rope.data_ptr(), y.data_ptr(), work.data_ptr(), B, T, nh, hs,
                                               BLK, C.byref(prefix[0]), L.stream_ptr())
    L.check(rc, "b2l_attention_nocache")
    return y


def _flat(dev, B, nh, hs, S, T=1, seed=0):
    """qkv [B, T, 3C] randn, logical caches [B, nh, S, hs] randn * 0.5 (bf16)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = torch.randn(B, T, 3 * nh * hs, device=dev, generator=g).bfloat16()
    kl = (torch.randn(B, nh, S, hs, device=dev, generator=g) * 0.5).bfloat16()
    vl = (torch.randn(B, nh, S, hs, device=dev, generator=g) * 0.5).bfloat16()
    return qkv, kl, vl


def _phys(logical, ring):
    """The physical cache holding `logical` at ring offset `ring`: physical slot (j + ring) % S = logical slot j."""
    return torch.roll(logical, ring, dims=2)


def _logical(phys, ring):
    return torch.roll(phys, -ring, dims=2)


def _rot(x, nh, p0):
    """The kernels' RoPE chain on the host: x [B, T, nh*hs] bf16 at positions p0.. -> [B, nh, T, hs] bf16."""
    B, T, C_ = x.shape
    rows = _rope(C_ // nh, None)[0][p0:p0 + T]
    return O.rope_apply(x.cpu().view(B, T, nh, C_ // nh), rows).transpose(1, 2)


# ============================================================================================== 1. exact invariances
ROW_POSITIONS = [63, 64, 255, 256, 257, 300, 767, 768, 1000, 1535, 2047, 2600]   # each side of every chunk edge; 2600: roll


@pytest.mark.parametrize("variant", ["fused", "adapter", "unfused"])
@pytest.mark.parametrize("nh", [32, 40, 52, 64])
def test_batch_rows_equal_batch1(dev, nh, variant):
    """Row b of a B-row launch equals the B = 1 launch on row b's cache: output and appended K / V rows, bit for bit.
    B in {2, 4, 16} at LLaMA head counts, on each side of every chunk size the fused kernel's split plan can pick, and in
    the roll branch (position >= S).  The split plan, and with it the fp32 order of the softmax and of the cross-CTA
    merge, must not depend on B."""
    S, hs = 2048, 128
    qkv, kl, vl = _flat(dev, 16, nh, hs, S, seed=nh)
    prefix = _prefix(dev, nh, {32: 1, 40: 10, 52: 64, 64: 10}[nh], hs, seed=nh) if variant == "adapter" else None
    flags = F_UNFUSED if variant == "unfused" else 0
    bad = []
    for B in (2, 4, 16):
        for pos in ROW_POSITIONS:
            ring = 777 if pos >= S else 0
            kb, vb = _phys(kl[:B], ring), _phys(vl[:B], ring)
            y = _launch(qkv[:B].clone(), kb, vb, pos, ring, nh, flags=flags, prefix=prefix)
            for b in range(B):
                k1, v1 = _phys(kl[b:b + 1], ring), _phys(vl[b:b + 1], ring)
                y1 = _launch(qkv[b:b + 1].clone(), k1, v1, pos, ring, nh, flags=flags, prefix=prefix)
                if not torch.equal(y[b], y1[0]):
                    bad.append((B, pos, b, int((y[b] != y1[0]).sum())))
                assert torch.equal(kb[b], k1[0]) and torch.equal(vb[b], v1[0]), (B, pos, b)
    assert not bad, f"(B, position, row, differing elements): {bad}"


RING_S = 1000   # not a multiple of 64
RINGS = [0, 1, 63, 64, 777, RING_S - 1]   # 777: the wrap falls at logical slot 223, inside a 64-row sub-tile / key tile
RING_DECODE = [0, 63, 230, 500, 999, 1300]   # 230: the new token's sub-tile holds the wrap at 223; 1300: roll
RING_PREFILL = [(0, 65), (200, 129), (700, 300)]   # (p0, T); 200..328 reads the key tile 192..255 that wraps at ring 777


@pytest.mark.parametrize("path", ["fused", "adapter", "unfused", "unfused-adapter", "hs64", "prefill", "prefill-hs64",
                                  "prefill-adapter"])
def test_ring_offset_invariance(dev, path):
    """The same logical cache stored at ring offsets {0, 1, 63, 64, 777, S - 1} gives the same y on every path, and the
    appended K / V rows land at (slot + ring) % S, the K row bit-equal to the host's RoPE chain."""
    B, nh, S = 2, 4, RING_S
    hs = 64 if "hs64" in path else 128
    flags = F_UNFUSED if path.startswith("unfused") else 0
    prefix = _prefix(dev, nh, 64, hs, seed=3) if "adapter" in path else None
    cases = [(p0, T) for p0, T in RING_PREFILL] if "prefill" in path else [(p, 1) for p in RING_DECODE]
    for ci, (p0, T) in enumerate(cases):
        qkv, kl, vl = _flat(dev, B, nh, hs, S, T=T, seed=10 + ci)
        slots = torch.arange(min(p0, S - 1), min(p0, S - 1) + T)
        k_want = _rot(qkv[:, :, nh * hs:2 * nh * hs], nh, p0)
        v_want = qkv[:, :, 2 * nh * hs:].cpu().view(B, T, nh, hs).transpose(1, 2)
        ref = None
        for ring in RINGS:
            kp, vp = _phys(kl, ring), _phys(vl, ring)
            y = _launch(qkv.clone(), kp, vp, p0, ring, nh, flags=flags, prefix=prefix)
            phys = (slots + ring) % S
            assert torch.equal(kp[:, :, phys].cpu(), k_want), (p0, ring)
            assert torch.equal(vp[:, :, phys].cpu(), v_want), (p0, ring)
            out = (y, _logical(kp, ring), _logical(vp, ring))
            if ref is None:
                ref = out
                assert bool(torch.isfinite(y).all())
            else:
                assert torch.equal(out[0], ref[0]), (p0, T, ring, int((out[0] != ref[0]).sum()))
                assert torch.equal(out[1], ref[1]) and torch.equal(out[2], ref[2]), (p0, ring)


@pytest.mark.parametrize("path", ["fused", "adapter", "unfused", "unfused-adapter", "prefill", "hs96"])
def test_head_and_row_permutation(dev, path):
    """Permuting the heads (and the batch rows) of q, k, v, the caches and the adapter prefix permutes y exactly: the
    (b, h) indexing and the per-(b, h) tickets, at up to 16 x 64 heads."""
    if path == "prefill":
        B, nh, hs, S, cases = 4, 16, 128, 512, [(40, 130), (0, 64)]
    elif path == "hs96":
        B, nh, hs, S, cases = 8, 16, 96, 512, [(300, 1), (40, 70)]
    else:
        B, nh, hs, S, cases = 16, 64, 128, 2048, [(300, 1), (1000, 1), (2047, 1)]
    flags = F_UNFUSED if path.startswith("unfused") else 0
    g = torch.Generator().manual_seed(5)
    ph, pb = torch.randperm(nh, generator=g).to(dev), torch.randperm(B, generator=g).to(dev)
    prefix = _prefix(dev, nh, 10, hs, seed=4) if "adapter" in path else None
    pprefix = None
    if prefix is not None:
        _, k, v, gate = prefix
        k, v, gate = k[ph].contiguous(), v[ph].contiguous(), gate[ph].contiguous()
        pprefix = (_L().AdapterPrefix(k.data_ptr(), v.data_ptr(), gate.data_ptr(), k.shape[1]), k, v, gate)
    for ci, (p0, T) in enumerate(cases):
        qkv, kc, vc = _flat(dev, B, nh, hs, S, T=T, seed=20 + ci)
        qkv_p = qkv.view(B, T, 3, nh, hs)[pb][:, :, :, ph].reshape(B, T, 3 * nh * hs).contiguous()
        kp, vp = kc[pb][:, ph].contiguous(), vc[pb][:, ph].contiguous()
        y = _launch(qkv.clone(), kc, vc, p0, 5, nh, flags=flags, prefix=prefix)
        yp = _launch(qkv_p, kp, vp, p0, 5, nh, flags=flags, prefix=pprefix)
        want = y.view(B, T, nh, hs)[pb][:, :, ph].reshape(B, T, nh * hs)
        assert torch.equal(yp, want), (p0, T, int((yp != want).sum()))
        assert torch.equal(kp, kc[pb][:, ph]) and torch.equal(vp, vc[pb][:, ph])


@pytest.mark.parametrize("variant", ["fused", "adapter"])
def test_repeated_launches_and_graph_replay(dev, variant):
    """Repeated launches give identical y, and so does a CUDA graph of one b2l_attention call replayed at three
    positions written on the device between replays: the cross-CTA tickets re-arm inside a graph as well (y is NaN
    before every launch, so a merge that never ran would show)."""
    B, nh, hs, S = 4, 40, 128, 2048
    positions = [300, 1000, 2047]   # 5, 4 and 6 CTAs per head
    qkv, kl, vl = _flat(dev, B, nh, hs, S, seed=30)
    prefix = _prefix(dev, nh, 64, hs, seed=30) if variant == "adapter" else None
    ke, ve, work = kl.clone(), vl.clone(), _work(B, nh, hs, 1, S, dev)
    eager = []
    for p in positions:
        a = _launch(qkv, ke, ve, p, 0, nh, prefix=prefix, work=work).clone()
        b = _launch(qkv, ke, ve, p, 0, nh, prefix=prefix, work=work)
        assert bool(torch.isfinite(a).all()) and torch.equal(a, b), p
        eager.append(a)
    kg, vg, work_g = kl.clone(), vl.clone(), _work(B, nh, hs, 1, S, dev)
    pos = torch.zeros(1, dtype=torch.int64, device=dev)
    ring = torch.zeros(1, dtype=torch.int32, device=dev)
    y = torch.empty(B, 1, nh * hs, device=dev, dtype=torch.bfloat16)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L = _L()
        args = (qkv.data_ptr(), kg.data_ptr(), vg.data_ptr(), _rope(hs, dev)[1].data_ptr(), pos.data_ptr(), ring.data_ptr(),
                y.data_ptr(), work_g.data_ptr(), B, 1, nh, hs, S, BLK, 0)
        if prefix is None:
            L.check(L.lib().b2l_attention(*args, L.stream_ptr()), "b2l_attention")
        else:
            L.check(L.lib().b2l_attention_adapter(*args, C.byref(prefix[0]), L.stream_ptr()), "b2l_attention_adapter")
    for _ in range(2):
        for p, want in zip(positions, eager):
            pos.fill_(p)
            y.fill_(NAN)
            graph.replay()
            assert torch.equal(y, want), p
    torch.cuda.synchronize()
    assert torch.equal(kg, ke) and torch.equal(vg, ve)


@pytest.mark.parametrize("path", ["fused", "adapter", "unfused", "unfused-adapter", "hs34", "prefill", "prefill-hs64",
                                  "nocache", "nocache-adapter"])
def test_value_scaling_is_exact(dev, path):
    """y(2^e V) = 2^e y(V) bit for bit for |e| <= 16 (the adapter prefix values scaled alike): every step after the
    scores is a product, a sum or a quotient of fp32 values that scale exactly."""
    B, nh, S = 2, 8, 2048
    hs = {"hs34": 34, "prefill-hs64": 64}.get(path, 128)
    flags = F_UNFUSED if path.startswith("unfused") else 0
    T = 130 if path.startswith(("prefill", "nocache")) else 1
    p0 = 1500 if T == 1 else 200
    qkv, kc, vc = _flat(dev, B, nh, hs, S, T=T, seed=40)
    prefix = _prefix(dev, nh, 10, hs, seed=40) if "adapter" in path else None

    def run(e):
        q = qkv.clone()
        q[:, :, 2 * nh * hs:] *= 2.0 ** e
        pre = None
        if prefix is not None:
            _, k, v, gate = prefix
            v = v * 2.0 ** e
            pre = (_L().AdapterPrefix(k.data_ptr(), v.data_ptr(), gate.data_ptr(), k.shape[1]), k, v, gate)
        if path.startswith("nocache"):
            return _nocache(q, nh, pre)
        return _launch(q, kc.clone(), vc * 2.0 ** e, p0, 123, nh, flags=flags, prefix=pre)

    y0 = run(0)
    assert bool(torch.isfinite(y0).all())
    for e in (-16, -5, 1, 7, 16):
        assert torch.equal(run(e), y0 * 2.0 ** e), e


@pytest.mark.parametrize("path", ["fused", "adapter", "unfused", "unfused-adapter", "hs64", "prefill", "prefill-hs64"])
def test_unread_slots_may_hold_nan(dev, path):
    """Logical slots >= L (the slots after the newest position) hold NaN in K and V: y stays finite and bit-equal to the
    run without them -- attention touches the valid slots 0..pos only."""
    B, nh, S, ring = 2, 4, RING_S, 777
    hs = 64 if "hs64" in path else 128
    flags = F_UNFUSED if path.startswith("unfused") else 0
    prefix = _prefix(dev, nh, 10, hs, seed=50) if "adapter" in path else None
    cases = [(0, 65), (200, 129), (1, 2)] if "prefill" in path else [(p, 1) for p in (0, 63, 64, 230, 500, 998)]
    for ci, (p0, T) in enumerate(cases):
        qkv, kl, vl = _flat(dev, B, nh, hs, S, T=T, seed=50 + ci)
        y = _launch(qkv.clone(), _phys(kl, ring), _phys(vl, ring), p0, ring, nh, flags=flags, prefix=prefix)
        kn, vn = kl.clone(), vl.clone()
        kn[:, :, p0 + T:] = NAN
        vn[:, :, p0 + T:] = NAN
        yn = _launch(qkv.clone(), _phys(kn, ring), _phys(vn, ring), p0, ring, nh, flags=flags, prefix=prefix)
        assert bool(torch.isfinite(yn).all()) and torch.equal(yn, y), (p0, T)


@pytest.mark.parametrize("hs", [64, 128])
@pytest.mark.parametrize("S", [64, 77, 1000])
def test_kv_unroll_is_a_logical_copy(dev, S, hs):
    L = _L()
    B, nh = 3, 5
    g = torch.Generator(device=dev).manual_seed(S + hs)
    kl = torch.randn(B, nh, S, hs, device=dev, generator=g).bfloat16()
    for ring in (0, 1, S - 1, S // 3):
        r = torch.tensor([ring], dtype=torch.int32, device=dev)
        out = torch.full_like(kl, NAN)
        L.check(L.lib().b2l_kv_unroll(_phys(kl, ring).data_ptr(), r.data_ptr(), out.data_ptr(), B, nh, S, hs, L.stream_ptr()),
                "b2l_kv_unroll")
        assert torch.equal(out, kl), (S, hs, ring)


def test_ring_advance_moves_one_slot_past_the_cache(dev):
    """b2l_ring_advance: the ring start moves by one slot (mod S) exactly when the call's last position is >= S, the
    roll of model.py:214-218."""
    L = _L()
    S = 100
    r = torch.zeros(1, dtype=torch.int32, device=dev)
    for positions, start, want in [([0], 0, 0), ([99], 7, 7), ([100], 7, 8), ([250], 99, 0), ([90, 95, 99], 3, 3),
                                   ([98, 99, 100], 3, 4), ([100, 101], 0, 1)]:
        r.fill_(start)
        pos = torch.tensor(positions, dtype=torch.int64, device=dev)
        L.check(L.lib().b2l_ring_advance(pos.data_ptr(), len(positions), r.data_ptr(), S, L.stream_ptr()), "ring_advance")
        assert int(r) == want, (positions, start)


@pytest.mark.parametrize("hs,T", [(128, 1), (64, 1), (128, 65), (64, 65)])
def test_rope_rows_flag_equals_the_table(dev, hs, T):
    """B2L_F_ROPE_ROWS (`rope` holds the T rows input_pos selects, the reference's call convention): the same y and the
    same cache rows as the whole table indexed by position, bit for bit (at T = 1, head_size 128 the flag takes the
    three-kernel path, so the table run does too)."""
    B, nh, S, p0, ring = 2, 8, 1000, 700, 333
    qkv, kc, vc = _flat(dev, B, nh, hs, S, T=T, seed=60)
    rows = _rope(hs, dev)[1][p0:p0 + T].contiguous()
    k1, v1, k2, v2 = kc.clone(), vc.clone(), kc.clone(), vc.clone()
    y1 = _launch(qkv.clone(), k1, v1, p0, ring, nh, flags=F_UNFUSED if T == 1 else 0)
    y2 = _launch(qkv.clone(), k2, v2, p0, ring, nh, flags=F_ROPE_ROWS, rope=rows)
    assert bool(torch.isfinite(y1).all())
    assert torch.equal(y1, y2) and torch.equal(k1, k2) and torch.equal(v1, v2)


# ============================================================================================== 2. against float64
def _half_ulp_bf16(x):
    """Half a bf16 ulp at |x| (float64), normal range."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


SERIAL = {"decode": 1, "per_query": 16, "prefill_tc": 1}    # online-softmax updates in series per 64 keys
ACC = {"decode": 6, "per_query": 32, "prefill_tc": 274}    # accumulation roundings (of 2u) in series per 64 keys


def _exact(qh, k, v, Lrow, hs, n_tiles, kind):
    """float64 attention and the per-element bar.  qh [G, T, hs] (the rotated bf16 queries), k / v [G, Lmax, hs] (the
    logical cache as the kernel holds it), Lrow [T] valid slots per query, n_tiles = ceil(keys / 64) (S for the split
    decode paths, whose merge visits every split of the cache), `kind` the path: "decode" (fused or split-S, one
    query), "per_query" (T > 1 at head sizes other than 128: one CTA streams all keys of a query, 4 warps), or
    "prefill_tc" (the tensor-core prefill kernel).  Returns (y, eps): y = softmax(q k^T / sqrt(hs)) v with the mask,
    and eps bounding |fp32 kernel result - y| before its final bf16 rounding.

    Derivation (u = 2^-24; every error is carried to first order, weights to all orders through expm1):
    * score s_j = q.k_j / sqrt(hs): the hs products are exact in fp32 (bf16 x bf16); each addition rounds by at most
      2u of the running sum of magnitudes, for any order, rounding to nearest on the CUDA cores and truncating in the
      tensor cores' fp32 accumulation (where up to 17 addends share one alignment, hs/16 MMAs: 2 hs + hs/8), plus the
      rounding of the scaled query (1u), rsqrtf (2 ulp) and the product with it (1u), 2u more for safety:
      |ds_j| <= (2 hs + hs/8 + 6) u A_j,  A_j = sum_i |q_i k_ji| / sqrt(hs).
    * weight p_j = exp(s_j - M) is built from one exp per online-softmax update along its path (the key's own, every
      later running-max correction, the warp / key-group / CTA / split merges): at most SERIAL n_tiles + 24 of them
      (a fused key group sees <= 5 updates per CTA, a split-S warp 16 per split, a prefill row one per key tile, a
      per-query warp 16 per 64 keys); __expf(x) is within (2 + 1.173|x|) ulp, the rounding of the subtraction adds
      |x| u, and the |x| of the chain add up to M - s_j:
      eta_j = |ds_j| + u (3 (SERIAL n_tiles + 24) + 3 (M - s_j)), relative error <= expm1(eta_j).
      Weights perturbed by relative errors e_j move y by sum_j pi_j e_j (v_j - y) / (1 - sum_j pi_j |e_j|).
    * accumulation of sum_j p_j v_j and of sum_j p_j (and the final quotient): at most 2u per fp32 operation of the
      running magnitude sum, over the deepest chain: 3 updates per 64 keys plus 2 merge steps per 64-key split on the
      decode paths (ACC 6), 2 per key of a per-query warp (32), one correction and 8 MMAs of 17 addends per key tile
      in the prefill kernel (274), and 64 for the in-CTA merges and the quotient:
      (ACC n_tiles + 64) u (sum_j pi_j |v_j| + |y|).
    * the prefill kernel feeds P to its second MMA as bf16 hi + lo: 2^-17 relative per weight, numerator only:
      2^-17 sum_j pi_j |v_j|.
    """
    G, T, _ = qh.shape
    Lmax = k.shape[1]
    s = torch.einsum("gtd,gjd->gtj", qh, k) / math.sqrt(hs)
    A = torch.einsum("gtd,gjd->gtj", qh.abs(), k.abs()) / math.sqrt(hs)
    mask = torch.arange(Lmax, device=qh.device).view(1, 1, Lmax) < Lrow.view(1, T, 1)
    s = s.masked_fill(~mask, -math.inf)
    M = s.amax(-1, keepdim=True)
    p = torch.exp(s - M)
    pi = p / p.sum(-1, keepdim=True)
    y = torch.einsum("gtj,gjd->gtd", pi, v)
    gap = torch.where(mask, M - s, torch.zeros_like(s))
    c_s = 2 * hs + hs // 8 + 6
    eta = c_s * U * A + U * (3 * (SERIAL[kind] * n_tiles + 24) + 3 * gap)
    w = pi * torch.expm1(eta)
    mag = torch.einsum("gtj,gjd->gtd", pi, v.abs())
    if G * T * Lmax * hs > 2 ** 26:   # |v_j - y| <= |v_j| + |y| keeps the [G, T, L, hs] tensor out of memory
        dev_term = torch.einsum("gtj,gjd->gtd", w, v.abs()) + w.sum(-1, keepdim=True) * y.abs()
    else:
        dev_term = torch.einsum("gtj,gtjd->gtd", w, (v.unsqueeze(1) - y.unsqueeze(2)).abs())
    dev_term = dev_term / (1 - w.sum(-1, keepdim=True))
    eps = dev_term + (ACC[kind] * n_tiles + 64) * U * (mag + y.abs())
    if kind == "prefill_tc":
        eps = eps + 2.0 ** -17 * mag
    return y, eps


def _check_exact(got, y, eps, what):
    """|got - y| <= half an ulp of bf16 at |y| + eps, plus eps; returns the share bit-equal to bf16(y)."""
    got = got.double()
    err = (got - y).abs()
    bar = _half_ulp_bf16(y.abs() + eps) + eps
    over = err > bar
    assert bool(torch.isfinite(got).all()), what
    assert not bool(over.any()), (what, int(over.sum()), float((err - bar).max()), float(err[over].max()))
    return float((got == y.float().bfloat16().double()).double().mean())


def _check_adapter_exact(got, y, eps, ay, eps_ay, gate, what):
    """The LLaMA-Adapter output bf16(rbf(y) + rbf(gate * rbf(ay))) (adapter.py:167 under bf16) against its exact form
    y + gate * ay: y the cache attention and ay the prefix attention, each within its own float64 bar (eps, eps_ay).
    Each rounding on the way adds half a bf16 ulp at the largest magnitude its operand can have, the fp32 product and
    sum one u each.  Returns the share bit-equal to the chain applied to the exact y and ay."""
    h = _half_ulp_bf16
    got = got.double()
    err_y = eps + h(y.abs() + eps)                   # rbf(y)
    ra = ay.abs() + eps_ay
    err_a = eps_ay + h(ra)                           # rbf(ay)
    t = gate * (ra + h(ra))                          # |gate * rbf(ay)|
    err_t = gate * err_a + U * t + h(t * (1 + U))    # rbf(fl(gate * rbf(ay)))
    err_s = err_y + err_t + U * (y.abs() + err_y + t + err_t)
    z = y + gate * ay
    bar = err_s + h(z.abs() + err_s)
    err = (got - z).abs()
    over = err > bar
    assert bool(torch.isfinite(got).all()), what
    assert not bool(over.any()), (what, int(over.sum()), float((err - bar).max()))
    f = lambda x: x.float().bfloat16().float()   # noqa: E731
    chain = (f(y) + f(gate.float() * f(ay))).bfloat16().double()
    return float((got == chain).double().mean())


def _shape_inputs(dev, dist, B, nh, hs, S, T, p0, seed):
    """qkv [B, T, 3C] and logical caches [B, nh, S, hs] for a score distribution (all bf16)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    C_ = nh * hs
    qkv, kl, vl = _flat(dev, B, nh, hs, S, T=T, seed=seed)
    q, k, v = qkv[..., :C_].view(B, T, nh, hs), qkv[..., C_:2 * C_].view(B, T, nh, hs), qkv[..., 2 * C_:].view(B, T, nh, hs)
    if dist == "sink":
        # slot 0 holds 90..99.9 % of the mass: its key points along the query's low-frequency RoPE pairs (they barely
        # rotate), every other key is small; its value row is small (the LLaMA pattern)
        n_lo = min(8, hs)
        lo = slice(hs - n_lo, hs)
        q[..., lo] = 2.0
        k.mul_(0.3)
        k[..., lo] = 0.0
        kl.mul_(0.3)
        kl[:, :, :, lo] = 0.0
        frac = 0.9 + 0.099 * torch.rand(nh, device=dev, generator=g)   # the sink's share per head
        gap = torch.log(frac / (1 - frac) * max(S - 1, 1))
        kl[:, :, 0, lo] = (gap * math.sqrt(hs) / (2.0 * n_lo)).view(1, nh, 1)
        vl[:, :, 0] = (torch.randn(B, nh, hs, device=dev, generator=g) * 0.02).bfloat16()
    elif dist == "massive":
        # massive channels on the lowest-frequency pairs: |k| up to 1e3, a near one-hot softmax and a large sum |q k|
        lo = slice(hs - 4, hs)
        q[..., lo] = 40.0 * torch.sign(torch.randn(B, T, nh, 4, device=dev, generator=g))
        k[..., lo] = ((torch.rand(B, T, nh, 4, device=dev, generator=g) * 2 - 1) * 1e3).bfloat16()
        kl[:, :, :, lo] = ((torch.rand(B, nh, S, 4, device=dev, generator=g) * 2 - 1) * 1e3).bfloat16()
    elif dist == "equal":   # every key equals the new token's rotated key: uniform weights, y = mean of V
        kr = _rot(qkv[..., C_:2 * C_], nh, p0)[:, :, :1].to(dev)
        kl.copy_(kr.expand(B, nh, S, hs))
    elif dist == "q0":
        q.zero_()
    elif dist == "cancel":   # large values of mixed sign: y is far smaller than sum pi |v|
        sgn = torch.sign(torch.randn(B, nh, S, hs, device=dev, generator=g))
        vl.copy_((sgn * (1000 + 30 * torch.randn(B, nh, S, hs, device=dev, generator=g))).bfloat16())
        v.copy_((torch.sign(torch.randn(B, T, nh, hs, device=dev, generator=g)) * 1000).bfloat16())
    return qkv, kl, vl


def _vs_float64(dev, path, dist, B, nh, hs, S, p0, T, ring, seed, stats=None, prefix=None):
    """One launch against float64: the appended K rows bit-equal to the host RoPE chain, every output within the bar
    (with `prefix`: the adapter output against its exact form).  The share of outputs bit-equal to the correctly rounded
    exact result is appended to stats[dist]."""
    qkv, kl, vl = _shape_inputs(dev, dist, B, nh, hs, S, T, p0, seed)
    C_ = nh * hs
    qh = _rot(qkv[..., :C_], nh, p0).to(dev).double()                    # [B, nh, T, hs]
    k_new = _rot(qkv[..., C_:2 * C_], nh, p0)
    kp, vp = _phys(kl, ring), _phys(vl, ring)
    y = _launch(qkv.clone(), kp, vp, p0, ring, nh, flags=F_UNFUSED if path.startswith("unfused") else 0, prefix=prefix)
    w0 = min(p0, S - 1)
    kg, vg = _logical(kp, ring), _logical(vp, ring)
    assert torch.equal(kg[:, :, w0:w0 + T].cpu(), k_new), (path, dist, S, p0)
    Lrow = torch.arange(w0 + 1, w0 + T + 1, device=dev)
    Lmax = w0 + T
    G = B * nh
    kind = "decode" if T == 1 else ("prefill_tc" if hs == 128 else "per_query")
    ye, eps = _exact(qh.reshape(G, T, hs), kg[:, :, :Lmax].reshape(G, Lmax, hs).double(),
                     vg[:, :, :Lmax].reshape(G, Lmax, hs).double(), Lrow, hs, -(-(S if T == 1 else Lmax) // 64), kind)
    got = y.view(B, T, nh, hs).transpose(1, 2).reshape(G, T, hs)
    what = (path, dist, S, p0, T, ring)
    if prefix is None:
        same = _check_exact(got, ye, eps, what)
    else:   # the prefix: alen keys of every head, all valid, one query; its loops run in series over the alen keys
        _, pk, pv, gate = prefix
        alen = pk.shape[1]
        pk = pk.unsqueeze(0).expand(B, -1, -1, -1).reshape(G, alen, hs).double()
        pv = pv.unsqueeze(0).expand(B, -1, -1, -1).reshape(G, alen, hs).double()
        ay, eps_ay = _exact(qh.reshape(G, T, hs), pk, pv, torch.full((T,), alen, device=dev), hs, 1, "decode")
        same = _check_adapter_exact(got, ye, eps, ay, eps_ay, gate.double().repeat(B).view(G, 1, 1), what)
    if stats is not None:
        stats.setdefault(dist, []).append(same)
    return same


DISTS = ["flat", "sink", "massive", "equal", "q0", "cancel"]
# least share of outputs bit-equal to the correctly rounded exact result, per distribution, over every case below.
# Measured on an H100 80GB HBM3 (700 W): flat 0.9974, sink 0.9972, massive 0.9939, equal 0.9998, q0 0.9992, cancel
# 0.9977 (the lowest of the decode, LLaMA-head and prefill cases).  A kernel that loses a key or a rescale falls far below.
SHARE = {"flat": 0.99, "sink": 0.99, "massive": 0.985, "equal": 0.995, "q0": 0.995, "cancel": 0.99}


def _check_shares(stats, what):
    print(what + ": bit-equal to the exact result: " + ", ".join(f"{d} {min(v):.4f}" for d, v in stats.items()))
    for d, v in stats.items():
        assert min(v) >= SHARE[d], (what, d, min(v))


def _plan(L, nh):
    """(keys per CTA, working CTAs per head) of the fused decode kernel: 3 CTAs per SM aimed at, shared by the n_head
    heads of a batch row, 64..256 keys per CTA (attn_decode_fused_kernel)."""
    want = max(1, 3 * torch.cuda.get_device_properties(0).multi_processor_count // nh)
    chunk = 256 if L <= 256 else min(256, max(64, 64 * -(-L // (64 * want))))
    return chunk, -(-L // chunk)


LLAMA_L = [200, 256, 1000, 2047, 4095]   # valid slots: one CTA of 4 sub-tiles (L <= 256), then 128..256-key chunks


@pytest.mark.parametrize("path", ["fused", "adapter", "unfused-adapter"])
@pytest.mark.parametrize("nh", [32, 40, 64])
def test_decode_llama_heads_vs_float64(dev, nh, path):
    """Single-token attention at the LLaMA head counts (7B, 13B, 65B), batch 1, S = 4096, every head against float64,
    for every score distribution.  At these head counts the fused kernel runs its production regime: one CTA streams
    four 64-key sub-tiles (L = 200, 256), and 128..256-key chunks are merged across up to 16 CTAs per head (L = 1000,
    2047, 4095).  The adapter output (prefix length 1, 10 or 64) against its exact form, on the fused kernel and on the
    three-kernel path with the prefix kernel."""
    S = 4096
    stats, plans = {}, set()
    for li, L_ in enumerate(LLAMA_L):
        plans.add(_plan(L_, nh))
        prefix = _prefix(dev, nh, (1, 10, 64)[li % 3], 128, seed=1300 + li) if "adapter" in path else None
        for di, dist in enumerate(DISTS):
            _vs_float64(dev, path, dist, 1, nh, 128, S, L_ - 1, 1, 0 if li % 2 == 0 else 1000, seed=1200 + 10 * li + di,
                        stats=stats, prefix=prefix)
    _check_shares(stats, f"decode {path} n_head={nh}")
    # the chunk sizes the fused kernel reached here
    assert (256, 1) in plans, plans                                 # 4 sub-tiles in one CTA, no merge
    assert {c for c, n in plans if n > 1} & {128, 192}, plans       # multi-sub-tile chunks merged across CTAs
    assert (256, 16) in plans, plans                                # 16 partials: the merge's second batch of 8


@pytest.mark.parametrize("path", ["fused", "unfused"])
@pytest.mark.parametrize("S", [64, 65, 300, 2048, 4096])
def test_decode_hs128_vs_float64(dev, S, path):
    """Single-token attention at head_size 128 (fused kernel, and the three-kernel path with EPL = 4) against float64,
    at the full cache, a middle position and (S = 300) the roll branch, for every score distribution."""
    stats = {}
    cases = [(S - 1, 0), (S // 2, 5), (S + 150, 37)] if S == 300 else [(S - 1, 0), (S // 2, 5)]
    for di, dist in enumerate(DISTS):
        for ci, (pos, ring) in enumerate(cases):
            _vs_float64(dev, path, dist, 2, 4, 128, S, pos, 1, ring, seed=100 * di + ci, stats=stats)
    _check_shares(stats, f"decode {path} S={S}")


@pytest.mark.parametrize("hs", [2, 34, 64, 96, 256])
def test_decode_generic_head_sizes_vs_float64(dev, hs):
    """The generic (EPL = 0) three-kernel path at head sizes other than 128."""
    for S in (65, 2048):
        for di, dist in enumerate(["flat", "sink", "q0", "cancel"] + (["massive", "equal"] if hs >= 8 else [])):
            for ci, (pos, ring) in enumerate([(S - 1, 0), (S // 2 + 3, 9)]):
                _vs_float64(dev, "generic", dist, 2, 4, hs, S, pos, 1, ring, seed=500 + 10 * di + ci)


PREFILL = [(T, p0) for T in (2, 63, 64, 65, 129, 2048) for p0 in (0, 1, 200)]


@pytest.mark.parametrize("T,p0", PREFILL)
def test_prefill_hs128_vs_float64(dev, T, p0):
    """The tensor-core prefill kernel (T > 1, head_size 128) against float64, with a rotated cache (ring 777) from p0 > 0
    on; flat and sink scores everywhere, the other distributions at T = 65."""
    S = 2304
    ring = 777 if p0 else 0
    dists = DISTS if T == 65 else ["flat", "sink"]
    stats = {}
    for di, dist in enumerate(dists):
        if dist == "equal":
            continue   # the new keys are rotated at T different positions
        _vs_float64(dev, "prefill", dist, 2, 4, 128, S, p0, T, ring, seed=700 + di, stats=stats)
    _check_shares(stats, f"prefill T={T} p0={p0}")


@pytest.mark.parametrize("hs", [64, 96])
def test_prefill_per_query_vs_float64(dev, hs):
    """T > 1 at head sizes other than 128 (one CTA per query on the three-kernel path)."""
    for ci, (T, p0, ring) in enumerate([(2, 0, 0), (65, 1, 777), (129, 200, 999)]):
        for di, dist in enumerate(["flat", "sink", "massive", "cancel"]):
            _vs_float64(dev, "prefill", dist, 2, 4, hs, 1000, p0, T, ring, seed=900 + 10 * ci + di)


@pytest.mark.parametrize("T", [2, 65, 2048])
@pytest.mark.parametrize("hs", [64, 128])
def test_nocache_vs_float64(dev, T, hs):
    """b2l_attention_nocache: causal attention over the T rows of qkv, k rotated in place bit-equal to the host chain."""
    B, nh = 2, 4
    C_ = nh * hs
    for di, dist in enumerate(["flat", "sink", "cancel"]):
        qkv, _, _ = _shape_inputs(dev, dist, B, nh, hs, 64, T, 0, seed=1100 + di)
        qh = _rot(qkv[..., :C_], nh, 0).to(dev).double()
        kr = _rot(qkv[..., C_:2 * C_], nh, 0)
        v = qkv[..., 2 * C_:].view(B, T, nh, hs).transpose(1, 2)
        q2 = qkv.clone()
        y = _nocache(q2, nh)
        assert torch.equal(q2[..., C_:2 * C_].cpu().view(B, T, nh, hs).transpose(1, 2), kr)
        G = B * nh
        ye, eps = _exact(qh.reshape(G, T, hs), kr.to(dev).reshape(G, T, hs).double(), v.reshape(G, T, hs).double(),
                         torch.arange(1, T + 1, device=dev), hs, -(-T // 64), "prefill_tc" if hs == 128 else "per_query")
        _check_exact(y.view(B, T, nh, hs).transpose(1, 2).reshape(G, T, hs), ye, eps, ("nocache", dist, T, hs))


# ============================================================================================== 4. the model-level promise
@pytest.mark.parametrize("kind", ["13B-q4", "13B-w8"])
def test_sampled_rows_bit_identical_to_batch1_past_position_256(dev, kind):
    """generate_batch on the exact 2..16-row steps of a two-Block model at the 13B widths (40 heads): a 300-token
    prompt, S = 512, N = 4 and 16 samples.  Every row's logits equal the teacher-forced batch-1 model's at every step,
    bit for bit, at positions where the fused attention splits each head over several CTAs."""
    import test_gpu_generate_batch as TG

    L = _L()
    model = TG._exact_model(dev, kind)
    try:
        prompt = TG._prompt(dev, model.config.vocab_size, T=300, seed=12)
        for n in (4, 16):
            ys, logs, qs = TG._sampled(model, prompt, n, 6, S=512, seed=80 + n)
            st = model._decode
            assert st is not None and st.B == n and st.args.flags & (L.F_Q4_BATCH_I8 if "q4" in kind else L.F_W8_BATCH)
            assert len({tuple(y.tolist()) for y in ys}) > 1
            TG._check_draws(ys, logs, qs, 300)
            TG._rows_vs_batch1(model, prompt, ys, logs, 512)
    finally:
        del model
        torch.cuda.empty_cache()

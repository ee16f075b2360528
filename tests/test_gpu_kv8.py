"""GPU: the fp8 KV cache (b2l_attention_kv8, B2L_F_KV_FP8, LLaMA.kv_cache_dtype = "fp8"), bit for bit unless stated.

1. Append exactness: the codes and scales a decode launch (with and without B2L_F_ROW_POS, at ring offsets with and
   without a wrap) or a prefill writes equal the number format restated (`quant`) on the rows the bf16 path writes.
2. Same arithmetic: with the new key zero and the new value on the e4m3 grid, the fp8 launch equals b2l_attention on a
   bf16 cache holding the values read back, at positions with one CTA per head and with several, with and without
   the adapter prefix.
3. Invariances: rows of a B-row launch equal B = 1; permuting heads and rows permutes y; graph replays repeat; unread
   slots may hold NaN codes and scales; scaling V by 2^e keeps the codes, moves the scale by 2^e and gives 2^e y.
4. Against float64 attention over the values read back (the new token's included), under the per-element bar
   tests/test_gpu_attention.py derives for the decode kernel (restated in `_exact`), on flat, sink, massive-channel
   and cancelling inputs.
5. Model level on a tiny head-size-128 model: prompt logits equal the no-cache forward; the whole-token step against
   the module path (bit for bit where the bf16 step is: llm.int8; within the bf16 model test's tolerance for
   gptq.int4 / gptq.int8 at batch 1); q4_batch_step / w8_batch_step rows equal the batch-1 fp8 model past position
   256; greedy generate_prompts / generate_stream equal generate() per prompt; logical_kv_caches equals the restatement.
6. Quality, reported (printed), not gated: bf16 against fp8 cache over 256 greedy decode steps.
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
E_MIN = -124


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as entry

    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def quant(x: torch.Tensor):
    """The number format (include/b2l.h, restated): x bf16 [..., hs] -> (codes float8_e4m3fn, scales fp32 [...]).
    e via frexp, the rounding by torch's e4m3fn conversion (tests/test_kv8_cpu.py pins it against an independent
    round-to-nearest-even restatement)."""
    xf = x.float()
    amax = xf.abs().amax(-1)
    bad = ~torch.isfinite(xf).all(-1)
    m, ex = torch.frexp(amax.double())
    e = torch.where(m <= 0.875, ex - 9, ex - 8).clamp_min(E_MIN)
    e = torch.where(amax == 0, torch.zeros_like(e), e)
    scale = torch.ldexp(torch.ones_like(amax), e.to(torch.int32))
    codes = (xf * torch.ldexp(torch.ones_like(amax), (-e).to(torch.int32)).unsqueeze(-1)).to(torch.float8_e4m3fn)
    codes = torch.where(bad.unsqueeze(-1), torch.full_like(codes.view(torch.uint8), 0x7f), codes.view(torch.uint8))
    codes = codes.view(torch.float8_e4m3fn)   # (float8 tensors are indexed and selected through their bytes)
    scale = torch.where(bad, torch.full_like(scale, math.nan), scale)
    return codes, scale


def back(codes: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """The values read back, float(code) * scale (fp32)."""
    return codes.float() * scale.unsqueeze(-1)


def _bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    if a.dtype == torch.float8_e4m3fn:
        return torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    return torch.equal(a.contiguous().view(torch.int32 if a.dtype == torch.float32 else torch.int16),
                       b.contiguous().view(torch.int32 if b.dtype == torch.float32 else torch.int16))


def _rope(dev, S):
    from lit_llama_b200.model import build_rope_cache

    return build_rope_cache(S, 128, torch.float32, dev).float().contiguous()


def _work(L, B, nh, S, dev, T=1):
    return torch.zeros(L.lib().b2l_attn_workspace_bytes(B, nh, 128, T, S) // 4 + 1, device=dev, dtype=torch.float32)


class Cache8:
    """An fp8 cache [B, nh, S, 128] in device memory."""

    def __init__(self, codes, ks, vcodes, vs):
        self.k, self.v, self.ks, self.vs = codes.contiguous(), vcodes.contiguous(), ks.contiguous(), vs.contiguous()

    @classmethod
    def random(cls, dev, B, nh, S, seed, kmag=1.0, vmag=1.0):
        g = torch.Generator(device=dev).manual_seed(seed)
        kc, ks = quant((torch.randn((B, nh, S, 128), device=dev, generator=g) * kmag).bfloat16())
        vc, vs = quant((torch.randn((B, nh, S, 128), device=dev, generator=g) * vmag).bfloat16())
        return cls(kc, ks, vc, vs)

    def clone(self):
        return Cache8(self.k.clone(), self.ks.clone(), self.v.clone(), self.vs.clone())

    def spec(self, L):
        return L.KV8Cache(self.k.data_ptr(), self.v.data_ptr(), self.ks.data_ptr(), self.vs.data_ptr())

    def values(self):
        return back(self.k, self.ks).bfloat16(), back(self.v, self.vs).bfloat16()


def _prefix(dev, nh, alen=10, seed=5):
    from lit_llama_b200 import _lib as L

    g = torch.Generator(device=dev).manual_seed(seed)
    k = torch.randn((nh, alen, 128), device=dev, generator=g).bfloat16()
    v = torch.randn((nh, alen, 128), device=dev, generator=g).bfloat16()
    gate = (torch.rand(nh, device=dev, generator=g) + 0.5).bfloat16()
    spec = L.AdapterPrefix(k.data_ptr(), v.data_ptr(), gate.data_ptr(), alen)
    spec._keep = (k, v, gate)
    return spec


def run8(L, qkv, cache, pos, ring, nh, rows=False, prefix=None):
    """b2l_attention_kv8 at T == 1 (qkv is not modified); returns y [B, 1, C]."""
    B, S = qkv.shape[0], cache.k.shape[2]
    dev = qkv.device
    y = torch.empty((B, 1, nh * 128), device=dev, dtype=torch.bfloat16)
    posv = torch.tensor(pos, dtype=torch.int64, device=dev)
    ringv = torch.tensor(ring, dtype=torch.int32, device=dev)
    spec = cache.spec(L)
    rc = L.lib().b2l_attention_kv8(qkv.data_ptr(), C.byref(spec), _rope(dev, S).data_ptr(), posv.data_ptr(),
                                   ringv.data_ptr(), y.data_ptr(), _work(L, B, nh, S, dev).data_ptr(), B, 1, nh, 128, S, S,
                                   L.F_ROW_POS if rows else 0, None if prefix is None else C.byref(prefix), L.stream_ptr())
    L.check(rc, "b2l_attention_kv8")
    torch.cuda.synchronize()
    return y


def run16(L, qkv, kc, vc, pos, ring, nh, rows=False, prefix=None):
    B, S = qkv.shape[0], kc.shape[2]
    dev = qkv.device
    y = torch.empty((B, 1, nh * 128), device=dev, dtype=torch.bfloat16)
    posv = torch.tensor(pos, dtype=torch.int64, device=dev)
    ringv = torch.tensor(ring, dtype=torch.int32, device=dev)
    args = (qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), _rope(dev, S).data_ptr(), posv.data_ptr(), ringv.data_ptr(),
            y.data_ptr(), _work(L, B, nh, S, dev).data_ptr(), B, 1, nh, 128, S, S, L.F_ROW_POS if rows else 0)
    lib = L.lib()
    rc = lib.b2l_attention(*args, L.stream_ptr()) if prefix is None else lib.b2l_attention_adapter(*args, C.byref(prefix), L.stream_ptr())
    L.check(rc, "b2l_attention")
    torch.cuda.synchronize()
    return y


def _qkv(dev, B, nh, seed, scale=1.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn((B, 1, 3 * nh * 128), device=dev, generator=g) * scale).bfloat16()


def _slot(p, ring, S):
    return (min(p, S - 1) + ring) % S


# ---------------------------------------------------------------------------------------------------------- 1. append
@pytest.mark.parametrize("rows", [False, True])
def test_decode_append_is_the_format_on_the_bf16_rows(L, dev, rows):
    nh, S = 2, 64
    cases = ([([5, 63, 70], [0, 7, 13]), ([64, 1, 200], [63, 0, 5])] if rows else
             [([40], [9]), ([80], [63]), ([0], [0])])
    for pos, ring in cases:
        B = len(pos) if rows else 3
        qkv = _qkv(dev, B, nh, seed=sum(pos))
        qkv[0, 0, nh * 128:nh * 128 + 5] = 0   # a partly zero key
        c8 = Cache8.random(dev, B, nh, S, seed=1)
        kc, vc = c8.values()
        run16(L, qkv, kc, vc, pos, ring, nh, rows)
        run8(L, qkv, c8, pos, ring, nh, rows)
        for b in range(B):
            p, r = (pos[b], ring[b]) if rows else (pos[0], ring[0])
            s = _slot(p, r, S)
            for codes, scales, ref in ((c8.k, c8.ks, kc), (c8.v, c8.vs, vc)):
                wc, ws = quant(ref[b, :, s])
                assert _bits_equal(codes[b, :, s], wc) and _bits_equal(scales[b, :, s], ws), (pos, ring, b)


def test_prefill_append_and_output(L, dev):
    """T > 1: the codes of slots (t + ring) % S equal the format on the rotated keys / values b2l_attention_nocache
    computes, and y equals it bit for bit (with and without the adapter prefix)."""
    B, T, nh, S = 2, 150, 2, 256
    lib = L.lib()
    for ring, prefix in ((0, None), (100, _prefix(dev, nh))):
        g = torch.Generator(device=dev).manual_seed(ring)
        qkv = torch.randn((B, T, 3 * nh * 128), device=dev, generator=g).bfloat16()
        rope = _rope(dev, S)
        q16, y16 = qkv.clone(), torch.empty((B, T, nh * 128), device=dev, dtype=torch.bfloat16)
        args = (q16.data_ptr(), rope.data_ptr(), y16.data_ptr(), _work(L, B, nh, T, dev, T).data_ptr(), B, T, nh, 128, S)
        rc = (lib.b2l_attention_nocache(*args, L.stream_ptr()) if prefix is None
              else lib.b2l_attention_nocache_adapter(*args, C.byref(prefix), L.stream_ptr()))
        L.check(rc, "nocache")
        c8 = Cache8.random(dev, B, nh, S, seed=2)
        q8, y8 = qkv.clone(), torch.empty_like(y16)
        ringv = torch.tensor([ring], dtype=torch.int32, device=dev)
        L.check(lib.b2l_attention_kv8(q8.data_ptr(), C.byref(c8.spec(L)), rope.data_ptr(), None, ringv.data_ptr(),
                                      y8.data_ptr(), _work(L, B, nh, S, dev, T).data_ptr(), B, T, nh, 128, S, S, 0,
                                      None if prefix is None else C.byref(prefix), L.stream_ptr()), "kv8 prefill")
        torch.cuda.synchronize()
        assert _bits_equal(y8, y16) and _bits_equal(q8, q16)
        C_ = nh * 128
        slots = (torch.arange(T, device=dev) + ring) % S
        for third, codes, scales in ((1, c8.k, c8.ks), (2, c8.v, c8.vs)):
            rows = q16[..., third * C_:(third + 1) * C_].view(B, T, nh, 128).transpose(1, 2)
            wc, ws = quant(rows)
            got = codes.view(torch.uint8)[:, :, slots].view(torch.float8_e4m3fn)
            assert _bits_equal(got, wc) and _bits_equal(scales[:, :, slots], ws), ring


# ---------------------------------------------------------------------------------------------------------- 2. same
def _grid_value(dev, B, nh, seed):
    """New values on the e4m3 grid times 2^-6 (amax 448 2^-6): the format reproduces them exactly."""
    g = torch.Generator(device=dev).manual_seed(seed)
    c = (torch.randn((B, nh, 128), device=dev, generator=g) * 40).to(torch.float8_e4m3fn).float()
    c[..., 3] = 448.0
    return (c * 2.0 ** -6).bfloat16()


@pytest.mark.parametrize("p0", [100, 255, 700, 1500, 2047])
@pytest.mark.parametrize("adapter", [False, True])
def test_fp8_launch_equals_bf16_launch_on_the_read_back_cache(L, dev, p0, adapter):
    B, nh, S = 3, 4, 2048
    qkv = _qkv(dev, B, nh, seed=p0)
    C_ = nh * 128
    qkv[..., C_:2 * C_] = 0                                    # new key: zero
    qkv[..., 2 * C_:] = _grid_value(dev, B, nh, p0).view(B, 1, C_)
    c8 = Cache8.random(dev, B, nh, S, seed=p0, kmag=2.0)
    kc, vc = c8.values()
    pre = _prefix(dev, nh) if adapter else None
    for rows, pos, ring in ((False, [p0], [17]), (True, [p0, max(p0 - 300, 0), min(p0 + 37, 2047)], [0, 5, 2040])):
        a = run8(L, qkv, c8.clone(), pos, ring, nh, rows, pre)
        b = run16(L, qkv, kc.clone(), vc.clone(), pos, ring, nh, rows, pre)
        assert _bits_equal(a, b), (rows, pos)


# ---------------------------------------------------------------------------------------------------------- 3. invariances
def test_rows_equal_batch1_and_permutations(L, dev):
    nh, S = 4, 2048
    pos, ring = [30, 300, 1100, 2047], [0, 3, 900, 5]
    B = len(pos)
    qkv = _qkv(dev, B, nh, seed=3)
    c8 = Cache8.random(dev, B, nh, S, seed=3)
    c_all = c8.clone()
    y = run8(L, qkv, c_all, pos, ring, nh, rows=True)
    for b in range(B):
        one = Cache8(c8.k[b:b + 1], c8.ks[b:b + 1], c8.v[b:b + 1], c8.vs[b:b + 1]).clone()
        y1 = run8(L, qkv[b:b + 1].contiguous(), one, [pos[b]], [ring[b]], nh)
        assert _bits_equal(y[b:b + 1], y1), b
        assert _bits_equal(one.k[0], c_all.k[b]) and _bits_equal(one.ks[0], c_all.ks[b])
    # rows reversed and heads permuted
    rp, hp = torch.tensor([3, 1, 0, 2], device=dev), torch.tensor([2, 0, 3, 1], device=dev)
    q3 = qkv.view(B, 1, 3, nh, 128)[rp][:, :, :, hp].reshape(B, 1, -1).contiguous()
    f8 = lambda t: t.view(torch.uint8)[rp][:, hp].view(torch.float8_e4m3fn)   # noqa: E731
    cp = Cache8(f8(c8.k), c8.ks[rp][:, hp], f8(c8.v), c8.vs[rp][:, hp])
    yp = run8(L, q3, cp, [pos[i] for i in rp.tolist()], [ring[i] for i in rp.tolist()], nh, rows=True)
    assert _bits_equal(yp, y.view(B, 1, nh, 128)[rp][:, :, hp].reshape(B, 1, -1))


def test_graph_replay_repeats_and_unread_slots_may_be_nan(L, dev):
    nh, S, B = 2, 1024, 2
    pos, ring = [600, 90], [1000, 0]
    qkv = _qkv(dev, B, nh, seed=4)
    c8 = Cache8.random(dev, B, nh, S, seed=4)
    y0 = run8(L, qkv, c8.clone(), pos, ring, nh, rows=True)
    # every slot no launch at these positions reads: NaN codes and scales
    nan = c8.clone()
    for b in range(B):
        L_ = min(pos[b], S - 1) + 1
        unread = (torch.arange(L_, S, device=dev) + ring[b]) % S
        nan.k.view(torch.uint8)[b][:, unread] = 0x7f
        nan.v.view(torch.uint8)[b][:, unread] = 0x7f
        nan.ks[b][:, unread] = math.nan
        nan.vs[b][:, unread] = math.nan
    assert _bits_equal(run8(L, qkv, nan, pos, ring, nh, rows=True), y0)
    # CUDA graph: three replays from the same cache state repeat
    lib = L.lib()
    c = c8.clone()
    start = c.clone()
    y = torch.empty((B, 1, nh * 128), device=dev, dtype=torch.bfloat16)
    posv, ringv = torch.tensor(pos, device=dev), torch.tensor(ring, dtype=torch.int32, device=dev)
    rope, work, spec = _rope(dev, S), _work(L, B, nh, S, dev), c.spec(L)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            lib.b2l_attention_kv8(qkv.data_ptr(), C.byref(spec), rope.data_ptr(), posv.data_ptr(), ringv.data_ptr(),
                                  y.data_ptr(), work.data_ptr(), B, 1, nh, 128, S, S, L.F_ROW_POS | L.F_PDL, None,
                                  s.cuda_stream)
    for _ in range(3):
        for t, t0 in ((c.k, start.k), (c.v, start.v), (c.ks, start.ks), (c.vs, start.vs)):
            t.copy_(t0)
        g.replay()
        torch.cuda.synchronize()
        assert _bits_equal(y, y0)


def test_value_scaling_by_powers_of_two(L, dev):
    nh, S, B = 2, 512, 2
    pos, ring = [400, 77], [3, 500]
    qkv = _qkv(dev, B, nh, seed=6)
    c8 = Cache8.random(dev, B, nh, S, seed=6)
    c0 = c8.clone()
    y0 = run8(L, qkv, c0, pos, ring, nh, rows=True)
    C_ = nh * 128
    for e in (-20, -3, 5, 30):
        q = qkv.clone()
        q[..., 2 * C_:] = (q[..., 2 * C_:].float() * 2.0 ** e).bfloat16()
        c = c8.clone()
        c.vs.mul_(2.0 ** e)
        y = run8(L, q, c, pos, ring, nh, rows=True)
        assert _bits_equal(c.v, c0.v) and torch.equal(c.vs, c0.vs * 2.0 ** e), e
        assert torch.equal(y.float(), y0.float() * 2.0 ** e), e


# ---------------------------------------------------------------------------------------------------------- 4. float64
def _half_ulp_bf16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


def _exact(qh, k, v, L_, n_tiles):
    """float64 attention of one query per group over L_ keys and tests/test_gpu_attention.py's bar for the decode
    kernel (SERIAL 1, ACC 6): scores within (2 hs + hs/8 + 6) u A_j, each weight within expm1 of that plus
    u (3 (n_tiles + 24) + 3 (M - s_j)), accumulations within (6 n_tiles + 64) u (sum pi |v| + |y|)."""
    hs = qh.shape[-1]
    s = torch.einsum("gd,gjd->gj", qh, k[:, :L_]) / math.sqrt(hs)
    A = torch.einsum("gd,gjd->gj", qh.abs(), k[:, :L_].abs()) / math.sqrt(hs)
    M = s.amax(-1, keepdim=True)
    pi = torch.softmax(s, -1)
    vv = v[:, :L_]
    y = torch.einsum("gj,gjd->gd", pi, vv)
    eta = (2 * hs + hs // 8 + 6) * U * A + U * (3 * (n_tiles + 24) + 3 * (M - s))
    w = pi * torch.expm1(eta)
    dev_term = torch.einsum("gj,gjd->gd", w, vv.abs()) + w.sum(-1, keepdim=True) * y.abs()
    dev_term = dev_term / (1 - w.sum(-1, keepdim=True))
    mag = torch.einsum("gj,gjd->gd", pi, vv.abs())
    return y, dev_term + (6 * n_tiles + 64) * U * (mag + y.abs())


@pytest.mark.parametrize("dist", ["flat", "sink", "massive", "cancel"])
@pytest.mark.parametrize("p0", [200, 1800])
def test_against_float64(L, dev, dist, p0):
    B, nh, S = 2, 4, 2048
    g = torch.Generator(device=dev).manual_seed(p0)
    kl = torch.randn((B, nh, S, 128), device=dev, generator=g)
    vl = torch.randn((B, nh, S, 128), device=dev, generator=g)
    qkv = _qkv(dev, B, nh, seed=p0)
    C_ = nh * 128
    q = qkv[..., :C_].view(B, nh, 128)
    if dist == "sink":   # slot 0 takes most of the mass through the low-frequency pairs
        q[..., 120:] = 2.0
        kl.mul_(0.3)
        kl[..., 120:] = 0.0
        kl[:, :, 0, 120:] = math.log(0.99 / 0.01 * S) * math.sqrt(128) / 16
        vl[:, :, 0] *= 0.02
    elif dist == "massive":
        q[..., 124:] = 40.0
        kl[..., 124:] = (torch.rand((B, nh, S, 4), device=dev, generator=g) * 2 - 1) * 1e3
    elif dist == "cancel":
        vl = torch.sign(vl) * (1000 + 30 * torch.randn((B, nh, S, 128), device=dev, generator=g))
        qkv[..., 2 * C_:] = (torch.sign(qkv[..., 2 * C_:].float()) * 1000).bfloat16()
    kc, ks = quant(kl.bfloat16())
    vc, vs = quant(vl.bfloat16())
    c8 = Cache8(kc, ks, vc, vs)
    ring = 0
    y = run8(L, qkv, c8, [p0], [ring], nh)
    kv_k, kv_v = back(c8.k, c8.ks).double(), back(c8.v, c8.vs).double()   # the new token included, as read back
    # the rotated query as the kernel forms it: rbf(rot(q)) (RoPE table row p0)
    rope = _rope(dev, S)[p0]
    qq = qkv[..., :C_].reshape(B * nh, 64, 2).float()
    c, s_ = rope[:, 0], rope[:, 1]
    qr = torch.stack((qq[..., 0] * c - qq[..., 1] * s_, qq[..., 1] * c + qq[..., 0] * s_), -1).reshape(B * nh, 128)
    qh = qr.bfloat16().double()
    L_ = p0 + 1
    yx, eps = _exact(qh, kv_k.view(B * nh, S, 128), kv_v.view(B * nh, S, 128), L_, (S + 63) // 64)
    got = y.view(B * nh, 128).double()
    bar = _half_ulp_bf16(yx.abs() + eps) + eps
    over = (got - yx).abs() > bar
    assert bool(torch.isfinite(got).all()) and not bool(over.any()), (dist, int(over.sum()))


# ---------------------------------------------------------------------------------------------------------- 5. model
CFG = dict(block_size=512, vocab_size=96, n_layer=2, n_head=2, n_embd=256)
RTOL, ATOL = 1e-3, 5e-3   # tests/test_gpu_model.py's fused-vs-module tolerance


def _tiny(dev, mode="gptq.int4", seed=1234):
    from gpu_util import build_tiny

    m, _, _ = build_tiny(dev, CFG, mode=mode, seed=seed)
    return m


def _decode(m, prompt, steps, S, dev):
    """Prefill then greedy `steps` batch-1 steps; returns the list of logits (prefill's last row first)."""
    out = [m(prompt.view(1, -1), S, torch.arange(prompt.numel(), device=dev))[0, -1].float()]
    tok, p = int(out[0].argmax()), prompt.numel()
    for i in range(steps):
        lg = m(torch.tensor([[tok]], device=dev), S, torch.tensor([p + i], device=dev))[0, -1].float()
        out.append(lg.clone())
        tok = int(lg.argmax())
    return out


def test_prompt_logits_equal_the_no_cache_forward(dev):
    m = _tiny(dev)
    m.kv_cache_dtype = "fp8"
    prompt = torch.randint(0, 96, (1, 37), generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad():
        want = m(prompt)
        got = m(prompt, 64, torch.arange(37, device=dev))
        assert torch.equal(got, want)
        with pytest.raises(ValueError, match="nonzero position"):
            m(prompt[:, :5], 64, torch.arange(37, 42, device=dev))
        with pytest.raises(RuntimeError, match="fp8 KV cache"):
            m.decode_tokens(prompt[:, :3], 64, torch.arange(37, 40, device=dev))


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8", "llm.int8"])
def test_step_against_module_path(dev, mode):
    prompt = torch.randint(0, 96, (20,), generator=torch.Generator().manual_seed(2)).to(dev)
    runs = []
    with torch.no_grad():
        for fast in (True, False):
            m = _tiny(dev, mode)
            m.kv_cache_dtype = "fp8"
            m.int8_step = True
            if not fast:
                m._fast_ok = False
            runs.append(_decode(m, prompt, 6, 64, dev))
            if mode == "llm.int8" and fast:
                assert m._decode is not None and m._decode.args.flags & 32768
    for a, b in zip(*runs):
        if mode == "llm.int8":   # the bf16 int8_step equals its module path bit for bit, and so does the fp8 one
            assert torch.equal(a, b)
        else:
            torch.testing.assert_close(a, b, rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_batched_rows_equal_batch1_past_256(dev, mode):
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, 96, (n,), generator=g).to(torch.int32).to(dev) for n in (270, 300, 5)]
    S = 512
    with torch.no_grad():
        m = _tiny(dev, mode)
        m.q4_batch_step = m.w8_batch_step = True
        m.kv_cache_dtype = "fp8"
        rows = [m.prefill_rows(prompts, S)]
        pos = torch.tensor([[p.numel()] for p in prompts], device=dev)
        toks = rows[0].argmax(-1).view(-1, 1).to(torch.int32)
        for _ in range(8):
            lg = m(toks, S, pos)[:, -1].float()
            rows.append(lg.clone())
            toks, pos = lg.argmax(-1).view(-1, 1).to(torch.int32), pos + 1
        assert m._decode.args.flags & 32768
        for b, p in enumerate(prompts):
            m.reset_cache()
            one = _decode(m, p, 8, S, dev)
            for i in range(9):
                assert torch.equal(rows[i][b].float(), one[i]), (b, i)


def test_generate_prompts_and_stream_equal_generate(dev):
    from lit_llama_b200.generate import generate, generate_prompts, generate_stream

    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, 96, (n,), generator=g).to(torch.int32).to(dev) for n in (9, 40, 3, 17, 25)]
    with torch.no_grad():
        m = _tiny(dev)
        m.q4_batch_step = True
        m.kv_cache_dtype = "fp8"
        want = []
        for p in prompts:
            m.reset_cache()
            want.append(generate(m, p, 12, max_seq_length=64, top_k=1))
        m.reset_cache()
        got = generate_prompts(m, prompts[:3], 12, max_seq_length=64, top_k=1)
        m.reset_cache()
        got_s = generate_stream(m, prompts, 12, batch_size=2, max_seq_length=64, top_k=1)
    for a, b in zip(got, want[:3]):
        assert torch.equal(a, b)
    for a, b in zip(got_s, want):
        assert torch.equal(a, b)


def test_logical_kv_caches_and_expand(dev):
    m = _tiny(dev)
    m.kv_cache_dtype = "fp8"
    S = 16
    prompt = torch.randint(0, 96, (1, 10), generator=torch.Generator().manual_seed(5)).to(dev)
    with torch.no_grad():
        m(prompt, S, torch.arange(10, device=dev))
        for i in range(12):   # past S: the ring rolls
            m(torch.tensor([[i + 1]], device=dev), S, torch.tensor([10 + i], device=dev))
        ring = int(m._ring.item())
        assert ring > 0
        for c, (lk, lv) in zip(m.kv_caches, m.logical_kv_caches()):
            for code, scale, got in ((c[0], c.k_scale, lk), (c[1], c.v_scale, lv)):
                idx = (torch.arange(S, device=dev) + ring) % S
                assert torch.equal(got, back(code, scale)[:, :, idx].bfloat16())
        m.expand_cache(3)
        assert m.kv_caches[0][0].shape[0] == 3 and torch.equal(m.kv_caches[0].k_scale[2], m.kv_caches[0].k_scale[0])
        assert _bits_equal(m.kv_caches[1][1][1], m.kv_caches[1][1][0])


# ---------------------------------------------------------------------------------------------------------- 6. quality
def test_quality_bf16_against_fp8_reported(dev, capsys):
    """Not gated: the largest |logit difference| and the greedy-token agreement of the fp8 cache against the bf16
    cache, each arm decoding its own greedy tokens for 256 steps after the same prompt."""
    prompt = torch.randint(0, 96, (16,), generator=torch.Generator().manual_seed(6)).to(dev)
    res = {}
    for mode in ("gptq.int4", "gptq.int8"):
        arms = []
        with torch.no_grad():
            for dt in (None, "fp8"):
                m = _tiny(dev, mode)
                m.kv_cache_dtype = dt
                arms.append(_decode(m, prompt, 256, 512, dev))
        a, b = arms
        same = [int(x.argmax()) == int(y.argmax()) for x, y in zip(a, b)]
        first = same.index(False) if False in same else len(same)
        dmax = max(float((x - y).abs().max()) for x, y in zip(a[:first + 1], b[:first + 1]))
        res[mode] = dict(agree=sum(same) / len(same), first_divergence=first, max_abs_dlogit_until_then=dmax)
    with capsys.disabled():
        print(f"\nfp8 vs bf16 KV cache, tiny head-size-128 models, 256 greedy steps: {res}")

"""-m gpu: the batch-1 GEMV (b2l_q4_gemv, b2l_w8_gemv) against a host restatement of its arithmetic, bit for bit.

The restatement follows q4_gemv_kernel step by step: the RMSNorm sum of bf16-rounded squares in the kernel's thread,
warp and block order, rms_rinv, the 2^sh choice from max|v|, X = rint(v 2^sh), the exact Σ level·X and Σ X, one fp32
rounding of (Σ level·X − zero·Σ X)·2^-sh, then the bf16 epilogue (affine, residual, SwiGLU).  Every 7B / 13B / 65B
linear shape runs, plus ragged N, on the default grid and on explicit grids of one and two CTAs per SM: the integer
contraction does not depend on how the row blocks are split, so every grid must give the same bits."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NT = 256        # prologue threads (8 consumer warps); thread t owns k = (c NT + t) 8 .. + 7 of chunk c
NDIG = 3        # balanced base-256 digits: |X| < 2^22

# (name, N, K, prologue, epilogue): the linears of one Block and the head, as the decode step runs them
_LAYERS = [("c_attn", 3, 1, "rms", "store"), ("c_proj", 1, 1, None, "res"), ("fc12", None, 1, "rms", "swiglu"),
           ("mlp_proj", 1, None, None, "res"), ("lm_head", "vocab", 1, "rms", "store")]
_MODELS = {"7B": (4096, 11008), "13B": (5120, 13824), "65B": (8192, 22016)}


def _shapes():
    out = []
    for m, (C_, H) in _MODELS.items():
        for name, nf, kf, pro, epi in _LAYERS:
            N = 32000 if nf == "vocab" else (2 * H if nf is None else nf * C_)
            K = H if kf is None else kf * C_
            out.append(pytest.param(N, K, pro, epi, id=f"{m}-{name}"))
    # ragged N (not a multiple of 16 or of two row blocks), every epilogue but SwiGLU (which needs N % 16 == 0)
    out += [pytest.param(4100, 4096, "rms", "store", id="ragged-4100"), pytest.param(12290, 4096, None, "res", id="ragged-12290"),
            pytest.param(40, 11008, "rms", "res", id="ragged-40"), pytest.param(8200, 64, None, "store", id="ragged-8200-K64")]
    return out


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _rbf(a):
    """fp32 -> bf16 -> fp32 (round to nearest even), as numpy float32."""
    return torch.from_numpy(np.array(a, dtype=np.float32)).bfloat16().float().numpy()


def _prologue(x, g, eps):
    """The kernel's activation row: (X int64 [K], sh).  x, g: bf16 values as float32 numpy [K] (g None: no RMSNorm)."""
    K = x.shape[0]
    nchunk = -(-K // (NT * 8))
    xp = np.zeros(nchunk * NT * 8, np.float32)
    xp[:K] = x
    xt = xp.reshape(nchunk, NT, 8)
    if g is not None:
        sq = _rbf(xt * xt)                        # HMUL2: exact product, one bf16 rounding
        ss = np.zeros(NT, np.float32)
        for c in range(nchunk):                   # per thread: chunks, then pairs (lo + hi first)
            for q in range(4):
                ss = (ss + (sq[c, :, 2 * q] + sq[c, :, 2 * q + 1])).astype(np.float32)
        v = ss.reshape(8, 32)
        for o in (16, 8, 4, 2, 1):                # warp_sum: xor butterfly; lane 0 is stored
            v = (v + v[:, np.arange(32) ^ o]).astype(np.float32)
        tot = np.float32(0)
        for w in range(8):
            tot = np.float32(tot + v[w, 0])
        ms = _rbf(np.float32(tot) / np.float32(K))
        t = _rbf(ms + np.float32(eps))
        rinv = _rbf(np.float32(1.0) / np.sqrt(t, dtype=np.float32))
        mx = np.float32(np.abs(_rbf(g * x)).max(initial=0.0))
        mx = np.float32(np.float32(mx * rinv) * np.float32(1.02))
        v = _rbf(g * _rbf(x * rinv))
    else:
        mx = np.float32(np.abs(x).max(initial=0.0))
        v = x
    e = int((np.array(mx, np.float32).view(np.uint32) >> 23) & 0xFF) - 127
    sh = max(-126, min(126, (8 * NDIG - 3) - e))
    X = np.rint(v.astype(np.float64) * 2.0 ** sh).astype(np.int64)   # fma(v, 2^sh, 1.5 2^23): half to even
    assert np.abs(X).max(initial=0) < 2 ** 22
    return X, sh


def _expected(lv, sc, z, x, g, eps, epi, res, aff, dev):
    """bf16 output of the kernel, restated on the host (SwiGLU's expf evaluated by torch on the device: the kernel and
    torch both call CUDA's expf)."""
    X, sh = _prologue(x, g, eps)
    # Σ level·X: integer products below 2^30 and sums below 2^53, so float64 arithmetic is exact in any order
    Xd = torch.from_numpy(X.astype(np.float64))
    tq = torch.cat([lv[i:i + 4096].double() @ Xd for i in range(0, lv.shape[0], 4096)])
    sum_x = float(X.sum())
    tf = ((tq - z.double() * sum_x) * 2.0 ** -sh).float()             # one fp32 rounding
    v = (sc.float() * tf).bfloat16().float()
    if aff is not None:
        s, b = aff
        v = (s.float() * (v + b.float()).bfloat16().float()).bfloat16().float()
    if epi == "res":
        return (v + res.float()).bfloat16()
    if epi == "swiglu":
        blocks = v.view(-1, 2, 8).to(dev)
        a, b = blocks[:, 0], blocks[:, 1]
        sl = (a / (1.0 + torch.exp(-a))).bfloat16().float()
        return (sl * b).bfloat16().reshape(-1).cpu()
    return v.bfloat16()


def _weights(N, K, bits, seed, sz_f32=False):
    g = torch.Generator().manual_seed(seed)
    maxq = 2 ** bits - 1
    lv = torch.randint(0, maxq + 1, (N, K), generator=g, dtype=torch.uint8)
    if bits == 4:
        qw = lv[:, 0::2] | (lv[:, 1::2] << 4)
    else:
        qw = lv
    qw = qw.t().contiguous().t()              # reference layout: byte [k / epb][o]
    dt = torch.float32 if sz_f32 else torch.bfloat16
    sc = (torch.rand(N, 1, generator=g) * 0.01 + 0.002).to(dt)
    z = torch.randint(0, maxq + 1, (N, 1), generator=g).to(dt)
    return lv, qw, sc, z


def _launch(bits, x, qt, sc, z, N, K, *, g, eps, epi, res, aff, grid, n_out):
    L = _L()
    y = torch.full((1, n_out), float("nan"), device=x.device, dtype=torch.bfloat16)
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                       sz_dtype=L.sz_dtype_of(sc), y=y.data_ptr(), ldy=n_out, M=1, N=N, K=K,
                       prologue=L.PRO_RMSNORM if g is not None else L.PRO_NONE,
                       norm_scale=None if g is None else g.data_ptr(), eps=eps,
                       epilogue={"store": L.EPI_STORE, "res": L.EPI_RESIDUAL, "swiglu": L.EPI_SWIGLU}[epi],
                       res=None if res is None else res.data_ptr(), ldres=N, split_k=grid, flags=0)
    if aff is not None:
        a.out_affine.scale, a.out_affine.bias = aff[0].data_ptr(), aff[1].data_ptr()
    fn = "b2l_w8_gemv" if bits == 8 else "b2l_q4_gemv"
    L.check(getattr(L.lib(), fn)(C.byref(a), L.stream_ptr()), fn)
    torch.cuda.synchronize()
    return y[0].cpu()


def _check(dev, bits, N, K, pro, epi, *, affine, sz_f32=False):
    from lit_llama_b200.quantization import tile_i8

    seed = N * 7 + K + bits
    lv, qw, sc, z = _weights(N, K, bits, seed, sz_f32)
    qt = tile_i8(qw.to(dev), N, K, bits)
    gen = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(K, generator=gen) * 1.5
    x[K // 3] = 900.0                                       # one massive channel, as LLaMA's hidden state has
    x = x.bfloat16()
    g = (1 + 0.2 * torch.randn(K, generator=gen)).bfloat16() if pro == "rms" else None
    g_np = None if g is None else g.float().numpy()
    res = (torch.randn(N, generator=gen) * 0.5).bfloat16() if epi == "res" else None
    aff = ((1 + 0.1 * torch.randn(N, generator=gen)).bfloat16(), (0.05 * torch.randn(N, generator=gen)).bfloat16()) if affine else None
    eps = 1e-5
    want = _expected(lv, sc.view(-1), z.view(-1), x.float().numpy(), g_np, eps, epi, res, aff, dev)
    n_out = N // 2 if epi == "swiglu" else N
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    to = lambda t: None if t is None else t.to(dev)
    args = dict(g=to(g), eps=eps, epi=epi, res=to(res), aff=None if aff is None else (to(aff[0]), to(aff[1])), n_out=n_out)
    xd, scd, zd = x.to(dev).view(1, K), sc.to(dev), z.to(dev)
    for grid in (0, sms, 2 * sms):            # the default grid, one CTA per SM, two CTAs per SM
        got = _launch(bits, xd, qt, scd, zd, N, K, grid=grid, **args)
        bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
        assert bad.numel() == 0, (f"bits={bits} N={N} K={K} grid={grid}: {bad.numel()} of {n_out} outputs differ, first "
                                  f"{int(bad[0])}: got {float(got[bad[0]])} want {float(want[bad[0]])}")


@pytest.mark.parametrize("N,K,pro,epi", _shapes())
def test_q4_gemv_equals_restatement(dev, N, K, pro, epi):
    _check(dev, 4, N, K, pro, epi, affine=False)


@pytest.mark.parametrize("N,K,pro,epi", _shapes())
def test_w8_gemv_equals_restatement(dev, N, K, pro, epi):
    _check(dev, 8, N, K, pro, epi, affine=False)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K,pro,epi", [(12288, 4096, "rms", "store"), (4096, 11008, None, "res"), (22016, 4096, "rms", "swiglu"),
                                         (4100, 4096, None, "store")])
def test_gemv_affine_equals_restatement(dev, bits, N, K, pro, epi):
    """LLaMA-Adapter v2's per-row scale and bias ahead of the epilogue (the AFFINE instantiations)."""
    _check(dev, bits, N, K, pro, epi, affine=True)


@pytest.mark.parametrize("bits", [4, 8])
def test_gemv_fp32_scales_equal_restatement(dev, bits):
    _check(dev, bits, 4096, 4096, "rms", "res", affine=False, sz_f32=True)

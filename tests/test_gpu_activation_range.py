"""-m gpu: the gptq linears across the activation range.

Every other linear test draws its activations from randn (row max about 4, RMSNorm weights 1 +- 0.1).  LLaMA's hidden
states are different: a few "massive" channels reach 1e3..1e4, RMSNorm weights span two orders of magnitude and the
massive channels carry small ones.  Three properties, for every entry point that serves gptq.int4 / gptq.int8:

1. power-of-two scale equivariance, bit for bit: y(2^e x) == 2^e y(x) (residual scaled alike), and for the RMSNorm
   prologue y(2^e g) == 2^e y(g) with x fixed (RMSNorm is not scale-invariant in x because of eps).  Every rounding in
   these kernels is relative to a power-of-two exponent, so a miss means a magnitude-dependent step;
2. mixed-magnitude batches: rows scaled by 2^e_r (e_r in -30..30) and a zero row give each row's unscaled result times
   2^e_r, so no scale is shared across rows;
3. massive-activation rows against float64 exact arithmetic, the RMSNorm row computed on the host by the kernel's
   chain (rms_rinv, then bf16(g bf16(x rinv))) and accepted with its own rinv or a one-ulp neighbour."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EXPS = [-40, -24, -16, -12, -8, -4, 4, 8, 12, 16, 24, 40]
SHAPES = [(130, 256), (12288, 4096), (1024, 22016)]   # ragged, 7B c_attn, the wide (K > 12288) prologue
CPROJ = (4096, 11008)                                  # 7B mlp.c_proj: its input carries the largest activations

# entry point -> (weight bits, batch sizes, fused RMSNorm / residual)
KINDS = {
    "q4_gemv": (4, (1,), True),
    "w8_gemv": (8, (1,), True),
    "q4_gemv_batch": (4, (2, 5, 8), True),
    "q4_gemv_batch_i8": (4, (2, 9, 16), True),
    "w8_gemv_batch": (8, (2, 9, 16), True),
    "q4_linear_tc": (4, (9, 16), True),
    "q4_gemm": (4, (17, 300), False),
    "w8_gemm": (8, (17, 300), False),
}
CASES = [(k, M) for k, (_, ms, _) in KINDS.items() for M in ms]
BATCH1 = ("q4_gemv", "w8_gemv")
GEMMS = ("q4_gemm", "w8_gemm")
# share of outputs bit-equal to the correctly rounded exact result: exact integer contraction (batch-1 and the digit
# batch kernels, whose rows equal batch-1 bit for bit) vs fp32 accumulation (f16 mma.sync, wgmma)
MIN_EQUAL = {"q4_gemv": 0.995, "w8_gemv": 0.995, "q4_gemv_batch_i8": 0.995, "w8_gemv_batch": 0.995,
             "q4_gemv_batch": 0.8, "q4_linear_tc": 0.98}


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


_WEIGHTS = {}


def _weights(dev, N, K, bits):
    """Random levels / scales / zeros (gpu_util.rand_q4) and every tiling of them, built once per shape."""
    key = (N, K, bits)
    if key not in _WEIGHTS:
        from gpu_util import rand_q4

        lv, qw, sc, z = rand_q4(N, K, dev, seed=N + K + bits, bits=bits)
        _WEIGHTS[key] = dict(lv=lv, qw=qw, sc=sc, z=z, N=N, K=K, bits=bits, tiles={})
    return _WEIGHTS[key]


def _tiled(w, kind):
    from gpu_util import tile, tile_mma
    from lit_llama_b200.quantization import tile_i8

    L = _L()
    if kind not in w["tiles"]:
        qw, N, K = w["qw"], w["N"], w["K"]
        if kind in ("q4_gemv", "q4_gemv_batch_i8", "w8_gemv", "w8_gemv_batch"):
            t = tile_i8(qw, N, K, w["bits"])
        elif kind == "q4_gemv_batch":
            t = tile_mma(L, qw, N, K)
        elif kind in ("q4_linear_tc", "q4_gemm"):
            t = tile(L, qw, N, K)
        else:
            t = qw   # b2l_w8_gemm reads quant_weight in the reference layout
        w["tiles"][kind] = t
    return w["tiles"][kind]


def _run(kind, w, x, *, g=None, res=None):
    """y = linear(x) through b2l_<kind> (the batch-1 kernels one row per call); `g`: RMSNorm prologue weight; `res`:
    residual epilogue."""
    L = _L()
    lib = L.lib()
    N, K = w["N"], w["K"]
    qt, sc, z = _tiled(w, kind), w["sc"], w["z"]
    M = x.shape[0]
    y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16)
    ws = None
    if kind == "q4_gemv_batch":
        ws = torch.zeros(lib.b2l_q4_gemv_batch_workspace_bytes(K), dtype=torch.uint8, device=x.device)
    elif kind in ("q4_gemv_batch_i8", "w8_gemv_batch"):
        ws = torch.zeros(lib.b2l_w8_gemv_batch_workspace_bytes(K, M), dtype=torch.uint8, device=x.device)
    calls = [(slice(r, r + 1)) for r in range(M)] if kind in BATCH1 else [slice(0, M)]
    for s in calls:
        xs, ys = x[s], y[s]
        a = L.Q4LinearArgs(x=xs.data_ptr(), ldx=x.stride(0), qw_tiled=qt.data_ptr(), scales=sc.data_ptr(),
                           zeros=z.data_ptr(), sz_dtype=L.sz_dtype_of(sc), y=ys.data_ptr(), ldy=N, M=xs.shape[0], N=N,
                           K=K, prologue=L.PRO_NONE if g is None else L.PRO_RMSNORM,
                           norm_scale=None if g is None else g.data_ptr(), eps=1e-5,
                           epilogue=L.EPI_STORE if res is None else L.EPI_RESIDUAL,
                           res=None if res is None else res[s].data_ptr(), ldres=N, split_k=0, flags=0,
                           workspace=None if ws is None else ws.data_ptr())
        L.check(getattr(lib, "b2l_" + kind)(C.byref(a), L.stream_ptr()), kind)
    torch.cuda.synchronize()
    return y


def _normal_range(t, e=0):
    """Every nonzero |t| * 2^e is a bf16 normal (>= 2^-126, finite)."""
    a = t.float().abs()
    nz = a[a > 0]
    if nz.numel():
        assert math.ldexp(float(nz.min()), e) >= 2.0 ** -126 and math.ldexp(float(nz.max()), e) < 2.0 ** 127, e


def _randn_rows(M, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g) * 2
    if M > 2:
        x[M // 2] = 0
    return x.bfloat16()


def _pow2(e):
    return torch.tensor(2.0 ** e).bfloat16()


# ---------------------------------------------------------------- 1. power-of-two scale equivariance
@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("kind,M", CASES)
@pytest.mark.parametrize("case", ["store", "residual", "rmsnorm"])
def test_power_of_two_scaling_is_exact(dev, kind, M, N, K, case):
    if case != "store" and not KINDS[kind][2]:
        pytest.skip("plain linear only")
    w = _weights(dev, N, K, KINDS[kind][0])
    gen = torch.Generator().manual_seed(M + N + K)
    x = _randn_rows(M, K, M + K).to(dev)
    res = (torch.randn(M, N, generator=gen) * 4).bfloat16().to(dev) if case == "residual" else None
    g = None
    if case == "rmsnorm":
        g = torch.exp(torch.empty(K).uniform_(math.log(0.02), math.log(2.5), generator=gen)).bfloat16().to(dev)
    y0 = _run(kind, w, x, g=g, res=res)
    assert not y0.isnan().any()
    for e in EXPS:
        s = _pow2(e).to(dev)
        if case == "rmsnorm":
            _normal_range(g, e)
            y = _run(kind, w, x, g=g * s)
        else:
            _normal_range(x, e)
            assert float(x.float().abs().amax(-1)[x.float().abs().amax(-1) > 0].min()) * 2.0 ** e >= 2.0 ** -100
            y = _run(kind, w, x * s, res=None if res is None else res * s)
        _normal_range(y0, e)
        assert torch.equal(y, y0 * s), (e, int((y != y0 * s).sum()), y.numel())


# ---------------------------------------------------------------- 2. rows of very different magnitudes in one batch
@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("kind,M", [c for c in CASES if c[1] > 1])
@pytest.mark.parametrize("case", ["store", "residual"])
def test_mixed_magnitude_rows_keep_their_own_scale(dev, kind, M, N, K, case):
    if case != "store" and not KINDS[kind][2]:
        pytest.skip("plain linear only")
    w = _weights(dev, N, K, KINDS[kind][0])
    gen = torch.Generator().manual_seed(3 * M + N + K)
    x = (torch.randn(M, K, generator=gen) * 2).bfloat16()
    res = (torch.randn(M, N, generator=gen) * 4).bfloat16() if case == "residual" else None
    er = torch.linspace(-30, 30, M).round()
    er = er[torch.randperm(M, generator=gen)]
    sc = torch.pow(2.0, er).bfloat16().view(M, 1)
    xs = x * sc
    xs[M // 2] = 0
    ys_want_zero = M // 2
    y0 = _run(kind, w, x.to(dev), res=None if res is None else res.to(dev))
    y = _run(kind, w, xs.to(dev), res=None if res is None else (res * sc).to(dev))
    for r in range(M):
        if r == ys_want_zero:
            want = torch.zeros(N, dtype=torch.bfloat16) if res is None else (res[r] * sc[r])
            assert torch.equal(y[r].cpu(), want), r
            continue
        _normal_range(y0[r], int(er[r]))
        assert torch.equal(y[r].cpu(), (y0[r].cpu() * sc[r])), (r, int(er[r]))


# ---------------------------------------------------------------- 3. massive activations against exact arithmetic
def _massive_rows(M, K, seed, big_lower=None):
    """Student-t (5 dof) bulk with 1..3 massive channels per row at 10^2.5..10^4, one of them at k % 16 < 8 and one at
    k % 16 >= 8 (the two fp16 halves of a k16 chunk of the 2..8-row kernel), and RMSNorm weights log-uniform in
    [0.02, 2.5] with about 0.01 on the massive channels.  big_lower: the value of row 0's lower-half channel."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=gen) / torch.sqrt((torch.randn(5, M, K, generator=gen) ** 2).mean(0))
    blk = torch.randint(0, K // 16, (3,), generator=gen)
    off = torch.randint(0, 8, (3,), generator=gen)
    lo, hi, third = int(16 * blk[0] + off[0]), int(16 * blk[1] + 8 + off[1]), int(16 * blk[2] + off[2] + 8 * (off[2] % 2))
    for r in range(M):
        chans = ([lo, hi, third] if r % 2 == 0 else [hi, lo, third])[: 1 + r % 3]
        for c in chans:
            mag = 10.0 ** (2.5 + 1.5 * float(torch.rand(1, generator=gen)))
            x[r, c] = mag if float(torch.rand(1, generator=gen)) < 0.5 else -mag
    if big_lower is not None:
        x[0, lo] = big_lower
    g = torch.exp(torch.empty(K).uniform_(math.log(0.02), math.log(2.5), generator=gen))
    g[[lo, hi, third]] = 0.01 * (0.8 + 0.4 * torch.rand(3, generator=gen))
    return x.bfloat16(), g.bfloat16(), (lo, hi, third)


def _rms_candidates(x, g, eps=1e-5):
    """The rows the kernel feeds its linear after RMSNorm: rinv by rms_rinv (b2l_common.cuh) on the exact sum of the
    bf16-rounded squares, then bf16(g bf16(x rinv)); and the same with rinv one bf16 ulp up or down (the kernel's fp32
    sum runs in its own order and may land rinv on the neighbouring value, which rescales the whole row)."""
    K = x.shape[1]
    ss = (x.float() * x.float()).bfloat16().double().sum(-1, keepdim=True).float()
    ms = (ss / K).bfloat16().float()
    t = (ms + torch.tensor(eps, dtype=torch.float32)).bfloat16().float()
    rinv = (1.0 / torch.sqrt(t)).bfloat16()
    bits = rinv.view(torch.int16)
    return [g * (x * r) for r in (rinv, (bits + 1).view(torch.bfloat16), (bits - 1).view(torch.bfloat16))]


def _digit_grid(x):
    """x on the activation grid of the int8-digit kernels without a prologue: 2^-sh with max|x| 2^sh in [2^21, 2^22),
    round to nearest even (q4_gemv.cu).  Elements more than 2^14 below the row's largest are rounded there."""
    xd = x.double()
    mx = xd.abs().amax(-1, keepdim=True)
    sh = 21 - torch.floor(torch.log2(mx))
    return torch.round(xd * torch.pow(2.0, sh)) * torch.pow(2.0, -sh)


def _check_gemm(kind, y, x, w):
    """The wgmma GEMMs multiply get_weight's bf16 matrix (the reference's dense branch): products exact, fp32
    accumulation, one bf16 rounding.  Massive channels put most of a row's magnitude into one product, and every later
    fp32 addition of the k loop rounds at that magnitude: the bar on Σ|x w| is the 8-bit instantiation's (2^-16, the
    same kernel), not the 2^-20 that randn rows meet."""
    from gpu_util import relerr

    wb = ((w["lv"].to(torch.bfloat16) - w["z"].to(torch.bfloat16)) * w["sc"].to(torch.bfloat16)).double()
    want = x.double() @ wb.t()
    mag = x.double().abs() @ wb.abs().t()
    err = (y.double() - want).abs()
    bound = want.abs() * 2.0 ** -8 + mag * 2.0 ** -16 + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    assert relerr(y, want) < 2.0 ** -9
    assert float((y == want.float().bfloat16()).float().mean()) > 0.98


@pytest.mark.parametrize("N,K", SHAPES + [CPROJ])
@pytest.mark.parametrize("kind,M", CASES)
def test_massive_activation_rows_vs_exact(dev, kind, M, N, K):
    """With RMSNorm where the entry point fuses it (the shapes of SHAPES), and as raw mlp.c_proj-like input rows at
    K = 11008 with a lower-half element of 70000 (beyond fp16's 65504) and no prologue."""
    from gpu_util import assert_q4_linear_close, ref_linear, relerr

    rows = 3 if kind in BATCH1 else M
    cproj = (N, K) == CPROJ
    w = _weights(dev, N, K, KINDS[kind][0])
    x, g, chans = _massive_rows(rows, K, seed=rows + N + K, big_lower=70000.0 if cproj else None)
    assert chans[0] % 16 < 8 <= chans[1] % 16
    if kind in GEMMS:
        _check_gemm(kind, _run(kind, w, x.to(dev)), x.to(dev), w)
        return
    if cproj:
        y = _run(kind, w, x.to(dev))
        assert float(x.float().abs().max()) > 65504
        assert relerr(y, ref_linear(x.to(dev), w["lv"], w["sc"], w["z"])) < 1e-3 + 2.0 ** -9
        # 70000 over a bulk of about 1 is 2^16: more than the 2^14 the digit kernels represent exactly, so those are
        # held to the exact linear of the row on their documented grid
        cands = [_digit_grid(x) if MIN_EQUAL[kind] > 0.99 else x]
    else:
        y = _run(kind, w, x.to(dev), g=g.to(dev))
        cands = _rms_candidates(x, g)
    for r in range(rows):
        errs = []
        for xh in cands:
            try:
                assert_q4_linear_close(y[r:r + 1], xh[r:r + 1].to(dev), w["lv"], w["sc"], w["z"], min_equal=MIN_EQUAL[kind])
                break
            except AssertionError as ex:
                errs.append(str(ex))
        else:
            raise AssertionError(f"row {r}: {errs}")

"""-m gpu: every llm.int8 entry point against the exact restatement of LLM.int8() (oracle.llama_oracle.int8_linear_exact).

Entry points: b2l_q8_gemv (the re-tiled copy, with and without a given outlier mask), b2l_q8_gemv_cb, b2l_q8_gemm
(M = 2..2048), b2l_q8_linear (M = 1) and b2l_q8_linear_batch (M = 2..16) with the RMSNorm prologue, the v2 affine and
the store / residual / SwiGLU epilogues.  Shapes: the 7B, 13B, 30B and 65B linears, a 32000-row lm_head, K = 32768 and a
ragged N = 130.

Every output must lie in its admissible set (compared bit for bit where the set has one value, so inf signs and NaN
positions count), and a least share must be bit-equal to the single-rounded value.  The mask, SCA and CA are exact and
so are held exactly through the identity probe: CB = 127 I with SCB = 127 / SCA_m gives y = CA[m, k] on inlier columns
and |y| > 127 on outlier columns, so a failure names the row and column whose CA, SCA or mask is wrong.

Input families, each for one edge: randn rows with a few outliers; LLaMA-like massive channels (τ carries most of |y|);
outlier products at fp16's edge (inf); |x| = 6.0 and 5.96875 (the largest bf16 below 6) in one row only; rint ties
(SCA = 127/32, inliers ±(2j+1)/64); x outside fp16's normal range (2^-16..2^-26 rows, 65280 and 65536 columns); the
saturated contraction (CA = CB = ±127 at K = 32768); mixed-magnitude batches with a zero row; SCB large enough that the
dequantised part overflows."""
import ctypes as C
import math

import pytest
import torch

from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu

THR = 6.0
EPS = 1e-5
MIN_EQUAL = 0.995   # share bit-equal to the single-rounded value

SHAPES = {"7b_attn": (12288, 4096), "7b_cproj": (4096, 4096), "7b_fc": (11008, 4096), "7b_proj": (4096, 11008),
          "13b_fc": (13824, 5120), "13b_proj": (5120, 13824), "30b_fc": (17920, 6656), "30b_proj": (6656, 17920),
          "65b_fc": (22016, 8192), "65b_proj": (8192, 22016), "lm_head": (32000, 4096), "k32768": (1024, 32768),
          "ragged": (130, 4096)}
FAMILIES = ["randn", "massive", "fp16edge", "threshold", "ties", "tiny", "saturated", "mixed", "bigscb"]


_SHARES = []   # (case, share bit-equal to the single-rounded value), printed at the end (pytest -s) for the floor


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)
    if _SHARES:
        low = sorted(_SHARES, key=lambda c: c[1])[:5]
        print("\nlowest bit-equal shares:", ", ".join(f"{w}: {100 * v:.3f} %" for w, v in low))


def _L():
    from lit_llama_b200 import _lib as L

    return L


# ---------------------------------------------------------------- inputs
def _gen(seed):
    return torch.Generator().manual_seed(seed)


_W = {}


def _weight(N, K, dev, salt=0):
    key = (N, K, salt)
    if key not in _W:
        if len(_W) > 4:
            _W.clear()
        g = torch.Generator(device=dev).manual_seed(N * 31 + K + salt)
        cb = torch.randint(-127, 128, (N, K), generator=g, device=dev, dtype=torch.int8)
        scb = torch.rand(N, generator=g, device=dev) * 0.2 + 0.01
        _W[key] = (cb, scb)
    return _W[key]


def _family(fam, M, K, N, dev, seed):
    """(x [M, K] bf16, a transform of (cb, scb) or None)."""
    g = _gen(seed)
    x = torch.randn(M, K, generator=g)
    wf = None
    if fam == "randn":
        for i in range(4):
            x[(3 * i) % M, (97 * i + 13) % K] = (6.5 + 2 * i) * (-1) ** i
    elif fam == "massive":
        chans = torch.randperm(K, generator=g)[:2 + seed % 7]
        mags = torch.pow(10.0, 2 + 2 * torch.rand(len(chans), generator=g)) * torch.sign(torch.randn(len(chans), generator=g))
        x[:, chans] = mags * (0.8 + 0.4 * torch.rand(M, len(chans), generator=g))
    elif fam == "fp16edge":
        c1, c2 = (5 * K) // 7, K // 3
        x[:, c1] = 3.0e4
        x[M - 1, c2] = -4.5e4
        wf = lambda cb, scb: (cb, scb * 0 + torch.linspace(0.5, 3.0, len(scb), device=scb.device))
    elif fam == "threshold":
        x.clamp_(-5.5, 5.5)
        x[0, 5] = 6.0
        x[M - 1, K - 1] = -6.0
        x[M // 2, K // 2] = 5.96875
        x[M - 1, 17] = -5.96875
    elif fam == "ties":
        j = torch.randint(0, 127, (M, K), generator=g)
        x = (2 * j + 1).float() / 64 * torch.sign(torch.randn(M, K, generator=g))
        x[:, 3] = 127 / 32
    elif fam == "tiny":
        e = torch.tensor([-16 - (r * 10) // max(M - 1, 1) for r in range(M)], dtype=torch.float32)
        x = x.clamp(-1.9, 1.9) * torch.pow(2.0, e).unsqueeze(1)
        if M == 1 and seed % 2:
            x = (torch.rand(1, K, generator=g) * 2 - 1) * 2.0 ** -26   # fp16 zero: SCA = 0
        x[0, 11] = 65280.0
        x[M - 1, K - 7] = -65536.0
        wf = lambda cb, scb: (_zero_col(cb, K - 7), scb)
    elif fam == "saturated":
        s = torch.sign(torch.randn(M, K, generator=g))
        s[s == 0] = 1
        x = s.clone()
        def wf(cb, scb):
            row = (127 * s[0]).to(torch.int8).to(cb.device)
            cb = cb.clone()
            n = min(cb.shape[0], 512)
            cb[:n] = row
            off = torch.arange(n, device=cb.device)
            cols = torch.arange(K, device=cb.device)
            cb[:n] = torch.where(cols.unsqueeze(0) < off.unsqueeze(1), (126 * s[0]).to(torch.int8).to(cb.device), cb[:n])
            return cb, scb * 0 + torch.linspace(0.5, 1.9, len(scb), device=scb.device)
    elif fam == "mixed":
        e = torch.linspace(-20, 10, M).round()
        x = x * torch.pow(2.0, e).unsqueeze(1)
        if M > 2:
            x[M // 2] = 0
        x[M - 1, 29] = 9.0
    elif fam == "bigscb":
        x[0, 7] = 8.5
        x[M - 1, 91] = -7.0
        wf = lambda cb, scb: (cb, torch.pow(10.0, torch.linspace(0, 4.7, len(scb), device=scb.device))[torch.randperm(len(scb), device=scb.device)])
    return x.bfloat16().to(dev), wf


def _zero_col(cb, k):
    cb = cb.clone()
    cb[::7, k] = 0   # inf * 0 = NaN on those outputs
    return cb


def _mask_words(mask):
    K = mask.numel()
    w = (mask.view(K // 32, 32).long() << torch.arange(32, device=mask.device)).sum(1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


# ---------------------------------------------------------------- entry points
def _gemv(x, cb, scb, mask=None, tiled=True):
    L = _L()
    lib = L.lib()
    M, K = x.shape
    N = cb.shape[0]
    y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16)
    mw = None if mask is None else _mask_words(mask)
    if tiled:
        wt = torch.empty(lib.b2l_q8_tiled_bytes(N, K), dtype=torch.uint8, device=x.device)
        L.check(lib.b2l_q8_tile(cb.data_ptr(), wt.data_ptr(), N, K, L.stream_ptr()), "b2l_q8_tile")
    for m in range(M):
        xm = x[m].contiguous()
        if tiled:
            L.check(lib.b2l_q8_gemv(xm.data_ptr(), wt.data_ptr(), cb.data_ptr(), scb.data_ptr(), None if mw is None else mw.data_ptr(),
                                    y[m].data_ptr(), N, K, THR, 0, L.stream_ptr()), "b2l_q8_gemv")
        else:
            L.check(lib.b2l_q8_gemv_cb(xm.data_ptr(), cb.data_ptr(), scb.data_ptr(), None, y[m].data_ptr(), N, K, THR, 0,
                                       L.stream_ptr()), "b2l_q8_gemv_cb")
    torch.cuda.synchronize()
    return y


def _gemm(x, cb, scb):
    L = _L()
    lib = L.lib()
    M, K = x.shape
    N = cb.shape[0]
    nb = lib.b2l_q8_gemm_workspace_bytes(M, K)
    work = torch.full((nb,), 0x55, dtype=torch.uint8, device=x.device)
    y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16)
    L.check(lib.b2l_q8_gemm(x.data_ptr(), K, cb.data_ptr(), scb.data_ptr(), work.data_ptr(), nb, y.data_ptr(), N, M, N, K, THR, 0,
                            L.stream_ptr()), "b2l_q8_gemm")
    torch.cuda.synchronize()
    return y


def _linear(x, w, w2=None, g=None, epi=None, res=None, aff=None):
    """b2l_q8_linear (M = 1) or b2l_q8_linear_batch (M = 2..16)."""
    L = _L()
    lib = L.lib()
    cb, scb = w
    M, K = x.shape
    N = cb.shape[0]
    epi = L.EPI_STORE if epi is None else epi
    y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16)
    a = L.Q8LinearArgs(x=x.data_ptr(), cb=cb.data_ptr(), scb=scb.data_ptr(), y=y.data_ptr(), N=N, K=K, threshold=THR,
                       prologue=L.PRO_RMSNORM if g is not None else L.PRO_NONE, norm_scale=None if g is None else g.data_ptr(),
                       eps=EPS, epilogue=epi, res=None if res is None else res.data_ptr(), flags=0)
    if w2 is not None:
        a.cb2, a.scb2 = w2[0].data_ptr(), w2[1].data_ptr()
    if aff is not None:
        a.out_affine = L.OutAffine(aff[0].data_ptr(), aff[1].data_ptr())
    if M == 1:
        L.check(lib.b2l_q8_linear(C.byref(a), L.stream_ptr()), "b2l_q8_linear")
    else:
        nb = lib.b2l_q8_linear_batch_workspace_bytes(K, M)
        ws = torch.full((nb,), 0x55, dtype=torch.uint8, device=x.device)
        L.check(lib.b2l_q8_linear_batch(C.byref(a), M, ws.data_ptr(), nb, L.stream_ptr()), "b2l_q8_linear_batch")
    torch.cuda.synchronize()
    return y


# ---------------------------------------------------------------- checks
def _report(y, A, what):
    ok = A.contains(y)
    if not bool(ok.all()):
        bad = torch.nonzero(~ok)
        m, o = bad[0].tolist()
        raise AssertionError(f"{what}: {bad.shape[0]} of {y.numel()} outputs outside their admissible set; first (row {m}, "
                             f"out {o}): got {float(y[m, o])}, set [{float(A.lo[m, o])}, {float(A.hi[m, o])}] nan={bool(A.nan[m, o])}, "
                             f"single-rounded {float(A.id[m, o])}")
    eq = (y.view(torch.int16) == A.id.view(torch.int16)) | (torch.isnan(y) & torch.isnan(A.id))
    share = float(eq.float().mean())
    _SHARES.append((what, share))
    assert share >= MIN_EQUAL, (what, share)
    return share


def _check_plain(y, x, cb, scb, what, mask=None):
    R = O.int8_linear_exact(x, cb, scb, THR, mask=mask)
    _report(y, R.out, what)
    return R


def _probe_weights(x, mask=None):
    """CB = 127 I per row block, SCB = 127 / SCA_m: y[m, m K + k] = CA[m, k] on inliers, |y| > 127 on outliers."""
    M, K = x.shape
    R = O.int8_linear_exact(x, torch.zeros(1, K, dtype=torch.int8, device=x.device), torch.ones(1, device=x.device), THR, mask=mask)
    cb = (127 * torch.eye(K, device=x.device)).to(torch.int8).repeat(M, 1)
    scb = (torch.tensor(127.0, device=x.device) / R.sca.clamp_min(2.0 ** -24)).repeat_interleave(K)
    return cb.contiguous(), scb.contiguous(), R


def _check_probe(y, R, what):
    M, K = R.ca.shape
    for m in range(M):
        ym = y[m, m * K:(m + 1) * K].float()
        inl = ~R.mask
        bad = torch.nonzero(inl & (ym != R.ca[m])).flatten()
        assert bad.numel() == 0, (f"{what}: row {m}, column {int(bad[0])}: y = {float(ym[bad[0]])}, CA = {float(R.ca[m, bad[0]])}, "
                                  f"SCA = {float(R.sca[m])}, {bad.numel()} columns wrong")
        # an outlier column of this row: |τ| = |x̂| 127 / SCA_m > 127 (a given mask may hold columns below SCA)
        big = R.mask & (R.xh[m].float().abs() > R.sca[m])
        bado = torch.nonzero(big & ~(ym.abs() > 127)).flatten()
        assert bado.numel() == 0, f"{what}: row {m}, outlier column {int(bado[0])}: y = {float(ym[bado[0]])} (mask wrong?)"


def _probe_rows(M, K, dev):
    g = _gen(M * 7 + K)
    x = torch.randn(M, K, generator=g) * 2
    x[0, 9] = 7.5
    x[M - 1, K - 3] = -6.0
    x[M // 2, 40] = 5.96875
    return x.bfloat16().to(dev)


ENTRIES = ["gemv", "gemv_mask", "gemv_cb", "gemm", "linear", "linear_batch"]


def _run_plain(entry, x, cb, scb, mask=None):
    if entry in ("gemv", "gemv_mask"):
        return _gemv(x, cb, scb, mask=mask)
    if entry == "gemv_cb":
        return _gemv(x, cb, scb, tiled=False)
    if entry == "gemm":
        return _gemm(x, cb, scb)
    return _linear(x, (cb, scb))


def _given_mask(x, K, seed):
    """gemv_mask: the derived mask plus three columns another row of the batch would have made outliers."""
    m = (x.float().half().float().abs() >= THR).any(0)
    extra = torch.randperm(K, generator=_gen(seed))[:3].to(x.device)
    m = m.clone()
    m[extra] = True
    return m


@pytest.mark.parametrize("entry", ENTRIES)
def test_identity_probe(dev, entry):
    M = 3 if entry in ("gemm", "linear_batch") else 1
    K = 256
    x = _probe_rows(M, K, dev)
    mask = _given_mask(x, K, 1) if entry == "gemv_mask" else None
    cb, scb, R = _probe_weights(x, mask)
    y = _run_plain(entry, x, cb, scb, mask)
    _check_probe(y, R, entry)
    _check_plain(y, x, cb, scb, entry, mask)


def _entry_M(entry, M):
    return 1 if entry in ("gemv", "gemv_mask", "gemv_cb", "linear") else M


def _case(entry, shape, fam, M, seed, dev):
    N, K = SHAPES[shape]
    M = _entry_M(entry, M)
    x, wf = _family(fam, M, K, N, dev, seed)
    cb, scb = _weight(N, K, dev)
    if wf is not None:
        cb, scb = wf(cb, scb)
    mask = _given_mask(x, K, seed) if entry == "gemv_mask" else None
    y = _run_plain(entry, x, cb, scb, mask)
    R = _check_plain(y, x, cb, scb, f"{entry} {shape} {fam} M={M}", mask)
    return x, y, R


# every entry point x every family at 7B attn.c_proj
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("entry,M", [("gemv", 1), ("gemv_mask", 1), ("gemv_cb", 1), ("gemm", 17), ("linear", 1), ("linear_batch", 9)])
def test_families(dev, entry, M, fam):
    if fam == "mixed" and _entry_M(entry, M) == 1:
        pytest.skip("a batch property")
    x, y, R = _case(entry, "7b_cproj", fam, M, seed=FAMILIES.index(fam) * 13 + ENTRIES.index(entry), dev=dev)
    if fam == "threshold":
        assert bool(R.mask[[5, x.shape[1] - 1]].all()) and not bool(R.mask[[17, x.shape[1] // 2]].any())
    if fam == "ties":
        assert bool((R.qs == 32).all())
        frac = (R.xh.float() * 32) - (R.xh.float() * 32).floor()
        assert float((frac == 0.5).float().mean()) > 0.99
    if fam == "fp16edge":
        assert bool(torch.isinf(y).any()) and bool(torch.isfinite(y).any())
    if fam == "tiny":
        assert bool(torch.isinf(R.xh).any()) and bool((R.xh.float().abs() == 65280).any())
        assert bool(torch.isnan(y).any())
    if fam == "bigscb":
        assert bool(torch.isinf(R.v).any())
    if fam == "saturated" and entry != "gemv_mask":   # (a given mask zeroes three columns of CA)
        assert float(R.t[0, 0]) == 127 * 127 * x.shape[1]
    if fam == "massive":
        y_abs = R.out.id.float().abs().double()
        assert float((R.tau.abs() > 0.5 * y_abs).double().mean()) > 0.5   # τ carries most of |y|


# every width through every entry point (families rotate), the 65B widths and K = 32768 on gemv_cb, gemm, linear_batch
_SWEEP = [(e, s, FAMILIES[(i + j) % len(FAMILIES)]) for i, s in enumerate(SHAPES) for j, e in enumerate(ENTRIES)]
_SWEEP = [(e, s, "randn" if f in ("mixed", "saturated") else f) for e, s, f in _SWEEP]
_SWEEP += [("gemv_cb", "k32768", "saturated"), ("gemm", "k32768", "saturated"), ("linear_batch", "k32768", "saturated"),
           ("gemv_cb", "65b_proj", "massive"), ("gemm", "65b_fc", "massive"), ("linear_batch", "65b_proj", "mixed")]


@pytest.mark.parametrize("entry,shape,fam", _SWEEP)
def test_shapes(dev, entry, shape, fam):
    _case(entry, shape, fam, M=5, seed=len(shape) + ENTRIES.index(entry), dev=dev)


@pytest.mark.parametrize("M", [2, 16, 17, 300, 2048])
@pytest.mark.parametrize("fam", ["randn", "mixed", "massive"])
def test_gemm_rows(dev, M, fam):
    _case("gemm", "7b_attn", fam, M=M, seed=M, dev=dev)


# ---------------------------------------------------------------- the fused step: RMSNorm prologue and epilogues
def _rms_candidates(x, g):
    """x̂ by the kernels' chain (rms_rinv on the exact sum of the bf16-rounded squares, then bf16(g bf16(x rinv))), with
    rinv itself and one bf16 ulp up and down: the kernels' fp32 sum runs in their own order."""
    K = x.shape[1]
    xf = x.float()
    ss = (xf * xf).bfloat16().double().sum(-1, keepdim=True).float()
    ms = (ss / K).bfloat16().float()
    t = (ms + torch.tensor(EPS, dtype=torch.float32, device=x.device)).bfloat16().float()
    rinv = (1.0 / torch.sqrt(t)).bfloat16()
    bits = rinv.view(torch.int16)
    return [g * (x * r) for r in (rinv, (bits + 1).view(torch.bfloat16), (bits - 1).view(torch.bfloat16))]


def _fused_inputs(fam, M, K, dev, seed, norm):
    if not norm:
        x, _ = _family(fam, M, K, 0, dev, seed)
        return x, None, [x]
    for attempt in range(20):   # a mask that no rinv candidate moves (no |x̂| within an ulp of 6)
        gen = _gen(seed + 1000 * attempt)
        x = torch.randn(M, K, generator=gen)
        g = torch.exp(torch.empty(K).uniform_(math.log(1e-2), math.log(1.0), generator=gen))
        if fam == "massive":
            chans = torch.randperm(K, generator=gen)[:2 + (seed + attempt) % 7]
            x[:, chans] = torch.pow(10.0, 2 + 2 * torch.rand(M, len(chans), generator=gen)) * torch.sign(torch.randn(len(chans), generator=gen))
            g[chans] = 0.3 + 0.7 * torch.rand(len(chans), generator=gen)
        else:
            g = g * 8
        x, g = x.bfloat16().to(dev), g.bfloat16().to(dev)
        cands = _rms_candidates(x, g)
        masks = [(c.float().half().float().abs() >= THR).any(0) for c in cands]
        if all(torch.equal(masks[0], m) for m in masks):
            return x, g, cands
    raise AssertionError("no input with a stable outlier mask")


def _interleave(N):
    """SWIGLU affine index of output o of cb (first) and of cb2 (second): 16 entries per 8 outputs."""
    o = torch.arange(N)
    return (o // 8) * 16 + o % 8, (o // 8) * 16 + 8 + o % 8


def _fused_adm(xh, w, w2, epi, res, aff, mask):
    L = _L()
    A = O.int8_linear_exact(xh, w[0], w[1], THR, mask=mask)
    adm, taus = A.out, [A]
    N = w[0].shape[0]
    if epi == L.EPI_SWIGLU:
        B = O.int8_linear_exact(xh, w2[0], w2[1], THR, mask=mask)
        a2 = B.out
        if aff is not None:
            i1, i2 = (i.to(xh.device) for i in _interleave(N))
            adm = O.int8_adm_affine(adm, aff[0][i1], aff[1][i1])
            a2 = O.int8_adm_affine(a2, aff[0][i2], aff[1][i2])
        return O.int8_adm_silu_mul(adm, a2), A
    if aff is not None:
        adm = O.int8_adm_affine(adm, aff[0], aff[1])
    if epi == L.EPI_RESIDUAL:
        adm = O.int8_adm_residual(adm, res)
    return adm, A


def _fused_case(dev, M, shape, fam, norm, epi_name, affine, seed):
    L = _L()
    epi = {"store": L.EPI_STORE, "residual": L.EPI_RESIDUAL, "swiglu": L.EPI_SWIGLU}[epi_name]
    N, K = SHAPES[shape]
    x, g, cands = _fused_inputs(fam, M, K, dev, seed, norm)
    w = _weight(N, K, dev)
    w2 = _weight(N, K, dev, salt=1) if epi == L.EPI_SWIGLU else None
    gen = torch.Generator(device=dev).manual_seed(seed)
    res = (torch.randn(M, N, generator=gen, device=dev) * 2).bfloat16() if epi == L.EPI_RESIDUAL else None
    aff = None
    if affine:
        n_aff = 16 * ((N + 7) // 8) if epi == L.EPI_SWIGLU else N
        s = (torch.rand(n_aff, generator=gen, device=dev) + 0.5) * torch.sign(torch.randn(n_aff, generator=gen, device=dev))
        aff = (s.bfloat16(), (torch.randn(n_aff, generator=gen, device=dev) * 0.1).bfloat16())
    y = _linear(x, w, w2, g, epi, res, aff)
    mask = (cands[0].float().half().float().abs() >= THR).any(0)
    adms = [_fused_adm(c, w, w2, epi, res, aff, mask) for c in cands]
    what = f"linear M={M} {shape} {fam} norm={norm} {epi_name} affine={affine}"
    eq = 0
    for m in range(M):   # each row fits one rinv candidate as a whole
        for adm, _ in adms:
            if _row_ok(adm, y, m):
                eq += int(((y[m].view(torch.int16) == adm.id[m].view(torch.int16)) | (torch.isnan(y[m]) & torch.isnan(adm.id[m]))).sum())
                break
        else:
            _report(y[m:m + 1], _row(adms[0][0], m), f"{what} row {m}")
    _SHARES.append((what, eq / y.numel()))
    assert eq / y.numel() >= MIN_EQUAL, (what, eq / y.numel())
    return adms[0][1], y


def _row(adm, m):
    return O.Adm(id=adm.id[m:m + 1], lo=adm.lo[m:m + 1], hi=adm.hi[m:m + 1], nan=adm.nan[m:m + 1])


def _row_ok(adm, y, m):
    return bool(_row(adm, m).contains(y[m:m + 1]).all())


_FUSED = [(norm, epi, aff) for norm in (False, True) for epi in ("store", "residual", "swiglu") for aff in (False, True)]
_EPI_SHAPE = {"store": "7b_attn", "residual": "7b_proj", "swiglu": "7b_fc"}


@pytest.mark.parametrize("norm,epi,affine", _FUSED)
@pytest.mark.parametrize("M", [1, 2, 9, 16])
def test_fused_step(dev, M, norm, epi, affine):
    fam = "massive" if norm or epi == "residual" else "randn"
    A, y = _fused_case(dev, M, _EPI_SHAPE[epi], fam, norm, epi, affine, seed=M * 100 + len(epi) + 2 * norm + affine)
    if fam == "massive" and norm:
        y_abs = A.out.id.float().abs().double()
        assert float((A.tau.abs() > 0.5 * y_abs).double().mean()) > 0.5   # τ carries most of |y|


@pytest.mark.parametrize("shape", ["13b_fc", "13b_proj", "30b_fc", "30b_proj", "65b_fc", "65b_proj", "lm_head", "k32768", "ragged"])
@pytest.mark.parametrize("M", [1, 16])
def test_fused_step_widths(dev, M, shape):
    epi = "residual" if shape.endswith("proj") else "store"
    _fused_case(dev, M, shape, "massive", True, epi, False, seed=M + len(shape))

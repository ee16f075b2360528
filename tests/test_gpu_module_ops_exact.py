"""-m gpu: the kernels of the module path against exact arithmetic.

The module path (every prefill, refill and no-cache window; llm.int8, dense and grouped / biased gptq decode; the TP
module path) runs the stand-alone kernels of csrc/elementwise.cu and csrc/q_generic.cu, and several fused kernels are
tested against them bit for bit.  Each is compared here with a restatement that never calls the library: torch in
float64 on the device, or the reference's own bf16 formula run by torch on the same device.

Bars, derived from the arithmetic (u = 2^-24, fp32's unit roundoff; gamma_n = n u / (1 - n u)):

* b2l_rmsnorm keeps model.py:270-277's rounding points: bf16 squares, an fp32 sum, ms = bf16(ss / C),
  t = bf16(ms + eps), rinv = bf16(1 / sqrt(t)), y = bf16(g bf16(x rinv)).  Only the fp32 sum's order is the
  kernel's own: it moves ss by at most gamma_C ss (< 2^-11 ss at C = 8192), which can move the bf16 ms, and through it
  rinv, by one bf16 ulp, and nothing else.  So a row equals the restatement bit for bit over the whole row with rinv
  or with rinv one bf16 ulp up or down.  The restatement sums in float64 (error below 2^-40 of ss) and holds the sum
  in fp32 as the kernel does: a row at 2^60 whose squares sum beyond fp32's range gives rinv = 0 in every summation
  order (the smallest partial sum that completes it already overflows), and so does torch's fp32-accumulating mean.
* b2l_silu_mul and b2l_add are model.py:252 and :166-167: one fp32 operation chain per element (silu through expf
  and an IEEE division) with the reference's bf16 rounding points.  torch evaluates the same chain in fp32 on the
  device, so the results are equal bit for bit.  Against float64 the chain carries a few fp32 roundings (expf is
  within 2 ulp, the add and the division within half an ulp each) before each bf16 rounding, so a bf16 result may
  take the other neighbour only where the exact value lies within 8 fp32 ulps of the midpoint between two bf16
  neighbours; everywhere else it is the correctly rounded value.  exp is evaluated in fp32, as the reference does:
  beyond 88.72 it is inf and silu(a) = -0.
* b2l_q_dequant is get_weight (quantization.py:392-411) evaluated in the output dtype: oracle.llama_oracle.dequant
  bit for bit.
* b2l_q_linear forms each w = (level - zero) scale in fp32 (two roundings, the same as qlinear_exact's fp32 dequant,
  so w is exact there), accumulates x w by fp32 FMA in a fixed order (at most ceil(K / epb / 8) epb FMAs per warp,
  7 warp adds and one bias add: n <= K + 9 roundings on any path) and rounds once to bf16.  Per element
  |y - e| <= 2^-8 (|e| + gamma_n m) + gamma_n m, with e the float64 result and m = sum |x w| + |bias| (half a bf16 ulp
  of the fp32 value is at most 2^-8 of it); normwise under 2^-9 (the bf16 rounding of values with spread significands
  has an RMS relative error near 2^-9.3, the fp32 error is far smaller); and the fp32 error is far below a bf16 ulp,
  so at least 98 % of the outputs equal bf16(e).  Each row's FMA sequence does not depend on how many rows share the launch:
  row m of an M-row call equals the one-row call on x[m] bit for bit.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS = 1e-5


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _nan_buffer(n, dev, offset=0, guard=16):
    """A NaN-filled bf16 buffer of offset + n + guard elements and its [offset, offset + n) view: an element the kernel
    never writes stays NaN, and so does every guard element."""
    buf = torch.full((offset + n + guard,), float("nan"), device=dev, dtype=torch.bfloat16)
    return buf, buf[offset:offset + n]


def _guards_untouched(buf, offset, n):
    assert bool(buf[:offset].isnan().all()) and bool(buf[offset + n:].isnan().all()), "a write outside the output"


def _gamma(n):
    return n * U / (1 - n * U)


def _massive_rows(M, K, dev, seed):
    """Student-t (5 dof) bulk with 1..3 massive channels per row at 10^2.5..10^4 and either sign, as LLaMA's hidden
    states carry them."""
    gen = _gen(dev, seed)
    x = torch.randn(M, K, generator=gen, device=dev) / torch.sqrt((torch.randn(5, M, K, generator=gen, device=dev) ** 2).mean(0))
    chans = torch.randint(0, K, (M, 3), generator=gen, device=dev)
    mags = torch.pow(10.0, 2.5 + 1.5 * torch.rand(M, 3, generator=gen, device=dev))
    mags = torch.where(torch.rand(M, 3, generator=gen, device=dev) < 0.5, mags, -mags)
    use = torch.arange(3, device=dev)[None, :] < (1 + torch.arange(M, device=dev) % 3)[:, None]
    rows = torch.arange(M, device=dev)[:, None].expand(M, 3)
    x[rows[use], chans[use]] = mags[use]
    return x.bfloat16()


def _log_uniform(n, dev, seed, lo=0.02, hi=2.5):
    gen = _gen(dev, seed)
    return torch.exp(torch.empty(n, device=dev).uniform_(math.log(lo), math.log(hi), generator=gen)).bfloat16()


# ================================================================ 1. b2l_rmsnorm
def _rmsnorm(x, g, y, rows, C_, eps=EPS):
    L = _L()
    L.check(L.lib().b2l_rmsnorm(x.data_ptr(), g.data_ptr(), y.data_ptr(), rows, C_, eps, L.stream_ptr()), "b2l_rmsnorm")
    torch.cuda.synchronize()


def _rms_candidates(x, g, eps=EPS):
    """The restatement with the row's rinv, one bf16 ulp up and one down (module docstring)."""
    C_ = x.shape[-1]
    xf = x.float()
    ss = (xf * xf).bfloat16().double().sum(-1, keepdim=True).float()
    ms = (ss / C_).bfloat16().float()
    t = (ms + torch.tensor(eps, dtype=torch.float32, device=x.device)).bfloat16().float()
    rinv = (1.0 / torch.sqrt(t)).bfloat16()
    bits = rinv.view(torch.int16)
    return [g * (x * r) for r in (rinv, (bits + 1).view(torch.bfloat16), (bits - 1).view(torch.bfloat16))]


RMS_WIDTHS = [(128, "aligned"), (4096, "aligned"), (5120, "aligned"), (6656, "aligned"), (8192, "aligned"),
              # the scalar path: a width that is not a multiple of 8, and each pointer off 16-byte alignment
              (4100, "aligned"), (4096, "x+1"), (4096, "y+1"), (4096, "g+1")]
RMS_FAMILIES = ["randn", "massive", "tiny", "huge", "special"]


def _rms_input(family, rows, C_, dev, seed):
    gen = _gen(dev, seed)
    if family == "massive":
        return _massive_rows(rows, C_, dev, seed)
    x = torch.randn(rows, C_, generator=gen, device=dev)
    if family == "tiny":
        x = x * 2.0 ** -60
    elif family == "huge":
        x = x * 2.0 ** 60
    elif family == "special":   # cycling: an all-zero row, a constant row, a randn row
        x[0::3] = 0
        x[1::3] = torch.linspace(-3.0, 3.0, len(range(1, rows, 3)), device=dev)[:, None]
    return x.bfloat16()


@pytest.mark.parametrize("family", RMS_FAMILIES)
@pytest.mark.parametrize("rows", [1, 7, 4096])
@pytest.mark.parametrize("C_,layout", RMS_WIDTHS)
def test_rmsnorm_rows_equal_restatement(dev, C_, layout, rows, family):
    """Every row bit for bit against the restatement with one of its three rinv candidates; at least 99.5 % of the
    elements bit-equal to model.py's formula evaluated by torch in bf16 on this device; an all-zero row is exactly 0."""
    seed = C_ * 7 + rows + RMS_FAMILIES.index(family) * 100003
    x = _rms_input(family, rows, C_, dev, seed)
    g = _log_uniform(C_, dev, seed + 1)
    n = rows * C_
    xo, yo, go = (1 if layout == s else 0 for s in ("x+1", "y+1", "g+1"))
    xbuf = torch.empty(n + xo, device=dev, dtype=torch.bfloat16)
    xbuf[xo:] = x.reshape(-1)
    gbuf = torch.empty(C_ + go, device=dev, dtype=torch.bfloat16)
    gbuf[go:] = g
    ybuf, y = _nan_buffer(n, dev, yo)
    _rmsnorm(xbuf[xo:], gbuf[go:], y, rows, C_)
    _guards_untouched(ybuf, yo, n)
    y = y.view(rows, C_)
    assert not bool(y.isnan().any())
    ok = torch.zeros(rows, dtype=torch.bool, device=dev)
    for cand in _rms_candidates(x, g):
        ok |= (y == cand).all(-1)
    assert bool(ok.all()), f"rows off the restatement: {(~ok).nonzero().flatten().tolist()[:8]}"
    ref = g * (x * torch.rsqrt(torch.mean(x * x, -1, keepdim=True) + EPS))
    assert float((y == ref).float().mean()) >= 0.995
    if family == "special":
        assert bool((y[0::3] == 0).all())
    if family == "tiny":   # eps dominates: rinv = bf16(1 / sqrt(bf16(eps))), y about 316 x g
        assert bool((y.float().abs() < 2.0 ** -40).all()) and bool((y != 0).any())


@pytest.mark.parametrize("C_,layout", [(4096, "aligned"), (4100, "aligned")])
@pytest.mark.parametrize("family", ["randn", "massive"])
def test_rmsnorm_row_permutation_and_power_of_two_weights(dev, C_, layout, family):
    """Permuting the rows permutes the output bit for bit (no state is shared across rows), and y(2^e g) == 2^e y(g):
    every rounding is relative to a power-of-two exponent and g enters only the last product."""
    rows = 33
    x = _rms_input(family, rows, C_, dev, C_ + rows)
    g = _log_uniform(C_, dev, C_ + 5)
    y0 = torch.empty_like(x)
    _rmsnorm(x, g, y0, rows, C_)
    perm = torch.randperm(rows, generator=_gen(dev, 3), device=dev)
    xp = x[perm].contiguous()
    yp = torch.empty_like(x)
    _rmsnorm(xp, g, yp, rows, C_)
    assert torch.equal(yp, y0[perm])
    nz = y0.float().abs()[y0 != 0]
    for e in (-24, -3, 5, 24):
        assert float(nz.min()) * 2.0 ** e >= 2.0 ** -126 and float(nz.max()) * 2.0 ** e < 2.0 ** 127
        assert float(g.float().min()) * 2.0 ** e >= 2.0 ** -126
        ys = torch.empty_like(x)
        _rmsnorm(x, (g.float() * 2.0 ** e).bfloat16(), ys, rows, C_)
        assert torch.equal(ys, (y0.float() * 2.0 ** e).bfloat16()), e


# ================================================================ 2. b2l_silu_mul, b2l_add
def _binary(op, a, b, y, n):
    L = _L()
    fn = L.lib().b2l_silu_mul if op == "silu_mul" else L.lib().b2l_add
    L.check(fn(a.data_ptr(), b.data_ptr(), y.data_ptr(), n, L.stream_ptr()), "b2l_" + op)
    torch.cuda.synchronize()


def _bf16_neighbours(v):
    """float64 v -> (its bf16 rounding through fp32, whether v lies within 8 fp32 ulps of the midpoint between two bf16
    neighbours, the neighbour below and the one above in magnitude)."""
    v32 = v.float()
    bits = v32.view(torch.int32)
    near = ((bits & 0xFFFF) - 0x8000).abs() <= 8
    trunc = bits & -65536
    lo = trunc.view(torch.float32).bfloat16()
    hi = (trunc + 65536).view(torch.float32).bfloat16()
    return v32.bfloat16(), near, lo, hi


def _same(y, c):
    return (y == c) | (y.isnan() & c.isnan())


def _restated_ok(op, a, b, y):
    """Elementwise: y is the float64 restatement's bf16 result, or (near a bf16 midpoint) its other neighbour."""
    a64, b64 = a.double(), b.double()
    if op == "add":
        rn, near, lo, hi = _bf16_neighbours(a64 + b64)
        return _same(y, rn) | (near & (_same(y, lo) | _same(y, hi)))
    e = torch.exp(-a64).float().double()   # exp in fp32, as the reference evaluates it: inf beyond 88.72
    rn, near, lo, hi = _bf16_neighbours(a64 / (1.0 + e))
    bf = b.float()
    ok = _same(y, (rn.float() * bf).bfloat16())
    return ok | (near & (_same(y, (lo.float() * bf).bfloat16()) | _same(y, (hi.float() * bf).bfloat16())))


def _torch_ref(op, a, b):
    return F.silu(a) * b if op == "silu_mul" else a + b


def _binary_values(family, n, dev, seed):
    gen = _gen(dev, seed)
    a = torch.randn(n, generator=gen, device=dev)
    b = torch.randn(n, generator=gen, device=dev)
    if family in ("tiny", "huge"):
        s = 2.0 ** (-100 if family == "tiny" else 100)
        a, b = a * s, b * s
    elif family == "specials":   # every pair of +-0, +-inf, NaN, +-1, +-bf16 max and the smallest bf16 subnormal
        sp = torch.tensor([0.0, -0.0, math.inf, -math.inf, math.nan, 1.0, -1.0, 3.3895313892515355e38, -3.3895313892515355e38,
                           2.0 ** -133, -(2.0 ** -133)], device=dev)
        k = sp.numel()
        pa, pb = sp.repeat_interleave(k), sp.repeat(k)
        reps = -(-n // (k * k))
        a, b = pa.repeat(reps)[:n].clone(), pb.repeat(reps)[:n].clone()
        a[k * k:] = torch.randn(max(0, n - k * k), generator=gen, device=dev)
    elif family == "exp_overflow":   # a in [-100, -80]: exp(-a) overflows fp32 below -88.72
        a = -80.0 - 20.0 * torch.rand(n, generator=gen, device=dev)
    elif family == "subnormal":   # bf16 subnormals (|v| < 2^-126) against each other and against normals
        mant = torch.randint(1, 128, (n,), generator=gen, device=dev).float()
        a = mant * 2.0 ** -133 * torch.where(torch.rand(n, generator=gen, device=dev) < 0.5, 1.0, -1.0)
        b = torch.where(torch.arange(n, device=dev) % 2 == 0, b, -a.flip(0) * 3)
    return a.bfloat16(), b.bfloat16()


def _check_binary(op, a, b, y):
    want = _torch_ref(op, a, b)
    same = _same(y, want)
    assert bool(same.all()), f"{int((~same).sum())} elements differ from torch, first at {int((~same).nonzero()[0])}"
    ok = _restated_ok(op, a, b, y)
    assert bool(ok.all()), f"{int((~ok).sum())} elements off the float64 restatement, first at {int((~ok).nonzero()[0])}"


BIN_NS = [1, 7, 8, 9, 4096, 4097, 11008, 11015, 16 * 11008, 2048 * 13824]   # n % 8 in {0, 1, 7} on the vector path
LAYOUTS = ["aligned", "a+1", "b+1", "y+1"]                                   # one pointer off: the scalar path


def _run_binary(op, a, b, layout, dev):
    """y = op(a, b) with a, b or y moved one element off 16-byte alignment per `layout`, y NaN-prefilled."""
    n = a.numel()
    offs = {k: 1 if layout == k + "+1" else 0 for k in ("a", "b", "y")}
    ins = []
    for name, t in (("a", a), ("b", b)):
        buf = torch.empty(n + offs[name], device=dev, dtype=torch.bfloat16)
        buf[offs[name]:] = t
        ins.append(buf[offs[name]:])
    ybuf, y = _nan_buffer(n, dev, offs["y"])
    _binary(op, ins[0], ins[1], y, n)
    _guards_untouched(ybuf, offs["y"], n)
    return y


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("n", BIN_NS)
@pytest.mark.parametrize("op", ["silu_mul", "add"])
def test_binary_paths(dev, op, n, layout):
    a, b = _binary_values("randn", n, dev, n + LAYOUTS.index(layout))
    y = _run_binary(op, a, b, layout, dev)
    assert not bool(y.isnan().any())
    _check_binary(op, a, b, y)


@pytest.mark.parametrize("family", ["tiny", "huge", "specials", "exp_overflow", "subnormal"])
@pytest.mark.parametrize("layout", ["aligned", "a+1"])
@pytest.mark.parametrize("n", [9, 11015, 16 * 11008 + 1])
@pytest.mark.parametrize("op", ["silu_mul", "add"])
def test_binary_values(dev, op, n, layout, family):
    a, b = _binary_values(family, n, dev, 7 * n + len(family))
    _check_binary(op, a, b, _run_binary(op, a, b, layout, dev))


@pytest.mark.parametrize("n", [9, 4097, 16 * 11008 + 7])
@pytest.mark.parametrize("alias", ["a", "b"])
@pytest.mark.parametrize("op", ["silu_mul", "add"])
def test_binary_in_place(dev, op, alias, n):
    """y = a and y = b (MLP.forward and the residual add may write over an input): the out-of-place result bit for bit."""
    a, b = _binary_values("randn", n, dev, n)
    want = torch.empty_like(a)
    _binary(op, a, b, want, n)
    a2, b2 = a.clone(), b.clone()
    y = a2 if alias == "a" else b2
    _binary(op, a2, b2, y, n)
    assert torch.equal(y, want)
    _check_binary(op, a, b, y)


# ================================================================ 3. b2l_embedding
def _embedding(idx, wte, out, n, C_, V):
    L = _L()
    rc = L.lib().b2l_embedding(idx.data_ptr(), 1 if idx.dtype == torch.int64 else 0, wte.data_ptr(), out.data_ptr(), n, C_, V,
                               L.stream_ptr())
    L.check(rc, "b2l_embedding")
    torch.cuda.synchronize()


V_EMB = 32000


@pytest.mark.parametrize("n", [1, 7, 4096])
@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("C_", [4096, 8192, 4100])
def test_embedding_rows(dev, C_, idx_dtype, n):
    gen = _gen(dev, C_ + n)
    wte = torch.randn(V_EMB, C_, generator=gen, device=dev).bfloat16()
    idx = torch.randint(0, V_EMB, (n,), generator=gen, device=dev)
    idx[0] = V_EMB - 1
    if n > 1:
        idx[-1] = 0
    idx = idx.to(idx_dtype)
    obuf, out = _nan_buffer(n * C_, dev)
    _embedding(idx, wte, out, n, C_, V_EMB)
    _guards_untouched(obuf, 0, n * C_)
    assert torch.equal(out.view(n, C_), wte[idx.long()])


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
def test_embedding_out_of_range_ids_read_row_0(dev, idx_dtype):
    """elementwise.cu documents it: an id outside [0, V) reads row 0 (torch would raise), so the kernel stays in
    bounds."""
    C_, V = 4096, 1000
    wte = torch.randn(V, C_, generator=_gen(dev, 1), device=dev).bfloat16()
    bad = [-1, V, V + 1, -(2 ** 31), 2 ** 31 - 1] + ([2 ** 40, -(2 ** 40), 2 ** 32] if idx_dtype == torch.int64 else [])
    ids = [5, V - 1] + bad + [0, 17]
    idx = torch.tensor(ids, dtype=idx_dtype, device=dev)
    out = torch.full((len(ids), C_), float("nan"), device=dev, dtype=torch.bfloat16)
    _embedding(idx, wte, out, len(ids), C_, V)
    want = wte[torch.tensor([i if 0 <= i < V else 0 for i in ids], device=dev)]
    assert torch.equal(out, want)


# ================================================================ 4. b2l_q_dequant, b2l_q_linear
def _pack(lv, bits):
    """levels (N, K) -> quant_weight (N, K / epb) in the reference layout, strides (1, N)."""
    epb = 8 // bits
    qw = torch.zeros((lv.shape[0], lv.shape[1] // epb), dtype=torch.uint8, device=lv.device)
    for nr in range(epb):
        qw |= lv[:, nr::epb] << (nr * bits)
    return qw.t().contiguous().t()


def _qweights(dev, N, K, bits, tile_cols, sz_dtype, seed):
    """Random levels, positive scales, and zeros that are integral (as GPTQ writes them) on even rows and fractional
    on odd rows: uniform in [0, 2^bits) in fp32, below 1 in bf16."""
    gen = _gen(dev, seed)
    tc = K if tile_cols == -1 else tile_cols
    ng = -(-K // tc)
    lv = torch.randint(0, 2 ** bits, (N, K), generator=gen, device=dev, dtype=torch.uint8)
    sc = (torch.rand(N, ng, generator=gen, device=dev) * 0.01 + 0.002).to(sz_dtype)
    zi = torch.randint(0, 2 ** bits, (N, ng), generator=gen, device=dev).float()
    zf = torch.rand(N, ng, generator=gen, device=dev) * (2.0 ** bits if sz_dtype == torch.float32 else 1.0)
    z = torch.where((torch.arange(N, device=dev) % 2 == 0)[:, None], zi, zf).to(sz_dtype)
    return lv, _pack(lv, bits), sc, z, tc


def _dequant(qw, sc, z, N, K, bits, tile_cols, out_dtype):
    L = _L()
    w = torch.full((N, K), float("nan"), device=qw.device, dtype=out_dtype)
    rc = L.lib().b2l_q_dequant(qw.data_ptr(), sc.data_ptr(), z.data_ptr(), L.sz_dtype_of(sc), w.data_ptr(),
                               L.B2L_BF16 if out_dtype == torch.bfloat16 else L.B2L_F32, N, K, bits, tile_cols, L.stream_ptr())
    L.check(rc, "b2l_q_dequant")
    return w


DQ_SHAPES = [(12288, 4096), (4096, 11008), (32000, 4096), (130, 200)]   # (out, in); 130 x 200: K/2 = 100, N not % 32


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("sz_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("tile_cols", [32, 128, -1, 96])   # -1: K (one group); 96 divides none of the K
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K", DQ_SHAPES)
def test_dequant_bit_exact(dev, N, K, bits, tile_cols, sz_dtype, out_dtype):
    lv, qw, sc, z, tc = _qweights(dev, N, K, bits, tile_cols, sz_dtype, seed=N + K + bits + tile_cols)
    if tile_cols == 96:
        assert K % tc != 0
    # get_weight's first rounding bf16(level - zero) is exercised: some differences are not bf16 numbers
    d = lv[:, :: tc].float() - z.float()
    assert bool((d.bfloat16().float() != d).any())
    w = _dequant(qw, sc, z, N, K, bits, tile_cols, out_dtype)
    with torch.device(dev):
        want = O.dequant(qw, sc, z, bits, tc, out_dtype)
    assert torch.equal(w, want)


def _q_linear(x, qw, sc, z, bias, N, K, bits, tile_cols, *, ldx=None, y=None, ldy=None):
    L = _L()
    M = x.shape[0]
    ldx = x.stride(0) if ldx is None else ldx
    if y is None:
        y = torch.full((M, N), float("nan"), device=x.device, dtype=torch.bfloat16)
        ldy = N
    rc = L.lib().b2l_q_linear(x.data_ptr(), ldx, qw.data_ptr(), sc.data_ptr(), z.data_ptr(), L.sz_dtype_of(sc),
                              None if bias is None else bias.data_ptr(), y.data_ptr(), ldy, M, N, K, bits, tile_cols,
                              L.stream_ptr())
    L.check(rc, "b2l_q_linear")
    torch.cuda.synchronize()
    return y


def _assert_linear_exact(y, x, qw, sc, z, bits, tc, bias=None):
    """The per-element, normwise and bit-equal-share bars of the module docstring."""
    K = x.shape[1]
    epb = 8 // bits
    n = -(-(K // epb) // 8) * epb + 9
    with torch.device(x.device):
        w = O.dequant(qw, sc.float(), z.float(), bits, tc, torch.float32).double()
        exact32 = O.qlinear_exact(x, qw, sc, z, bits, tc, bias)
    e = x.double() @ w.t()
    m = x.double().abs() @ w.abs().t()
    if bias is not None:
        e, m = e + bias.double(), m + bias.double().abs()
    g = _gamma(n)
    err = (y.double() - e).abs()
    bound = 2.0 ** -8 * (e.abs() + g * m) + g * m + 2.0 ** -133
    assert bool((err <= bound).all()), float((err / bound).max())
    assert float((y.double() - e).norm() / e.norm()) < 2.0 ** -9
    assert float((y == exact32.bfloat16()).float().mean()) >= 0.98


# name -> (N, K, bits, tile_cols, scale / zero dtype, bias, ldx pad, ldy pad)
QL_CASES = {
    "q4_row": (4096, 4096, 4, -1, torch.bfloat16, False, 0, 0),
    "q4_g128_bias_vec1": (4098, 4096, 4, 128, torch.bfloat16, True, 0, 0),
    "q8_g96_f32_bias": (4096, 11008, 8, 96, torch.float32, True, 0, 0),
    "q8_row_f32_vec1_ld": (4098, 4096, 8, -1, torch.float32, False, 8, 5),
    "q4_g32_f32_ld": (12288, 4096, 4, 32, torch.float32, False, 24, 3),
}
QL_MS = [1, 2, 3, 4, 5, 8, 17, 300]   # MT = 1, 2, 4; several m0 passes, 5 and 17 with a partial last one


@pytest.mark.parametrize("family", ["randn", "massive"])
@pytest.mark.parametrize("M", QL_MS)
@pytest.mark.parametrize("case", list(QL_CASES))
def test_q_linear_vs_exact(dev, case, M, family):
    N, K, bits, tile_cols, sz_dtype, has_bias, xpad, ypad = QL_CASES[case]
    seed = N + K + bits + tile_cols
    lv, qw, sc, z, tc = _qweights(dev, N, K, bits, tile_cols, sz_dtype, seed)
    gen = _gen(dev, seed + M)
    bias = (torch.randn(N, generator=gen, device=dev) * 0.5).bfloat16() if has_bias else None
    xs = _massive_rows(M, K, dev, seed + M) if family == "massive" else torch.randn(M, K, generator=gen, device=dev).bfloat16()
    xbuf = torch.zeros(M, K + xpad, device=dev, dtype=torch.bfloat16)
    xbuf[:, :K] = xs
    x = xbuf[:, :K]
    ybuf = torch.full((M, N + ypad), float("nan"), device=dev, dtype=torch.bfloat16)
    y = _q_linear(x, qw, sc, z, bias, N, K, bits, tile_cols, ldx=K + xpad, y=ybuf, ldy=N + ypad)
    assert bool(ybuf[:, N:].isnan().all())   # ldy > N: the padding is not written
    y = ybuf[:, :N]
    _assert_linear_exact(y, xs, qw, sc, z, bits, tc, bias)
    # the same call again, and each row alone: bit for bit
    again = _q_linear(x, qw, sc, z, bias, N, K, bits, tile_cols, ldx=K + xpad)
    assert torch.equal(again, y)
    if M > 1:
        for r in range(M):
            assert torch.equal(_q_linear(xs[r:r + 1], qw, sc, z, bias, N, K, bits, tile_cols), y[r:r + 1]), r


def _layer(dev, N, K, bits, tile_cols, bias, seed):
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    lv, qw, sc, z, tc = _qweights(dev, N, K, bits, tile_cols, torch.bfloat16, seed)
    lin = ColBlockQuantizedLinear(K, N, bias, bits=bits, tile_cols=tile_cols).to(dev)
    lin.quant_weight.copy_(qw)
    lin.scales = sc.clone()
    lin.zeros = z.clone()
    if bias:
        lin.bias = (torch.randn(N, generator=_gen(dev, seed + 1), device=dev) * 0.5).bfloat16()
    return lin, qw, sc, z


@pytest.mark.parametrize("kind,M", [(k, M) for k in ("grouped", "bias", "offset_input") for M in (1, 5, 17, 300)] + [("k96", 17)])
def test_forward_routes_to_q_linear(dev, kind, M):
    """ColBlockQuantizedLinear.forward on the layers kernel_at sends to the generic kernel (grouped; biased; an input
    view 2 bytes off 16-byte alignment; 4 bits at K = 96, which only M > 16 sends there): a direct b2l_q_linear call
    bit for bit, and the bars of the module docstring."""
    N, K = (640, 96) if kind == "k96" else (1024, 4096)
    tile_cols = 128 if kind == "grouped" else -1
    lin, qw, sc, z = _layer(dev, N, K, 4, tile_cols, kind == "bias", seed=N + M)
    gen = _gen(dev, M)
    if kind == "offset_input":
        buf = torch.randn(M * K + 1, generator=gen, device=dev).bfloat16()
        x = buf[1:].view(M, K)
        assert x.data_ptr() % 16 == 2
    else:
        x = torch.randn(M, K, generator=gen, device=dev).bfloat16()
    aligned = x.data_ptr() % 16 == 0
    assert lin.kernel_at(M, aligned) == "q_linear"
    y = lin(x)
    torch.cuda.synchronize()
    assert torch.equal(y, _q_linear(x, qw, sc, z, lin.bias, N, K, 4, tile_cols))
    _assert_linear_exact(y, x, qw, sc, z, 4, K if tile_cols == -1 else tile_cols, lin.bias)


@pytest.mark.parametrize("M", [1, 5, 300])
@pytest.mark.parametrize("layout", ["reference", "row_major"])
def test_qlinear_4bit_weight_vs_exact(dev, M, layout):
    """The drop-in for the reference's Triton launcher: (N, K/2) weights in the reference layout, or row-major, which
    it re-lays out; per-row scales and zeros."""
    from lit_llama_b200.quantization import qlinear_4bit_weight

    N, K = 4096, 4096
    lv, qw, sc, z, tc = _qweights(dev, N, K, 4, -1, torch.bfloat16, seed=M)
    w = qw if layout == "reference" else qw.contiguous()
    assert (tuple(w.stride()) == (1, N)) == (layout == "reference")
    x = torch.randn(M, K, generator=_gen(dev, M + 1), device=dev).bfloat16()
    y = qlinear_4bit_weight(x, w, sc, z)
    torch.cuda.synchronize()
    _assert_linear_exact(y, x, qw, sc, z, 4, tc)


# ================================================================ 5. a grouped gptq.int4 model on the module path
CFG128 = dict(block_size=64, vocab_size=256, n_layer=2, n_head=4, n_embd=512)   # head_size 128
PROMPT = torch.tensor([5, 100, 3, 7, 200, 9, 31])
TOKS = [77, 12, 9, 150, 42]


def _run_model(model, dev, S, toks):
    T = PROMPT.numel()
    with torch.no_grad():
        out = [model(PROMPT.view(1, -1).to(dev), S, torch.arange(T, device=dev))]
        for i, t in enumerate(toks):
            out.append(model(torch.full((1, 1), t, device=dev), S, torch.tensor([T + i], device=dev)))
    torch.cuda.synchronize()
    return out


def _want(oracle, S, toks):
    T = PROMPT.numel()
    oracle.reset_cache()
    out = [oracle.forward(PROMPT.view(1, -1), S, torch.arange(T))]
    for i, t in enumerate(toks):
        out.append(oracle.forward(torch.full((1, 1), t), S, torch.tensor([T + i])))
    return out


def _close(got, want, bar=2e-2):
    for a, b in zip(got, want):
        a, b = a.float().cpu(), b.float().cpu()
        assert float((a - b).norm() / b.norm()) < bar


def test_grouped_gptq_int4_model_vs_oracle(dev):
    """tile_cols = 128 (4 groups per c_attn row, 12 per mlp.c_proj row): every linear runs b2l_q_linear, the decode
    step is the module-by-module sequence (eager, then replayed as a CUDA graph), against the oracle's exact-linear
    arithmetic at the bars of the head_size-128 LoRA model tests: prefill, decode, the roll branch, greedy tokens."""
    import lit_llama_b200 as P
    from gpu_util import build_tiny

    for graph_after in (0, 2):
        model, oracle, sd = build_tiny(dev, CFG128, "gptq.int4", seed=77, tile_cols=128, exact_linears=True)
        assert sd["transformer.h.0.attn.c_attn.scales"].shape == (3 * 512, 4)
        for blk in model.transformer.h:
            for lin in (blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_fc1, blk.mlp.c_fc2, blk.mlp.c_proj):
                assert lin.tile_cols == 128 and all(lin.kernel_at(M) == "q_linear" for M in (1, 7))
        model.graph_after = graph_after
        got = _run_model(model, dev, 32, TOKS)
        assert model._decode is None
        mg = model._module_graph
        assert (mg is not None and mg["graph"] is not None) == (graph_after > 0)
        _close(got, _want(oracle, 32, TOKS))
    model.reset_cache()
    roll_toks = [3, 17, 40, 41, 2, 77]    # positions 7..12 in an 8-slot cache
    roll = [t[:, -1] for t in _run_model(model, dev, 8, roll_toks)]
    _close(roll, [t[:, -1] for t in _want(oracle, 8, roll_toks)])
    model.reset_cache()
    oracle.reset_cache()
    greedy = P.generate(model, PROMPT.to(torch.int32).to(dev), 12, top_k=1).cpu()
    assert (greedy == O.generate(oracle, PROMPT.to(torch.int32), 12, top_k=1)).float().mean() >= 0.9

"""CPU checks of the exact LLM.int8() restatement (oracle.llama_oracle.int8_linear_exact) before any kernel is measured
against it in test_gpu_int8_exact.py:

1. an fp32 evaluation of the kernels' own chain (q8_common.cuh's order: fmaf products exact, so fmaf = mul + add) lands
   in the admissible set, on random inputs and on inputs built to sit within an fp32 ulp of an fp16 midpoint;
2. away from midpoints the set has one element, so the bar is not vacuous;
3. the constructions the GPU file relies on do what they claim;
4. the restatement equals int8_linear (the double-rounding oracle) except where that double rounding differs, and
   int8_linear itself lies in the admissible set."""
import pytest
import torch

from oracle import llama_oracle as O

THR = 6.0


def _kernel_chain(x, cb, scb, mask=None):
    """q8_gemv.cu / q8_gemm.cu / q8_gemv_batch.cu in fp32, step for step: (bf16 out, fp16 dequantised part)."""
    xh = x.float().half().float()
    mask = (xh.abs() >= THR).any(0) if mask is None else mask
    a_in = xh.masked_fill(mask, 0.0)
    sca = a_in.abs().amax(1)
    qs = torch.where(sca > 0, torch.tensor(127.0) / sca, torch.zeros_like(sca))
    ca = torch.round(a_in * qs.unsqueeze(1)).clamp(-127, 127).masked_fill(mask, 0.0)
    t = (ca.double() @ cb.double().t()).float()                      # (float)t
    c = torch.tensor(1.0) / torch.tensor(127.0 * 127.0)              # 1.0f / (127.0f * 127.0f)
    v = (t * ((sca.unsqueeze(1) * scb.unsqueeze(0)) * c)).half()     # q8_dequant
    if not bool(mask.any()):
        return v.float().bfloat16(), v
    wsc = scb / torch.tensor(127.0)
    w = (cb[:, mask].float() * wsc.unsqueeze(1)).half().float()      # q8_outlier_weight
    term = torch.zeros(x.shape[0], cb.shape[0])
    for j, k in enumerate(torch.nonzero(mask).flatten().tolist()):   # fmaf, k ascending
        term = term + xh[:, k:k + 1] * w[:, j].unsqueeze(0)
    return (v.float() + term.half().float()).half().float().bfloat16(), v   # q8_add_outliers; (out, v)


def _weights(N, K, g, lo=0.01, hi=0.21):
    cb = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8)
    scb = torch.rand(N, generator=g) * (hi - lo) + lo
    return cb, scb


def _rows(M, K, g, n_out=3):
    x = torch.randn(M, K, generator=g) * 1.5
    for i in range(n_out):
        x[i % M, (53 * i + 7) % K] = (6.5 + 3 * i) * (-1) ** i
    return x.bfloat16()


@pytest.mark.parametrize("M,N,K,n_out,floor", [(1, 300, 256, 0, 0.995), (4, 257, 512, 3, 0.995), (16, 130, 1024, 9, 0.995),
                                               (3, 500, 128, 40, 0.98)])
def test_kernel_chain_lands_in_set_random(M, N, K, n_out, floor):
    """floor: the share of one-element sets.  With 40 outlier columns about one output in fifty has an outlier weight
    within its bound of an fp16 midpoint, whose |x̂_k| ulp16(w_k) widens that output's set."""
    g = torch.Generator().manual_seed(M * 1000 + N + K)
    cb, scb = _weights(N, K, g)
    x = _rows(M, K, g, n_out)
    R = O.int8_linear_exact(x, cb, scb)
    y, yv = _kernel_chain(x, cb, scb)
    assert bool(R.out.contains(y).all())
    assert bool(R.out.contains(R.out.id).all())
    single = R.out.single()
    assert float(single.float().mean()) >= floor, float(single.float().mean())
    assert float((y.view(torch.int16) == R.out.id.view(torch.int16)).float().mean()) >= 0.995


def _midpoints_near(v):
    """An fp16 midpoint next to v (same sign): halfway between fp16(|v|) and the fp16 value above it."""
    h = O.round_to(v.double().abs(), torch.float16)
    up = (h.view(torch.int16) + 1).view(torch.float16)
    return torch.sign(v) * (h.double() + up.double()) / 2


def test_dequantised_part_at_fp16_midpoints():
    """SCA = 127/32 (qs = 32) and x on the 1/32 grid make every CA exact; SCB is then solved so that t SCA SCB / 127²
    sits within an fp32 ulp of an fp16 midpoint.  The kernel chain must land in the set, the set must have two
    elements there for most outputs, and the single-rounded value must be one of them."""
    g = torch.Generator().manual_seed(7)
    K, N = 256, 2000
    x = torch.randint(-126, 127, (1, K), generator=g).float() / 32
    x[0, 0] = 127 / 32
    cb, scb0 = _weights(N, K, g)
    R0 = O.int8_linear_exact(x, cb, scb0)
    assert float(R0.qs[0]) == 32.0 and bool((R0.ca == x * 32).all())
    t = R0.t[0]
    keep = t.abs() > 1000
    mid = _midpoints_near(t * float(R0.sca[0]) * scb0.double() / 16129.0)
    scb = (mid * 16129.0 / (t * float(R0.sca[0]))).float().abs()
    scb = torch.where(keep, scb, scb0)
    R = O.int8_linear_exact(x, cb, scb)
    y, yv = _kernel_chain(x, cb, scb)
    e = R.t[0] * float(R.sca[0]) * scb.double() / 16129.0
    assert bool(((e - mid).abs() <= mid.abs() * 2.0 ** -23)[keep].all())
    assert bool(R.out.contains(y).all())
    v16 = lambda t: t.view(torch.int16)
    assert bool(((v16(yv) == v16(R.v_lo)) | (v16(yv) == v16(R.v_hi))).all())
    two = (v16(R.v_lo) != v16(R.v_hi))[0]
    assert float(two[keep].float().mean()) > 0.9, float(two[keep].float().mean())
    assert bool(((v16(R.v) == v16(R.v_lo)) | (v16(R.v) == v16(R.v_hi))).all())


def test_outlier_weight_at_fp16_midpoints():
    """SCB solved so that CB SCB / 127 of the outlier column sits at an fp16 midpoint: w_k has two candidates, and the
    τ bound carries |x̂_k| ulp16(w_k) for them."""
    g = torch.Generator().manual_seed(8)
    K, N = 256, 1500
    x = (torch.randn(2, K, generator=g)).bfloat16()
    x[0, 17] = 40.0
    x[1, 17] = -24.0
    cb, _ = _weights(N, K, g)
    cb[:, 17] = torch.randint(1, 128, (N,), generator=g).to(torch.int8)
    w_target = torch.rand(N, generator=g).double() * 3 + 0.05
    mid = _midpoints_near(w_target)
    scb = (mid * 127.0 / cb[:, 17].double()).float()
    R = O.int8_linear_exact(x, cb, scb)
    y, yv = _kernel_chain(x, cb, scb)
    assert bool(R.out.contains(y).all())
    assert float((R.tau_bound > 40 * 2.0 ** -14).float().mean()) > 0.5


def test_constructions():
    """What the GPU file's input families claim of their values."""
    # rint ties: SCA = 127/32 gives qs = 32 exactly, (2j+1)/64 * 32 = j + 1/2 exactly, rounded to even
    sca = torch.tensor(127 / 32).bfloat16().half().float()
    assert float(sca) == 127 / 32
    qs = torch.tensor(127.0) / sca
    assert float(qs) == 32.0
    j = torch.arange(0, 126)
    v = ((2 * j + 1).float() / 64).bfloat16().half().float()
    assert bool((v == (2 * j + 1).float() / 64).all())
    p = v * qs
    assert bool((p == j.float() + 0.5).all())
    assert bool((torch.round(p) == 2 * torch.round(j.float() / 2 + 0.25)).all())   # even neighbour
    # threshold: 5.96875 is the largest bf16 below 6; 5.984375 is not a bf16 (it rounds to 6)
    assert float(torch.tensor(5.96875).bfloat16()) == 5.96875
    assert float(torch.nextafter(torch.tensor(5.96875), torch.tensor(7.0)).bfloat16()) in (5.96875, 6.0)
    assert float((torch.tensor(5.96875).bfloat16().view(torch.int16) + 1).view(torch.bfloat16)) == 6.0
    assert float(torch.tensor(5.984375).bfloat16()) == 6.0
    # fp16's range from bf16: 65280 is the largest bf16 that stays finite, 65536 the first that is inf
    assert float(torch.tensor(65280.0).bfloat16().half()) == 65280.0
    assert float((torch.tensor(65280.0).bfloat16().view(torch.int16) + 1).view(torch.bfloat16)) == 65536.0
    assert torch.isinf(torch.tensor(65536.0).bfloat16().half())
    # rows at 2^-16 .. 2^-24 become fp16 subnormals; at most 2^-25 in magnitude they become zero
    assert 0 < float(torch.tensor(2.0 ** -16).half()) < 2.0 ** -14
    assert float(torch.tensor(2.0 ** -25).half()) == 0.0 and float(torch.tensor(2.0 ** -24).half()) == 2.0 ** -24
    # the saturated contraction: 127² 32768 = 16129 2^15 is exact in fp32 (14 significant bits); one 126 in place of a
    # 127 gives 528514945, which is not
    t_max = 127 * 127 * 32768
    assert t_max == 528515072 and t_max < 2 ** 31
    assert int(torch.tensor(t_max, dtype=torch.float64).float()) == t_max
    assert int(torch.tensor(t_max - 127, dtype=torch.float64).float()) != t_max - 127


def test_round_to_is_single_rounding():
    """round_to rounds float64 once: at a value just above an fp16 midpoint that fp32 would round onto it, it rounds
    up, where .float().half() rounds to even (down)."""
    lo = torch.tensor(1.0, dtype=torch.float64)
    mid = lo + 2.0 ** -11                       # midpoint of 1 and 1 + 2^-10
    e = mid + 2.0 ** -40                        # fp32 rounds this to the midpoint
    assert float(e.float()) == float(mid)
    assert float(e.float().half()) == 1.0
    assert float(O.round_to(e, torch.float16)) == 1.0 + 2.0 ** -10
    assert float(O.round_to(mid, torch.float16)) == 1.0
    b = torch.tensor(1.0 + 2.0 ** -8 + 2.0 ** -40, dtype=torch.float64)   # just above a bf16 midpoint
    assert float(O.round_to(b, torch.bfloat16)) == 1.0 + 2.0 ** -7
    assert torch.isinf(O.round_to(torch.tensor(65520.0, dtype=torch.float64), torch.float16))
    assert float(O.round_to(torch.tensor(65519.99, dtype=torch.float64), torch.float16)) == 65504.0
    assert float(O.round_to(torch.tensor(3.0 * 2.0 ** -26, dtype=torch.float64), torch.float16)) == 2.0 ** -24


def test_special_values():
    """inf from fp16(x) and from a large SCB, NaN from inf · 0, and an all-zero row (SCA = 0)."""
    g = torch.Generator().manual_seed(9)
    K, N = 256, 64
    cb, scb = _weights(N, K, g)
    x = torch.randn(4, K, generator=g).bfloat16()
    x[0, 3] = 65536.0          # fp16 inf
    x[1, 5] = -65280.0
    x[2] = 0.0
    x[3] = ((torch.rand(K, generator=g) * 2 - 1) * 2.0 ** -26).bfloat16()   # below 2^-25: fp16 zero
    cb[::7, 3] = 0             # inf * 0
    scb[::5] = 5e4             # dequantised part beyond fp16
    R = O.int8_linear_exact(x, cb, scb)
    y, yv = _kernel_chain(x, cb, scb)
    assert bool(R.out.contains(y).all())
    assert float(R.sca[2]) == 0.0 and float(R.sca[3]) == 0.0
    assert bool(torch.isnan(R.out.id[0, ::7]).all()) and bool(torch.isinf(R.out.id).any())
    assert bool(torch.isfinite(R.out.id[2]).all())


def test_silu_mul_set():
    g = torch.Generator().manual_seed(10)
    y1 = (torch.randn(4000, generator=g) * 4).bfloat16()
    y1[:4] = torch.tensor([-100.0, -89.0, float("inf"), float("-inf")])
    y2 = (torch.randn(4000, generator=g) * 2).bfloat16()
    A = O.int8_adm_silu_mul(O.Adm.of(y1, [y1]), O.Adm.of(y2, [y2]))
    s = (y1.float() / (1.0 + torch.exp(-y1.float()))).bfloat16()     # silu_mul1 (b2l_common.cuh)
    got = (s.float() * y2.float()).bfloat16()
    assert bool(A.contains(got).all())
    assert bool(A.contains(A.id).all())
    assert bool(torch.isnan(got[3])) and bool(A.nan[3])              # silu(-inf) = -inf / inf
    assert float(A.single().float().mean()) > 0.99
    assert float((got.view(torch.int16) == A.id.view(torch.int16)).float().mean()) > 0.99


@pytest.mark.parametrize("M,N,K,n_out", [(1, 512, 512, 2), (8, 300, 1024, 6), (16, 257, 256, 20)])
def test_restatement_vs_double_rounding_oracle(M, N, K, n_out):
    g = torch.Generator().manual_seed(M + 17 * N + K)
    cb, scb = _weights(N, K, g)
    x = _rows(M, K, g, n_out)
    R = O.int8_linear_exact(x, cb, scb)
    old = O.int8_linear(x, cb, scb)
    # int8_linear's 127.0 / sca is reciprocal-then-multiply: where that moves a product across a .5 tie its CA differs
    a = x.float().half().float().masked_fill(R.mask, 0.0)
    ca_old = torch.round(a * (127.0 / R.sca.clamp_min(1e-30)).unsqueeze(1)).clamp(-127, 127)
    same = (ca_old == R.ca).all(1)
    assert float(same.float().mean()) >= 0.5
    assert bool(R.out.contains(old)[same].all())
    differ = old.view(torch.int16) != R.out.id.view(torch.int16)
    assert float(differ[same].float().mean()) < 5e-3, int(differ[same].sum())
    # the exact parts agree with the oracle's
    a = x.float().half().float()
    assert torch.equal(R.mask, (a.abs() >= THR).any(0))


def test_signed_zero_sets():
    """Corners -0 and +0 admit both zeros; corners that are all -0 admit -0 only."""
    z = torch.tensor([0.0, -0.0]).bfloat16()
    both = O.Adm.of(z[0:1], [z[1:2], z[0:1]])
    assert bool(both.contains(z[0:1]).all()) and bool(both.contains(z[1:2]).all())
    neg = O.Adm.of(z[1:2], [z[1:2], z[1:2]])
    assert bool(neg.contains(z[1:2]).all()) and not bool(neg.contains(z[0:1]).any())

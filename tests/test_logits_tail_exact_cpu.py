"""CPU checks of the exact restatements of the logits tail (oracle.llama_oracle.topk_softmax_exact, draw_exact,
nll_exact) before any kernel is measured against them in test_gpu_logits_tail_exact.py:

1. the kept set equals an independent sort of IEEE-ordered keys (-0 == +0, NaN largest);
2. the float64 probability, rounded to bf16, lies in every admissible set, and away from bf16 midpoints the set is one value;
3. an fp32 evaluation of the sampling kernel's chain, in its order and with expf perturbed by up to 2 ulp, lands in the
   set for every input family of the GPU file;
4. the input constructions do what they claim (the threshold on +0 with -0 entries kept, the tie block across the
   k-th rank, one high-byte bin, all 256 bins, the temperature that overflows and the one that underflows);
5. nll_exact's bound holds for an fp32 evaluation of the NLL kernels' chain in their order (numpy, expf / logf
   perturbed by ±2 ulp), at logits where exp without the max subtraction overflows and with -inf tiles."""
import math

import numpy as np
import pytest
import torch

from oracle import llama_oracle as O
from test_gpu_logits_tail_exact import FAMILIES, NLL_FAMILIES, nll_inputs, rounded_tie_q, sampling_inputs, tie_positions

F32 = np.float32


def _perturb(y, rng, ulps):
    """fp32 y moved by a random number of ulps in [-ulps, ulps] (not past 0 or inf)."""
    y = y.astype(F32).copy()
    steps = rng.integers(-ulps, ulps + 1, size=y.shape)
    for s in range(1, ulps + 1):
        up = steps >= s
        dn = steps <= -s
        y[up] = np.nextafter(y[up], F32(np.inf))
        y[dn] = np.nextafter(y[dn], F32(0))
    return y


def _expf(d, rng):
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(d.astype(np.float64)).astype(F32)
    fin = np.isfinite(e) & (e > 0)
    e[fin] = _perturb(e[fin], rng, 2)
    return e


def _bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=F32)).bfloat16()


def _sampling_chain(x, T, k, rng):
    """topk_softmax_kernel in fp32 numpy for one row: (probs bf16 [V]).  Kept set and d as the kernel makes them
    (keys with -0 stored as +0); the sum per thread over its vectors 8 elements at a time, then the two butterflies."""
    V = x.numel()
    inv = F32(1.0) / F32(T)
    s = (x.float().numpy() * inv).astype(F32)
    s = torch.from_numpy(s).bfloat16().float().numpy()
    s = np.where(s == 0, F32(0), s)                                         # -0 stored as +0
    with np.errstate(invalid="ignore"):
        if 0 < k < V:
            key = np.where(np.isnan(s), np.inf, s)
            thr = np.sort(key)[::-1][k - 1]
            kept = np.isnan(s) | (key >= thr)
        else:
            kept = np.ones(V, bool)
        gmax = np.max(np.where(np.isnan(s), -np.inf, s)).astype(F32)
        d = (s - gmax).astype(F32)
        e = _expf(d, rng)
        e = np.where(kept & (s != -np.inf), e, F32(0))
    Vp = (V + 7) // 8 * 8
    ep = np.zeros(Vp, F32)
    ep[:V] = e
    nvp = Vp // 8
    rounds = -(-nvp // 1024)
    vec = np.zeros((rounds * 1024, 8), F32)
    vec[:nvp] = ep.reshape(nvp, 8)
    vec = vec.reshape(rounds, 1024, 8)
    acc = np.zeros(1024, F32)
    with np.errstate(invalid="ignore"):
        for r in range(rounds):
            for j in range(8):
                acc = (acc + vec[r, :, j]).astype(F32)
        w = acc.reshape(32, 32)
        for o in (16, 8, 4, 2, 1):
            w = (w + w[:, np.arange(32) ^ o]).astype(F32)
        t = w[:, 0].copy()
        for o in (16, 8, 4, 2, 1):
            t = (t + t[np.arange(32) ^ o]).astype(F32)
        total = t[0]
        e2 = _expf(d, rng)
        p = np.where(kept & (s != -np.inf), (e2 / total).astype(F32), F32(0))
    return _bf16(p)


@pytest.mark.parametrize("V", [1, 7, 9, 130, 8193, 32769])
def test_kernel_chain_lands_in_set_for_every_family(V):
    rng = np.random.default_rng(V)
    for fi, fam in enumerate(FAMILIES):
        x, T, k = sampling_inputs(fam, 2, V, seed=V * 31 + fi)
        R = O.topk_softmax_exact(x, T, k)
        assert bool(R.probs.contains(R.probs.id).all()), fam
        for b in range(2):
            p = _sampling_chain(x[b], T, k, rng)
            ok = R.probs.contains(p.view(1, -1))[0] if x.shape[0] == 1 else \
                O.topk_softmax_exact(x[b:b + 1], T, k).probs.contains(p.view(1, -1))[0]
            assert bool(ok.all()), (fam, b, int((~ok).sum()))


def _ieee_key(v):
    """A total order on float values for sorting: -0 == +0, NaN above +inf."""
    return math.inf if math.isnan(v) else (0.0 if v == 0 else v)


@pytest.mark.parametrize("fam", FAMILIES)
def test_kept_set_against_sorted_keys(fam):
    for V in (7, 130, 8193):
        x, T, k = sampling_inputs(fam, 2, V, seed=V + 3)
        R = O.topk_softmax_exact(x, T, k)
        for b in range(2):
            vals = [float(v) for v in R.scaled[b].float()]
            if 0 < k < V:
                thr = sorted((_ieee_key(v) for v in vals), reverse=True)[k - 1]
                want = [math.isnan(v) or _ieee_key(v) >= thr for v in vals]
            else:
                want = [True] * V
            assert R.kept[b].tolist() == want, (fam, V, b)


def test_float64_value_in_set_and_single_away_from_midpoints():
    g = torch.Generator().manual_seed(1)
    for V, T, k in ((32000, 0.8, 200), (50257, 1.0, 0), (130, 2.0, 4)):
        x = (torch.randn(4, V, generator=g) * 3).bfloat16()
        R = O.topk_softmax_exact(x, T, k)
        p = R.p.float()
        fin = R.kept & torch.isfinite(R.p)
        # the float64 value, rounded once, and its float32 rounding rounded again, are in the set
        assert bool(R.probs.contains(O.round_to(R.p, torch.bfloat16)).all())
        assert bool(R.probs.contains(p.bfloat16()).all())
        # away from a bf16 midpoint by more than the bound: one value
        mid_gap = (R.p - O.round_to(R.p, torch.bfloat16).double()).abs()
        ulp = torch.pow(2.0, torch.floor(torch.log2(R.p.clamp_min(1e-300))) - 7)
        far = fin & ((ulp / 2 - mid_gap) > 2 * R.bound) & (R.p > 2.0 ** -120)
        assert bool(R.probs.single()[far].all())
        assert float(R.probs.single()[fin].float().mean()) > 0.995
        assert torch.allclose(R.p.sum(-1), torch.ones(4, dtype=torch.float64), atol=1e-12)


def test_constructions():
    """What the GPU file's input families claim of their values."""
    V = 8193
    # ±0 at the threshold: the k-th largest is 0, -0 entries are kept, and enough +0 sit above the k-th rank that a
    # key order with -0 < +0 would put the threshold on +0 and drop them
    x, T, k = sampling_inputs("zero_thr", 3, V, seed=1)
    R = O.topk_softmax_exact(x, T, k)
    for b in range(3):
        s = R.scaled[b].float()
        assert float(R.thr[b]) == 0.0
        neg0 = (s == 0) & torch.signbit(s)
        pos0 = (s == 0) & ~torch.signbit(s)
        assert bool(R.kept[b][neg0].all()) and int(neg0.sum()) > 100
        assert int((s > 0).sum()) + int(pos0.sum()) >= k
    # T = 3e38 rounds every scaled value to ±0: both signs present, the threshold 0, everything kept
    x, T, k = sampling_inputs("t_under", 2, V, seed=2)
    R = O.topk_softmax_exact(x, T, k)
    s = R.scaled.float()
    assert bool((s == 0).all()) and bool(torch.signbit(s).any()) and bool((~torch.signbit(s)).any())
    assert bool(R.kept.all()) and 0 < k < V
    # T = 1e-37 overflows some scaled values to +inf: the row is NaN
    x, T, k = sampling_inputs("t_over", 2, 32000, seed=3)
    R = O.topk_softmax_exact(x, T, k)
    assert bool((R.scaled.float() == float("inf")).any(1).all()) and bool(torch.isnan(R.probs.id).any(1).all())
    # the tie block straddles the k-th rank: more kept entries than k
    x, T, k = sampling_inputs("tie70", 2, V, seed=4)
    R = O.topk_softmax_exact(x, T, k)
    assert bool((R.kept.sum(1) == 130).all()) and k < 130 and float(R.thr[0]) == 2.0
    # one high byte of the key (exponents 128 and 129), and every one of the 256
    key = lambda s: torch.where(torch.signbit(s), ~s.view(torch.int16).int() & 0xFFFF, (s.view(torch.int16).int() & 0xFFFF) | 0x8000)
    x, T, k = sampling_inputs("onebin", 1, V, seed=5)
    assert (key(O.topk_softmax_exact(x, T, k).scaled) >> 8).unique().numel() == 1
    x, T, k = sampling_inputs("allbins", 1, 51200, seed=6)
    assert (key(O.topk_softmax_exact(x, T, k).scaled) >> 8).unique().numel() >= 250
    # the k-th value in the lowest and in the highest bin
    for fam, want in (("kth_lowest", 0), ("kth_highest", 255)):
        x, T, k = sampling_inputs(fam, 1, V, seed=7)
        R = O.topk_softmax_exact(x, T, k)
        assert int(key(R.thr.bfloat16())[0, 0]) >> 8 == want, fam
    # subnormals: exponent field 0, nonzero
    x, _, _ = sampling_inputs("subnormal", 1, V, seed=8)
    assert bool(((x.view(torch.int16) & 0x7F80) == 0).all()) and bool((x != 0).all())
    # -inf inside the kept set
    x, T, k = sampling_inputs("neginf_kept", 1, V, seed=9)
    R = O.topk_softmax_exact(x, T, k)
    assert float(R.thr[0]) == float("-inf") and bool(R.kept.all()) and int((R.probs.id != 0).sum()) == 5
    # tie positions: each pair lies where its name says (thread t holds vectors t + 1024 j, lane t % 32, warp t / 32)
    for Vt in (9, 130, 8193, 32769, 50257):
        for name, (a, b) in tie_positions(Vt).items():
            assert 0 <= a < b < Vt, (name, Vt)
            ta, tb = (a // 8) % 1024, (b // 8) % 1024
            if name.startswith("thread"):
                assert ta == tb
            elif name == "lanes":
                assert ta // 32 == tb // 32 and ta != tb
            elif name.startswith("warps"):
                assert ta // 32 != tb // 32
            else:
                assert b >= Vt - Vt % 8


@pytest.mark.parametrize("V", [9, 130, 8193, 32769, 50257])
def test_rounded_tie_construction(V):
    """The GPU file's rounded ties: for p = bf16(1 / V) the two quotients differ in fp32 and agree in bf16, both above
    p / 4 (every other entry), so draw_exact picks the lower index and an unrounded argmax the higher one."""
    P = float(torch.tensor(1.0 / V).bfloat16())
    qa, qb = rounded_tie_q(P)
    p = torch.full((1, 4), P).bfloat16()
    q = torch.tensor([[4.0, qa, qb, 4.0]]).bfloat16()
    r = p.float() / q.float()
    assert float(r[0, 1]) < float(r[0, 2]) and float(r[0, 1].bfloat16()) == float(r[0, 2].bfloat16())
    assert O.draw_exact(p, q).tolist() == [1] and int(torch.argmax(r)) == 2


def test_draw_exact_rules():
    p = torch.tensor([[0.25, 0.5, 0.5, 0.0], [float("nan"), 0.1, float("nan"), 0.2], [0.0, 0.0, 0.0, 0.0]]).bfloat16()
    q = torch.tensor([[1.0, 2.0, 2.0, 1.0], [1.0, 1.0, 1.0, 1.0], [1.0, 1.0, 1.0, 1.0]]).bfloat16()
    assert O.draw_exact(p, q).tolist() == [0, 0, 0]
    assert torch.equal(O.draw_exact(p[:2], q[:2]), torch.argmax((p[:2] / q[:2]), dim=-1))
    # rounding of p / q to bf16 makes near-equal quotients equal: the lower index wins
    p = torch.tensor([[0.5, 0.95703125]]).bfloat16()
    q = torch.tensor([[0.5234375, 1.0]]).bfloat16()
    r = p.float() / q.float()
    assert float(r[0, 0]) < float(r[0, 1]) and float(r[0, 0].bfloat16()) == float(r[0, 1])
    assert O.draw_exact(p, q).tolist() == [0]


# ------------------------------------------------------------------ NLL
def _nll_chain(logits, t, rng):
    """logits_nll_tile_kernel + nll_combine_kernel in fp32 numpy, in their order (nll_common.cuh)."""
    L = logits.float().numpy()
    M, N = L.shape
    nt = -(-N // 128)
    out = np.empty(M, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for m in range(M):
            tg = int(t[m])
            if tg < 0 or tg >= N:
                out[m] = np.nan
                continue
            mxs, ss = [], []
            for j in range(nt):
                v = np.full(128, -np.inf, F32)
                seg = L[m, j * 128:(j + 1) * 128]
                v[:seg.size] = seg
                lanes = v.reshape(16, 4, 2).transpose(1, 0, 2).reshape(4, 32)   # lane q: columns 8c + 2q + e
                mx = F32(np.max(np.where(np.isnan(lanes), -np.inf, lanes))) if not np.isnan(lanes).all() else F32(np.nan)
                base = F32(0) if mx == -np.inf else mx
                e = _expf((lanes - base).astype(F32), rng)
                acc = np.zeros(4, F32)
                for i in range(32):
                    acc = (acc + e[:, i]).astype(F32)
                acc = (acc + acc[[1, 0, 3, 2]]).astype(F32)
                acc = (acc + acc[[2, 3, 0, 1]]).astype(F32)
                mxs.append(mx)
                ss.append(acc[0])
            mx = F32(max((x for x in mxs if not np.isnan(x)), default=-np.inf))
            s = F32(0)
            for mj, sj in zip(mxs, ss):
                s = F32(s + F32(sj * _expf(np.array([F32(mj - mx)]), rng)[0]))
            ls = np.log(np.float64(s)).astype(F32) if s > 0 else F32(np.log(np.float64(s)))
            if np.isfinite(ls) and ls != 0:
                ls = _perturb(np.array([ls]), rng, 1)[0]
            out[m] = F32(F32(mx + ls) - F32(L[m, tg]))
    return torch.from_numpy(out)


@pytest.mark.parametrize("N", [1, 2, 127, 128, 129, 1000, 4097])
def test_nll_bound_holds_for_the_kernel_chain(N):
    rng = np.random.default_rng(N)
    for fi, fam in enumerate(NLL_FAMILIES):
        logits, t = nll_inputs(fam, 12, N, seed=N + fi)
        R = O.nll_exact(logits, t)
        got = _nll_chain(logits, t, rng).double()
        assert torch.equal(torch.isnan(got), torch.isnan(R.nll)), (fam, got.tolist(), R.nll.tolist())
        inf = torch.isinf(R.nll)
        assert torch.equal(torch.isinf(got), inf) and bool((got[inf] == R.nll[inf]).all()), fam
        fin = torch.isfinite(R.nll)
        err = (got - R.nll).abs()
        assert bool((err <= R.bound)[fin].all()), (fam, err[fin].max().item(), R.bound[fin].min().item())


def test_nll_exact_special_values():
    N = 300
    x = torch.randn(6, N).bfloat16()
    t = torch.tensor([3, 4, 5, 6, N, -1])
    x[0, 3] = float("nan")
    x[1, 4] = float("inf")
    x[2, 5] = float("-inf")
    x[3, :] = float("-inf")
    R = O.nll_exact(x, t)
    assert torch.isnan(R.nll[[0, 1, 3, 4, 5]]).all() and float(R.nll[2]) == float("inf")
    # equal rows: log N, and the bound is a few fp32 ulps of it
    e = O.nll_exact(torch.full((2, 32000), 2.5).bfloat16(), torch.tensor([0, 31999]))
    assert bool(((e.nll - math.log(32000)).abs() < 1e-12).all()) and float(e.bound.max()) < 64 * 2.0 ** -24 * math.log(32000)

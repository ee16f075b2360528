"""-m gpu: the two kernels that consume the logits against exact arithmetic.

Sampling (topk_softmax_kernel, csrc/sampling.cu) through b2l_topk_softmax, b2l_topk_softmax_sample, _rows and
_sample_rows, against oracle.llama_oracle.topk_softmax_exact: the kept set exactly, every probability in its admissible
set, a least share bit-equal to the single-rounded value, and the token equal to draw_exact (argmax(bf16(p / q)), ties
to the lowest index, NaN first) on the kernel's own probabilities, always in 0..V-1.  V from 1 to 51200 (102400 for
probabilities only: the shared-memory limits with and without noise; one above each is refused), past 32768 the
kernel's reload path, B in {1, 3, 16} with ld = V, V + 3 and 0.  Input families, each for one edge: randn at several
σ; every value in one high-byte bin (the second radix pass decides); values over all 256 bins; all equal; a 70-value
tie block across the k-th rank; the k-th value in the lowest and in the highest bin; negative logits only; bf16
subnormals; ±0 at the threshold; -inf inside the kept set and all but one entry -inf; a NaN logit; temperatures 0.05..20,
one that overflows the scaled logits to inf and one that underflows them to zero.  Constructed noise puts equal maxima
of bf16(p / q) in one thread, in lanes of one warp, across warps and in the V % 8 tail, both exactly equal quotients
and quotients that only the bf16 rounding of p / q makes equal.

NLL (logits_nll_tile_kernel + nll_combine_kernel, and the NLL epilogue of the q4 / w8 GEMMs) against
oracle.llama_oracle.nll_exact: every nll[m] within the derived bound, NaN and inf exactly where the contract puts them,
the fp64 window sum within M 2^-53 Σ|nll| of the exact sum of the returned values, repeated launches bit-identical, and
the fused GEMM paths bit-identical to the standalone kernel at logits of about ±60."""
import ctypes as C
import math
import struct

import pytest
import torch

from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu

MIN_EQUAL = 0.999  # share of probabilities bit-equal to the single-rounded value, per launch (measured: 100 %)
_SHARES = []       # (case, share), the lowest printed at the end (pytest -s)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)
    if _SHARES:
        worst = {}
        for fam, v in _SHARES:
            worst[fam] = min(worst.get(fam, 1.0), v)
        print("\nlowest bit-equal share per family:", ", ".join(f"{f}: {100 * v:.3f} %" for f, v in sorted(worst.items())))


def _L():
    from lit_llama_b200 import _lib as L

    return L


# ---------------------------------------------------------------- sampling inputs
def sampling_inputs(fam: str, B: int, V: int, seed: int):
    """(logits [B, V] bf16 on the CPU, temperature, top_k) for one input family."""
    g = torch.Generator().manual_seed(seed)
    k = min(max(V // 4, 1), 200) if V > 1 else 0
    T = 0.8
    if fam.startswith("randn"):
        sig = {"randn": 3.0, "randn_small": 0.3, "randn_big": 40.0}[fam]
        x = torch.randn(B, V, generator=g) * sig
        T = {"randn": 0.8, "randn_small": 0.05, "randn_big": 20.0}[fam]
    elif fam == "onebin":          # exponents 128 and 129: one high byte of the key, the second pass decides
        x = torch.rand(B, V, generator=g) * 5.9 + 2
        T = 1.0
    elif fam == "allbins":         # |x| from 1e-38 to 3e38, both signs: every high byte
        mag = torch.pow(10.0, torch.rand(B, V, generator=g) * 76.4 - 38)
        x = mag * torch.where(torch.rand(B, V, generator=g) < 0.5, -1.0, 1.0)
        x = x.clamp(-3e38, 3e38)
        T = 1.0
        k = max(V // 3, 1) if V > 1 else 0
    elif fam == "equal":
        x = torch.full((B, V), 1.5)
    elif fam == "tie70":           # 60 distinct values above a block of 70 equal ones, the k-th rank inside the block
        x = torch.randn(B, V, generator=g) - 10
        n_top = min(60, V // 3)
        n_tie = min(70, V - n_top)
        for b in range(B):
            p = torch.randperm(V, generator=g)
            x[b, p[:n_top]] = torch.linspace(3, 9, n_top)
            x[b, p[n_top:n_top + n_tie]] = 2.0
        k = n_top + max(n_tie // 2, 1) if V > 1 else 0
        T = 1.0
    elif fam == "kth_lowest":      # the k-th value among -(1.7..3.3)e38 (high byte 0)
        x = -(torch.rand(B, V, generator=g) * 1.6e38 + 1.7e38)
        n_up = max(V // 5, 1)
        x[:, :n_up] = torch.randn(B, n_up, generator=g)
        k = min(n_up + max(V // 3, 1), V - 1) if V > 2 else 0
        T = 1.0
    elif fam == "kth_highest":     # the k-th value among (1.7..3.3)e38 (high byte 255)
        x = torch.randn(B, V, generator=g)
        n_up = min(max(V // 5, 2), V)
        x[:, :n_up] = torch.rand(B, n_up, generator=g) * 1.6e38 + 1.7e38
        k = max(n_up // 2, 1) if V > 1 else 0
        T = 1.0
    elif fam == "negative":
        x = -(torch.randn(B, V, generator=g).abs() * 3 + 5)
    elif fam == "subnormal":       # exponent field 0: every bf16 subnormal magnitude, both signs
        bits = torch.randint(1, 0x80, (B, V), generator=g) - 0x8000 * torch.randint(0, 2, (B, V), generator=g)
        x = bits.to(torch.int16).view(torch.bfloat16).float()   # negative int16: the sign bit set
        T = 1.0
    elif fam == "zero_thr":        # a few positives, then +0 / -0 mixed; the k-th largest is 0 with -0 in the kept set
        x = -(torch.rand(B, V, generator=g) * 4 + 0.5)
        n_pos = max(V // 10, 0)
        n_zero = max(V // 3, 1)
        for b in range(B):
            p = torch.randperm(V, generator=g)
            x[b, p[:n_pos]] = torch.rand(n_pos, generator=g) + 1
            z = p[n_pos:n_pos + n_zero]
            x[b, z] = 0.0
            x[b, z[::2]] = -0.0
        k = n_pos + max(n_zero // 4, 1) if V > 1 else 0
        T = 1.0
    elif fam == "t_under":         # T = 3e38: every scaled value rounds to ±0, the threshold is 0
        x = torch.randn(B, V, generator=g) * 1e-3
        T = 3e38
        k = max(V // 5, 1) if V > 1 else 0
    elif fam == "t_over":          # T = 1e-37: the scaled logits overflow to ±inf
        x = torch.randn(B, V, generator=g) * 10
        T = 1e-37
    elif fam == "neginf_kept":     # five finite logits, the rest -inf, k past them: -inf inside the kept set
        x = torch.full((B, V), float("-inf"))
        n = min(5, V)
        x[:, :n] = torch.randn(B, n, generator=g)
        k = min(n + 15, V - 1) if V > n + 1 else 0
    elif fam == "one_finite":      # all but one entry -inf
        x = torch.full((B, V), float("-inf"))
        for b in range(B):
            x[b, int(torch.randint(0, V, (1,), generator=g))] = 0.25 * b - 1
    elif fam == "nan":             # one NaN logit (k >= 2, so the threshold stays a number)
        x = torch.randn(B, V, generator=g) * 3
        for b in range(B):
            x[b, int(torch.randint(0, V, (1,), generator=g))] = float("nan")
        k = 0 if V < 3 else max(k, 2)
    else:
        raise ValueError(fam)
    return x.bfloat16(), T, k


FAMILIES = ["randn", "randn_small", "randn_big", "onebin", "allbins", "equal", "tie70", "kth_lowest", "kth_highest",
            "negative", "subnormal", "zero_thr", "t_under", "t_over", "neginf_kept", "one_finite", "nan"]
VOCABS = [1, 7, 8, 9, 130, 8191, 8192, 8193, 32000, 32768, 32769, 50257, 51200]


def _rows_buf(x, ld, dev):
    """x [B, V] into a 16-byte aligned device buffer with rows ld apart (ld = 0: x has one row, read by every CTA)."""
    B, V = x.shape
    if ld == 0:
        buf = torch.empty(V + 8, dtype=torch.bfloat16, device=dev)
        buf[:V] = x[0].to(dev)
        return buf
    buf = torch.full((B * ld + 8,), float("nan"), dtype=torch.bfloat16, device=dev)
    buf[: B * ld].view(B, ld)[:, :V] = x.to(dev)
    return buf


def _noise(B, V, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.empty(B, V, dtype=torch.bfloat16, device=dev).exponential_(1, generator=g)


def _launch(dev, x, T, k, ld, q=None, single=False):
    """probs [B, V] and tokens [B] (None without noise) from one launch of the row (or, single, the B = 1) entry point."""
    L = _L()
    B, V = x.shape
    buf = _rows_buf(x, ld, dev)
    probs = torch.full((B, V), float("nan"), dtype=torch.bfloat16, device=dev)
    if q is None:
        if single:
            rc = L.lib().b2l_topk_softmax(buf.data_ptr(), T, k, probs.data_ptr(), V, None)
        else:
            rc = L.lib().b2l_topk_softmax_rows(buf.data_ptr(), ld, T, k, probs.data_ptr(), B, V, None)
        tok = None
    else:
        tok = torch.full((B,), -7, dtype=torch.int64, device=dev)
        if single:
            rc = L.lib().b2l_topk_softmax_sample(buf.data_ptr(), T, k, q.data_ptr(), probs.data_ptr(), tok.data_ptr(), V, None)
        else:
            rc = L.lib().b2l_topk_softmax_sample_rows(buf.data_ptr(), ld, T, k, q.data_ptr(), probs.data_ptr(), tok.data_ptr(),
                                                       B, V, None)
    assert rc == 0, L.lib().b2l_last_error()
    torch.cuda.synchronize()
    return probs.cpu(), None if tok is None else tok.cpu()


def _check_probs(case, x, T, k, probs, record=True):
    R = O.topk_softmax_exact(x, T, k)
    A = R.probs
    ok = A.contains(probs)
    if not bool(ok.all()):
        b, i = [int(v) for v in (~ok).nonzero()[0]]
        raise AssertionError(f"{case}: p[{b}, {i}] = {float(probs[b, i])!r} outside [{float(A.lo[b, i])!r}, "
                             f"{float(A.hi[b, i])!r}] (kept {bool(R.kept[b, i])}, s {float(R.scaled[b, i])!r}, "
                             f"thr {float(R.thr[b, 0])!r}); {int((~ok).sum())} outside")
    # the kept set: nonzero exactly on kept entries, except where the set admits 0 (an underflowing probability)
    admits0 = A.contains(torch.zeros_like(probs))
    nz = (probs != 0) & ~torch.isnan(probs)
    assert bool((~nz | R.kept).all()), case
    assert bool((nz | ~R.kept | admits0 | torch.isnan(probs)).all()), case
    if record:
        same = (probs.view(torch.int16) == A.id.view(torch.int16)) | (torch.isnan(probs) & torch.isnan(A.id))
        share = float(same.float().mean())
        _SHARES.append((case.split("/")[0], share))
        assert share >= MIN_EQUAL, (case, share)
    return R


def _check_draw(case, probs, q, tok):
    want = O.draw_exact(probs, q.cpu())
    V = probs.shape[-1]
    assert bool(((tok >= 0) & (tok < V)).all()), (case, tok.tolist())
    assert torch.equal(tok, want), (case, tok.tolist(), want.tolist())


@pytest.mark.parametrize("V", VOCABS)
def test_sampling_families(dev, V):
    """Every family at B = 3 (ld = V + 3, with the draw), randn and ±0 also at B = 16 (ld = V) and B = 3 (ld = 0)."""
    for fi, fam in enumerate(FAMILIES):
        x, T, k = sampling_inputs(fam, 3, V, seed=V * 31 + fi)
        case = f"{fam}/V={V}/k={k}/T={T}"
        probs, _ = _launch(dev, x, T, k, V + 3)
        _check_probs(case, x, T, k, probs)
        q = _noise(3, V, dev, seed=fi + V)
        p2, tok = _launch(dev, x, T, k, V + 3, q=q)
        assert torch.equal(p2.view(torch.int16), probs.view(torch.int16)), case
        _check_draw(case, p2, q, tok)
    for fam in ("randn", "zero_thr", "tie70"):
        x, T, k = sampling_inputs(fam, 16, V, seed=V + 5)
        q = _noise(16, V, dev, seed=V + 6)
        probs, tok = _launch(dev, x, T, k, V, q=q)
        _check_probs(f"{fam}/B=16/V={V}", x, T, k, probs)
        _check_draw(f"{fam}/B=16/V={V}", probs, q, tok)
        x1 = x[:1].expand(3, V)
        probs, tok = _launch(dev, x1, T, k, 0, q=q[:3].contiguous())
        _check_probs(f"{fam}/ld=0/V={V}", x1, T, k, probs)
        _check_draw(f"{fam}/ld=0/V={V}", probs, q[:3], tok)


@pytest.mark.parametrize("V", [1, 9, 8193, 32769, 51200])
def test_single_row_entry_points(dev, V):
    """b2l_topk_softmax / b2l_topk_softmax_sample equal row 0 of the row entry points, and hold the same sets."""
    for fam in ("randn", "zero_thr", "nan", "t_over"):
        x, T, k = sampling_inputs(fam, 1, V, seed=V + 77)
        q = _noise(1, V, dev, seed=V + 78)
        p1, _ = _launch(dev, x, T, k, V, single=True)
        p2, tok = _launch(dev, x, T, k, V, q=q, single=True)
        p3, tok3 = _launch(dev, x, T, k, V, q=q)
        _check_probs(f"{fam}/single/V={V}", x, T, k, p1, record=False)
        assert torch.equal(p1.view(torch.int16), p2.view(torch.int16))
        assert torch.equal(p1.view(torch.int16), p3.view(torch.int16)) and torch.equal(tok, tok3)
        _check_draw(f"{fam}/single/V={V}", p2, q, tok)


@pytest.mark.parametrize("V", [51201, 102400])
def test_probabilities_up_to_the_smem_limit(dev, V):
    """102400 is the limit without noise; 51201 is past the limit with noise but fine without."""
    for fam in ("randn", "tie70", "zero_thr"):
        x, T, k = sampling_inputs(fam, 3, V, seed=V)
        probs, _ = _launch(dev, x, T, k, V + 3)
        _check_probs(f"{fam}/V={V}", x, T, k, probs)


def test_vocabulary_too_large_is_refused(dev):
    L = _L()
    buf = torch.zeros(102408 * 2, dtype=torch.bfloat16, device=dev)
    q = torch.ones(102408 * 2, dtype=torch.bfloat16, device=dev)
    probs = torch.zeros_like(buf)
    tok = torch.zeros(2, dtype=torch.int64, device=dev)
    lib = L.lib()
    assert lib.b2l_topk_softmax_rows(buf.data_ptr(), 102401, 1.0, 0, probs.data_ptr(), 1, 102401, None) == -2
    assert b"too large" in lib.b2l_last_error()
    assert lib.b2l_topk_softmax(buf.data_ptr(), 1.0, 0, probs.data_ptr(), 102401, None) == -2
    assert lib.b2l_topk_softmax_sample_rows(buf.data_ptr(), 51201, 1.0, 0, q.data_ptr(), None, tok.data_ptr(), 1, 51201,
                                            None) == -2
    assert b"too large" in lib.b2l_last_error()
    assert lib.b2l_topk_softmax_sample(buf.data_ptr(), 1.0, 0, q.data_ptr(), None, tok.data_ptr(), 51201, None) == -2
    assert lib.b2l_topk_softmax_sample_rows(buf.data_ptr(), 51200, 1.0, 0, q.data_ptr(), None, tok.data_ptr(), 1, 51200,
                                            None) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the draw's tie-break
def tie_positions(V: int):
    """Pairs (a, b) of indices, a < b, where equal maxima of bf16(p / q) exercise one level of the kernel's reduction:
    thread t holds vectors t, t + 1024, ... (8 elements each), lane t % 32 of warp t / 32."""
    out = {}
    if V >= 8:
        out["thread"] = (2, 6)                                            # one vector
    if V >= 8 * 1024 + 8:
        out["thread_rounds"] = (8 * 5 + 1, 8 * (1024 + 5) + 3)            # one thread, two rounds
    if V >= 8 * 20:
        out["lanes"] = (8 * 3 + 7, 8 * 17 + 0)                           # warp 0, lanes 3 and 17
    if V >= 8 * 700:
        out["warps"] = (8 * 40 + 4, 8 * 650 + 4)                         # warps 1 and 20
    if V >= 8 * 1024 + 8:
        out["warps_reversed"] = (8 * 1000 + 2, 8 * 1024 + 1)             # warp 31 round 0 vs warp 0 round 1
    if V % 8 and V > 8:
        out["tail"] = (V - V % 8 - 8 + 1, V - 1)                         # the last full vector and the tail
        out["tail_only"] = (V - V % 8, V - 1) if V % 8 > 1 else out["tail"]
    return out


def rounded_tie_q(P: float):
    """(q_a, q_b), bf16 values in [0.5, 1), with fl32(P / q_a) < fl32(P / q_b) but bf16(P / q_a) == bf16(P / q_b):
    only the bf16 rounding of p / q makes the two quotients equal."""
    q = torch.arange(0x3F00, 0x3F80, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    r = torch.tensor(P, dtype=torch.float32) / q
    rb = r.bfloat16().float()
    for v in rb.unique():
        sel = (rb == v).nonzero().view(-1)
        if sel.numel() >= 2 and float(r[sel].min()) < float(r[sel].max()):
            return float(q[sel[int(r[sel].argmin())]]), float(q[sel[int(r[sel].argmax())]])
    raise AssertionError(P)


@pytest.mark.parametrize("V", [9, 130, 8193, 32769, 50257])
def test_draw_tie_break_at_every_reduction_level(dev, V):
    """All logits equal (every p the same bf16 value); q = 1 except q = 1/2 at the pair, so bf16(p / q) takes its
    maximum at exactly those two entries: the token must be the lower index, in either order of arrival."""
    x = torch.full((1, V), 0.5).bfloat16()
    pairs = tie_positions(V)
    assert pairs
    for name, (a, b) in pairs.items():
        for extra in (None, "first"):
            q = torch.ones(1, V)
            at = [a, b]
            if extra == "first":   # a third maximum elsewhere: still the lowest index wins
                at.append(V - 1 if b != V - 1 else 0)
            q[0, at] = 0.5
            qd = q.bfloat16().to(dev)
            for k in (0, V):
                probs, tok = _launch(dev, x, 1.0, k, V, q=qd)
                want = min(at)
                _check_draw(f"tie/{name}/V={V}", probs, qd, tok)
                assert int(tok[0]) == want, (name, a, b, int(tok[0]))
        # a tie made by the rounding of p / q alone: the exact quotient is larger at b, the bf16 ones are equal
        P = float(_launch(dev, x, 1.0, 0, V)[0][0, 0])
        qa, qb = rounded_tie_q(P)
        q = torch.full((1, V), 4.0)
        q[0, a], q[0, b] = qa, qb
        qd = q.bfloat16().to(dev)
        probs, tok = _launch(dev, x, 1.0, 0, V, q=qd)
        _check_draw(f"rounded_tie/{name}/V={V}", probs, qd, tok)
        assert int(tok[0]) == a, (name, a, b, int(tok[0]))


def test_draw_nan_and_filtered(dev):
    """A NaN logit makes every kept probability NaN: the token is the first kept entry (torch.argmax ranks NaN first),
    never an out-of-range id and never a filtered entry."""
    V = 1000
    x = (torch.randn(1, V, generator=torch.Generator().manual_seed(3)) * 2).bfloat16()
    x[0, 700] = float("nan")
    for k, T in ((0, 1.0), (50, 1.0), (50, 1e-37)):
        q = _noise(1, V, dev, seed=k)
        probs, tok = _launch(dev, x, T, k, V, q=q)
        R = _check_probs(f"nan_draw/k={k}", x, T, k, probs, record=False)
        first_kept = int(R.kept[0].nonzero()[0])
        assert int(tok[0]) == first_kept, (k, int(tok[0]), first_kept)
        _check_draw(f"nan_draw/k={k}", probs, q, tok)


# ---------------------------------------------------------------- NLL
def _nll_launch(dev, logits, t, ldl):
    """(nll fp32 [M], nll_sum fp64) from b2l_logits_nll on logits [M, N] stored with leading dimension ldl."""
    L = _L()
    M, N = logits.shape
    buf = torch.full((M * ldl + 2,), float("nan"), dtype=torch.bfloat16, device=dev)
    buf[: M * ldl].view(M, ldl)[:, :N] = logits.to(dev)
    tt = t.to(dev)
    nll = torch.full((M,), 7.0, dtype=torch.float32, device=dev)
    s = torch.zeros((), dtype=torch.float64, device=dev)
    ws = torch.empty(max(L.lib().b2l_nll_workspace_bytes(M, N), 16), dtype=torch.uint8, device=dev)
    a = L.NLLArgs(targets=tt.data_ptr(), targets_i64=1 if tt.dtype == torch.int64 else 0, nll=nll.data_ptr(),
                  nll_sum=s.data_ptr(), workspace=ws.data_ptr())
    rc = L.lib().b2l_logits_nll(buf.data_ptr(), ldl, M, N, C.byref(a), None)
    assert rc == 0, L.lib().b2l_last_error()
    torch.cuda.synchronize()
    return nll.cpu(), float(s.cpu())


def nll_inputs(fam: str, M: int, N: int, seed: int):
    """(logits [M, N] bf16 on the CPU, targets int64 [M])."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, N, (M,), generator=g)
    if fam == "big100":
        x = (torch.rand(M, N, generator=g) * 200 - 100)
    elif fam == "huge":          # ±3e38; the targets sit on logits >= 0 so that the loss stays below fp32's range
        x = (torch.rand(M, N, generator=g) * 6 - 3) * 1e38
        x[torch.arange(M), t] = x[torch.arange(M), t].abs()
    elif fam == "equal":
        x = torch.full((M, N), 2.5)
    elif fam == "argmax":
        x = torch.randn(M, N, generator=g) * 4
        t = x.bfloat16().float().argmax(1)
    elif fam == "edges":         # targets at 127 / 128 (the tile edge), 0 and N - 1
        x = torch.randn(M, N, generator=g) * 4
        ed = torch.tensor([min(127, N - 1), min(128, N - 1), 0, N - 1])
        t = ed[torch.arange(M) % 4]
    elif fam == "neginf_scatter":
        x = torch.randn(M, N, generator=g) * 4
        x[torch.rand(M, N, generator=g) < 0.3] = float("-inf")
        x[torch.arange(M), t] = 1.0
    elif fam == "neginf_tile":   # one whole aligned 128-column tile at -inf (the last tile when N <= 128: whole row)
        x = torch.randn(M, N, generator=g) * 4
        tile = 1 if N > 256 else 0
        x[:, tile * 128:(tile + 1) * 128] = float("-inf")
        if N > 128:
            lo, hi = (tile + 1) * 128 if tile == 0 else 0, N if tile == 0 else 128
            t = torch.randint(lo, min(hi, N), (M,), generator=g)
    elif fam == "specials":      # NaN / +inf / -inf target logits, out-of-range targets, NaN and +inf off target
        x = torch.randn(M, N, generator=g) * 4
        r = torch.arange(M)
        x[r[0::6], t[0::6]] = float("nan")
        x[r[1::6], t[1::6]] = float("inf")
        x[r[2::6], t[2::6]] = float("-inf")
        t[3::6] = torch.where(torch.arange(t[3::6].numel()) % 2 == 0, N, -1)
        if N > 1:
            x[r[4::6], (t[4::6] + 1) % N] = float("nan")
    else:
        raise ValueError(fam)
    return x.bfloat16(), t


NLL_FAMILIES = ["big100", "huge", "equal", "argmax", "edges", "neginf_scatter", "neginf_tile", "specials"]


def _check_nll(case, logits, t, nll, s):
    R = O.nll_exact(logits, t)
    got = nll.double()
    nan_want = torch.isnan(R.nll)
    assert torch.equal(torch.isnan(got), nan_want), (case, torch.isnan(got).nonzero().view(-1)[:8].tolist(),
                                                       nan_want.nonzero().view(-1)[:8].tolist())
    inf_want = torch.isinf(R.nll)
    assert torch.equal(torch.isinf(got), inf_want) and bool((got[inf_want] == R.nll[inf_want]).all()), case
    fin = torch.isfinite(R.nll)
    err = (got - R.nll).abs()
    bad = fin & ~(err <= R.bound)
    if bool(bad.any()):
        m = int(bad.nonzero()[0])
        raise AssertionError(f"{case}: nll[{m}] = {float(got[m])!r}, exact {float(R.nll[m])!r}, error {float(err[m]):.3g} "
                             f"> bound {float(R.bound[m]):.3g}; {int(bad.sum())} rows")
    vals = nll.tolist()
    if any(math.isnan(v) for v in vals):
        assert math.isnan(s), case
    elif any(math.isinf(v) for v in vals):
        assert s == sum(v for v in vals if math.isinf(v)), case
    else:
        exact = math.fsum(vals)
        assert abs(s - exact) <= len(vals) * 2.0 ** -53 * sum(abs(v) for v in vals), case


@pytest.mark.parametrize("N", [1, 2, 127, 128, 129, 32000, 32001])
def test_nll_families(dev, N):
    for fi, fam in enumerate(NLL_FAMILIES):
        for M, odd in ((7, True), (300 if N > 1000 else 2047, False)):
            if fam == "neginf_tile" and N <= 128 and M > 7:
                continue
            logits, t = nll_inputs(fam, M, N, seed=N * 13 + fi + M)
            ldl = N + (N % 2 == 0 if odd else N % 2)   # odd: 2-byte loads; even: the paired loads
            ti = t.to(torch.int32) if odd else t
            nll, s = _nll_launch(dev, logits, ti, ldl)
            _check_nll(f"{fam}/N={N}/M={M}/ldl={ldl}", logits, t, nll, s)
            nll2, s2 = _nll_launch(dev, logits, ti, ldl)
            assert torch.equal(nll.view(torch.int32), nll2.view(torch.int32)), fam
            assert struct.pack("<d", s) == struct.pack("<d", s2) or (math.isnan(s) and math.isnan(s2)), fam


def test_nll_whole_row_families_at_m2047(dev):
    """The largest window (M = 2047) at the vocabulary width, equal rows (loss log N up to the bound) and -inf tiles."""
    N, M = 32000, 2047
    for fam in ("equal", "neginf_tile", "big100"):
        logits, t = nll_inputs(fam, M, N, seed=M + len(fam))
        nll, s = _nll_launch(dev, logits, t, N)
        _check_nll(f"{fam}/N={N}/M={M}", logits, t, nll, s)
        if fam == "equal":
            assert float((nll.double() - math.log(N)).abs().max()) <= float(O.nll_exact(logits, t).bound.max())


def _gptq_linear(dev, bits, N, K, seed, amp):
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.device(dev):
        lin = ColBlockQuantizedLinear(K, N, False, bits=bits, tile_cols=-1)
    epb = 8 // bits
    lin.quant_weight.copy_(torch.randint(0, 256, (N, K // epb), generator=g, device=dev, dtype=torch.uint8))
    lv = 2 ** bits
    lin.scales = ((torch.rand(N, 1, generator=g, device=dev) + 0.5) * (amp / (lv * K ** 0.5))).to(torch.bfloat16)
    lin.zeros = torch.randint(lv // 2 - lv // 8, lv // 2 + lv // 8, (N, 1), generator=g, device=dev).to(torch.bfloat16)
    return lin


def _fused_nll(dev, lin, x, t, kind):
    L = _L()
    M, N, K = t.numel(), lin.out_features, x.shape[1]
    nll = torch.full((M,), 7.0, dtype=torch.float32, device=dev)
    s = torch.zeros((), dtype=torch.float64, device=dev)
    ws = torch.empty(max(L.lib().b2l_nll_workspace_bytes(M, N), 16), dtype=torch.uint8, device=dev)
    a = L.NLLArgs(targets=t.data_ptr(), targets_i64=1, nll=nll.data_ptr(), nll_sum=s.data_ptr(), workspace=ws.data_ptr())
    wt = lin.tiled() if kind == "q4" else lin.reference_quant_weight()
    g = L.Q4LinearArgs(x=x.data_ptr(), ldx=x.stride(0), qw_tiled=wt.data_ptr(), scales=lin.scales.data_ptr(),
                       zeros=lin.zeros.data_ptr(), sz_dtype=L.sz_dtype_of(lin.scales), y=None, ldy=0, M=M, N=N, K=K,
                       prologue=L.PRO_NONE, norm_scale=None, eps=0.0, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0,
                       flags=0)
    fn = "b2l_q4_gemm_nll" if kind == "q4" else "b2l_w8_gemm_nll"
    rc = getattr(L.lib(), fn)(C.byref(g), C.byref(a), None)
    assert rc == 0, L.lib().b2l_last_error()
    torch.cuda.synchronize()
    return nll.cpu(), float(s.cpu())


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K,M", [(32000, 4096, 300), (1000, 512, 129), (999, 512, 40)])
def test_fused_gemm_nll_bit_identical_at_large_logits(dev, bits, N, K, M):
    """The q4 / w8 GEMM's NLL epilogue against b2l_logits_nll on the logits the plain GEMM writes, with the scales
    raised so that the logits reach about ±60, and both within the bound of nll_exact."""
    lin = _gptq_linear(dev, bits, N, K, seed=N + K + bits, amp=50.0)
    g = torch.Generator(device=dev).manual_seed(M + bits)
    x = torch.randn(M + 1, K, generator=g, device=dev).to(torch.bfloat16)
    t = torch.randint(0, N, (M,), generator=g, device=dev)
    t[: min(M, 4)] = torch.tensor([0, 127, 128, N - 1][: min(M, 4)], device=dev)
    logits = lin(x)[:M].contiguous()
    torch.cuda.synchronize()
    amax = float(logits.float().abs().max())
    assert 30 < amax < 150, amax
    got = _fused_nll(dev, lin, x, t, "q4" if bits == 4 else "w8")
    want = _nll_launch(dev, logits, t, N)
    assert torch.equal(got[0].view(torch.int32), want[0].view(torch.int32)), float((got[0] - want[0]).abs().max())
    assert got[1] == want[1]
    _check_nll(f"fused{bits}/N={N}/M={M}", logits.cpu(), t.cpu(), got[0], got[1])

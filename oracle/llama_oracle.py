"""CPU oracle for the lit-llama quantized decode path.  TEST INFRASTRUCTURE ONLY.

This module restates, on the CPU, the arithmetic of the reference hot path
(SURVEY.md section 8a) as plain functions over torch CPU tensors.  It exists to
*check* the CUDA path; nothing under `lit-llama_b200/` may import it.  Only
`tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference`
legs of `bench.py` use it.

Pinning: the reference's own tests hold no golden vectors for quantization.py
(SURVEY.md section 8c); the pin is therefore the reference itself, executed in the
build container by `oracle/make_golden.py`, whose outputs are committed under
`tests/golden/` and compared against this restatement by
`tests/test_oracle_golden.py`.  The gptq.int4/int8 + model.py + generate.py part
is pinned that way.  The llm.int8 part restates the published bitsandbytes
LLM.int8() algorithm (bitsandbytes is unpinned in pyproject.toml:19, absent from
the reference checkout and not installed) and is therefore **parity unpinned**.

Every function cites the reference lines (relative to the reference checkout) it follows.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

Tensor = torch.Tensor


# ----------------------------------------------------------------------------
# lit_llama/utils.py
# ----------------------------------------------------------------------------
def find_multiple(n: int, k: int) -> int:
    """lit_llama/utils.py:38-41."""
    r = n % k
    return n if r == 0 else n + (k - r)


MODEL_SIZES = {4096: "7B", 5120: "13B", 6656: "30B", 8192: "65B"}  # utils.py:20-25
CONFIGS = {  # model.py:42-47
    "7B": dict(n_layer=32, n_head=32, n_embd=4096),
    "13B": dict(n_layer=40, n_head=40, n_embd=5120),
    "30B": dict(n_layer=60, n_head=52, n_embd=6656),
    "65B": dict(n_layer=80, n_head=64, n_embd=8192),
}


def n_hidden_for(n_embd: int) -> int:
    """model.py:243-245: SwiGLU hidden width."""
    return find_multiple(int(2 * (4 * n_embd) / 3), 256)


# ----------------------------------------------------------------------------
# lit_llama/quantization.py : round-to-nearest parameters + packing
# ----------------------------------------------------------------------------
def rtn_params(w: Tensor, bits: int) -> Tuple[Tensor, Tensor]:
    """Per-output-row asymmetric min/max grid.  quantization.py:477-513
    (perchannel=True, sym=False).  Returns (scale, zero), both (out, 1)."""
    maxq = 2**bits - 1
    lo = torch.clamp(w.amin(dim=1), max=0.0)
    hi = torch.clamp(w.amax(dim=1), min=0.0)
    dead = (lo == 0) & (hi == 0)
    lo = torch.where(dead, torch.full_like(lo, -1.0), lo)
    hi = torch.where(dead, torch.full_like(hi, 1.0), hi)
    scale = (hi - lo) / maxq
    zero = torch.round(-lo / scale)
    return scale.reshape(-1, 1), zero.reshape(-1, 1)


def rtn_levels(w: Tensor, scale: Tensor, zero: Tensor, bits: int) -> Tensor:
    """Integer levels q = clamp(round(w/scale)+zero, 0, maxq).  quantization.py:471-475."""
    return torch.clamp(torch.round(w / scale) + zero, 0, 2**bits - 1)


def pack_levels(levels: Tensor, bits: int) -> Tensor:
    """levels (out, in) in [0, 2^bits) -> uint8 (out, in/epb) stored with strides
    (1, out), i.e. memory is row-major (in/epb, out).  Entry `nr` of a byte sits at
    bit nr*bits and holds column epb*j+nr.  quantization.py:350-359, 386-390."""
    epb = 8 // bits
    lv = levels.to(torch.uint8)
    out, inf = lv.shape
    packed = torch.zeros((out, inf // epb), dtype=torch.uint8)
    for nr in range(epb):
        packed |= lv[:, nr::epb] << (nr * bits)
    return packed.t().contiguous().t()


def pack_weight(w: Tensor, scales: Tensor, zeros: Tensor, bits: int, tile_cols: int) -> Tensor:
    """ColBlockQuantizedLinear.pack_weight, quantization.py:376-390: divide by the
    group's scale, add the zero, clamp, *truncate* to uint8 (no rounding: the
    caller passes scale*(q-zero) so the quotient is integral up to fp error)."""
    w = w.clone()
    for g in range(scales.size(1)):
        sl = slice(g * tile_cols, (g + 1) * tile_cols)
        w[:, sl] /= scales[:, g : g + 1]
        w[:, sl] += zeros[:, g : g + 1]
    return pack_levels(w.clamp_(0, 2**bits - 1).to(torch.uint8), bits)


def unpack_levels(qw: Tensor, bits: int) -> Tensor:
    """uint8 (out, in/epb) -> int levels (out, in).  quantization.py:398-402."""
    epb = 8 // bits
    mask = (1 << bits) - 1
    out, packed_cols = qw.shape
    lv = torch.empty((out, packed_cols * epb), dtype=torch.uint8)
    for nr in range(epb):
        lv[:, nr::epb] = (qw >> (nr * bits)) & mask
    return lv


def dequant(qw: Tensor, scales: Tensor, zeros: Tensor, bits: int, tile_cols: int, dtype=torch.float32) -> Tensor:
    """ColBlockQuantizedLinear.get_weight, quantization.py:392-411.  The level is
    written into a `dtype` tensor, the zero subtracted and the scale multiplied *in
    that dtype* (so in bf16 each weight carries one bf16 rounding)."""
    w = unpack_levels(qw, bits).float().to(dtype)
    for g in range(scales.size(1)):
        sl = slice(g * tile_cols, (g + 1) * tile_cols)
        w[:, sl] -= zeros[:, g : g + 1]
        w[:, sl] *= scales[:, g : g + 1]
    return w


def qlinear(x: Tensor, qw: Tensor, scales: Tensor, zeros: Tensor, bits: int, tile_cols: int,
            bias: Optional[Tensor] = None) -> Tensor:
    """ColBlockQuantizedLinear.forward dense branch, quantization.py:422-423: the
    weight is re-materialised in x.dtype on every call, then F.linear."""
    return torch.nn.functional.linear(x, dequant(qw, scales, zeros, bits, tile_cols, x.dtype), bias)


def qlinear_exact(x: Tensor, qw: Tensor, scales: Tensor, zeros: Tensor, bits: int, tile_cols: int,
                  bias: Optional[Tensor] = None) -> Tensor:
    """Same contraction with exact fp32 dequant (level-zero)*scale and fp64
    accumulation - the arithmetic of the reference's GPU kernel
    (quantization.py:259-269: fp32 dequant, fp32 accumulate) without its TF32 dot.
    Returned in fp32; used as the tight numerical target for the CUDA kernels."""
    w = dequant(qw, scales.float(), zeros.float(), bits, tile_cols, torch.float32).double()
    y = x.double() @ w.t()
    if bias is not None:
        y = y + bias.double()
    return y.float()


# ----------------------------------------------------------------------------
# LLM.int8()  (restatement of bitsandbytes; parity unpinned - see module docstring)
# ----------------------------------------------------------------------------
def int8_quantize_weight(w: Tensor) -> Tuple[Tensor, Tensor]:
    """quantization.py:69-77 -> bnb.functional.double_quant on W.half(): row-wise
    absmax scaling to int8.  Returns CB int8 (out,in) and SCB fp32 (out,)."""
    wh = w.half().float()
    scb = wh.abs().amax(dim=1)
    cb = torch.round(wh * (127.0 / scb.clamp_min(1e-30)).unsqueeze(1)).clamp_(-127, 127).to(torch.int8)
    return cb, scb


def int8_linear(x: Tensor, cb: Tensor, scb: Tensor, threshold: float = 6.0) -> Tensor:
    """bnb.matmul / MatMul8bitLt.forward with has_fp16_weights=False,
    threshold=6.0 (quantization.py:47): activations go to fp16; columns of A that
    hold any |a| >= threshold are handled in fp16 against the dequantised weight
    columns, the rest row-wise absmax-quantised to int8; int32 GEMM; dequant by
    SCA*SCB/127^2; sum; cast back to x.dtype."""
    shape = x.shape
    a = x.reshape(-1, shape[-1]).half().float()
    outlier_cols = (a.abs() >= threshold).any(dim=0)
    a_in = a.clone()
    a_in[:, outlier_cols] = 0
    sca = a_in.abs().amax(dim=1)
    ca = torch.round(a_in * (127.0 / sca.clamp_min(1e-30)).unsqueeze(1)).clamp_(-127, 127)
    acc = ca.double() @ cb.double().t()  # exact int32 contraction
    y = (acc * (sca.double().unsqueeze(1) * scb.double().unsqueeze(0) / (127.0 * 127.0))).float()
    y = y.half().float()
    if outlier_cols.any():
        w_sub = (cb[:, outlier_cols].float() * (scb / 127.0).unsqueeze(1)).half().float()
        y = (y + (a[:, outlier_cols] @ w_sub.t()).half().float()).half().float()
    return y.to(x.dtype).reshape(*shape[:-1], cb.shape[0])


# LLM.int8() held exactly.  int8_linear above rounds the dequantised part fp64 -> fp32 -> fp16 (a double rounding);
# int8_linear_exact is the single-rounding statement of the same algorithm, with threshold θ:
#   x̂ = fp16(x);  O = {k : some row has |x̂[m,k]| >= θ};  SCA_m = max_{k∉O} |x̂[m,k]|;  qs = fl32(127 / SCA_m) (0 if 0)
#   CA = clamp(rint_even(fl32(x̂ qs)), ±127), 0 on O;  t = CA · CB[o] (exact);  v = fp16(t SCA_m SCB_o / 127²)
#   w_k = fp16(CB[o,k] SCB_o / 127);  τ = Σ_{k∈O} x̂_k w_k;  y = fp16(fl32(v + fp16(τ))) if O ≠ ∅ else v;  out = bf16(y)
# Steps with exact operands (mask, SCA, qs, CA, t, the fp32 add of two fp16 values, every conversion) are reproduced
# bit for bit.  Where a kernel chooses the evaluation order, the result is an admissible set: the correctly rounded
# value R(e), plus its neighbours across fp16 / bf16 midpoints that lie within the derived bound b of the exact e.
# Rounding is monotone, so a value computed within b of e rounds into [R(e - b), R(e + b)]; y, the bf16 store and the
# epilogue are monotone in each operand, so every set is an interval [lo, hi] of the output format (one value away
# from midpoints; then it is compared bit for bit), plus NaN where a corner of it is NaN.  Bounds, u = 2^-24 and
# γ_n = n u / (1 - n u):
#   v: (float)t, fl32(1/127²), sca·scb, ·(1/127²), t·that: five fp32 roundings, |err| <= γ_5 |v|;
#   w_k: fl32(SCB / 127), then fl32(CB · that): two roundings, γ_2 |w_k|;
#   τ: a chain of n = |O| fmaf, |err| <= γ_n Σ|x̂_k w_k|, plus |x̂_k| ulp16(w_k) for each w_k with two candidates;
#   silu: expf within 2 ulp (no fast math), then 1 + e and the IEEE division: |err| <= (2·2u + 2u + γ_2)|silu| < 7u|silu|.
# float64 slack (the fp64 products, and a float64 GEMM that may reorder its sum) is added on top of each.
INT8_U = 2.0 ** -24


def _gamma(n):
    return n * INT8_U / (1.0 - n * INT8_U)


def round_to(e: Tensor, dtype) -> Tensor:
    """float64 -> fp16 / bf16 / fp32 rounded once to nearest even (overflow to inf, subnormals, signed zero).  A plain
    .to(dtype) may go through fp32 and round twice, so the fp32 step rounds to odd: fp32 carries more than two extra
    bits over fp16 and bf16, and rounding to odd first makes the second rounding the correctly rounded one."""
    e = e.double()
    f = e.float()
    if dtype == torch.float32:
        return f
    inexact = (f.double() != e) & torch.isfinite(e)
    toward0 = torch.where(f.double().abs() > e.abs(), torch.nextafter(f, torch.zeros_like(f)), f)
    bits = toward0.view(torch.int32)
    odd = torch.where(inexact, bits | 1, bits).view(torch.float32)
    return odd.to(dtype)


def ulp16(w: Tensor) -> Tensor:
    """The spacing of fp16 at |w| (subnormal spacing 2^-24 included)."""
    a = w.double().abs().clamp_min(2.0 ** -14)
    return torch.pow(2.0, torch.floor(torch.log2(a)) - 10)


def _around(e: Tensor, b: Tensor, dtype):
    """(R(e), R(e - b), R(e + b)); a non-finite e keeps its own value."""
    b = torch.where(torch.isfinite(e) & torch.isfinite(b), b, torch.zeros_like(b))
    return round_to(e, dtype), round_to(e - b, dtype), round_to(e + b, dtype)


@dataclass
class Adm:
    """An admissible set: the values of [lo, hi] in the output format (lo == hi bitwise: that value alone), and NaN
    where nan; `id` is the single-rounded value."""
    id: Tensor
    lo: Tensor
    hi: Tensor
    nan: Tensor

    @staticmethod
    def of(id: Tensor, corners) -> "Adm":
        c = torch.stack([x.float() for x in corners])
        isn = torch.isnan(c)
        lo = torch.where(isn, float("inf"), c).amin(0)
        hi = torch.where(isn, float("-inf"), c).amax(0)
        none = isn.all(0)
        lo = torch.where(none, float("nan"), lo)
        hi = torch.where(none, float("nan"), hi)
        # signed zero: -0 and +0 corners give [-0, +0]; corners of one value keep its bits
        neg0 = ((c == 0) & (torch.signbit(c))).any(0)
        pos0 = ((c == 0) & ~torch.signbit(c)).any(0)
        lo = torch.where((lo == 0) & neg0, -0.0, lo)
        hi = torch.where((hi == 0) & pos0, 0.0, hi)
        same = (c.view(torch.int32) == c[0:1].view(torch.int32)).all(0)
        lo = torch.where(same, c[0], lo)
        hi = torch.where(same, c[0], hi)
        return Adm(id=id, lo=lo.to(id.dtype), hi=hi.to(id.dtype), nan=isn.any(0))

    def contains(self, y: Tensor) -> Tensor:
        yb, lb, hb = (t.view(torch.int16) for t in (y, self.lo, self.hi))
        single = lb == hb
        yf, lo, hi = y.float(), self.lo.float(), self.hi.float()
        return (torch.isnan(y) & self.nan) | (single & (yb == lb)) | (~single & (yf >= lo) & (yf <= hi))

    def single(self) -> Tensor:
        return self.lo.view(torch.int16) == self.hi.view(torch.int16)

    def width(self) -> Tensor:
        """Steps of the output format from lo to hi (0: one value)."""
        return _ordinal(self.hi) - _ordinal(self.lo)


def _ordinal(x: Tensor) -> Tensor:
    """16-bit float bits -> integers in the order of the values (-0 and +0 adjacent)."""
    b = x.view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF) - 1, b)


def _from_ordinal(o: Tensor, dtype) -> Tensor:
    b = torch.where(o < 0, (-(o + 1)) | 0x8000, o)
    return b.to(torch.int32).to(torch.int16).view(dtype) if dtype != torch.int16 else b


def _tau_exact(xo: Tensor, w: Tensor) -> Tensor:
    """Σ_k xo[m,k] w[o,k] in float64; elementwise when an operand is not finite, so inf·0 and inf - inf give NaN exactly
    as the kernels' fp32 chain does (a GEMM library may not)."""
    if bool(torch.isfinite(xo).all()) and bool(torch.isfinite(w).all()):
        return xo @ w.t()
    return torch.stack([(xo[m].unsqueeze(0) * w).sum(-1) for m in range(xo.shape[0])])


@dataclass
class Int8Exact:
    """int8_linear_exact's result.  Exact parts: xh (fp16 x̂), mask, sca, qs, ca, t (float64).  Per output: v (fp16
    single-rounded dequantised part) and its set [v_lo, v_hi], tau (float64 exact τ) and tau_bound, and `out`, the bf16 output's Adm."""
    xh: Tensor
    mask: Tensor
    sca: Tensor
    qs: Tensor
    ca: Tensor
    t: Tensor
    v: Tensor
    v_lo: Tensor
    v_hi: Tensor
    tau: Tensor
    tau_bound: Tensor
    out: Adm


def int8_linear_exact(x: Tensor, cb: Tensor, scb: Tensor, threshold: float = 6.0, mask: Optional[Tensor] = None) -> Int8Exact:
    """The exact restatement above for x [M, K] (bf16 or fp32 values; after the RMSNorm prologue when there is one)
    against CB [N, K] int8 and SCB [N] fp32.  mask: a given outlier mask (bool [K]) instead of the derived one.  Runs on
    x's device: the float64 contractions of integers are exact in any order below 2^53.  qs is the IEEE quotient, as
    the kernels' 127.0f / SCA (int8_linear's `127.0 / sca` is torch's reciprocal-then-multiply, which can differ by an
    ulp and move a product onto or off a .5 tie)."""
    xh = x.float().half()
    a = xh.float()
    if mask is None:
        mask = (a.abs() >= threshold).any(0)
    mask = mask.to(device=a.device, dtype=torch.bool)
    a_in = a.masked_fill(mask, 0.0)
    sca = a_in.abs().amax(1)
    qs = torch.where(sca > 0, torch.tensor(127.0, dtype=torch.float32, device=a.device) / sca, torch.zeros_like(sca))
    ca = torch.round(a_in * qs.unsqueeze(1)).clamp_(-127, 127).masked_fill_(mask, 0.0)
    t = ca.double() @ cb.double().t() + 0.0   # + 0.0: an all-zero sum is +0, as the kernels' int32 t converts
    scbd = scb.double()
    ev = t * sca.double().unsqueeze(1) * scbd.unsqueeze(0) / 16129.0
    v_id, v_lo, v_hi = _around(ev, ev.abs() * (_gamma(5) + 2.0 ** -48), torch.float16)
    n = int(mask.sum())
    M, N = t.shape
    bf = lambda y: y.float().bfloat16()
    if n == 0:
        tau = torch.zeros(M, N, dtype=torch.float64, device=a.device)
        tb = torch.zeros_like(tau)
        out = Adm.of(bf(v_id), [bf(v_lo), bf(v_hi)])
    else:
        ew = cb[:, mask].double() * scbd.unsqueeze(1) / 127.0
        w = round_to(ew, torch.float16).double()
        wb = ew.abs() * (_gamma(2) + 2.0 ** -48)
        amb = (round_to(ew - wb, torch.float16) != round_to(ew + wb, torch.float16)).double() * ulp16(w)
        xo = a[:, mask].double()
        tau = _tau_exact(xo, w) + 0.0   # the kernels' chain starts from +0
        s1 = _tau_exact(xo.abs(), w.abs())
        s2 = _tau_exact(xo.abs(), amb) if bool(amb.any()) else torch.zeros_like(s1)
        tb = _gamma(n) * (s1 + s2) + s2 + 2.0 ** -40 * s1
        t_id, t_lo, t_hi = _around(tau, tb, torch.float16)
        add = lambda p, q: bf((p.float() + q.float()).half())   # bf16(fp16(fl32(v + fp16(τ))))
        out = Adm.of(add(v_id, t_id), [add(p, q) for p in (v_lo, v_hi) for q in (t_lo, t_hi)])
    return Int8Exact(xh=xh, mask=mask, sca=sca, qs=qs, ca=ca, t=t, v=v_id, v_lo=v_lo, v_hi=v_hi, tau=tau, tau_bound=tb, out=out)


def int8_affine(y: Tensor, s: Tensor, b: Tensor) -> Tensor:
    """LLaMA-Adapter v2's affine on a bf16 linear output: bf16(s · bf16(y + b)) (adapter_v2.py:30-33), exact."""
    return ((y.float() + b.float()).bfloat16().float() * s.float()).bfloat16()


def int8_adm_affine(y: Adm, s: Tensor, b: Tensor) -> Adm:
    f = lambda t: int8_affine(t, s, b)
    r = Adm.of(f(y.id), [f(y.lo), f(y.hi)])   # monotone either way (the sign of s)
    r.nan = r.nan | y.nan
    return r


def int8_adm_residual(y: Adm, res: Tensor) -> Adm:
    f = lambda t: (t.float() + res.float()).bfloat16()
    r = Adm.of(f(y.id), [f(y.lo), f(y.hi)])
    r.nan = r.nan | y.nan
    return r


def _silu_bf16(y1: Tensor):
    """bf16(silu(y1)): (correctly rounded, lowest, highest) over the kernels' fp32 y / (1 + expf(-y)) within 7u and the
    host's own fp32 evaluation of it (which also carries the non-finite cases and expf's overflow below -88.7)."""
    a = y1.double()
    e = a / (1.0 + torch.exp(-a))
    s_id, s_lo, s_hi = _around(e, e.abs() * (7 * INT8_U + 2.0 ** -48), torch.bfloat16)
    y1f = y1.float()
    s_host = (y1f / (1.0 + torch.exp(-y1f))).bfloat16()
    return s_id, [s_lo, s_hi, s_host]


SILU_ARGMIN = -1.2784645   # silu falls below it and rises above it; silu(SILU_ARGMIN) = -0.2784645


def int8_adm_silu_mul(y1: Adm, y2: Adm) -> Adm:
    """SwiGLU's bf16(bf16(silu(y1)) · y2) (model.py:252).  silu is monotone on each side of its minimum, so over y1's
    interval it ranges between its values at the ends, and down to the minimum where the interval straddles it; the
    product is monotone in each factor, so its corners bound it."""
    mul = lambda s, t: (s.float() * t.float()).bfloat16()
    s_id, _ = _silu_bf16(y1.id)
    ends = _silu_bf16(y1.lo)[1] + _silu_bf16(y1.hi)[1]
    straddle = (y1.lo.float() < SILU_ARGMIN) & (y1.hi.float() > SILU_ARGMIN)
    s_min = _silu_bf16(torch.full_like(y1.lo, SILU_ARGMIN, dtype=torch.float64))[1]
    ends += [torch.where(straddle, m.float(), ends[0].float()).bfloat16() for m in s_min]
    s = Adm.of(s_id, ends)
    r = Adm.of(mul(s_id, y2.id), [mul(p, q) for p in (s.lo, s.hi) for q in (y2.lo, y2.hi)])
    r.nan = r.nan | s.nan | y2.nan
    return r


# ----------------------------------------------------------------------------
# The logits tail held exactly: generate.py:68-76 (temperature, top-k, softmax, multinomial) and the next-token NLL of
# evaluate/*.py, as csrc/sampling.cu and csrc/nll.cu compute them
# ----------------------------------------------------------------------------
# Sampling, per row of bf16 logits l [V] at temperature T and top-k k:
#   s_i = bf16(fl32(l_i · fl32(1 / fl32(T))))            ATen's scalar-reciprocal path and the kernel: two roundings
#   thr = the k-th largest s in IEEE order (NaN largest, as torch.topk); kept = {i : !(s_i < thr)}, so -0 and +0 are
#         equal; k = 0 or k >= V keeps every entry
#   gmax = max of the non-NaN s;  d_i = fl32(s_i - gmax) (bit for bit);  p*_i = exp(d_i) / Σ_kept exp(d_j) in float64
# The kernel's p_i = bf16(fl32(expf(d_i) / Σ̂)) lies within ε p*_i of p*_i, with u = 2^-24:
#   expf within 2 ulp (<= 4u relative) in the numerator and in each term of the sum; the sum in the kernel's order,
#   m = 8 ⌈Vp / 8192⌉ sequential terms per thread and then 5 + 5 butterfly levels, γ_{m+10}; one IEEE division, u:
#   ε = (1 + 4u)(1 + u) / ((1 - 4u)(1 - γ_{m+10})) - 1, plus an absolute 2^-147 for expf and the division where they
#   return fp32 subnormals.  A probability's admissible set is [bf16(p* - b), bf16(p* + b)], one value away from bf16
#   midpoints; the single-rounded value is round_to(p*, bf16).
# Special cases, as torch's op sequence defines them: a NaN among the kept s (a NaN logit) or a +inf kept (the scaled
# logits overflow, inf - inf) makes the softmax NaN.  Contract for such a row: every kept entry above -inf is NaN, every
# other entry 0 (the filter removed it, or exp(-inf) is 0, before the softmax; torch spreads the NaN over them as well),
# and the draw is the first NaN entry, as torch.argmax(p / q) ranks NaN first.  A kept -inf has probability 0.  A row with no kept value above
# -inf has no distribution (torch: NaN); the kernel writes zeros and draws token 0, and the oracle states exactly that.
SAMP_THREADS = 1024


def _samp_eps(V: int) -> float:
    vp = (V + 7) // 8 * 8
    m = 8 * (-(-vp // (8 * SAMP_THREADS)))
    u = INT8_U
    return (1 + 4 * u) * (1 + u) / ((1 - 4 * u) * (1 - _gamma(m + 10))) - 1 + 2.0 ** -48


@dataclass
class TopkExact:
    """topk_softmax_exact's result for logits [..., V]: the scaled bf16 values, the threshold (fp32; -inf: no filter),
    the kept mask, gmax, d (fp32, bit for bit), p* (float64), the bound b and `probs`, the bf16 probabilities' Adm."""
    scaled: Tensor
    thr: Tensor
    kept: Tensor
    gmax: Tensor
    d: Tensor
    p: Tensor
    bound: Tensor
    probs: Adm


def topk_softmax_exact(logits: Tensor, temperature: float, top_k: int) -> TopkExact:
    lf = logits.float()
    V = lf.shape[-1]
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(temperature, dtype=torch.float32)
    s = (lf * inv).bfloat16()
    sf = s.float()
    if 0 < top_k < V:
        thr = torch.topk(sf, top_k, dim=-1).values[..., -1:]
    else:
        thr = torch.full_like(sf[..., :1], float("-inf"))
    kept = ~(sf < thr)
    gmax = torch.where(torch.isnan(sf), float("-inf"), sf).amax(-1, keepdim=True)
    d = sf - gmax
    dd = d.double()
    e = torch.where(kept & (sf != float("-inf")), torch.exp(dd), torch.zeros_like(dd))
    tot = e.sum(-1, keepdim=True)
    nan_row = torch.isnan(tot)
    p = e / tot
    eps = _samp_eps(V)
    b = p.abs() * eps + 2.0 ** -147
    b = torch.where(torch.isfinite(p), b, torch.zeros_like(b))
    lo = round_to(torch.clamp(p - b, min=0.0), torch.bfloat16)
    hi = round_to(p + b, torch.bfloat16)
    pid = round_to(p, torch.bfloat16)
    # the contracts above: NaN rows keep NaN at kept entries and 0 at filtered ones; rows with nothing above -inf are 0
    zero = torch.zeros_like(pid)
    empty = (tot == 0) & ~nan_row
    nan_kept = nan_row & kept & (sf != float("-inf"))
    nanv = torch.full_like(pid, float("nan"))
    fix = lambda t: torch.where(nan_kept, nanv, torch.where((nan_row & ~kept) | empty, zero, t))
    probs = Adm.of(fix(pid), [fix(lo), fix(hi)])
    return TopkExact(scaled=s, thr=thr, kept=kept, gmax=gmax, d=d, p=p, bound=b, probs=probs)


def draw_exact(probs: Tensor, q: Tensor) -> Tensor:
    """torch.multinomial(probs, 1) as argmax(probs / q) on bf16 tensors: r = bf16(fl32(p / q)), the first maximum, with
    NaN ranked above everything (torch.argmax's rule).  Exact given the probabilities.  int64 [...]."""
    r = (probs.float() / q.float()).bfloat16().float()
    isn = torch.isnan(r)
    V = r.shape[-1]
    idx = torch.arange(V).expand_as(r)
    first_nan = torch.where(isn, idx, V).amin(-1)
    rr = torch.where(isn, float("-inf"), r)
    top = rr.amax(-1, keepdim=True)
    first_max = torch.where(rr == top, idx, V).amin(-1)
    return torch.where(isn.any(-1), first_nan, first_max).to(torch.int64)


# Next-token NLL (nll.cu / nll_common.cuh / the NLL epilogue of q4_gemm.cu) of bf16 logits L [M, N] against targets t:
#   nll_m = logsumexp_n L[m, n] - L[m, t_m], computed as: per 128-column tile j, mx_j = max and
#   s_j = Σ_i expf(fl32(v_i - mx_j)) (each lane 32 sequential terms, then 2 butterfly adds); the combine
#   mx = max_j mx_j, ŝ = Σ_j fl32(s_j · expf(fl32(mx_j - mx))) sequentially over the n_tiles tiles; then
#   fl32(fl32(mx + logf(ŝ)) - L[m, t]).  A tile whose columns are all -inf contributes s_j = 0.
# Absolute bound, u = 2^-24, E_j = Σ_i e^{d_ij}, A_j = Σ_i |d_ij| e^{d_ij}, w_j = e^{Δ_j}, Δ_j = mx_j - mx:
#   a rounded difference d(1 + δ) moves e^d by at most u |d| e^d; expf 4u; the tile sum γ_34; the product u; the
#   combine sum γ_{n_tiles}:  |ŝ - S| <= (γ_34 + 9u + γ_{n_tiles}) S + u Σ_j w_j (A_j + |Δ_j| E_j)  (first order, ×1.01);
#   logf within 1 ulp (<= 2u |log ŝ|), |log ŝ - log S| <= ρ / (1 - ρ), ρ = |ŝ - S| / S; then the roundings of
#   mx + log ŝ and of the final subtraction, u each.
# NaN where torch's cross_entropy gives NaN: a NaN or +inf logit in the row, an all -inf row, a target outside
# 0..N-1; +inf where the target's logit is -inf (and the row has a finite logit).
NLL_TILE = 128


@dataclass
class NLLExact:
    """nll_exact's result: nll (float64 [M], NaN / +inf in the special cases) and bound (float64 [M], 0 there)."""
    nll: Tensor
    bound: Tensor


def nll_exact(logits: Tensor, targets: Tensor) -> NLLExact:
    Lf = logits.double()
    M, N = Lf.shape
    t = targets.long().view(-1)
    nt = -(-N // NLL_TILE)
    pad = torch.full((M, nt * NLL_TILE - N), float("-inf"), dtype=torch.float64)
    T = torch.cat([Lf, pad], 1).view(M, nt, NLL_TILE)
    u = INT8_U
    fin = torch.where(torch.isnan(T), float("-inf"), T)
    mxj = fin.amax(-1)                                   # [M, nt]
    live = mxj > float("-inf")
    mxj0 = torch.where(live, mxj, torch.zeros_like(mxj))
    dij = torch.where(T > float("-inf"), T - mxj0.unsqueeze(-1), torch.full_like(T, float("-inf")))
    eij = torch.exp(dij)
    Ej = eij.sum(-1)
    Aj = torch.where(eij > 0, dij.abs() * eij, torch.zeros_like(eij)).sum(-1)
    mx = mxj.amax(-1, keepdim=True)
    mx0 = torch.where(mx > float("-inf"), mx, torch.zeros_like(mx))
    dj = torch.where(live, mxj - mx0, torch.full_like(mxj, float("-inf")))
    wj = torch.exp(dj)
    S = (wj * Ej).sum(-1)
    err_s = (_gamma(34) + 9 * u + _gamma(nt)) * S + u * (wj * (Aj + torch.where(live, dj.abs(), torch.zeros_like(dj)) * Ej)).sum(-1)
    err_s = err_s * 1.01 + 2.0 ** -140 * N
    lnS = torch.log(S)
    rho = err_s / S
    rho = rho / (1 - rho)
    ls_err = rho + 2 * u * (lnS.abs() + rho)
    mxv = mx.squeeze(-1)
    a = (mxv + lnS).abs() + ls_err
    r_err = ls_err + u * a * (1 + u)
    ok_t = (t >= 0) & (t < N)
    lt = Lf.gather(1, t.clamp(0, N - 1).view(-1, 1)).squeeze(1)
    nll = mxv + lnS - lt
    bound = (r_err + u * (nll.abs() + r_err)) * (1 + 1e-9)
    bad = torch.isnan(Lf).any(1) | (Lf == float("inf")).any(1) | ~(Lf > float("-inf")).any(1) | ~ok_t
    nll = torch.where(bad, float("nan"), torch.where(lt == float("-inf"), float("inf"), nll))
    bound = torch.where(torch.isfinite(nll), bound, torch.zeros_like(bound))
    return NLLExact(nll=nll, bound=bound)


# ----------------------------------------------------------------------------
# lit_llama/model.py
# ----------------------------------------------------------------------------
def rmsnorm(x: Tensor, scale: Tensor, eps: float = 1e-5) -> Tensor:
    """RMSNorm.forward, model.py:270-277, evaluated in x.dtype with no upcast:
    mean(x*x) -> +eps -> rsqrt -> x*that -> scale*that."""
    ms = torch.mean(x * x, dim=-1, keepdim=True)
    return scale * (x * torch.rsqrt(ms + eps))


def rope_table(seq_len: int, n_elem: int, base: int = 10000) -> Tensor:
    """build_rope_cache, model.py:280-303, for the integer-`idx` call made by
    LLaMA.forward (model.py:128-134): fp32 (seq_len, n_elem/2, 2) of (cos, sin)."""
    theta = 1.0 / (base ** (torch.arange(0, n_elem, 2, dtype=torch.float32) / n_elem))
    ang = torch.outer(torch.arange(seq_len, dtype=torch.float32), theta)
    return torch.stack((torch.cos(ang), torch.sin(ang)), dim=-1)


def rope_apply(x: Tensor, rows: Tensor) -> Tensor:
    """apply_rope, model.py:306-323.  x (B,T,nh,hs); rows (T,hs/2,2) fp32.
    Interleaved pairs rotate in fp32, result cast back to x.dtype."""
    B, T, nh, hs = x.shape
    xp = x.float().reshape(B, T, nh, hs // 2, 2)
    c = rows[:T, :, 0].reshape(1, T, 1, hs // 2)
    s = rows[:T, :, 1].reshape(1, T, 1, hs // 2)
    even = xp[..., 0] * c - xp[..., 1] * s
    odd = xp[..., 1] * c + xp[..., 0] * s
    return torch.stack((even, odd), dim=-1).reshape(B, T, nh, hs).to(x.dtype)


def sdpa(q: Tensor, k: Tensor, v: Tensor, mask: Tensor) -> Tensor:
    """model.py:230 semantics: softmax(q k^T / sqrt(hs) masked) v.  Evaluated in
    fp32 from the stored-dtype operands, one rounding to q.dtype at the end."""
    att = (q.float() @ k.float().transpose(-2, -1)) * (1.0 / math.sqrt(q.size(-1)))
    att = att.masked_fill(~mask, float("-inf"))
    return (torch.softmax(att, dim=-1) @ v.float()).to(q.dtype)


@dataclass
class QLin:
    """One linear layer of the model in whichever storage the mode uses."""
    kind: str  # "dense" | "gptq" | "gptq_exact" | "int8"
    weight: Optional[Tensor] = None  # dense
    qw: Optional[Tensor] = None
    scales: Optional[Tensor] = None
    zeros: Optional[Tensor] = None
    bits: int = 4
    tile_cols: int = -1
    cb: Optional[Tensor] = None
    scb: Optional[Tensor] = None

    def __call__(self, x: Tensor) -> Tensor:
        if self.kind == "dense":
            return torch.nn.functional.linear(x, self.weight)
        if self.kind == "gptq":
            return qlinear(x, self.qw, self.scales, self.zeros, self.bits, self.tile_cols)
        if self.kind == "gptq_exact":  # arithmetic of the reference's GPU kernel: fp32 dequant, fp32+ accumulate
            return qlinear_exact(x, self.qw, self.scales, self.zeros, self.bits, self.tile_cols).to(x.dtype)
        return int8_linear(x, self.cb, self.scb)


@dataclass
class OracleLLaMA:
    """Functional restatement of lit_llama.model.LLaMA for inference with a KV cache."""
    n_layer: int
    n_head: int
    n_embd: int
    block_size: int
    padded_vocab_size: int
    wte: Tensor
    lm_head: QLin
    ln_f: Tensor
    layers: List[Dict[str, object]]  # keys: rms_1, rms_2 (Tensor); c_attn, c_proj, c_fc1, c_fc2, mlp_proj (QLin)
    rope: Optional[Tensor] = None
    kv: List[Tuple[Tensor, Tensor]] = field(default_factory=list)

    @staticmethod
    def from_state_dict(sd: Dict[str, Tensor], n_layer: int, n_head: int, block_size: int,
                        mode: Optional[str] = None, exact_linears: bool = False) -> "OracleLLaMA":
        """Builds from a reference-format state dict (keys as produced by
        lit_llama.model.LLaMA under utils.quantization(mode)).  `exact_linears` selects the
        arithmetic of the reference's GPU branch (quantization.py:259-269: fp32 dequant and
        accumulate, no per-weight bf16 rounding) instead of its dense CPU branch (:392-423)."""

        def lin(prefix: str) -> QLin:
            if prefix + ".quant_weight" in sd:
                qw = sd[prefix + ".quant_weight"]
                sc = sd[prefix + ".scales"]
                bits = 4 if mode in (None, "gptq.int4") else 8
                epb = 8 // bits
                in_features = qw.shape[1] * epb
                n_groups = sc.shape[1]
                tile_cols = in_features if n_groups == 1 else -(-in_features // n_groups)
                return QLin("gptq_exact" if exact_linears else "gptq", qw=qw, scales=sc, zeros=sd[prefix + ".zeros"], bits=bits,
                            tile_cols=tile_cols)
            w = sd[prefix + ".weight"]
            if mode == "llm.int8":
                cb, scb = int8_quantize_weight(w)
                return QLin("int8", cb=cb, scb=scb)
            return QLin("dense", weight=w)

        wte = sd["transformer.wte.weight"]
        layers = []
        for i in range(n_layer):
            p = f"transformer.h.{i}."
            layers.append(dict(
                rms_1=sd[p + "rms_1.scale"], rms_2=sd[p + "rms_2.scale"],
                c_attn=lin(p + "attn.c_attn"), c_proj=lin(p + "attn.c_proj"),
                c_fc1=lin(p + "mlp.c_fc1"), c_fc2=lin(p + "mlp.c_fc2"), mlp_proj=lin(p + "mlp.c_proj"),
            ))
        return OracleLLaMA(n_layer=n_layer, n_head=n_head, n_embd=wte.shape[1], block_size=block_size,
                           padded_vocab_size=wte.shape[0], wte=wte, lm_head=lin("lm_head"),
                           ln_f=sd["transformer.ln_f.scale"], layers=layers)

    def reset_cache(self) -> None:
        """model.py:140-145."""
        self.kv = []

    def _attn(self, x: Tensor, lay, rope: Tensor, mask: Tensor, S: int, input_pos: Optional[Tensor], li: int) -> Tensor:
        """CausalSelfAttention.forward, model.py:185-237."""
        B, T, C = x.shape
        hs = C // self.n_head
        q, k, v = lay["c_attn"](x).split(C, dim=2)
        q = rope_apply(q.view(B, T, self.n_head, hs), rope).transpose(1, 2)
        k = rope_apply(k.view(B, T, self.n_head, hs), rope).transpose(1, 2)
        v = v.view(B, T, self.n_head, hs).transpose(1, 2)
        if input_pos is not None:
            ck, cv = self.kv[li]
            if int(input_pos[-1]) >= S:  # model.py:214-218: sliding window by one slot
                input_pos = torch.tensor(S - 1)
                ck = torch.roll(ck, -1, dims=2)
                cv = torch.roll(cv, -1, dims=2)
            k = ck.index_copy(2, input_pos.reshape(-1), k)
            v = cv.index_copy(2, input_pos.reshape(-1), v)
            self.kv[li] = (k, v)
        y = sdpa(q, k, v, mask)
        return lay["c_proj"](y.transpose(1, 2).contiguous().view(B, T, C))

    def forward(self, idx: Tensor, max_seq_length: Optional[int] = None, input_pos: Optional[Tensor] = None) -> Tensor:
        """LLaMA.forward, model.py:76-122 (+ Block.forward :156-168, MLP.forward :251-254)."""
        B, T = idx.shape
        S = self.block_size if max_seq_length is None else max_seq_length
        assert T <= S <= self.block_size
        hs = self.n_embd // self.n_head
        if self.rope is None:
            self.rope = rope_table(self.block_size, hs)
        tril = torch.tril(torch.ones(self.block_size, self.block_size, dtype=torch.bool))
        if input_pos is not None:
            rope = self.rope.index_select(0, input_pos)
            mask = tril.index_select(0, input_pos)[:, :S].reshape(1, 1, T, S)
        else:
            rope = self.rope[:T]
            mask = tril[:T, :T].reshape(1, 1, T, T)
        x = self.wte[idx]
        if input_pos is not None and not self.kv:
            shape = (B, self.n_head, S, hs)
            self.kv = [(torch.zeros(shape, dtype=x.dtype), torch.zeros(shape, dtype=x.dtype)) for _ in range(self.n_layer)]
        for li, lay in enumerate(self.layers):
            x = x + self._attn(rmsnorm(x, lay["rms_1"]), lay, rope, mask, S, input_pos, li)
            h = rmsnorm(x, lay["rms_2"])
            x = x + lay["mlp_proj"](torch.nn.functional.silu(lay["c_fc1"](h)) * lay["c_fc2"](h))
        return self.lm_head(rmsnorm(x, self.ln_f))


def generate(model, idx: Tensor, max_new_tokens: int, *, max_seq_length: Optional[int] = None,
             temperature: float = 1.0, top_k: Optional[int] = None, eos_id: Optional[int] = None) -> Tensor:
    """generate.py:20-91.  `model` needs .forward(idx, max_seq_length, input_pos)
    and .block_size.  Sampling uses torch.multinomial so the RNG stream is the
    reference's."""
    T = idx.size(0)
    T_new = T + max_new_tokens
    if max_seq_length is None:
        max_seq_length = min(T_new, model.block_size)
    out = torch.empty(T_new, dtype=idx.dtype)
    out[:T] = idx
    input_pos = torch.arange(0, T)
    for _ in range(max_new_tokens):
        x = out.index_select(0, input_pos).view(1, -1)
        logits = model.forward(x, max_seq_length, input_pos)[0, -1] / temperature
        if top_k is not None:
            v, _ = torch.topk(logits, min(top_k, logits.size(-1)))
            logits = torch.where(logits < v[[-1]], -float("inf"), logits)
        probs = torch.softmax(logits, dim=-1)
        nxt = torch.multinomial(probs, num_samples=1).to(dtype=idx.dtype)
        input_pos = input_pos[-1:] + 1
        out = out.index_copy(0, input_pos, nxt)
        if eos_id is not None and int(nxt) == eos_id:
            return out[: int(input_pos)]
    return out


# ----------------------------------------------------------------------------
# Synthetic weights (SURVEY.md section 8d) - shared by tests, smoke and bench
# ----------------------------------------------------------------------------
def synth_state_dict(n_layer: int, n_head: int, n_embd: int, vocab_size: int, mode: Optional[str],
                     dtype=torch.bfloat16, seed: int = 1234, tile_cols: int = -1) -> Dict[str, Tensor]:
    """Random-init weights with the reference initialiser's statistics
    (model.py:70-74: N(0, 0.02/sqrt(2 n_layer))), RMSNorm scales near 1, quantised
    round-to-nearest with the reference formulas (rtn_params / rtn_levels /
    pack_levels).  Keys, shapes, dtypes and strides match what the reference model
    holds under utils.quantization(mode)."""
    g = torch.Generator().manual_seed(seed)
    std = 0.02 / math.sqrt(2 * n_layer)
    V = find_multiple(vocab_size, 64)
    nh = n_hidden_for(n_embd)
    sd: Dict[str, Tensor] = {}

    def put_linear(prefix: str, out_f: int, in_f: int) -> None:
        w = torch.randn(out_f, in_f, generator=g) * std
        if mode in ("gptq.int4", "gptq.int8"):
            bits = 4 if mode == "gptq.int4" else 8
            tc = in_f if tile_cols == -1 else tile_cols
            ng = -(-in_f // tc)
            scales = torch.empty(out_f, ng)
            zeros = torch.empty(out_f, ng)
            lv = torch.empty(out_f, in_f)
            for gi in range(ng):
                sl = slice(gi * tc, (gi + 1) * tc)
                s, z = rtn_params(w[:, sl], bits)
                s = s.to(dtype).float()  # the stored scale is what every consumer sees
                scales[:, gi : gi + 1], zeros[:, gi : gi + 1] = s, z
                lv[:, sl] = rtn_levels(w[:, sl], s, z, bits)
            sd[prefix + ".quant_weight"] = pack_levels(lv, bits)
            sd[prefix + ".scales"] = scales.to(dtype)
            sd[prefix + ".zeros"] = zeros.to(dtype)
        else:
            sd[prefix + ".weight"] = w.to(dtype)

    put_linear("lm_head", V, n_embd)
    sd["transformer.wte.weight"] = (torch.randn(V, n_embd, generator=g) * 0.02).to(dtype)
    for i in range(n_layer):
        p = f"transformer.h.{i}."
        sd[p + "rms_1.scale"] = (1.0 + 0.1 * torch.randn(n_embd, generator=g)).to(dtype)
        put_linear(p + "attn.c_attn", 3 * n_embd, n_embd)
        put_linear(p + "attn.c_proj", n_embd, n_embd)
        sd[p + "rms_2.scale"] = (1.0 + 0.1 * torch.randn(n_embd, generator=g)).to(dtype)
        put_linear(p + "mlp.c_fc1", nh, n_embd)
        put_linear(p + "mlp.c_fc2", nh, n_embd)
        put_linear(p + "mlp.c_proj", n_embd, nh)
    sd["transformer.ln_f.scale"] = (1.0 + 0.1 * torch.randn(n_embd, generator=g)).to(dtype)
    return sd

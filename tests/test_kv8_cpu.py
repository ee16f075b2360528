"""CPU: the fp8 KV cache.  b2l_kv8_cache, b2l_attention_kv8 and b2l_decode_args::kv8 against the header (ctypes
binding, struct layout, every existing offset unchanged), their refusals before any launch, LLaMA.kv_cache_dtype, and
the number format of include/b2l.h restated here (`kv8_quantize`) against torch.float8_e4m3fn on ties, the 448
boundary, subnormal codes, all-zero vectors, the bf16 extremes and non-finite inputs.

The restatement: amax = max |x_i|; e = 0 when amax == 0, else the smallest integer with amax 2^-e <= 448, raised to
-124; code_i = e4m3(x_i 2^-e) rounded to nearest even; scale = 2^e; the value read back is float(code_i) * scale in
fp32.  A vector with a non-finite element is stored as NaN codes (0x7f) and a NaN scale.  The e4m3 rounding here is
computed on the e4m3 grid in float64 (round half to even of x / quantum), not by torch."""
import ctypes as C
import math
import os
import subprocess

import pytest
import torch

import __graft_entry__ as entry
import lit_llama_b200 as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_MIN = -124


def kv8_exponent(amax: float) -> int:
    """The scale exponent of a vector with largest magnitude amax (finite)."""
    if amax == 0.0:
        return 0
    m, ex = math.frexp(amax)                 # amax = m 2^ex, m in [0.5, 1)
    e = ex - 9 if m <= 0.875 else ex - 8     # (2 m) 2^8 <= 448, else one binade up
    assert amax * 2.0 ** -e <= 448 < amax * 2.0 ** -(e - 1)
    return max(e, E_MIN)


def e4m3_rne(y: float) -> float:
    """y (|y| <= 448) rounded to nearest even on the e4m3fn grid, as a float."""
    a = abs(y)
    if a == 0.0:
        return math.copysign(0.0, y)
    quantum = 2.0 ** -9 if a < 2.0 ** -6 else 2.0 ** (math.frexp(a)[1] - 1 - 3)   # 3 mantissa bits
    q = a / quantum                                                               # exact
    r = math.floor(q)
    if q - r > 0.5 or (q - r == 0.5 and r % 2 == 1):
        r += 1
    return math.copysign(r * quantum, y)


def kv8_quantize(x: torch.Tensor):
    """x bf16 [..., hs] -> (values e4m3fn codes as float64 [..., hs], scale float64 [...], read-back float32 [..., hs])."""
    xs = x.double().reshape(-1, x.shape[-1])
    codes, scales = torch.empty_like(xs), torch.empty(xs.shape[0], dtype=torch.float64)
    for r in range(xs.shape[0]):
        row = xs[r].tolist()
        if not all(math.isfinite(v) for v in row):
            codes[r] = math.nan
            scales[r] = math.nan
            continue
        e = kv8_exponent(max(abs(v) for v in row))
        scales[r] = 2.0 ** e
        codes[r] = torch.tensor([e4m3_rne(v * 2.0 ** -e) for v in row], dtype=torch.float64)
    back = (codes.float() * scales.float().unsqueeze(-1))
    sh = x.shape
    return codes.view(sh), scales.view(sh[:-1]), back.view(sh)


def _torch_codes(x: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """torch's e4m3fn conversion of x 2^-e (fp32 product), as the float value of each code."""
    inv = torch.where(torch.isfinite(scales), 1.0 / scales, torch.ones_like(scales)).float()
    return (x.float() * inv.unsqueeze(-1)).to(torch.float8_e4m3fn).double()


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Equal including the sign of zero, NaN equal to NaN."""
    a, b = a.double(), b.double()
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((a == b) & (torch.signbit(a) == torch.signbit(b)) | nan).all())


def _vec(vals, hs=128, fill=0.0):
    x = torch.full((hs,), fill, dtype=torch.float64)
    x[:len(vals)] = torch.tensor(vals, dtype=torch.float64)
    return x.bfloat16()


BF16_MAX = float(torch.finfo(torch.bfloat16).max)
CASES = {
    # amax 448 (e = 0): exact e4m3 ties round to the even neighbour, in every binade and among subnormals
    "ties": _vec([448.0, 1.0625, 1.1875, -1.3125, 17.0, 19.0, -288.0, 2.0 ** -10, 3 * 2.0 ** -10, -5 * 2.0 ** -10,
                  2.0 ** -6 + 2.0 ** -10, 0.01171875]),
    "ties_scaled": _vec([448.0 * 2.0 ** -20, 1.0625 * 2.0 ** -20, 19.0 * 2.0 ** -20, -288.0 * 2.0 ** -20]),
    # the 448 boundary: 448 stays at e = 0, the next bf16 value (450) moves to e = 1; 448 2^k -> e = k
    "at_448": _vec([448.0, -447.0, 100.0]),
    "above_448": _vec([450.0, 448.0, -449.0]),
    "448_times_2^40": _vec([448.0 * 2.0 ** 40, 3.0 * 2.0 ** 40]),
    "just_below_2^9": _vec([510.0, 1.0]),
    # subnormal codes next to a large element
    "subnormal_codes": _vec([448.0] + [k * 2.0 ** -9 for k in range(1, 8)] + [-(k + 0.5) * 2.0 ** -9 for k in range(8)]),
    "zero": _vec([]),
    "signed_zero": _vec([-0.0, 0.0, -0.0]),
    # bf16 extremes: the largest finite value (reads back as inf: the one inexact read-back), the smallest normal and
    # subnormal, a vector of subnormals only (e = -124: 2^-133 is code 2^-9)
    "bf16_max": _vec([BF16_MAX, -1.875 * 2.0 ** 127, 1.0]),
    "bf16_min_normal": _vec([2.0 ** -126, -2.0 ** -126, 2.0 ** -127]),
    "bf16_subnormals": _vec([2.0 ** -133, -2.0 ** -133, 3 * 2.0 ** -133, 2.0 ** -127]),
    "randn": (torch.randn(128, generator=torch.Generator().manual_seed(0)) * 3).bfloat16(),
    "massive": _vec([1000.0, -0.001, 3.0, 0.5]),
    "nan": _vec([1.0, math.nan, 2.0]),
    "inf": _vec([1.0, -math.inf, 2.0]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_quantizer_restatement_agrees_with_torch_e4m3fn(case):
    x = CASES[case]
    codes, scale, back = kv8_quantize(x)
    if case in ("nan", "inf"):
        assert bool(torch.isnan(codes).all()) and math.isnan(float(scale)) and bool(torch.isnan(back).all())
        return
    e = math.frexp(float(scale))[1] - 1
    assert float(scale) == 2.0 ** e and E_MIN <= e <= 120
    # torch's conversion of the scaled inputs agrees code for code (sign of zero included)
    assert _same(codes, _torch_codes(x, scale)), case
    assert bool((codes.abs() <= 448).all())
    # the read-back value is float(code) * scale, exact in fp32, and a bf16 number -- except at the top of the bf16
    # range, where a code of 256+ at e = 120 overflows
    want = codes * float(scale)
    finite = want.abs() < 2.0 ** 128
    assert _same(back.double()[finite], want[finite])
    assert bool(torch.isinf(back[~finite]).all())
    assert _same(back[finite].bfloat16().double(), back[finite].double())
    # every nonzero input reads back nonzero (E_MIN maps the smallest bf16 subnormal onto the smallest e4m3 subnormal)
    # unless it is at most half an e4m3 subnormal of this vector's scale (the tie rounds to the even zero)
    tiny = x.double().abs() <= 2.0 ** -10 * float(scale)
    assert bool(((x.double() == 0) | tiny | (back.double() != 0)).all())


def test_exponent_and_boundaries():
    assert kv8_exponent(448.0) == 0 and kv8_exponent(450.0) == 1 and kv8_exponent(224.0) == -1
    assert kv8_exponent(0.0) == 0 and kv8_exponent(2.0 ** -133) == E_MIN and kv8_exponent(2.0 ** -116) == E_MIN
    assert kv8_exponent(BF16_MAX) == 120
    assert kv8_quantize(CASES["bf16_subnormals"])[2][0].item() == 2.0 ** -133
    assert kv8_quantize(CASES["zero"])[1].item() == 1.0
    # scaling the input by 2^k moves the exponent by k and leaves the codes (away from the E_MIN clamp)
    x = CASES["randn"]
    c0, s0, _ = kv8_quantize(x)
    for k in (-30, -1, 1, 17):
        c, s, _ = kv8_quantize((x.double() * 2.0 ** k).bfloat16())
        assert _same(c, c0) and float(s) == float(s0) * 2.0 ** k


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_binding_and_layout_match_the_header(L, tmp_path):
    """b2l_kv8_cache and the kv8 member appended to b2l_decode_args agree with the C compiler; the offsets of
    b2l_decode_args are pinned (kv8 sits behind lora_row_set, the last field before it); the prototypes bind."""
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "typedef int (*att_t)(void*, const b2l_kv8_cache*, const void*, const int64_t*, const int32_t*, void*, void*, int,"
        " int, int, int, int, int, int, const b2l_adapter_prefix*, b2l_stream_t);\n"
        "typedef int (*unroll_t)(const void*, const float*, const int32_t*, void*, int, int, int, int, b2l_stream_t);\n"
        "int main(void){ att_t a = b2l_attention_kv8; unroll_t u = b2l_kv8_unroll, r = b2l_kv8_unroll_rows;\n"
        "(void)a; (void)u; (void)r;\n"
        'printf("%zu %zu %zu %zu %zu %zu %zu %zu %d\\n", sizeof(b2l_kv8_cache), offsetof(b2l_kv8_cache, v), '
        "offsetof(b2l_kv8_cache, k_scale), offsetof(b2l_kv8_cache, v_scale), sizeof(b2l_decode_args), "
        "offsetof(b2l_decode_args, kv8), offsetof(b2l_decode_args, lora_row_set), offsetof(b2l_decode_args, flags), "
        "B2L_F_KV_FP8);\nreturn 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(prog), "-o", str(exe) + ".o"],
                   check=True)
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe), "-Wl,--unresolved-symbols=ignore-all"],
                   check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    K, D = L.KV8Cache, L.DecodeArgs
    assert out == [C.sizeof(K), K.v.offset, K.k_scale.offset, K.v_scale.offset, C.sizeof(D), D.kv8.offset,
                   D.lora_row_set.offset, D.flags.offset, L.F_KV_FP8]
    # b2l_decode_args ends with kv8: 336 bytes, lora_row_set at 320, flags at 200
    assert (D.lora_row_set.offset, D.flags.offset, D.kv8.offset) == (320, 200, 328) and C.sizeof(D) == 336
    assert L.F_KV_FP8 == 32768
    fn = L._SIGS["b2l_attention_kv8"]
    assert fn[0] is C.c_int and len(fn[1]) == 16 and fn[1][1] is C.POINTER(L.KV8Cache)


P16 = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its checks


def _kv(L, **kw):
    a = dict(k=P16, v=P16 + 4096, k_scale=P16 + 8192, v_scale=P16 + 12288)
    a.update(kw)
    return L.KV8Cache(**a)


def test_attention_kv8_refuses_before_any_launch(L):
    lib = L.lib()

    def call(kv=None, input_pos=P16, B=2, T=1, nh=4, hs=128, S=64, block=64, flags=0, prefix=None, **ptr):
        p = dict(qkv=P16, rope=P16, ring=P16, y=P16, work=P16)
        p.update(ptr)
        kv = _kv(L) if kv is None else kv
        rc = lib.b2l_attention_kv8(p["qkv"], C.byref(kv), p["rope"], input_pos, p["ring"], p["y"], p["work"], B, T, nh, hs,
                                   S, block, flags, prefix, None)
        return rc, lib.b2l_last_error().decode()

    for kw, code, words in [
        (dict(hs=64), -2, ["head_size 128"]),
        (dict(hs=256), -2, ["head_size 128"]),
        (dict(flags=L.F_STEPWISE), -2, ["B2L_F_STEPWISE"]),
        (dict(flags=8), -2, ["B2L_F_ATTN_UNFUSED"]),
        (dict(flags=L.F_ROPE_ROWS), -2, ["B2L_F_ROPE_ROWS"]),
        (dict(T=5), -2, ["T > 1", "nonzero position"]),                 # a prefill with positions
        (dict(T=5, input_pos=None, flags=L.F_ROW_POS), -2, ["B2L_F_ROW_POS"]),
        (dict(input_pos=None), -1, ["input_pos"]),
        (dict(kv=_kv(L, k_scale=None)), -1, ["null fp8 cache"]),
        (dict(kv=_kv(L, v=P16 + 8)), -1, ["16-byte aligned"]),
        (dict(qkv=None), -1, ["null pointer"]),
        (dict(T=65, input_pos=None), -1, ["bad shape"]),
        (dict(prefix=C.byref(L.AdapterPrefix(P16, P16, P16, 65))), -2, ["adapter prefix length"]),
    ]:
        rc, msg = call(**kw)
        assert rc == code and "b2l_attention_kv8" in msg and all(w in msg for w in words), (kw, rc, msg)


def _decode(L, n_layer=2, B=4, n_head=4, n_embd=512, **kw):
    layers = (L.Layer * n_layer)()
    kv8 = (L.KV8Cache * n_layer)(*[_kv(L) for _ in range(n_layer)])
    d = L.DecodeArgs(n_layer=n_layer, n_head=n_head, n_embd=n_embd, n_hidden=2048, vocab=128, B=B, S=64, layers=layers,
                     wte=16, ln_f=16, rope=16, idx=16, input_pos=16, ring_start=16, block_size=64, x=16, qkv=16, att=16,
                     hid=16, attn_work=16, logits=16, flags=L.F_PDL | L.F_ROW_POS | L.F_KV_FP8,
                     kv8=C.cast(kv8, C.POINTER(L.KV8Cache)))
    for k, v in kw.items():
        setattr(d, k, v)
    d._keep = [layers, kv8]
    return d


def test_decode_step_refusals(L):
    lib = L.lib()

    def refused(code, *words, **kw):
        rc = lib.b2l_decode_step(C.byref(_decode(L, **kw)), None)
        msg = lib.b2l_last_error().decode()
        assert rc == code and "b2l_decode_step" in msg and all(w in msg for w in words), (kw.keys(), rc, msg)

    refused(-2, "B2L_F_KV_FP8", "B2L_F_STEPWISE", flags=L.F_PDL | L.F_STEPWISE | L.F_KV_FP8 | L.F_Q4_BATCH_I8,
            batch_work=P16)
    refused(-2, "B2L_F_ATTN_UNFUSED", flags=L.F_PDL | L.F_KV_FP8 | 8)
    refused(-2, "head_size 128", n_head=8)
    refused(-1, "kv8", kv8=None)
    # the launch count is the fused attention's (one launch per layer)
    assert lib.b2l_decode_step_launches(C.byref(_decode(L))) == lib.b2l_decode_step_launches(
        C.byref(_decode(L, flags=L.F_PDL | L.F_ROW_POS)))


def test_kv_cache_dtype_is_read_at_allocation():
    m = P.LLaMA(P.LLaMAConfig(block_size=16, vocab_size=64, n_layer=1, n_head=1, n_embd=128))
    assert m.kv_cache_dtype is None
    with pytest.raises(ValueError, match="'fp16'"):
        m.kv_cache_dtype = "fp16"
    m.kv_cache_dtype = "fp8"
    m._new_kv_store(2, 16, torch.device("cpu"))
    c = m.kv_caches[0]
    k, v = c
    assert isinstance(c, P.model.FP8KVCache) and k.dtype == torch.float8_e4m3fn and tuple(k.shape) == (2, 1, 16, 128)
    assert c.k_scale.dtype == torch.float32 and tuple(c.v_scale.shape) == (2, 1, 16)
    with pytest.raises(RuntimeError, match="reset_cache"):
        m.kv_cache_dtype = None
    m.kv_cache_dtype = "fp8"   # unchanged: allowed
    assert "fp8 KV cache" in m._decode_route(2, stepwise=True)   # decode_tokens and generate_speculative refuse it
    m.reset_cache()
    m.kv_cache_dtype = None
    m._new_kv_store(1, 16, torch.device("cpu"))
    assert m.kv_caches[0][0].dtype == torch.bfloat16 and not isinstance(m.kv_caches[0], P.model.FP8KVCache)


def test_tp_model_refuses_fp8():
    from lit_llama_b200.tp import TPLLaMA

    m = TPLLaMA(P.LLaMAConfig(block_size=16, vocab_size=64, n_layer=1, n_head=2, n_embd=128), 0, 1, 256)
    m.kv_cache_dtype = None
    with pytest.raises(ValueError, match="bf16 KV cache"):
        m.kv_cache_dtype = "fp8"

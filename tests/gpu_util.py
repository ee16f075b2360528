"""Helpers shared by the -m gpu parity tests."""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from diag import gemv_batch_call, gemv_call, rand_q4, ref_linear, relerr, tc_call, tile, tile_i8, tile_mma  # noqa: E402,F401


def build_tiny(dev, cfg, mode="gptq.int4", seed=1234, tile_cols=-1, exact_linears=False):
    """A tiny model under `mode` and its oracle on the same synthetic weights.  `tile_cols` != -1 (gptq modes): one
    (scale, zero) per group of that many input columns, each linear built as utils.quantization builds it but with
    that group size."""
    import functools

    import lit_llama_b200 as P
    from lit_llama_b200.quantization import ColBlockQuantizedLinear
    from lit_llama_b200.utils import quantization
    from oracle import llama_oracle as O

    if tile_cols != -1 and mode not in ("gptq.int4", "gptq.int8"):
        raise ValueError(f"build_tiny: tile_cols applies to gptq.int4 / gptq.int8, not {mode}")
    sd = O.synth_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"], None if mode == "llm.int8" else mode,
                            dtype=torch.bfloat16, seed=seed, tile_cols=tile_cols)  # llm.int8 loads a float checkpoint and quantises on load
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization(mode):
            if tile_cols != -1:   # quantization() restores torch.nn.Linear on exit
                torch.nn.Linear = functools.partial(ColBlockQuantizedLinear, bits=4 if mode == "gptq.int4" else 8,
                                                    tile_cols=tile_cols)
            model = P.LLaMA(P.LLaMAConfig(**cfg))
    finally:
        torch.set_default_dtype(prev)
    model.load_state_dict(sd)
    oracle = O.OracleLLaMA.from_state_dict(sd, cfg["n_layer"], cfg["n_head"], cfg["block_size"], mode, exact_linears=exact_linears)
    return model.eval(), oracle, sd


def assert_q4_linear_close(y, x, lv, sc, z, min_equal=0.8):
    """An int4 linear output against exact arithmetic: every element within the final bf16 rounding (2^-8
    relative) plus 2^-12 of the row's magnitude sum_k |(lv - z) s x| (the 2..8-row kernel accumulates
    lv x + 64 x over half of k in fp32, DESIGN.md Numerics), and at least `min_equal` of the
    elements bit-equal to the correctly rounded result (the batch-1 kernel is exact integer arithmetic up to one
    fp32 and one bf16 rounding: callers pass min_equal=0.995 for it)."""
    want = ref_linear(x, lv, sc, z)
    mag = x.double().abs() @ ((lv.double() - z.double()) * sc.double()).abs().t()
    err = (y.double() - want).abs()
    bound = want.abs() * 2.0 ** -8 + mag * 2.0 ** -12 + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    assert relerr(y, want) < 1e-3 + 2.0 ** -9
    n_bad = int((y != want.float().bfloat16()).sum())
    assert n_bad <= max(2, round((1.0 - min_equal) * y.numel())), (n_bad, y.numel())

"""CPU: LLaMA._decode_route, the one place the Python side picks the whole-token decode step's route (csrc/api.cu's
RouteId) from the weight kind, B, LLaMA-Adapter v2 affines, the opt-ins int8_step / w8_batch_step / q4_batch_step and
quantization.BATCH_GEMV: each route's flags, tiling and workspace, for every setting at B = 1..16 and stepwise
T = 2..16, and the refusals decode_tokens and generate_speculative raise."""
import itertools

import pytest
import torch

import lit_llama_b200 as P
from lit_llama_b200 import _lib as L
from lit_llama_b200 import adapter as PA
from lit_llama_b200 import adapter_v2 as PV
from lit_llama_b200 import quantization as Q
from lit_llama_b200.utils import quantization
from oracle import llama_oracle as O

CFG = dict(block_size=16, vocab_size=64, n_layer=1, n_head=1, n_embd=128)

# name: (B2L_F_* bits, weight tiling and _fc12 kind, kernel whose workspace batch_work holds)
ROUTES = {
    "q4_gemv": (0, "i8", None),
    "q4_batch": (0, "mma", "q4_gemv_batch"),
    "q4_tc": (0, "tc", None),
    "q4_batch_i8": (L.F_Q4_BATCH_I8, "i8", "w8_gemv_batch"),
    "w8_gemv": (L.F_W8, "i8", None),
    "w8_batch": (L.F_W8 | L.F_W8_BATCH, "i8", "w8_gemv_batch"),
    "q8": (L.F_Q8, None, None),
    "q8_batch": (L.F_Q8 | L.F_Q8_BATCH, None, "q8_linear_batch"),
}
# model: (how it is built, the weight kind _fast_ok holds, has v2 affines)
MODELS = {
    "gptq.int4": ("gptq.int4", "q4", False),
    "gptq.int8": ("gptq.int8", "w8", False),
    "dense": (None, False, False),
    "llm.int8": (None, "q8", False),          # _int8_decode_ok needs CUDA tensors: the kind is set
    "gptq.int4+v2": ("gptq.int4", "q4", True),
    "gptq.int8+v2": ("gptq.int8", "w8", True),
    "llm.int8+v2": (None, "q8", True),
    "gptq.int4 forced off": ("gptq.int4", False, False),   # tests set _fast_ok = False for the module path
}
KNOBS = list(itertools.product((False, True), repeat=4))   # int8_step, w8_batch_step, q4_batch_step, BATCH_GEMV
NEEDS = "needs a gptq.int4 or gptq.int8 model the fused decode step runs with its row-exact batch kernels"


def _model(name: str):
    mode, kind, v2 = MODELS[name]
    with quantization(mode):
        m = PA.LLaMA(PA.LLaMAConfig(**CFG)) if v2 else P.LLaMA(P.LLaMAConfig(**CFG))
        if v2:
            PV.add_adapter_v2_parameters_to_linear_layers(m)
    m.load_state_dict(O.synth_state_dict(1, 1, 128, 64, mode, dtype=torch.bfloat16), strict=False)
    assert m._fast_decode_ok() == {"gptq.int4": "q4", "gptq.int8": "w8", None: False}[mode], name
    m._fast_ok = kind
    assert m._has_affines() == v2
    return m


def _expected(kind, affines: bool, B: int, int8_step: bool, w8_batch_step: bool, q4_batch_step: bool,
              batch_gemv: bool):
    """The route of a plain step (forward, T = 1) at B rows, or None (module by module)."""
    if kind == "q8":
        return ("q8" if B == 1 else "q8_batch") if int8_step else None
    if kind == "w8":
        return "w8_gemv" if B == 1 else ("w8_batch" if w8_batch_step and not affines else None)
    if kind == "q4":
        if B == 1:
            return "q4_gemv"
        if affines:
            return None
        return "q4_batch_i8" if q4_batch_step else ("q4_batch" if B <= 8 and batch_gemv else "q4_tc")
    return None


def _check(route, name):
    if name is None:
        assert isinstance(route, str) and route, route
        return
    assert not isinstance(route, str), (name, route)
    assert (route.name, route.flags, route.tiling, route.work) == (name, *ROUTES[name])


@pytest.mark.parametrize("model", list(MODELS))
def test_decode_route_table(model, monkeypatch):
    m = _model(model)
    kind, affines = MODELS[model][1], MODELS[model][2]
    for int8_step, w8_batch_step, q4_batch_step, batch_gemv in KNOBS:
        monkeypatch.setattr(m, "int8_step", int8_step)
        monkeypatch.setattr(m, "w8_batch_step", w8_batch_step)
        monkeypatch.setattr(m, "q4_batch_step", q4_batch_step)
        monkeypatch.setattr(Q, "BATCH_GEMV", batch_gemv)
        for B in range(1, 17):
            want = _expected(kind, affines, B, int8_step, w8_batch_step, q4_batch_step, batch_gemv)
            _check(m._decode_route(B), want)
        # stepwise (decode_tokens): the row-exact batch kernels whatever the opt-ins say
        for T in range(2, 17):
            r = m._decode_route(T, stepwise=True)
            if kind in ("q4", "w8") and not affines:
                _check(r, "q4_batch_i8" if kind == "q4" else "w8_batch")
            else:
                assert NEEDS in r and "not dense, llm.int8, LLaMA-Adapter v2, or grouped / biased gptq" in r, r
    assert m._fast_ok == kind   # the resolver keeps the cached kind


@pytest.mark.parametrize("model", ["gptq.int4", "gptq.int8"])
def test_decode_route_refuses_stepwise_on_fp8_cache(model):
    m = _model(model)
    m.kv_cache_dtype = "fp8"
    msg = "does not run on an fp8 KV cache (kv_cache_dtype='fp8'): speculative verify keeps a bf16 cache"
    for T in (2, 5, 16):
        assert m._decode_route(T, stepwise=True) == msg
    m._new_kv_store(1, 16, torch.device("cpu"))
    assert m._decode_route(2, stepwise=True) == msg
    _check(m._decode_route(1), "q4_gemv" if model == "gptq.int4" else "w8_gemv")   # the plain step runs fp8 caches
    m._fast_ok = None   # the refusal comes before the weight kind is looked at
    m._decode_route(2, stepwise=True)
    assert m._fast_ok is None


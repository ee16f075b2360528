"""LLaMA-Adapter v2 (reference: lit_llama/adapter_v2.py) on the H100 path.

Same public names, signatures and state-dict keys as the reference, so `generate/adapter_v2.py` (build the model,
`add_adapter_v2_parameters_to_linear_layers`, base checkpoint, then adapter checkpoint, both `strict=False`, then
`generate()`) runs unchanged through `patch_reference()`.  The model class stays `lit_llama_b200.adapter.LLaMA`.

v2 is v1 plus a per-output-feature scale and bias on every linear, lm_head included:
`adapter_scale * (linear(x) + adapter_bias)` (adapter_v2.py:30-33), with the reference's bf16 rounding points, and
trainable RMSNorm scales (weights only).  The linears are found whatever `torch.nn.Linear` is bound to: torch's class,
`ColBlockQuantizedLinear` (gptq.int4 / gptq.int8) and `Linear8bitLt` (llm.int8), so v2 also runs over quantized
bases, which the reference cannot (its `isinstance(module, nn.Linear)` fails once `quantization()` made the name a
`functools.partial`, and its forward reads `layer.weight`).

  * module by module (prefill, no cache, B >= 2, llm.int8, dense): the linear's own forward, then the affine in place
    on its output (`b2l_linear_affine`);
  * the whole-token decode step at B == 1 (gptq.int4, gptq.int8): the affine runs inside each linear's launch
    (`b2l_decode_args::affines`), so the step enqueues as many kernels as without it.
Loading any of these parameters (or an RMSNorm scale) bumps the weight generation, so a captured decode graph and the
adapter prefix are rebuilt for the next token.
"""
import torch
import torch.nn as nn
from torch import Tensor

from . import _lib as L
from .adapter import LLaMA  # noqa: F401  (the reference module exposes the model class under this name)
from .int8 import Linear8bitLt
from .model import RMSNorm, affine_of
from .quantization import ColBlockQuantizedLinear, weights_changed

_TORCH_LINEAR = nn.modules.linear.Linear   # torch's class; `torch.nn.Linear` itself is swapped by quantization()
_LINEARS = (_TORCH_LINEAR, ColBlockQuantizedLinear, Linear8bitLt)


def get_adapter_substrings():
    """adapter_v2.py:11-15: names of the parameters v2 trains (v1's prefix and gate, the linears' scale and bias, the
    RMSNorm scales)."""
    return ["adapter_wte", "gating_factor", "adapter_scale", "adapter_bias", "rms_1", "rms_2", "ln_f"]


def mark_only_adapter_v2_as_trainable(model: LLaMA) -> None:
    """adapter_v2.py:18-21."""
    subs = get_adapter_substrings()
    for name, param in model.named_parameters():
        param.requires_grad = any(s in name for s in subs)


def adapter_v2_state_from_state_dict(state_dict: dict) -> dict:
    """adapter_v2.py:24-27."""
    subs = get_adapter_substrings()
    return {name: param for name, param in state_dict.items() if any(s in name for s in subs)}


def linear_affine(y: Tensor, scale: Tensor, bias: Tensor) -> Tensor:
    """y = bf16(scale * bf16(y + bias)) per output feature, in place on the GPU (b2l_linear_affine).  y: bf16 CUDA
    [..., N], contiguous; scale / bias: bf16 [N]."""
    L.require_cuda_bf16(y, "adapter_v2 linear")
    N = y.shape[-1]
    rc = L.lib().b2l_linear_affine(y.data_ptr(), N, y.numel() // N, N, scale.data_ptr(), bias.data_ptr(), L.stream_ptr())
    L.check(rc, "b2l_linear_affine")
    return y


def adapter_v2_new_forward(self, input: Tensor) -> Tensor:
    """adapter_v2.py:30-33: the layer's own forward (torch's, gptq's or llm.int8's), then the affine."""
    y = type(self).forward(self, input)
    if not y.is_contiguous():
        y = y.contiguous()
    scale, bias = affine_of(self)
    return linear_affine(y, scale, bias)


def _bump_generation(module, incompatible_keys) -> None:
    weights_changed()


def _out_features(layer: nn.Module) -> int:
    n = getattr(layer, "out_features", None)
    if n is None:
        raise TypeError(f"{type(layer).__name__} has no out_features")
    return n


def _device(layer: nn.Module) -> torch.device:
    for t in list(layer.parameters(recurse=False)) + list(layer.buffers(recurse=False)):
        return t.device
    return torch.device("cpu")


def adapter_v2_linear_with_bias_and_scale(layer):
    """adapter_v2.py:36-41: `adapter_bias` (zeros) and `adapter_scale` (ones) of size out_features, in the default
    dtype on the layer's device, and the forward above bound to the instance."""
    from .lora import LoRALayer

    if isinstance(layer, LoRALayer):
        raise ValueError("LLaMA-Adapter v2 over a LoRA layer is unsupported (the reference never combines them)")
    n, dev = _out_features(layer), _device(layer)
    layer.adapter_bias = torch.nn.Parameter(torch.zeros(n, device=dev), requires_grad=True)
    layer.adapter_scale = torch.nn.Parameter(torch.ones(n, device=dev), requires_grad=True)
    layer.forward = adapter_v2_new_forward.__get__(layer, layer.__class__)
    if not getattr(layer, "_adapter_v2_hooked", False):
        layer.register_load_state_dict_post_hook(_bump_generation)
        layer._adapter_v2_hooked = True
    return layer


def add_adapter_v2_parameters_to_linear_layers(model):
    """adapter_v2.py:44-47, for every linear of the model, lm_head included, whatever class `torch.nn.Linear` was
    when it was built.  The RMSNorm scales (trainable in v2) also bump the weight generation when loaded."""
    for module in model.modules():
        if isinstance(module, _LINEARS):
            adapter_v2_linear_with_bias_and_scale(module)
        elif isinstance(module, RMSNorm) and not getattr(module, "_adapter_v2_hooked", False):
            module.register_load_state_dict_post_hook(_bump_generation)
            module._adapter_v2_hooked = True

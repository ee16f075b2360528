"""LoRA (reference: lit_llama/lora.py) on the H100 path.

Same public names, signatures, parameter names, shapes and state-dict keys as the reference, so `generate/lora.py`
(base checkpoint, then LoRA checkpoint, both `strict=False`, then `eval()` and `generate()`) runs unchanged through
`patch_reference()`.  `lora()` swaps `lit_llama_b200.model.CausalSelfAttention`, the name `Block` resolves.

`c_attn` is a `MergedLinear` over whatever `torch.nn.Linear` is when the model is built:

  * torch's own class (a dense model): the reference's layer.  `train(False)` merges `scaling * B.A` into `weight`
    and `train(True)` takes it out again, with the reference's torch arithmetic (lora.py:243-280), so after `eval()`
    c_attn is a dense linear like every other one.
  * under `quantization(mode)` (gptq.int4, gptq.int8, llm.int8): a LoRA layer over that quantized class.  A quantized
    base cannot absorb the update, so it is never merged: the forward is the base's, then `b2l_lora_apply` adds the
    unmerged term of lora.py:308-326 in place (no dropout: inference only).  State-dict keys are the base's buffers
    plus `lora_A` / `lora_B`.  gptq.int4 / gptq.int8 models decode on the whole-token step, which adds the term
    between c_attn and the attention (`b2l_decode_args::loras`); the kernel reads `lora_A` / `lora_B` in place, and
    loading them bumps the weight generation so every baked pointer is rebuilt.

Multi-LoRA: `add_lora_adapter` registers more adapters on such a model (adapter 0 is its own lora_A / lora_B, -1 the
base alone).  `LLaMA.prefill_rows` / `refill_rows` and `generate_prompts` / `generate_stream` with `adapters=` pick
one per prompt: each row of the batched decode step then adds its own adapter's term (`b2l_lora_apply_rows`), and
each prompt's prefill adds its adapter's (`b2l_lora_apply` on its tokens).
"""
import ctypes as C
import functools
import math
from contextlib import contextmanager
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import model as llama
from .quantization import weights_changed

_TORCH_LINEAR = nn.modules.linear.Linear   # torch's class; `torch.nn.Linear` itself is swapped by quantization()


class LoRALayer:
    """lora.py:59-89."""

    def __init__(self, r: int, lora_alpha: int, lora_dropout: float, merge_weights: bool):
        self.r = r
        self.lora_alpha = lora_alpha
        self.lora_dropout = nn.Dropout(p=lora_dropout) if lora_dropout > 0.0 else (lambda x: x)
        self.merged = False
        self.merge_weights = merge_weights

    def _init_lora(self, in_features: int, out_features: int, enable_lora: List[bool], like: torch.Tensor) -> None:
        """lora_A (r n_on, in), lora_B (out / len(enable_lora) n_on, r), scaling and the zero_pad row mask
        (lora.py:139-191); A kaiming-uniform, B zero (lora.py:196-203)."""
        assert out_features % len(enable_lora) == 0, "The length of enable_lora must divide out_features"
        self.enable_lora = enable_lora
        if self.r > 0 and any(enable_lora):
            n_on = sum(enable_lora)
            self.lora_A = nn.Parameter(like.new_zeros((self.r * n_on, in_features)))
            self.lora_B = nn.Parameter(like.new_zeros((out_features // len(enable_lora) * n_on, self.r)))
            self.scaling = self.lora_alpha / self.r
            ind = like.new_zeros((out_features,), dtype=torch.bool).view(len(enable_lora), -1)
            ind[enable_lora, :] = True
            self.lora_ind = ind.view(-1)

    def _reset_lora(self) -> None:
        if hasattr(self, "lora_A"):
            nn.init.kaiming_uniform_(self.lora_A, a=math.sqrt(5))
            nn.init.zeros_(self.lora_B)

    @property
    def _has_lora(self) -> bool:
        return self.r > 0 and any(self.enable_lora)

    def zero_pad(self, x: torch.Tensor) -> torch.Tensor:
        """lora.py:205-241: the update of the enabled groups spread over out_features, zeros in the disabled groups.
        Like the reference, the padded dimension is the last one of x.transpose(0, 1): dim 0 of a 2-D weight update,
        the last dim of a (B, T, n_on part) activation."""
        xt = x.transpose(0, 1)
        out = xt.new_zeros((*xt.shape[:-1], self.out_features))
        out[..., self.lora_ind] = xt
        return out.transpose(0, 1)

    def lora_weights(self) -> Tuple[L.LoRA, Tuple[torch.Tensor, ...]]:
        """The b2l_lora of this layer and the bf16 tensors it points at (the parameters themselves when they are
        bf16 CUDA tensors, so a later in-place load is read by a captured graph)."""
        def bf16(p: torch.Tensor) -> torch.Tensor:
            t = p.detach()
            if t.dtype != torch.bfloat16:
                t = t.to(torch.bfloat16)
            return t.contiguous()

        A, B = bf16(self.lora_A), bf16(self.lora_B)
        mask = sum(1 << g for g, on in enumerate(self.enable_lora) if on)
        spec = L.LoRA(A.data_ptr(), B.data_ptr(), float(self.scaling), self.r, len(self.enable_lora), mask)
        return spec, (A, B)

    def _add_lora(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """y (the base linear's output for x) += zero_pad(B . (A . x)) * scaling in place, lora.py:313-325, on the GPU
        (b2l_lora_apply)."""
        L.require_cuda_bf16(x, "MergedLinear.forward")
        L.require_cuda_bf16(y, "MergedLinear.forward")
        K, N = x.shape[-1], y.shape[-1]
        x2 = x.reshape(-1, K)
        if x2.stride(-1) != 1 or x2.stride(0) % 8 != 0 or x2.data_ptr() % 16 != 0:
            x2 = x2.contiguous()
        if not y.is_contiguous():
            y = y.contiguous()
        spec, keep = self.lora_weights()
        rc = L.lib().b2l_lora_apply(C.byref(spec), x2.data_ptr(), x2.stride(0), None, 0.0, y.data_ptr(), N, x2.shape[0],
                                    N, K, 0, L.stream_ptr())
        L.check(rc, "b2l_lora_apply")
        del keep   # the launch is enqueued: the caching allocator reuses the memory in stream order
        return y


class MergedLinear(_TORCH_LINEAR, LoRALayer):
    """lora.py:92-326.  Constructed while `torch.nn.Linear` is a quantized class (inside `quantization(mode)`), it
    returns a LoRA layer over that class instead (never merged; see the module docstring)."""

    def __new__(cls, *args, **kwargs):
        base = torch.nn.Linear
        if cls is MergedLinear and base is not _TORCH_LINEAR:
            extra = {}
            if isinstance(base, functools.partial):   # gptq: partial(ColBlockQuantizedLinear, bits=..., tile_cols=-1)
                base, extra = base.func, dict(base.keywords)
            qcls = _quantized_merged_linear(base)
            obj = object.__new__(qcls)
            obj.__init__(*args, _base_kwargs=extra, **kwargs)
            return obj
        return super().__new__(cls)

    def __init__(self, in_features: int, out_features: int, r: int = 0, lora_alpha: int = 1, lora_dropout: float = 0.0,
                 enable_lora: List[bool] = [False], fan_in_fan_out: bool = False, merge_weights: bool = True, **kwargs):
        _TORCH_LINEAR.__init__(self, in_features, out_features, **kwargs)
        LoRALayer.__init__(self, r=r, lora_alpha=lora_alpha, lora_dropout=lora_dropout, merge_weights=merge_weights)
        self.fan_in_fan_out = fan_in_fan_out
        self._init_lora(in_features, out_features, enable_lora, self.weight)
        if self._has_lora:
            self.weight.requires_grad = False
        self.reset_parameters()
        if fan_in_fan_out:
            self.weight.data = self.weight.data.T

    def reset_parameters(self):
        """lora.py:196-203."""
        _TORCH_LINEAR.reset_parameters(self)
        self._reset_lora()

    def _t(self, w: torch.Tensor) -> torch.Tensor:
        return w.T if self.fan_in_fan_out else w

    def train(self, mode: bool = True):
        """lora.py:243-280: eval merges scaling * conv1d(A, B) into weight, train takes it out (same torch ops)."""
        _TORCH_LINEAR.train(self, mode)
        if self.merge_weights and (self.merged if mode else not self.merged):
            if self._has_lora:
                delta = F.conv1d(self.lora_A.data.unsqueeze(0), self.lora_B.data.unsqueeze(-1),
                                 groups=sum(self.enable_lora)).squeeze(0)
                self.weight.data += (-1 if mode else 1) * self.zero_pad(self._t(delta * self.scaling))
            self.merged = not mode
        return self

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """lora.py:282-326: merged, the dense linear; unmerged, the dense linear plus the LoRA term on the GPU."""
        result = F.linear(x, self._t(self.weight), bias=self.bias)
        if self.merged or not self._has_lora:
            return result
        return self._add_lora(x, result)


class _QuantizedLoRA(LoRALayer):
    """MergedLinear over a quantized base class (the second base of the concrete class): the base's buffers, forward
    and kernels, plus lora_A / lora_B and the unmerged term."""

    _base: type = None
    #: the per-row adapter choice LLaMA sets around a multi-LoRA call (None: lora_A / lora_B on every row):
    #: ("rows", sel) row m adds adapter sel[m] (device int32, >= M entries); ("one", k, sel) every row adds adapter k;
    #: ("segments", [(start, len, k), ...]) the packed prompts of refill_rows, each its own adapter
    _lora_route = None

    def __init__(self, in_features: int, out_features: int, r: int = 0, lora_alpha: int = 1, lora_dropout: float = 0.0,
                 enable_lora: List[bool] = [False], fan_in_fan_out: bool = False, merge_weights: bool = True, *,
                 _base_kwargs=None, **kwargs):
        if fan_in_fan_out:
            raise ValueError("MergedLinear over a quantized base: fan_in_fan_out=True is unsupported")
        self._base.__init__(self, in_features, out_features, **kwargs, **(_base_kwargs or {}))
        LoRALayer.__init__(self, r=r, lora_alpha=lora_alpha, lora_dropout=lora_dropout, merge_weights=merge_weights)
        self.fan_in_fan_out = False
        like = torch.empty(0, device=self._device())
        self._init_lora(in_features, out_features, enable_lora, like)
        self._reset_lora()

    def _device(self) -> torch.device:
        return next(t.device for t in list(self._buffers.values()) + list(self._parameters.values()) if t is not None)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = self._base.forward(self, x)
        if not self._has_lora:
            return y
        return self._add_lora(x, y) if self._lora_route is None else self._add_lora_route(x, y)

    @property
    def _adapters(self) -> List[Tuple[torch.Tensor, torch.Tensor, float, int]]:
        """The adapters add_lora_adapter registered (1, 2, ...): (lora_A, lora_B, scaling, r), bf16 on the device.
        Plain attributes, not parameters: state_dict() does not change."""
        if "_extra_adapters" not in self.__dict__:
            self.__dict__["_extra_adapters"] = []
        return self.__dict__["_extra_adapters"]

    def lora_set(self, k: int) -> Tuple[L.LoRA, tuple]:
        """The b2l_lora of adapter k (0: lora_A / lora_B) and the tensors it points at."""
        if k == 0:
            return self.lora_weights()
        A, B, scaling, r = self._adapters[k - 1]
        mask = sum(1 << g for g, on in enumerate(self.enable_lora) if on)
        return L.LoRA(A.data_ptr(), B.data_ptr(), float(scaling), r, len(self.enable_lora), mask), (A, B)

    def _add_lora_route(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """y += each row's adapter term under _lora_route (the module path of a multi-LoRA model)."""
        L.require_cuda_bf16(x, "MergedLinear.forward")
        L.require_cuda_bf16(y, "MergedLinear.forward")
        K, N = x.shape[-1], y.shape[-1]
        x2 = x.reshape(-1, K)
        if x2.stride(-1) != 1 or x2.stride(0) % 8 != 0 or x2.data_ptr() % 16 != 0:
            x2 = x2.contiguous()
        if not y.is_contiguous():
            y = y.contiguous()
        M, lib, route = x2.shape[0], L.lib(), self._lora_route
        if route[0] == "rows":   # decode: row m adds adapter sel[m]
            n = 1 + len(self._adapters)
            specs = [self.lora_set(k) for k in range(n)]
            arr = (L.LoRA * n)(*[sp for sp, _ in specs])
            rc = lib.b2l_lora_apply_rows(arr, n, route[1].data_ptr(), x2.data_ptr(), x2.stride(0), None, 0.0, y.data_ptr(),
                                         N, M, N, K, 0, L.stream_ptr())
            L.check(rc, "b2l_lora_apply_rows")
            return y
        segs = [(0, M, route[1])] if route[0] == "one" else route[1]
        for start, n_rows, k in segs:   # one launch per prompt on its rows: a row's term does not depend on M
            if k < 0:
                continue
            spec, keep = self.lora_set(k)
            rc = lib.b2l_lora_apply(C.byref(spec), x2.data_ptr() + start * x2.stride(0) * 2, x2.stride(0), None, 0.0,
                                    y.data_ptr() + start * N * 2, N, n_rows, N, K, 0, L.stream_ptr())
            L.check(rc, "b2l_lora_apply")
        return y

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        """lora_A / lora_B are copied in place (the decode step's pointers stay valid); the rest goes to the base's own
        loader (which may consume `weight` itself, like Linear8bitLt).  Loading bumps the weight generation."""
        lora = {name: self._parameters.pop(name) for name in ("lora_A", "lora_B") if name in self._parameters}
        try:
            with torch.no_grad():
                for name, p in lora.items():
                    key = prefix + name
                    if key not in state_dict:
                        missing_keys.append(key)
                        continue
                    v = state_dict.pop(key)
                    if v.shape != p.shape:
                        error_msgs.append(f"size mismatch for {key}: copying a param with shape {tuple(v.shape)}, "
                                          f"the shape in current model is {tuple(p.shape)}.")
                        continue
                    p.copy_(v)
            super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                          error_msgs)
        finally:
            self._parameters.update(lora)
        weights_changed()


_QUANT_CLASSES: Dict[type, type] = {}


def lora_layers(model: nn.Module) -> List[Tuple[str, "_QuantizedLoRA"]]:
    """(name, layer) of every LoRA layer over a quantized base that carries a term."""
    return [(n, m) for n, m in model.named_modules() if isinstance(m, _QuantizedLoRA) and m._has_lora]


def add_lora_adapter(model: nn.Module, lora_state_dict: Dict[str, torch.Tensor], alpha: float = 16) -> int:
    """Register one more LoRA adapter on a LoRA model over a quantized base (built under `lora(...)` and
    `quantization(...)`) and return its id: 1, 2, ... (adapter 0 is the model's own lora_A / lora_B, -1 the base
    alone).  `lora_state_dict` is what `lora_state_dict()` or finetune/lora.py save: the `...c_attn.lora_A` /
    `lora_B` of every LoRA layer.  r comes from the shapes (1..64), scaling = alpha / r, enable_lora is the model's.
    The tensors are copied once, as bf16 on the model's device; `state_dict()` does not change.  Rows pick adapters
    through `adapters=` of LLaMA.prefill_rows / refill_rows and generate_prompts / generate_stream."""
    if any(isinstance(m, MergedLinear) for m in model.modules()):
        raise ValueError("add_lora_adapter: a dense base merges its LoRA into the weights on eval(); per-row adapters "
                         "need a quantized base (gptq.int4, gptq.int8 or llm.int8)")
    layers = lora_layers(model)
    if not layers:
        raise ValueError("add_lora_adapter: the model has no LoRA layers (build it under lora(...) and quantization(...))")
    want = {f"{n}.{p}" for n, _ in layers for p in ("lora_A", "lora_B")}
    got = set(lora_state_dict)
    if got != want:
        missing, extra = sorted(want - got), sorted(got - want)
        raise ValueError(f"add_lora_adapter: the state dict does not match the model's LoRA layers "
                         f"(missing {missing[:4]}{'...' if len(missing) > 4 else ''}, "
                         f"unexpected {extra[:4]}{'...' if len(extra) > 4 else ''})")
    if len(layers[0][1]._adapters) >= L.LORA_MAX_SETS - 1:
        raise ValueError(f"add_lora_adapter: {L.LORA_MAX_SETS - 1} adapters are registered already (the most one "
                         "decode step serves besides the model's own)")
    staged = []
    for n, lay in layers:
        A, B = lora_state_dict[f"{n}.lora_A"], lora_state_dict[f"{n}.lora_B"]
        n_on, n_g = sum(lay.enable_lora), len(lay.enable_lora)
        r = A.shape[0] // n_on if A.dim() == 2 else 0
        if (A.dim() != 2 or B.dim() != 2 or A.shape[0] != r * n_on or not 1 <= r <= L.LORA_MAX_R
                or A.shape[1] != lay.in_features or tuple(B.shape) != (lay.out_features // n_g * n_on, r)):
            raise ValueError(f"add_lora_adapter: {n}: lora_A {tuple(A.shape)} / lora_B {tuple(B.shape)} do not fit "
                             f"enable_lora={lay.enable_lora} on a [{lay.out_features}, {lay.in_features}] linear "
                             f"(lora_A [r*{n_on}, {lay.in_features}], lora_B [{lay.out_features // n_g}*{n_on}, r], "
                             f"r 1..{L.LORA_MAX_R})")
        staged.append((lay, A, B, r))
    dev = layers[0][1]._device()
    for lay, A, B, r in staged:
        a = torch.empty(A.shape, dtype=torch.bfloat16, device=dev)
        b = torch.empty(B.shape, dtype=torch.bfloat16, device=dev)
        a.copy_(A)
        b.copy_(B)
        lay._adapters.append((a, b, alpha / r, r))
    weights_changed()
    return len(layers[0][1]._adapters)


def _quantized_merged_linear(base: type) -> type:
    cls = _QUANT_CLASSES.get(base)
    if cls is None:
        cls = _QUANT_CLASSES[base] = type("MergedLinear", (_QuantizedLoRA, base),
                                          {"_base": base, "__module__": __name__,
                                           "__qualname__": f"MergedLinear[{base.__name__}]"})
    return cls


def mark_only_lora_as_trainable(model: nn.Module, bias: str = "none") -> None:
    """lora.py:329-361."""
    for n, p in model.named_parameters():
        if "lora_" not in n:
            p.requires_grad = False
    if bias == "none":
        return
    if bias == "all":
        for n, p in model.named_parameters():
            if "bias" in n:
                p.requires_grad = True
    elif bias == "lora_only":
        for m in model.modules():
            if isinstance(m, LoRALayer) and getattr(m, "bias", None) is not None:
                m.bias.requires_grad = True
    else:
        raise NotImplementedError


def lora_state_dict(model: nn.Module, bias: str = "none") -> Dict[str, torch.Tensor]:
    """lora.py:364-395."""
    sd = model.state_dict()
    if bias == "none":
        return {k: v for k, v in sd.items() if "lora_" in k}
    if bias == "all":
        return {k: v for k, v in sd.items() if "lora_" in k or "bias" in k}
    if bias == "lora_only":
        out = {}
        for k, v in sd.items():
            if "lora_" in k:
                out[k] = v
                b = k.split("lora_")[0] + "bias"
                if b in sd:
                    out[b] = sd[b]
        return out
    raise NotImplementedError


@dataclass
class LoRAConfig:
    """lora.py:398-402."""
    r: float = 0.0
    alpha: float = 1.0
    dropout: float = 0.0


class CausalSelfAttention(llama.CausalSelfAttention):
    """lora.py:405-446: model.CausalSelfAttention with c_attn a MergedLinear on q and v (`enable_lora=[True, False,
    True]`)."""
    lora_config = None

    def __init__(self, config: llama.LLaMAConfig) -> None:
        nn.Module.__init__(self)
        assert config.n_embd % config.n_head == 0
        self.c_attn = MergedLinear(in_features=config.n_embd, out_features=3 * config.n_embd, r=self.lora_config.r,
                                   lora_alpha=self.lora_config.alpha, lora_dropout=self.lora_config.dropout,
                                   enable_lora=[True, False, True], fan_in_fan_out=False, merge_weights=True, bias=False)
        self.c_proj = nn.Linear(config.n_embd, config.n_embd, bias=False)
        self.n_head = config.n_head
        self.n_embd = config.n_embd
        self.block_size = config.block_size
        self.rope_cache = None
        self._ring: Optional[torch.Tensor] = None
        self._ring_shared = False

    def _lora(self):
        c = self.c_attn
        if not isinstance(c, _QuantizedLoRA) or not c._has_lora:
            return None   # a dense MergedLinear merges on eval(); the fused step runs quantized models only
        return c.lora_weights()


@contextmanager
def lora(r, alpha, dropout, enabled: bool = True):
    """lora.py:449-478: inside, `lit_llama_b200.model.CausalSelfAttention` is the LoRA variant."""
    if not enabled:
        yield
        return
    CausalSelfAttention.lora_config = LoRAConfig(r=r, alpha=alpha, dropout=dropout)
    previous = llama.CausalSelfAttention
    llama.CausalSelfAttention = CausalSelfAttention
    try:
        yield
    finally:
        llama.CausalSelfAttention = previous
        CausalSelfAttention.lora_config = None

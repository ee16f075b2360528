"""CPU oracle for LoRA inference (reference: lit_llama/lora.py).  TEST INFRASTRUCTURE ONLY.

The reference merges its LoRA update into a dense `c_attn` on `eval()` and refuses a quantized base
(generate/lora.py:61-62), so for gptq / llm.int8 models there is no reference run to pin against.  This module
restates the reference's UNMERGED MergedLinear forward (lora.py:308-326) on top of oracle/llama_oracle.py's linears:

    result = base(x);  after_A = F.linear(x, lora_A);  after_B = grouped conv1d(after_A, lora_B);
    result += zero_pad(after_B) * scaling

every step in x's dtype like the reference.  `lora_branch` is pinned bit for bit against the reference's own
MergedLinear by tests/golden/tiny_lora_bf16.pt (oracle/make_golden_lora.py).  A module of its own, so the base oracle
and the fixtures it is pinned by stay untouched.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle import llama_oracle as O

Tensor = torch.Tensor
QV = [True, False, True]   # lora.py:436, LoRA on q and v


def lora_branch(x: Tensor, result: Tensor, A: Tensor, B: Tensor, scaling: float, enable_lora: List[bool]) -> Tensor:
    """lora.py:313-325 for x (..., in) with at least 2 dims and result = base(x) (..., out): returns a new tensor."""
    n_on = sum(enable_lora)
    out_features = result.shape[-1]
    after_a = F.linear(x, A)
    after_b = F.conv1d(after_a.transpose(-2, -1), B.unsqueeze(-1), groups=n_on).transpose(-2, -1)
    ind = torch.zeros(out_features, dtype=torch.bool).view(len(enable_lora), -1)
    ind[enable_lora, :] = True
    padded = after_b.new_zeros((*after_b.shape[:-1], out_features))
    padded[..., ind.view(-1)] = after_b
    return result + padded * scaling


class LoRALin:
    """A layer of the oracle model: its base linear (O.QLin) plus the unmerged LoRA term."""

    def __init__(self, base: O.QLin, A: Tensor, B: Tensor, scaling: float, enable_lora: List[bool]):
        self.base, self.A, self.B, self.scaling, self.enable_lora = base, A, B, scaling, enable_lora

    def __call__(self, x: Tensor) -> Tensor:
        return lora_branch(x, self.base(x), self.A, self.B, self.scaling, self.enable_lora)


def lora_weights(n_layer: int, n_embd: int, r: int = 8, seed: int = 4321, b_std: float = 0.05, zero_b: bool = False,
                 dtype=torch.bfloat16, layers: Optional[List[int]] = None) -> Dict[str, Tensor]:
    """Random LoRA weights for c_attn on q and v: lora_A like the reference's init (kaiming-uniform, lora.py:202),
    lora_B ~ N(0, b_std) instead of its zero init (zero_b: the reference's initial state), for `layers` (default all)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    bound = 1.0 / math.sqrt(n_embd)   # kaiming_uniform_(a=sqrt(5)) on a fan_in of n_embd
    for i in (range(n_layer) if layers is None else layers):
        p = f"transformer.h.{i}.attn.c_attn."
        out[p + "lora_A"] = ((torch.rand(2 * r, n_embd, generator=g) * 2 - 1) * bound).to(dtype)
        b = torch.randn(2 * n_embd, r, generator=g) * b_std
        out[p + "lora_B"] = (torch.zeros_like(b) if zero_b else b).to(dtype)
    return out


def from_state_dict(sd: Dict[str, Tensor], n_layer: int, n_head: int, block_size: int, mode: Optional[str] = None,
                    exact_linears: bool = False, r: int = 8, alpha: float = 16) -> O.OracleLLaMA:
    """OracleLLaMA whose c_attn carries the unmerged LoRA term wherever `sd` has lora_A / lora_B."""
    m = O.OracleLLaMA.from_state_dict(sd, n_layer, n_head, block_size, mode, exact_linears)
    for i, lay in enumerate(m.layers):
        p = f"transformer.h.{i}.attn.c_attn."
        if p + "lora_A" in sd:
            lay["c_attn"] = LoRALin(lay["c_attn"], sd[p + "lora_A"], sd[p + "lora_B"], alpha / r, QV)
    return m

"""CPU oracle for LLaMA-Adapter v2 inference (reference: lit_llama/adapter_v2.py).  TEST INFRASTRUCTURE ONLY.

Extends oracle/adapter_oracle.py's OracleAdapterLLaMA: every linear of every Block and lm_head becomes
`adapter_scale * (linear(x) + adapter_bias)` (adapter_v2.py:30-33) in the activations' dtype, so a bf16 model rounds
after the add and after the multiply like the reference.  The v1 prefix keys / values go through the wrapped c_attn,
as in the reference.  The RMSNorm scales are ordinary weights here.  Pinned by tests/golden/tiny_adapter_v2_bf16.pt
(oracle/make_golden_adapter_v2.py runs the unmodified reference).  A module of its own, so the v1 oracle and the
fixtures it is pinned by stay untouched.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch

from oracle import adapter_oracle as A

Tensor = torch.Tensor

# oracle layer key -> reference module path inside transformer.h.<i>
LAYER_LINEARS = {"c_attn": "attn.c_attn", "c_proj": "attn.c_proj", "c_fc1": "mlp.c_fc1", "c_fc2": "mlp.c_fc2",
                 "mlp_proj": "mlp.c_proj"}


def linear_prefixes(n_layer: int):
    """Module paths of every linear adapter v2 wraps, lm_head included."""
    return ["lm_head"] + [f"transformer.h.{i}.{p}" for i in range(n_layer) for p in LAYER_LINEARS.values()]


def adapter_v2_state_dict(n_layer: int, n_head: int, n_embd: int, vocab_size: int, mode: Optional[str],
                          prompt_length: int = 10, start_layer: int = 2, dtype=torch.bfloat16, seed: int = 1234,
                          adapter_seed: int = 4321, v2_seed: int = 2468, identity: bool = False,
                          zero_gates: bool = False) -> Dict[str, Tensor]:
    """A v2 checkpoint on top of A.adapter_state_dict (base weights, prefix, gates): every linear gets `adapter_scale`
    with |s| in [0.5, 1.5] and either sign and `adapter_bias` ~ N(0, 0.05^2) (the order of the linears' outputs), and
    every RMSNorm scale is redrawn in [0.5, 1.5] (away from 1).  A kernel that skipped the affine, or read it in the
    wrong row order, is then far off.  `identity`: scale 1 and bias 0 (the reference's initial values); the norm
    scales are drawn all the same."""
    sd = A.adapter_state_dict(n_layer, n_head, n_embd, vocab_size, mode, prompt_length, start_layer, dtype=dtype,
                              seed=seed, adapter_seed=adapter_seed, zero_gates=zero_gates)
    g = torch.Generator().manual_seed(v2_seed)
    for p in linear_prefixes(n_layer):
        key = p + (".scales" if p + ".scales" in sd else ".weight")
        n = sd[key].shape[0]
        s = (0.5 + torch.rand(n, generator=g)) * torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
        b = 0.05 * torch.randn(n, generator=g)
        sd[p + ".adapter_scale"] = (torch.ones(n) if identity else s).to(dtype)
        sd[p + ".adapter_bias"] = (torch.zeros(n) if identity else b).to(dtype)
    for k in list(sd):
        if k.endswith("rms_1.scale") or k.endswith("rms_2.scale") or k == "transformer.ln_f.scale":
            sd[k] = (0.5 + torch.rand(sd[k].shape[0], generator=g)).to(dtype)
    return sd


@dataclass
class AffineLin:
    """adapter_v2.py:30-33 around one oracle linear."""
    lin: object
    scale: Tensor
    bias: Tensor

    def __call__(self, x: Tensor) -> Tensor:
        y = self.lin(x)
        return self.scale.to(y.dtype) * (y + self.bias.to(y.dtype))


class OracleAdapterV2LLaMA(A.OracleAdapterLLaMA):
    """OracleAdapterLLaMA whose linears carry the v2 affine."""

    @staticmethod
    def from_state_dict(sd: Dict[str, Tensor], n_layer: int, n_head: int, block_size: int, mode: Optional[str] = None,
                        exact_linears: bool = False) -> "OracleAdapterV2LLaMA":
        base = A.OracleAdapterLLaMA.from_state_dict(sd, n_layer, n_head, block_size, mode, exact_linears)
        m = OracleAdapterV2LLaMA(**{f: getattr(base, f) for f in base.__dataclass_fields__})

        def wrap(lin, prefix):
            if prefix + ".adapter_scale" not in sd:
                return lin
            return AffineLin(lin, sd[prefix + ".adapter_scale"], sd[prefix + ".adapter_bias"])

        m.lm_head = wrap(m.lm_head, "lm_head")
        for i, lay in enumerate(m.layers):
            for key, path in LAYER_LINEARS.items():
                lay[key] = wrap(lay[key], f"transformer.h.{i}.{path}")
        return m

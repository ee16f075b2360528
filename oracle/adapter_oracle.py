"""CPU oracle for LLaMA-Adapter inference (reference: lit_llama/adapter.py).  TEST INFRASTRUCTURE ONLY.

Extends oracle/llama_oracle.py's OracleLLaMA with the adapter's prefix attention (adapter.py:149-167): from
`adapter_start_layer` on, the k / v thirds of c_attn(adapter_wte.weight) (no RMSNorm, no RoPE, cached per cache
lifetime, recomputed without a cache), attended by the rotated q with a softmax of their own, gated per head and
added to the cache attention with the reference's bf16 rounding points.  Pinned by tests/golden/tiny_adapter_int4_bf16.pt
(oracle/make_golden_adapter.py runs the unmodified reference).  A module of its own on top of llama_oracle.py, so
the base oracle and the fixtures it is pinned by stay untouched.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, Optional, Tuple

import torch

from oracle import llama_oracle as O

Tensor = torch.Tensor


def adapter_state_dict(n_layer: int, n_head: int, n_embd: int, vocab_size: int, mode: Optional[str],
                       prompt_length: int = 10, start_layer: int = 2, dtype=torch.bfloat16, seed: int = 1234,
                       adapter_seed: int = 4321, zero_gates: bool = False) -> Dict[str, Tensor]:
    """Synthetic weights of lit_llama.adapter.LLaMA: O.synth_state_dict for the base model, with wte / lm_head cut to
    `vocab_size` rows (the adapter model does not pad the vocabulary, adapter.py:232-235), plus `adapter_wte` ~ N(0, 1)
    and random non-zero per-head gates (|g| in [0.5, 1.5], either sign) in every layer from `start_layer` on."""
    sd = O.synth_state_dict(n_layer, n_head, n_embd, vocab_size, mode, dtype=dtype, seed=seed)
    for k in ("transformer.wte.weight", "lm_head.weight"):
        if k in sd:
            sd[k] = sd[k][:vocab_size].contiguous()
    for k in ("lm_head.quant_weight",):
        if k in sd:
            sd[k] = sd[k][:vocab_size].t().contiguous().t()
    for k in ("lm_head.scales", "lm_head.zeros"):
        if k in sd:
            sd[k] = sd[k][:vocab_size].contiguous()
    g = torch.Generator().manual_seed(adapter_seed)
    for i in range(start_layer, n_layer):
        p = f"transformer.h.{i}.attn."
        sd[p + "adapter_wte.weight"] = torch.randn(prompt_length, n_embd, generator=g).to(dtype)
        gate = (0.5 + torch.rand(n_head, generator=g)) * torch.where(torch.rand(n_head, generator=g) < 0.5, -1.0, 1.0)
        sd[p + "gating_factor"] = (torch.zeros(n_head) if zero_gates else gate).reshape(1, n_head, 1, 1).to(dtype)
    return sd


@dataclass
class OracleAdapterLLaMA(O.OracleLLaMA):
    """OracleLLaMA plus the adapter prefix attention of adapter.py:149-167."""
    adapters: Dict[int, Tuple[Tensor, Tensor]] = field(default_factory=dict)   # layer -> (adapter_wte, gating_factor)
    akv: Dict[int, Tuple[Tensor, Tensor]] = field(default_factory=dict)        # prefix k / v of the cache's lifetime

    @staticmethod
    def from_state_dict(sd: Dict[str, Tensor], n_layer: int, n_head: int, block_size: int, mode: Optional[str] = None,
                        exact_linears: bool = False) -> "OracleAdapterLLaMA":
        base = O.OracleLLaMA.from_state_dict(sd, n_layer, n_head, block_size, mode, exact_linears)
        m = OracleAdapterLLaMA(**{f: getattr(base, f) for f in base.__dataclass_fields__})
        for i in range(n_layer):
            p = f"transformer.h.{i}.attn."
            if p + "adapter_wte.weight" in sd:
                gate = sd[p + "gating_factor"]
                if gate.dim() < 4:   # adapter.py:184-186: legacy checkpoints hold one value for all heads
                    gate = gate.reshape(1, 1, 1, 1).repeat(1, n_head, 1, 1)
                m.adapters[i] = (sd[p + "adapter_wte.weight"], gate)
        return m

    def reset_cache(self) -> None:
        """adapter.py:250-252."""
        self.kv = []
        self.akv = {}

    def _attn(self, x: Tensor, lay, rope: Tensor, mask: Tensor, S: int, input_pos: Optional[Tensor], li: int) -> Tensor:
        """adapter.py:88-174."""
        B, T, C = x.shape
        nh = self.n_head
        hs = C // nh
        q, k, v = lay["c_attn"](x).split(C, dim=2)
        q = O.rope_apply(q.view(B, T, nh, hs), rope).transpose(1, 2)
        k = O.rope_apply(k.view(B, T, nh, hs), rope).transpose(1, 2)
        v = v.view(B, T, nh, hs).transpose(1, 2)
        if input_pos is not None:
            ck, cv = self.kv[li]
            if int(input_pos[-1]) >= S:
                input_pos = torch.tensor(S - 1)
                ck = torch.roll(ck, -1, dims=2)
                cv = torch.roll(cv, -1, dims=2)
            k = ck.index_copy(2, input_pos.reshape(-1), k)
            v = cv.index_copy(2, input_pos.reshape(-1), v)
            self.kv[li] = (k, v)
        y = O.sdpa(q, k, v, mask)
        if li in self.adapters:
            wte, gate = self.adapters[li]
            if input_pos is not None and li in self.akv:
                ak, av = self.akv[li]
            else:
                aT = wte.shape[0]
                _, ak, av = lay["c_attn"](wte.reshape(1, aT, C).to(x.dtype)).split(C, dim=2)
                ak = ak.view(1, aT, nh, hs).repeat(B, 1, 1, 1).transpose(1, 2)
                av = av.view(1, aT, nh, hs).repeat(B, 1, 1, 1).transpose(1, 2)
                if input_pos is not None:
                    self.akv[li] = (ak, av)
            ay = O.sdpa(q, ak, av, torch.ones(T, ak.shape[-2], dtype=torch.bool))
            y = y + gate.to(y.dtype) * ay
        return lay["c_proj"](y.transpose(1, 2).contiguous().view(B, T, C))

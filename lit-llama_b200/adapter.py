"""LLaMA-Adapter (reference: lit_llama/adapter.py) on the H100 path.

Same classes, constructor signatures, parameter names, shapes and state-dict keys as the reference, so
`generate/adapter.py` (base checkpoint, then adapter checkpoint, both `strict=False`, then `generate()`) runs
unchanged through `patch_reference()`.  The classes subclass `model.py`: the forward, the fused decode step, the
module-by-module path, CUDA graphs and `compact()` are the base model's.  What is added:

  * the prefix keys / values: the k and v thirds of `c_attn(adapter_wte.weight)` (adapter.py:155-160, no RMSNorm, no
    RoPE), computed through the layer's own `c_attn` once per cache lifetime into one allocation
    `[layer][2][n_head][aT][hs]` (recomputed when any weight changes); the no-cache forward recomputes them per call
    like the reference;
  * the attention entry points `b2l_attention_adapter` / `b2l_attention_nocache_adapter`, and `adapters` in the
    whole-token decode step: `y + gating_factor * softmax(q ak^T / sqrt(hs)) av` (adapter.py:164-167) with the
    reference's bf16 rounding points, inside the fused decode attention kernel at head_size 128.
"""
import dataclasses
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
from typing_extensions import Self

from . import _lib as L
from . import model as llama
from .model import KVCache, llama_configs
from .quantization import WEIGHTS_GENERATION, weights_changed


@dataclass
class LLaMAConfig(llama.LLaMAConfig):
    """adapter.py:55-58."""
    adapter_prompt_length: int = 10
    adapter_start_layer: int = 2

    @classmethod
    def from_name(cls, name: str) -> Self:
        return cls(**llama_configs[name])


class CausalSelfAttention(llama.CausalSelfAttention):
    """adapter.py:61-190: model.CausalSelfAttention plus, from `adapter_start_layer` on, `adapter_wte` and
    `gating_factor`."""

    def __init__(self, config: LLaMAConfig, block_idx: int) -> None:
        super().__init__(config)
        if block_idx >= config.adapter_start_layer:
            self.adapter_wte = nn.Embedding(config.adapter_prompt_length, config.n_embd)
            self.gating_factor = torch.nn.Parameter(torch.zeros(1, config.n_head, 1, 1))
        self.block_idx = block_idx
        self.adapter_prompt_length = config.adapter_prompt_length
        self.adapter_start_layer = config.adapter_start_layer
        self._cached_prefix: Optional[L.AdapterPrefix] = None   # set by LLaMA for the cache's lifetime
        self._keep = None

    @property
    def has_adapter(self) -> bool:
        return self.block_idx >= self.adapter_start_layer and self.adapter_prompt_length > 0

    def prefix_kv(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """adapter.py:155-159: the prefix keys and values, each bf16 [n_head][aT][hs], through this layer's c_attn."""
        aT, C_ = self.adapter_prompt_length, self.n_embd
        if aT > L.ADAPTER_MAX_LEN:
            raise RuntimeError(f"adapter_prompt_length {aT} unsupported: the attention kernels take at most "
                               f"{L.ADAPTER_MAX_LEN} prefix positions")
        w = self.adapter_wte.weight
        if w.dtype != torch.bfloat16:
            w = w.to(torch.bfloat16)
        kv = self.c_attn(w.reshape(1, aT, C_))[0]   # (aT, 3C)
        hs = C_ // self.n_head
        ak = kv[:, C_:2 * C_].reshape(aT, self.n_head, hs).transpose(0, 1).contiguous()
        av = kv[:, 2 * C_:].reshape(aT, self.n_head, hs).transpose(0, 1).contiguous()
        return ak, av

    def gate(self) -> torch.Tensor:
        """gating_factor as bf16 [n_head]."""
        return self.gating_factor.detach().reshape(-1).to(torch.bfloat16).contiguous()

    def _adapter_prefix(self, cached: bool) -> Optional[L.AdapterPrefix]:
        if not self.has_adapter:
            return None
        if cached and self._cached_prefix is not None:
            return self._cached_prefix
        # no cache (adapter.py:154-160 recomputes on every call), or a stand-alone cached call outside LLaMA
        with torch.no_grad():
            ak, av = self.prefix_kv()
            g = self.gate()
        self._keep = (ak, av, g)   # alive until the next call; the launches are on the current stream
        return L.AdapterPrefix(ak.data_ptr(), av.data_ptr(), g.data_ptr(), self.adapter_prompt_length)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        """adapter.py:176-190: old checkpoints hold one gating value for all heads.  Loading also invalidates the
        decode state / graphs and the prefix store (they bake the prefix and the gate)."""
        name = prefix + "gating_factor"
        if name in state_dict:
            tensor = state_dict[name]
            tensor = tensor._load_tensor() if hasattr(tensor, "_load_tensor") else tensor
            if len(tensor.shape) < 4:
                state_dict[name] = tensor.reshape(1, 1, 1, 1).repeat(1, self.n_head, 1, 1)
            else:
                state_dict[name] = tensor
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
        weights_changed()


class Block(llama.Block):
    """adapter.py:193-219: model.Block with the adapter attention."""

    def __init__(self, config: LLaMAConfig, block_idx: int) -> None:
        object.__setattr__(self, "_block_idx", block_idx)   # read by _attention during model.Block.__init__
        super().__init__(config)

    def _attention(self, config: LLaMAConfig) -> nn.Module:
        return CausalSelfAttention(config, self._block_idx)


class LLaMA(llama.LLaMA):
    """adapter.py:222-304: model.LLaMA whose Blocks know their index.  Like the reference, wte and lm_head have
    `vocab_size` rows (not the padded size)."""

    def __init__(self, config: LLaMAConfig) -> None:
        assert config.vocab_size is not None and config.block_size is not None
        super().__init__(dataclasses.replace(config, padded_vocab_size=config.vocab_size))
        self.adapter_kv_caches: List[Optional[KVCache]] = []
        self._adapter_store: Optional[torch.Tensor] = None   # [layer][2][n_head][aT][hs]
        self._adapter_gates: Optional[torch.Tensor] = None   # [layer][n_head]
        self._adapter_arr = None
        self._adapter_gen = None

    def _block(self, config: LLaMAConfig, block_idx: int) -> nn.Module:
        return Block(config, block_idx)

    @classmethod
    def from_name(cls, name: str) -> Self:
        return cls(LLaMAConfig.from_name(name))

    def reset_cache(self) -> None:
        super().reset_cache()
        self.adapter_kv_caches.clear()
        self._adapter_gen = None

    def expand_cache(self, B: int) -> None:
        """model.LLaMA.expand_cache; the prefix store does not depend on B, so only its (B, nh, aT, hs) views follow."""
        super().expand_cache(B)
        self._prefix_views(B)

    def refill_rows(self, prompts, rows, max_seq_length: int, adapters=None) -> torch.Tensor:
        """model.LLaMA.refill_rows (prefill_rows too); the prefix store is brought up to date first, since the packed
        prefill reads it, and the prefix views follow B as in expand_cache."""
        self._check_prompts(prompts, max_seq_length, "refill_rows")
        if self._adapter_layers() and (self._adapter_gen != WEIGHTS_GENERATION[0] or self._adapter_arr is None):
            self._build_prefixes(1, prompts[0].device)
        out = super().refill_rows(prompts, rows, max_seq_length, adapters)
        self._prefix_views(self._kv_store.shape[2])
        return out

    def _prefix_views(self, B: int) -> None:
        self.adapter_kv_caches = [None if c is None else (c[0][:1].expand(B, -1, -1, -1), c[1][:1].expand(B, -1, -1, -1))
                                  for c in self.adapter_kv_caches]

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        self._adapter_store = self._adapter_gates = self._adapter_arr = None
        self._adapter_gen = None
        for blk in self.transformer.h:
            blk.attn._cached_prefix = None
        return out

    def _adapter_layers(self) -> List[int]:
        return [i for i, blk in enumerate(self.transformer.h) if blk.attn.has_adapter]

    def _adapter_prefixes(self):
        return self._adapter_arr

    @torch.no_grad()
    def _build_prefixes(self, B: int, device: torch.device) -> None:
        """adapter.py:151-160 once per cache lifetime: every adapter layer's prefix keys / values through its own
        c_attn, into one allocation (kept, and refilled in place, while the shape stays)."""
        cfg = self.config
        layers = self._adapter_layers()
        nh, hs, aT = cfg.n_head, cfg.n_embd // cfg.n_head, cfg.adapter_prompt_length
        shape = (cfg.n_layer, 2, nh, aT, hs)
        st = self._adapter_store
        if st is None or st.shape != shape or st.device != device:
            self._adapter_store = torch.zeros(shape, device=device, dtype=torch.bfloat16)
            self._adapter_gates = torch.zeros((cfg.n_layer, nh), device=device, dtype=torch.bfloat16)
            self._drop_steps()   # they point at the old store
        st, gates = self._adapter_store, self._adapter_gates
        arr = (L.AdapterPrefix * cfg.n_layer)()
        for i in layers:
            attn = self.transformer.h[i].attn
            ak, av = attn.prefix_kv()
            st[i, 0].copy_(ak)
            st[i, 1].copy_(av)
            gates[i].copy_(attn.gate())
            arr[i] = L.AdapterPrefix(st[i, 0].data_ptr(), st[i, 1].data_ptr(), gates[i].data_ptr(), aT)
        for i, blk in enumerate(self.transformer.h):
            blk.attn._cached_prefix = arr[i] if i in layers else None
        self._adapter_arr = arr
        # parity with the reference's attribute: (B, nh, aT, hs) views of the store, None where a layer has no adapter
        self.adapter_kv_caches = [(st[i, 0].unsqueeze(0).expand(B, -1, -1, -1), st[i, 1].unsqueeze(0).expand(B, -1, -1, -1))
                                  if i in layers else None for i in range(cfg.n_layer)]
        self._adapter_gen = WEIGHTS_GENERATION[0]

    def forward(self, idx: torch.Tensor, max_seq_length: Optional[int] = None, input_pos: Optional[torch.Tensor] = None):
        if input_pos is not None and self._adapter_layers():
            if not self.kv_caches or self._adapter_gen != WEIGHTS_GENERATION[0] or self._adapter_arr is None:
                self._build_prefixes(idx.size(0), idx.device)
        return super().forward(idx, max_seq_length, input_pos)


def mark_only_adapter_as_trainable(model: LLaMA) -> None:
    """adapter.py:307-311."""
    for name, param in model.named_parameters():
        param.requires_grad = "adapter_wte" in name or "gating_factor" in name


def adapter_state_from_state_dict(state_dict: dict) -> dict:
    """adapter.py:313-315."""
    return {name: param for name, param in state_dict.items() if "adapter_wte" in name or "gating_factor" in name}

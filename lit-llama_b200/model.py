"""Drop-in LLaMA modules (reference: lit_llama/model.py) backed by libb200llama.

Same classes, constructor signatures, parameter/buffer names and forward signatures as
the reference, so `with quantization(mode): model = LLaMA.from_name(name)` followed by
`model.load_state_dict(checkpoint)` and the reference's `generate()` work unchanged.
Every forward runs hand-written sm_90a kernels (include/b2l.h); tensors must be CUDA
bf16 - there is no CPU fallback.

Two execution paths behind `LLaMA.forward`:
  * decode (T == 1 with a KV cache, B <= 16, every Linear a per-row gptq.int4 / gptq.int8 or an llm.int8 layer): one C
    call enqueues the whole token (`b2l_decode_step`), replayed as a CUDA graph, on the route `LLaMA._decode_route`
    picks from the weight kind, B and the opt-ins documented on LLaMA (each route's kernels: csrc/api.cu kRoutes).
  * everything else (prefill on the wgmma GEMM, no-cache forward, other Linear kinds): module by module.
"""
import ctypes as C
import math
import os
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Callable, List, Optional, Tuple, Union

import torch
import torch.nn as nn
from typing_extensions import Self

from . import _lib as L
from .quantization import WEIGHTS_GENERATION
from .utils import find_multiple

MaskCache = torch.Tensor
RoPECache = torch.Tensor
KVCache = Tuple[torch.Tensor, torch.Tensor]


class FP8KVCache(tuple):
    """One layer's fp8 KV cache (LLaMA.kv_cache_dtype = "fp8"): unpacks as (k, v), the e4m3 codes [B, nh, S, hs] in the
    bf16 cache's slot order, with the fp32 scales [B, nh, S] beside them as k_scale / v_scale (include/b2l.h states
    the number format)."""

    def __new__(cls, k: torch.Tensor, v: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor) -> "FP8KVCache":
        self = super().__new__(cls, (k, v))
        self.k_scale, self.v_scale = k_scale, v_scale
        return self


@dataclass
class LLaMAConfig:
    """model.py:25-40."""
    block_size: int = 2048
    vocab_size: int = 32000
    padded_vocab_size: Optional[int] = None
    n_layer: int = 32
    n_head: int = 32
    n_embd: int = 4096

    def __post_init__(self):
        if self.padded_vocab_size is None:
            self.padded_vocab_size = find_multiple(self.vocab_size, 64)

    @classmethod
    def from_name(cls, name: str) -> Self:
        return cls(**llama_configs[name])


llama_configs = {  # model.py:43-48
    "7B": dict(n_layer=32, n_head=32, n_embd=4096),
    "13B": dict(n_layer=40, n_head=40, n_embd=5120),
    "30B": dict(n_layer=60, n_head=52, n_embd=6656),
    "65B": dict(n_layer=80, n_head=64, n_embd=8192),
}


def _linear(module: nn.Module, x: torch.Tensor) -> torch.Tensor:
    return module(x)


def affine_of(lin: nn.Module) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """(adapter_scale, adapter_bias) of a LLaMA-Adapter v2 linear (lit_llama_b200.adapter_v2) as contiguous bf16
    tensors (the parameters themselves when they already are), or None for a plain linear."""
    if not hasattr(lin, "adapter_scale"):
        return None

    def bf16(p: torch.Tensor) -> torch.Tensor:
        t = p.detach()
        return (t if t.dtype == torch.bfloat16 else t.to(torch.bfloat16)).contiguous()

    return bf16(lin.adapter_scale), bf16(lin.adapter_bias)


class RMSNorm(nn.Module):
    """model.py:257-277; the kernel keeps the reference's bf16 rounding points."""

    def __init__(self, size: int, dim: int = -1, eps: float = 1e-5) -> None:
        super().__init__()
        self.scale = nn.Parameter(torch.ones(size))
        self.eps = eps
        self.dim = dim

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        L.require_cuda_bf16(x, "RMSNorm.forward")
        if self.dim not in (-1, x.dim() - 1):
            raise RuntimeError("RMSNorm: only dim=-1 is implemented")
        xc = x.contiguous()
        C_ = xc.shape[-1]
        y = torch.empty_like(xc)
        scale = self.scale if self.scale.dtype == torch.bfloat16 else self.scale.to(torch.bfloat16)
        rc = L.lib().b2l_rmsnorm(xc.data_ptr(), scale.data_ptr(), y.data_ptr(), xc.numel() // C_, C_, float(self.eps), L.stream_ptr())
        L.check(rc, "b2l_rmsnorm")
        return y


def build_rope_cache(seq_len: int, n_elem: int, dtype: torch.dtype, device: torch.device, base: int = 10000) -> RoPECache:
    """model.py:280-303.  Table construction is one-time host-side setup (torch ops)."""
    theta = 1.0 / (base ** (torch.arange(0, n_elem, 2, dtype=dtype, device=device) / n_elem))
    seq_idx = torch.arange(seq_len, dtype=dtype, device=device)
    idx_theta = torch.outer(seq_idx, theta).float()
    cache = torch.stack([torch.cos(idx_theta), torch.sin(idx_theta)], dim=-1)
    if dtype in (torch.float16, torch.bfloat16, torch.int8):
        cache = cache.half()
    return cache


def apply_rope(x: torch.Tensor, rope_cache: RoPECache) -> torch.Tensor:
    """model.py:306-323 as a stand-alone op: x (B, T, n_head, hs) -> rotated copy.
    (Inside the model the rotation is fused with the KV append, see b2l_attention.)"""
    L.require_cuda_bf16(x, "apply_rope")
    B, T, nh, hs = x.shape
    qkv = torch.zeros((B, T, 3, nh, hs), device=x.device, dtype=x.dtype)
    qkv[:, :, 0] = x
    rows = rope_cache[:T].float().contiguous()
    y = torch.empty((B, T, nh * hs), device=x.device, dtype=x.dtype)
    work = torch.empty(L.lib().b2l_attn_workspace_bytes(B, nh, hs, T, T) // 4 + 1, device=x.device, dtype=torch.float32)
    rc = L.lib().b2l_attention_nocache(qkv.data_ptr(), rows.data_ptr(), y.data_ptr(), work.data_ptr(), B, T, nh, hs, T, L.stream_ptr())
    L.check(rc, "b2l_attention_nocache")
    return qkv[:, :, 0].contiguous()


class CausalSelfAttention(nn.Module):
    """model.py:171-237."""

    def __init__(self, config: LLaMAConfig) -> None:
        super().__init__()
        assert config.n_embd % config.n_head == 0
        self.c_attn = nn.Linear(config.n_embd, 3 * config.n_embd, bias=False)
        self.c_proj = nn.Linear(config.n_embd, config.n_embd, bias=False)
        self.n_head = config.n_head
        self.n_embd = config.n_embd
        self.block_size = config.block_size
        self._ring: Optional[torch.Tensor] = None  # shared by LLaMA; private when used stand-alone
        self._ring_shared = False

    def forward(
        self,
        x: torch.Tensor,
        rope: RoPECache,
        mask: MaskCache,
        max_seq_length: int,
        input_pos: Optional[torch.Tensor] = None,
        kv_cache: Optional[KVCache] = None,
        *,
        _rope_is_table: bool = False,
        _ragged: Optional[L.Ragged] = None,
    ) -> Tuple[torch.Tensor, Optional[KVCache]]:
        """`mask` is accepted for signature parity and ignored: the kernel derives the
        causal mask from input_pos exactly as model.py:94-96 builds it from tril.  A 2-D input_pos of shape (B, 1)
        puts each row's one token at its own position, with its own ring offset (B2L_F_ROW_POS).  `_ragged`
        (LLaMA.refill_rows): x (1, N, C) holds the packed prompts it describes, each prefilled into its own row of
        kv_cache at positions 0.. (b2l_attention_ragged, b2l_attention_ragged_kv8 on an fp8 cache; input_pos is
        ignored)."""
        L.require_cuda_bf16(x, "CausalSelfAttention.forward")
        B, T, C_ = x.size()
        hs = C_ // self.n_head
        qkv = self.c_attn(x)
        if not qkv.is_contiguous():
            qkv = qkv.contiguous()
        y = torch.empty((B, T, C_), device=x.device, dtype=x.dtype)
        lib = L.lib()
        rope32 = rope if rope.dtype == torch.float32 else rope.float()
        rope32 = rope32.contiguous()
        prefix = self._adapter_prefix(kv_cache is not None)   # LLaMA-Adapter layers only (adapter.py)
        if _ragged is not None:
            cache_k, cache_v = kv_cache
            tail = (C.byref(_ragged), self._ring.data_ptr(), y.data_ptr(), B * T, cache_k.shape[0], self.n_head, hs,
                    cache_k.shape[2], rope32.shape[0], None if prefix is None else C.byref(prefix), L.stream_ptr())
            if isinstance(kv_cache, FP8KVCache):
                kv8 = L.KV8Cache(cache_k.data_ptr(), cache_v.data_ptr(), kv_cache.k_scale.data_ptr(), kv_cache.v_scale.data_ptr())
                L.check(lib.b2l_attention_ragged_kv8(qkv.data_ptr(), C.byref(kv8), rope32.data_ptr(), *tail),
                        "b2l_attention_ragged_kv8")
            else:
                L.check(lib.b2l_attention_ragged(qkv.data_ptr(), cache_k.data_ptr(), cache_v.data_ptr(), rope32.data_ptr(),
                                                 *tail), "b2l_attention_ragged")
        elif kv_cache is None:
            work = torch.empty(lib.b2l_attn_workspace_bytes(B, self.n_head, hs, T, T) // 4 + 1, device=x.device, dtype=torch.float32)
            rows = rope32 if not _rope_is_table else rope32[:T]
            if prefix is None:
                rc = lib.b2l_attention_nocache(qkv.data_ptr(), rows.data_ptr(), y.data_ptr(), work.data_ptr(), B, T,
                                               self.n_head, hs, rows.shape[0], L.stream_ptr())
                L.check(rc, "b2l_attention_nocache")
            else:
                rc = lib.b2l_attention_nocache_adapter(qkv.data_ptr(), rows.data_ptr(), y.data_ptr(), work.data_ptr(), B, T,
                                                       self.n_head, hs, rows.shape[0], C.byref(prefix), L.stream_ptr())
                L.check(rc, "b2l_attention_nocache_adapter")
        else:
            cache_k, cache_v = kv_cache
            S = cache_k.shape[2]
            assert S == max_seq_length and cache_k.is_contiguous() and cache_v.is_contiguous()
            pos = input_pos.reshape(-1).to(torch.int64)
            rows = input_pos.dim() == 2   # one position (and ring offset) per row
            if rows and (T != 1 or pos.numel() != B):
                raise ValueError(f"CausalSelfAttention: a 2-D input_pos is one position per row, shape ({B}, 1); got "
                                 f"{tuple(input_pos.shape)} for T={T}")
            n_ring = B if rows else 1
            if self._ring is None or self._ring.device != x.device:
                self._ring = torch.zeros(n_ring, dtype=torch.int32, device=x.device)
            if not self._ring_shared:  # stand-alone use: this module owns the roll state (model.py:214-218)
                if self._ring.numel() != n_ring:   # every row starts from the shared offset
                    self._ring = self._ring[:1].expand(n_ring).contiguous()
                if rows:
                    L.check(lib.b2l_ring_advance_rows(pos.data_ptr(), B, self._ring.data_ptr(), S, L.stream_ptr()),
                            "b2l_ring_advance_rows")
                else:
                    L.check(lib.b2l_ring_advance(pos.data_ptr(), T, self._ring.data_ptr(), S, L.stream_ptr()), "b2l_ring_advance")
            if self._ring.numel() != n_ring:
                raise RuntimeError(f"CausalSelfAttention: the KV ring holds {self._ring.numel()} offsets, this call needs {n_ring}")
            work = torch.zeros(lib.b2l_attn_workspace_bytes(B, self.n_head, hs, T, S) // 4 + 1, device=x.device, dtype=torch.float32)
            flags = (0 if _rope_is_table else 4) | (L.F_ROW_POS if rows else 0)  # B2L_F_ROPE_ROWS
            args = (qkv.data_ptr(), cache_k.data_ptr(), cache_v.data_ptr(), rope32.data_ptr(), pos.data_ptr(),
                    self._ring.data_ptr(), y.data_ptr(), work.data_ptr(), B, T, self.n_head, hs, S, rope32.shape[0], flags)
            if isinstance(kv_cache, FP8KVCache):   # T > 1: a prefill at positions 0..T-1 (LLaMA.forward checks them)
                kv8 = L.KV8Cache(cache_k.data_ptr(), cache_v.data_ptr(), kv_cache.k_scale.data_ptr(), kv_cache.v_scale.data_ptr())
                L.check(lib.b2l_attention_kv8(qkv.data_ptr(), C.byref(kv8), rope32.data_ptr(), pos.data_ptr() if T == 1 else None,
                                              self._ring.data_ptr(), y.data_ptr(), work.data_ptr(), B, T, self.n_head, hs, S,
                                              rope32.shape[0], flags, None if prefix is None else C.byref(prefix),
                                              L.stream_ptr()), "b2l_attention_kv8")
            elif prefix is None:
                L.check(lib.b2l_attention(*args, L.stream_ptr()), "b2l_attention")
            else:
                L.check(lib.b2l_attention_adapter(*args, C.byref(prefix), L.stream_ptr()), "b2l_attention_adapter")
        y = self.c_proj(y)
        return y, kv_cache

    def _adapter_prefix(self, cached: bool) -> Optional[L.AdapterPrefix]:
        """The LLaMA-Adapter prefix this layer attends to besides the cache (lit_llama_b200.adapter); None here."""
        return None

    def _lora(self):
        """(b2l_lora, tensors it points at) of a quantized LoRA c_attn (lit_llama_b200.lora); None here."""
        return None


class MLP(nn.Module):
    """model.py:240-254."""

    def __init__(self, config: LLaMAConfig) -> None:
        super().__init__()
        hidden_dim = 4 * config.n_embd
        n_hidden = int(2 * hidden_dim / 3)
        n_hidden = find_multiple(n_hidden, 256)
        self.c_fc1 = nn.Linear(config.n_embd, n_hidden, bias=False)
        self.c_fc2 = nn.Linear(config.n_embd, n_hidden, bias=False)
        self.c_proj = nn.Linear(n_hidden, config.n_embd, bias=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        L.require_cuda_bf16(x, "MLP.forward")
        a = self.c_fc1(x).contiguous()
        b = self.c_fc2(x).contiguous()
        h = torch.empty_like(a)
        L.check(L.lib().b2l_silu_mul(a.data_ptr(), b.data_ptr(), h.data_ptr(), a.numel(), L.stream_ptr()), "b2l_silu_mul")
        return self.c_proj(h)


def _add(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    a, b = a.contiguous(), b.contiguous()
    y = torch.empty_like(a)
    L.check(L.lib().b2l_add(a.data_ptr(), b.data_ptr(), y.data_ptr(), a.numel(), L.stream_ptr()), "b2l_add")
    return y


class Block(nn.Module):
    """model.py:148-168."""

    def __init__(self, config: LLaMAConfig) -> None:
        super().__init__()
        self.rms_1 = RMSNorm(config.n_embd)
        self.attn = self._attention(config)
        self.rms_2 = RMSNorm(config.n_embd)
        self.mlp = MLP(config)

    def _attention(self, config: LLaMAConfig) -> nn.Module:
        """The Block's attention (lit_llama_b200.adapter passes the block index down, adapter.py:200)."""
        return CausalSelfAttention(config)

    def forward(
        self,
        x: torch.Tensor,
        rope: RoPECache,
        mask: MaskCache,
        max_seq_length: int,
        input_pos: Optional[torch.Tensor] = None,
        kv_cache: Optional[KVCache] = None,
        **kw,
    ) -> Tuple[torch.Tensor, Optional[KVCache]]:
        h, new_kv_cache = self.attn(self.rms_1(x), rope, mask, max_seq_length, input_pos, kv_cache, **kw)
        x = _add(x, h)
        x = _add(x, self.mlp(self.rms_2(x)))
        return x, new_kv_cache


def _graph_step(st, graph_after: int, enqueue: Callable[[], None]) -> None:
    """One call of a decode step whose state `st` holds `graph` and `calls`: replay st.graph if captured, else capture
    `enqueue` on call graph_after + 1 (never with graph_after == 0) and replay it, else run `enqueue` eagerly."""
    if st.graph is not None:
        st.graph.replay()
    elif graph_after and st.calls >= graph_after:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            enqueue()
        st.graph = g
        g.replay()
    else:
        enqueue()
    st.calls += 1


class _ModuleGraph(SimpleNamespace):
    """The module-by-module step's `_graph_step` state, key and static buffers; fields also read as items ("graph")."""

    def __getitem__(self, name: str):
        return getattr(self, name)


def _interleave_rows(a: torch.Tensor, b: torch.Tensor, g: int) -> torch.Tensor:
    """Rows (dim 0) of a and b as [g rows of a | g rows of b] per block: the fc1|fc2 order of the fused SwiGLU linear."""
    n = a.shape[0]
    return torch.stack((a.reshape(n // g, g, *a.shape[1:]), b.reshape(n // g, g, *b.shape[1:])), dim=1).reshape(2 * n, *a.shape[1:])


def _fc12_weights(mlp: nn.Module, q1: torch.Tensor, q2: torch.Tensor, kind: str):
    """(tiling, scales, zeros) of c_fc1 and c_fc2 (quant_weight q1 / q2 in the reference layout) interleaved (8 rows / 8
    rows per 16-row block for the batch-1 and 2..8-row kernels, 64 / 64 per 128-row tile for the wgmma kernel) and
    re-tiled for `kind` ("i8", "mma" or "tc", as _Route.tiling), so one tile holds silu's argument and its multiplier
    and SwiGLU runs in the epilogue.  "i8" tiles 4-bit layers with b2l_q4_tile_i8 and 8-bit ones with b2l_w8_tile_i8."""
    nh, K = mlp.c_fc1.out_features, mlp.c_fc1.in_features
    g = 8 if kind != "tc" else 64
    assert nh % g == 0
    qw = _interleave_rows(q1, q2, g).t().contiguous().t()  # reference layout (1, 2nh)
    scales = _interleave_rows(mlp.c_fc1.scales, mlp.c_fc2.scales, g).contiguous()
    zeros = _interleave_rows(mlp.c_fc1.zeros, mlp.c_fc2.zeros, g).contiguous()
    lib = L.lib()
    if kind == "i8":
        from .quantization import tile_i8

        tiled = tile_i8(qw, 2 * nh, K, mlp.c_fc1.bits)
    elif kind == "mma":
        tiled = torch.empty(lib.b2l_q4_tiled_mma_bytes(2 * nh, K), dtype=torch.uint8, device=qw.device)
        L.check(lib.b2l_q4_tile_mma(qw.data_ptr(), tiled.data_ptr(), 2 * nh, K, L.stream_ptr()), "b2l_q4_tile_mma")
    else:
        tiled = torch.empty(lib.b2l_q4_tiled_bytes(2 * nh, K), dtype=torch.uint8, device=qw.device)
        L.check(lib.b2l_q4_tile(qw.data_ptr(), tiled.data_ptr(), 2 * nh, K, L.stream_ptr()), "b2l_q4_tile")
    return tiled, scales, zeros


@dataclass(frozen=True)
class _Route:
    """One route of b2l_decode_step, named as csrc/api.cu's RouteId: the B2L_F_* bits it adds to the step's flags, the
    tiling every gptq weight is read in ("i8": tiled_i8() as qw_mma, the resident copy of a compacted model; "mma":
    tiled_mma() as qw_mma; "tc": tiled() as qw_tiled; None: llm.int8's CB / SCB in place), which is also _fc12's kind,
    and the kernel whose workspace batch_work holds (None: no batch_work)."""
    name: str
    flags: int
    tiling: Optional[str]
    work: Optional[str]


_ROUTES = {r.name: r for r in (
    _Route("q4_gemv", 0, "i8", None),
    _Route("q4_batch", 0, "mma", "q4_gemv_batch"),
    _Route("q4_tc", 0, "tc", None),
    _Route("q4_batch_i8", L.F_Q4_BATCH_I8, "i8", "w8_gemv_batch"),   # the two batch kernels share their workspace
    _Route("w8_gemv", L.F_W8, "i8", None),
    _Route("w8_batch", L.F_W8 | L.F_W8_BATCH, "i8", "w8_gemv_batch"),
    _Route("q8", L.F_Q8, None, None),
    _Route("q8_batch", L.F_Q8 | L.F_Q8_BATCH, None, "q8_linear_batch"),
)}


class _DecodeState:
    """Static buffers + the C argument block of b2l_decode_step on `route` for one (B, S)."""

    def __init__(self, model: "LLaMA", route: _Route, B: int, S: int, device: torch.device, idx_dtype: torch.dtype,
                 row_pos: bool = False, stepwise: bool = False) -> None:
        from .quantization import ColBlockQuantizedLinear, batch_workspace

        cfg = model.config
        C_, nh = cfg.n_embd, cfg.n_head
        hs = C_ // nh
        bf = dict(device=device, dtype=torch.bfloat16)
        self.B, self.S, self.row_pos = B, S, row_pos
        self.generation = WEIGHTS_GENERATION[0]   # raw weight pointers below are valid for this generation only
        self.idx = torch.zeros(B, dtype=idx_dtype, device=device)
        # B2L_F_ROW_POS: one position per row (and model._ring holds one offset per row); B2L_F_STEPWISE: the B rows are
        # consecutive tokens of one sequence, one position each; else one shared position
        self.pos = torch.zeros(B if (row_pos or stepwise) else 1, dtype=torch.int64, device=device)
        self.x = torch.empty((B, C_), **bf)
        self.qkv = torch.empty((B, 3 * C_), **bf)
        self.att = torch.empty((B, C_), **bf)
        n_hidden = model.transformer.h[0].mlp.c_fc1.out_features
        self.hid = torch.empty((B, n_hidden), **bf)
        self.logits = torch.empty((B, 1, cfg.padded_vocab_size), **bf)
        lib = L.lib()
        self.work = torch.zeros(lib.b2l_attn_workspace_bytes(B, nh, hs, 1, S) // 4 + 1, device=device, dtype=torch.float32)
        self.keep = []  # tensors the argument block points into
        q8 = route.tiling is None
        mma = route.tiling != "tc"   # the tiling goes in qw_mma (else qw_tiled)
        if route.work == "q4_gemv_batch":   # one per device, shared by every state
            self.batch_ws = batch_workspace(device, max(C_, n_hidden))
        elif route.work is not None:
            nb = getattr(lib, f"b2l_{route.work}_workspace_bytes")(max(C_, n_hidden), B)
            self.batch_ws = torch.empty(nb, dtype=torch.uint8, device=device)
        else:
            self.batch_ws = None

        def q4(lin: ColBlockQuantizedLinear) -> L.Q4Weight:
            t = {"i8": lin.tiled_i8, "mma": lin.tiled_mma, "tc": lin.tiled}[route.tiling]()
            self.keep.append(t)   # a compacted layer hands out transient tilings: this state owns the ones it points at
            return L.Q4Weight(None if mma else t.data_ptr(), t.data_ptr() if mma else None, lin.scales.data_ptr(),
                              lin.zeros.data_ptr(), lin.out_features, lin.in_features)

        def bf16(p: torch.Tensor) -> torch.Tensor:
            t = p.detach()
            if t.dtype != torch.bfloat16:
                t = t.to(torch.bfloat16)
                self.keep.append(t)
            return t

        def q8w(lin) -> L.Q8Weight:
            return L.Q8Weight(lin.weight.data.data_ptr(), lin.weight.SCB.data_ptr(), lin.out_features, lin.in_features)

        layers = (L.Layer * cfg.n_layer)()
        q8_layers = (L.Q8Layer * cfg.n_layer)() if q8 else None
        # fp8 KV cache: every layer's attention reads its codes and scales (B2L_F_KV_FP8)
        kv8 = isinstance(model.kv_caches[0], FP8KVCache)
        kv8_arr = (L.KV8Cache * cfg.n_layer)() if kv8 else None
        for i, c in enumerate(model.kv_caches if kv8 else ()):
            kv8_arr[i] = L.KV8Cache(c[0].data_ptr(), c[1].data_ptr(), c.k_scale.data_ptr(), c.v_scale.data_ptr())
        for i, blk in enumerate(model.transformer.h):
            k, v = model.kv_caches[i]
            rms = dict(rms_1=bf16(blk.rms_1.scale).data_ptr(), rms_2=bf16(blk.rms_2.scale).data_ptr())
            if q8:   # layers[i] supplies the norms and the KV cache only
                mlp = blk.mlp
                q8_layers[i] = L.Q8Layer(q8w(blk.attn.c_attn), q8w(blk.attn.c_proj), q8w(mlp.c_fc1), q8w(mlp.c_fc2),
                                         q8w(mlp.c_proj))
                layers[i] = L.Layer(**rms, k_cache=k.data_ptr(), v_cache=v.data_ptr())
                continue
            fc12 = model._fc12(i, route.tiling)
            layers[i] = L.Layer(
                **rms, c_attn=q4(blk.attn.c_attn), c_proj=q4(blk.attn.c_proj),
                c_fc12=L.Q4Weight(None if mma else fc12[0].data_ptr(), fc12[0].data_ptr() if mma else None,
                                  fc12[1].data_ptr(), fc12[2].data_ptr(), 2 * n_hidden, C_),
                mlp_proj=q4(blk.mlp.c_proj), k_cache=k.data_ptr(), v_cache=v.data_ptr())
        self.layers = layers
        lin0 = model.lm_head
        self.args = L.DecodeArgs(
            n_layer=cfg.n_layer, n_head=nh, n_embd=C_, n_hidden=n_hidden, vocab=cfg.padded_vocab_size, B=B, S=S,
            sz_dtype=0 if q8 else L.sz_dtype_of(lin0.scales), eps=float(model.transformer.ln_f.eps), layers=layers,
            wte=bf16(model.transformer.wte.weight).data_ptr(), ln_f=bf16(model.transformer.ln_f.scale).data_ptr(),
            lm_head=L.Q4Weight() if q8 else q4(lin0), rope=model.rope_cache.data_ptr(), idx=self.idx.data_ptr(),
            idx_is_i64=1 if idx_dtype == torch.int64 else 0, input_pos=self.pos.data_ptr(),
            ring_start=model._ring.data_ptr(), block_size=cfg.block_size, x=self.x.data_ptr(), qkv=self.qkv.data_ptr(),
            att=self.att.data_ptr(), hid=self.hid.data_ptr(), attn_work=self.work.data_ptr(),
            logits=self.logits.data_ptr(),
            flags=(model.decode_flags | route.flags | (L.F_ROW_POS if row_pos else 0) | (L.F_STEPWISE if stepwise else 0)
                   | (L.F_KV_FP8 if kv8 else 0)),
            batch_work=None if self.batch_ws is None else self.batch_ws.data_ptr())
        if kv8:
            self.keep.append(kv8_arr)
            self.args.kv8 = C.cast(kv8_arr, C.POINTER(L.KV8Cache))
        if q8:
            self.q8_layers = q8_layers
            self.args.q8_layers = C.cast(q8_layers, C.POINTER(L.Q8Layer))
            self.args.q8_lm_head = q8w(lin0)
            self.args.q8_threshold = float(lin0.threshold)
        adapters = model._adapter_prefixes()
        if adapters is not None:   # LLaMA-Adapter: the step's attention adds each layer's gated prefix term
            self.keep.append(adapters)
            self.args.adapters = C.cast(adapters, C.POINTER(L.AdapterPrefix))
        # multi-LoRA (a per-row adapter choice is set): each row adds its own adapter's term, the choice copied into
        # lora_rows before every step; otherwise LoRA: the step adds each layer's low-rank term behind c_attn
        self.lora_rows = None
        sets = None if stepwise or model._lora_route is None else model._lora_sets(self.keep)
        loras = None if sets is not None else model._loras(self.keep)
        if sets is not None:
            self.lora_rows = torch.full((B,), -1, dtype=torch.int32, device=device)
            self.args.lora_sets = C.cast(sets[0], C.POINTER(L.LoRA))
            self.args.n_lora_sets = sets[1]
            self.args.lora_row_set = self.lora_rows.data_ptr()
        if loras is not None:
            self.args.loras = C.cast(loras, C.POINTER(L.LoRA))
        affines = model._affines(self.keep)
        if affines is not None:    # LLaMA-Adapter v2 (B == 1, llm.int8 at any B): every linear's launch applies them
            self.args.affines = C.cast(affines[0], C.POINTER(L.LayerAffine))
            self.args.lm_head_affine = affines[1]
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.calls = 0

    def enqueue(self) -> None:
        L.check(L.lib().b2l_decode_step(C.byref(self.args), L.stream_ptr()), "b2l_decode_step")


class LLaMA(nn.Module):
    """model.py:51-145."""

    #: replay the decode step as a CUDA graph after this many eager steps (0 = never)
    graph_after: int = 2
    #: flags passed to b2l_decode_step (1 = programmatic dependent launch)
    decode_flags: int = 1
    #: return a fresh logits tensor per call like the reference (False: a view of the static buffer)
    copy_logits: bool = True
    #: decode of an llm.int8 model (plain, LLaMA-Adapter v1 / v2 or LoRA) at batch 1..16 on the whole-token step
    #: (b2l_decode_step under B2L_F_Q8: b2l_q8_linear with RMSNorm / residual / SwiGLU / affine fused at batch 1, and
    #: with B2L_F_Q8_BATCH b2l_q8_linear_batch at 2..16), bit-identical to the module path.  Opt-in (B2L_INT8_STEP=1):
    #: by default llm.int8 decodes module by module, and so do batches over 16.
    int8_step: bool = os.environ.get("B2L_INT8_STEP", "0") == "1"
    #: batched (B = 2..16) decode of a gptq.int8 model (plain, LLaMA-Adapter v1 or LoRA) on the whole-token step
    #: (b2l_decode_step under B2L_F_W8 | B2L_F_W8_BATCH: b2l_w8_gemv_batch on the resident batch-1 tilings, each row
    #: bit-identical to b2l_w8_gemv on that row).  Opt-in (B2L_W8_BATCH_STEP=1): by default batched gptq.int8 decodes
    #: module by module, on the wgmma GEMM.
    w8_batch_step: bool = os.environ.get("B2L_W8_BATCH_STEP", "0") == "1"
    #: batched (B = 2..16) decode of a gptq.int4 model (plain, LLaMA-Adapter v1 or LoRA) on the resident batch-1
    #: tilings (b2l_decode_step under B2L_F_Q4_BATCH_I8: b2l_q4_gemv_batch_i8, each row bit-identical to b2l_q4_gemv on
    #: that row), so a compacted model holds no second weight copy while it decodes a batch.  Opt-in
    #: (B2L_Q4_BATCH_STEP=1): by default batches of 2..8 run b2l_q4_gemv_batch and 9..16 b2l_q4_linear_tc.
    q4_batch_step: bool = os.environ.get("B2L_Q4_BATCH_STEP", "0") == "1"

    def __init__(self, config: LLaMAConfig) -> None:
        super().__init__()
        assert config.padded_vocab_size is not None
        self.config = config

        self.lm_head = nn.Linear(config.n_embd, config.padded_vocab_size, bias=False)
        self.transformer = nn.ModuleDict(
            dict(
                wte=nn.Embedding(config.padded_vocab_size, config.n_embd),
                h=nn.ModuleList(self._block(config, i) for i in range(config.n_layer)),
                ln_f=RMSNorm(config.n_embd),
            )
        )

        self.rope_cache: Optional[RoPECache] = None
        self.mask_cache: Optional[MaskCache] = None  # kept for attribute parity; never materialised
        self.kv_caches: List[KVCache] = []
        self._ring: Optional[torch.Tensor] = None
        self._kv_store: Optional[torch.Tensor] = None
        self._kv_scale: Optional[torch.Tensor] = None   # fp8 cache: the scales [n_layer, 2, B, nh, S] beside _kv_store
        self._decode: Optional[_DecodeState] = None
        self._verify = {}   # T -> _DecodeState of decode_tokens (B2L_F_STEPWISE), each with its own CUDA graph
        self._module_graph = None  # CUDA graph of the module-by-module decode step (non-fused Linear kinds)
        # the fused step can run every Linear (checked once, _fast_decode_ok): "q4" (per-row gptq.int4), "w8" (per-row
        # gptq.int8), "q8" (llm.int8), False (module path); _decode_route picks the route from it
        self._fast_ok: Union[None, bool, str] = None
        self._fc12_cache = {}
        self._lora_route = None   # multi-LoRA: the adapter choice of the current call (lora._QuantizedLoRA._lora_route)
        self._lora_sel: Optional[torch.Tensor] = None   # device int32 [16]: each cache row's adapter (-1: none)

    def _block(self, config: LLaMAConfig, block_idx: int) -> nn.Module:
        """Block `block_idx` of the stack (lit_llama_b200.adapter passes the index down, adapter.py:236)."""
        return Block(config)

    _kv_cache_dtype: Optional[str] = None

    @property
    def kv_cache_dtype(self) -> Optional[str]:
        """The KV cache's number format: None (bf16, the default) or "fp8" (e4m3 codes with a power-of-two fp32 scale per
        row, head and slot, include/b2l.h: half the bytes per cached token).  Read when the cache is allocated; it cannot
        change while a cache exists (reset_cache() first).  Under "fp8", kv_caches holds FP8KVCache entries, every
        attention reads and appends codes (b2l_attention_kv8, the decode step's B2L_F_KV_FP8), a prefill starts at
        position 0, and refill_rows packs the prompts a bf16 cache would pack (b2l_attention_ragged_kv8);
        decode_tokens (speculative verify) refuses it."""
        return self._kv_cache_dtype

    @kv_cache_dtype.setter
    def kv_cache_dtype(self, value: Optional[str]) -> None:
        if value not in (None, "fp8"):
            raise ValueError(f"LLaMA.kv_cache_dtype: {value!r}; None (bf16) or 'fp8'")
        if value != self._kv_cache_dtype and self._kv_store is not None:
            raise RuntimeError(f"LLaMA.kv_cache_dtype: a {self._kv_cache_dtype or 'bf16'} KV cache exists; reset_cache() "
                               "before changing its format")
        self._kv_cache_dtype = value

    def _new_kv_store(self, B: int, S: int, device: torch.device) -> None:
        """A zeroed B-row KV store in the kv_cache_dtype format (and its scales), with kv_caches its per-layer views."""
        cfg = self.config
        shape = (cfg.n_layer, 2, B, cfg.n_head, S, cfg.n_embd // cfg.n_head)
        if self._kv_cache_dtype == "fp8":
            self._kv_store = torch.zeros(shape, device=device, dtype=torch.uint8).view(torch.float8_e4m3fn)
            self._kv_scale = torch.zeros(shape[:-1], device=device, dtype=torch.float32)
        else:
            self._kv_store = torch.zeros(shape, device=device, dtype=torch.bfloat16)
            self._kv_scale = None
        self._set_kv_views()

    def _set_kv_views(self) -> None:
        """kv_caches: the per-layer views of _kv_store (and _kv_scale under fp8)."""
        st, sc = self._kv_store, self._kv_scale
        if sc is None:
            self.kv_caches = [(st[i, 0], st[i, 1]) for i in range(self.config.n_layer)]
        else:
            self.kv_caches = [FP8KVCache(st[i, 0], st[i, 1], sc[i, 0], sc[i, 1]) for i in range(self.config.n_layer)]

    def _adapter_prefixes(self):
        """HOST array [n_layer] of b2l_adapter_prefix for b2l_decode_args::adapters, or None (no adapter)."""
        return None

    def _loras(self, keep: list):
        """HOST array [n_layer] of b2l_lora for b2l_decode_args::loras, or None (no LoRA layer); what it points at is
        appended to `keep`."""
        terms = [blk.attn._lora() for blk in self.transformer.h]
        if all(t is None for t in terms):
            return None
        arr = (L.LoRA * len(terms))()
        for i, t in enumerate(terms):
            if t is not None:
                arr[i] = t[0]
                keep.append(t[1])
        keep.append(arr)
        return arr

    def _lora_sets(self, keep: list):
        """(HOST array [n_sets][n_layer] of b2l_lora, n_sets) for b2l_decode_args::lora_sets: set k is adapter k of
        every LoRA layer (lit_llama_b200.lora.add_lora_adapter), r == 0 in a layer without one; None when no layer has
        LoRA.  What it points at is appended to `keep`."""
        from .lora import _QuantizedLoRA

        cs = [blk.attn.c_attn for blk in self.transformer.h]
        lay = [c if isinstance(c, _QuantizedLoRA) and c._has_lora else None for c in cs]
        if all(c is None for c in lay):
            return None
        n_sets = 1 + len(next(c for c in lay if c is not None)._adapters)
        n = len(lay)
        arr = (L.LoRA * (n_sets * n))()
        for i, c in enumerate(lay):
            for k in range(n_sets if c is not None else 0):
                spec, t = c.lora_set(k)
                arr[k * n + i] = spec
                keep.append(t)
        keep.append(arr)
        return arr, n_sets

    def _set_lora_route(self, route) -> None:
        """The per-row adapter choice every LoRA c_attn and the decode step read (None: today's single adapter)."""
        from .lora import lora_layers

        if (route is None) != (self._lora_route is None):
            self._module_graph = None   # it was captured for the other kind of c_attn term
        self._lora_route = route
        for _, lay in lora_layers(self):
            lay._lora_route = route

    def _check_adapters(self, adapters, n: int, who: str) -> List[int]:
        """adapters: one id per prompt, -1 (the base alone), 0 (the model's own LoRA) or one add_lora_adapter returned."""
        from .lora import lora_layers

        layers = lora_layers(self)
        if not layers:
            raise ValueError(f"{who}: adapters= needs a LoRA model over a quantized base (lit_llama_b200.lora)")
        ids = [int(a) for a in adapters]
        top = len(layers[0][1]._adapters)
        if len(ids) != n or not all(-1 <= a <= top for a in ids):
            raise ValueError(f"{who}: adapters {ids} must be {n} ids in -1..{top}")
        return ids

    def _has_affines(self) -> bool:
        return any(hasattr(m, "adapter_scale") for m in self.modules())

    def _affines(self, keep: list):
        """(HOST array [n_layer] of b2l_layer_affine, lm_head's b2l_out_affine) for b2l_decode_args::affines /
        lm_head_affine, or None (no LLaMA-Adapter v2 linear); what they point at is appended to `keep`.  c_fc1 and
        c_fc2's vectors are interleaved 8 / 8 like the batch-1 fc1|fc2 tiling (_fc12 "i8")."""
        if not self._has_affines():
            return None

        def spec(t) -> L.OutAffine:
            if t is None:
                return L.OutAffine()
            keep.extend(t)
            return L.OutAffine(t[0].data_ptr(), t[1].data_ptr())

        arr = (L.LayerAffine * len(self.transformer.h))()
        for i, blk in enumerate(self.transformer.h):
            mlp = blk.mlp
            f1, f2 = affine_of(mlp.c_fc1), affine_of(mlp.c_fc2)
            fc12 = None
            if f1 is not None or f2 is not None:
                nh = mlp.c_fc1.out_features
                like = (f1 or f2)[0]
                one, zero = torch.ones(nh, dtype=like.dtype, device=like.device), torch.zeros(nh, dtype=like.dtype, device=like.device)
                f1, f2 = f1 or (one, zero), f2 or (one, zero)
                fc12 = tuple(_interleave_rows(a, b, 8) for a, b in zip(f1, f2))
            arr[i] = L.LayerAffine(spec(affine_of(blk.attn.c_attn)), spec(affine_of(blk.attn.c_proj)), spec(fc12),
                                   spec(affine_of(mlp.c_proj)))
        keep.append(arr)
        return arr, spec(affine_of(self.lm_head))

    def _init_weights(self, module: nn.Module) -> None:
        """model.py:70-74."""
        if isinstance(module, nn.Linear) and hasattr(module, "weight"):
            torch.nn.init.normal_(module.weight, mean=0.0, std=0.02 / math.sqrt(2 * self.config.n_layer))
        elif isinstance(module, nn.Embedding):
            torch.nn.init.normal_(module.weight, mean=0.0, std=0.02 / math.sqrt(2 * self.config.n_layer))

    @classmethod
    def from_name(cls, name: str) -> Self:
        return cls(LLaMAConfig.from_name(name))

    def build_rope_cache(self, idx: torch.Tensor) -> RoPECache:
        """model.py:128-134: called with the integer token tensor, so the table is fp32."""
        return build_rope_cache(seq_len=self.config.block_size, n_elem=self.config.n_embd // self.config.n_head,
                                dtype=idx.dtype, device=idx.device)

    def build_mask_cache(self, idx: torch.Tensor) -> MaskCache:
        """model.py:136-138 (provided for parity; the kernels never read a mask tensor)."""
        ones = torch.ones((self.config.block_size, self.config.block_size), device=idx.device, dtype=torch.bool)
        return torch.tril(ones).unsqueeze(0).unsqueeze(0)

    def reset_cache(self) -> None:
        """model.py:140-145."""
        self.kv_caches.clear()
        self._kv_store = None
        self._kv_scale = None
        self._drop_steps()
        if self._lora_route is not None:
            self._set_lora_route(None)
        if self._ring is not None:
            if self._ring.numel() != 1:   # back to one shared ring offset
                self._set_ring(torch.zeros(1, dtype=torch.int32, device=self._ring.device))
            else:
                self._ring.zero_()

    def _set_ring(self, ring: torch.Tensor) -> None:
        """The KV ring offset(s) every layer reads: int32 [1] shared by all rows, or [B] after a per-row step."""
        self._ring = ring
        for blk in self.transformer.h:
            blk.attn._ring, blk.attn._ring_shared = ring, True
        self._drop_steps()   # they point at the old ring

    @staticmethod
    def _check_prompts(prompts: List[torch.Tensor], max_seq_length: int, who: str) -> None:
        if not 1 <= len(prompts) <= 16:
            raise ValueError(f"{who}: {len(prompts)} prompts; 1..16 (the batched decode step's range)")
        for p in prompts:
            if p.dim() != 1 or p.numel() == 0:
                raise ValueError(f"{who}: every prompt must be a non-empty 1-D token tensor, got {tuple(p.shape)}")
            if not p.is_cuda:
                raise RuntimeError(f"{who}: prompt is on {p.device}; lit_llama_b200 runs on CUDA only (no CPU fallback)")
            if p.numel() > max_seq_length:
                raise ValueError(f"{who}: a prompt of {p.numel()} tokens does not fit max_seq_length={max_seq_length}")

    @torch.no_grad()
    def prefill_rows(self, prompts: List[torch.Tensor], max_seq_length: int, adapters=None) -> torch.Tensor:
        """Prefill 1..16 different prompts (1-D token tensors of any lengths <= max_seq_length) into one B-row KV cache
        and return each prompt's last-position logits, (B, vocab).

        A fresh B-row cache, then `refill_rows(prompts, range(B), max_seq_length)`: row b's cache is bit for bit the one
        `generate()` builds for prompts[b] (no padded (B, T_max) prefill, which would cost more and round
        differently).  The ring offsets start per row at zero: the next step passes a (B, 1) `input_pos`, row b's first
        new token at position len(prompts[b]).  `adapters` (multi-LoRA): one adapter id per prompt, as refill_rows."""
        self._check_prompts(prompts, max_seq_length, "prefill_rows")
        if adapters is not None:
            self._check_adapters(adapters, len(prompts), "prefill_rows")
        B, dev = len(prompts), prompts[0].device
        self.reset_cache()
        self._prepare(prompts[0].view(1, -1), max_seq_length)
        self._new_kv_store(B, max_seq_length, dev)
        self._set_ring(torch.zeros(B, dtype=torch.int32, device=dev))
        return self.refill_rows(prompts, range(B), max_seq_length, adapters)

    @torch.no_grad()
    def refill_rows(self, prompts: List[torch.Tensor], rows, max_seq_length: int, adapters=None) -> torch.Tensor:
        """Prefill prompts[i] into row rows[i] of the existing B-row KV cache (prefill_rows) and return each prompt's
        last-position logits, (n, vocab): row rows[i] then holds, bit for bit, the cache `generate()` builds for
        prompts[i], with its ring offset at zero, and its next token goes in at position len(prompts[i]).

        The prompts `_pack_plan` admits run through ONE packed prefill (M = sum of their lengths on every linear, the
        ragged attention b2l_attention_ragged or, on an fp8 cache, b2l_attention_ragged_kv8, lm_head on their last rows
        only), split into consecutive passes in input order only when the device's free memory cannot hold the whole
        pack's activations (`_packed_passes`); each of the others runs the batch-1 prefill into its row ("alone").
        Other rows keep their cache contents, positions and ring offsets, and the B-row decode state and its CUDA graph
        stay the same objects (the KV store and the ring tensor change in place), so a decode loop can refill finished
        rows between two steps (generate_stream).

        `adapters` (multi-LoRA, lit_llama_b200.lora.add_lora_adapter): one id per prompt, -1 for the base alone.  Each
        prompt's prefill adds its adapter's term on its own tokens, and row rows[i] then decodes with adapters[i] (the
        other rows keep theirs; rows never given one use adapter 0) until reset_cache().  None: the model's own LoRA on
        every row, as without multi-LoRA; refused once rows carry adapters."""
        rows = [int(r) for r in rows]
        self._check_prompts(prompts, max_seq_length, "refill_rows")
        if adapters is not None:
            adapters = self._check_adapters(adapters, len(prompts), "refill_rows")
        elif self._lora_route is not None:
            raise ValueError("refill_rows: the cache's rows carry adapters (prefill_rows(adapters=...)); pass adapters=")
        store = self._kv_store
        if store is None or self._ring is None or self._ring.numel() != store.shape[2]:
            raise RuntimeError("refill_rows: no B-row KV cache to refill (prefill_rows builds one)")
        B = store.shape[2]
        if len(rows) != len(prompts) or len(set(rows)) != len(rows) or not all(0 <= r < B for r in rows):
            raise ValueError(f"refill_rows: rows {rows} must name {len(prompts)} distinct rows of 0..{B - 1}")
        if store.shape[4] != max_seq_length:
            raise ValueError(f"refill_rows: max_seq_length={max_seq_length} against a cache of {store.shape[4]}")
        self._prepare(prompts[0].view(1, -1), max_seq_length)
        packed = self._pack_plan([p.numel() for p in prompts])
        out: List[Optional[torch.Tensor]] = [None] * len(prompts)
        ad = adapters if adapters is not None else [None] * len(prompts)
        if packed:
            dev = prompts[0].device
            free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
            for part in self._packed_passes([prompts[i].numel() for i in packed], self._packed_token_bytes(), free):
                ids = [packed[j] for j in part]
                logits = self._prefill_packed([prompts[i] for i in ids], [rows[i] for i in ids], max_seq_length,
                                              [ad[i] for i in ids])
                for j, i in enumerate(ids):
                    out[i] = logits[j]
        alone = [i for i in range(len(prompts)) if i not in packed]
        for i, lg in zip(alone, self._prefill_alone([prompts[i] for i in alone], [rows[i] for i in alone], max_seq_length,
                                                    [ad[i] for i in alone])):
            out[i] = lg
        if adapters is not None:   # the refilled rows decode with their prompts' adapters from the next step on
            if self._lora_sel is None or self._lora_sel.device != prompts[0].device:
                self._lora_sel = torch.zeros(16, dtype=torch.int32, device=prompts[0].device)
            if self._lora_route is None:
                self._lora_sel.zero_()   # rows never given an adapter keep the model's own (adapter 0)
            self._lora_sel[torch.tensor(rows, device=self._lora_sel.device)] = torch.tensor(
                adapters, dtype=torch.int32, device=self._lora_sel.device)
            self._set_lora_route(("rows", self._lora_sel))
        return torch.stack(out)

    def _linears(self) -> List[nn.Module]:
        lins = [self.lm_head]
        for blk in self.transformer.h:
            lins += [blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_fc1, blk.mlp.c_fc2, blk.mlp.c_proj]
        return lins

    def _pack_plan(self, lengths: List[int]) -> List[int]:
        """Indices of the prompts (given by length) that refill_rows prefills packed: those whose own batch-1 prefill
        runs every linear on the same row-exact kernel as the pack does (quantization.packs_at), so each keeps its
        batch-1 bits; [] for head sizes other than 128 (the ragged attention's) and for models with any linear outside
        that dispatch (dense, llm.int8, whose rows interact through the batch outlier mask).  The cache's format does
        not enter: an fp8 cache packs the same prompts as a bf16 one."""
        from .quantization import packs_at

        cfg = self.config
        if cfg.n_embd // cfg.n_head != 128:
            return []
        lins = self._linears()
        cand = [i for i, T in enumerate(lengths) if packs_at(lins, T, T)]
        N = sum(lengths[i] for i in cand)
        if not all(packs_at(lins, lengths[i], N) for i in cand):
            return []
        return cand

    def _packed_token_bytes(self) -> int:
        """Device bytes of bf16 activations one token of a packed prefill can hold at once: the Block's widest point is
        the MLP, where x, rms_2(x), c_fc1's, c_fc2's and silu_mul's outputs and c_proj's output are alive (4 C + 3 H
        elements); 2 C more cover the linears' own temporaries (LoRA and v2 affine terms)."""
        cfg = self.config
        n_hidden = find_multiple(int(2 * 4 * cfg.n_embd / 3), 256)
        return 2 * (6 * cfg.n_embd + 3 * n_hidden)

    @staticmethod
    def _packed_passes(lengths: List[int], token_bytes: int, free_bytes: int) -> List[List[int]]:
        """The packed prompts (given by length) as consecutive passes in input order, as indices into `lengths`: one
        pass whenever every token fits `free_bytes` at `token_bytes` each, else each pass takes prompts while they fit,
        and at least one.  Each prompt keeps its batch-1 bits in any pass: the linears are row-exact at any M (no
        split-K, fixed tiles) and packs_at holds at every pass total N >= T."""
        cap = max(0, free_bytes) // max(1, token_bytes)
        passes: List[List[int]] = []
        n = 0
        for i, T in enumerate(lengths):
            if passes and n + T <= cap:
                passes[-1].append(i)
                n += T
            else:
                passes.append([i])
                n = T
        return passes

    def _prefill_packed(self, prompts: List[torch.Tensor], rows: List[int], max_seq_length: int,
                        adapters: List[Optional[int]]) -> torch.Tensor:
        """The packed prefill of refill_rows: the prompts back to back as one (1, N) sequence through the module path
        at M = N, the attention ragged (each prompt into its row at positions 0..), lm_head on each prompt's last row
        on the kernel its batch-1 prefill ran it on at M = len (the GEMM, not the 2..16-row kernel M = n would pick)."""
        from .quantization import kernel_at

        seqs = L.Ragged()
        seqs.n_seq = len(prompts)
        N = 0
        for j, (p, r) in enumerate(zip(prompts, rows)):
            seqs.row[j], seqs.start[j], seqs.len[j] = r, N, p.numel()
            N += p.numel()
        dev = prompts[0].device
        toks = torch.cat([p.to(torch.int64) for p in prompts]).view(1, N)
        route = self._lora_route
        if adapters[0] is not None:   # multi-LoRA: each prompt's tokens add its adapter's term
            self._set_lora_route(("segments", [(seqs.start[j], seqs.len[j], a) for j, a in enumerate(adapters)]))
        try:
            h = self._forward_hidden(toks, max_seq_length, None, ragged=seqs)
        finally:
            self._set_lora_route(route)
        last = torch.tensor([seqs.start[j] + seqs.len[j] - 1 for j in range(len(prompts))], device=dev)
        x = h[0].index_select(0, last)
        y = self.lm_head.run(x, kernel_at(self.lm_head, N))
        aff = affine_of(self.lm_head)
        if aff is not None:   # LLaMA-Adapter v2: the affine its forward applies after the linear
            from .adapter_v2 import linear_affine

            linear_affine(y, *aff)
        return y

    def _prefill_alone(self, prompts: List[torch.Tensor], rows: List[int], max_seq_length: int,
                       adapters: List[Optional[int]]) -> List[torch.Tensor]:
        """The batch-1 prefill of each prompt into its row: the model is pointed at that row of the KV store and its
        ring offset (ring[r:r+1], zeroed) for the call, and the B-row decode state and module graph are put back after
        (a one-token prompt runs, and replaces, the batch-1 step state)."""
        ring, store, scale, caches = self._ring, self._kv_store, self._kv_scale, self.kv_caches
        decode, module_graph, route = self._decode, self._module_graph, self._lora_route
        out = []
        try:
            for p, r, a in zip(prompts, rows, adapters):
                if a is not None:   # multi-LoRA: the prompt's adapter on every token (a one-token prompt's step too)
                    self._set_lora_route(("one", a, torch.full((1,), a, dtype=torch.int32, device=p.device)))
                one = ring[r:r + 1]
                one.zero_()
                self._ring = one
                for blk in self.transformer.h:
                    blk.attn._ring = one
                self._kv_store = store[:, :, r:r + 1]
                self._kv_scale = None if scale is None else scale[:, :, r:r + 1]
                self._set_kv_views()   # contiguous
                self._decode, self._module_graph = None, None
                out.append(self(p.view(1, -1), max_seq_length, torch.arange(p.numel(), device=p.device))[0, -1].clone())
        finally:
            self._ring, self._kv_store, self._kv_scale, self.kv_caches = ring, store, scale, caches
            for blk in self.transformer.h:
                blk.attn._ring = ring
            self._set_lora_route(route)
            self._decode, self._module_graph = decode, module_graph
        return out

    def expand_cache(self, B: int) -> None:
        """Broadcast a batch-1 KV cache to B rows: every row then holds the prompt's keys and values, so B samples of one
        prompt decode from one batch-1 prefill (generate_batch) instead of a (B, T) prefill at B times the GEMM work.
        One device copy of the KV store; `kv_caches` become views of the new store, the ring offset (shared by all rows)
        is kept, and the decode state and module graph, which point at the old store, are rebuilt on the next step.
        `reset_cache()` returns the model to batch 1."""
        if self._kv_store is None:
            raise RuntimeError("expand_cache: no KV cache yet (run the prompt through forward with input_pos first)")
        n_layer, two, B0, nh, S, hs = self._kv_store.shape
        if B == B0:
            return
        if B0 != 1 or B < 1:
            raise ValueError(f"expand_cache: the cache holds {B0} rows; only a batch-1 cache expands (to {B} rows)")
        if self._kv_scale is None:
            self._kv_store = self._kv_store.expand(n_layer, two, B, nh, S, hs).contiguous()
        else:   # fp8: the codes (copied as bytes) and their scales
            self._kv_store = self._kv_store.view(torch.uint8).expand(n_layer, two, B, nh, S, hs).contiguous().view(
                torch.float8_e4m3fn)
            self._kv_scale = self._kv_scale.expand(n_layer, two, B, nh, S).contiguous()
        self._set_kv_views()
        self._drop_steps()

    # ------------------------------------------------------------------ helpers
    def _fc12(self, i: int, kind: str):
        """_fc12_weights of layer i for `kind`, cached while c_fc1 and c_fc2's weights stay the same."""
        mlp = self.transformer.h[i].mlp
        hit = self._fc12_cache.get((i, kind))
        if hit is not None and getattr(mlp.c_fc1, "_released", False):
            return hit[1]     # compacted: this copy IS the layer's weights (compact())
        q1, q2 = mlp.c_fc1.reference_quant_weight(), mlp.c_fc2.reference_quant_weight()
        key = (kind, q1.data_ptr(), q1._version, q2.data_ptr(), q2._version)
        if hit is not None and hit[0] == key:
            return hit[1]
        val = _fc12_weights(mlp, q1, q2, kind)
        self._fc12_cache[(i, kind)] = (key, val)
        return val

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        # the interleaved fc1|fc2 copies are plain tensors of this module: they move with it (a compacted model has no other)
        self._fc12_cache = {k: (key, tuple(fn(t) for t in val)) for k, (key, val) in self._fc12_cache.items()}
        self._drop_steps()
        self._fast_ok = None
        return out

    def _drop_steps(self) -> None:
        """Forget every cached decode step (the fused one, decode_tokens' and the module graph): each bakes pointers
        into the KV store, the ring, the adapter prefixes and the weights."""
        self._decode, self._verify, self._module_graph = None, {}, None

    def _drop_stale(self, st) -> bool:
        """Whether the step state `st` was built before a linear was reloaded, repacked or moved.  If so, everything that
        bakes weight pointers is dropped: every step, _fast_ok, and the interleaved fc1|fc2 copies the reference buffers
        can rebuild (not those compact() made the ONLY copy of both layers: still released, nothing was loaded)."""
        if st is None or st.generation == WEIGHTS_GENERATION[0]:
            return False
        self._drop_steps()
        self._fast_ok = None
        self._fc12_cache = {k: v for k, v in self._fc12_cache.items() if k[1] == "i8" and self._fc12_is_only_copy(k[0])}
        return True

    def _fc12_is_only_copy(self, i: int) -> bool:
        mlp = self.transformer.h[i].mlp
        return getattr(mlp.c_fc1, "_released", False) and getattr(mlp.c_fc2, "_released", False)

    def _fc12_tiling(self, i: int) -> torch.Tensor:
        """The interleaved fc1|fc2 batch-1 tiling of layer i: a compacted c_fc1 / c_fc2's weights (the prefill GEMM
        reads its half in place)."""
        return self._fc12_cache[(i, "i8")][1][0]

    def _fc_from_fc12(self, i: int, which: int) -> torch.Tensor:
        """c_fc1 (which = 0) or c_fc2 (1) of layer i in the reference layout, rebuilt from the interleaved batch-1
        tiling (compacted models keep only that copy): untile (a permutation, by bit width) and take every other 8
        rows."""
        tiled, _, _ = self._fc12_cache[(i, "i8")][1]
        mlp = self.transformer.h[i].mlp
        nh, K, epb = mlp.c_fc1.out_features, mlp.c_fc1.in_features, mlp.c_fc1.entries_per_byte
        name = "b2l_w8_untile_i8" if mlp.c_fc1.bits == 8 else "b2l_q4_untile_i8"
        both = torch.empty((K // epb, 2 * nh), dtype=torch.uint8, device=tiled.device).t()
        L.check(getattr(L.lib(), name)(tiled.data_ptr(), both.data_ptr(), 2 * nh, K, L.stream_ptr()), name)
        return both.contiguous().reshape(nh // 8, 2, 8, K // epb)[:, which].reshape(nh, K // epb).t().contiguous().t()

    def compact(self) -> "LLaMA":
        """Keep ONE resident copy of every gptq.int4 (or, uniformly, gptq.int8) weight: the batch-1 decode tiling
        (c_fc1 / c_fc2: the interleaved fc1|fc2 tiling).  The reference-layout buffers and the per-kernel duplicates are freed; `state_dict()`, prefill
        and batched decode rebuild what they need transiently from that copy (bit-exact permutations).  7B: 3.3 GB of
        weights + 0.26 GB embedding + KV cache instead of 2-3 copies (the reference's gptq.int4 figure is "~5 GB",
        howto/inference.md:37).  Returns self."""
        import functools

        if self._fast_ok is None:
            self._fast_ok = self._fast_decode_ok()
        if self._fast_ok not in ("q4", "w8"):   # llm.int8 ("q8") already holds one copy: CB, read in place
            raise RuntimeError("compact() needs a gptq.int4 or gptq.int8 model the fused batch-1 decode step can run "
                               "(one bit width for every linear)")
        for i, blk in enumerate(self.transformer.h):
            self._fc12(i, "i8")
            for kind in ("mma", "tc"):
                self._fc12_cache.pop((i, kind), None)
            for lin in (blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_proj):
                lin.release_reference_layout()
            fc12 = functools.partial(self._fc12_tiling, i)
            blk.mlp.c_fc1.release_reference_layout(source=functools.partial(self._fc_from_fc12, i, 0), half=(fc12, 0))
            blk.mlp.c_fc2.release_reference_layout(source=functools.partial(self._fc_from_fc12, i, 1), half=(fc12, 1))
        self.lm_head.release_reference_layout()
        self._drop_steps()   # rebuilt on the next step (B > 1 states hold their transient tilings)
        torch.cuda.empty_cache()
        return self

    def _fast_decode_ok(self) -> Union[bool, str]:
        """"q4" / "w8" when every Linear is a per-row gptq.int4 / gptq.int8 layer the fused step can run, "q8" when every
        Linear is a bias-free llm.int8 layer b2l_q8_linear can run (one threshold throughout), else False."""
        from .int8 import Linear8bitLt
        from .quantization import ColBlockQuantizedLinear

        if isinstance(self.lm_head, Linear8bitLt):
            return "q8" if self._int8_decode_ok() else False
        if not isinstance(self.lm_head, ColBlockQuantizedLinear):
            return False
        kind = "w8" if self.lm_head.bits == 8 else "q4"

        def ok(m):
            if not isinstance(m, ColBlockQuantizedLinear):
                return False
            return m.w8_gemv_capable if kind == "w8" else (m.tc_capable and m.gemv_capable)

        dt = self.lm_head.scales.dtype
        if self.config.n_embd % 8 != 0 or not all(ok(m) and m.scales.dtype == dt for m in self._linears()):
            return False
        return kind if all(blk.mlp.c_fc1.out_features % 64 == 0 for blk in self.transformer.h) else False

    def _int8_decode_ok(self) -> bool:
        from .int8 import Linear8bitLt

        thr = self.lm_head.threshold

        def ok(m) -> bool:
            if not isinstance(m, Linear8bitLt) or m.bias is not None or m.threshold != thr:
                return False
            cb, scb = m.weight.data, getattr(m.weight, "SCB", None)
            return (m.in_features % 128 == 0 and m.in_features <= Linear8bitLt.MAX_IN_FEATURES and cb.is_cuda
                    and cb.dtype == torch.int8 and cb.is_contiguous() and cb.data_ptr() % 16 == 0 and scb is not None
                    and scb.dtype == torch.float32 and scb.is_contiguous() and scb.device == cb.device)

        return all(ok(m) for m in self._linears())

    def logical_kv_caches(self) -> List[KVCache]:
        """kv_caches in the reference's slot order.  Identical to `kv_caches` until the
        roll branch (model.py:214-218) has triggered; afterwards the physical tensors are
        a ring and this returns the un-rotated copies the reference would hold.  An fp8 cache returns the values read
        back from it (float(code) * scale), as bf16."""
        out = []
        lib = L.lib()
        if self._kv_scale is not None:   # fp8: the values read back, bf16
            name = "b2l_kv8_unroll_rows" if self._ring.numel() > 1 else "b2l_kv8_unroll"
            unroll = getattr(lib, name)
            for c in self.kv_caches:
                B, nh, S, hs = c[0].shape
                pair = []
                for code, scale in ((c[0], c.k_scale), (c[1], c.v_scale)):
                    o = torch.empty((B, nh, S, hs), device=code.device, dtype=torch.bfloat16)
                    L.check(unroll(code.data_ptr(), scale.data_ptr(), self._ring.data_ptr(), o.data_ptr(), B, nh, S, hs,
                                   L.stream_ptr()), name)
                    pair.append(o)
                out.append(tuple(pair))
            return out
        name = "b2l_kv_unroll_rows" if self._ring.numel() > 1 else "b2l_kv_unroll"   # one ring offset per row, or shared
        unroll = getattr(lib, name)
        for k, v in self.kv_caches:
            B, nh, S, hs = k.shape
            ko, vo = torch.empty_like(k), torch.empty_like(v)
            L.check(unroll(k.data_ptr(), self._ring.data_ptr(), ko.data_ptr(), B, nh, S, hs, L.stream_ptr()), name)
            L.check(unroll(v.data_ptr(), self._ring.data_ptr(), vo.data_ptr(), B, nh, S, hs, L.stream_ptr()), name)
            out.append((ko, vo))
        return out

    # ------------------------------------------------------------------ forward
    def forward(
        self, idx: torch.Tensor, max_seq_length: Optional[int] = None, input_pos: Optional[torch.Tensor] = None
    ) -> Union[torch.Tensor, Tuple[torch.Tensor, List[KVCache]]]:
        B, T = idx.size()
        # a (B, 1) input_pos: one token per row, each at its own position with its own ring offset (B2L_F_ROW_POS);
        # at B == 1 that is the shared form
        rows = input_pos is not None and input_pos.dim() == 2
        if rows and (T != 1 or tuple(input_pos.shape) != (B, 1)):
            raise ValueError(f"LLaMA.forward: a 2-D input_pos is one position per row, shape ({B}, 1) for T == 1; got "
                             f"{tuple(input_pos.shape)} with T={T}")
        max_seq_length = self._prepare(idx, max_seq_length)
        if rows:
            if B == 1:
                input_pos, rows = input_pos.reshape(1), False
        elif input_pos is not None and self._ring.numel() > 1:
            raise RuntimeError("LLaMA.forward: the cache holds one position per row (prefill_rows); pass input_pos of "
                               "shape (B, 1), or reset_cache() first")

        if input_pos is not None and not self.kv_caches:
            self._new_kv_store(B, max_seq_length, idx.device)
            self._drop_steps()
        if input_pos is not None and T > 1 and self._kv_scale is not None:
            # an fp8 cache is prefilled from position 0 (one host read of the positions)
            if input_pos.numel() != T or not bool((input_pos.reshape(-1) == torch.arange(T, device=input_pos.device)).all()):
                raise ValueError("LLaMA.forward: an fp8 KV cache (kv_cache_dtype='fp8') takes a multi-token prompt at "
                                 "positions 0..T-1 only; a prefill at a nonzero position is not supported")
        if rows:
            if self._kv_store.shape[2] != B:
                raise ValueError(f"LLaMA.forward: {B} rows against a KV cache of {self._kv_store.shape[2]}")
            if self._ring.numel() != B:   # after expand_cache: every row starts from the shared ring offset
                self._set_ring(self._ring.expand(B).contiguous())

        # ---- decode: one C call per token, replayed as a CUDA graph
        st = None
        if input_pos is not None and T == 1 and B <= 16 and idx.dtype in (torch.int32, torch.int64):
            st = None if self._drop_stale(self._decode) else self._decode
            if (st is None or st.B != B or st.S != max_seq_length or st.idx.dtype != idx.dtype or st.idx.device != idx.device
                    or st.row_pos != rows or (st.lora_rows is None) != (self._lora_route is None)):
                route = self._decode_route(B)
                st = self._decode = (_DecodeState(self, route, B, max_seq_length, idx.device, idx.dtype, rows)
                                     if isinstance(route, _Route) else None)
        if st is not None:
            st.idx.copy_(idx.reshape(-1))
            st.pos.copy_(input_pos.reshape(-1) if rows else input_pos.reshape(-1)[-1:])
            if st.lora_rows is not None:   # multi-LoRA: each row's adapter, as the route gives it
                r = self._lora_route
                if r[0] == "segments":
                    raise RuntimeError("LLaMA.forward: a packed prefill's adapter segments do not decode")
                st.lora_rows.copy_(r[2].expand(B) if r[0] == "one" else r[1][:B])
            _graph_step(st, self.graph_after, st.enqueue)
            return st.logits.clone() if self.copy_logits else st.logits

        # ---- single-token decode the fused step does not run (llm.int8, grouped or biased gptq, dense, gptq.int8 at
        #      B >= 2): the module-by-module launch sequence, replayed as a CUDA graph once warm
        if input_pos is not None and T == 1 and self.graph_after and idx.dtype in (torch.int32, torch.int64):
            route = self._lora_route   # a multi-LoRA c_attn reads its adapter choice from the tensor the route names
            key = (B, max_seq_length, idx.dtype, idx.device, WEIGHTS_GENERATION[0],
                   None if route is None else (route[0], route[-1].data_ptr() if route[0] != "segments" else None), rows)
            mg = self._module_graph
            if mg is None or mg.key != key:
                mg = self._module_graph = _ModuleGraph(
                    key=key, calls=0, graph=None, idx=torch.zeros((B, 1), dtype=idx.dtype, device=idx.device),
                    pos=torch.zeros((B, 1) if rows else (1,), dtype=torch.int64, device=idx.device), out=None)
            mg.idx.copy_(idx)
            mg.pos.copy_(input_pos if rows else input_pos.reshape(-1)[-1:])
            def enqueue() -> None:
                mg.out = self._forward_modules(mg.idx, max_seq_length, mg.pos)
            _graph_step(mg, self.graph_after, enqueue)
            # the eager warm-up calls return a fresh tensor each; a graph's output is its static buffer
            return mg.out.clone() if self.copy_logits and mg.graph is not None else mg.out
        return self._forward_modules(idx, max_seq_length, input_pos)

    @torch.no_grad()
    def decode_tokens(self, idx: torch.Tensor, max_seq_length: int, input_pos: torch.Tensor) -> torch.Tensor:
        """Run T = 2..16 consecutive tokens of ONE sequence through the whole-token decode step in one call (the verify
        step of speculative decoding): idx (1, T) at positions input_pos (T,) = p..p+T-1, all < max_seq_length, on the
        batch-1 KV cache.  Returns (T, vocab) logits; row t equals, bit for bit, the logits `forward` returns for token t
        alone at input_pos[t] after tokens 0..t-1 (b2l_decode_step under B2L_F_STEPWISE: the row-exact batch linears
        and, per query, the attention of a T == 1 launch), and the cache ends as those T batch-1 steps leave it.

        gptq.int4 and gptq.int8 models the fused batch-1 step runs (compacted or not, plain, LLaMA-Adapter v1 or LoRA);
        dense, llm.int8, LLaMA-Adapter v2 and grouped or biased gptq models are refused.  One step state per T, each
        replayed as its own CUDA graph."""
        if idx.dim() != 2 or idx.shape[0] != 1 or not 2 <= idx.shape[1] <= 16:
            raise ValueError(f"decode_tokens: idx must be (1, T) with T in 2..16, got {tuple(idx.shape)}")
        T = idx.shape[1]
        if input_pos.dim() != 1 or input_pos.numel() != T:
            raise ValueError(f"decode_tokens: input_pos must be ({T},), got {tuple(input_pos.shape)}")
        if idx.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"decode_tokens: idx dtype {idx.dtype}; int32 or int64")
        max_seq_length = self._prepare(idx, max_seq_length)
        route = self._decode_route(T, stepwise=True)
        if isinstance(route, str):
            raise RuntimeError(f"decode_tokens: {route}")
        if self._ring.numel() != 1 or (self._kv_store is not None and self._kv_store.shape[2] != 1):
            raise RuntimeError("decode_tokens: the KV cache holds more than one sequence; reset_cache() first")
        if not self.kv_caches:
            self._new_kv_store(1, max_seq_length, idx.device)
            self._drop_steps()
        if self._kv_store.shape[4] != max_seq_length:
            raise ValueError(f"decode_tokens: max_seq_length={max_seq_length} against a cache of {self._kv_store.shape[4]}")
        st = self._verify.get(T)
        if self._drop_stale(st) or (st is not None and (st.idx.dtype != idx.dtype or st.idx.device != idx.device)):
            self._verify, self._fast_ok = {}, None   # weight pointers or the step's inputs changed
            return self.decode_tokens(idx, max_seq_length, input_pos)
        if st is None:
            st = self._verify[T] = _DecodeState(self, route, T, max_seq_length, idx.device, idx.dtype, stepwise=True)
        st.idx.copy_(idx.reshape(-1))
        st.pos.copy_(input_pos)
        _graph_step(st, self.graph_after, st.enqueue)
        out = st.logits.view(T, -1)
        return out.clone() if self.copy_logits else out

    def _decode_route(self, B: int, stepwise: bool = False) -> Union[_Route, str]:
        """The route b2l_decode_step runs B rows on (stepwise: decode_tokens' B consecutive tokens of one sequence), or
        why the fused step does not run them: forward then goes module by module, and decode_tokens refuses with it.
        The one place the Python side picks the step's kernels (csrc/api.cu resolve_route reads the flags it sets)."""
        from . import quantization

        if stepwise and (self._kv_cache_dtype == "fp8" or self._kv_scale is not None):
            return "does not run on an fp8 KV cache (kv_cache_dtype='fp8'): speculative verify keeps a bf16 cache"
        if self._fast_ok is None:
            self._fast_ok = self._fast_decode_ok()
        kind, affines = self._fast_ok, self._has_affines()
        if stepwise:   # the row-exact batch kernels whatever the opt-ins say: each row must equal the batch-1 step
            if kind in ("q4", "w8") and not affines:
                return _ROUTES["q4_batch_i8" if kind == "q4" else "w8_batch"]
            return ("needs a gptq.int4 or gptq.int8 model the fused decode step runs with its row-exact batch kernels "
                    "(not dense, llm.int8, LLaMA-Adapter v2, or grouped / biased gptq)")
        if kind == "q8" and self.int8_step:   # LLaMA-Adapter v2 affines at any B
            return _ROUTES["q8" if B == 1 else "q8_batch"]
        if kind in ("q4", "w8") and B == 1:
            return _ROUTES[kind + "_gemv"]
        if kind == "w8" and self.w8_batch_step and not affines:
            return _ROUTES["w8_batch"]
        if kind == "q4" and not affines:
            return _ROUTES["q4_batch_i8" if self.q4_batch_step else
                           "q4_batch" if B <= 8 and quantization.BATCH_GEMV else "q4_tc"]
        return f"the fused step runs no route for this model at batch {B} with these opt-ins"

    def _prepare(self, idx: torch.Tensor, max_seq_length: Optional[int]) -> int:
        """model.py:79-91: the shape checks, and the RoPE table and KV ring on idx's device.  Returns max_seq_length."""
        B, T = idx.size()
        if not idx.is_cuda:
            raise RuntimeError(f"LLaMA.forward: idx is on {idx.device}; lit_llama_b200 runs on CUDA only (no CPU fallback)")

        block_size = self.config.block_size
        if max_seq_length is None:
            max_seq_length = block_size
        assert T <= max_seq_length, f"Cannot forward sequence of length {T}, max seq length is only {max_seq_length}"
        assert max_seq_length <= block_size, f"Cannot attend to {max_seq_length}, block size is only {block_size}"
        assert T <= block_size, f"Cannot forward sequence of length {T}, block size is only {block_size}"

        if self.rope_cache is None or self.rope_cache.device != idx.device:
            self.rope_cache = self.build_rope_cache(idx).float().contiguous()
        if self._ring is None or self._ring.device != idx.device:
            self._set_ring(torch.zeros(1, dtype=torch.int32, device=idx.device))
        return max_seq_length

    def _forward_modules(self, idx: torch.Tensor, max_seq_length: int, input_pos: Optional[torch.Tensor]) -> torch.Tensor:
        """Prefill, no-cache forward and non-fused decode: one kernel (or two) per reference module."""
        return self.lm_head(self._forward_hidden(idx, max_seq_length, input_pos))  # (b, t, vocab_size)

    def _forward_hidden(self, idx: torch.Tensor, max_seq_length: int, input_pos: Optional[torch.Tensor],
                        ragged: Optional[L.Ragged] = None) -> torch.Tensor:
        """_forward_modules up to lm_head's input: the embedding, the Blocks and ln_f (lit_llama_b200.evaluate runs
        lm_head with the loss in its epilogue instead).  `ragged`: idx (1, N) holds the packed prompts of refill_rows."""
        B, T = idx.size()
        x = torch.empty((B, T, self.config.n_embd), device=idx.device, dtype=torch.bfloat16)
        wte = self.transformer.wte.weight
        if wte.dtype != torch.bfloat16:
            raise RuntimeError(f"wte dtype {wte.dtype} unsupported; the model must be bf16 (model.to(torch.bfloat16))")
        idx_c = idx.contiguous()
        if idx_c.dtype not in (torch.int32, torch.int64):
            idx_c = idx_c.to(torch.int64)
        rc = L.lib().b2l_embedding(idx_c.data_ptr(), 1 if idx_c.dtype == torch.int64 else 0, wte.data_ptr(), x.data_ptr(),
                                   B * T, self.config.n_embd, wte.shape[0], L.stream_ptr())
        L.check(rc, "b2l_embedding")

        if ragged is not None:
            for i, block in enumerate(self.transformer.h):
                x, _ = block(x, self.rope_cache, None, max_seq_length, None, self.kv_caches[i], _rope_is_table=True,
                             _ragged=ragged)
        elif input_pos is None:  # proxy for use_cache=False (model.py:104-106)
            for block in self.transformer.h:
                x, _ = block(x, self.rope_cache, None, max_seq_length, _rope_is_table=True)
        else:
            pos = input_pos.reshape(-1).to(torch.int64)
            if input_pos.dim() == 2:   # one position per row (T == 1): each row's ring advances on its own
                L.check(L.lib().b2l_ring_advance_rows(pos.data_ptr(), B, self._ring.data_ptr(), max_seq_length, L.stream_ptr()),
                        "b2l_ring_advance_rows")
                pos = pos.view(B, 1)
            else:
                L.check(L.lib().b2l_ring_advance(pos.data_ptr(), T, self._ring.data_ptr(), max_seq_length, L.stream_ptr()), "b2l_ring_advance")
            for i, block in enumerate(self.transformer.h):
                x, self.kv_caches[i] = block(x, self.rope_cache, None, max_seq_length, pos, self.kv_caches[i], _rope_is_table=True)

        return self.transformer.ln_f(x)

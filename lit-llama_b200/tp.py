"""Tensor-parallel decode across GPUs of one node (SURVEY.md section 8e; new capability - the
reference has no multi-GPU inference, every script is `L.Fabric(devices=1)`).

Megatron-style sharding of the reference Block (split dims as recorded by the reference's own
checkpoint converter, scripts/convert_checkpoint.py:56-64):

  c_attn    (3C, C)   column-parallel BY HEADS inside each of q, k, v   -> local [q_r; k_r; v_r]
  attention           local heads, local KV cache
  attn.c_proj (C, C)  row-parallel over `in` (the local heads' slice)   -> all-reduce(sum)
  c_fc1/c_fc2         column-parallel
  mlp.c_proj          row-parallel                                       -> all-reduce(sum)
  lm_head   (V, C)    column-parallel + all-gather of the logits
  wte, RMSNorm scales replicated

Two all-reduces per Block are needed for exact semantics (rms_2 needs the full post-attention
residual, model.py:165-167).  One process per GPU, `torch.distributed` (NCCL over NVLink) for the
exchange; every local op is the same kernel the single-GPU path uses (include/b2l.h).  Row-parallel
int4 linears keep their per-row scale/zero on every rank: `y = s*(sum_k lv*x - z*sum_k x)` is linear in
the K slice, so each rank's kernel uses its LOCAL sum(x) and the partial results simply add.

The per-rank partial products are rounded to bf16 before the reduction (the kernels' output
dtype), so a TP result can differ from the single-GPU one by one bf16 ulp per reduction.
"""
import ctypes as C
import os
import sys
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib as L
from .model import LLaMAConfig, RMSNorm, _add, _fc12_weights, _graph_step, build_rope_cache
from .quantization import ColBlockQuantizedLinear


# ----------------------------------------------------------------------------- sharding (host logic, any device)
def _rows(t: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    return t.index_select(0, idx.to(t.device))


def shard_linear(sd: Dict[str, torch.Tensor], prefix: str, *, rows: Optional[torch.Tensor] = None,
                 k_range: Optional[Tuple[int, int]] = None) -> Dict[str, torch.Tensor]:
    """One linear of a reference-format gptq.int4 state dict, restricted to output `rows`
    (column-parallel) or to the input range `k_range` (row-parallel).  Packed weights keep
    the reference layout (uint8 (out, in/2), strides (1, out))."""
    qw, sc, z = sd[prefix + ".quant_weight"], sd[prefix + ".scales"], sd[prefix + ".zeros"]
    if sc.shape[1] != 1:
        raise RuntimeError("tensor parallelism supports one (scale, zero) per output row (gptq.int4 as produced by --quantize gptq.int4)")
    if rows is not None:
        qw, sc, z = _rows(qw, rows), _rows(sc, rows), _rows(z, rows)
    if k_range is not None:
        k0, k1 = k_range
        assert k0 % 2 == 0 and k1 % 2 == 0
        qw = qw[:, k0 // 2 : k1 // 2]
    return {prefix + ".quant_weight": qw.t().contiguous().t(), prefix + ".scales": sc.contiguous(), prefix + ".zeros": z.contiguous()}


def shard_state_dict(sd: Dict[str, torch.Tensor], rank: int, world: int, n_head: int) -> Dict[str, torch.Tensor]:
    """The slice of a full gptq.int4 checkpoint that rank `rank` of `world` holds."""
    C = sd["transformer.wte.weight"].shape[1]
    V = sd["lm_head.scales"].shape[0]
    assert n_head % world == 0 and V % world == 0, "n_head and the padded vocabulary must divide by the TP degree"
    hs = C // n_head
    nh_l = n_head // world
    heads = torch.arange(rank * nh_l, (rank + 1) * nh_l)
    head_rows = (heads.unsqueeze(1) * hs + torch.arange(hs).unsqueeze(0)).reshape(-1)  # rows of one of q/k/v for the local heads
    qkv_rows = torch.cat([head_rows, C + head_rows, 2 * C + head_rows])
    out: Dict[str, torch.Tensor] = {}
    n_layer = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer.h."))
    for i in range(n_layer):
        p = f"transformer.h.{i}."
        nh = sd[p + "mlp.c_fc1.scales"].shape[0]
        assert nh % world == 0
        f_rows = torch.arange(rank * (nh // world), (rank + 1) * (nh // world))
        out.update(shard_linear(sd, p + "attn.c_attn", rows=qkv_rows))
        out.update(shard_linear(sd, p + "attn.c_proj", k_range=(rank * nh_l * hs, (rank + 1) * nh_l * hs)))
        out.update(shard_linear(sd, p + "mlp.c_fc1", rows=f_rows))
        out.update(shard_linear(sd, p + "mlp.c_fc2", rows=f_rows))
        out.update(shard_linear(sd, p + "mlp.c_proj", k_range=(rank * (nh // world), (rank + 1) * (nh // world))))
        out[p + "rms_1.scale"] = sd[p + "rms_1.scale"]
        out[p + "rms_2.scale"] = sd[p + "rms_2.scale"]
    out.update(shard_linear(sd, "lm_head", rows=torch.arange(rank * (V // world), (rank + 1) * (V // world))))
    out["transformer.wte.weight"] = sd["transformer.wte.weight"]
    out["transformer.ln_f.scale"] = sd["transformer.ln_f.scale"]
    return out


# ----------------------------------------------------------------------------- the sharded model
def _q4(in_f: int, out_f: int) -> ColBlockQuantizedLinear:
    return ColBlockQuantizedLinear(in_f, out_f, False, bits=4, tile_cols=-1)


class _TPAttention(nn.Module):
    def __init__(self, C: int, C_l: int) -> None:
        super().__init__()
        self.c_attn = _q4(C, 3 * C_l)
        self.c_proj = _q4(C_l, C)


class _TPMLP(nn.Module):
    def __init__(self, C: int, nh_l: int) -> None:
        super().__init__()
        self.c_fc1 = _q4(C, nh_l)
        self.c_fc2 = _q4(C, nh_l)
        self.c_proj = _q4(nh_l, C)


class _TPBlock(nn.Module):
    def __init__(self, C: int, C_l: int, nh_l: int) -> None:
        super().__init__()
        self.rms_1 = RMSNorm(C)
        self.attn = _TPAttention(C, C_l)
        self.rms_2 = RMSNorm(C)
        self.mlp = _TPMLP(C, nh_l)


class _TPDecodeState:
    """Batch-1 decode step of one rank as a fixed launch sequence over static buffers (captured once into a CUDA graph,
    all-reduces included: b2l_tp_allreduce over peer memory, or NCCL when that is unavailable): the single-GPU path's fused kernels on the local shards --
      [rms_1 + c_attn(local heads)] -> fused attention (local heads) -> [c_proj (K = local heads) (+ residual on rank 0)]
      -> all-reduce -> [rms_2 + c_fc1|c_fc2 (local columns) + SwiGLU] -> [mlp.c_proj (K = local columns) (+ residual on
      rank 0)] -> all-reduce; finally [ln_f + lm_head (local vocabulary rows)] -> all-gather.
    The residual enters the sum exactly once (rank 0's epilogue), so all-reduce(sum) leaves x + sum_r partial_r on every
    rank (model.py:166-167).  Two all-reduces per Block (SURVEY section 7.6)."""

    def __init__(self, m: "TPLLaMA", S: int, dev: torch.device, idx_dtype: torch.dtype) -> None:
        cfg, lib = m.config, L.lib()
        Cd, hs, nh_l, world = cfg.n_embd, m.hs, m.nh_l, m.world
        C_l = nh_l * hs
        bf = dict(device=dev, dtype=torch.bfloat16)
        self.idx = torch.zeros(1, dtype=idx_dtype, device=dev)
        self.pos = torch.zeros(1, dtype=torch.int64, device=dev)
        self.x = torch.empty((1, Cd), **bf)
        self.qkv = torch.empty((1, 3 * C_l), **bf)
        self.att = torch.empty((1, C_l), **bf)
        hid_l = m.transformer.h[0].mlp.c_fc1.out_features
        self.hid = torch.empty((1, hid_l), **bf)
        V_l = m.lm_head.out_features
        self.logits_l = torch.empty((1, V_l), **bf)
        self.logits = torch.empty((world, V_l), **bf)
        self.work = torch.zeros(lib.b2l_attn_workspace_bytes(1, nh_l, hs, 1, S) // 4 + 1, device=dev, dtype=torch.float32)
        self.keep: List[torch.Tensor] = []
        szd = L.sz_dtype_of(m.lm_head.scales)
        eps = float(m.transformer.ln_f.eps)

        def bf16(p: torch.Tensor) -> torch.Tensor:
            t = p.detach()
            if t.dtype != torch.bfloat16:
                t = t.to(torch.bfloat16)
            self.keep.append(t)
            return t

        def gemv(tiled, scales, zeros, N, K, x, y, pro, ns, epi, res):
            self.keep += [tiled, scales, zeros]
            return L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=tiled.data_ptr(), scales=scales.data_ptr(), zeros=zeros.data_ptr(),
                                  sz_dtype=szd, y=y.data_ptr(), ldy=N, M=1, N=N, K=K, prologue=pro,
                                  norm_scale=None if ns is None else ns.data_ptr(), eps=eps, epilogue=epi,
                                  res=None if res is None else res.data_ptr(), ldres=N, split_k=0, flags=L.F_PDL)

        def lin(l: ColBlockQuantizedLinear, x, y, pro=L.PRO_NONE, ns=None, epi=L.EPI_STORE, res=None):
            return gemv(l.tiled_i8(), l.scales, l.zeros, l.out_features, l.in_features, x, y, pro, ns, epi, res)

        rank0 = m.rank == 0
        self.ops = []   # ("gemv", args) | ("attn", layer index) | ("allreduce", tensor) | ("allgather",)
        for i, blk in enumerate(m.transformer.h):
            self.ops.append(("gemv", lin(blk.attn.c_attn, self.x, self.qkv, L.PRO_RMSNORM, bf16(blk.rms_1.scale))))
            self.ops.append(("attn", i))
            self.ops.append(("gemv", lin(blk.attn.c_proj, self.att, self.x, epi=L.EPI_RESIDUAL if rank0 else L.EPI_STORE, res=self.x if rank0 else None)))
            self.ops.append(("allreduce", self.x))
            t, sc, z = _fc12_weights(blk.mlp, blk.mlp.c_fc1.quant_weight, blk.mlp.c_fc2.quant_weight, "i8")
            self.ops.append(("gemv", gemv(t, sc, z, 2 * hid_l, Cd, self.x, self.hid, L.PRO_RMSNORM, bf16(blk.rms_2.scale), L.EPI_SWIGLU, None)))
            self.ops.append(("gemv", lin(blk.mlp.c_proj, self.hid, self.x, epi=L.EPI_RESIDUAL if rank0 else L.EPI_STORE, res=self.x if rank0 else None)))
            self.ops.append(("allreduce", self.x))
        self.ops.append(("gemv", lin(m.lm_head, self.x, self.logits_l, L.PRO_RMSNORM, bf16(m.transformer.ln_f.scale))))
        self.ops.append(("allgather",))
        self.m, self.S = m, S
        self.comm = m.tp_comm(dev)
        self.wte = bf16(m.transformer.wte.weight)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.calls = 0
        self.n_kernels = sum(1 for o in self.ops if o[0] in ("gemv", "attn")) + 2

    def enqueue(self) -> None:
        m, lib, sp = self.m, L.lib(), L.stream_ptr()
        cfg = m.config
        L.check(lib.b2l_ring_advance(self.pos.data_ptr(), 1, m._ring.data_ptr(), self.S, sp), "b2l_ring_advance")
        L.check(lib.b2l_embedding(self.idx.data_ptr(), 1 if self.idx.dtype == torch.int64 else 0, self.wte.data_ptr(), self.x.data_ptr(), 1,
                                  cfg.n_embd, self.wte.shape[0], sp), "b2l_embedding")
        for op in self.ops:
            if op[0] == "gemv":
                L.check(lib.b2l_q4_gemv(C.byref(op[1]), sp), "b2l_q4_gemv")
            elif op[0] == "attn":
                k_c, v_c = m.kv_caches[op[1]]
                L.check(lib.b2l_attention(self.qkv.data_ptr(), k_c.data_ptr(), v_c.data_ptr(), m.rope_cache.data_ptr(), self.pos.data_ptr(),
                                          m._ring.data_ptr(), self.att.data_ptr(), self.work.data_ptr(), 1, 1, m.nh_l, m.hs, self.S,
                                          cfg.block_size, L.F_PDL, sp), "b2l_attention")
            elif op[0] == "allreduce":
                if self.comm is not None:   # one-shot sum over peer memory (NVLink), in place, inside the PDL chain
                    L.check(lib.b2l_tp_allreduce(C.byref(self.comm), op[1].data_ptr(), op[1].data_ptr(), op[1].numel(), L.F_PDL, sp),
                            "b2l_tp_allreduce")
                elif m.world > 1:
                    dist.all_reduce(op[1], op=dist.ReduceOp.SUM, group=m.group)
            else:
                if m.world > 1:
                    dist.all_gather_into_tensor(self.logits, self.logits_l, group=m.group)
                else:
                    self.logits.copy_(self.logits_l)


class TPLLaMA(nn.Module):
    """LLaMA.forward (model.py:76-122) with every quantized linear sharded over `group`.
    State-dict keys equal the reference's, so `load_state_dict(shard_state_dict(full, rank, world, n_head))` works."""

    def __init__(self, config: LLaMAConfig, rank: int, world: int, n_hidden: int, group=None) -> None:
        super().__init__()
        assert config.n_head % world == 0 and n_hidden % world == 0 and config.padded_vocab_size % world == 0
        self.config, self.rank, self.world, self.group = config, rank, world, group
        C = config.n_embd
        self.hs = C // config.n_head
        self.nh_l = config.n_head // world
        C_l = self.nh_l * self.hs
        self.lm_head = _q4(C, config.padded_vocab_size // world)
        self.transformer = nn.ModuleDict(dict(
            wte=nn.Embedding(config.padded_vocab_size, C),
            h=nn.ModuleList(_TPBlock(C, C_l, n_hidden // world) for _ in range(config.n_layer)),
            ln_f=RMSNorm(C),
        ))
        self.rope_cache: Optional[torch.Tensor] = None
        self.kv_caches: List[Tuple[torch.Tensor, torch.Tensor]] = []
        self._ring: Optional[torch.Tensor] = None
        self._work: Optional[torch.Tensor] = None
        self._decode: Optional[_TPDecodeState] = None
        #: replay the batch-1 decode step as a CUDA graph (NCCL collectives included) after this many eager steps (0 = never)
        self.graph_after = 2
        #: fused per-rank decode step (batch 1, head_size 128, K % 64 == 0); False: module by module
        self.fast_decode = True
        self._comm, self._comm_keep, self._comm_tried = None, None, False

    def reset_cache(self) -> None:
        self.kv_caches.clear()
        self._decode = None
        if self._ring is not None:
            self._ring.zero_()

    @property
    def kv_cache_dtype(self) -> None:
        """Always None: the tensor-parallel step keeps a bf16 KV cache (LLaMA.kv_cache_dtype)."""
        return None

    @kv_cache_dtype.setter
    def kv_cache_dtype(self, value) -> None:
        if value is not None:
            raise ValueError(f"TPLLaMA.kv_cache_dtype: {value!r} is not supported; the tensor-parallel decode step keeps "
                             "a bf16 KV cache")

    def tp_comm(self, dev: torch.device) -> Optional["L.TPComm"]:
        """The peer-memory exchange of b2l_tp_allreduce (csrc/tp_allreduce.cu), created once per model (a collective
        call: every rank must get here).  Buffers come from torch's symmetric memory -- allocation + peer mapping
        only, the all-reduce itself is this library's kernel.  None when world == 1, when B2L_TP_ALLREDUCE=nccl, or
        when the peer mapping is unavailable (said once on stderr): the step then uses NCCL all-reduces."""
        if self._comm_tried:
            return self._comm
        self._comm_tried = True
        if self.world == 1 or os.environ.get("B2L_TP_ALLREDUCE", "ll") == "nccl":
            return None
        lib = L.lib()
        C_ = self.config.n_embd
        try:
            import torch.distributed._symmetric_memory as symm

            nbytes = lib.b2l_tp_buffer_bytes(self.world, C_)
            buf = symm.empty(nbytes, dtype=torch.uint8, device=dev)
            buf.zero_()
            hdl = symm.rendezvous(buf, self.group if self.group is not None else dist.group.WORLD)
            ptrs = [int(p) for p in hdl.buffer_ptrs]
            assert len(ptrs) == self.world
        except Exception as e:  # noqa: BLE001 -- any failure of the optional peer mapping selects the NCCL path, loudly
            print(f"[lit_llama_b200.tp] peer-memory exchange unavailable ({type(e).__name__}: {e}); using NCCL all-reduces", file=sys.stderr, flush=True)
            return None
        words = torch.zeros(32, dtype=torch.int32, device=dev)   # [0..15] epochs, [16] status
        comm = L.TPComm()
        for r in range(self.world):
            comm.peer_buf[r] = ptrs[r]
        comm.rank, comm.world, comm.max_elems = self.rank, self.world, C_
        comm.epoch, comm.status = words.data_ptr(), words.data_ptr() + 64
        self._comm, self._comm_keep = comm, (buf, hdl, words)
        torch.cuda.synchronize(dev)
        dist.barrier(group=self.group)   # every rank's buffer is zeroed before anyone pushes
        return comm

    def tp_check(self) -> None:
        """Raises if a bounded wait inside b2l_tp_allreduce ever timed out (a peer stopped issuing its calls)."""
        if self._comm is not None:
            torch.cuda.synchronize()
            if int(self._comm_keep[2][16]) != 0:
                raise RuntimeError("b2l_tp_allreduce: a wait for a peer's partial row timed out; results are invalid")

    def _all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    @torch.no_grad()
    def forward(self, idx: torch.Tensor, max_seq_length: Optional[int] = None, input_pos: Optional[torch.Tensor] = None) -> torch.Tensor:
        B, T = idx.shape
        if not idx.is_cuda:
            raise RuntimeError("TPLLaMA.forward: CUDA only (no CPU fallback)")
        if input_pos is None:
            raise RuntimeError("TPLLaMA implements the KV-cache path (input_pos given), which is what generate() uses")
        cfg, dev, lib = self.config, idx.device, L.lib()
        S = cfg.block_size if max_seq_length is None else max_seq_length
        C, hs, nh_l = cfg.n_embd, self.hs, self.nh_l
        if self.rope_cache is None:
            self.rope_cache = build_rope_cache(cfg.block_size, hs, idx.dtype, dev).float().contiguous()
        if self._ring is None:
            self._ring = torch.zeros(1, dtype=torch.int32, device=dev)
        if not self.kv_caches:
            shape = (B, nh_l, S, hs)
            self.kv_caches = [(torch.zeros(shape, device=dev, dtype=torch.bfloat16), torch.zeros(shape, device=dev, dtype=torch.bfloat16))
                              for _ in range(cfg.n_layer)]
            self._work = torch.zeros(lib.b2l_attn_workspace_bytes(B, nh_l, hs, T, S) // 4 + 1, device=dev, dtype=torch.float32)
        if self._work.numel() * 4 < lib.b2l_attn_workspace_bytes(B, nh_l, hs, T, S):
            self._work = torch.zeros(lib.b2l_attn_workspace_bytes(B, nh_l, hs, T, S) // 4 + 1, device=dev, dtype=torch.float32)
        pos = input_pos.reshape(-1).to(torch.int64)
        wte = self.transformer.wte.weight
        if wte.dtype != torch.bfloat16:
            raise RuntimeError("TPLLaMA: the model must be bf16")
        # ---- batch-1 decode: the fused per-rank step, graph-replayed
        C_l, hid_l = nh_l * hs, self.transformer.h[0].mlp.c_fc1.out_features
        if (self.fast_decode and B == 1 and T == 1 and hs == 128 and C % 64 == 0 and C_l % 64 == 0 and hid_l % 64 == 0 and hid_l % 8 == 0
                and self.lm_head.out_features % 16 == 0 and idx.dtype in (torch.int32, torch.int64) and self.lm_head.gemv_capable):
            st = self._decode
            if st is None or st.S != S or st.idx.dtype != idx.dtype:
                st = self._decode = _TPDecodeState(self, S, dev, idx.dtype)
            st.idx.copy_(idx.reshape(-1))
            st.pos.copy_(pos[-1:])
            _graph_step(st, self.graph_after, st.enqueue)
            return st.logits.reshape(1, 1, -1).clone()
        idx_c = idx.contiguous() if idx.dtype in (torch.int32, torch.int64) else idx.to(torch.int64).contiguous()
        x = torch.empty((B, T, C), device=dev, dtype=torch.bfloat16)
        L.check(lib.b2l_embedding(idx_c.data_ptr(), 1 if idx_c.dtype == torch.int64 else 0, wte.data_ptr(), x.data_ptr(), B * T, C,
                                  wte.shape[0], L.stream_ptr()), "b2l_embedding")
        L.check(lib.b2l_ring_advance(pos.data_ptr(), T, self._ring.data_ptr(), S, L.stream_ptr()), "b2l_ring_advance")
        for i, blk in enumerate(self.transformer.h):
            qkv = blk.attn.c_attn(blk.rms_1(x)).contiguous()               # (B, T, 3*C_l): local heads of q | k | v
            k_c, v_c = self.kv_caches[i]
            y = torch.empty((B, T, nh_l * hs), device=dev, dtype=torch.bfloat16)
            rc = lib.b2l_attention(qkv.data_ptr(), k_c.data_ptr(), v_c.data_ptr(), self.rope_cache.data_ptr(), pos.data_ptr(),
                                   self._ring.data_ptr(), y.data_ptr(), self._work.data_ptr(), B, T, nh_l, hs, S, cfg.block_size, 0,
                                   L.stream_ptr())
            L.check(rc, "b2l_attention")
            x = _add(x, self._all_reduce(blk.attn.c_proj(y)))              # row-parallel partials -> sum  (model.py:166)
            h = blk.rms_2(x)
            a, b = blk.mlp.c_fc1(h).contiguous(), blk.mlp.c_fc2(h).contiguous()
            g = torch.empty_like(a)
            L.check(lib.b2l_silu_mul(a.data_ptr(), b.data_ptr(), g.data_ptr(), a.numel(), L.stream_ptr()), "b2l_silu_mul")
            x = _add(x, self._all_reduce(blk.mlp.c_proj(g)))               # (model.py:167)
        logits_l = self.lm_head(self.transformer.ln_f(x)).contiguous()     # (B, T, V / world)
        if self.world == 1:
            return logits_l
        parts = [torch.empty_like(logits_l) for _ in range(self.world)]
        dist.all_gather(parts, logits_l, group=self.group)
        return torch.cat(parts, dim=-1)

"""Drop-in quantized linears (reference: lit_llama/quantization.py).

`ColBlockQuantizedLinear` keeps the reference's constructor, attributes, buffers
(names, shapes, dtypes, strides) and `state_dict` keys (quantization.py:340-374), so a
`llama-gptq.4bit.pth` produced by the reference's quantize/gptq.py loads unchanged.
`forward` runs hand-written sm_90a kernels through the C ABI of include/b2l.h (M = 1: exact int8-digit MMA GEMV;
2..8: f16 MMA batch kernel; 9..16: wgmma with weights from registers; > 16: wgmma 128 x 128 tile GEMM; gptq.int8:
the same GEMV at M = 1 and the same GEMM for M >= 2); there is no Triton, no library GEMM, no dense fallback and no
CPU path.
"""
import ctypes as C
import os
from typing import Optional

import torch

from . import _lib as L


# 2..8 activation rows go through the mma.sync batch kernel (B2L_BATCH_GEMV=0: wgmma kernel instead)
BATCH_GEMV = os.environ.get("B2L_BATCH_GEMV", "1") != "0"
_BATCH_WS = {}
_BATCH_WS_OLD = []

#: bumped whenever a quantized linear's storage may have changed (load_state_dict, pack_weight, .to()/_apply): the
#: decode state of LLaMA bakes raw pointers to the re-tiled weights into a C argument block / CUDA graph and rebuilds
#: when this differs from the value it was built at
WEIGHTS_GENERATION = [0]


def weights_changed() -> None:
    WEIGHTS_GENERATION[0] += 1


def batch_workspace(device, K: int) -> torch.Tensor:
    """Scratch of b2l_q4_gemv_batch (activation fragments), one per device, grown to the largest K seen.
    Launches of one stream are serialised, so every layer can share it."""
    need = L.lib().b2l_q4_gemv_batch_workspace_bytes(int(K))
    ws = _BATCH_WS.get(device)
    if ws is None or ws.numel() < need:
        if ws is not None:
            _BATCH_WS_OLD.append(ws)  # captured CUDA graphs may still point at it: never freed
        ws = _BATCH_WS[device] = torch.zeros(need, dtype=torch.uint8, device=device)
    return ws


class ColBlockQuantizedLinear(torch.nn.Module):
    """Weight-only int4 / int8 linear with per-row (or per column-group) scale and zero.

    Same signature as the reference class (quantization.py:340-374).  Storage:
    `quant_weight` uint8 (out, in/epb) with strides (1, out); entry nr of a byte holds
    column epb*j+nr at bit nr*bits (quantization.py:386-390).  `scales`/`zeros`
    (out, ceil(in/tile_cols)) in the default dtype; `bias` (out,) or None.
    """

    def __init__(self, in_features, out_features, bias: bool, *, bits, tile_cols):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        self.tile_cols = tile_cols if tile_cols != -1 else self.in_features
        self.bits = bits
        self.entries_per_byte = 8 // bits
        assert self.entries_per_byte > 0 and self.entries_per_byte * self.bits == 8
        assert in_features % self.entries_per_byte == 0
        self.register_buffer(
            "quant_weight",
            torch.empty((self.out_features, self.in_features // self.entries_per_byte), dtype=torch.uint8).t().contiguous().t(),
        )
        n_groups = (self.in_features + self.tile_cols - 1) // self.tile_cols
        self.register_buffer("scales", torch.empty((self.out_features, n_groups)))
        self.register_buffer("zeros", torch.empty_like(self.scales))
        assert isinstance(bias, bool)
        if bias:
            self.register_buffer("bias", torch.empty((self.out_features,)))
        else:
            self.register_buffer("bias", None)
        self._tiled = None        # load-time re-tilings for the kernels (not part of state_dict)
        self._tiled_key = None
        self._tiled_mma = None
        self._tiled_mma_key = None
        self._tiled_i8 = None
        self._tiled_i8_key = None
        self._released = False    # reference-layout buffer freed (release_reference_layout): one copy of the weights
        self._source = None       # released + no own tiling: callable returning the reference-layout tensor
        self._half = None         # ... and (callable returning the interleaved tiling that holds it, 0 / 1: which half)

    # ------------------------------------------------------------------ packing (load-time, any device)
    def pack_weight(self, weight):
        """quantization.py:376-390: weight = scale * (level - zero) -> packed levels."""
        weight = weight.to(device=self.quant_weight.device, copy=True)
        for j in range(self.scales.size(1)):
            sl = slice(j * self.tile_cols, (j + 1) * self.tile_cols)
            weight[:, sl] /= self.scales[:, j : j + 1]
            weight[:, sl] += self.zeros[:, j : j + 1]
        weight = weight.clamp_(min=0, max=2**self.bits - 1).to(dtype=torch.uint8)
        self.quant_weight.zero_()
        for nr in range(self.entries_per_byte):
            self.quant_weight += weight[:, nr :: self.entries_per_byte] << (nr * self.bits)
        self._tiled = self._tiled_mma = self._tiled_i8 = None
        weights_changed()

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # a checkpoint with this layer's levels is coming: the buffer it is copied into has to exist again.  A dict
        # without them (e.g. adapter weights loaded with strict=False) leaves a compacted layer's only copy alone.
        if self._released and prefix + "quant_weight" in state_dict:
            self.quant_weight = torch.empty((self.in_features // self.entries_per_byte, self.out_features), dtype=torch.uint8,
                                            device=self.scales.device).t()
            self._released, self._source, self._half = False, None, None
            self._tiled = self._tiled_mma = self._tiled_i8 = None
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)   # copies in place: pointers stay, contents (and _version) change
        weights_changed()

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        if self._released:   # checkpoints keep the reference's layout: rebuilt from the kernel tiling (a permutation)
            destination[prefix + "quant_weight"] = self.reference_quant_weight()

    # ------------------------------------------------------------------ one resident copy of the weights
    def reference_quant_weight(self) -> torch.Tensor:
        """`quant_weight` in the reference layout (uint8 (out, in/epb), strides (1, out), quantization.py:350-359).  The
        registered buffer itself unless release_reference_layout() freed it: then a TRANSIENT tensor rebuilt from the
        batch-1 kernel's tiling (b2l_q4_untile_i8 / b2l_w8_untile_i8: pure permutations, tested bit-exact) or by
        `_source`."""
        if not self._released:
            return self.quant_weight
        if self._source is not None:
            return self._source()
        out = torch.empty((self.in_features // self.entries_per_byte, self.out_features), dtype=torch.uint8,
                          device=self._tiled_i8.device).t()
        name = "b2l_w8_untile_i8" if self.bits == 8 else "b2l_q4_untile_i8"
        L.check(getattr(L.lib(), name)(self._tiled_i8.data_ptr(), out.data_ptr(), self.out_features, self.in_features, L.stream_ptr()),
                name)
        return out

    def release_reference_layout(self, source=None, half=None) -> None:
        """Free the reference-layout buffer: the decode kernels read only their own tiling, so keeping both doubles
        the weight memory (the reference's selling point for gptq.int4 is "~5 GB", howto/inference.md:37).
        `state_dict()` and the prefill / batch tilings are then rebuilt on demand from the batch-1 tiling -- or from
        `source()` (c_fc1 / c_fc2, whose decode copy is the interleaved fc1|fc2 tiling owned by the model), in which
        case this module keeps no tiling of its own.  `half` = (tiling, h) then says where the prefill GEMM finds the
        layer: rows 8 h .. 8 h + 7 of every 16-row block of the tensor `tiling()` returns.  Loading a state dict
        brings the buffer back."""
        if self._released:
            return
        if not self.scales.is_cuda:
            raise RuntimeError(f"release_reference_layout: the layer is on {self.scales.device}; its tiling is built on CUDA only")
        if not (self.gemv_capable or self.w8_gemv_capable):
            raise RuntimeError("release_reference_layout needs a gptq.int4 / gptq.int8 layer the batch-1 kernel can run "
                               "(per-row scales, no bias, in % 64 == 0)")
        if half is not None and source is None:
            raise ValueError("release_reference_layout: `half` describes a layer held in another tiling; pass its `source` too")
        if source is None:
            self.tiled_i8()
        self._released, self._source, self._half = True, source, half
        self.quant_weight = torch.empty((self.out_features, 0), dtype=torch.uint8, device=self.scales.device)
        self._tiled = self._tiled_mma = None
        if source is not None:
            self._tiled_i8 = None

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        self._tiled = self._tiled_mma = None   # another device / dtype: the tilings are rebuilt on demand
        if self._released and self._source is None and self._tiled_i8 is not None:
            self._tiled_i8 = fn(self._tiled_i8)   # the only copy of a compacted layer travels with the module (uint8: casts leave it alone)
        else:
            self._tiled_i8 = None
        weights_changed()
        return out

    # ------------------------------------------------------------------ device paths
    def _check_layout(self):
        if self._released:
            return
        qw = self.quant_weight
        if tuple(qw.stride()) != (1, self.out_features) and qw.numel() > 0 and self.out_features > 1 and qw.shape[1] > 1:
            raise RuntimeError(
                f"quant_weight strides {tuple(qw.stride())} differ from the reference layout (1, {self.out_features})")
        if not self.scales.is_contiguous() or not self.zeros.is_contiguous():
            raise RuntimeError("scales/zeros must be contiguous")

    def get_weight(self, dtype=torch.float):
        """quantization.py:392-411, on the GPU, bit-exact with the reference arithmetic."""
        L.require_cuda_bf16(torch.empty(0, device=self.scales.device, dtype=torch.bfloat16), "get_weight")
        self._check_layout()
        if dtype not in (torch.bfloat16, torch.float32):
            raise RuntimeError(f"get_weight dtype {dtype} unsupported (bf16 or fp32)")
        out = torch.empty((self.out_features, self.in_features), device=self.scales.device, dtype=dtype)
        qw = self.reference_quant_weight()
        rc = L.lib().b2l_q_dequant(qw.data_ptr(), self.scales.data_ptr(), self.zeros.data_ptr(),
                                   L.sz_dtype_of(self.scales), out.data_ptr(),
                                   L.B2L_BF16 if dtype == torch.bfloat16 else L.B2L_F32, self.out_features,
                                   self.in_features, self.bits, self.tile_cols, L.stream_ptr())
        L.check(rc, "b2l_q_dequant")
        return out

    @property
    def tc_capable(self) -> bool:
        """Eligible for the wgmma kernels: 4 bits, one (scale, zero) per row, K % 32 == 0, no bias."""
        return (self.bits == 4 and self.scales.shape[1] == 1 and self.in_features % 32 == 0 and self.bias is None
                and self.zeros.dtype == self.scales.dtype)

    def tiled(self) -> torch.Tensor:
        """The [N/128][K/32][128][16 B] re-tiling (b2l_q4_tile), rebuilt when quant_weight changes."""
        qw = self.reference_quant_weight()
        key = (qw.data_ptr(), qw._version)
        if self._released or self._tiled is None or self._tiled_key != key:
            self._check_layout()
            nbytes = L.lib().b2l_q4_tiled_bytes(self.out_features, self.in_features)
            t = torch.empty(nbytes, dtype=torch.uint8, device=qw.device)
            L.check(L.lib().b2l_q4_tile(qw.data_ptr(), t.data_ptr(), self.out_features, self.in_features, L.stream_ptr()),
                    "b2l_q4_tile")
            if self._released:
                return t          # transient: a released layer keeps ONE resident copy (callers hold the tensor while it is in use)
            self._tiled, self._tiled_key = t, key
        return self._tiled

    def tiled_i8(self) -> torch.Tensor:
        """The re-tiling of the batch-1 kernel (int8-MMA fragments): [N/16][K/64][32 lanes][16 B] of packed nibbles
        (b2l_q4_tile_i8) at 4 bits, [N/16][K/64][2][32 lanes][16 B] of levels (b2l_w8_tile_i8) at 8 bits."""
        if self._released and self._source is None:
            return self._tiled_i8     # the resident copy
        qw = self.reference_quant_weight()
        key = (qw.data_ptr(), qw._version)
        if self._released or self._tiled_i8 is None or self._tiled_i8_key != key:
            self._check_layout()
            t = tile_i8(qw, self.out_features, self.in_features, self.bits)
            if self._released:        # c_fc1 / c_fc2 after compaction: transient, from the interleaved copy
                return t
            self._tiled_i8, self._tiled_i8_key = t, key
        return self._tiled_i8

    def gemm_weight(self):
        """(weights, flags) for b2l_q4_gemm / b2l_w8_gemm: a released layer's resident batch-1 tiling with
        B2L_F_GEMM_I8 (c_fc1 / c_fc2: half of the interleaved fc1|fc2 tiling), else b2l_q4_tile's tiling (4 bits) or
        quant_weight itself (8 bits), rebuilt by `source()` for a released layer given no `half`.  The GEMM's result
        is the same bit for bit either way."""
        if self._released and self._source is None:
            return self._tiled_i8, L.F_GEMM_I8
        if self._half is not None:
            tiling, h = self._half
            return tiling(), L.F_GEMM_I8 | (L.F_GEMM_I8_HI if h else L.F_GEMM_I8_LO)
        if self.bits == 8:
            self._check_layout()
            return self.reference_quant_weight(), 0
        return self.tiled(), 0

    def tiled_mma(self) -> torch.Tensor:
        """The [N/16][K/64][32 lanes][16 B] re-tiling of the 2..8-row kernel (b2l_q4_tile_mma: f16-MMA fragments)."""
        qw = self.reference_quant_weight()
        key = (qw.data_ptr(), qw._version)
        if self._released or self._tiled_mma is None or self._tiled_mma_key != key:
            self._check_layout()
            nbytes = L.lib().b2l_q4_tiled_mma_bytes(self.out_features, self.in_features)
            t = torch.empty(nbytes, dtype=torch.uint8, device=qw.device)
            L.check(L.lib().b2l_q4_tile_mma(qw.data_ptr(), t.data_ptr(), self.out_features, self.in_features, L.stream_ptr()),
                    "b2l_q4_tile_mma")
            if self._released:
                return t
            self._tiled_mma, self._tiled_mma_key = t, key
        return self._tiled_mma

    @property
    def gemv_capable(self) -> bool:
        return self.tc_capable and self.in_features % 64 == 0 and self.in_features <= 24576

    @property
    def w8_capable(self) -> bool:
        """gptq.int8 on the wgmma GEMM (M >= 2): 8 bits, one (scale, zero) per row, K % 64 == 0, no bias."""
        return (self.bits == 8 and self.scales.shape[1] == 1 and self.in_features % 64 == 0 and self.bias is None
                and self.zeros.dtype == self.scales.dtype)

    @property
    def w8_gemv_capable(self) -> bool:
        """gptq.int8 on the batch-1 kernel (M == 1): w8_capable and K <= 24576."""
        return self.w8_capable and self.in_features <= 24576

    def kernel_at(self, M: int, aligned: bool = True) -> str:
        """The kernel `forward` runs for M activation rows (`aligned`: the rows are 16-byte aligned, their stride a
        multiple of 8 elements, as a contiguous input's are).  The one place this dispatch policy lives: `forward`
        and the packed prefill (LLaMA.refill_rows, which packs a prompt only where this answer is the same at its own
        length and at the pack's) both ask it."""
        if self.w8_gemv_capable and aligned and M == 1:
            return "w8_gemv"
        if self.w8_capable and aligned:
            return "w8_gemm"
        if self.gemv_capable and aligned and M == 1:
            return "q4_gemv"
        if self.gemv_capable and aligned and M <= 8 and BATCH_GEMV:
            return "q4_gemv_batch"
        if self.tc_capable and aligned and M <= 16:
            return "q4_linear_tc"
        if self.tc_capable and aligned and self.in_features % 64 == 0:
            return "q4_gemm"
        return "q_linear"

    def forward(self, inp):
        return self.run(inp)

    def run(self, inp, kernel: Optional[str] = None):
        """forward on `kernel` (a `kernel_at` answer the input qualifies for), or on `kernel_at`'s choice (None)."""
        L.require_cuda_bf16(inp, "ColBlockQuantizedLinear.forward")
        if self.scales.device != inp.device:
            raise RuntimeError("input and quant_weight are on different devices")
        shape = inp.shape
        x = inp.reshape(-1, shape[-1])
        if x.stride(-1) != 1:
            x = x.contiguous()
        M, K, N = x.shape[0], self.in_features, self.out_features
        assert shape[-1] == K, "incompatible dimensions"
        y = torch.empty((M, N), device=inp.device, dtype=inp.dtype)
        if M == 0:
            return y.reshape(*shape[:-1], N)
        aligned = x.data_ptr() % 16 == 0 and x.stride(0) % 8 == 0
        if kernel is None:
            kernel = self.kernel_at(M, aligned)
        # `wt` keeps a transient tiling (released layers) alive until its launch is enqueued; the caching allocator
        # hands freed blocks out in stream order, so the kernel has finished before anybody else writes there
        if kernel in ("w8_gemv", "q4_gemv"):
            wt = self.tiled_i8()
            a = L.Q4LinearArgs(
                x=x.data_ptr(), ldx=x.stride(0), qw_tiled=wt.data_ptr(), scales=self.scales.data_ptr(),
                zeros=self.zeros.data_ptr(), sz_dtype=L.sz_dtype_of(self.scales), y=y.data_ptr(), ldy=N, M=1, N=N, K=K,
                prologue=L.PRO_NONE, norm_scale=None, eps=0.0, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=0)
            L.check(getattr(L.lib(), "b2l_" + kernel)(C.byref(a), L.stream_ptr()), "b2l_" + kernel)
        elif kernel in ("w8_gemm", "q4_gemm"):
            # prefill-shaped, 128 x 128 wgmma tiles, weights dequantised on the fly with get_weight's roundings; a
            # compacted layer's GEMM reads its resident batch-1 tiling
            wt, flags = self.gemm_weight()
            a = L.Q4LinearArgs(
                x=x.data_ptr(), ldx=x.stride(0), qw_tiled=wt.data_ptr(), scales=self.scales.data_ptr(),
                zeros=self.zeros.data_ptr(), sz_dtype=L.sz_dtype_of(self.scales), y=y.data_ptr(), ldy=N,
                M=M, N=N, K=K, prologue=L.PRO_NONE, norm_scale=None, eps=0.0, epilogue=L.EPI_STORE, res=None,
                ldres=0, split_k=0, flags=flags)
            L.check(getattr(L.lib(), "b2l_" + kernel)(C.byref(a), L.stream_ptr()), "b2l_" + kernel)
        elif kernel == "q4_gemv_batch":
            # 2..8 rows: the mma.sync tile has 8 columns, one per row (csrc/q4_gemv_batch.cu)
            wt = self.tiled_mma()
            a = L.Q4LinearArgs(
                x=x.data_ptr(), ldx=x.stride(0), qw_tiled=wt.data_ptr(), scales=self.scales.data_ptr(),
                zeros=self.zeros.data_ptr(), sz_dtype=L.sz_dtype_of(self.scales), y=y.data_ptr(), ldy=N, M=M, N=N, K=K,
                prologue=L.PRO_NONE, norm_scale=None, eps=0.0, epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=0,
                workspace=batch_workspace(inp.device, K).data_ptr())
            L.check(L.lib().b2l_q4_gemv_batch(C.byref(a), L.stream_ptr()), "b2l_q4_gemv_batch")
        elif kernel == "q4_linear_tc":
            wt = self.tiled()
            a = L.Q4LinearArgs(
                x=x.data_ptr(), ldx=x.stride(0), qw_tiled=wt.data_ptr(), scales=self.scales.data_ptr(),
                zeros=self.zeros.data_ptr(), sz_dtype=L.sz_dtype_of(self.scales), y=y.data_ptr(), ldy=N,
                M=M, N=N, K=K, prologue=L.PRO_NONE, norm_scale=None, eps=0.0, epilogue=L.EPI_STORE, res=None,
                ldres=0, split_k=0, flags=0)
            L.check(L.lib().b2l_q4_linear_tc(C.byref(a), L.stream_ptr()), "b2l_q4_linear_tc")
        elif kernel == "q_linear":
            self._check_layout()
            qw = self.reference_quant_weight()
            rc = L.lib().b2l_q_linear(x.data_ptr(), x.stride(0), qw.data_ptr(), self.scales.data_ptr(),
                                      self.zeros.data_ptr(), L.sz_dtype_of(self.scales),
                                      None if self.bias is None else self.bias.to(inp.dtype).data_ptr(), y.data_ptr(), N,
                                      M, N, K, self.bits, self.tile_cols, L.stream_ptr())
            L.check(rc, "b2l_q_linear")
        else:
            raise ValueError(f"ColBlockQuantizedLinear: unknown kernel {kernel!r}")
        return y.reshape(*shape[:-1], N)


#: kernels each of whose output rows depends on its own activation row and the weights only, whatever M is and
#: wherever the row falls in a tile (fixed 128 x 128 tiles, no split-K): prompts packed into one launch of these keep
#: the bits of their own batch-1 prefill
ROW_EXACT_KERNELS = ("q4_gemm", "w8_gemm")


def kernel_at(lin: torch.nn.Module, M: int) -> Optional[str]:
    """The kernel a linear runs for M contiguous activation rows (ColBlockQuantizedLinear.kernel_at), or None for a
    linear without that dispatch (dense, llm.int8: never packed)."""
    return lin.kernel_at(M) if isinstance(lin, ColBlockQuantizedLinear) else None


def packs_at(linears, T: int, N: int) -> bool:
    """Whether a T-token prompt may join a packed prefill of N tokens: its own batch-1 prefill at M = T runs every one
    of `linears` on the same row-exact kernel as the pack at M = N."""
    for lin in linears:
        k = kernel_at(lin, T)
        if k not in ROW_EXACT_KERNELS or kernel_at(lin, N) != k:
            return False
    return True


def tile_i8(qw: torch.Tensor, N: int, K: int, bits: int) -> torch.Tensor:
    """The batch-1 kernel's tiling of quant_weight `qw` (reference layout) for `bits` 4 or 8: a new tensor."""
    if not qw.is_cuda:
        raise RuntimeError(f"tile_i8: quant_weight is on {qw.device}; the tiling kernels run on CUDA only")
    kind = "w8" if bits == 8 else "q4"
    t = torch.empty(getattr(L.lib(), f"b2l_{kind}_tiled_i8_bytes")(N, K), dtype=torch.uint8, device=qw.device)
    L.check(getattr(L.lib(), f"b2l_{kind}_tile_i8")(qw.data_ptr(), t.data_ptr(), N, K, L.stream_ptr()), f"b2l_{kind}_tile_i8")
    return t


def qlinear_4bit_weight(inp, weight, scales, zeros):
    """Same call as the reference's Triton launcher (quantization.py:284-333):
    `weight` is quant_weight (N, K/2) in the reference layout, scales/zeros (N, 1)."""
    L.require_cuda_bf16(inp, "qlinear_4bit_weight")
    N, K = weight.shape[0], weight.shape[1] * 2
    assert inp.shape[-1] == K, "incompatible dimensions"
    assert scales.shape == (N, 1) and zeros.shape == (N, 1)
    x = inp.reshape(-1, K).contiguous()
    y = torch.empty((x.shape[0], N), device=inp.device, dtype=inp.dtype)
    if tuple(weight.stride()) != (1, N):
        weight = weight.t().contiguous().t()
    scales, zeros = scales.contiguous(), zeros.contiguous()
    rc = L.lib().b2l_q_linear(x.data_ptr(), K, weight.data_ptr(), scales.data_ptr(), zeros.data_ptr(), L.sz_dtype_of(scales),
                              None, y.data_ptr(), N, x.shape[0], N, K, 4, K, L.stream_ptr())
    L.check(rc, "b2l_q_linear")
    return y.reshape(*inp.shape[:-1], N)

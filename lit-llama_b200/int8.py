"""Drop-in `Linear8bitLt` (reference: lit_llama/quantization.py:38-77, a subclass of
bitsandbytes' `bnb.nn.Linear8bitLt` with has_fp16_weights=False, threshold=6.0).

Same construction-time behaviour: the weight is quantised row-wise to int8 as soon as the
module exists and again whenever a float `*.weight` arrives through `load_state_dict`
(quantization.py:52-77); `weight.CB` (int8, (out, in)) and `weight.SCB` (fp32 row absmax)
are attributes of the parameter like in bitsandbytes.  The forward is the LLM.int8()
algorithm on the tensor cores (csrc/q8_gemv.cu for one row, csrc/q8_gemm.cu for more) - no bitsandbytes,
no CPU path.

bitsandbytes is not part of the reference tree (unpinned dependency, pyproject.toml:19), so the
arithmetic follows the published algorithm (parity with the reference is unpinned, see DESIGN.md).
"""
import torch

from . import _lib as L
from .quantization import weights_changed


def quantize_rows_int8(weight: torch.Tensor):
    """quantization.py:69-77 (`bnb.functional.double_quant` on W.half(), row statistics only):
    CB = round(W * 127 / rowabsmax) int8, SCB = rowabsmax fp32."""
    wh = weight.contiguous().half().float()
    scb = wh.abs().amax(dim=1)
    cb = torch.round(wh * (127.0 / scb.clamp_min(1e-30)).unsqueeze(1)).clamp_(-127, 127).to(torch.int8)
    return cb.contiguous(), scb.contiguous()


class Linear8bitLt(torch.nn.Module):
    def __init__(self, input_features, output_features, bias=True, **kwargs):
        super().__init__()
        self.in_features = input_features
        self.out_features = output_features
        self.threshold = 6.0
        w = torch.empty((output_features, input_features))
        torch.nn.init.kaiming_uniform_(w, a=5 ** 0.5)  # nn.Linear's default, what bnb inherits
        self.weight = torch.nn.Parameter(torch.empty((output_features, input_features), dtype=torch.int8), requires_grad=False)
        if bias:
            self.bias = torch.nn.Parameter(torch.zeros(output_features), requires_grad=False)
        else:
            self.register_parameter("bias", None)
        self._tiled = None
        self._tiled_key = None
        self._quantize_weight(w.to(self.weight.device))

    def _quantize_weight(self, weight: torch.Tensor) -> None:
        """quantization.py:69-77."""
        cb, scb = quantize_rows_int8(weight.to(self.weight.device))
        self.weight.data = cb
        setattr(self.weight, "CB", cb)
        setattr(self.weight, "SCB", scb)
        self._tiled = None
        weights_changed()

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        # keep the statistics next to the (possibly moved) int8 weight; dtype casts leave int8 alone
        scb = getattr(self.weight, "SCB", None)
        if scb is not None:
            self.weight.SCB = scb.to(self.weight.device)
            self.weight.CB = self.weight.data
        self._tiled = None
        weights_changed()
        return out

    def _load_from_state_dict(self, local_state_dict, prefix, *args, **kwargs):
        """quantization.py:52-67: a float `*.weight` is re-quantised; int8 weights (a state dict saved
        from this module) are taken as they are when `*.SCB` travels with them."""
        wkey = prefix + "weight"
        if wkey in local_state_dict:
            w = local_state_dict.pop(wkey)
            if w.dtype == torch.int8:
                scb = local_state_dict.pop(prefix + "SCB", None)
                if scb is None:
                    raise RuntimeError(f"{wkey} is int8 but {prefix}SCB is missing")
                self.weight.data = w.to(self.weight.device).contiguous()
                self.weight.CB = self.weight.data
                self.weight.SCB = scb.to(self.weight.device).float().contiguous()
                self._tiled = None
                weights_changed()
            else:
                self._quantize_weight(w)
        local_state_dict.pop(prefix + "SCB", None)
        if any(k.startswith(prefix) for k in local_state_dict):
            super()._load_from_state_dict(local_state_dict, prefix, *args, **kwargs)

    def tiled(self) -> torch.Tensor:
        """CB re-tiled for `b2l_q8_gemv` (b2l_q8_tile), built on demand and cached.  forward does not use it: both of
        its kernels read CB directly, so a model that only runs forward holds one copy of its int8 weights."""
        cb = self.weight.data
        key = (cb.data_ptr(), cb._version)
        if self._tiled is None or self._tiled_key != key:
            lib = L.lib()
            t = torch.empty(lib.b2l_q8_tiled_bytes(self.out_features, self.in_features), dtype=torch.uint8, device=cb.device)
            L.check(lib.b2l_q8_tile(cb.data_ptr(), t.data_ptr(), self.out_features, self.in_features, L.stream_ptr()), "b2l_q8_tile")
            self._tiled, self._tiled_key = t, key
        return self._tiled

    MAX_IN_FEATURES = 32768  # the kernels' limit (csrc/q8_gemv.cu, csrc/q8_gemm.cu); LLaMA-65B's n_hidden is 22016

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        L.require_cuda_bf16(x, "Linear8bitLt.forward")
        if self.in_features % 128 != 0 or self.in_features > self.MAX_IN_FEATURES:
            raise RuntimeError(f"Linear8bitLt: in_features {self.in_features} unsupported (multiple of 128, <= {self.MAX_IN_FEATURES})")
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        M, K, N = x2.shape[0], self.in_features, self.out_features
        y = torch.empty((M, N), device=x.device, dtype=x.dtype)
        lib = L.lib()
        cb, scb = self.weight.data, self.weight.SCB
        if M == 1:
            rc = lib.b2l_q8_gemv_cb(x2.data_ptr(), cb.data_ptr(), scb.data_ptr(), None, y.data_ptr(), N, K, self.threshold, 0,
                                    L.stream_ptr())
            L.check(rc, "b2l_q8_gemv_cb")
        else:  # outlier columns are a property of the whole batch (any row over the threshold)
            nbytes = lib.b2l_q8_gemm_workspace_bytes(M, K)
            work = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            rc = lib.b2l_q8_gemm(x2.data_ptr(), K, cb.data_ptr(), scb.data_ptr(), work.data_ptr(), nbytes, y.data_ptr(), N,
                                 M, N, K, self.threshold, 0, L.stream_ptr())
            L.check(rc, "b2l_q8_gemm")
        if self.bias is not None:
            y = y + self.bias.to(y.dtype)
        return y.reshape(*shape[:-1], N)

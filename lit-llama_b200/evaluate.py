"""evaluate/{full,lora,adapter,adapter_v2}.py of the reference (perplexity over 2048-token windows) on the H100 path.

The reference scripts run `logits = model(inp)[0]` per window and then torch's
`cross_entropy(logits[:-1], inp[0, 1:], reduction="sum")`: a (T, vocab) logits tensor is written and read again, and on
bf16 logits the window's loss comes back as a bf16 scalar (about 3 significant digits of a sum in the thousands).
Here the loss is computed by the project's kernels, with fp32 per-token NLL and an fp64 window sum:

  * `window_nll(model, inp)` runs the embedding, the Blocks and ln_f like `model(inp)` with no cache, then lm_head:
      - a plain gptq.int4 lm_head (per-row scales, no bias) for windows of more than 16 tokens, or a plain gptq.int8
        one for 2 or more: the loss inside the lm_head GEMM's epilogue (`b2l_q4_gemm_nll` / `b2l_w8_gemm_nll`), so the
        logits are never written;
      - every other lm_head (dense, llm.int8, short gptq.int4 windows, LLaMA-Adapter v2's affine): `lm_head(x)`, then
        `b2l_logits_nll` on those logits.
    Both give bit-identical results on the same logits, and equal `model(inp)` followed by `b2l_logits_nll`.
  * `perplexity(model, encoded)` follows the reference loop: trim to 256 * block_size tokens, windows of 2048 with a
    ragged last one, T - 1 predicted tokens per window, the windows summed on the device and read once.
  * `main()` / `cli()` mirror the four scripts' arguments, selected with `--kind`.
"""
import ctypes as C
import math
import sys
import time
from pathlib import Path
from typing import Callable, Optional, Tuple

import torch

from . import _lib as L
from .quantization import ColBlockQuantizedLinear

NLLFn = Callable[[torch.nn.Module, torch.Tensor], Tuple[torch.Tensor, torch.Tensor]]


def _nll_args(targets: torch.Tensor, M: int, N: int) -> Tuple[L.NLLArgs, tuple]:
    """The argument block for M rows of N columns and the tensors it points at: (nll fp32 [M], nll_sum fp64 scalar,
    workspace)."""
    dev = targets.device
    nll = torch.empty(M, dtype=torch.float32, device=dev)
    s = torch.empty((), dtype=torch.float64, device=dev)
    ws = torch.empty(max(L.lib().b2l_nll_workspace_bytes(M, N), 16), dtype=torch.uint8, device=dev)
    a = L.NLLArgs(targets=targets.data_ptr(), targets_i64=1 if targets.dtype == torch.int64 else 0,
                  nll=nll.data_ptr(), nll_sum=s.data_ptr(), workspace=ws.data_ptr())
    return a, (nll, s, ws)


def _targets(t: torch.Tensor) -> torch.Tensor:
    if t.dtype not in (torch.int32, torch.int64):
        t = t.to(torch.int64)
    return t.contiguous()


def logits_nll(logits: torch.Tensor, targets: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(nll fp32 [M], nll_sum fp64 scalar) of rows 0..M-1 of bf16 `logits` [>= M, N] (unit column stride) against
    `targets` [M] (b2l_logits_nll).  A target outside 0..N-1 gives NaN for its row."""
    L.require_cuda_bf16(logits, "logits_nll")
    if logits.stride(-1) != 1:
        logits = logits.contiguous()
    N = logits.shape[-1]
    l2 = logits.reshape(-1, N)
    t = _targets(targets)
    M = t.numel()
    if M > l2.shape[0]:
        raise ValueError(f"logits_nll: {M} targets for {l2.shape[0]} rows of logits")
    a, (nll, s, _ws) = _nll_args(t, M, N)
    L.check(L.lib().b2l_logits_nll(l2.data_ptr(), l2.stride(0), M, N, C.byref(a), L.stream_ptr()), "b2l_logits_nll")
    return nll, s


def _fused_kind(lm: torch.nn.Module, T: int, x: torch.Tensor) -> Optional[str]:
    """"q4" / "w8" when lm_head over the T rows of x runs on the wgmma GEMM (ColBlockQuantizedLinear.forward's
    dispatch), so the loss can go in its epilogue; None otherwise."""
    if type(lm) is not ColBlockQuantizedLinear or hasattr(lm, "adapter_scale"):
        return None
    if not (x.data_ptr() % 16 == 0 and x.stride(0) % 8 == 0):
        return None
    if lm.w8_capable and T >= 2:
        return "w8"
    if lm.tc_capable and lm.in_features % 64 == 0 and T > 16:
        return "q4"
    return None


@torch.no_grad()
def lm_head_nll(lm: torch.nn.Module, x: torch.Tensor, targets: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(nll fp32 [T-1], nll_sum fp64 scalar) of `lm` over the T rows of x ([..., T, K], the rows of one window)
    against `targets` [T-1]: the loss in the lm_head GEMM's epilogue when `lm` runs on the wgmma GEMM, else `lm(x)`
    then b2l_logits_nll.  Bit-identical either way."""
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    T = x2.shape[0]
    targets = _targets(targets)
    kind = _fused_kind(lm, T, x2)
    if kind is None:
        return logits_nll(lm(x), targets)
    N, M = lm.out_features, targets.numel()
    a, (nll, s, _ws) = _nll_args(targets, M, N)
    if kind == "q4":
        wt = lm.tiled()   # transient on a compacted layer: held until the launch is enqueued
        fn = "b2l_q4_gemm_nll"
    else:
        lm._check_layout()
        wt = lm.reference_quant_weight()
        fn = "b2l_w8_gemm_nll"
    g = L.Q4LinearArgs(
        x=x2.data_ptr(), ldx=x2.stride(0), qw_tiled=wt.data_ptr(), scales=lm.scales.data_ptr(), zeros=lm.zeros.data_ptr(),
        sz_dtype=L.sz_dtype_of(lm.scales), y=None, ldy=0, M=M, N=N, K=K, prologue=L.PRO_NONE, norm_scale=None, eps=0.0,
        epilogue=L.EPI_STORE, res=None, ldres=0, split_k=0, flags=0)
    L.check(getattr(L.lib(), fn)(C.byref(g), C.byref(a), L.stream_ptr()), fn)
    return nll, s


@torch.no_grad()
def window_nll(model: torch.nn.Module, inp: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """One window (B = 1): (nll fp32 [T-1], nll_sum fp64 scalar tensor) of predicting inp[0, m+1] from inp[0, :m+1],
    on the device.  Equal, bit for bit, to `b2l_logits_nll` on the logits `model(inp)` returns."""
    if inp.dim() != 2 or inp.size(0) != 1:
        raise ValueError(f"window_nll: inp must be (1, T), got {tuple(inp.shape)}")
    inp = inp.contiguous()
    max_seq_length = model._prepare(inp, None)
    x = model._forward_hidden(inp, max_seq_length, None)
    return lm_head_nll(model.lm_head, x, inp[0, 1:])


def perplexity(model: torch.nn.Module, encoded: torch.Tensor, block_size: int = 2048,
               nll_fn: NLLFn = window_nll) -> Tuple[float, float, int]:
    """evaluate/full.py:113-130: (perplexity, summed NLL, predicted tokens) of the token sequence `encoded` ((n,) or
    (1, n)), trimmed to 256 * model.config.block_size tokens and cut into windows of `block_size` (the last one may
    be shorter, down to one token).  Each window predicts its own T - 1 next tokens; nothing is predicted across a
    window boundary.  The window sums stay on the device; the result is read once."""
    enc = encoded.reshape(-1)[: 256 * model.config.block_size]
    total, n_tokens = None, 0
    for i in range(0, enc.numel(), block_size):
        inp = enc[i : i + block_size].view(1, -1)
        _, s = nll_fn(model, inp)
        total = s.clone() if total is None else total.add_(s)
        n_tokens += inp.size(1) - 1
    if n_tokens == 0:
        raise ValueError("perplexity needs at least two tokens")
    nll_sum = float(total.item())
    return math.exp(nll_sum / n_tokens), nll_sum, n_tokens


def load_eval_data(dataset_name: str) -> str:
    """evaluate/full.py:26-46: the test split of wikitext-2, ptb or the first c4 validation shard (needs `datasets`
    and its cache or network)."""
    from datasets import load_dataset

    if dataset_name == "wikitext":
        testdata = load_dataset("wikitext", "wikitext-2-raw-v1", split="test")
        return "\n\n".join(testdata["text"])
    if dataset_name == "ptb":
        testdata = load_dataset("ptb_text_only", "penn_treebank", split="test")
        return "\n\n".join(testdata["sentence"])
    if dataset_name == "c4":
        testdata = load_dataset("allenai/c4", "allenai--c4",
                                data_files={"validation": "en/c4-validation.00000-of-00008.json.gz"}, split="validation")
        return " ".join(testdata[:1100]["text"])
    raise ValueError("invalid dataset name (wikitext, ptb, c4 are allowed)")


def load_model(kind: str, checkpoint_path: Path, quantize: Optional[str], lora_path: Optional[Path] = None,
               adapter_path: Optional[Path] = None, device: torch.device = torch.device("cuda", 0)) -> torch.nn.Module:
    """The model of one of the four scripts, in bf16 on `device`: full (evaluate/full.py), LoRA r=8 alpha=16 on
    c_attn (evaluate/lora.py), LLaMA-Adapter (evaluate/adapter.py) or LLaMA-Adapter v2 (evaluate/adapter_v2.py).
    The base checkpoint is loaded first, then the fine-tuned weights, both with strict=False like the reference."""
    from contextlib import ExitStack

    from .utils import llama_model_lookup, quantization

    checkpoint = torch.load(checkpoint_path, map_location="cpu", weights_only=True, mmap=True)
    name = llama_model_lookup(checkpoint)
    extra = None
    if kind == "full":
        from .model import LLaMA
    elif kind == "lora":
        from .lora import lora
        from .model import LLaMA

        extra = lora_path
    elif kind in ("adapter", "adapter_v2"):
        from .adapter import LLaMA

        extra = adapter_path
    else:
        raise ValueError(f"unknown kind {kind!r} (full, lora, adapter, adapter_v2)")
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)   # what Fabric's bf16-true does inside init_module
    try:
        with ExitStack() as stack:
            stack.enter_context(torch.device(device))
            stack.enter_context(quantization(mode=quantize))
            if kind == "lora":
                stack.enter_context(lora(r=8, alpha=16, dropout=0.05, enabled=True))   # evaluate/lora.py:26-30
            model = LLaMA.from_name(name)
            if kind == "adapter_v2":
                from .adapter_v2 import add_adapter_v2_parameters_to_linear_layers

                add_adapter_v2_parameters_to_linear_layers(model)
    finally:
        torch.set_default_dtype(prev)
    model.load_state_dict(checkpoint, strict=extra is None)
    if extra is not None:
        model.load_state_dict(torch.load(extra, map_location="cpu", weights_only=True, mmap=True), strict=False)
    return model.eval()


def main(
    datasets: str = "wikitext,ptb,c4",
    *,
    kind: str = "full",
    checkpoint_path: Path = Path("checkpoints/lit-llama/7B/lit-llama.pth"),
    tokenizer_path: Path = Path("checkpoints/lit-llama/tokenizer.model"),
    quantize: Optional[str] = None,
    lora_path: Path = Path("out/lora/alpaca/lit-llama-lora-finetuned.pth"),
    adapter_path: Optional[Path] = None,
    text_path: Optional[Path] = None,
    instruction_tuning: Optional[bool] = None,
) -> None:
    """evaluate/{full,lora,adapter,adapter_v2}.py without Fabric: bf16 on cuda:0 (the reference's default dtype is
    float32, which this path does not run), the same printed lines.  `text_path` evaluates a local UTF-8 text file
    instead of `datasets` (no download).  Like the reference, the lora / adapter / adapter_v2 kinds first wrap the
    text as an Alpaca instruction, with `generate_prompt` of the lit-llama checkout's scripts/prepare_alpaca.py
    (which must be importable; `instruction_tuning=False` skips the wrapping)."""
    from sentencepiece import SentencePieceProcessor

    checkpoint_path, tokenizer_path = Path(checkpoint_path), Path(tokenizer_path)
    assert checkpoint_path.is_file(), checkpoint_path
    assert tokenizer_path.is_file(), tokenizer_path
    if adapter_path is None:
        adapter_path = Path(f"out/{kind}/alpaca/lit-llama-adapter-finetuned.pth")
    if instruction_tuning is None:
        instruction_tuning = kind != "full"
    device = torch.device("cuda", 0)

    print("Loading model ...", file=sys.stderr)
    t0 = time.time()
    model = load_model(kind, checkpoint_path, quantize, Path(lora_path), Path(adapter_path), device)
    print(f"Time to load model: {time.time() - t0:.02f} seconds.", file=sys.stderr)
    sp = SentencePieceProcessor(model_file=str(tokenizer_path))

    total_toks = 0
    t0 = time.perf_counter()
    sources = [(Path(text_path).name, None)] if text_path is not None else [(ds, ds) for ds in datasets.split(",")]
    for dsname, ds in sources:
        test_string = Path(text_path).read_text(encoding="utf-8") if ds is None else load_eval_data(ds)
        if instruction_tuning:
            from scripts.prepare_alpaca import generate_prompt

            test_string = generate_prompt({"instruction": test_string, "input": ""})
        encoded = torch.tensor([sp.bos_id()] + sp.encode(test_string), dtype=torch.int64, device=device)
        ppl, _, toks = perplexity(model, encoded)
        print(f"Perplexity on {dsname}: {ppl:.2f}")
        total_toks += toks

    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    print(f"\n\nTime for inference: {t:.02f} sec total, {total_toks / t:.02f} tokens/sec", file=sys.stderr)
    print(f"Memory used: {torch.cuda.max_memory_reserved() / 1e9:.02f} GB", file=sys.stderr)


def cli(argv=None) -> None:
    import argparse

    ap = argparse.ArgumentParser(description=main.__doc__)
    ap.add_argument("--datasets", default="wikitext,ptb,c4")
    ap.add_argument("--kind", default="full", choices=["full", "lora", "adapter", "adapter_v2"])
    ap.add_argument("--checkpoint_path", type=Path, default=Path("checkpoints/lit-llama/7B/lit-llama.pth"))
    ap.add_argument("--tokenizer_path", type=Path, default=Path("checkpoints/lit-llama/tokenizer.model"))
    ap.add_argument("--quantize", default=None, choices=[None, "llm.int8", "gptq.int4", "gptq.int8"])
    ap.add_argument("--lora_path", type=Path, default=Path("out/lora/alpaca/lit-llama-lora-finetuned.pth"))
    ap.add_argument("--adapter_path", type=Path, default=None)
    ap.add_argument("--text_path", type=Path, default=None)
    ap.add_argument("--no_instruction_tuning", action="store_true",
                    help="lora / adapter / adapter_v2: evaluate the raw text, not the Alpaca-wrapped one")
    a = vars(ap.parse_args(argv))
    a["instruction_tuning"] = False if a.pop("no_instruction_tuning") else None
    main(**a)


if __name__ == "__main__":
    cli()

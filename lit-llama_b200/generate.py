"""generate.py of the reference (generate.py:20-91, 94-155) over the H100 modules.

`generate()` keeps the reference's Python token loop and torch sampling ops (so the
RNG stream of `torch.multinomial` is the reference's); the model call inside it is one
CUDA-graph replay per token.  `main()` mirrors the reference CLI with argparse
(jsonargparse and lightning are not dependencies of this path)."""
import os
import sys
import time
from pathlib import Path
from typing import Optional

import torch

from . import _lib as L
from .model import LLaMA
from .utils import llama_model_lookup, quantization


_TORCH_MULTINOMIAL = torch.multinomial


def sample_probs(logits_row: torch.Tensor, temperature: float = 1.0, top_k: Optional[int] = None) -> torch.Tensor:
    """generate.py:68-75: probabilities of the next token from the last position's logits
    (V,) bf16: temperature, top-k filter and softmax fused in one kernel (b2l_topk_softmax)."""
    L.require_cuda_bf16(logits_row, "sample_probs")
    x = logits_row.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()  # the kernel reads 16-byte vectors
    V = x.numel()
    probs = torch.empty_like(x)
    k = 0 if top_k is None else min(int(top_k), V)
    L.check(L.lib().b2l_topk_softmax(x.data_ptr(), float(temperature), k, probs.data_ptr(), V, L.stream_ptr()), "b2l_topk_softmax")
    return probs


def sample_token(logits_row: torch.Tensor, temperature: float = 1.0, top_k: Optional[int] = None) -> torch.Tensor:
    """generate.py:68-76: the next token (shape (1,), int64) drawn from the last position's logits.
    `torch.multinomial(probs, num_samples=1)` is `argmax(probs / q)` with `q = empty_like(probs).exponential_(1)`
    (ATen/native/Distributions.cpp); q is drawn here with torch -- the RNG consumption of multinomial, so for the same
    generator state the token equals `torch.multinomial(sample_probs(...), 1)` -- and everything else is one
    launch (b2l_topk_softmax_sample) instead of multinomial's dozen."""
    L.require_cuda_bf16(logits_row, "sample_token")
    x = logits_row.contiguous()
    if x.data_ptr() % 16:
        x = x.clone()  # the kernel reads 16-byte vectors
    V = x.numel()
    q = torch.empty_like(x).exponential_(1)
    token = torch.empty(1, dtype=torch.int64, device=x.device)
    k = 0 if top_k is None else min(int(top_k), V)
    L.check(L.lib().b2l_topk_softmax_sample(x.data_ptr(), float(temperature), k, q.data_ptr(), None, token.data_ptr(), V, L.stream_ptr()),
            "b2l_topk_softmax_sample")
    return token


@torch.no_grad()
def generate(
    model: LLaMA,
    idx: torch.Tensor,
    max_new_tokens: int,
    *,
    max_seq_length: Optional[int] = None,
    temperature: float = 1.0,
    top_k: Optional[int] = None,
    eos_id: Optional[int] = None,
) -> torch.Tensor:
    """generate.py:20-91: `idx` (T,) prompt -> (T + max_new_tokens,) tokens."""
    T = idx.size(0)
    T_new = T + max_new_tokens
    if max_seq_length is None:
        max_seq_length = min(T_new, model.config.block_size)

    device, dtype = idx.device, idx.dtype
    empty = torch.empty(T_new, dtype=dtype, device=device)
    empty[:T] = idx
    idx = empty
    input_pos = torch.arange(0, T, device=device)

    for _ in range(max_new_tokens):
        x = idx.index_select(0, input_pos).view(1, -1)
        logits = model(x, max_seq_length, input_pos)
        if torch.multinomial is _TORCH_MULTINOMIAL:
            idx_next = sample_token(logits[0, -1], temperature, top_k).to(dtype=dtype)  # generate.py:68-76: RNG draw + one launch
        else:
            # torch.multinomial has been replaced (the reference's tests/test_generate.py:26-54 patches it to record
            # the draws): keep calling it, on the fused probabilities
            idx_next = torch.multinomial(sample_probs(logits[0, -1], temperature, top_k), num_samples=1).to(dtype=dtype)
        input_pos = input_pos[-1:] + 1
        idx = idx.index_copy(0, input_pos, idx_next)
        if eos_id is not None and idx_next == eos_id:
            return idx[:input_pos]  # include the EOS token
    return idx


def main(
    prompt: str = "Hello, my name is",
    *,
    num_samples: int = 1,
    max_new_tokens: int = 50,
    top_k: int = 200,
    temperature: float = 0.8,
    checkpoint_path: Path = Path("checkpoints/lit-llama/7B/lit-llama.pth"),
    tokenizer_path: Path = Path("checkpoints/lit-llama/tokenizer.model"),
    quantize: Optional[str] = None,
) -> None:
    """generate.py:94-155 without Fabric: bf16 on cuda:0, same prints on stderr."""
    from sentencepiece import SentencePieceProcessor

    checkpoint_path, tokenizer_path = Path(checkpoint_path), Path(tokenizer_path)
    assert checkpoint_path.is_file(), checkpoint_path
    assert tokenizer_path.is_file(), tokenizer_path
    device = torch.device("cuda", 0)

    print("Loading model ...", file=sys.stderr)
    t0 = time.time()
    checkpoint = torch.load(checkpoint_path, map_location="cpu", weights_only=True, mmap=True)
    name = llama_model_lookup(checkpoint)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)  # what Fabric's bf16-true does inside init_module
    try:
        with torch.device(device), quantization(mode=quantize):
            model = LLaMA.from_name(name)
    finally:
        torch.set_default_dtype(prev)
    model.load_state_dict(checkpoint)
    print(f"Time to load model: {time.time() - t0:.02f} seconds.", file=sys.stderr)
    model.eval()
    if quantize in ("gptq.int4", "gptq.int8") and os.environ.get("B2L_COMPACT", "1") != "0":
        try:
            model.compact()   # one resident copy of the weights (the reference-layout buffers come back on state_dict())
        except RuntimeError:  # a layer the fused decode step cannot run (grouped scales, odd widths): keep everything
            pass

    sp = SentencePieceProcessor(model_file=str(tokenizer_path))
    encoded = torch.tensor([sp.bos_id()] + sp.encode(prompt), dtype=torch.int, device=device)
    prompt_length = encoded.size(0)

    torch.manual_seed(1234)
    for i in range(num_samples):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        y = generate(model, encoded, max_new_tokens, temperature=temperature, top_k=top_k)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        model.reset_cache()
        print(sp.decode(y.tolist()))
        tokens_generated = y.size(0) - prompt_length
        print(f"Time for inference {i + 1}: {t:.02f} sec total, {tokens_generated / t:.02f} tokens/sec", file=sys.stderr)
    print(f"Memory used: {torch.cuda.max_memory_reserved() / 1e9:.02f} GB", file=sys.stderr)


def cli() -> None:
    import argparse

    ap = argparse.ArgumentParser(description=main.__doc__)
    ap.add_argument("--prompt", default="Hello, my name is")
    ap.add_argument("--num_samples", type=int, default=1)
    ap.add_argument("--max_new_tokens", type=int, default=50)
    ap.add_argument("--top_k", type=int, default=200)
    ap.add_argument("--temperature", type=float, default=0.8)
    ap.add_argument("--checkpoint_path", type=Path, default=Path("checkpoints/lit-llama/7B/lit-llama.pth"))
    ap.add_argument("--tokenizer_path", type=Path, default=Path("checkpoints/lit-llama/tokenizer.model"))
    ap.add_argument("--quantize", default=None, choices=[None, "llm.int8", "gptq.int4", "gptq.int8"])
    a = ap.parse_args()
    main(**vars(a))


if __name__ == "__main__":
    cli()

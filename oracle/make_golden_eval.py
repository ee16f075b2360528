"""Generates tests/golden/tiny_eval_int4.pt by running the UNMODIFIED reference's evaluation loop on the CPU.

    python oracle/make_golden_eval.py        (the lit-llama checkout is found as oracle/make_golden.py finds it)

The model is the tiny gptq.int4 model of make_golden.golden_model (block_size 64, vocab 96 padded to 128, the same
synthetic weights).  Two token sequences are cut into 64-token windows exactly like evaluate/full.py:120-129 does
(`range(0, n, block_size)`): one of 229 tokens (a ragged last window of 37) and one of 129 (a last window of 1
token).  Per window the loop's own expression is recorded,
    cross_entropy(logits[:-1], inp[0, 1:].long(), reduction="sum"),
on an fp32 model and on a bf16 model (where it returns a bf16 scalar), plus reduction="none" of the fp32 model and of
the bf16 model's logits upcast to fp32.  TEST INFRASTRUCTURE.
"""
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import llama_oracle as O  # noqa: E402
from oracle.make_golden import build_ref_model  # noqa: E402  (puts the reference and oracle/_shim on sys.path)

OUT = os.path.join(ROOT, "tests", "golden")
CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)
BLOCK = 64
LENGTHS = (229, 129)


@torch.no_grad()
def evaluate_like_reference(model, encoded: torch.Tensor) -> dict:
    """evaluate/full.py:113-130 on the CPU, keeping every window's loss."""
    encoded = encoded[None, : 256 * model.config.block_size]
    sums, nones, nlls, toks = [], [], 0, 0
    for i in range(0, encoded.shape[1], BLOCK):
        inp = encoded[:, i : i + BLOCK]
        logits = model(inp)[0]
        nll = F.cross_entropy(logits[:-1], inp[0, 1:].to(dtype=torch.long), reduction="sum")
        nones.append(F.cross_entropy(logits[:-1].float(), inp[0, 1:].to(dtype=torch.long), reduction="none"))
        sums.append(nll.clone())
        toks += inp.size(1) - 1
        nlls += nll.item()
    return dict(window_sums=sums, window_nll_f32=nones, nlls=nlls, toks=toks, ppl=math.exp(nlls / toks))


def main():
    g = torch.Generator().manual_seed(2024)
    seqs = [torch.randint(0, CFG["vocab_size"], (n,), generator=g) for n in LENGTHS]
    out = dict(cfg=CFG, seed=1234, block=BLOCK, seqs=seqs)
    for dtype, tag in ((torch.float32, "f32"), (torch.bfloat16, "bf16")):
        sd = O.synth_state_dict(CFG["n_layer"], CFG["n_head"], CFG["n_embd"], CFG["vocab_size"], "gptq.int4", dtype=dtype,
                                seed=1234)
        m = build_ref_model(CFG, sd, "gptq.int4", dtype)
        out[tag] = [evaluate_like_reference(m, s) for s in seqs]
    torch.save(out, os.path.join(OUT, "tiny_eval_int4.pt"))
    for tag in ("f32", "bf16"):
        for n, r in zip(LENGTHS, out[tag]):
            print(tag, n, [float(s) for s in r["window_sums"]], r["toks"], r["ppl"])


if __name__ == "__main__":
    main()

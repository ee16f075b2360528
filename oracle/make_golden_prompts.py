"""Generates tests/golden/tiny_prompts_int4_bf16.pt by running the UNMODIFIED reference on the CPU:

    python oracle/make_golden_prompts.py

Writes only that file (the fixtures of oracle/make_golden.py are not regenerated): the reference's greedy
`generate()` (top_k=1, 12 new tokens) on the tiny gptq.int4 bf16 model of tiny_int4_bf16.pt, for 4 prompts of
different lengths (3, 16, 40, 7), one prompt at a time.  tests/test_gpu_generate_prompts.py holds each row of
`generate_prompts` to these tokens.  Needs the lit-llama checkout (default /root/reference; LIT_LLAMA_DIR overrides
it) and oracle/_shim.  TEST INFRASTRUCTURE.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import llama_oracle as O  # noqa: E402
from oracle.make_golden import OUT, build_ref_model, ref_generate  # noqa: E402  (puts the reference on sys.path)

LENGTHS = (3, 16, 40, 7)
NEW = 12


@torch.no_grad()
def main():
    cfg = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)
    sd = O.synth_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"], "gptq.int4",
                            dtype=torch.bfloat16, seed=1234)
    m = build_ref_model(cfg, sd, "gptq.int4", torch.bfloat16)
    g = torch.Generator().manual_seed(17)
    prompts = [torch.randint(0, cfg["vocab_size"], (n,), generator=g) for n in LENGTHS]
    gen = []
    for i, p in enumerate(prompts):
        if i:
            m.reset_cache()
        m.kv_caches.clear()
        gen.append(ref_generate.generate(m, p.to(torch.int32), NEW, top_k=1).clone())
    out = dict(cfg=cfg, seed=1234, prompts=prompts, max_new_tokens=NEW, gen_greedy=gen)
    path = os.path.join(OUT, "tiny_prompts_int4_bf16.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()

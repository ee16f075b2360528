"""Generates the LLaMA-Adapter fixtures under tests/golden/ by running the UNMODIFIED reference on the CPU:

    python oracle/make_golden_adapter.py

Writes only new files (the fixtures of oracle/make_golden.py are not regenerated):
  * tiny_adapter_int4_bf16.pt: lit_llama.adapter.LLaMA under quantization("gptq.int4"), bf16, n_layer 3,
    adapter_start_layer 1, random non-zero gates: prefill + 3 decode steps, the no-cache forward, the roll branch and
    greedy / sampled generate() tokens;
  * reference_adapter_surface.json: the names lit_llama.adapter and generate/adapter.py bind.
Needs the lit-llama checkout (default /root/reference; LIT_LLAMA_DIR overrides it) and oracle/_shim.  TEST INFRASTRUCTURE.

This is a separate generator, and the adapter restatement a separate module (oracle/adapter_oracle.py, built on
oracle/llama_oracle.py), rather than an `adapter` target of oracle/make_golden.py and more code in llama_oracle.py:
the existing generator and oracle, and every fixture they pin, stay byte for byte as they were, and running this
script cannot regenerate any of them.
"""
import importlib.util
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("LIT_LLAMA_DIR", "/root/reference")
sys.path.insert(0, os.path.join(HERE, "_shim"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

import generate as ref_generate  # noqa: E402  (reference generate.py)
import lit_llama.adapter as ref_adapter  # noqa: E402
from lit_llama.utils import quantization  # noqa: E402

from oracle import adapter_oracle as A  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CFG = dict(block_size=64, vocab_size=96, n_layer=3, n_head=4, n_embd=128, adapter_prompt_length=10, adapter_start_layer=1)
SEED, ADAPTER_SEED = 1234, 4321


def state_dict():
    return A.adapter_state_dict(CFG["n_layer"], CFG["n_head"], CFG["n_embd"], CFG["vocab_size"], "gptq.int4",
                                CFG["adapter_prompt_length"], CFG["adapter_start_layer"], dtype=torch.bfloat16,
                                seed=SEED, adapter_seed=ADAPTER_SEED)


@torch.no_grad()
def golden_adapter_model():
    sd = state_dict()
    with quantization("gptq.int4"):
        m = ref_adapter.LLaMA(ref_adapter.LLaMAConfig(**CFG))
    m = m.to(torch.bfloat16)
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    m.eval()
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, CFG["vocab_size"], (7,), generator=g)
    out = dict(cfg=CFG, seed=SEED, adapter_seed=ADAPTER_SEED, prompt=prompt, state_dict_keys=sorted(m.state_dict().keys()))
    S = 16
    logits = [m(prompt.view(1, -1), S, torch.arange(7))]
    nxt = [11, 5, 90]
    for i, t in enumerate(nxt):
        logits.append(m(torch.tensor([[t]]), S, torch.tensor([7 + i])))
    out["steps_tokens"] = nxt
    out["steps_logits"] = [l.clone() for l in logits]
    m.reset_cache()
    out["nocache_logits"] = m(prompt.view(1, -1)).clone()
    m.reset_cache()
    S2 = 8
    roll = [m(prompt.view(1, -1), S2, torch.arange(7))[:, -1].clone()]
    toks = [3, 17, 40, 41, 2, 77]
    for i, t in enumerate(toks):
        roll.append(m(torch.tensor([[t]]), S2, torch.tensor([7 + i]))[:, -1].clone())
    out["roll_tokens"] = toks
    out["roll_logits"] = roll
    m.reset_cache()
    out["gen_greedy"] = ref_generate.generate(m, prompt.to(torch.int32), 12, top_k=1).clone()
    m.reset_cache()
    torch.manual_seed(1234)
    out["gen_sampled"] = ref_generate.generate(m, prompt.to(torch.int32), 12, temperature=0.8, top_k=20).clone()
    m.reset_cache()
    torch.save(out, os.path.join(OUT, "tiny_adapter_int4_bf16.pt"))


def golden_adapter_surface():
    """`name -> "defining_module.qualname"` for every class or function lit_llama.adapter and generate/adapter.py
    bind (the format of reference_surface.json)."""
    spec = importlib.util.spec_from_file_location("ref_generate_adapter", os.path.join(REF, "generate", "adapter.py"))
    gen_adapter = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_adapter)
    out = {}
    for key, mod in (("adapter", ref_adapter), ("generate_adapter", gen_adapter)):
        names = {}
        for name, obj in sorted(vars(mod).items()):
            origin = getattr(obj, "__module__", None)
            if name.startswith("__") or not callable(obj) or not isinstance(origin, str):
                continue
            if origin.startswith("lit_llama") or origin == mod.__name__:
                names[name] = f"{origin}.{getattr(obj, '__qualname__', name)}"
        out[key] = names
    with open(os.path.join(OUT, "reference_adapter_surface.json"), "w") as f:
        json.dump({"modules": out}, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    os.makedirs(OUT, exist_ok=True)
    golden_adapter_surface()
    golden_adapter_model()
    for f in ("tiny_adapter_int4_bf16.pt", "reference_adapter_surface.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()

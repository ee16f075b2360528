"""Generates the LoRA fixtures under tests/golden/ by running the UNMODIFIED reference on the CPU:

    python oracle/make_golden_lora.py

Writes only new files (the fixtures of oracle/make_golden.py and make_golden_adapter.py are not regenerated):
  * tiny_lora_bf16.pt:
      - a tiny dense LoRA model (the reference's lora() context, r 8, alpha 16, dropout 0.05, random non-zero lora_B,
        bf16) after eval(): prefill + 3 decode steps, the no-cache forward, the roll branch, greedy / sampled
        generate() tokens, and every layer's merged c_attn.weight;
      - stand-alone unmerged MergedLinear layers (lora_dropout 0) on random inputs: q / v and a 4-group pattern,
        which pin the branch arithmetic and the zero_pad layout;
  * reference_lora_surface.json: the names lit_llama.lora and generate/lora.py bind.
Needs the lit-llama checkout (default /root/reference; LIT_LLAMA_DIR overrides it) and oracle/_shim.  TEST INFRASTRUCTURE.
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
import lit_llama.lora as ref_lora  # noqa: E402
import lit_llama.model as ref_model  # noqa: E402

from oracle import llama_oracle as O  # noqa: E402
from oracle import lora_oracle as LO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)
LORA = dict(r=8, alpha=16, dropout=0.05)   # generate/lora.py:22-24
SEED, LORA_SEED = 1234, 4321


def state_dict():
    sd = O.synth_state_dict(CFG["n_layer"], CFG["n_head"], CFG["n_embd"], CFG["vocab_size"], None, dtype=torch.bfloat16,
                            seed=SEED)
    sd.update(LO.lora_weights(CFG["n_layer"], CFG["n_embd"], r=LORA["r"], seed=LORA_SEED))
    return sd


@torch.no_grad()
def golden_lora_model(out):
    sd = state_dict()
    with ref_lora.lora(**LORA):
        m = ref_model.LLaMA(ref_model.LLaMAConfig(**CFG))
    m = m.to(torch.bfloat16)
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert isinstance(m.transformer.h[0].attn.c_attn, ref_lora.MergedLinear)
    m.eval()
    assert m.transformer.h[0].attn.c_attn.merged
    out.update(cfg=CFG, lora=LORA, seed=SEED, lora_seed=LORA_SEED, state_dict_keys=sorted(m.state_dict().keys()))
    out["merged_c_attn"] = [blk.attn.c_attn.weight.detach().clone() for blk in m.transformer.h]
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, CFG["vocab_size"], (7,), generator=g)
    out["prompt"] = prompt
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


@torch.no_grad()
def golden_merged_linear(out):
    """Stand-alone unmerged MergedLinear layers (train mode, lora_dropout 0) on (B, T, in) inputs.  The reference's
    zero_pad transposes dims 0 and 1, so its unmerged forward only accepts inputs with at least 3 dims; a 2-D input
    is recorded as (1, M, in)."""
    g = torch.Generator().manual_seed(77)
    cases = []
    for in_f, out_f, r, alpha, enable, shapes in (
            (128, 384, 8, 16, [True, False, True], [(1, 6), (2, 5)]),
            (64, 256, 4, 6, [False, True, True, False], [(1, 3), (3, 4)])):
        layer = ref_lora.MergedLinear(in_f, out_f, r=r, lora_alpha=alpha, lora_dropout=0.0, enable_lora=enable,
                                      bias=False).to(torch.bfloat16)
        layer.weight.copy_((torch.randn(out_f, in_f, generator=g) * 0.05).to(torch.bfloat16))
        layer.lora_A.copy_((torch.rand(layer.lora_A.shape, generator=g) * 0.2 - 0.1).to(torch.bfloat16))
        layer.lora_B.copy_((torch.randn(layer.lora_B.shape, generator=g) * 0.05).to(torch.bfloat16))
        assert layer.training and not layer.merged
        for shape in shapes:
            x = torch.randn(*shape, in_f, generator=g).to(torch.bfloat16)
            cases.append(dict(in_features=in_f, out_features=out_f, r=r, alpha=alpha, enable_lora=enable,
                              weight=layer.weight.clone(), lora_A=layer.lora_A.clone(), lora_B=layer.lora_B.clone(),
                              x=x, y=layer(x).clone()))
    out["merged_linear_cases"] = cases


def golden_lora_surface():
    """`name -> "defining_module.qualname"` for every class or function lit_llama.lora and generate/lora.py bind (the
    format of reference_surface.json)."""
    spec = importlib.util.spec_from_file_location("ref_generate_lora", os.path.join(REF, "generate", "lora.py"))
    gen_lora = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_lora)
    out = {}
    for key, mod in (("lora", ref_lora), ("generate_lora", gen_lora)):
        names = {}
        for name, obj in sorted(vars(mod).items()):
            origin = getattr(obj, "__module__", None)
            if name.startswith("__") or not callable(obj) or not isinstance(origin, str):
                continue
            if origin.startswith("lit_llama") or origin == mod.__name__:
                names[name] = f"{origin}.{getattr(obj, '__qualname__', name)}"
        out[key] = names
    with open(os.path.join(OUT, "reference_lora_surface.json"), "w") as f:
        json.dump({"modules": out}, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    os.makedirs(OUT, exist_ok=True)
    golden_lora_surface()
    out = {}
    golden_lora_model(out)
    golden_merged_linear(out)
    torch.save(out, os.path.join(OUT, "tiny_lora_bf16.pt"))
    for f in ("tiny_lora_bf16.pt", "reference_lora_surface.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()

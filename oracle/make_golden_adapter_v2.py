"""Generates the LLaMA-Adapter v2 fixtures under tests/golden/ by running the UNMODIFIED reference on the CPU:

    python oracle/make_golden_adapter_v2.py

Writes only new files (no other generator's fixtures are regenerated):
  * tiny_adapter_v2_bf16.pt: lit_llama.adapter.LLaMA with v2's linear scale and bias, bf16, n_layer 3,
    adapter_start_layer 1, non-trivial scales / biases / norm scales (oracle/adapter_v2_oracle.py), on two bases:
      - "dense": the reference's own add_adapter_v2_parameters_to_linear_layers;
      - "gptq.int4": the reference's modules under quantization("gptq.int4").  The reference cannot attach v2 to
        them (its isinstance(module, nn.Linear) raises once torch.nn.Linear is a functools.partial, and its forward
        reads layer.weight), so this script attaches adapter_bias / adapter_scale itself and binds
        forward = adapter_scale * (ref_forward(x) + adapter_bias): adapter_v2_new_forward with the reference's own
        CPU linear, F.linear(x, get_weight(), bias), in place of F.linear(x, W, b).
    For each: prefill + 3 decode steps, the no-cache forward, the roll branch and greedy / sampled generate() tokens.
  * reference_adapter_v2_surface.json: the names lit_llama.adapter_v2 and generate/adapter_v2.py bind.
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
import lit_llama.adapter as ref_adapter  # noqa: E402
import lit_llama.adapter_v2 as ref_v2  # noqa: E402
import lit_llama.quantization as ref_quant  # noqa: E402
from lit_llama.utils import quantization  # noqa: E402

from oracle import adapter_v2_oracle as A2  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CFG = dict(block_size=64, vocab_size=96, n_layer=3, n_head=4, n_embd=128, adapter_prompt_length=10, adapter_start_layer=1)
SEED, ADAPTER_SEED, V2_SEED = 1234, 4321, 2468


def state_dict(mode):
    return A2.adapter_v2_state_dict(CFG["n_layer"], CFG["n_head"], CFG["n_embd"], CFG["vocab_size"], mode,
                                    CFG["adapter_prompt_length"], CFG["adapter_start_layer"], dtype=torch.bfloat16,
                                    seed=SEED, adapter_seed=ADAPTER_SEED, v2_seed=V2_SEED)


def attach_v2_to_quantized(model):
    """v2's parameters and forward on the reference's ColBlockQuantizedLinear modules (see the module docstring)."""
    for module in model.modules():
        if isinstance(module, ref_quant.ColBlockQuantizedLinear):
            n = module.out_features
            module.adapter_bias = torch.nn.Parameter(torch.zeros(n))
            module.adapter_scale = torch.nn.Parameter(torch.ones(n))
            ref_forward = module.forward   # the class's forward, bound: F.linear(x, get_weight(), bias) on the CPU

            def forward(x, self=module, ref_forward=ref_forward):
                return self.adapter_scale * (ref_forward(x) + self.adapter_bias)

            module.forward = forward


@torch.no_grad()
def run(mode):
    sd = state_dict(mode)
    if mode is None:
        m = ref_adapter.LLaMA(ref_adapter.LLaMAConfig(**CFG))
        ref_v2.add_adapter_v2_parameters_to_linear_layers(m)
    else:
        with quantization(mode):
            m = ref_adapter.LLaMA(ref_adapter.LLaMAConfig(**CFG))
        attach_v2_to_quantized(m)
    m = m.to(torch.bfloat16)
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    m.eval()
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, CFG["vocab_size"], (7,), generator=g)
    out = dict(prompt=prompt, state_dict_keys=sorted(m.state_dict().keys()))
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
    return out


def golden_adapter_v2_model():
    out = dict(cfg=CFG, seed=SEED, adapter_seed=ADAPTER_SEED, v2_seed=V2_SEED,
               bases={"dense": run(None), "gptq.int4": run("gptq.int4")})
    torch.save(out, os.path.join(OUT, "tiny_adapter_v2_bf16.pt"))


def golden_adapter_v2_surface():
    """`name -> "defining_module.qualname"` for every class or function lit_llama.adapter_v2 and generate/adapter_v2.py
    bind (the format of reference_surface.json)."""
    spec = importlib.util.spec_from_file_location("ref_generate_adapter_v2", os.path.join(REF, "generate", "adapter_v2.py"))
    gen_v2 = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_v2)
    out = {}
    for key, mod in (("adapter_v2", ref_v2), ("generate_adapter_v2", gen_v2)):
        names = {}
        for name, obj in sorted(vars(mod).items()):
            origin = getattr(obj, "__module__", None)
            if name.startswith("__") or not callable(obj) or not isinstance(origin, str):
                continue
            if origin.startswith("lit_llama") or origin == mod.__name__:
                names[name] = f"{origin}.{getattr(obj, '__qualname__', name)}"
        out[key] = names
    with open(os.path.join(OUT, "reference_adapter_v2_surface.json"), "w") as f:
        json.dump({"modules": out}, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    os.makedirs(OUT, exist_ok=True)
    golden_adapter_v2_surface()
    golden_adapter_v2_model()
    for f in ("tiny_adapter_v2_bf16.pt", "reference_adapter_v2_surface.json"):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()

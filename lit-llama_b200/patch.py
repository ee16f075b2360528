"""Plug the H100 modules into an UNMODIFIED reference checkout.

The reference resolves its classes through module globals at construction time
(lit_llama/model.py:61,152,154 and the torch.nn.Linear swap of utils.py:156-162 - the
same trick its own lora() context uses, lit_llama/lora.py:472-476).  After

    import lit_llama, lit_llama_b200
    lit_llama_b200.patch_reference(lit_llama)

the reference's own `generate.py` (`main()`, `--quantize gptq.int4`) builds H100
modules: `lit_llama.LLaMA`, `lit_llama.model.{LLaMA,Block,CausalSelfAttention,MLP,
RMSNorm,apply_rope,build_rope_cache}`, `lit_llama.quantization.{ColBlockQuantizedLinear,
Linear8bitLt}`, `lit_llama.utils.{quantization,EmptyInitOnDevice,lazy_load}` and, when the
package has it, `lit_llama.adapter.{LLaMA,LLaMAConfig,Block,CausalSelfAttention}` (LLaMA-Adapter,
`generate/adapter.py`) and `lit_llama.lora.{lora,MergedLinear,LoRALayer,LoRAConfig,CausalSelfAttention,
mark_only_lora_as_trainable,lora_state_dict}` (LoRA, `generate/lora.py`) and `lit_llama.adapter_v2.{get_adapter_substrings,
mark_only_adapter_v2_as_trainable,adapter_v2_state_from_state_dict,adapter_v2_new_forward,
adapter_v2_linear_with_bias_and_scale,add_adapter_v2_parameters_to_linear_layers}` (LLaMA-Adapter v2,
`generate/adapter_v2.py`) all point at this package.
"""
import sys


def patch_reference(lit_llama_module=None):
    from . import model as m, quantization as q, utils as u

    if lit_llama_module is None:
        import lit_llama as lit_llama_module  # noqa: N813
    ref_model = sys.modules[lit_llama_module.__name__ + ".model"]
    ref_utils = sys.modules[lit_llama_module.__name__ + ".utils"]
    ref_quant = sys.modules.get(lit_llama_module.__name__ + ".quantization")
    if ref_quant is None:
        import importlib

        ref_quant = importlib.import_module(lit_llama_module.__name__ + ".quantization")
    saved = {}
    for name in ("LLaMA", "LLaMAConfig", "Block", "CausalSelfAttention", "MLP", "RMSNorm", "apply_rope", "build_rope_cache"):
        saved[("model", name)] = getattr(ref_model, name)
        setattr(ref_model, name, getattr(m, name))
        if hasattr(lit_llama_module, name):
            saved[("pkg", name)] = getattr(lit_llama_module, name)
            setattr(lit_llama_module, name, getattr(m, name))
    saved[("quant", "ColBlockQuantizedLinear")] = ref_quant.ColBlockQuantizedLinear
    ref_quant.ColBlockQuantizedLinear = q.ColBlockQuantizedLinear
    from . import int8 as i8

    saved[("quant", "Linear8bitLt")] = getattr(ref_quant, "Linear8bitLt", None)  # absent when bitsandbytes is not installed
    ref_quant.Linear8bitLt = i8.Linear8bitLt
    saved[("quant", "qlinear_4bit_weight")] = getattr(ref_quant, "qlinear_4bit_weight", None)
    ref_quant.qlinear_4bit_weight = q.qlinear_4bit_weight
    # The offline converter stays the reference's own (quantize/gptq.py + quantization.GPTQQuantizer, host-side torch,
    # out of the decode path): it builds `ColBlockQuantizedLinear` through the name patched above and calls
    # pack_weight(), so it converts straight into H100 modules.
    for name in ("EmptyInitOnDevice", "lazy_load"):
        saved[("utils", name)] = getattr(ref_utils, name, None)
        setattr(ref_utils, name, getattr(u, name))
    saved[("utils", "quantization")] = ref_utils.quantization
    ref_utils.quantization = u.quantization
    # LLaMA-Adapter (lit_llama/adapter.py), when the package has it
    ref_adapter = sys.modules.get(lit_llama_module.__name__ + ".adapter")
    if ref_adapter is None:
        import importlib

        try:
            ref_adapter = importlib.import_module(lit_llama_module.__name__ + ".adapter")
        except ImportError:
            ref_adapter = None
    if ref_adapter is not None:
        from . import adapter as a

        for name in ("LLaMA", "LLaMAConfig", "Block", "CausalSelfAttention"):
            saved[("adapter", name)] = getattr(ref_adapter, name, None)
            setattr(ref_adapter, name, getattr(a, name))
    # LoRA (lit_llama/lora.py), when the package has it
    ref_lora = sys.modules.get(lit_llama_module.__name__ + ".lora")
    if ref_lora is None:
        import importlib

        try:
            ref_lora = importlib.import_module(lit_llama_module.__name__ + ".lora")
        except ImportError:
            ref_lora = None
    if ref_lora is not None:
        from . import lora as lo

        for name in ("LoRALayer", "MergedLinear", "LoRAConfig", "CausalSelfAttention", "lora", "mark_only_lora_as_trainable",
                     "lora_state_dict"):
            saved[("lora", name)] = getattr(ref_lora, name, None)
            setattr(ref_lora, name, getattr(lo, name))
    # LLaMA-Adapter v2 (lit_llama/adapter_v2.py), when the package has it
    ref_v2 = sys.modules.get(lit_llama_module.__name__ + ".adapter_v2")
    if ref_v2 is None:
        import importlib

        try:
            ref_v2 = importlib.import_module(lit_llama_module.__name__ + ".adapter_v2")
        except ImportError:
            ref_v2 = None
    if ref_v2 is not None:
        from . import adapter_v2 as a2

        for name in ("get_adapter_substrings", "mark_only_adapter_v2_as_trainable", "adapter_v2_state_from_state_dict",
                     "adapter_v2_new_forward", "adapter_v2_linear_with_bias_and_scale",
                     "add_adapter_v2_parameters_to_linear_layers"):
            saved[("adapter_v2", name)] = getattr(ref_v2, name, None)
            setattr(ref_v2, name, getattr(a2, name))
    for mod in list(sys.modules.values()):  # scripts that did `from lit_llama.utils import quantization`
        if mod is not None and getattr(mod, "quantization", None) is saved[("utils", "quantization")]:
            setattr(mod, "quantization", u.quantization)
        if mod is not None and getattr(mod, "LLaMA", None) is saved[("model", "LLaMA")]:
            setattr(mod, "LLaMA", m.LLaMA)
        # generate/adapter.py did `from lit_llama.adapter import LLaMA`
        if ref_adapter is not None and mod is not None and saved[("adapter", "LLaMA")] is not None \
                and getattr(mod, "LLaMA", None) is saved[("adapter", "LLaMA")]:
            setattr(mod, "LLaMA", a.LLaMA)
        # generate/lora.py did `from lit_llama.lora import lora`
        if ref_lora is not None and mod is not None and saved[("lora", "lora")] is not None \
                and getattr(mod, "lora", None) is saved[("lora", "lora")]:
            setattr(mod, "lora", lo.lora)
        # generate/adapter_v2.py did `from lit_llama.adapter_v2 import add_adapter_v2_parameters_to_linear_layers`
        name = "add_adapter_v2_parameters_to_linear_layers"
        if ref_v2 is not None and mod is not None and saved[("adapter_v2", name)] is not None \
                and getattr(mod, name, None) is saved[("adapter_v2", name)]:
            setattr(mod, name, getattr(a2, name))
    return saved

"""lit-llama_b200: H100 (sm_90a) quantized-decode path for Lightning-AI/lit-llama.

Mirrors the reference's public surface for this path (lit_llama/__init__.py):
`LLaMA, LLaMAConfig, RMSNorm, build_rope_cache, apply_rope`, the quantized linears of
`lit_llama/quantization.py` and `utils.quantization()` of `lit_llama/utils.py` (import it
as `from lit_llama_b200.utils import quantization`, like the reference), all backed
by hand-written CUDA in `csrc/` behind the C ABI of `include/b2l.h`.
"""
from .model import LLaMA, LLaMAConfig, Block, CausalSelfAttention, MLP, RMSNorm, build_rope_cache, apply_rope
from .quantization import ColBlockQuantizedLinear
from .int8 import Linear8bitLt
from .utils import find_multiple, llama_model_lookup
from .generate import (generate, generate_batch, generate_prompts, generate_speculative, generate_stream, sample_probs,
                       sample_token)
from .patch import patch_reference
from .tp import TPLLaMA, shard_state_dict
from . import evaluate

__all__ = [
    "LLaMA", "LLaMAConfig", "Block", "CausalSelfAttention", "MLP", "RMSNorm", "build_rope_cache", "apply_rope",
    "ColBlockQuantizedLinear", "Linear8bitLt", "find_multiple", "llama_model_lookup", "generate", "generate_batch", "generate_prompts", "generate_speculative", "generate_stream", "sample_probs", "sample_token", "patch_reference", "TPLLaMA", "shard_state_dict",
    "evaluate",
]

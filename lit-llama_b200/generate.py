"""generate.py of the reference (generate.py:20-91, 94-155) over the H100 modules.

`generate()` keeps the reference's Python token loop and torch sampling ops (so the
RNG stream of `torch.multinomial` is the reference's); the model call inside it is one
CUDA-graph replay per token.  `generate_batch()` draws up to 16 samples of one prompt
at once: one batch-1 prefill, then one batched decode step and one sampling launch per
token for all samples.  `generate_prompts()` continues up to 16 different prompts at
once: one batch-1 prefill per prompt into its row of the cache, then one batched decode
step at per-row positions and one sampling launch per token.  `generate_stream()` decodes any number of
prompts on up to 16 rows, refilling each finished row with the next prompt while the others keep decoding
(continuous batching).  `generate_speculative()`
lets a small draft model, or prompt lookup over the sequence's own n-grams, propose up to 15 tokens that the model
verifies in one step (speculative sampling); its greedy output is `generate()`'s token for token.
`main()` mirrors the reference CLI with argparse
(jsonargparse and lightning are not dependencies of this path)."""
import os
import re
import sys
import time
from collections import deque
from pathlib import Path
from typing import List, Optional, Sequence, Union

import torch

from . import _lib as L
from .model import LLaMA
from .utils import llama_model_lookup, quantization


_TORCH_MULTINOMIAL = torch.multinomial


#: most samples generate_batch() draws at once: the range of the batched decode step (B = 2..16)
MAX_SAMPLES = 16


def _rows(logits: torch.Tensor):
    """(x, ld) for the row entry points: (B, V) logits with unit stride along V and 16-byte aligned, rows ld >= V
    elements apart, or ld = 0 for one row expanded to B rows (`row.expand(B, -1)`); read in place when they already
    are, else copied."""
    B, V = logits.shape
    if B > 1 and logits.stride(0) == 0:   # one row for every sample
        row = logits[0].contiguous()
        if row.data_ptr() % 16:
            row = row.clone()
        return row, 0
    x = logits
    if (V > 1 and x.stride(1) != 1) or (B > 1 and x.stride(0) < V):
        x = x.contiguous()
    if x.data_ptr() % 16:
        x = x.clone(memory_format=torch.contiguous_format)   # the kernel reads 16-byte vectors
    return x, (x.stride(0) if B > 1 else V)


def sample_probs(logits_row: torch.Tensor, temperature: float = 1.0, top_k: Optional[int] = None) -> torch.Tensor:
    """generate.py:68-75: probabilities of the next token from the last position's logits
    (V,) bf16: temperature, top-k filter and softmax fused in one kernel (b2l_topk_softmax_rows on one row).
    (B, V) logits give (B, V) probabilities, every row in the same launch, each row bit-equal to the (V,) call on it."""
    L.require_cuda_bf16(logits_row, "sample_probs")
    rows = logits_row if logits_row.dim() == 2 else logits_row.reshape(1, -1)   # (V,): one row
    x, ld = _rows(rows)
    B, V = rows.shape
    probs = torch.empty((B, V), dtype=x.dtype, device=x.device)
    k = 0 if top_k is None else min(int(top_k), V)
    L.check(L.lib().b2l_topk_softmax_rows(x.data_ptr(), ld, float(temperature), k, probs.data_ptr(), B, V, L.stream_ptr()),
            "b2l_topk_softmax_rows")
    return probs if logits_row.dim() == 2 else probs.view(logits_row.shape)


def sample_token(logits_row: torch.Tensor, temperature: float = 1.0, top_k: Optional[int] = None) -> torch.Tensor:
    """generate.py:68-76: the next token (shape (1,), int64) drawn from the last position's logits.
    `torch.multinomial(probs, num_samples=1)` is `argmax(probs / q)` with `q = empty_like(probs).exponential_(1)`
    (ATen/native/Distributions.cpp); q is drawn here with torch -- the RNG consumption of multinomial, so for the same
    generator state the token equals `torch.multinomial(sample_probs(...), 1)` -- and everything else is one
    launch (b2l_topk_softmax_sample_rows) instead of multinomial's dozen.
    (B, V) logits give (B,) tokens: q is one [B, V] draw, as multinomial makes on [B, V] probabilities, so token b
    equals `torch.multinomial(sample_probs(logits), 1)[b]`, and all rows are drawn in one launch."""
    L.require_cuda_bf16(logits_row, "sample_token")
    rows = logits_row if logits_row.dim() == 2 else logits_row.reshape(1, -1)   # (V,): one row
    x, ld = _rows(rows)
    B, V = rows.shape
    q = torch.empty((B, V), dtype=x.dtype, device=x.device).exponential_(1)
    tokens = torch.empty(B, dtype=torch.int64, device=x.device)
    k = 0 if top_k is None else min(int(top_k), V)
    L.check(L.lib().b2l_topk_softmax_sample_rows(x.data_ptr(), ld, float(temperature), k, q.data_ptr(), None, tokens.data_ptr(),
                                                 B, V, L.stream_ptr()), "b2l_topk_softmax_sample_rows")
    return tokens


def _draw(rows: torch.Tensor, temperature: float, top_k: Optional[int], dtype: torch.dtype) -> torch.Tensor:
    """One token per row of `rows` ((V,) or (B, V) logits), as `dtype`: sample_token (one RNG draw and one launch for
    all rows), or, while torch.multinomial is replaced (the reference's tests/test_generate.py:26-54 patches it to record
    the draws), torch.multinomial on the fused probabilities."""
    if torch.multinomial is _TORCH_MULTINOMIAL:
        return sample_token(rows, temperature, top_k).to(dtype=dtype)
    return torch.multinomial(sample_probs(rows, temperature, top_k), num_samples=1).view(-1).to(dtype=dtype)


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
        idx_next = _draw(logits[0, -1], temperature, top_k, dtype)   # generate.py:68-76
        input_pos = input_pos[-1:] + 1
        idx = idx.index_copy(0, input_pos, idx_next)
        if eos_id is not None and idx_next == eos_id:
            return idx[:input_pos]  # include the EOS token
    return idx


@torch.no_grad()
def generate_batch(
    model: LLaMA,
    idx: torch.Tensor,
    num_samples: int,
    max_new_tokens: int,
    *,
    max_seq_length: Optional[int] = None,
    temperature: float = 1.0,
    top_k: Optional[int] = None,
    eos_id: Optional[int] = None,
) -> List[torch.Tensor]:
    """`num_samples` (1..16) continuations of one prompt `idx` (T,), drawn together: a list of `num_samples` 1-D
    tensors, each the prompt plus that sample's new tokens (generate.py:20-91 per row).

    The prompt is prefilled once, at batch 1, and `LLaMA.expand_cache` copies its KV cache to every row; the first
    tokens are all drawn from the prefill's last position.  Each later token is one batched model call (whatever path
    the model runs at B = num_samples) and one sampling launch for all rows; positions are shared, so the roll branch
    (model.py:214-218) applies when T + max_new_tokens > max_seq_length.  Row b's token is
    `torch.multinomial(probs, 1)[b]` of the step's [B, V] probabilities, with multinomial's RNG consumption, so
    `num_samples=1` gives `generate()`'s tokens for the same seed.

    With `eos_id`, a row that draws it ends there, the eos token included; finished rows keep riding along (their
    later tokens are dropped) and the loop stops once every row has finished, reading one flag per step.  The cache
    is left at B = num_samples: call `model.reset_cache()` before the next prompt, as after `generate()`."""
    if not 1 <= int(num_samples) <= MAX_SAMPLES:
        raise ValueError(f"generate_batch: num_samples = {num_samples}; 1..{MAX_SAMPLES} (the batched decode step's range)")
    if idx.dim() != 1:
        raise ValueError(f"generate_batch: idx must be one prompt of shape (T,), got {tuple(idx.shape)}")
    if not idx.is_cuda:
        raise RuntimeError(f"generate_batch: idx is on {idx.device}; lit_llama_b200 runs on CUDA only (no CPU fallback)")
    B = int(num_samples)
    T = idx.size(0)
    T_new = T + max_new_tokens
    if max_seq_length is None:
        max_seq_length = min(T_new, model.config.block_size)

    device, dtype = idx.device, idx.dtype
    out = torch.empty((B, T_new), dtype=dtype, device=device)
    out[:, :T] = idx
    input_pos = torch.arange(0, T, device=device)
    x = idx.view(1, -1)
    end = torch.full((B,), T_new, dtype=torch.int64, device=device) if eos_id is not None else None
    done = torch.zeros(B, dtype=torch.bool, device=device) if eos_id is not None else None

    for i in range(max_new_tokens):
        logits = model(x, max_seq_length, input_pos)
        if i == 0:
            model.expand_cache(B)
            rows = logits[0, -1].expand(B, -1)   # every sample's first token comes from the prompt's last position
        else:
            rows = logits[:, -1]
        idx_next = _draw(rows, temperature, top_k, dtype)
        input_pos = input_pos[-1:] + 1
        out[:, T + i] = idx_next
        x = idx_next.view(B, 1)
        if eos_id is not None:
            hit = (idx_next == eos_id) & ~done
            end = torch.where(hit, T + i + 1, end)   # include the eos token
            done |= hit
            if bool(done.all()):
                break
    if end is None:
        return list(out.unbind(0))
    return [out[b, :n] for b, n in enumerate(end.tolist())]


#: most draft tokens one generate_speculative() round proposes: the verify step runs 2..16 tokens
MAX_DRAFT = 15

#: longest n-gram prompt lookup matches (b2l_ngram_propose)
MAX_NGRAM = 16


@torch.no_grad()
def generate_speculative(
    model: LLaMA,
    draft: Optional[LLaMA],
    idx: torch.Tensor,
    max_new_tokens: int,
    *,
    num_draft: int = 4,
    max_seq_length: Optional[int] = None,
    temperature: float = 1.0,
    top_k: Optional[int] = None,
    eos_id: Optional[int] = None,
    stats: Optional[dict] = None,
    max_ngram: int = 3,
    min_ngram: int = 1,
) -> torch.Tensor:
    """Speculative sampling: `idx` (T,) prompt -> (T + max_new_tokens,) tokens like `generate()`, with draft tokens
    that `model` verifies several at a time.  `draft` (a smaller model over the same vocabulary) proposes them, or,
    with `draft=None`, prompt lookup: the tokens that followed the most recent earlier occurrence of the sequence's
    last g tokens, g = max_ngram down to min_ngram (1..16; the rule of `b2l_ngram_propose`, include/b2l.h).

    `model` (and the draft) prefill the prompt at batch 1 and the first token is drawn from `model`'s prefill logits
    as in `generate()`.  Each round proposes k = num_draft (1..15) tokens with their probability rows q: k batch-1
    draft steps, each sampling its token with the fused kernel, or the proposal of one `b2l_ngram_propose` launch
    (q one-hot).  Then one `LLaMA.decode_tokens` of `model` over the pending token and the k proposed tokens, and one
    `b2l_spec_accept` launch, which accepts token t while u_t q_t(x_t) < p_t(x_t) and draws the next token from the
    residual max(0, p_j - q_j) at the first rejection j (from p_k when all are accepted), so every emitted token is
    distributed as `model`'s own samples.  The round's only host synchronisation is one 4-byte read of the number
    accepted (with `eos_id`, the first eos among the emitted tokens travels in the same word).  When all k are
    accepted the draft also consumes the last of them.  Rejected cache slots of either model are left stale: they are
    never read and are overwritten later.

    Prompt lookup launches the next round's proposer right behind the accept, over the history extended by the
    round's emitted tokens on the device, so the same read also carries the next proposal count, and a round uses
    min(k, count) of them.  A count of 0 runs one plain target step (`model` + `sample_token`), then the proposer,
    then the same one read.

    With top_k=1 a token is accepted exactly when it is the target's argmax, and `decode_tokens` rows are bit-identical
    to the batch-1 step, so the output equals `generate(model, ..., top_k=1)` token for token whatever is proposed.

    k shrinks so that the verified positions stay below max_seq_length and no round overshoots max_new_tokens; from
    the point where no draft token fits (the roll branch included) the tail runs `generate()`'s plain target steps.
    With `eos_id` the output ends at the first eos, which is included.  `stats`, when given, receives "rounds",
    "proposed" / "accepted" (lists: draft tokens per round), "num_draft", "tail_steps" and "lookup_misses" (plain
    steps prompt lookup ran for want of a proposal; 0 with a draft model).  Call `reset_cache()` on the model(s)
    before the next prompt, as after `generate()`."""
    if not 1 <= int(num_draft) <= MAX_DRAFT:
        raise ValueError(f"generate_speculative: num_draft = {num_draft}; 1..{MAX_DRAFT} (the verify step runs 2..16 tokens)")
    if draft is None:
        if not 1 <= int(min_ngram) <= int(max_ngram) <= MAX_NGRAM:
            raise ValueError(f"generate_speculative: min_ngram = {min_ngram}, max_ngram = {max_ngram}; "
                             f"1 <= min_ngram <= max_ngram <= {MAX_NGRAM}")
    elif draft.config.padded_vocab_size != model.config.padded_vocab_size:
        raise ValueError(f"generate_speculative: the draft's padded_vocab_size {draft.config.padded_vocab_size} differs from "
                         f"the target's {model.config.padded_vocab_size}")
    if idx.dim() != 1:
        raise ValueError(f"generate_speculative: idx must be one prompt of shape (T,), got {tuple(idx.shape)}")
    why = model._decode_route(int(num_draft) + 1, stepwise=True)
    if isinstance(why, str):
        raise RuntimeError(f"generate_speculative: the target's verify step (LLaMA.decode_tokens) {why}")
    if not idx.is_cuda:
        raise RuntimeError(f"generate_speculative: idx is on {idx.device}; lit_llama_b200 runs on CUDA only (no CPU fallback)")
    T = idx.size(0)
    T_new = T + max_new_tokens
    if max_seq_length is None:
        max_seq_length = min(T_new, model.config.block_size)
    S = max_seq_length
    device, dtype = idx.device, idx.dtype
    V = model.config.padded_vocab_size
    lib = L.lib()
    kmax = int(num_draft)
    k_top = 0 if top_k is None else min(int(top_k), V)
    out = torch.empty(T_new, dtype=torch.int64 if draft is None else dtype, device=device)   # lookup reads it as int64
    out[:T] = idx
    st = {} if stats is None else stats
    st.update(rounds=0, proposed=[], accepted=[], num_draft=kmax, tail_steps=0, lookup_misses=0)
    if max_new_tokens <= 0:
        return out.to(dtype)

    pos_all = torch.arange(0, max(T_new, S), device=device)
    logits = model(idx.view(1, -1), S, pos_all[:T])
    if draft is not None:
        draft(idx.view(1, -1), S, pos_all[:T])
    # tokens stay int64 on the device (one step state per model: its idx dtype never changes)
    tok = sample_token(logits[0, -1], temperature, top_k)   # generate()'s first token
    out[T] = tok[0]
    n = 1                                  # tokens emitted; the last one (tok) is in neither cache yet

    q = torch.empty((kmax, V), dtype=torch.bfloat16, device=device)   # the proposals' probability rows
    dtok = torch.empty((kmax + 1, 1), dtype=torch.int64, device=device)   # d_1..d_k, then the target's next token
    nacc = torch.zeros(1, dtype=torch.int32, device=device)
    steps = torch.arange(kmax + 1, device=device)
    count = torch.zeros(1, dtype=torch.int32, device=device)   # prompt lookup: the proposal's length
    none = torch.zeros(1, dtype=torch.int32, device=device)    # a plain step accepts nothing

    def propose(base_len: int, grown: bool) -> None:
        """b2l_ngram_propose over out[:base_len], plus the last round's nacc + 1 tokens when `grown`."""
        L.check(lib.b2l_ngram_propose(out.data_ptr(), base_len, nacc.data_ptr() if grown else None, int(min_ngram),
                                      int(max_ngram), kmax, dtok.data_ptr(), q.data_ptr(), count.data_ptr(), V,
                                      L.stream_ptr()), "b2l_ngram_propose")

    def read(em: torch.Tensor, acc: torch.Tensor):
        """The one host read of a round or plain step: (number accepted, index of the first eos among the emitted
        tokens em[:acc + 1] or 255, the next proposal count), packed in one word."""
        w = acc.long()[0]
        if eos_id is not None:
            hit = (em == eos_id) & (steps[:em.numel()] <= w)
            w = w | (torch.where(hit, steps[:em.numel()], 255).min() << 8)
        if draft is None:
            w = w | (count.long()[0] << 16)
        w = int(w.to(torch.int32).item())
        return w & 255, (w >> 8) & 255 if eos_id is not None else 255, w >> 16

    def plain_step() -> None:
        """generate()'s target step: the pending token in, the next one drawn and emitted."""
        nonlocal tok, n
        p = T + n - 1
        logits = model(tok.view(1, 1), S, pos_all[p:p + 1])
        tok = sample_token(logits[0, -1], temperature, top_k)
        out[T + n] = tok[0]
        n += 1

    if draft is None:
        propose(T + 1, False)
        _, e, c = read(tok, none)
        if e != 255:
            return out[:T + 1].to(dtype)
    elif eos_id is not None and int(tok[0]) == eos_id:
        return out[:T + 1]

    while n < max_new_tokens:
        p = T + n - 1                       # position of the pending token
        k = min(kmax, S - 1 - p, max_new_tokens - n - 1)
        if k < 1:
            break
        if draft is None:
            k = min(k, c)
            if k == 0:                      # no proposal: one plain target step, then the proposer again
                plain_step()
                st["lookup_misses"] += 1
                propose(T + n, False)
                _, e, c = read(tok, none)
                if e != 255:
                    return out[:T + n].to(dtype)
                continue
        else:
            x = tok.view(1, 1)
            for i in range(k):              # k batch-1 draft steps: tok, d_1 .. d_{k-1}
                dl = draft(x, S, pos_all[p + i:p + i + 1])[0, -1].contiguous()
                noise = torch.empty_like(dl).exponential_(1)
                L.check(lib.b2l_topk_softmax_sample(dl.data_ptr(), float(temperature), k_top, noise.data_ptr(),
                                                    q[i].data_ptr(), dtok[i].data_ptr(), V, L.stream_ptr()),
                        "b2l_topk_softmax_sample")
                x = dtok[i].view(1, 1)
        vidx = torch.cat((tok.view(1, 1), dtok[:k].view(1, k)), dim=1)
        tl = model.decode_tokens(vidx, S, pos_all[p:p + k + 1])
        u = torch.rand(k, device=device)
        noise = torch.empty(V, dtype=torch.bfloat16, device=device).exponential_(1)
        L.check(lib.b2l_spec_accept(tl.data_ptr(), V, float(temperature), k_top, q.data_ptr(), dtok.data_ptr(), u.data_ptr(),
                                    noise.data_ptr(), nacc.data_ptr(), dtok[k].data_ptr(), k + 1, V, L.stream_ptr()),
                "b2l_spec_accept")
        # the round's tokens: d_1..d_a, then the target's token (at slot a); later slots are overwritten by later rounds
        em = torch.where(steps[:k + 1] < nacc.long(), dtok[:k + 1, 0], dtok[k, 0]).to(out.dtype)
        out[T + n:T + n + k + 1] = em
        tok = dtok[k].clone()
        if draft is None:                   # the next proposal, over the history grown by this round's a + 1 tokens
            propose(T + n, True)
        a, e, c = read(em, nacc)
        st["rounds"] += 1
        st["proposed"].append(k)
        st["accepted"].append(a)
        if e != 255:
            return out[:T + n + e + 1].to(dtype)
        if draft is not None and a == k:    # every draft token accepted: the draft also consumes d_k
            draft(dtok[k - 1].view(1, 1), S, pos_all[p + k:p + k + 1])
        n += a + 1

    # the tail: generate()'s plain target steps (no draft token fits below max_seq_length, or one token is left)
    while n < max_new_tokens:
        plain_step()
        st["tail_steps"] += 1
        if eos_id is not None and tok == eos_id:
            return out[:T + n].to(dtype)
    return out.to(dtype)


@torch.no_grad()
def generate_prompts(
    model: LLaMA,
    prompts: List[torch.Tensor],
    max_new_tokens: int,
    *,
    max_seq_length: Optional[int] = None,
    temperature: float = 1.0,
    top_k: Optional[int] = None,
    eos_id: Optional[int] = None,
    adapters: Optional[Sequence[int]] = None,
) -> List[torch.Tensor]:
    """Continuations of 1..16 different prompts (1-D tensors of any lengths), decoded together: a list of 1-D tensors,
    row b the prompt `prompts[b]` plus its new tokens (generate.py:20-91 per row), each of `prompts[0]`'s dtype.

    `generate_stream` on B = len(prompts) rows, so no row is ever refilled: `LLaMA.prefill_rows` runs each prompt
    through the batch-1 prefill into its own row of one cache; the first tokens are drawn from those last positions.
    Each later token is one batched model call with a (B, 1) `input_pos`, row b at position len(prompts[b]) + i with
    its own KV ring (each row takes the roll branch, model.py:214-218, on its own once it passes max_seq_length), and
    one sampling launch for all rows.  max_seq_length defaults to min(longest prompt + max_new_tokens, block_size).
    Row b's token is `torch.multinomial(probs, 1)[b]` of the step's [B, V] probabilities, so one prompt gives
    `generate()`'s tokens for the same seed.

    With `eos_id`, a row that draws it ends there, the eos token included; finished rows keep riding along (their later
    tokens are dropped) and the loop stops once every row has finished, reading the step's eos flags once per step.
    The cache is left at B rows: call `model.reset_cache()` before a batch-1 `generate()`.

    `adapters` (multi-LoRA, lit_llama_b200.lora.add_lora_adapter): one adapter id per prompt (-1: the base alone);
    prompt b is prefilled and decoded with its own adapter (LLaMA.prefill_rows)."""
    B = len(prompts)
    if not 1 <= B <= MAX_SAMPLES:
        raise ValueError(f"generate_prompts: {B} prompts; 1..{MAX_SAMPLES} (the batched decode step's range)")
    ys = generate_stream(model, prompts, max_new_tokens, batch_size=B, max_seq_length=max_seq_length,
                         temperature=temperature, top_k=top_k, eos_id=eos_id, adapters=adapters, _who="generate_prompts")
    return [y.to(prompts[0].dtype) for y in ys]


@torch.no_grad()
def generate_stream(
    model: LLaMA,
    prompts: List[torch.Tensor],
    max_new_tokens: Union[int, Sequence[int]],
    *,
    batch_size: int = MAX_SAMPLES,
    max_seq_length: Optional[int] = None,
    temperature: float = 1.0,
    top_k: Optional[int] = None,
    eos_id: Optional[int] = None,
    stats: Optional[dict] = None,
    adapters: Optional[Sequence[int]] = None,
    _who: str = "generate_stream",
) -> List[torch.Tensor]:
    """Continuations of any number of prompts (1-D tensors of any lengths) on B = min(batch_size, len(prompts)) rows
    (batch_size 1..16), refilling each finished row with the next prompt while the others keep decoding (continuous
    batching): a list of 1-D tensors in input order, prompt i plus its new tokens (generate.py:20-91 per prompt).

    `max_new_tokens` is one int for every prompt or one per prompt.  The first B prompts go through
    `LLaMA.prefill_rows`.  Each later step is one batched model call with a (B, 1) `input_pos` and one sampling launch
    for all rows; a row finishes when it has its prompt's `max_new_tokens` or draws `eos_id` (included).  The rows
    that finish in a step take the next prompts in input order, all in one `LLaMA.refill_rows` call behind the next
    step's model call, and their first tokens are drawn from the refill's logits in that step's sampling launch.  Once
    no prompt is left, finished rows ride along and their tokens are dropped.  With `eos_id` the host reads the step's
    eos hits (B flags) once per step; without it, it knows from the counts when each row finishes.
    max_seq_length (S) defaults to min(max over prompts of T_i + new_i, block_size); each row takes the roll branch
    (model.py:214-218) on its own, and a refill restarts its row's ring.

    Draws are argmax(probs / q) of their row's probabilities (sample_token).  On the exact batched steps
    (`q4_batch_step`, `w8_batch_step`) every row is bit-identical to the batch-1 model, so with top_k=1 prompt i gets
    `generate(model, prompts[i], new_i, max_seq_length=S, top_k=1, eos_id=eos_id)` token for token, whichever row and
    step admit it.  With len(prompts) <= batch_size and one `max_new_tokens` no row is refilled: that is
    `generate_prompts`.  `stats`, when given, receives "steps" (sampling launches), "refills"
    (prompts admitted after the first prefill), "packed" / "alone" (prompts prefilled in a packed pass / one at a time,
    LLaMA.refill_rows) and "idle_row_steps" (row-steps whose token was dropped).  The cache is left at B rows: call
    `model.reset_cache()` before a batch-1 `generate()`.

    `adapters` (multi-LoRA, lit_llama_b200.lora.add_lora_adapter): one adapter id per prompt (-1: the base alone).
    Prompt i is prefilled and decoded with adapter i; a refilled row moves to its new prompt's adapter in the step
    its prefill runs.  On the exact batched steps prompt i then gets `generate()`'s tokens on a batch-1 model that
    carries only that adapter."""
    n = len(prompts)
    if n == 0:
        raise ValueError(f"{_who}: no prompts")
    if adapters is not None and len(adapters) != n:
        raise ValueError(f"{_who}: {len(adapters)} adapters for {n} prompts")
    if not 1 <= int(batch_size) <= MAX_SAMPLES:
        raise ValueError(f"{_who}: batch_size = {batch_size}; 1..{MAX_SAMPLES} (the batched decode step's range)")
    for p in prompts:
        if p.dim() != 1 or p.numel() == 0:
            raise ValueError(f"{_who}: every prompt must be a non-empty 1-D sequence of shape (T,), got {tuple(p.shape)}")
    for p in prompts:
        if not p.is_cuda:
            raise RuntimeError(f"{_who}: a prompt is on {p.device}; lit_llama_b200 runs on CUDA only (no CPU fallback)")
    news = [int(max_new_tokens)] * n if isinstance(max_new_tokens, int) else [int(m) for m in max_new_tokens]
    if len(news) != n or min(news) < 0:
        raise ValueError(f"{_who}: max_new_tokens must be one int >= 0, or one per prompt ({n}), got {max_new_tokens}")
    Ts = [p.numel() for p in prompts]
    S = max_seq_length
    if S is None:
        S = min(max(T + m for T, m in zip(Ts, news)), model.config.block_size)
    if max(Ts) > S:
        raise ValueError(f"{_who}: a prompt of {max(Ts)} tokens is longer than max_seq_length={S}")
    st = {} if stats is None else stats
    st.update(steps=0, refills=0, packed=0, alone=0, idle_row_steps=0)
    device, dtype = prompts[0].device, prompts[0].dtype
    queue = deque(i for i in range(n) if news[i] > 0)
    if not queue:
        return [p.clone() for p in prompts]

    def admit(ids: List[int]) -> None:
        if stats is None:   # the pack plan walks every linear per prompt: host time spent only for the caller's stats
            return
        k = len(model._pack_plan([Ts[i] for i in ids]))
        st["packed"] += k
        st["alone"] += len(ids) - k

    B = min(int(batch_size), len(queue))
    serving: List[Optional[int]] = [queue.popleft() for _ in range(B)]   # the prompt each row decodes (None: idle)
    done = [0] * n                          # new tokens prompt i has so far
    first, row_of = [0] * n, [0] * n        # the step that drew prompt i's first token, and its row
    hist = []                               # every step's (B,) tokens
    pending = []                            # (row, prompt): refilled behind the next step's model call
    input_pos = torch.tensor([Ts[i] for i in serving], dtype=torch.int64, device=device).view(B, 1)
    admit(serving)
    step = 0
    while True:
        if step == 0:
            first_rows = [prompts[i] for i in serving]
            rows = (model.prefill_rows(first_rows, S) if adapters is None
                    else model.prefill_rows(first_rows, S, [adapters[i] for i in serving]))
        else:
            rows = model(x, S, input_pos)[:, -1]
            input_pos = input_pos + 1
            if pending:   # the finished rows rode along in that call; now they take their new prompts
                ids = [i for _, i in pending]
                admit(ids)
                ridx = torch.tensor([r for r, _ in pending], device=device)
                new_rows = ([prompts[i] for i in ids], [r for r, _ in pending], S)
                rows[ridx] = (model.refill_rows(*new_rows) if adapters is None
                              else model.refill_rows(*new_rows, [adapters[i] for i in ids]))
                input_pos[ridx] = torch.tensor([Ts[i] for i in ids], dtype=torch.int64, device=device).view(-1, 1)
                st["refills"] += len(ids)
                pending = []
        idx_next = _draw(rows, temperature, top_k, dtype)
        hist.append(idx_next)
        x = idx_next.view(B, 1)
        hits = (idx_next == eos_id).tolist() if eos_id is not None else None   # the step's one host read
        for b, i in enumerate(serving):
            if i is None:
                st["idle_row_steps"] += 1
                continue
            if done[i] == 0:
                first[i], row_of[i] = step, b
            done[i] += 1
            if done[i] == news[i] or (hits is not None and hits[b]):
                serving[b] = queue.popleft() if queue else None
                if serving[b] is not None:
                    pending.append((b, serving[b]))
        step += 1
        if all(i is None for i in serving):
            break
    st["steps"] = step
    H = torch.stack(hist)
    return [torch.cat((p.to(dtype), H[first[i]:first[i] + done[i], row_of[i]])) for i, p in enumerate(prompts)]


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
    batch_size: int = 1,
    prompts_file: Optional[Path] = None,
    draft_checkpoint_path: Optional[Path] = None,
    draft_quantize: Optional[str] = None,
    num_draft: int = 4,
    stream: bool = False,
    lora_path: Optional[Sequence[Path]] = None,
    lora_alpha: float = 16,
    kv_cache: Optional[str] = None,
    lookup_ngram: int = 0,
) -> None:
    """generate.py:94-155 without Fabric: bf16 on cuda:0, same prints on stderr.  `batch_size` > 1 draws the samples
    in groups of up to `batch_size` (at most 16) through `generate_batch`, on the model's exact batched decode step.
    `prompts_file` (one prompt per line) replaces `prompt`: the prompts are decoded in groups of `batch_size` through
    `generate_prompts`, `num_samples` times each; with `stream` they go through `generate_stream` on `batch_size` rows,
    each finished row taking the next prompt.  `draft_checkpoint_path` (with `draft_quantize`) loads a draft model
    and decodes each sample with `generate_speculative`, `num_draft` draft tokens per round.  `lora_path` (one or
    more LoRA checkpoints over a quantized base) builds the model under `lora(r, lora_alpha, 0)`, r from the first
    file, loads the first as adapter 0 (generate/lora.py's way) and registers the others with `add_lora_adapter`;
    with `prompts_file` a line may then start with `<k>\t` to decode with adapter k (adapter 0 without it).
    `kv_cache` "fp8" gives the model an fp8 KV cache (LLaMA.kv_cache_dtype; not with a draft model).  `lookup_ngram`
    N > 0 decodes each sample with `generate_speculative(draft=None, max_ngram=N)`: prompt lookup proposes up to
    `num_draft` tokens per round from the sequence's own n-grams, no draft model."""
    if not 1 <= batch_size <= MAX_SAMPLES:
        raise ValueError(f"batch_size = {batch_size}; 1..{MAX_SAMPLES}")
    from sentencepiece import SentencePieceProcessor

    checkpoint_path, tokenizer_path = Path(checkpoint_path), Path(tokenizer_path)
    assert checkpoint_path.is_file(), checkpoint_path
    assert tokenizer_path.is_file(), tokenizer_path
    device = torch.device("cuda", 0)

    loras = [torch.load(p, map_location="cpu", weights_only=True) for p in lora_path or []]

    def load(path: Path, mode: Optional[str], loras=()) -> LLaMA:
        print("Loading model ...", file=sys.stderr)
        t0 = time.time()
        checkpoint = torch.load(path, map_location="cpu", weights_only=True, mmap=True)
        name = llama_model_lookup(checkpoint)
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.bfloat16)  # what Fabric's bf16-true does inside init_module
        # LoRA: r from the first adapter's lora_A (q and v enabled: 2 r rows), as generate/lora.py builds it
        r = next(v.shape[0] // 2 for k, v in loras[0].items() if k.endswith("lora_A")) if loras else 0
        try:
            with torch.device(device), quantization(mode=mode), lora_ctx(r=r, alpha=lora_alpha, dropout=0.0, enabled=bool(loras)):
                m = LLaMA.from_name(name)
        finally:
            torch.set_default_dtype(prev)
        m.load_state_dict(checkpoint, strict=not loras)
        if loras:
            m.load_state_dict(loras[0], strict=False)
            for sd in loras[1:]:
                add_lora_adapter(m, sd, alpha=lora_alpha)
        print(f"Time to load model: {time.time() - t0:.02f} seconds.", file=sys.stderr)
        m.eval()
        if mode in ("gptq.int4", "gptq.int8") and os.environ.get("B2L_COMPACT", "1") != "0":
            try:
                m.compact()   # one resident copy of the weights (the reference-layout buffers come back on state_dict())
            except RuntimeError:  # a layer the fused decode step cannot run (grouped scales, odd widths): keep everything
                pass
        return m

    from .lora import add_lora_adapter, lora as lora_ctx

    model = load(checkpoint_path, quantize, loras)
    model.kv_cache_dtype = kv_cache
    draft = None
    if draft_checkpoint_path is not None:
        assert Path(draft_checkpoint_path).is_file(), draft_checkpoint_path
        draft = load(Path(draft_checkpoint_path), draft_quantize)

    sp = SentencePieceProcessor(model_file=str(tokenizer_path))
    encoded = torch.tensor([sp.bos_id()] + sp.encode(prompt), dtype=torch.int, device=device)

    def timed(k: int, run, prompts: List[torch.Tensor]) -> None:
        """Inference number k: run() (one output per prompt) between two synchronises, then the caches reset and the
        outputs and the rate printed."""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ys = run()
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        for m in (model, draft):
            if m is not None:
                m.reset_cache()
        for y in ys:
            print(sp.decode(y.tolist()))
        tokens_generated = sum(y.size(0) - p.size(0) for y, p in zip(ys, prompts))
        print(f"Time for inference {k}: {t:.02f} sec total, {tokens_generated / t:.02f} tokens/sec", file=sys.stderr)

    torch.manual_seed(1234)
    if batch_size > 1 or prompts_file is not None:
        # the exact 2..16-row decode step of each quantized base (each row bit-identical to the batch-1 step on it);
        # without it a compacted gptq.int4 model re-tiles every linear at B >= 2 and gptq.int8 runs module by module
        if quantize == "gptq.int4":
            model.q4_batch_step = True
        elif quantize == "gptq.int8":
            model.w8_batch_step = True
        elif quantize == "llm.int8":
            model.int8_step = True
    if prompts_file is not None:
        lines = [ln for ln in Path(prompts_file).read_text().splitlines() if ln.strip()]
        adapters = None
        if loras:   # "<k>\t" in front of a line picks adapter k
            picks = [re.match(r"(-?\d+)\t(.*)", ln) for ln in lines]
            adapters = [int(m.group(1)) if m else 0 for m in picks]
            lines = [m.group(2) if m else ln for m, ln in zip(picks, lines)]
        prompts = [torch.tensor([sp.bos_id()] + sp.encode(ln), dtype=torch.int, device=device) for ln in lines]
        k = 0
        for _ in range(num_samples):
            if stream:
                k += 1
                timed(k, lambda: generate_stream(model, prompts, max_new_tokens, batch_size=batch_size,
                                                 temperature=temperature, top_k=top_k, adapters=adapters), prompts)
                continue
            for first in range(0, len(prompts), batch_size):
                group = prompts[first:first + batch_size]
                k += 1
                timed(k, lambda: generate_prompts(model, group, max_new_tokens, temperature=temperature, top_k=top_k,
                                                  adapters=None if adapters is None else adapters[first:first + batch_size]),
                      group)
    elif batch_size == 1:
        def one() -> torch.Tensor:
            if lookup_ngram > 0:
                return generate_speculative(model, None, encoded, max_new_tokens, num_draft=num_draft,
                                            max_ngram=lookup_ngram, temperature=temperature, top_k=top_k)
            if draft is None:
                return generate(model, encoded, max_new_tokens, temperature=temperature, top_k=top_k)
            return generate_speculative(model, draft, encoded, max_new_tokens, num_draft=num_draft,
                                        temperature=temperature, top_k=top_k)

        for i in range(num_samples):
            timed(i + 1, lambda: [one()], [encoded])
    else:
        for i, first in enumerate(range(0, num_samples, batch_size)):
            n = min(batch_size, num_samples - first)
            timed(i + 1, lambda: generate_batch(model, encoded, n, max_new_tokens, temperature=temperature, top_k=top_k),
                  [encoded] * n)
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
    ap.add_argument("--batch_size", type=int, default=1,
                    help=f"samples drawn together per generate_batch call (1..{MAX_SAMPLES}; 1: one generate() per sample); "
                         "with --prompts_file, prompts decoded together per generate_prompts call")
    ap.add_argument("--prompts_file", type=Path, default=None,
                    help="a text file of prompts, one per line, decoded in groups of --batch_size (replaces --prompt)")
    ap.add_argument("--stream", action="store_true",
                    help="with --prompts_file: decode the whole file through generate_stream on --batch_size rows, each "
                         "finished row taking the next prompt (continuous batching)")
    ap.add_argument("--draft_checkpoint_path", type=Path, default=None,
                    help="a smaller model's checkpoint: decode with generate_speculative, this model proposing tokens")
    ap.add_argument("--draft_quantize", default=None, choices=[None, "llm.int8", "gptq.int4", "gptq.int8"])
    ap.add_argument("--num_draft", type=int, default=4, help=f"draft tokens per speculative round (1..{MAX_DRAFT})")
    ap.add_argument("--lora_path", type=Path, action="append", default=None,
                    help="a LoRA checkpoint over a quantized base (repeatable): the first is adapter 0, the next 1, 2, ...; "
                         "a --prompts_file line starting with '<k>\\t' decodes with adapter k")
    ap.add_argument("--lora_alpha", type=float, default=16, help="LoRA alpha of every --lora_path (scaling = alpha / r)")
    ap.add_argument("--kv_cache", default=None, choices=[None, "fp8"],
                    help="fp8: e4m3 keys and values with a power-of-two scale per slot and head, half the KV cache's bytes "
                         "(default: bf16)")
    ap.add_argument("--lookup_ngram", type=int, default=0,
                    help=f"N in 1..{MAX_NGRAM}: speculative decoding without a draft model, --num_draft tokens per round "
                         "proposed by prompt lookup (the continuation of the latest earlier match of the last N..1 "
                         "tokens); 0: off")
    a = ap.parse_args()
    if a.kv_cache == "fp8" and a.draft_checkpoint_path is not None:
        ap.error("--kv_cache fp8 does not combine with --draft_checkpoint_path (the verify step keeps a bf16 cache)")
    if a.draft_checkpoint_path is not None and (a.batch_size != 1 or a.prompts_file is not None):
        ap.error("--draft_checkpoint_path decodes one sequence at a time (batch_size 1, no prompts_file)")
    if a.lookup_ngram:
        if not 1 <= a.lookup_ngram <= MAX_NGRAM:
            ap.error(f"--lookup_ngram {a.lookup_ngram}: 1..{MAX_NGRAM}, or 0 (off)")
        if a.draft_checkpoint_path is not None:
            ap.error("--lookup_ngram does not combine with --draft_checkpoint_path (lookup replaces the draft model)")
        if a.kv_cache == "fp8":
            ap.error("--kv_cache fp8 does not combine with --lookup_ngram (the verify step keeps a bf16 cache)")
        if a.batch_size != 1 or a.prompts_file is not None:
            ap.error("--lookup_ngram decodes one sequence at a time (batch_size 1, no prompts_file)")
    if a.stream and a.prompts_file is None:
        ap.error("--stream decodes a --prompts_file")
    main(**vars(a))


if __name__ == "__main__":
    cli()

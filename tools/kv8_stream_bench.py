"""Packed refill into an fp8 KV cache (b2l_attention_ragged_kv8) against one prompt at a time, and continuous batching on
the fp8 cache against bf16, on synthetic seeded weights (tools/diag.py `_random_w8_model`), compacted:

  (a) refill time: `prefill_rows` of the first 16 prompts of tools/stream_bench.py's workload (16..512 tokens) on 7B
      gptq.int4 (`q4_batch_step`) and gptq.int8 (`w8_batch_step`), in three arms: fp8 packed, fp8 one at a time (the
      pack plan emptied, as before packing on fp8 existed) and bf16 packed, in ms;
  (b) stream throughput: `generate_stream` of stream_bench's 64 prompts on 16 rows, fp8 against bf16, sampled tokens
      per second (every prefill included);
  (c) 65B gptq.int4, fp8 cache, 16 rows, max_seq_length 2048: `prefill_rows` of 16 prompts of 1536 tokens, packed
      against one at a time: time, peak allocated memory, and the passes the free-memory bound chose
      (--skip-65b leaves it out).

    python tools/kv8_stream_bench.py [--rounds 3] [--models q4,w8] [--skip-65b] [--out kv8_stream_bench.json]

The arms of each part run in one process, alternated round by round (the order rotates every round), each timed as
wall time between two torch.cuda.synchronize() calls; medians over rounds are reported.  The GPU name and power limit
are read in the same run and printed with the numbers.
"""
import argparse
import contextlib
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from samples_bench import _wall, gpu_facts  # noqa: E402
from stream_bench import ROWS, workload  # noqa: E402


@contextlib.contextmanager
def _alone(model):
    """Every prompt prefilled on its own (the pack plan emptied)."""
    model._pack_plan = lambda lengths: []
    try:
        yield
    finally:
        del model._pack_plan


def _set_format(model, fmt):
    model.reset_cache()
    model.kv_cache_dtype = fmt


def _passes(model, prompts):
    """The passes refill_rows would split the packed prompts into on the device as it is now."""
    packed = model._pack_plan([p.numel() for p in prompts])
    dev = prompts[0].device
    free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    return packed, model._packed_passes([prompts[i].numel() for i in packed], model._packed_token_bytes(), free)


def bench_model(kind: str, rounds: int) -> dict:
    import lit_llama_b200 as P
    from diag import _random_w8_model

    dev = torch.device("cuda", 0)
    model = _random_w8_model("7B", dev, seed=1234, bits=4 if kind == "q4" else 8)
    model.compact()
    if kind == "q4":
        model.q4_batch_step = True
    else:
        model.w8_batch_step = True
    lengths, news = workload()
    g = torch.Generator().manual_seed(16)
    prompts = [torch.randint(0, 32000, (t,), generator=g).to(torch.int32).to(dev) for t in lengths]
    kw = dict(temperature=0.8, top_k=200)
    useful = sum(news)
    pre, S = prompts[:ROWS], max(lengths[:ROWS])

    def refill(fmt, alone=False):
        def run():
            _set_format(model, fmt)
            with _alone(model) if alone else contextlib.nullcontext():
                model.prefill_rows(pre, S)
            torch.cuda.synchronize()
        return run

    stats = {}

    def stream(fmt):
        def run():
            _set_format(model, fmt)
            ys = P.generate_stream(model, prompts, news, batch_size=ROWS, stats=stats.setdefault(fmt or "bf16", {}), **kw)
            assert [y.numel() for y in ys] == [t + m for t, m in zip(lengths, news)]
        return run

    # (a) the three refill arms give the same logits and fp8 caches (packed = alone, bit for bit)
    out = {}
    for name, fmt, alone in (("fp8_packed", "fp8", False), ("fp8_alone", "fp8", True)):
        _set_format(model, fmt)
        with _alone(model) if alone else contextlib.nullcontext():
            lg = model.prefill_rows(pre, S)
        out[name] = (lg, model._kv_store.view(torch.uint8).clone(), model._kv_scale.clone())
    same = all(torch.equal(a, b) for a, b in zip(out["fp8_packed"], out["fp8_alone"]))
    del out
    torch.manual_seed(0)
    # warm-up: every decode state, graph and allocator size the timed rounds use
    for fmt in ("fp8", None):
        _set_format(model, fmt)
        P.generate_stream(model, prompts[:20], [4] * 20, batch_size=ROWS, **kw)
        refill(fmt)()
    refill("fp8", alone=True)()
    arms_a = [("fp8_packed", refill("fp8")), ("fp8_alone", refill("fp8", alone=True)), ("bf16_packed", refill(None))]
    arms_b = [("fp8_stream", stream("fp8")), ("bf16_stream", stream(None))]
    t = {name: [] for name, _ in arms_a + arms_b}
    for r in range(rounds):
        for arms in (arms_a, arms_b):
            k = r % len(arms)
            for name, fn in arms[k:] + arms[:k]:
                t[name].append(_wall(fn))
    med = {k: statistics.median(v) for k, v in t.items()}
    _set_format(model, "fp8")
    packed, passes = _passes(model, pre)
    model.reset_cache()
    res = dict(model=f"7B {'gptq.int4' if kind == 'q4' else 'gptq.int8'} (compacted, synthetic)",
               prefill_prompts=ROWS, prefill_tokens=sum(lengths[:ROWS]), packed_of_16=len(packed),
               passes=len(passes), fp8_packed_equals_alone=same,
               fp8_packed_ms=1e3 * med["fp8_packed"], fp8_alone_ms=1e3 * med["fp8_alone"],
               bf16_packed_ms=1e3 * med["bf16_packed"], alone_over_packed=med["fp8_alone"] / med["fp8_packed"],
               stream_prompts=len(prompts), sampled_tokens=useful,
               fp8_stream_tok_s=useful / med["fp8_stream"], bf16_stream_tok_s=useful / med["bf16_stream"],
               fp8_over_bf16_stream=med["bf16_stream"] / med["fp8_stream"], stream_stats=stats,
               runs_s={k: v for k, v in t.items()})
    del model
    torch.cuda.empty_cache()
    return res


def bench_65b() -> dict:
    from diag import _random_w8_model

    dev = torch.device("cuda", 0)
    S, T = 2048, 1536
    torch.cuda.empty_cache()
    model = _random_w8_model("65B", dev, seed=1234, bits=4)
    model.compact()
    model.q4_batch_step = True
    model.kv_cache_dtype = "fp8"
    torch.cuda.synchronize()
    weights = torch.cuda.memory_allocated()
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, 32000, (T,), generator=g).to(torch.int32).to(dev) for _ in range(ROWS)]
    res = dict(model="65B gptq.int4 (compacted, synthetic), fp8 cache", rows=ROWS, prompt_tokens=T, max_seq_length=S,
               weights_gib=weights / 2 ** 30)
    for name in ("packed", "alone"):
        model.reset_cache()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        if name == "packed":   # the plan on an allocated cache, the state refill_rows plans in
            model._new_kv_store(ROWS, S, dev)
            packed, passes = _passes(model, prompts)
            res.update(packed_of_16=len(packed), passes=[len(p) for p in passes],
                       free_gib_beside_cache=torch.cuda.mem_get_info(dev)[0] / 2 ** 30)
            model.reset_cache()
        with _alone(model) if name == "alone" else contextlib.nullcontext():
            res[f"{name}_s"] = _wall(lambda: model.prefill_rows(prompts, S))
        res[f"{name}_peak_allocated_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
        res["kv_store_gib"] = (model._kv_store.numel() + model._kv_scale.numel() * 4) / 2 ** 30
    res["alone_over_packed"] = res["alone_s"] / res["packed_s"]
    del model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", default="q4,w8")
    ap.add_argument("--skip-65b", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv8_stream_bench needs a GPU")
    facts = gpu_facts()
    print(f"GPU (name, power limit, max SM clock): {facts}", flush=True)
    results = []
    for kind in [k for k in a.models.split(",") if k]:
        res = bench_model(kind, a.rounds)
        results.append(res)
        print(f"{res['model']}: prefill_rows of {ROWS} prompts ({res['prefill_tokens']} tokens, {res['packed_of_16']} "
              f"packed, {res['passes']} pass): fp8 packed {res['fp8_packed_ms']:.1f} ms, fp8 one at a time "
              f"{res['fp8_alone_ms']:.1f} ms (x{res['alone_over_packed']:.2f}), bf16 packed {res['bf16_packed_ms']:.1f} ms;"
              f" fp8 packed == alone bit for bit: {res['fp8_packed_equals_alone']}", flush=True)
        print(f"  generate_stream, {res['stream_prompts']} prompts on {ROWS} rows, {res['sampled_tokens']} sampled "
              f"tokens: fp8 {res['fp8_stream_tok_s']:.0f} tok/s, bf16 {res['bf16_stream_tok_s']:.0f} tok/s "
              f"(x{res['fp8_over_bf16_stream']:.2f}); stats {res['stream_stats']}", flush=True)
    if not a.skip_65b:
        try:
            res = bench_65b()
        except torch.cuda.OutOfMemoryError as e:
            res = dict(error=f"out of memory: {e}")
        results.append(res)
        print(f"65B: {res}", flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(gpu=facts, results=results), f, indent=1)


if __name__ == "__main__":
    main()

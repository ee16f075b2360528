"""Continuous batching against the grouped loop, on 7B gptq.int4 (compacted, `q4_batch_step`) and 7B gptq.int8
(compacted, `w8_batch_step`) with synthetic seeded weights (tools/diag.py `_random_w8_model`).

Workload: 64 prompts with lengths spread evenly over 16..512 tokens and per-prompt new-token counts spread evenly over
32..256, both shuffled with a seed.  The counts stand in for eos, which random weights do not draw in any meaningful way.

  (a) decode: `generate_prompts` in groups of 16 in input order (what `main --prompts_file` does), each group run to
      its longest count and every prompt cut to its own, against `generate_stream` on 16 rows; sampled tokens per
      second = the sum of the counts / wall time (every prefill included);
  (b) prefill: the first 16 prompts through `prefill_rows` (one packed pass for every prompt of 17 tokens or more)
      against the per-prompt batch-1 prefill loop, in ms;
  (c) what a refill costs next to a decode step: one 16-row decode step, and `refill_rows` of one prompt of 17, 264
      and 512 tokens into a 16-row cache (median of 5 each), in ms.

    python tools/stream_bench.py [--rounds 3] [--models q4,w8] [--out stream_bench.json]

The arms of each part run in one process, alternated round by round (the order flips every round), each timed as wall
time between two torch.cuda.synchronize() calls; medians over rounds are reported.  The GPU name and power limit are
read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import random
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from samples_bench import _wall, gpu_facts  # noqa: E402

N_PROMPTS, ROWS = 64, 16


def workload(seed: int = 64):
    """(prompt lengths, new-token counts): each spread evenly over its range, shuffled independently."""
    rng = random.Random(seed)
    lengths = [16 + (512 - 16) * i // (N_PROMPTS - 1) for i in range(N_PROMPTS)]
    news = [32 + (256 - 32) * i // (N_PROMPTS - 1) for i in range(N_PROMPTS)]
    rng.shuffle(lengths)
    rng.shuffle(news)
    return lengths, news


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

    def grouped():
        out = []
        for first in range(0, N_PROMPTS, ROWS):
            group, counts = prompts[first:first + ROWS], news[first:first + ROWS]
            ys = P.generate_prompts(model, group, max(counts), **kw)
            out += [y[:p.numel() + m] for y, p, m in zip(ys, group, counts)]
            model.reset_cache()
        assert [y.numel() for y in out] == [t + m for t, m in zip(lengths, news)]

    stats = {}

    def stream():
        ys = P.generate_stream(model, prompts, news, batch_size=ROWS, stats=stats, **kw)
        model.reset_cache()
        assert [y.numel() for y in ys] == [t + m for t, m in zip(lengths, news)]

    pre = prompts[:ROWS]
    S = max(lengths[:ROWS])

    def packed():
        model.prefill_rows(pre, S)
        model.reset_cache()

    def alone():
        for p in pre:
            model(p.view(1, -1), S, torch.arange(p.numel(), device=dev))
            model.reset_cache()

    torch.manual_seed(0)
    # warm-up: every decode state, graph and allocator size the timed rounds use
    P.generate_stream(model, prompts[:20], [4] * 20, batch_size=ROWS, **kw)
    model.reset_cache()
    P.generate_prompts(model, prompts[:ROWS], 4, **kw)
    model.reset_cache()
    packed()
    alone()
    t = {"grouped": [], "stream": [], "packed": [], "alone": []}
    for r in range(rounds):
        for name, fn in ((("grouped", grouped), ("stream", stream)) if r % 2 == 0 else (("stream", stream), ("grouped", grouped))):
            t[name].append(_wall(fn))
        for name, fn in ((("packed", packed), ("alone", alone)) if r % 2 == 0 else (("alone", alone), ("packed", packed))):
            t[name].append(_wall(fn))
    med = {k: statistics.median(v) for k, v in t.items()}
    # (c) one decode step and one single-prompt refill on a 16-row cache at the stream's S
    S_all = max(a + b for a, b in zip(lengths, news))
    model.prefill_rows(pre, S_all)
    pos = torch.tensor(lengths[:ROWS], device=dev).view(ROWS, 1)
    x = torch.zeros((ROWS, 1), dtype=torch.int32, device=dev)
    step_s = []
    for i in range(25):
        step_s.append(_wall(lambda: model(x, S_all, pos + i)))
    one = {}
    for n in (17, 264, 512):
        p = torch.randint(0, 32000, (n,), generator=g).to(torch.int32).to(dev)
        one[n] = 1e3 * statistics.median(_wall(lambda: model.refill_rows([p], [0], S_all)) for _ in range(5))
    model.reset_cache()
    res = dict(model=f"7B {'gptq.int4' if kind == 'q4' else 'gptq.int8'} (compacted, synthetic)", prompts=N_PROMPTS,
               rows=ROWS, sampled_tokens=useful, prefill_prompts=ROWS, prefill_tokens=sum(lengths[:ROWS]),
               packed_of_16=len(model._pack_plan(lengths[:ROWS])),
               grouped_tok_s=useful / med["grouped"], stream_tok_s=useful / med["stream"],
               stream_over_grouped=med["grouped"] / med["stream"], grouped_s=t["grouped"], stream_s=t["stream"],
               stream_stats=dict(stats),
               packed_ms=1e3 * med["packed"], alone_ms=1e3 * med["alone"], alone_over_packed=med["alone"] / med["packed"],
               packed_runs_ms=[1e3 * x for x in t["packed"]], alone_runs_ms=[1e3 * x for x in t["alone"]],
               step_ms=1e3 * statistics.median(step_s[5:]), refill_one_ms=one)
    del model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--models", default="q4,w8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench needs a GPU")
    facts = gpu_facts()
    print(f"GPU (name, power limit, max SM clock): {facts}", flush=True)
    results = []
    for kind in a.models.split(","):
        res = bench_model(kind, a.rounds)
        results.append(res)
        print(f"{res['model']}: {N_PROMPTS} prompts on {ROWS} rows, {res['sampled_tokens']} sampled tokens: grouped "
              f"{res['grouped_tok_s']:.0f} tok/s, stream {res['stream_tok_s']:.0f} tok/s "
              f"(x{res['stream_over_grouped']:.2f}); stream stats {res['stream_stats']}", flush=True)
        print(f"  prefill of {ROWS} prompts ({res['prefill_tokens']} tokens, {res['packed_of_16']} packed): packed "
              f"{res['packed_ms']:.1f} ms, one at a time {res['alone_ms']:.1f} ms (x{res['alone_over_packed']:.2f})",
              flush=True)
        print(f"  one 16-row decode step {res['step_ms']:.2f} ms; refill of one prompt: "
              + ", ".join(f"{n} tokens {ms:.1f} ms" for n, ms in res["refill_one_ms"].items()), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(gpu=facts, results=results), f, indent=1)


if __name__ == "__main__":
    main()

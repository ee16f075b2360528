"""Speculative decoding on one GPU: what a verify step costs and what a round costs, on synthetic gptq.int4 weights.

1. `LLaMA.decode_tokens` at T = 2..16 against the batch-1 step, at positions ~64 / ~1024 / ~2000, for each model
   (CUDA events around 20 replays of each CUDA graph after warm-up; the median of 5 repetitions).
2. End-to-end tokens/s of `generate_speculative(top_k=1)` against `generate(top_k=1)`, run alternately, medians:
   draft = the smallest model's own weights (every draft token accepted: the upper bound) and the smallest model
   drafting for the largest.

Acceptance on random weights says nothing about real checkpoints, so the script reports per-round costs and the
expected speedup formula of speculative sampling, (1 - a^(k+1)) / (1 - a) * t_target / (k t_draft + t_verify) for an
acceptance rate a, evaluated at a few a; the card name and power limit are read in the same run and printed with the
numbers.  Prints one JSON object.

  python tools/spec_bench.py [--models 7B,65B] [--new 128] [--reps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timed(fn, n=20, reps=5):
    """Median over `reps` of the mean ms of n calls of fn, CUDA events around them."""
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / n)
    return statistics.median(out)


def step_costs(model, dev, positions, Ts, S=2048):
    """{pos: {"T=1": ms of the batch-1 step, "T=t": ms of decode_tokens at t}}: the cache filled to `pos` first."""
    V = model.config.vocab_size
    res = {}
    for pos in positions:
        model.reset_cache()
        model(torch.randint(0, V, (1, pos), device=dev), S, torch.arange(pos, device=dev))
        tok = torch.randint(0, V, (1, 1), device=dev)
        p1 = torch.tensor([pos], device=dev)
        r = {"T=1": timed(lambda: model(tok, S, p1))}
        for T in Ts:
            idx = torch.randint(0, V, (1, T), device=dev)
            pp = torch.arange(pos, pos + T, device=dev)
            r[f"T={T}"] = timed(lambda: model.decode_tokens(idx, S, pp))
        res[pos] = r
    model.reset_cache()
    return res


def e2e(P, target, draft, dev, n_new, reps, k):
    """Alternated runs of generate and generate_speculative (top_k = 1): median tokens/s of each, the rounds'
    acceptance, and whether the two outputs agree (random weights can tie for the top logit; top_k = 1 keeps every
    tied token and the draw between them depends on the RNG stream, which the two drivers consume differently)."""
    V = target.config.vocab_size
    prompt = torch.randint(0, V, (32,), generator=torch.Generator().manual_seed(0)).to(dev)
    plain, spec, acc = [], [], None
    for r in range(reps + 1):   # the first pair warms up
        for which in ("plain", "spec"):
            target.reset_cache()
            draft.reset_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stats = {}
            if which == "plain":
                y = P.generate(target, prompt, n_new, top_k=1)
            else:
                y2 = P.generate_speculative(target, draft, prompt, n_new, num_draft=k, top_k=1, stats=stats)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if r > 0:
                (plain if which == "plain" else spec).append(n_new / dt)
            if which == "spec":
                acc = stats
    target.reset_cache()
    draft.reset_cache()
    return dict(generate_tok_s=statistics.median(plain), speculative_tok_s=statistics.median(spec), rounds=acc["rounds"],
                mean_accepted=sum(acc["accepted"]) / max(1, acc["rounds"]), num_draft=k,
                tokens_equal=bool(torch.equal(y, y2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="7B,65B")
    ap.add_argument("--positions", default="64,1024,2000")
    ap.add_argument("--Ts", default="2,3,4,5,8,12,16")
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--num_draft", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_bench: needs a GPU (no CPU timing is meaningful)")
    import __graft_entry__ as entry

    entry.build()
    import lit_llama_b200 as P
    from diag import _random_w8_model

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    out = dict(card=card(), costs={}, e2e={})
    names = a.models.split(",")
    Ts = [int(t) for t in a.Ts.split(",")]
    models = {}
    for i, name in enumerate(names):
        models[name] = _random_w8_model(name, dev, seed=10 + i, bits=4).compact()
        out["costs"][name] = step_costs(models[name], dev, [int(p) for p in a.positions.split(",")], Ts)
        print(json.dumps({name: out["costs"][name]}), file=sys.stderr, flush=True)
    k = a.num_draft
    # draft = the target's own weights (acceptance 1): the smallest model, whose two copies fit beside the largest
    twin = _random_w8_model(names[0], dev, seed=10, bits=4).compact()
    out["e2e"][f"{names[0]} <- {names[0]} (same weights)"] = e2e(P, models[names[0]], twin, dev, a.new, a.reps, k)
    del twin
    torch.cuda.empty_cache()
    if len(names) > 1:
        out["e2e"][f"{names[-1]} <- {names[0]}"] = e2e(P, models[names[-1]], models[names[0]], dev, a.new, a.reps, k)
    # the expected speedup formula at position ~1024 for the last pair, from the measured per-step costs
    tgt, drf = out["costs"][names[-1]][1024], out["costs"][names[0]][1024]
    t_t, t_d, t_v = tgt["T=1"], drf["T=1"], tgt.get(f"T={k + 1}")
    if t_v is not None:
        out["expected_speedup_at_1024"] = {
            f"a={al}": round((1 - al ** (k + 1)) / (1 - al) * t_t / (k * t_d + t_v), 3) for al in (0.5, 0.7, 0.8, 0.9)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

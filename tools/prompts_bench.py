"""N different prompts: N sequential generate() calls against one generate_prompts(N), on 7B gptq.int4 (compacted,
`q4_batch_step`) and 7B gptq.int8 (compacted, `w8_batch_step`) with synthetic seeded weights (tools/diag.py
`_random_w8_model`).  Prompt lengths spread evenly over 16..512 tokens, 256 new tokens per prompt, N in {1, 2, 4, 8, 16}.

    python tools/prompts_bench.py [--rounds 3] [--new 256] [--models q4,w8] [--out prompts_bench.json]

Both arms run in one process, alternated round by round (the order flips every round), each timed as wall time between
two torch.cuda.synchronize() calls around the whole work (every prefill included).  Reported: sampled tokens per second
(N x new tokens / time, median over rounds) and generate_prompts / sequential.  The GPU name and power limit are read in
the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from samples_bench import _wall, gpu_facts  # noqa: E402


def lengths(n: int):
    """n prompt lengths spread evenly over 16..512."""
    return [16] if n == 1 else [16 + (512 - 16) * i // (n - 1) for i in range(n)]


def bench_model(kind: str, rounds: int, new: int, ns) -> dict:
    import lit_llama_b200 as P
    from diag import _random_w8_model

    dev = torch.device("cuda", 0)
    model = _random_w8_model("7B", dev, seed=1234, bits=4 if kind == "q4" else 8)
    model.compact()
    if kind == "q4":
        model.q4_batch_step = True
    else:
        model.w8_batch_step = True
    g = torch.Generator().manual_seed(16)
    prompts = {n: [torch.randint(0, 32000, (t,), generator=g).to(torch.int32).to(dev) for t in lengths(n)] for n in ns}
    kw = dict(temperature=0.8, top_k=200)

    def seq(n):
        for p in prompts[n]:
            P.generate(model, p, new, **kw)
            model.reset_cache()

    def batch(n):
        ys = P.generate_prompts(model, prompts[n], new, **kw)
        model.reset_cache()
        assert len(ys) == n and all(y.numel() == p.numel() + new for y, p in zip(ys, prompts[n]))

    torch.manual_seed(0)
    for n in ns:   # warm-up: decode states, graphs, allocator
        seq(1)
        batch(n)
    times = {n: {"seq": [], "batch": []} for n in ns}
    for r in range(rounds):
        for n in ns:
            arms = [("seq", seq), ("batch", batch)]
            for name, fn in (arms if r % 2 == 0 else arms[::-1]):
                times[n][name].append(_wall(lambda: fn(n)))
    out = {}
    for n in ns:
        ts, tb = statistics.median(times[n]["seq"]), statistics.median(times[n]["batch"])
        out[n] = dict(lengths=lengths(n), seq_s=ts, batch_s=tb, seq_tok_s=n * new / ts, batch_tok_s=n * new / tb,
                      ratio=ts / tb, seq_all=times[n]["seq"], batch_all=times[n]["batch"])
        print(f"7B gptq.{'int4' if kind == 'q4' else 'int8'} N={n:2d}: sequential {ts:6.2f} s = {n * new / ts:7.1f} tok/s | "
              f"generate_prompts {tb:6.2f} s = {n * new / tb:7.1f} tok/s | x{ts / tb:.2f} "
              f"(seq {', '.join(f'{t:.2f}' for t in times[n]['seq'])}; batch {', '.join(f'{t:.2f}' for t in times[n]['batch'])})",
              flush=True)
    del model
    torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--models", default="q4,w8")
    ap.add_argument("--ns", default="1,2,4,8,16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prompts_bench needs a CUDA device")
    card = gpu_facts()
    print(f"card: {card}", flush=True)
    ns = [int(n) for n in args.ns.split(",")]
    result = dict(card=card, new=args.new, rounds=args.rounds)
    for kind in args.models.split(","):
        result[kind] = bench_model(kind, args.rounds, args.new, ns)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

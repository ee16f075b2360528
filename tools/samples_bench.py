"""N samples of one prompt: N sequential generate() calls against one generate_batch(N), on 7B gptq.int4 (compacted,
`q4_batch_step`) and 7B gptq.int8 (compacted, `w8_batch_step`) with synthetic seeded weights (tools/diag.py
`_random_w8_model`).  A 16-token prompt, 256 new tokens per sample, N in {1, 2, 4, 8, 16}.

    python tools/samples_bench.py [--rounds 3] [--new 256] [--models q4,w8] [--out samples_bench.json]

Both arms run in one process, alternated round by round (the order flips every round), each timed as wall time between
two torch.cuda.synchronize() calls around the whole call (prefill included).  Reported: sampled tokens per second
(N x new tokens / time, median over rounds) and batch / sequential.  Then the sampling launch alone at B = 16, V = 32000
(top_k 200, temperature 0.8): one b2l_topk_softmax_sample_rows launch against 16 b2l_topk_softmax_sample launches, and
sample_token on (16, V) against 16 sample_token calls on (V,) (the Exp(1) draw included), CUDA events over many
repetitions.  The GPU name and power limit are read in the same run and printed with the numbers.
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


def gpu_facts() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _wall(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


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
    prompt = torch.randint(0, 32000, (16,), generator=torch.Generator().manual_seed(16)).to(torch.int32).to(dev)
    kw = dict(temperature=0.8, top_k=200)

    def seq(n):
        for _ in range(n):
            P.generate(model, prompt, new, **kw)
            model.reset_cache()

    def batch(n):
        ys = P.generate_batch(model, prompt, n, new, **kw)
        model.reset_cache()
        assert len(ys) == n and all(y.numel() == 16 + new for y in ys)

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
        out[n] = dict(seq_s=ts, batch_s=tb, seq_tok_s=n * new / ts, batch_tok_s=n * new / tb, ratio=ts / tb,
                      seq_all=times[n]["seq"], batch_all=times[n]["batch"])
        print(f"7B gptq.{'int4' if kind == 'q4' else 'int8'} N={n:2d}: sequential {ts:6.2f} s = {n * new / ts:7.1f} tok/s | "
              f"generate_batch {tb:6.2f} s = {n * new / tb:7.1f} tok/s | x{ts / tb:.2f} "
              f"(seq {', '.join(f'{t:.2f}' for t in times[n]['seq'])}; batch {', '.join(f'{t:.2f}' for t in times[n]['batch'])})",
              flush=True)
    del model
    torch.cuda.empty_cache()
    return out


def _events(fn, reps: int) -> float:
    """Mean GPU time of one fn() in us, CUDA events around `reps` calls."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def bench_sampling(reps: int = 300, rounds: int = 3) -> dict:
    import lit_llama_b200 as P
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda", 0)
    B, V, k, temp = 16, 32000, 200, 0.8
    logits = (torch.randn(B, V, device=dev) * 3).bfloat16()
    q = torch.empty((B, V), dtype=torch.bfloat16, device=dev).exponential_(1)
    tok = torch.empty(B, dtype=torch.int64, device=dev)
    lib, s = L.lib(), L.stream_ptr()

    def rows():
        lib.b2l_topk_softmax_sample_rows(logits.data_ptr(), V, temp, k, q.data_ptr(), None, tok.data_ptr(), B, V, s)

    def singles():
        for b in range(B):
            lib.b2l_topk_softmax_sample(logits[b].data_ptr(), temp, k, q[b].data_ptr(), None, tok[b:].data_ptr(), V, s)

    res = {"rows_us": [], "singles_us": [], "sample_token_rows_us": [], "sample_token_singles_us": []}
    for _ in range(rounds):
        res["rows_us"].append(_events(rows, reps))
        res["singles_us"].append(_events(singles, reps // 4))
        res["sample_token_rows_us"].append(_events(lambda: P.sample_token(logits, temp, k), reps))
        res["sample_token_singles_us"].append(_events(lambda: [P.sample_token(logits[b], temp, k) for b in range(B)], reps // 4))
    med = {key: statistics.median(v) for key, v in res.items()}
    print(f"sampling at B = 16, V = 32000, top_k 200: one rows launch {med['rows_us']:.1f} us | 16 single-row launches "
          f"{med['singles_us']:.1f} us | sample_token (16, V) {med['sample_token_rows_us']:.1f} us | 16 x sample_token (V,) "
          f"{med['sample_token_singles_us']:.1f} us  (rounds: {res})", flush=True)
    return dict(median=med, all=res)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--models", default="q4,w8")
    ap.add_argument("--ns", default="1,2,4,8,16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("samples_bench needs a CUDA device")
    card = gpu_facts()
    print(f"card: {card}", flush=True)
    ns = [int(n) for n in args.ns.split(",")]
    result = dict(card=card, prompt=16, new=args.new, rounds=args.rounds, sampling=bench_sampling())
    for kind in args.models.split(","):
        result[kind] = bench_model(kind, args.rounds, args.new, ns)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

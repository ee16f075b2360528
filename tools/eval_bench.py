"""Perplexity evaluation on 7B gptq.int4 (bench.py's synthetic weights), 2048-token windows:
lit_llama_b200.evaluate.window_nll (the loss in lm_head's GEMM epilogue) against what the reference's evaluate scripts
run on this path, `model(inp)` followed by torch's cross_entropy(logits[:-1], inp[1:], reduction="sum").

    python tools/eval_bench.py [--windows 8] [--rounds 4] [--compact] [--out eval_bench.json]

Both arms run in one process on the same windows, alternated round by round, timed with CUDA events around all the
windows of a round.  Peak memory is torch.cuda.max_memory_allocated() above what the model holds, per arm.  The GPU
name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_facts() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--block", type=int, default=2048)
    ap.add_argument("--compact", action="store_true", help="one resident weight copy (LLaMA.compact())")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")

    import bench
    import lit_llama_b200.evaluate as E

    dev = torch.device("cuda", 0)
    model = bench.build_synthetic_model("7B", dev, seed=1234)
    if args.compact:
        model.compact()
    g = torch.Generator(device=dev).manual_seed(7)
    wins = [torch.randint(0, 32000, (1, args.block), generator=g, device=dev) for _ in range(args.windows)]

    def ours():
        tot = torch.zeros((), dtype=torch.float64, device=dev)
        for w in wins:
            tot += E.window_nll(model, w)[1]
        return tot

    def torch_loop():
        tot = torch.zeros((), dtype=torch.float64, device=dev)
        with torch.inference_mode():
            for w in wins:
                logits = model(w)[0]
                tot += F.cross_entropy(logits[:-1], w[0, 1:].long(), reduction="sum")   # bf16 scalar, like the scripts
        return tot

    arms = {"window_nll": ours, "model+cross_entropy": torch_loop}
    sums = {k: float(f()) for k, f in arms.items()}   # warm-up: every shape and torch's kernel choices
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    times = {k: [] for k in arms}
    peaks = {k: 0 for k in arms}
    for r in range(args.rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(list(arms)))
        for k in order:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arms[k]()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / len(wins))
            peaks[k] = max(peaks[k], torch.cuda.max_memory_allocated() - base)
    # the same windows' exact loss in fp32 on model(inp)'s logits, for the numerics column
    with torch.inference_mode():
        exact = sum(float(F.cross_entropy(model(w)[0, :-1].float(), w[0, 1:], reduction="sum").double()) for w in wins)
    res = {
        "gpu": gpu_facts(), "model": "7B gptq.int4 synthetic", "compact": args.compact, "windows": args.windows,
        "window_tokens": args.block, "rounds": args.rounds,
        "ms_per_window": {k: {"min": min(v), "median": sorted(v)[len(v) // 2], "all": [round(t, 3) for t in v]}
                          for k, v in times.items()},
        "peak_extra_bytes": peaks,
        "nll_sum": sums, "nll_sum_fp32_torch": exact,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

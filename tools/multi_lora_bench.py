"""Multi-LoRA serving on 7B gptq.int4 (compacted, `q4_batch_step`, B = 16, r = 8) with synthetic seeded weights
(tools/diag.py `_random_w8_model`, LoRA terms from oracle/lora_oracle.py `lora_weights`).

  (a) ms per 16-row decode step with no LoRA, (b) with one adapter on every row (`b2l_decode_args::loras`) and (c)
      with 16 distinct adapters, one per row (`lora_sets`), at positions 128 and 1024: CUDA events around 20 graph
      replays, the three arms alternated round by round (order rotating), medians over rounds;
  the bytes (c) adds per step: 16 adapters' lora_A + lora_B;
  generate_stream sampled tokens per second over 64 prompts spread across 16 adapters (one call with adapters=),
      against serving the same prompts adapter by adapter (load that adapter's lora_A / lora_B, one generate_stream
      per adapter), wall time between two synchronisations, alternated;
  resident GiB (torch.cuda.memory_allocated) of the model with 1 and with 16 adapters.

    python tools/multi_lora_bench.py [--rounds 3] [--out multi_lora_bench.json]

The GPU name and power limit are read in the same run and printed with the numbers.
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

ROWS, R, N_PROMPTS = 16, 8, 64


def _models(dev):
    """(plain model, LoRA model, bytes the LoRA model holds): the same base weights, both compacted."""
    import lit_llama_b200.lora as PL
    from diag import _random_w8_model

    plain = _random_w8_model("7B", dev, seed=1234, bits=4)
    plain.compact()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with PL.lora(r=R, alpha=16, dropout=0.0):
        lora = _random_w8_model("7B", dev, seed=1234, bits=4)
    lora.compact()
    torch.cuda.synchronize()
    for m in (plain, lora):
        m.q4_batch_step = True
    return plain, lora, before


def _adapter(k: int):
    from oracle import lora_oracle as LO

    return LO.lora_weights(32, 4096, r=R, seed=500 + k)


def _step_ms(model, adapters, pos: int, S: int, dev) -> callable:
    """A timer of 20 decode steps of `model` at position `pos` on 16 rows (adapters: None or one id per row)."""
    g = torch.Generator().manual_seed(pos)
    prompts = [torch.randint(0, 32000, (8,), generator=g).to(torch.int32).to(dev) for _ in range(ROWS)]
    model.reset_cache()
    model.prefill_rows(prompts, S, adapters)
    p = torch.full((ROWS, 1), pos, device=dev)
    x = torch.zeros((ROWS, 1), dtype=torch.int32, device=dev)
    for _ in range(4):   # eager steps, then the graph capture
        model(x, S, p)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run() -> float:
        e0.record()
        for _ in range(20):
            model(x, S, p)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / 20

    return run


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_lora_bench needs a GPU")
    import lit_llama_b200 as P
    import lit_llama_b200.lora as PL

    facts = gpu_facts()
    print(f"GPU (name, power limit, max SM clock): {facts}", flush=True)
    dev = torch.device("cuda", 0)
    plain, model, before = _models(dev)
    model.load_state_dict(_adapter(0), strict=False)
    torch.cuda.synchronize()
    mem1 = torch.cuda.memory_allocated()
    sds = [_adapter(k) for k in range(ROWS)]
    for k in range(1, ROWS):
        PL.add_lora_adapter(model, sds[k])
    torch.cuda.synchronize()
    mem16 = torch.cuda.memory_allocated()
    adapter_bytes = sum(v.numel() * 2 for v in sds[0].values())
    # the LoRA model's own bytes: what was allocated after the plain model was built (no KV cache yet)
    res = dict(gpu=facts, model="7B gptq.int4 (compacted, synthetic)", rows=ROWS, r=R,
               adapter_bytes=adapter_bytes, added_bytes_per_step_c=ROWS * adapter_bytes,
               resident_gib_1_adapter=(mem1 - before) / 2 ** 30, resident_gib_16_adapters=(mem16 - before) / 2 ** 30)

    steps = {}
    for pos in (128, 1024):
        S = pos + 64
        arms = {"a_no_lora": (plain, None), "b_one_adapter": (model, None), "c_16_adapters": (model, list(range(ROWS)))}
        t = {k: [] for k in arms}
        names = list(arms)
        for r in range(a.rounds):   # each timing builds its arm's cache, step state and graph first
            for name in names[r % 3:] + names[:r % 3]:
                m, ads = arms[name]
                t[name].append(_step_ms(m, ads, pos, S, dev)())
        steps[pos] = {k: statistics.median(v) for k, v in t.items()}
        steps[pos]["runs"] = t
        print(f"pos {pos}: " + ", ".join(f"{k} {v:.3f} ms" for k, v in steps[pos].items() if k != "runs"), flush=True)
    res["step_ms"] = steps
    plain.reset_cache()
    model.reset_cache()

    g = torch.Generator().manual_seed(64)
    lengths = [16 + (128 - 16) * i // (N_PROMPTS - 1) for i in range(N_PROMPTS)]
    news = [32 + 32 * (i % 3) for i in range(N_PROMPTS)]
    prompts = [torch.randint(0, 32000, (n,), generator=g).to(torch.int32).to(dev) for n in lengths]
    ads = [i % ROWS for i in range(N_PROMPTS)]
    kw = dict(temperature=0.8, top_k=200, batch_size=ROWS)

    def multi():
        P.generate_stream(model, prompts, news, adapters=ads, **kw)
        model.reset_cache()

    def by_adapter():   # adapter k's weights loaded as adapter 0, then its prompts
        for k in range(ROWS):
            idx = [i for i in range(N_PROMPTS) if ads[i] == k]
            model.load_state_dict(sds[k], strict=False)
            P.generate_stream(model, [prompts[i] for i in idx], [news[i] for i in idx], **kw)
            model.reset_cache()

    torch.manual_seed(0)
    multi()
    by_adapter()
    t = {"multi": [], "by_adapter": []}
    for r in range(a.rounds):
        for name, fn in ((("multi", multi), ("by_adapter", by_adapter)) if r % 2 == 0 else
                         (("by_adapter", by_adapter), ("multi", multi))):
            t[name].append(_wall(fn))
    model.load_state_dict(sds[0], strict=False)
    useful = sum(news)
    res.update(stream_sampled_tokens=useful, multi_tok_s=useful / statistics.median(t["multi"]),
               by_adapter_tok_s=useful / statistics.median(t["by_adapter"]), stream_runs_s=t)
    print(f"generate_stream, {N_PROMPTS} prompts over {ROWS} adapters, {useful} sampled tokens: one call "
          f"{res['multi_tok_s']:.0f} tok/s, adapter by adapter {res['by_adapter_tok_s']:.0f} tok/s", flush=True)
    print(f"resident: {res['resident_gib_1_adapter']:.3f} GiB with 1 adapter, {res['resident_gib_16_adapters']:.3f} GiB "
          f"with 16; (c) streams {res['added_bytes_per_step_c'] / 2 ** 20:.1f} MiB of adapters per step", flush=True)
    print(json.dumps(res, default=str))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()

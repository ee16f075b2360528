"""fp8 KV cache (LLaMA.kv_cache_dtype = "fp8") against the bf16 cache, on synthetic seeded weights
(tools/diag.py `_random_w8_model`):

  (a) ms per decode step of 7B gptq.int4 (compacted, `q4_batch_step`) at B in {1, 8, 16} rows and positions
      {256, 1024, 2047} (max_seq_length 2048): CUDA events around 20 graph replays, the bf16 and fp8 arms alternated
      round by round (order rotating), medians over rounds;
  (b) the attention kernel's share of that step: one layer's attention launch (b2l_attention / b2l_attention_kv8 on a
      [B, 32, 2048, 128] cache, the step's shape) timed alone with CUDA events over 50 launches, times 32 layers, over
      the step time of (a);
  (c) the peak allocated memory of compacted 65B gptq.int4 decoding 16 rows at max_seq_length 2048 with the fp8 cache
      (prefill_rows of 16 prompts, then 4 steps at position 2047), where the model fits (--skip-65b leaves it out).

    python tools/kv8_bench.py [--rounds 3] [--skip-65b] [--out kv8_bench.json]

The GPU name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from samples_bench import gpu_facts  # noqa: E402

S = 2048
ROWS = (1, 8, 16)
POSITIONS = (256, 1024, 2047)


def _step_timer(model, B: int, pos: int, dev):
    """A timer of 20 decode steps of `model` at position `pos` on B rows (fresh cache in the model's format)."""
    g = torch.Generator().manual_seed(pos + B)
    prompts = [torch.randint(0, 32000, (8,), generator=g).to(torch.int32).to(dev) for _ in range(B)]
    model.reset_cache()
    model.prefill_rows(prompts, S)
    p = torch.full((B, 1), pos, device=dev)
    x = torch.zeros((B, 1), dtype=torch.int32, device=dev)
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


def _attention_ms(fp8: bool, B: int, pos: int, dev, nh: int = 32, hs: int = 128) -> float:
    """One layer's decode attention launch at the step's shape, alone: ms per launch over 50 launches."""
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.model import build_rope_cache

    lib = L.lib()
    g = torch.Generator(device=dev).manual_seed(7)
    qkv = torch.randn((B, 1, 3 * nh * hs), device=dev, generator=g).bfloat16()
    rope = build_rope_cache(S, hs, torch.float32, dev).float().contiguous()
    posv = torch.full((B,), pos, dtype=torch.int64, device=dev)
    ring = torch.zeros(B, dtype=torch.int32, device=dev)
    y = torch.empty((B, 1, nh * hs), device=dev, dtype=torch.bfloat16)
    work = torch.zeros(lib.b2l_attn_workspace_bytes(B, nh, hs, 1, S) // 4 + 1, device=dev, dtype=torch.float32)
    flags = L.F_ROW_POS
    if fp8:
        k = (torch.randn((B, nh, S, hs), device=dev, generator=g) * 64).to(torch.float8_e4m3fn)
        v = (torch.randn((B, nh, S, hs), device=dev, generator=g) * 64).to(torch.float8_e4m3fn)
        ks = torch.full((B, nh, S), 2.0 ** -6, device=dev)
        vs = ks.clone()
        kv = L.KV8Cache(k.data_ptr(), v.data_ptr(), ks.data_ptr(), vs.data_ptr())

        def launch():
            return lib.b2l_attention_kv8(qkv.data_ptr(), C.byref(kv), rope.data_ptr(), posv.data_ptr(), ring.data_ptr(),
                                         y.data_ptr(), work.data_ptr(), B, 1, nh, hs, S, S, flags, None, L.stream_ptr())
    else:
        k = torch.randn((B, nh, S, hs), device=dev, generator=g).bfloat16()
        v = torch.randn((B, nh, S, hs), device=dev, generator=g).bfloat16()

        def launch():
            return lib.b2l_attention(qkv.data_ptr(), k.data_ptr(), v.data_ptr(), rope.data_ptr(), posv.data_ptr(),
                                     ring.data_ptr(), y.data_ptr(), work.data_ptr(), B, 1, nh, hs, S, S, flags,
                                     L.stream_ptr())
    for _ in range(5):
        L.check(launch(), "attention")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        launch()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 50


def _peak_65b(dev) -> dict:
    from diag import _random_w8_model

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = _random_w8_model("65B", dev, seed=1234, bits=4)
    model.compact()
    model.q4_batch_step = True
    model.kv_cache_dtype = "fp8"
    torch.cuda.synchronize()
    weights = torch.cuda.memory_allocated()
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, 32000, (16,), generator=g).to(torch.int32).to(dev) for _ in range(16)]
    model.prefill_rows(prompts, S)
    p = torch.full((16, 1), S - 1, device=dev)
    x = torch.zeros((16, 1), dtype=torch.int32, device=dev)
    for _ in range(4):
        model(x, S, p)
    torch.cuda.synchronize()
    out = dict(weights_gib=weights / 2 ** 30, kv_store_gib=(model._kv_store.numel() + model._kv_scale.numel() * 4) / 2 ** 30,
               peak_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
    del model
    torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-65b", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv8_bench needs a GPU")
    from diag import _random_w8_model

    facts = gpu_facts()
    print(f"GPU (name, power limit, max SM clock): {facts}", flush=True)
    dev = torch.device("cuda", 0)
    model = _random_w8_model("7B", dev, seed=1234, bits=4)
    model.compact()
    model.q4_batch_step = True
    res = dict(gpu=facts, model="7B gptq.int4 (compacted, synthetic), q4_batch_step", max_seq_length=S, steps={})
    for B in ROWS:
        for pos in POSITIONS:
            t = {"bf16": [], "fp8": []}
            names = list(t)
            for r in range(a.rounds):   # each timing builds its arm's cache, step state and graph first
                for name in names[r % 2:] + names[:r % 2]:
                    model.reset_cache()
                    model.kv_cache_dtype = "fp8" if name == "fp8" else None
                    t[name].append(_step_timer(model, B, pos, dev)())
            model.reset_cache()
            model.kv_cache_dtype = None
            att = {k: 32 * _attention_ms(k == "fp8", B, pos, dev) for k in names}
            row = {k: statistics.median(v) for k, v in t.items()}
            row.update({f"attn_{k}_ms": att[k] for k in names})
            row.update({f"attn_share_{k}": att[k] / row[k] for k in names})
            row["fp8_over_bf16"] = row["fp8"] / row["bf16"]
            row["runs"] = t
            res["steps"][f"B{B}_pos{pos}"] = row
            print(f"B={B:2d} pos={pos:4d}: step bf16 {row['bf16']:.3f} ms, fp8 {row['fp8']:.3f} ms "
                  f"(x{row['fp8_over_bf16']:.3f}); attention 32 layers bf16 {att['bf16']:.3f} ms "
                  f"({row['attn_share_bf16']:.0%}), fp8 {att['fp8']:.3f} ms ({row['attn_share_fp8']:.0%})", flush=True)
    del model
    if not a.skip_65b:
        try:
            res["65B_16rows_fp8"] = _peak_65b(dev)
        except torch.cuda.OutOfMemoryError as e:   # reported, not hidden: the model does not fit this device
            res["65B_16rows_fp8"] = dict(error=f"out of memory: {e}")
        print(f"65B gptq.int4 compacted, 16 rows x {S}, fp8 cache: {res['65B_16rows_fp8']}", flush=True)
    print(json.dumps({k: v for k, v in res.items() if k != "steps"}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

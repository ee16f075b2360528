"""The prefill GEMM on the resident batch-1 tilings (B2L_F_GEMM_I8) against its own sources, and what a refill of a
compacted model costs next to the same model uncompacted.  Synthetic seeded weights (tools/diag.py `_random_w8_model`).

  (a) GEMM: b2l_q4_gemm / b2l_w8_gemm on b2l_q4_tile_i8 / b2l_w8_tile_i8 ("i8"; c_fc1 also as half of the interleaved
      fc1|fc2 tiling, "half") against b2l_q4_tile / quant_weight ("own"), at every 7B and 65B linear shape and
      M in 17, 64, 512, 2048.  Kernel time by CUDA events around 5 launches, the arms alternated (order flipping)
      over 9 rounds; median and spread (min..max) of the per-launch times.  The weights of a shape are one copy per arm,
      so a small one may sit in the 50 MB L2 for both arms alike;
  (b) refill_rows of one prompt of 17 / 264 / 512 tokens into a 16-row cache: 7B, the same weights uncompacted (the
      floor: every GEMM reads a layout it already holds) and then compacted, median of 7 each;
  (c) one compacted refill of 264 tokens under torch.profiler (CUDA activities), saved as a chrome trace with a
      kernel table under the output directory.

    python tools/compact_prefill_bench.py [--parts a,b,c] [--models q4,w8] [--out DIR]
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

from samples_bench import _wall, gpu_facts  # noqa: E402

# (model, linear, N, K): N output rows, K input features
SHAPES = [("7B", "c_attn", 12288, 4096), ("7B", "attn.c_proj", 4096, 4096), ("7B", "c_fc1", 11008, 4096),
          ("7B", "mlp.c_proj", 4096, 11008), ("7B", "lm_head", 32000, 4096),
          ("65B", "c_attn", 24576, 8192), ("65B", "attn.c_proj", 8192, 8192), ("65B", "c_fc1", 22016, 8192),
          ("65B", "mlp.c_proj", 8192, 22016), ("65B", "lm_head", 32000, 8192)]
MS = (17, 64, 512, 2048)


def _gemm_fn(L, bits, x, wt, sc, z, y, N, flags):
    M, K = x.shape
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=wt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                       sz_dtype=L.B2L_BF16, y=y.data_ptr(), ldy=N, M=M, N=N, K=K, prologue=0, norm_scale=None, eps=0.0,
                       epilogue=0, res=None, ldres=0, split_k=0, flags=flags)
    f = getattr(L.lib(), "b2l_w8_gemm" if bits == 8 else "b2l_q4_gemm")
    return lambda: L.check(f(C.byref(a), L.stream_ptr()), "gemm")


def _event_us(fn, n=5):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return 1e3 * s.elapsed_time(e) / n


def part_a(bits: int, rounds: int = 9) -> list:
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.quantization import tile_i8

    dev = torch.device("cuda", 0)
    lib = L.lib()
    g = torch.Generator(device=dev).manual_seed(bits)
    out = []
    for model, name, N, K in SHAPES:
        qw = torch.randint(0, 256, (K * bits // 8, N), dtype=torch.uint8, device=dev, generator=g).t()
        sc = (torch.rand(N, 1, device=dev, generator=g) * 0.01 + 0.002).bfloat16()
        z = torch.randint(0, 2**bits, (N, 1), device=dev, generator=g).bfloat16()
        if bits == 8:
            own = qw
        else:
            own = torch.empty(lib.b2l_q4_tiled_bytes(N, K), dtype=torch.uint8, device=dev)
            L.check(lib.b2l_q4_tile(qw.data_ptr(), own.data_ptr(), N, K, L.stream_ptr()), "b2l_q4_tile")
        arms = {"own": (own, 0), "i8": (tile_i8(qw, N, K, bits), L.F_GEMM_I8)}
        if name == "c_fc1":   # c_fc1 of a compacted model: the low half of the 2N-row fc1|fc2 tiling (here fc2 = fc1)
            kb = K * bits // 8
            both = torch.stack((qw.reshape(N // 8, 8, kb), qw.reshape(N // 8, 8, kb)), dim=1).reshape(2 * N, kb)
            arms["half"] = (tile_i8(both.t().contiguous().t(), 2 * N, K, bits), L.F_GEMM_I8 | L.F_GEMM_I8_LO)
            del both
        for M in MS:
            x = torch.randn(M, K, device=dev, generator=g).bfloat16()
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            fns = {k: _gemm_fn(L, bits, x, wt, sc, z, y, N, fl) for k, (wt, fl) in arms.items()}
            ys = {}
            for k, f in fns.items():   # warm-up, and the arms agree bit for bit
                f()
                ys[k] = y.clone()
            assert all(torch.equal(v, ys["own"]) for v in ys.values()), (model, name, M)
            t = {k: [] for k in fns}
            names = list(fns)
            for r in range(rounds):
                for k in (names if r % 2 == 0 else names[::-1]):
                    t[k].append(_event_us(fns[k]))
            row = dict(model=model, linear=name, N=N, K=K, M=M, bits=bits)
            for k, v in t.items():
                row[k + "_us"] = statistics.median(v)
                row[k + "_spread_us"] = [min(v), max(v)]
            row["i8_over_own"] = row["i8_us"] / row["own_us"]
            if "half_us" in row:
                row["half_over_own"] = row["half_us"] / row["own_us"]
            out.append(row)
            print(f"  {bits}-bit {model} {name} N={N} K={K} M={M}: own {row['own_us']:.1f} us "
                  f"[{min(t['own']):.1f}..{max(t['own']):.1f}], i8 {row['i8_us']:.1f} us [{min(t['i8']):.1f}..{max(t['i8']):.1f}] "
                  f"(x{row['i8_over_own']:.3f})" + (f", half {row['half_us']:.1f} us (x{row['half_over_own']:.3f})" if "half_us" in row else ""),
                  flush=True)
        del qw, own, arms
        torch.cuda.empty_cache()
    return out


def part_bc(kind: str, parts: str, out_dir: str) -> dict:
    from diag import _random_w8_model

    dev = torch.device("cuda", 0)
    model = _random_w8_model("7B", dev, seed=1234, bits=4 if kind == "q4" else 8)
    g = torch.Generator().manual_seed(16)
    pre = [torch.randint(0, 32000, (n,), generator=g).to(torch.int32).to(dev) for n in range(16, 16 + 16 * 30, 30)]
    one = {n: torch.randint(0, 32000, (n,), generator=g).to(torch.int32).to(dev) for n in (17, 264, 512)}
    S = 1024
    res = dict(model=f"7B {'gptq.int4' if kind == 'q4' else 'gptq.int8'} (synthetic)")

    def refills():
        model.reset_cache()
        model.prefill_rows(pre, S)
        for p in one.values():   # warm-up (and, uncompacted, the prefill GEMM's own layouts are built here)
            model.refill_rows([p], [0], S)
        return {n: 1e3 * statistics.median(_wall(lambda: model.refill_rows([p], [0], S)) for _ in range(7)) for n, p in one.items()}

    if "b" in parts:
        res["uncompacted_refill_ms"] = refills()
    model.compact()
    if "b" in parts:
        res["compacted_refill_ms"] = refills()
        res["compacted_over_uncompacted"] = {n: res["compacted_refill_ms"][n] / res["uncompacted_refill_ms"][n] for n in one}
        print(f"  {res['model']} refill of one prompt into a 16-row cache: "
              + ", ".join(f"{n} tokens {res['uncompacted_refill_ms'][n]:.1f} ms uncompacted / {res['compacted_refill_ms'][n]:.1f} ms "
                          f"compacted (x{res['compacted_over_uncompacted'][n]:.3f})" for n in one), flush=True)
    if "c" in parts:
        from torch.profiler import ProfilerActivity, profile

        model.reset_cache()
        model.prefill_rows(pre, S)
        model.refill_rows([one[264]], [0], S)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            model.refill_rows([one[264]], [0], S)
            torch.cuda.synchronize()
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, f"compact_refill_{kind}.pt.trace.json"))
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
        with open(os.path.join(out_dir, f"compact_refill_{kind}.txt"), "w") as f:
            f.write(table)
        print(table, flush=True)
    model.reset_cache()
    del model
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--parts", default="a,b,c")
    ap.add_argument("--models", default="q4,w8")
    ap.add_argument("--out", default=os.path.join("profiles", "compact_prefill"))   # profiles/ is git-ignored
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compact_prefill_bench needs a GPU")
    facts = gpu_facts()
    print(f"GPU (name, power limit, max SM clock): {facts}", flush=True)
    result = dict(gpu=facts)
    for kind in a.models.split(","):
        bits = 4 if kind == "q4" else 8
        if "a" in a.parts:
            result[f"gemm_{kind}"] = part_a(bits)
        if "b" in a.parts or "c" in a.parts:
            result[f"refill_{kind}"] = part_bc(kind, a.parts, a.out)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "compact_prefill_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

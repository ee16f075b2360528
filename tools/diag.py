"""GPU diagnostics: exercises every kernel against torch math and PRINTS errors instead
of asserting, section by section, each in its own subprocess with a timeout (a hung
kernel only loses its section).  Usage on the GPU box:

    python tools/diag.py            # all sections
    python tools/diag.py tc_small   # one section
"""
import ctypes as C
import gc
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SECTIONS = ["generic", "tile", "tc_small", "tc_shapes", "tc_modes", "gemv", "grid_flag", "hmma_rate", "imma_rate", "consumer_rate", "bench_gemm", "bench_tc", "trace", "bench_layers", "bench_gemv", "bench_step", "bench_ctx", "bench_13b_b8", "bench_sizes", "batch_debug", "bench_step_int8", "bench_q8_gemm", "bench_q8_gemv", "bench_w8_gemv", "bench_w8_gemm", "bench_step_w8", "bench_q4_batch", "bench_step_q4_batch", "bench_step_adapter", "bench_step_adapter_v2", "bench_step_lora", "bench_lora_kernel", "lora_timeline", "timeline"]


_DLIB = None


def dlib():
    """tools/libb200diag.so (include/b2l_diag.h): the micro-benchmarks live outside the product library."""
    global _DLIB
    if _DLIB is None:
        h = C.CDLL(os.path.join(ROOT, "tools", "libb200diag.so"))
        vp, ci = C.c_void_p, C.c_int
        for name, args in {"b2l_debug_grid_flag": [vp, vp, ci, ci, vp], "b2l_debug_hmma_rate": [vp, ci, ci, ci, ci, vp],
                           "b2l_debug_imma_rate": [vp, ci, ci, ci, ci, vp],
                           "b2l_debug_consumer_rate": [vp, ci, ci, ci, ci, vp]}.items():
            getattr(h, name).restype = ci
            getattr(h, name).argtypes = args
        h.b2l_diag_last_error.restype = C.c_char_p
        _DLIB = h
    return _DLIB


def dcheck(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {dlib().b2l_diag_last_error().decode()}")


def rand_q4(N, K, dev, seed=0, sz_dtype=None, groups=1, bits=4):
    import torch

    g = torch.Generator(device="cpu").manual_seed(seed)
    sz_dtype = sz_dtype or torch.bfloat16
    maxq = 2**bits - 1
    lv = torch.randint(0, maxq + 1, (N, K), generator=g, dtype=torch.uint8)
    epb = 8 // bits
    qw = torch.zeros((N, K // epb), dtype=torch.uint8)
    for nr in range(epb):
        qw |= lv[:, nr::epb] << (nr * bits)
    qw = qw.t().contiguous().t()
    scales = (torch.rand(N, groups, generator=g) * 0.01 + 0.002).to(sz_dtype)
    zeros = torch.randint(0, maxq + 1, (N, groups), generator=g).to(sz_dtype)
    return lv.to(dev), qw.to(dev), scales.to(dev), zeros.to(dev)


def ref_linear(x, lv, scales, zeros, tile_cols=None):
    import torch

    N, K = lv.shape
    tc = K if tile_cols is None else tile_cols
    ng = scales.shape[1]
    w = lv.double()
    for g in range(ng):
        sl = slice(g * tc, (g + 1) * tc)
        w[:, sl] = (w[:, sl] - zeros[:, g : g + 1].double()) * scales[:, g : g + 1].double()
    return (x.double() @ w.t())


def relerr(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def tc_call(L, x, qt, scales, zeros, N, K, *, y=None, prologue=0, norm_scale=None, eps=1e-5, epilogue=0, res=None,
            split_k=0, flags=0, n_out=None):
    import torch

    M = x.shape[0]
    n_out = n_out or N
    if y is None:
        y = torch.zeros((M, n_out), device=x.device, dtype=torch.bfloat16)
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=x.stride(0), qw_tiled=qt.data_ptr(), scales=scales.data_ptr(),
                       zeros=zeros.data_ptr(), sz_dtype=L.sz_dtype_of(scales), y=y.data_ptr(), ldy=y.stride(0), M=M, N=N,
                       K=K, prologue=prologue, norm_scale=None if norm_scale is None else norm_scale.data_ptr(),
                       eps=eps, epilogue=epilogue, res=None if res is None else res.data_ptr(),
                       ldres=0 if res is None else res.stride(0), split_k=split_k, flags=flags)
    rc = L.lib().b2l_q4_linear_tc(C.byref(a), L.stream_ptr())
    if rc != 0:
        return None, f"rc={rc}: {L.lib().b2l_last_error().decode()}"
    return y, None


def tile(L, qw, N, K):
    import torch

    qt = torch.empty(L.lib().b2l_q4_tiled_bytes(N, K), dtype=torch.uint8, device=qw.device)
    L.check(L.lib().b2l_q4_tile(qw.data_ptr(), qt.data_ptr(), N, K, L.stream_ptr()), "tile")
    return qt


def tile_mma(L, qw, N, K):
    import torch

    qt = torch.empty(L.lib().b2l_q4_tiled_mma_bytes(N, K), dtype=torch.uint8, device=qw.device)
    L.check(L.lib().b2l_q4_tile_mma(qw.data_ptr(), qt.data_ptr(), N, K, L.stream_ptr()), "tile_mma")
    return qt


def tile_i8(L, qw, N, K):
    import torch

    qt = torch.empty(L.lib().b2l_q4_tiled_i8_bytes(N, K), dtype=torch.uint8, device=qw.device)
    L.check(L.lib().b2l_q4_tile_i8(qw.data_ptr(), qt.data_ptr(), N, K, L.stream_ptr()), "tile_i8")
    return qt


def gemv_call(L, x, qt, scales, zeros, N, K, *, y=None, prologue=0, norm_scale=None, eps=1e-5, epilogue=0, res=None, grid=0,
              flags=0, n_out=None):
    import torch

    n_out = n_out or N
    if y is None:
        y = torch.zeros((1, n_out), device=x.device, dtype=torch.bfloat16)
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=scales.data_ptr(), zeros=zeros.data_ptr(),
                       sz_dtype=L.sz_dtype_of(scales), y=y.data_ptr(), ldy=n_out, M=1, N=N, K=K, prologue=prologue,
                       norm_scale=None if norm_scale is None else norm_scale.data_ptr(), eps=eps, epilogue=epilogue,
                       res=None if res is None else res.data_ptr(), ldres=N, split_k=grid, flags=flags)
    rc = L.lib().b2l_q4_gemv(C.byref(a), L.stream_ptr())
    if rc != 0:
        return None, f"rc={rc}: {L.lib().b2l_last_error().decode()}"
    return y, None


def gemv_batch_call(L, x, qt, scales, zeros, N, K, *, y=None, prologue=0, norm_scale=None, eps=1e-5, epilogue=0, res=None, grid=0,
                    flags=0, n_out=None):
    """b2l_q4_gemv_batch on x (M, K), M <= 8."""
    import torch

    M = x.shape[0]
    n_out = n_out or N
    if y is None:
        y = torch.zeros((M, n_out), device=x.device, dtype=torch.bfloat16)
    ws = torch.zeros(L.lib().b2l_q4_gemv_batch_workspace_bytes(K), dtype=torch.uint8, device=x.device)
    a = L.Q4LinearArgs(x=x.data_ptr(), ldx=x.stride(0), qw_tiled=qt.data_ptr(), scales=scales.data_ptr(), zeros=zeros.data_ptr(),
                       sz_dtype=L.sz_dtype_of(scales), y=y.data_ptr(), ldy=n_out, M=M, N=N, K=K, prologue=prologue,
                       norm_scale=None if norm_scale is None else norm_scale.data_ptr(), eps=eps, epilogue=epilogue,
                       res=None if res is None else res.data_ptr(), ldres=N, split_k=grid, flags=flags, workspace=ws.data_ptr())
    rc = L.lib().b2l_q4_gemv_batch(C.byref(a), L.stream_ptr())
    if rc != 0:
        return None, f"rc={rc}: {L.lib().b2l_last_error().decode()}"
    torch.cuda.synchronize()
    return y, None


def sec_gemv():
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    for (N, K, grid) in [(16, 64, 0), (16, 128, 0), (32, 2048, 0), (48, 4096, 0), (130, 256, 0), (4096, 4096, 0), (4096, 4096, 7),
                         (12288, 4096, 0), (4096, 11008, 0), (32000, 4096, 0), (22016, 4096, 0), (128, 6400, 0)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=N + K)
        qt = tile_i8(L, qw, N, K)
        back = torch.empty_like(qw)
        L.check(L.lib().b2l_q4_untile_i8(qt.data_ptr(), back.data_ptr(), N, K, L.stream_ptr()), "untile_i8")
        x = torch.randn(1, K, device=dev).bfloat16()
        y, err = gemv_call(L, x, qt, sc, z, N, K, grid=grid)
        torch.cuda.synchronize()
        if err:
            print(f"gemv N={N} K={K} grid={grid}: {err}")
            continue
        want = ref_linear(x, lv, sc, z)
        wb = want.float().bfloat16()
        print(f"gemv N={N} K={K} grid={grid}: roundtrip={bool(torch.equal(back, qw))} relerr={relerr(y, want):.3e} "
              f"exact_bf16_frac={float((y == wb).float().mean()):.4f}")
        if N == 16 and K == 64:
            print("   got ", [round(float(v), 4) for v in y[0, :8]])
            print("   want", [round(float(v), 4) for v in want[0, :8]])
    N, K = 512, 1024
    lv, qw, sc, z = rand_q4(N, K, dev, seed=5)
    qt = tile_i8(L, qw, N, K)
    x = (torch.randn(1, K, device=dev) * 0.7).bfloat16()
    g = (1 + 0.1 * torch.randn(K, device=dev)).bfloat16()
    ms = torch.mean(x * x, dim=-1, keepdim=True)
    xn = g * (x * torch.rsqrt(ms + 1e-5))
    y, err = gemv_call(L, x, qt, sc, z, N, K, prologue=1, norm_scale=g)
    torch.cuda.synchronize()
    print("gemv rmsnorm prologue:", err or f"relerr={relerr(y, ref_linear(xn, lv, sc, z)):.3e}")
    res = torch.randn(1, N, device=dev).bfloat16()
    y, err = gemv_call(L, x, qt, sc, z, N, K, epilogue=1, res=res)
    torch.cuda.synchronize()
    want = (ref_linear(x, lv, sc, z).float().bfloat16() + res)
    print("gemv residual:", err or f"relerr={relerr(y, want):.3e} exact={float((y == want).float().mean()):.4f}")
    buf = res.clone()
    y, err = gemv_call(L, x, qt, sc, z, N, K, epilogue=1, res=buf, y=buf)
    torch.cuda.synchronize()
    print("gemv in-place residual:", err or f"relerr={relerr(buf, want):.3e}")
    full = ref_linear(x, lv, sc, z).float().bfloat16().reshape(1, N // 16, 2, 8)
    a, b = full[:, :, 0].reshape(1, -1), full[:, :, 1].reshape(1, -1)
    want = torch.nn.functional.silu(a) * b
    y, err = gemv_call(L, x, qt, sc, z, N, K, epilogue=2, n_out=N // 2)
    torch.cuda.synchronize()
    print("gemv swiglu:", err or f"relerr={relerr(y, want):.3e} exact={float((y == want).float().mean()):.4f}")
    y, err = gemv_call(L, x, qt, sc, z, N, K, flags=1)
    torch.cuda.synchronize()
    print("gemv pdl flag:", err or f"relerr={relerr(y, ref_linear(x, lv, sc, z)):.3e}")


def sec_bench_gemv():
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    lib = L.lib()
    for (name, N, K) in [("c_attn", 12288, 4096), ("c_proj", 4096, 4096), ("fc12", 22016, 4096), ("mlp_proj", 4096, 11008), ("lm_head", 32000, 4096)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=3)
        n_copies = max(4, int(400e6 // (N * K // 2)) + 1)
        qts = [tile_i8(L, qw, N, K) for _ in range(n_copies)]
        x = torch.randn(1, K, device=dev).bfloat16()
        y = torch.zeros(1, N, device=dev, dtype=torch.bfloat16)
        for grid in (0,):
            for flags in (1, 17):
                args = [L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                                       sz_dtype=0, y=y.data_ptr(), ldy=N, M=1, N=N, K=K, prologue=0, norm_scale=None, eps=1e-5,
                                       epilogue=0, res=None, ldres=N, split_k=grid, flags=flags) for qt in qts]
                if lib.b2l_q4_gemv(C.byref(args[0]), L.stream_ptr()) != 0:
                    print(f"{name} grid={grid}: {lib.b2l_last_error().decode()[:90]}")
                    continue
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for a in args:
                        lib.b2l_q4_gemv(C.byref(a), L.stream_ptr())
                us = _time(g.replay, iters=10, warm=2) / n_copies
                print(f"gemv {name} N={N} K={K} grid={grid or 296} pdl={flags}: {us:.2f} us/launch  {(N * K / 2) / us / 1e3:.0f} GB/s")
        del qts


def sec_generic():
    import torch
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    dev = torch.device("cuda")
    for bits, groups, N, K, M in [(4, 1, 24, 64, 3), (4, 4, 24, 128, 1), (8, 1, 16, 64, 5), (8, 3, 8, 96, 2), (4, 1, 130, 256, 1),
                                  (4, 1, 4096, 4096, 1), (4, 1, 12288, 4096, 2)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=bits + N, groups=groups, bits=bits)
        tc = K // groups
        lin = ColBlockQuantizedLinear(K, N, False, bits=bits, tile_cols=tc if groups > 1 else -1).to(dev)
        lin.quant_weight.copy_(qw); lin.scales = sc; lin.zeros = z
        x = torch.randn(M, K, device=dev).bfloat16()
        y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        rc = L.lib().b2l_q_linear(x.data_ptr(), K, lin.quant_weight.data_ptr(), sc.data_ptr(), z.data_ptr(), L.sz_dtype_of(sc), None,
                                  y.data_ptr(), N, M, N, K, bits, tc, L.stream_ptr())
        torch.cuda.synchronize()
        want = ref_linear(x, lv, sc, z, tc)
        print(f"generic bits={bits} groups={groups} N={N} K={K} M={M}: rc={rc} relerr={relerr(y, want):.2e}")
        for dt in (torch.float32, torch.bfloat16):
            w = lin.get_weight(dt)
            wr = lv.float().to(dt)
            for g in range(groups):
                sl = slice(g * tc, (g + 1) * tc)
                wr[:, sl] -= z[:, g : g + 1]
                wr[:, sl] *= sc[:, g : g + 1]
            print(f"   dequant {dt}: bit-exact={bool(torch.equal(w, wr))}")


def sec_tile():
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    for N, K in [(128, 64), (130, 256), (4096, 4096), (96, 128)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=N)
        qt = tile(L, qw, N, K)
        back = torch.empty_like(qw)
        L.check(L.lib().b2l_q4_untile(qt.data_ptr(), back.data_ptr(), N, K, L.stream_ptr()), "untile")
        torch.cuda.synchronize()
        # independent check of the documented layout on the host
        w = qt.view(torch.int32).reshape(-1, K // 32, 128, 4).cpu()
        lvc = lv.cpu()
        ok = True
        for (nt, ks, r, i) in [(0, 0, 0, 0), (0, K // 32 - 1, 5, 3), ((N - 1) // 128, 1 % (K // 32), (N - 1) % 128, 2)]:
            word = int(w[nt, ks, r, i]) & 0xFFFFFFFF
            o = nt * 128 + r
            for s in range(8):
                k = ks * 32 + 8 * i + (2 * s if s < 4 else 2 * (s - 4) + 1)
                ok &= ((word >> (4 * s)) & 0xF) == int(lvc[o, k])
        print(f"tile N={N} K={K}: roundtrip={bool(torch.equal(back, qw))} layout_spot={ok}")


def sec_tc_small():
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    N, K, M = 128, 64, 1
    lv, qw, sc, z = rand_q4(N, K, dev, seed=1)
    qt = tile(L, qw, N, K)
    x = torch.randn(M, K, device=dev).bfloat16()
    y, err = tc_call(L, x, qt, sc, z, N, K, split_k=1)
    torch.cuda.synchronize()
    print("tc_small first call:", err or "launched")
    want = ref_linear(x, lv, sc, z)
    print(f"  N=128 K=64 M=1 S=1 relerr={relerr(y, want):.3e}")
    print("  got ", [round(float(v), 4) for v in y[0, :6]])
    print("  want", [round(float(v), 4) for v in want[0, :6]])
    # hypotheses if wrong: pair order swapped inside an A fragment / B rows
    xs = x.clone().reshape(M, K // 2, 2).flip(-1).reshape(M, K)
    print(f"  hypothesis pair-swapped relerr={relerr(y, ref_linear(xs, lv, sc, z)):.3e}")
    xh = x.clone().reshape(M, K // 16, 2, 8).flip(2).reshape(M, K)
    print(f"  hypothesis k-halves-swapped relerr={relerr(y, ref_linear(xh, lv, sc, z)):.3e}")
    for (N, K, M, S) in [(128, 64, 1, 1), (128, 128, 1, 1), (128, 256, 3, 1), (128, 256, 1, 2), (256, 512, 1, 4), (256, 1024, 8, 8),
                         (128, 96, 1, 1), (384, 4096, 1, 4), (130, 256, 2, 2), (128, 1024, 16, 2), (128, 1024, 9, 2)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=N + K)
        qt = tile(L, qw, N, K)
        x = torch.randn(M, K, device=dev).bfloat16()
        for flags in (0, 2):
            if flags == 2 and M > 8:
                continue
            y, err = tc_call(L, x, qt, sc, z, N, K, split_k=S, flags=flags)
            torch.cuda.synchronize()
            if err:
                print(f"  N={N} K={K} M={M} S={S} flags={flags}: {err}")
                continue
            want = ref_linear(x, lv, sc, z)
            wb = want.float().bfloat16()
            print(f"  N={N} K={K} M={M} S={S} flags={flags}: relerr={relerr(y, want):.3e} exact_bf16_frac={float((y == wb).float().mean()):.4f}")


def sec_tc_shapes():
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    for (N, K) in [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008), (32000, 4096)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=N % 1000 + K)
        qt = tile(L, qw, N, K)
        for M in (1, 8):
            x = torch.randn(M, K, device=dev).bfloat16()
            for S in (0, 1, 2, 4, 8):
                y, err = tc_call(L, x, qt, sc, z, N, K, split_k=S)
                torch.cuda.synchronize()
                if err:
                    print(f"  N={N} K={K} M={M} S={S}: {err}")
                    continue
                want = ref_linear(x, lv, sc, z)
                print(f"  N={N} K={K} M={M} S={S}: relerr={relerr(y, want):.3e}")
        del lv, qw, qt


def sec_tc_modes():
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    N, K, M = 512, 1024, 2
    lv, qw, sc, z = rand_q4(N, K, dev, seed=5)
    qt = tile(L, qw, N, K)
    x = (torch.randn(M, K, device=dev) * 0.7).bfloat16()
    g = (1 + 0.1 * torch.randn(K, device=dev)).bfloat16()
    # rmsnorm prologue (bf16 rounding points of model.py:270-277 via torch bf16 ops)
    ms = torch.mean(x * x, dim=-1, keepdim=True)
    xn = g * (x * torch.rsqrt(ms + 1e-5))
    y, err = tc_call(L, x, qt, sc, z, N, K, prologue=1, norm_scale=g, eps=1e-5)
    torch.cuda.synchronize()
    print("rmsnorm prologue:", err or f"relerr={relerr(y, ref_linear(xn, lv, sc, z)):.3e}")
    # residual epilogue
    res = torch.randn(M, N, device=dev).bfloat16()
    y, err = tc_call(L, x, qt, sc, z, N, K, epilogue=1, res=res)
    torch.cuda.synchronize()
    want = (ref_linear(x, lv, sc, z).float().bfloat16() + res)
    print("residual epilogue:", err or f"relerr={relerr(y, want):.3e} exact={float((y == want).float().mean()):.4f}")
    # in-place residual
    buf = res.clone()
    y, err = tc_call(L, x, qt, sc, z, N, K, epilogue=1, res=buf, y=buf)
    torch.cuda.synchronize()
    print("in-place residual:", err or f"relerr={relerr(buf, want):.3e}")
    # swiglu: rows interleaved [64 a | 64 b]
    full = ref_linear(x, lv, sc, z).float().bfloat16().reshape(M, N // 128, 2, 64)
    a, b = full[:, :, 0].reshape(M, -1), full[:, :, 1].reshape(M, -1)
    want = torch.nn.functional.silu(a) * b
    y, err = tc_call(L, x, qt, sc, z, N, K, epilogue=2, n_out=N // 2)
    torch.cuda.synchronize()
    print("swiglu epilogue:", err or f"relerr={relerr(y, want):.3e} exact={float((y == want).float().mean()):.4f}")
    # pdl flag outside a chain
    y, err = tc_call(L, x, qt, sc, z, N, K, flags=1)
    torch.cuda.synchronize()
    print("pdl flag:", err or f"relerr={relerr(y, ref_linear(x, lv, sc, z)):.3e}")
    # fp32 scales/zeros
    lv, qw, sc, z = rand_q4(N, K, dev, seed=6, sz_dtype=torch.float32)
    qt = tile(L, qw, N, K)
    y, err = tc_call(L, x, qt, sc, z, N, K)
    torch.cuda.synchronize()
    print("fp32 scales:", err or f"relerr={relerr(y, ref_linear(x, lv, sc, z)):.3e}")


def _time(fn, iters=20, warm=3):
    import torch

    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us


def make_args(L, x, qt, scales, zeros, N, K, y, *, prologue=0, norm_scale=None, epilogue=0, res=None, split_k=0, flags=0, trace=None):
    return L.Q4LinearArgs(x=x.data_ptr(), ldx=x.stride(0), qw_tiled=qt.data_ptr(), scales=scales.data_ptr(),
                          zeros=zeros.data_ptr(), sz_dtype=L.sz_dtype_of(scales), y=y.data_ptr(), ldy=y.stride(0), M=x.shape[0], N=N,
                          K=K, prologue=prologue, norm_scale=None if norm_scale is None else norm_scale.data_ptr(), eps=1e-5,
                          epilogue=epilogue, res=None if res is None else res.data_ptr(), ldres=0 if res is None else res.stride(0),
                          split_k=split_k, flags=flags, trace=None if trace is None else trace.data_ptr())


def sec_grid_flag():
    """Grid-wide arrive-and-wait through a global counter: the cost of a dependency without a kernel boundary."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    rounds = 16
    for cps in (1, 2):
        out = torch.zeros(2 * rounds, dtype=torch.int64, device=dev)
        out[rounds:] = 2**62
        counter = torch.zeros(1, dtype=torch.int32, device=dev)
        dcheck(dlib().b2l_debug_grid_flag(out.data_ptr(), counter.data_ptr(), cps, rounds, L.stream_ptr()), "grid_flag")
        torch.cuda.synchronize()
        o = out.cpu()
        print(f"ctas_per_sm={cps}: arrive-and-wait ns per round, max over CTAs {o[:rounds].tolist()}  min {o[rounds:].tolist()}", flush=True)


def sec_hmma_rate():
    """Legacy tensor pipe: cycles per mma.sync.m16n8k16 per SM sub-partition, by warps / chains / unpack."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    out = torch.zeros(2, dtype=torch.int64, device=dev)
    iters = 512
    for unpack in (0, 1):
        for warps in (4, 8, 16, 20):
            for chains in (1, 2, 4, 8):
                dcheck(dlib().b2l_debug_hmma_rate(out.data_ptr(), warps, chains, iters, unpack, L.stream_ptr()), "hmma_rate")
                torch.cuda.synchronize()
                dcheck(dlib().b2l_debug_hmma_rate(out.data_ptr(), warps, chains, iters, unpack, L.stream_ptr()), "hmma_rate")
                torch.cuda.synchronize()
                cyc = int(out[0])
                per_smsp = (warps / 4) * iters * 8
                print(f"unpack={unpack} warps={warps:2d} chains={chains}: {cyc} cycles, {cyc / (iters * 8):.1f} clk per MMA per warp, "
                      f"{cyc / per_smsp:.2f} clk per MMA per sub-partition", flush=True)


def sec_imma_rate():
    """Legacy integer tensor pipe: cycles per mma.sync.m16n8k32 (u8 x s8) per SM sub-partition, by warps / chains / ALU ops."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    out = torch.zeros(2, dtype=torch.int64, device=dev)
    iters = 512
    for n_alu in (0, 2, 4):
        for warps in (4, 8, 16, 20):
            for chains in (1, 2, 4, 8):
                for _ in range(2):
                    dcheck(dlib().b2l_debug_imma_rate(out.data_ptr(), warps, chains, iters, n_alu, L.stream_ptr()), "imma_rate")
                    torch.cuda.synchronize()
                cyc = int(out[0])
                per_smsp = (warps / 4) * iters * 8
                print(f"n_alu={n_alu} warps={warps:2d} chains={chains}: {cyc} cycles, {cyc / (iters * 8):.1f} clk per MMA per warp, "
                      f"{cyc / per_smsp:.2f} clk per MMA per sub-partition", flush=True)


def sec_consumer_rate():
    """The decode consumer loop on shared-memory-resident stages: what bounds it -- LDS, IMMA issue, or their sum?"""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    out = torch.zeros(2, dtype=torch.int64, device=dev)
    iters = 200
    names = {1: "weights LDS", 2: "digit LDS", 3: "both LDS", 4: "IMMA only", 5: "weights LDS + IMMA", 7: "all", 15: "all, unused lanes predicated off",
             13: "weights LDS + IMMA + (digits off)"}
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for warps in (16, 8):
        for ctas in (1, sms):
            for mode in (1, 2, 3, 4, 5, 7, 15):
                for _ in range(2):
                    dcheck(dlib().b2l_debug_consumer_rate(out.data_ptr(), warps, iters, mode, ctas, L.stream_ptr()), "consumer_rate")
                    torch.cuda.synchronize()
                cyc = int(out[0]) / (iters * 8)
                print(f"warps={warps:2d} ctas={ctas:3d} mode={mode:2d} ({names.get(mode, '')}): {cyc:.0f} cycles per 16 KB stage  "
                      f"-> {16384 / cyc:.1f} B/clk/SM = {16384 / cyc * 1.98 * sms / 1e3:.1f} TB/s-equivalent at 1.98 GHz", flush=True)


def sec_bench_gemm():
    """The wgmma prefill GEMM at the 13B widths, M = 4096 (BASELINE configs[3] prefill 8 x 512), next to torch.matmul
    (library bf16 GEMM on a dense weight of the same shape) as the tensor-pipe yardstick."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    M = int(os.environ.get("B2L_GEMM_M", "4096"))
    for (name, N, K) in [("c_attn", 15360, 5120), ("c_proj", 5120, 5120), ("fc1", 13824, 5120), ("mlp_proj", 5120, 13824), ("7B c_attn", 12288, 4096)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=3)
        qt = tile(L, qw, N, K)
        x = torch.randn(M, K, device=dev).bfloat16()
        y = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        a = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(), sz_dtype=0, y=y.data_ptr(), ldy=N,
                           M=M, N=N, K=K, prologue=0, norm_scale=None, eps=0.0, epilogue=0, res=None, ldres=0, split_k=0, flags=0)
        fn = lambda: L.check(L.lib().b2l_q4_gemm(C.byref(a), L.stream_ptr()), "gemm")
        us = _time(fn, iters=10, warm=2)
        w = torch.randn(N, K, device=dev).bfloat16()
        us_t = _time(lambda: torch.matmul(x, w.t()), iters=10, warm=2)
        fl = 2.0 * M * N * K
        print(f"gemm {name} M={M} N={N} K={K}: {us:.0f} us = {fl / us / 1e6:.0f} TFLOP/s   | torch.matmul bf16: {us_t:.0f} us = {fl / us_t / 1e6:.0f} TFLOP/s", flush=True)


def sec_bench_tc():
    """The 9..16-row wgmma linear on the 7B shapes at M = 16: weight copies rotated past the 50 MB L2, CUDA events;
    GB/s of packed weights."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    M = int(os.environ.get("B2L_TC_M", "16"))
    for (name, N, K) in [("c_attn", 12288, 4096), ("c_proj", 4096, 4096), ("fc12", 22016, 4096), ("mlp_proj", 4096, 11008), ("lm_head", 32000, 4096)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=3)
        n_copies = max(2, int(200e6 // (N * K // 2)) + 1)
        qts = [tile(L, qw, N, K) for _ in range(n_copies)]
        x = torch.randn(M, K, device=dev).bfloat16()
        y = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        args = [make_args(L, x, qt, sc, z, N, K, y) for qt in qts]

        def run():
            for a in args:
                L.check(L.lib().b2l_q4_linear_tc(C.byref(a), L.stream_ptr()), "tc")

        us = _time(run, iters=10, warm=2) / n_copies
        print(f"tc {name} M={M} N={N} K={K}: {us:.1f} us = {N * K / 2 / us / 1e3:.0f} GB/s of packed weights", flush=True)
        del qts


def sec_trace():
    """clock64 stamps of CTA 0 of one launch: where does a CTA spend its time?"""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    for (name, N, K, S) in [("c_attn", 12288, 4096, 4), ("c_proj", 4096, 4096, 8), ("mlp_proj", 4096, 11008, 8)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=3)
        qt = tile(L, qw, N, K)
        x = torch.randn(1, K, device=dev).bfloat16()
        g = torch.ones(K, device=dev, dtype=torch.bfloat16)
        y = torch.zeros(1, N, device=dev, dtype=torch.bfloat16)
        tr = torch.zeros(256, dtype=torch.int64, device=dev)
        a = make_args(L, x, qt, sc, z, N, K, y, prologue=1, norm_scale=g, split_k=S, trace=tr)
        for rep in range(2):  # second launch: weights of CTA 0 may be L2-warm, code is warm
            tr.zero_()
            flush = torch.empty(200 * 1024 * 1024, dtype=torch.uint8, device=dev).fill_(1)
            L.check(L.lib().b2l_q4_linear_tc(C.byref(a), L.stream_ptr()), "tc")
            torch.cuda.synchronize()
            t = tr.cpu().tolist()
            t0 = t[0]
            rel = lambda i: (t[i] - t0) if t[i] else None
            nst = (K // 32 // S + 1) // 2
            print(f"{name} S={S} rep={rep} stages={nst}: pdl_wait={rel(2)} x_ready={rel(3)} acc_done={rel(104)} "
                  f"csync1={rel(105)} epi={rel(106)} end={rel(107)}")
            k = min(nst, 20)
            print("   tma_issue ", [rel(108 + i) for i in range(k)])
            print("   w_full    ", [rel(4 + i) for i in range(k)])
            print("   mma_done  ", [rel(44 + i) for i in range(k)])
            del flush


def sec_bench_layers():
    """GPU time of the int4 linear per 7B shape: `n_copies` launches on distinct weight
    copies (> L2) captured in one CUDA graph, so the host cost of a launch is not in it."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    lib = L.lib()
    for (name, N, K) in [("c_attn", 12288, 4096), ("c_proj", 4096, 4096), ("fc12", 22016, 4096), ("mlp_proj", 4096, 11008), ("lm_head", 32000, 4096)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=3)
        n_copies = max(4, int(400e6 // (N * K // 2)) + 1)
        qts = [tile(L, qw, N, K) for _ in range(n_copies)]
        x = torch.randn(1, K, device=dev).bfloat16()
        y = torch.zeros(1, N, device=dev, dtype=torch.bfloat16)
        for S in (0, 1, 2, 3, 4, 6, 8):
            for flags in (0,):
                args = [make_args(L, x, qt, sc, z, N, K, y, split_k=S, flags=flags) for qt in qts]
                if lib.b2l_q4_linear_tc(C.byref(args[0]), L.stream_ptr()) != 0:
                    print(f"{name} S={S} flags={flags}: {lib.b2l_last_error().decode()[:90]}")
                    continue
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for a in args:
                        lib.b2l_q4_linear_tc(C.byref(a), L.stream_ptr())
                us = _time(g.replay, iters=10, warm=2) / n_copies
                print(f"{name} N={N} K={K} S={S} flags={flags}: {us:.2f} us/launch  {(N * K / 2) / us / 1e3:.0f} GB/s  ({n_copies} launches/graph)")
        del qts


def sec_bench_step():
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization
    from bench import build_synthetic_model

    dev = torch.device("cuda")
    model = build_synthetic_model("7B", dev)
    S = 2048
    for pdl in (1, 0):
        for graph_after in (2, 0):
            model.reset_cache()
            model.decode_flags = pdl
            model.graph_after = graph_after
            model.copy_logits = False
            idx = torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32)
            with torch.no_grad():
                model(idx, S, torch.arange(16, device=dev))
                tok = torch.randint(0, 32000, (1, 1), device=dev, dtype=torch.int32)
                pos = [torch.tensor([16 + i], device=dev) for i in range(64)]
                for i in range(4):
                    model(tok, S, pos[i])
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(4, 64):
                    model(tok, S, pos[i])
                e1.record()
                torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 60 * 1e3
            print(f"decode step 7B pos~16-80 pdl={pdl} graph={graph_after > 0}: {us:.1f} us/token  {1e6 / us:.1f} tok/s")


def sec_bench_ctx():
    """Decode step time against context length (graph + PDL): what single-token attention costs."""
    import torch
    from bench import build_synthetic_model

    dev = torch.device("cuda")
    model = build_synthetic_model("7B", dev)
    S = 2048
    model.copy_logits = False
    tok = torch.randint(0, 32000, (1, 1), device=dev, dtype=torch.int32)
    with torch.no_grad():
        model(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
        t16 = None
        for p0 in (16, 120, 136, 512, 1024, 1536, 1990):
            pos = [torch.tensor([p0 + i], device=dev) for i in range(48)]
            for i in range(6):
                model(tok, S, pos[i])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(6, 46):
                model(tok, S, pos[i])
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 40 * 1e3
            t16 = t16 or us
            print(f"decode step 7B pos~{p0 + 6}-{p0 + 46}: {us:.1f} us/token  (+{(us - t16) / 32:.2f} us per layer over pos 16)")


def _decode_us(model, B, S, dev, p0=512, n=24):
    import torch

    tok = torch.randint(0, 32000, (B, 1), device=dev, dtype=torch.int32)
    pos = [torch.tensor([p0 + i], device=dev) for i in range(n + 6)]
    with torch.no_grad():
        for i in range(6):
            model(tok, S, pos[i])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(6, 6 + n):
            model(tok, S, pos[i])
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


def sec_bench_13b_b8():
    """BASELINE.json configs[3]: LLaMA-13B gptq.int4, batch 8, prefill 512 then decode (ctx 2048)."""
    import torch
    from bench import build_synthetic_model

    dev = torch.device("cuda")
    model = build_synthetic_model("13B", dev)
    model.copy_logits = False
    B, T, S = 8, 512, 2048
    idx = torch.randint(0, 32000, (B, T), device=dev, dtype=torch.int32)
    with torch.no_grad():
        for rep in range(2):
            model.reset_cache()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model(idx, S, torch.arange(T, device=dev))
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
        print(f"13B gptq.int4 prefill B={B} T={T}: {ms:.1f} ms  ({B * T / ms * 1e3:.0f} tokens/s; wgmma tile GEMM for every linear)")
        if os.environ.get("B2L_PREFILL_PROFILE"):
            from torch.profiler import ProfilerActivity, profile
            model.reset_cache()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                model(idx, S, torch.arange(T, device=dev))
                torch.cuda.synchronize()
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=14, max_name_column_width=60))
    us = _decode_us(model, B, S, dev, p0=T)
    from lit_llama_b200.quantization import BATCH_GEMV
    print(f"13B gptq.int4 decode B={B} pos~{T}: {us:.0f} us/step  {B * 1e6 / us:.0f} tokens/s  "
          f"({'mma.sync batch kernel' if BATCH_GEMV else 'wgmma kernel'}, M={B})")


def sec_bench_sizes():
    """Batch-1 decode of every LLaMA size the reference names (lit_llama/model.py llama_configs)."""
    import torch
    from bench import build_synthetic_model

    dev = torch.device("cuda")
    for name in ("13B", "30B", "65B"):
        model = build_synthetic_model(name, dev)
        model.copy_logits = False
        with torch.no_grad():
            model(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), 2048, torch.arange(16, device=dev))
        us = _decode_us(model, 1, 2048, dev, p0=16, n=32)
        cfg = model.config
        nh = [m for m in model.transformer.h[0].mlp.modules() if hasattr(m, "quant_weight")][0].quant_weight.shape[0]
        w_bytes = cfg.n_layer * (4 * cfg.n_embd * cfg.n_embd + 3 * cfg.n_embd * nh) // 2 + cfg.padded_vocab_size * cfg.n_embd // 2
        print(f"{name} gptq.int4 decode B=1 pos~16-50: {us:.0f} us/token  {1e6 / us:.1f} tok/s  "
              f"({w_bytes / us / 1e3:.0f} GB/s of packed weights = {w_bytes / us / 1e3 / 6573.2:.3f} of measured HBM peak)")
        del model
        torch.cuda.empty_cache()


def sec_batch_debug():
    """B = 2 decode on the tiny model: batch kernel vs batch-1 kernel, with and without PDL / fast path."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from gpu_util import build_tiny

    dev = torch.device("cuda")
    cfg = dict(block_size=32, vocab_size=96, n_layer=2, n_head=4, n_embd=128)
    idx = torch.tensor([[3, 17, 40], [9, 9, 1]], device=dev)
    for flags in (1, 0):
        for fast in (True, False):
            model, _, _ = build_tiny(dev, cfg)
            model.decode_flags = flags
            model.graph_after = 0
            if not fast:
                model._fast_ok = False
            with torch.no_grad():
                pre2 = model(idx, 16, torch.arange(3, device=dev)).clone()
                both = model(torch.tensor([[5], [60]], device=dev), 16, torch.tensor([3], device=dev)).clone()
                model.reset_cache()
                if not fast:
                    model._fast_ok = False
                pre1 = model(idx[1:], 16, torch.arange(3, device=dev)).clone()
                one = model(torch.tensor([[60]], device=dev), 16, torch.tensor([3], device=dev)).clone()
            print(f"pdl={flags} fast={fast}: prefill row diff {float((pre2[1:].float() - pre1.float()).abs().max()):.4g}  "
                  f"decode row diff {float((both[1:].float() - one.float()).abs().max()):.4g}  (|logits| max {float(one.float().abs().max()):.3g})", flush=True)


def _card():
    """The card and its power limit, printed beside every absolute number."""
    import torch

    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        pl = "power limit unknown"
    return f"{torch.cuda.get_device_name()} ({pl})"


def _q8_tiled_forward(cb_forward):
    """Linear8bitLt.forward before b2l_q8_gemv_cb: at M = 1, b2l_q8_gemv on the cached re-tiled copy (Linear8bitLt.tiled)."""
    import torch
    from lit_llama_b200 import _lib as L

    def forward(self, x):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        if x2.shape[0] != 1:
            return cb_forward(self, x)
        y = torch.empty(self.out_features, dtype=x.dtype, device=x.device)
        L.check(L.lib().b2l_q8_gemv(x2.data_ptr(), self.tiled().data_ptr(), self.weight.data.data_ptr(), self.weight.SCB.data_ptr(), None,
                                    y.data_ptr(), self.out_features, self.in_features, self.threshold, 0, L.stream_ptr()), "b2l_q8_gemv")
        return y.reshape(*shape[:-1], self.out_features)

    return forward


def _int8_old_vs_new(model, S, dev, rounds=3):
    """7B batch-1 decode with Linear8bitLt.forward (CB read directly) and the parent's forward (re-tiled copy), alternated
    in one process.  Each run writes the same tokens at the same positions, then decodes one fixed token whose logits
    must be bit-identical between the two."""
    import torch
    import lit_llama_b200 as P

    new_forward = P.Linear8bitLt.forward
    old_forward = _q8_tiled_forward(new_forward)
    us = {"new": [], "old": []}
    logits = {}
    try:
        for _ in range(rounds):
            for kind, fwd in (("new", new_forward), ("old", old_forward)):
                P.Linear8bitLt.forward = fwd
                model._module_graph = None   # the graph bakes the launches: capture it again with this forward
                torch.manual_seed(0)
                us[kind].append(_decode_us(model, 1, S, dev, p0=2000, n=24))
                with torch.no_grad():
                    out = model(torch.tensor([[1234]], device=dev, dtype=torch.int32), S, torch.tensor([2040], device=dev)).clone()
                if kind in logits:
                    assert torch.equal(out, logits[kind]), f"{kind} forward is not deterministic"
                logits[kind] = out
    finally:
        P.Linear8bitLt.forward = new_forward
    assert torch.equal(logits["new"], logits["old"]), "CB-direct and tiled batch-1 decode give different logits"
    fmt = lambda v: " ".join(f"{x:.1f}" for x in v)
    print(f"  7B decode B=1, alternated: new forward (CB read directly) {fmt(us['new'])} us/token | parent forward (re-tiled copy) "
          f"{fmt(us['old'])} us/token | logits bit-identical", flush=True)


def sec_bench_step_int8():
    """--quantize llm.int8 (BASELINE config 2) at 7B, 13B, 30B and 65B: a 512-token prompt (the M >= 2 GEMM) and batch-1
    decode at ctx ~2048 (module path replayed as a CUDA graph).  B2L_INT8_SIZES picks the sizes.  The peak memory is
    taken before 7B's old-against-new decode comparison, which builds the parent's re-tiled copy."""
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    dev = torch.device("cuda")
    print(_card(), flush=True)
    S = 2048
    for name in os.environ.get("B2L_INT8_SIZES", "7B,13B,30B,65B").split(","):
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.bfloat16)
        try:
            with torch.device(dev), quantization("llm.int8"):
                model = P.LLaMA.from_name(name)
        finally:
            torch.set_default_dtype(prev)
        model.eval()
        model.copy_logits = False
        w8 = sum(m.weight.numel() for m in model.modules() if isinstance(m, P.Linear8bitLt))
        idx = torch.randint(0, 32000, (1, 512), device=dev, dtype=torch.int32)
        with torch.no_grad():
            prompt_us = _time(lambda: model(idx, S, torch.arange(512, device=dev)), iters=5, warm=2)
            model.reset_cache()
            us = _decode_us(model, 1, S, dev, p0=2000, n=24)
        print(f"{name} llm.int8: prompt 512 tokens {prompt_us / 1e3:.2f} ms ({512e6 / prompt_us:.0f} tok/s) | decode B=1 ctx~2000-2030 "
              f"graph={model._module_graph['graph'] is not None}: {us:.1f} us/token {1e6 / us:.1f} tok/s ({w8 / us / 1e3:.0f} GB/s of int8 weights) | "
              f"{torch.cuda.max_memory_allocated() / 2**30:.1f} GiB peak", flush=True)
        if name == "7B":
            _int8_old_vs_new(model, S, dev)
        del model
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()


def _time_graph(fn, reps):
    """GPU time of one fn() in us: `reps` calls captured into a CUDA graph (as the model replays decode), so host launch
    overhead is not part of the number; the graph is replayed 3 times, the median kept."""
    import torch

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    ts = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    return sorted(ts)[1]



def _w8_args(L, x, qt, sc, z, N, K, y, M=1, flags=0):
    return L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(), sz_dtype=L.B2L_BF16,
                          y=y.data_ptr(), ldy=N, M=M, N=N, K=K, prologue=0, norm_scale=None, eps=1e-5, epilogue=0, res=None, ldres=0,
                          split_k=0, flags=flags)


def sec_bench_w8_gemv():
    """gptq.int8 batch-1 kernel (b2l_w8_gemv) next to the int4 one (b2l_q4_gemv) and the generic kernel (b2l_q_linear at
    bits 8) on the same shapes, CUDA events around CUDA-graph replays in one process.  Each shape cycles through enough
    weight copies (>= 200 MB of 8-bit levels) that no call finds its weights in the 50 MB L2.  GB/s counts the weight
    bytes each kernel reads per call: N K at 8 bits, N K / 2 at 4 bits."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    shapes = [("7B c_attn", 12288, 4096), ("7B attn.c_proj", 4096, 4096), ("7B fc1|fc2", 22016, 4096), ("7B mlp.c_proj", 4096, 11008),
              ("7B lm_head", 32000, 4096), ("13B c_fc1", 13824, 5120), ("13B mlp.c_proj", 5120, 13824), ("65B c_fc1", 22016, 8192),
              ("65B mlp.c_proj", 8192, 22016)]
    for (name, N, K) in shapes:
        ncopy = max(2, -(-200_000_000 // (N * K)))
        x = torch.randn(1, K, device=dev).bfloat16()
        sc = (torch.rand(N, 1, device=dev) * 0.01 + 0.002).bfloat16()
        z = torch.randint(0, 256, (N, 1), device=dev).bfloat16()
        y = torch.empty(1, N, device=dev, dtype=torch.bfloat16)
        w8, q4, ref = [], [], []
        for i in range(ncopy):
            qw = torch.randint(0, 256, (K, N), device=dev, dtype=torch.uint8).t()     # reference layout: [K][N]
            t = torch.empty(lib.b2l_w8_tiled_i8_bytes(N, K), dtype=torch.uint8, device=dev)
            L.check(lib.b2l_w8_tile_i8(qw.data_ptr(), t.data_ptr(), N, K, L.stream_ptr()), "w8 tile")
            w8.append(t)
            t4 = torch.empty(lib.b2l_q4_tiled_i8_bytes(N, K), dtype=torch.uint8, device=dev)
            L.check(lib.b2l_q4_tile_i8(qw.data_ptr(), t4.data_ptr(), N, K, L.stream_ptr()), "q4 tile")   # any bytes: timing only
            q4.append(t4)
            if i < 2:
                ref.append(qw)
        a8 = [_w8_args(L, x, t, sc, z, N, K, y) for t in w8]
        a4 = [_w8_args(L, x, t, sc, z, N, K, y) for t in q4]
        reps = ncopy * max(1, -(-8_000_000_000 // (ncopy * N * K)))
        f8 = lambda: [lib.b2l_w8_gemv(C.byref(a8[i % ncopy]), L.stream_ptr()) for i in range(reps)]
        f4 = lambda: [lib.b2l_q4_gemv(C.byref(a4[i % ncopy]), L.stream_ptr()) for i in range(reps)]
        fg = lambda: [lib.b2l_q_linear(x.data_ptr(), K, ref[i % 2].data_ptr(), sc.data_ptr(), z.data_ptr(), L.B2L_BF16, None, y.data_ptr(),
                                       N, 1, N, K, 8, K, L.stream_ptr()) for i in range(8)]
        r8, r4 = [], []
        for _ in range(3):
            r8.append(_time_graph(f8, 1) / reps)
            r4.append(_time_graph(f4, 1) / reps)
        rg = _time_graph(fg, 1) / 8
        u8, u4 = sorted(r8)[1], sorted(r4)[1]
        print(f"{name} N={N} K={K}: w8_gemv {u8:.1f} us = {N * K / u8 / 1e3:.0f} GB/s | q4_gemv {u4:.1f} us = {N * K / 2 / u4 / 1e3:.0f} GB/s "
              f"| generic bits=8 {rg:.1f} us = {N * K / rg / 1e3:.0f} GB/s (L2-warm: 2 copies)", flush=True)
        del w8, q4, ref
        torch.cuda.empty_cache()


def sec_bench_w8_gemm():
    """gptq.int8 GEMM (b2l_w8_gemm, reference-layout levels) next to the int4 GEMM (b2l_q4_gemm), the generic kernel at
    bits 8 (small M only) and torch.matmul on a dense bf16 weight, CUDA events around CUDA-graph replays, same run.
    TFLOP/s counts 2 M N K."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    for (name, N, K) in [("7B c_attn", 12288, 4096), ("7B mlp.c_proj", 4096, 11008), ("13B c_attn", 15360, 5120), ("13B mlp.c_proj", 5120, 13824)]:
        qw = torch.randint(0, 256, (K, N), device=dev, dtype=torch.uint8).t()
        sc = (torch.rand(N, 1, device=dev) * 0.01 + 0.002).bfloat16()
        z = torch.randint(0, 256, (N, 1), device=dev).bfloat16()
        q4 = torch.empty(lib.b2l_q4_tiled_bytes(N, K), dtype=torch.uint8, device=dev)
        L.check(lib.b2l_q4_tile(qw.data_ptr(), q4.data_ptr(), N, K, L.stream_ptr()), "q4 tile")   # any bytes: timing only
        wd = torch.randn(N, K, device=dev).bfloat16()
        for M in (2, 8, 64, 512, 4096):
            x = torch.randn(M, K, device=dev).bfloat16()
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            a8, a4 = _w8_args(L, x, qw, sc, z, N, K, y, M=M), _w8_args(L, x, q4, sc, z, N, K, y, M=M)
            it = 20 if M <= 64 else 4
            u8 = _time_graph(lambda: L.check(lib.b2l_w8_gemm(C.byref(a8), L.stream_ptr()), "w8 gemm"), it)
            u4 = _time_graph(lambda: L.check(lib.b2l_q4_gemm(C.byref(a4), L.stream_ptr()), "q4 gemm"), it)
            ut = _time_graph(lambda: torch.matmul(x, wd.t()), it)
            gen = ""
            if M <= 8:
                ug = _time_graph(lambda: lib.b2l_q_linear(x.data_ptr(), K, qw.data_ptr(), sc.data_ptr(), z.data_ptr(), L.B2L_BF16, None,
                                                          y.data_ptr(), N, M, N, K, 8, K, L.stream_ptr()), it)
                gen = f" | generic bits=8 {ug:.1f} us"
            op = 2.0 * M * N * K
            print(f"{name} N={N} K={K} M={M}: w8_gemm {u8:.1f} us = {op / u8 / 1e6:.1f} TFLOP/s | q4_gemm {u4:.1f} us = {op / u4 / 1e6:.1f} "
                  f"TFLOP/s | torch.matmul bf16 {ut:.1f} us = {op / ut / 1e6:.1f} TFLOP/s{gen}", flush=True)
        del qw, q4, wd
        torch.cuda.empty_cache()


def _random_w8_model(name, dev, seed=0, n_layer=None, bits=8):
    """A gptq.int8 (bits = 4: gptq.int4) LLaMA at `name`'s widths (`n_layer` blocks if given) with random per-row
    levels, zeros and scales.  The scales give every linear a gain of about one (rms (level - zero) is about 76 at 8
    bits, 4.6 at 4), as in a trained model: with larger gains the attention scores saturate and the softmax turns
    rounding differences into different outputs."""
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200.quantization import ColBlockQuantizedLinear, weights_changed
    from lit_llama_b200.utils import quantization

    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("gptq.int8" if bits == 8 else "gptq.int4"):
            cfg = P.LLaMAConfig.from_name(name)
            if n_layer is not None:
                cfg.n_layer = n_layer
            model = P.LLaMA(cfg)
    finally:
        torch.set_default_dtype(prev)
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, ColBlockQuantizedLinear):
                m.quant_weight.copy_(torch.randint(0, 256, m.quant_weight.shape, generator=g, device=dev, dtype=torch.uint8))
                rms, zlo, zhi = (76, 96, 160) if bits == 8 else (4.6, 6, 10)
                m.scales.copy_((torch.rand(m.scales.shape, generator=g, device=dev) + 0.5) / (rms * m.in_features ** 0.5))
                m.zeros.copy_(torch.randint(zlo, zhi, m.zeros.shape, generator=g, device=dev))
            elif isinstance(m, P.RMSNorm):
                m.scale.fill_(1)
        model.transformer.wte.weight.normal_(0, 1, generator=g)
    weights_changed()
    return model.eval()


def _generic_forward(self, inp):
    """ColBlockQuantizedLinear.forward of the parent commit for gptq.int8: every call on the generic kernel."""
    import torch
    from lit_llama_b200 import _lib as L

    x = inp.reshape(-1, inp.shape[-1]).contiguous()
    y = torch.empty((x.shape[0], self.out_features), device=inp.device, dtype=inp.dtype)
    qw = self.reference_quant_weight()
    L.check(L.lib().b2l_q_linear(x.data_ptr(), x.stride(0), qw.data_ptr(), self.scales.data_ptr(), self.zeros.data_ptr(),
                                 L.sz_dtype_of(self.scales), None, y.data_ptr(), self.out_features, x.shape[0], self.out_features,
                                 self.in_features, self.bits, self.tile_cols, L.stream_ptr()), "b2l_q_linear")
    return y.reshape(*inp.shape[:-1], self.out_features)


def _w8_exact_anchor(dev, n_layer=4, T=16, steps=4, S=64):
    """Which path is nearer the exact result: the first `n_layer` blocks of a random 7B gptq.int8 model, a T-token
    prompt and `steps` decode steps, on the fused step and on the parent's path (generic kernel), both against the
    oracle with exact linears (fp64 dequantisation and accumulation, one rounding to bf16; every other op with the
    reference's bf16 rounding points).  Prints the largest normwise logit distance over the steps."""
    import torch
    from lit_llama_b200.quantization import ColBlockQuantizedLinear
    from oracle import llama_oracle as O

    model = _random_w8_model("7B", dev, seed=9, n_layer=n_layer)
    cfg = model.config
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    oracle = O.OracleLLaMA.from_state_dict(sd, n_layer, cfg.n_head, cfg.block_size, "gptq.int8", exact_linears=True)
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(0, 32000, (1, T), generator=g)
    toks = torch.randint(0, 32000, (steps,), generator=g).tolist()

    def run(fwd):
        fwd.reset_cache()
        dv = "cpu" if fwd is oracle else dev
        out = [fwd.forward(prompt.to(dv), S, torch.arange(T, device=dv))[:, -1]]
        for i, t in enumerate(toks):
            out.append(fwd.forward(torch.tensor([[t]], device=dv), S, torch.tensor([T + i], device=dv)).reshape(1, -1))
        return [o.float().cpu() for o in out]

    new_forward = ColBlockQuantizedLinear.forward
    with torch.no_grad():
        want = run(oracle)
        fused = run(model)
        assert model._decode is not None
        try:
            ColBlockQuantizedLinear.forward = _generic_forward
            model._fast_ok = False
            generic = run(model)
        finally:
            ColBlockQuantizedLinear.forward = new_forward
            model._fast_ok = None
    d = lambda a, b: max(float((x - y).norm() / y.norm()) for x, y in zip(a, b))
    print(f"  7B widths, {n_layer} blocks, {T}-token prompt + {steps} decode steps, logits against the oracle with exact linears: "
          f"fused step {d(fused, want):.2e} | parent path (generic kernel) {d(generic, want):.2e} | between the two "
          f"{d(fused, generic):.2e}", flush=True)
    del model
    gc.collect()
    torch.cuda.empty_cache()


def sec_bench_step_w8():
    """--quantize gptq.int8 at 7B, 13B, 30B and 65B (random levels, compacted: one resident copy): a 512-token prompt (the
    wgmma GEMM) and batch-1 decode at ctx ~2000 (the fused step, CUDA graph).  B2L_W8_SIZES picks the sizes.  For 7B
    the fused step is alternated with the parent's path (module by module on the generic kernel) before compaction, and
    both are compared with an exact evaluation of the first blocks (_w8_exact_anchor)."""
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    dev = torch.device("cuda")
    print(_card(), flush=True)
    S = 2048
    for name in os.environ.get("B2L_W8_SIZES", "7B,13B,30B,65B").split(","):
        model = _random_w8_model(name, dev, seed=8)
        model.copy_logits = False
        if name == "7B":
            new_forward = ColBlockQuantizedLinear.forward
            us = {"fused": [], "generic": []}
            logits = {}
            try:
                for _ in range(2):
                    for kind in ("fused", "generic"):
                        ColBlockQuantizedLinear.forward = new_forward if kind == "fused" else _generic_forward
                        model.reset_cache()
                        model._fast_ok = None if kind == "fused" else False
                        model._module_graph = None
                        torch.manual_seed(0)   # the same tokens at the same positions: the KV caches agree
                        us[kind].append(_decode_us(model, 1, S, dev, p0=2000, n=24))
                        with torch.no_grad():
                            logits[kind] = model(torch.tensor([[1234]], device=dev, dtype=torch.int32), S,
                                                 torch.tensor([2040], device=dev)).float().clone()
            finally:
                ColBlockQuantizedLinear.forward = new_forward
                model._fast_ok = None
            a, b = logits["fused"], logits["generic"]
            print(f"  7B decode B=1, alternated: fused step {' '.join(f'{v:.1f}' for v in us['fused'])} us/token | parent path (generic "
                  f"kernel) {' '.join(f'{v:.1f}' for v in us['generic'])} us/token | logits rel. diff {float((a - b).norm() / b.norm()):.2e}",
                  flush=True)
            model.reset_cache()
            _w8_exact_anchor(dev)
        model.compact()
        torch.cuda.reset_peak_memory_stats()
        levels = sum(m.out_features * m.in_features for m in model.modules() if isinstance(m, ColBlockQuantizedLinear))
        idx = torch.randint(0, 32000, (1, 512), device=dev, dtype=torch.int32)
        with torch.no_grad():
            prompt_us = _time(lambda: model(idx, S, torch.arange(512, device=dev)), iters=3, warm=1)
            model.reset_cache()
            us = _decode_us(model, 1, S, dev, p0=2000, n=24)
        print(f"{name} gptq.int8: prompt 512 tokens {prompt_us / 1e3:.2f} ms | decode B=1 ctx~2000-2030 fused="
              f"{model._decode is not None and model._decode.graph is not None}: {us:.1f} us/token {1e6 / us:.1f} tok/s "
              f"({levels / us / 1e3:.0f} GB/s of levels) | {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB peak", flush=True)
        del model
        gc.collect()   # a compacted model's c_fc1 / c_fc2 refer back to it (their layout source): a cycle
        torch.cuda.empty_cache()


def sec_bench_q8_gemm():
    """The llm.int8 GEMM (b2l_q8_gemm) against the per-row loop it replaced (b2l_q8_outlier_mask + M x b2l_q8_gemv with
    the batch mask) and torch.matmul on a dense bf16 weight of the same shape, CUDA events around CUDA-graph replays, same
    run.  TOP/s counts
    2 M N K int8 operations per call (the bf16 matmul does the same count in FLOP)."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    for (name, N, K) in [("7B c_attn", 12288, 4096), ("7B mlp.c_proj", 4096, 11008), ("13B c_fc1", 13824, 5120), ("13B mlp.c_proj", 5120, 13824)]:
        cb = torch.randint(-127, 128, (N, K), device=dev, dtype=torch.int8)
        scb = torch.rand(N, device=dev) * 0.2 + 0.01
        wt = torch.empty(lib.b2l_q8_tiled_bytes(N, K), dtype=torch.uint8, device=dev)
        L.check(lib.b2l_q8_tile(cb.data_ptr(), wt.data_ptr(), N, K, L.stream_ptr()), "tile")
        wd = torch.randn(N, K, device=dev).bfloat16()
        for M in (2, 8, 64, 512, 4096):
            x = torch.randn(M, K, device=dev).bfloat16()
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            nbytes = lib.b2l_q8_gemm_workspace_bytes(M, K)
            work = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            mask = torch.empty(K // 32, dtype=torch.int32, device=dev)
            gemm = lambda: L.check(lib.b2l_q8_gemm(x.data_ptr(), K, cb.data_ptr(), scb.data_ptr(), work.data_ptr(), nbytes, y.data_ptr(), N,
                                                   M, N, K, 6.0, 0, L.stream_ptr()), "gemm")

            def loop():
                lib.b2l_q8_outlier_mask(x.data_ptr(), K, M, K, 6.0, mask.data_ptr(), L.stream_ptr())
                for m in range(M):
                    lib.b2l_q8_gemv(x[m].data_ptr(), wt.data_ptr(), cb.data_ptr(), scb.data_ptr(), mask.data_ptr(), y[m].data_ptr(),
                                    N, K, 6.0, 0, L.stream_ptr())

            it = 20 if M <= 64 else 4
            us_g = _time_graph(gemm, it)
            us_l = _time_graph(loop, it if M <= 64 else 1)
            us_t = _time_graph(lambda: torch.matmul(x, wd.t()), it)
            op = 2.0 * M * N * K
            print(f"{name} N={N} K={K} M={M}: gemm {us_g:.1f} us = {op / us_g / 1e6:.1f} TOP/s | per-row loop {us_l:.1f} us "
                  f"({us_l / us_g:.1f}x the gemm) | torch.matmul bf16 {us_t:.1f} us = {op / us_t / 1e6:.1f} TFLOP/s", flush=True)
        del cb, wt, wd
        torch.cuda.empty_cache()


def sec_bench_q8_gemv():
    """The batch-1 llm.int8 kernel from its two weight sources: b2l_q8_gemv on the re-tiled copy against b2l_q8_gemv_cb on
    CB itself, CUDA events around CUDA-graph replays, alternated in one process (5 rounds, each number is the median of 3
    replays).  Each shape cycles through enough weight copies (>= 200 MB) that no call finds its weights in the 50 MB L2,
    as in a decode step.  GB/s counts the int8 weight bytes N K per call.  The input row has three outlier columns."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    shapes = [("7B c_attn", 12288, 4096), ("7B attn.c_proj", 4096, 4096), ("7B c_fc1", 11008, 4096), ("7B mlp.c_proj", 4096, 11008),
              ("7B lm_head", 32000, 4096), ("13B c_fc1", 13824, 5120), ("13B mlp.c_proj", 5120, 13824), ("30B c_fc1", 17920, 6656),
              ("30B mlp.c_proj", 6656, 17920), ("65B c_fc1", 22016, 8192), ("65B mlp.c_proj", 8192, 22016)]
    for (name, N, K) in shapes:
        ncopy = max(2, -(-200_000_000 // (N * K)))
        cbs = [torch.randint(-127, 128, (N, K), device=dev, dtype=torch.int8) for _ in range(ncopy)]
        scbs = [torch.rand(N, device=dev) * 0.2 + 0.01 for _ in range(ncopy)]
        wts = []
        for cb in cbs:
            wts.append(torch.empty(lib.b2l_q8_tiled_bytes(N, K), dtype=torch.uint8, device=dev))
            L.check(lib.b2l_q8_tile(cb.data_ptr(), wts[-1].data_ptr(), N, K, L.stream_ptr()), "tile")
        x = torch.randn(K, device=dev)
        x[[7, K // 3, K - 5]] = torch.tensor([9.0, -7.5, 6.5], device=dev)
        x = x.bfloat16()
        ys = [torch.empty(N, device=dev, dtype=torch.bfloat16) for _ in range(ncopy)]
        y2 = [torch.empty(N, device=dev, dtype=torch.bfloat16) for _ in range(ncopy)]
        reps = ncopy * max(1, -(-8_000_000_000 // (ncopy * N * K)))   # >= 8 GB of weights per replay

        def tiled():
            for i in range(reps):
                c = i % ncopy
                lib.b2l_q8_gemv(x.data_ptr(), wts[c].data_ptr(), cbs[c].data_ptr(), scbs[c].data_ptr(), None, ys[c].data_ptr(), N, K, 6.0, 0,
                                L.stream_ptr())

        def direct():
            for i in range(reps):
                c = i % ncopy
                lib.b2l_q8_gemv_cb(x.data_ptr(), cbs[c].data_ptr(), scbs[c].data_ptr(), None, y2[c].data_ptr(), N, K, 6.0, 0, L.stream_ptr())

        tiled()
        direct()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(ys, y2)), name
        t_t, t_c = [], []
        for _ in range(5):
            t_t.append(_time_graph(tiled, 1) / reps)
            t_c.append(_time_graph(direct, 1) / reps)
        med = lambda v: sorted(v)[len(v) // 2]
        fmt = lambda v: " ".join(f"{u:.2f}" for u in v)
        print(f"{name} N={N} K={K} ({ncopy} copies): tiled {med(t_t):.2f} us = {N * K / med(t_t) / 1e3:.0f} GB/s [{fmt(t_t)}] | "
              f"CB direct {med(t_c):.2f} us = {N * K / med(t_c) / 1e3:.0f} GB/s [{fmt(t_c)}] | CB/tiled {med(t_c) / med(t_t):.3f}", flush=True)
        del cbs, scbs, wts, ys, y2
        torch.cuda.empty_cache()


def sec_bench_step_adapter():
    """LLaMA-Adapter on the fused step: 7B gptq.int4 synthetic weights compacted, batch-1 decode at ctx ~2000 under the
    graph, with a random adapter (aT = 10, start layer 2, non-zero gates) against the same weights without it,
    alternated in one process.  The prefix term runs inside the fused attention launch (5 n_layer + 3 launches)."""
    import ctypes

    import torch
    import lit_llama_b200 as P
    from lit_llama_b200 import adapter as PA
    from lit_llama_b200.utils import quantization
    from bench import build_synthetic_model, synth_state

    dev = torch.device("cuda")
    sd = synth_state("7B", 1234, dev)
    plain = build_synthetic_model("7B", dev, state=sd).compact()
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("gptq.int4"):
            ada = PA.LLaMA.from_name("7B")
    finally:
        torch.set_default_dtype(prev)
    g = torch.Generator(device=dev).manual_seed(7)
    with torch.no_grad():
        own = ada.state_dict()
        for k, v in sd.items():
            own[k].copy_(v)
        for blk in ada.transformer.h[ada.config.adapter_start_layer:]:
            blk.attn.adapter_wte.weight.copy_(torch.randn(blk.attn.adapter_wte.weight.shape, generator=g, device=dev))
            blk.attn.gating_factor.copy_((torch.rand(blk.attn.gating_factor.shape, generator=g, device=dev) + 0.5))
    del sd, own
    ada = ada.eval().compact()
    torch.cuda.empty_cache()
    S = 2048
    for m in (plain, ada):
        m.copy_logits = False
        with torch.no_grad():
            m(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
    lib = P._lib.lib()
    res = {"plain": [], "adapter": []}
    for r in range(4):
        for name, m in (("plain", plain), ("adapter", ada)):
            res[name].append(_decode_us(m, 1, S, dev, p0=1960, n=24))
            if r == 0:
                n = lib.b2l_decode_step_launches(ctypes.byref(m._decode.args))
                print(f"{name}: fused step {m._decode is not None}, graph {m._decode.graph is not None}, {n} launches", flush=True)
    a, b = min(res["plain"]), min(res["adapter"])
    print(f"7B gptq.int4 compacted, batch 1, ctx ~1966-1990, graph + PDL on {_card()}")
    print(f"  plain   : {' '.join(f'{x:.1f}' for x in res['plain'])} us/token (best {a:.1f})")
    print(f"  adapter : {' '.join(f'{x:.1f}' for x in res['adapter'])} us/token (best {b:.1f})  -> {100 * (b - a) / a:+.2f} %")


def sec_bench_step_adapter_v2():
    """LLaMA-Adapter v2 on the fused step: 7B gptq.int4 (synth_state) and 7B gptq.int8 (_random_w8_model) weights,
    compacted, batch-1 decode at ctx ~2000 under the graph.  On the same base weights: the plain model, the v1-adapter
    model (aT = 10, start layer 2, non-zero gates) and the v2 model (the same prefix plus a non-trivial scale and bias
    on every linear), alternated in one process over 4 rounds.  The affine runs inside each linear's launch."""
    import ctypes

    import torch
    import lit_llama_b200 as P
    from lit_llama_b200 import adapter as PA
    from lit_llama_b200 import adapter_v2 as PV
    from lit_llama_b200.quantization import weights_changed
    from lit_llama_b200.utils import quantization
    from bench import build_synthetic_model, synth_state

    dev = torch.device("cuda")
    print(_card(), flush=True)
    S = 2048
    for mode in ("gptq.int4", "gptq.int8"):
        if mode == "gptq.int4":
            sd = synth_state("7B", 1234, dev)
            plain = build_synthetic_model("7B", dev, state=sd)
        else:
            plain = _random_w8_model("7B", dev, seed=8)
            sd = {k: v.clone() for k, v in plain.state_dict().items()}

        def adapter_model(v2):
            prev = torch.get_default_dtype()
            torch.set_default_dtype(torch.bfloat16)
            try:
                with torch.device(dev), quantization(mode):
                    m = PA.LLaMA.from_name("7B")
                    if v2:
                        PV.add_adapter_v2_parameters_to_linear_layers(m)
            finally:
                torch.set_default_dtype(prev)
            g = torch.Generator(device=dev).manual_seed(7)
            with torch.no_grad():
                own = m.state_dict()
                for k, v in sd.items():
                    own[k].copy_(v)
                for blk in m.transformer.h[m.config.adapter_start_layer:]:
                    blk.attn.adapter_wte.weight.copy_(torch.randn(blk.attn.adapter_wte.weight.shape, generator=g, device=dev))
                    blk.attn.gating_factor.copy_(torch.rand(blk.attn.gating_factor.shape, generator=g, device=dev) + 0.5)
                for lin in m.modules():
                    if hasattr(lin, "adapter_scale"):
                        lin.adapter_scale.copy_(torch.rand(lin.adapter_scale.shape, generator=g, device=dev) * 0.2 + 0.9)
                        lin.adapter_bias.copy_(torch.randn(lin.adapter_bias.shape, generator=g, device=dev) * 0.01)
            weights_changed()
            return m.eval().compact()

        models = {"plain": plain.compact(), "v1": adapter_model(False), "v2": adapter_model(True)}
        del sd
        torch.cuda.empty_cache()
        for m in models.values():
            m.copy_logits = False
            with torch.no_grad():
                m(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
        lib = P._lib.lib()
        res = {k: [] for k in models}
        for r in range(4):
            for name, m in models.items():
                res[name].append(_decode_us(m, 1, S, dev, p0=1960, n=24))
                if r == 0:
                    n = lib.b2l_decode_step_launches(ctypes.byref(m._decode.args))
                    print(f"{mode} {name}: fused step {m._decode is not None}, graph {m._decode.graph is not None}, {n} launches",
                          flush=True)
        best = {k: min(v) for k, v in res.items()}
        print(f"7B {mode} compacted, batch 1, ctx ~1966-1990, graph + PDL on {_card()}")
        for name in models:
            print(f"  {name:5s}: {' '.join(f'{x:.1f}' for x in res[name])} us/token (best {best[name]:.1f}, "
                  f"{100 * (best[name] - best['plain']) / best['plain']:+.2f} % vs plain, "
                  f"{100 * (best[name] - best['v1']) / best['v1']:+.2f} % vs v1)", flush=True)
        del models, plain
        gc.collect()
        torch.cuda.empty_cache()


def _lora_7b(dev):
    """7B gptq.int4 synthetic weights, compacted, without and with a random r = 8 LoRA on q and v in all 32 layers
    (alpha 16, non-zero lora_B): (plain, lora) on the same base weights."""
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200 import lora as PL
    from lit_llama_b200.utils import quantization
    from bench import build_synthetic_model, synth_state

    sd = synth_state("7B", 1234, dev)
    plain = build_synthetic_model("7B", dev, state=sd).compact()
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("gptq.int4"), PL.lora(r=8, alpha=16, dropout=0.05):
            lm = P.LLaMA.from_name("7B")
    finally:
        torch.set_default_dtype(prev)
    g = torch.Generator(device=dev).manual_seed(7)
    with torch.no_grad():
        own = lm.state_dict()
        for k, v in sd.items():
            own[k].copy_(v)
        for blk in lm.transformer.h:
            c = blk.attn.c_attn
            c.lora_A.copy_((torch.rand(c.lora_A.shape, generator=g, device=dev) * 2 - 1) / 64)
            c.lora_B.copy_(torch.randn(c.lora_B.shape, generator=g, device=dev) * 0.05)
    del sd, own
    lm = lm.eval().compact()
    torch.cuda.empty_cache()
    return plain, lm


def sec_bench_step_lora():
    """LoRA on the fused step: 7B gptq.int4 synthetic weights compacted, batch-1 decode at ctx ~2000 under the graph,
    with a random r = 8 LoRA on q and v in all 32 layers (alpha 16, non-zero lora_B) against the same weights without
    it, alternated in one process; then a 512-token prompt with and without it.  The LoRA model's step is one launch
    per layer longer (5 n_layer + 3 + n_layer)."""
    import ctypes
    import time

    import torch
    import lit_llama_b200 as P

    dev = torch.device("cuda")
    plain, lm = _lora_7b(dev)
    S = 2048
    for m in (plain, lm):
        m.copy_logits = False
        with torch.no_grad():
            m(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
    lib = P._lib.lib()
    res = {"plain": [], "lora": []}
    for r in range(4):
        for name, m in (("plain", plain), ("lora", lm)):
            res[name].append(_decode_us(m, 1, S, dev, p0=1960, n=24))
            if r == 0:
                n = lib.b2l_decode_step_launches(ctypes.byref(m._decode.args))
                print(f"{name}: fused step {m._decode is not None}, graph {m._decode.graph is not None}, {n} launches", flush=True)
    a, b = min(res["plain"]), min(res["lora"])
    card = _card()
    print(f"7B gptq.int4 compacted, batch 1, ctx ~1966-1990, graph + PDL on {card}")
    print(f"  plain : {' '.join(f'{x:.1f}' for x in res['plain'])} us/token (best {a:.1f})")
    print(f"  lora  : {' '.join(f'{x:.1f}' for x in res['lora'])} us/token (best {b:.1f})  -> {100 * (b - a) / a:+.2f} %, "
          f"{(b - a) / 32:.2f} us per layer")
    prompt = torch.randint(0, 32000, (1, 512), device=dev, dtype=torch.int32)
    pres = {"plain": [], "lora": []}
    for r in range(4):
        for name, m in (("plain", plain), ("lora", lm)):
            m.reset_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                m(prompt, S, torch.arange(512, device=dev))
            torch.cuda.synchronize()
            pres[name].append((time.perf_counter() - t0) * 1e3)
    pa, pb = min(pres["plain"][1:]), min(pres["lora"][1:])
    print(f"512-token prompt on {card}: plain {' '.join(f'{x:.2f}' for x in pres['plain'])} ms (best {pa:.2f}), "
          f"lora {' '.join(f'{x:.2f}' for x in pres['lora'])} ms (best {pb:.2f}) -> {100 * (pb - pa) / pa:+.2f} %")


def sec_bench_lora_kernel():
    """b2l_lora_apply alone on the 7B c_attn shape (r = 8, q and v): GPU time per launch in a graph of back-to-back
    launches, with and without the RMSNorm prologue, over M.  Back to back, each launch waits for the previous one
    (no PDL), so this is the kernel's own latency, not the dependency link inside the step."""
    import ctypes

    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    C_, r = 4096, 8
    A = ((torch.rand(2 * r, C_, device=dev) * 2 - 1) / 64).to(torch.bfloat16)
    B = (torch.randn(2 * C_, r, device=dev) * 0.05).to(torch.bfloat16)
    sc = torch.ones(C_, device=dev, dtype=torch.bfloat16)
    spec = L.LoRA(A.data_ptr(), B.data_ptr(), 2.0, r, 3, 0b101)
    lib = L.lib()
    for M in (1, 4, 16, 512):
        x = torch.randn(M, C_, device=dev).to(torch.bfloat16)
        y = torch.zeros(M, 3 * C_, device=dev, dtype=torch.bfloat16)
        row = []
        for norm in (None, sc):
            def fn():
                lib.b2l_lora_apply(ctypes.byref(spec), x.data_ptr(), C_, None if norm is None else norm.data_ptr(), 1e-5,
                                   y.data_ptr(), 3 * C_, M, 3 * C_, C_, 0, L.stream_ptr())
            row.append(_time_graph(fn, 200))
        print(f"M={M}: {row[0]:.2f} us plain input, {row[1]:.2f} us with the RMSNorm prologue", flush=True)
    print(f"on {_card()}")


def sec_lora_timeline():
    """Where a LoRA layer's time goes in the fused step (7B gptq.int4, compacted, r = 8 on q and v, one eager step at
    ctx ~1970, PDL on): %globaltimer stamps of c_attn, the attention and c_proj of layers 4..5, the plain model and the
    LoRA model on the same weights.  The LoRA launch itself has no stamps: it sits between c_attn's end and the
    attention's wait_done."""
    import torch

    dev = torch.device("cuda")
    plain, lm = _lora_7b(dev)
    S, pos0 = 2048, 1960
    tok = torch.randint(0, 32000, (1, 1), device=dev, dtype=torch.int32)
    for name, model in (("plain", plain), ("lora", lm)):
        model.graph_after = 0
        model.copy_logits = False
        with torch.no_grad():
            model(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
            for rep in range(3):
                for i in range(3):
                    model(tok, S, torch.tensor([pos0 + i], device=dev))
                st = model._decode
                n = 5 * model.config.n_layer + 1
                tl = torch.zeros((n, 64), dtype=torch.int64, device=dev)
                tl[:, 0] = 2**62
                tl[:, 60] = 2**62
                tl[:, 61] = 2**62
                st.args.timeline = tl.data_ptr()
                model(tok, S, torch.tensor([pos0 + 3], device=dev))
                torch.cuda.synchronize()
                st.args.timeline = None
                t = tl.cpu()
                l4, l5 = 5 * 4, 5 * 5

                def us(a, b):
                    return (int(a) - int(b)) / 1e3

                print(f"{name} rep {rep}: layer 4 -> 5 start {us(t[l5, 0], t[l4, 0]):.2f} us | c_attn start->end "
                      f"{us(t[l4, 4], t[l4, 0]):.2f} | c_attn end -> attn start {us(t[l4 + 1, 0], t[l4, 4]):.2f} | "
                      f"c_attn end -> attn wait_done {us(t[l4 + 1, 1], t[l4, 4]):.2f} | attn wait_done -> end "
                      f"{us(t[l4 + 1, 4], t[l4 + 1, 1]):.2f} | attn end -> c_proj end {us(t[l4 + 2, 4], t[l4 + 1, 4]):.2f} | "
                      f"whole step {us(t[n - 1, 4], t[0, 0]):.1f} us", flush=True)
    print(f"on {_card()}")


def sec_timeline():
    """%globaltimer stamps of every launch of one eager decode step (7B): who overlaps whom."""
    import torch
    from bench import build_synthetic_model

    dev = torch.device("cuda")
    model = build_synthetic_model("7B", dev)
    S = 2048
    model.graph_after = 0
    model.copy_logits = False
    pos0 = int(os.environ.get("B2L_TL_POS", "64"))
    with torch.no_grad():
        model(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
        tok = torch.randint(0, 32000, (1, 1), device=dev, dtype=torch.int32)
        for pdl in (1, 0):
            model.decode_flags = pdl
            model._decode = None
            for i in range(3):
                model(tok, S, torch.tensor([pos0 + i], device=dev))
            st = model._decode
            n = 5 * model.config.n_layer + 1
            tl = torch.zeros((n, 64), dtype=torch.int64, device=dev)
            tl[:, 0] = 2**62
            tl[:, 60] = 2**62
            tl[:, 61] = 2**62
            st.args.timeline = tl.data_ptr()
            model(tok, S, torch.tensor([pos0 + 3], device=dev))
            torch.cuda.synchronize()
            st.args.timeline = None
            t = tl.cpu()
            names = ["c_attn", "attn", "c_proj", "fc12", "mlp_proj"]
            base = int(t[5 * 4, 0])
            print(f"--- pdl={pdl} pos={pos0 + 3}: layers 4-5, ns relative to layer 4 c_attn start; "
                  "start(min) | wait_done(max) | x_ready(max) | loop_done(max) | end(max) | x_loaded(tid0) | after_ss_bar(tid0)")
            for li in range(5 * 4, 5 * 6 + 1):
                r = [int(v) - base if int(v) not in (0, 2**62) else None for v in t[li, :7]]
                extra = ""
                if li % 5 != 1:
                    extra = f"  | x_ready min..max {int(t[li, 60]) - base}..{r[2]}  loop_done min..max {int(t[li, 61]) - base}..{r[3]}"
                if li % 5 == 1:
                    b1 = int(t[li, 0])
                    extra = "  | CTA(0,0): " + " ".join(str(int(t[li, 8 + i]) - b1) for i in range(24) if int(t[li, 8 + i]))
                print(f"  L{li // 5} {names[li % 5]:9s} {r}{extra}")
            for li in (20, 23):  # layer 4 c_attn and fc12: CTA 0 per-stage stamps
                b0 = int(t[li, 0])
                st = [(int(t[li, 8 + 2 * i]) - b0, int(t[li, 9 + 2 * i]) - b0) for i in range(12) if int(t[li, 8 + 2 * i])]
                pi = [int(t[li, 40 + i]) - b0 for i in range(12) if int(t[li, 40 + i])]
                print(f"  {names[li % 5]} CTA0: wait_done={(int(t[li, 1]) - b0)} x_ready={(int(t[li, 2]) - b0)} stages(full_seen, done)={st} tma_issue={pi}")
            tot = int(t[n - 1, 4]) - int(t[0, 0])
            print(f"  whole step (first start -> lm_head end): {tot / 1e3:.1f} us; layer 4 start -> layer 5 start: "
                  f"{(int(t[25, 0]) - int(t[20, 0])) / 1e3:.2f} us")


def sec_precision():
    """How far the batch-1 kernel's fp32 accumulation is from exact arithmetic, in bf16 ulps of the result:
    fraction of outputs that differ from the correctly rounded fp64 result, and the largest distance."""
    import torch
    from lit_llama_b200 import _lib as L

    dev = torch.device("cuda")
    for N, K in [(4096, 4096), (4096, 11008), (2048, 22016)]:
        lv, qw, sc, z = rand_q4(N, K, dev, seed=3)
        qm, qt = tile_i8(L, qw, N, K), (tile(L, qw, N, K) if K <= 11008 else None)
        g = torch.Generator(device="cpu").manual_seed(5)
        base = torch.randn(1, K, generator=g)
        spike = base.clone(); spike[0, 16 * 7 + 2] = 60.0; spike[0, 16 * 90 + 11] = -45.0
        for name, xf in [("randn", base), ("randn+0.5", base + 0.5), ("|randn|", base.abs()), ("spikes", spike)]:
            x = xf.to(dev).bfloat16()
            want = ref_linear(x, lv, sc, z)
            wb = want.float().bfloat16()
            ulp = torch.maximum(want.abs(), torch.tensor(1e-30, device=dev, dtype=torch.float64)).log2().floor().sub(7).exp2()
            y, err = gemv_call(L, x, qm, sc, z, N, K)
            assert err is None, err
            line = f"N={N} K={K} x={name:10s} gemv: differ {float((y != wb).float().mean()):.4f}  max |y-exact| {float(((y.double() - want).abs() / ulp).max()):.3f} ulp"
            if qt is not None:
                y2, err = tc_call(L, torch.cat([x, x]), qt, sc, z, N, K)
                assert err is None, err
                line += f" | wgmma: differ {float((y2[0:1] != wb).float().mean()):.4f}  max {float(((y2[0:1].double() - want).abs() / ulp).max()):.3f} ulp"
            print(line, flush=True)


def sec_bench_q8_linear():
    """b2l_q8_linear (the llm.int8 linear of the B2L_F_Q8 step) per 7B / 13B / 65B shape, next to b2l_q8_gemv_cb (the
    module path's linear) and b2l_w8_gemv (gptq.int8, the same bytes of int8 weights): us per launch (200 launches in
    a graph, PDL on for the fused kernels) and GB/s of weights streamed."""
    import ctypes

    import torch
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.int8 import quantize_rows_int8
    from lit_llama_b200.quantization import tile_i8

    dev = torch.device("cuda")
    print(_card(), flush=True)
    shapes = [("7B c_attn", 12288, 4096, 0), ("7B c_proj", 4096, 4096, 0), ("7B fc1|fc2", 11008, 4096, 1),
              ("7B mlp.c_proj", 4096, 11008, 0), ("13B c_attn", 15360, 5120, 0), ("13B fc1|fc2", 13824, 5120, 1),
              ("13B mlp.c_proj", 5120, 13824, 0), ("65B c_attn", 24576, 8192, 0), ("65B fc1|fc2", 22016, 8192, 1),
              ("65B mlp.c_proj", 8192, 22016, 0), ("lm_head", 32000, 4096, 0)]
    lib = L.lib()
    for name, N, K, glu in shapes:
        cb, scb = quantize_rows_int8(torch.randn(N, K, device=dev) * 0.05)
        cb2, scb2 = quantize_rows_int8(torch.randn(N, K, device=dev) * 0.05) if glu else (cb, scb)
        x = torch.randn(K, device=dev).bfloat16()
        g = (torch.rand(K, device=dev) + 0.5).bfloat16()
        y = torch.empty(N, device=dev, dtype=torch.bfloat16)
        a = L.Q8LinearArgs(x=x.data_ptr(), cb=cb.data_ptr(), scb=scb.data_ptr(), cb2=cb2.data_ptr(), scb2=scb2.data_ptr(),
                           y=y.data_ptr(), N=N, K=K, threshold=6.0, prologue=L.PRO_NONE if K > 8192 else L.PRO_RMSNORM,
                           norm_scale=g.data_ptr(), eps=1e-5, epilogue=L.EPI_SWIGLU if glu else L.EPI_STORE, flags=L.F_PDL)
        fused = _time_graph(lambda: lib.b2l_q8_linear(ctypes.byref(a), L.stream_ptr()), 200)
        cbs = [(cb, scb)] + ([(cb2, scb2)] if glu else [])
        module = _time_graph(lambda: [lib.b2l_q8_gemv_cb(x.data_ptr(), c.data_ptr(), s.data_ptr(), None, y.data_ptr(), N, K, 6.0, 0,
                                                         L.stream_ptr()) for c, s in cbs], 200)
        nw = N * (2 if glu else 1)
        qw = torch.randint(0, 256, (K, nw), dtype=torch.uint8, device=dev)
        qt = tile_i8(qw, nw, K, 8)
        sc, z = torch.rand(nw, device=dev).bfloat16(), torch.full((nw,), 128.0, device=dev).bfloat16()
        y2 = torch.empty(nw, device=dev, dtype=torch.bfloat16)
        w8 = None
        if K <= 24576:
            wa = L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=qt.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(), sz_dtype=0,
                                y=y2.data_ptr(), ldy=nw, M=1, N=nw, K=K, flags=L.F_PDL)
            w8 = _time_graph(lambda: lib.b2l_w8_gemv(ctypes.byref(wa), L.stream_ptr()), 200)
        gb = nw * K / 1e3
        print(f"{name:15s} N={nw:6d} K={K:6d}: q8_linear {fused:7.1f} us {gb / fused:6.0f} GB/s | q8_gemv_cb x{len(cbs)} {module:7.1f} us "
              f"{gb / module:6.0f} GB/s" + (f" | w8_gemv {w8:7.1f} us {gb / w8:6.0f} GB/s" if w8 else ""), flush=True)
        del cb, cb2, qw, qt
        torch.cuda.empty_cache()


def sec_bench_step_q8():
    """llm.int8 batch-1 decode at ctx ~2000: the B2L_F_Q8 step (LLaMA.int8_step) against the module path (both replayed
    as CUDA graphs), alternated over 3 rounds in one process, for the sizes in B2L_INT8_SIZES (default 7B,65B) and for
    7B with a LLaMA-Adapter v1 prefix (aT = 10, start layer 2).  The last token's logits must be bit-identical."""
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200 import adapter as PA
    from lit_llama_b200.utils import quantization

    dev = torch.device("cuda")
    print(_card(), flush=True)
    S = 2048
    runs = [(n, False) for n in os.environ.get("B2L_INT8_SIZES", "7B,65B").split(",")] + [("7B", True)]
    for name, adapter in runs:
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.bfloat16)
        try:
            with torch.device(dev), quantization("llm.int8"):
                if adapter:
                    model = PA.LLaMA(PA.LLaMAConfig(**dict(P.LLaMAConfig.from_name(name).__dict__, adapter_prompt_length=10,
                                                            adapter_start_layer=2)))
                    for blk in model.transformer.h:
                        if hasattr(blk.attn, "gating_factor"):
                            blk.attn.gating_factor.data.fill_(0.5)
                else:
                    model = P.LLaMA.from_name(name)
        finally:
            torch.set_default_dtype(prev)
        model.eval()
        model.copy_logits = False
        torch.cuda.reset_peak_memory_stats()
        us = {True: [], False: []}
        logits = {}
        for _ in range(3):
            for fused in (True, False):
                model.int8_step = fused
                model.reset_cache()
                with torch.no_grad():
                    model(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
                torch.manual_seed(0)
                us[fused].append(_decode_us(model, 1, S, dev, p0=2000, n=24))
                assert (model._decode is not None) == fused
                with torch.no_grad():
                    logits[fused] = model(torch.tensor([[1234]], device=dev, dtype=torch.int32), S,
                                          torch.tensor([2040], device=dev)).clone()
        fmt = lambda v: " ".join(f"{u:.1f}" for u in v)
        print(f"{name}{' adapter' if adapter else ''} llm.int8 decode B=1 ctx~2000: fused step {fmt(us[True])} us/token | module path "
              f"{fmt(us[False])} us/token | logits bit-identical: {torch.equal(logits[True], logits[False])} | "
              f"peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB", flush=True)
        del model
        torch.cuda.empty_cache()


def sec_bench_w8_batch():
    """gptq.int8 at 2..16 rows: b2l_w8_gemv_batch (resident b2l_w8_tile_i8 tiling, fused prologue / epilogue as in the
    step) at M = 2, 4, 8, 16 next to b2l_w8_gemv at M = 1 and b2l_w8_gemm (the module path's GEMM, reference-layout
    levels) at the same M, for the 7B / 13B / 65B linears.  us per launch: 200 launches in a CUDA graph, PDL on for the
    fused kernels, the weights rotated over enough copies (>= 200 MB) that no launch finds them in the 50 MB L2.  GB/s
    counts N K bytes of levels per launch (the batch kernel also reads 3 M K bytes of digits, from L2)."""
    import ctypes

    import torch
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.quantization import tile_i8

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    # (name, N, K, prologue, epilogue): fused as b2l_decode_step fuses them
    R, NO, ST, RE, SW = L.PRO_RMSNORM, L.PRO_NONE, L.EPI_STORE, L.EPI_RESIDUAL, L.EPI_SWIGLU
    shapes = [("7B c_attn", 12288, 4096, R, ST), ("7B attn.c_proj", 4096, 4096, NO, RE), ("7B fc1|fc2", 22016, 4096, R, SW),
              ("7B mlp.c_proj", 4096, 11008, NO, RE), ("7B lm_head", 32000, 4096, R, ST),
              ("13B c_attn", 15360, 5120, R, ST), ("13B attn.c_proj", 5120, 5120, NO, RE), ("13B fc1|fc2", 27648, 5120, R, SW),
              ("13B mlp.c_proj", 5120, 13824, NO, RE), ("13B lm_head", 32000, 5120, R, ST),
              ("65B c_attn", 24576, 8192, R, ST), ("65B attn.c_proj", 8192, 8192, NO, RE), ("65B fc1|fc2", 44032, 8192, R, SW),
              ("65B mlp.c_proj", 8192, 22016, NO, RE), ("65B lm_head", 32000, 8192, R, ST)]
    for name, N, K, pro, epi in shapes:
        ncopy = max(2, -(-200_000_000 // (N * K)))
        sc = (torch.rand(N, device=dev) * 0.01 + 0.002).bfloat16()
        z = torch.randint(96, 160, (N,), device=dev).bfloat16()
        g = (torch.rand(K, device=dev) + 0.5).bfloat16()
        ref = [torch.randint(0, 256, (K, N), device=dev, dtype=torch.uint8).t() for _ in range(ncopy)]
        til = [tile_i8(q, N, K, 8) for q in ref]
        n_out = N // 2 if epi == SW else N
        line = f"{name:16s} N={N:6d} K={K:6d}:"
        for M in (1, 2, 4, 8, 16):
            x = torch.randn(M, K, device=dev).bfloat16()
            y = torch.empty(M, n_out, device=dev, dtype=torch.bfloat16)
            res = torch.randn(M, N, device=dev).bfloat16()
            ws = torch.empty(max(16, lib.b2l_w8_gemv_batch_workspace_bytes(K, M)), dtype=torch.uint8, device=dev)
            fused = [L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=t.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                                    sz_dtype=L.B2L_BF16, y=y.data_ptr(), ldy=n_out, M=M, N=N, K=K, prologue=pro,
                                    norm_scale=g.data_ptr(), eps=1e-5, epilogue=epi, res=res.data_ptr(), ldres=N, flags=L.F_PDL,
                                    workspace=ws.data_ptr()) for t in til]
            fn = lib.b2l_w8_gemv if M == 1 else lib.b2l_w8_gemv_batch
            uf = _time_graph(lambda: [L.check(fn(ctypes.byref(fused[i % ncopy]), L.stream_ptr()), "w8 fused") for i in range(200)], 1) / 200
            line += f" | M={M} {'w8_gemv' if M == 1 else 'batch'} {uf:7.1f} us {N * K / uf / 1e3:5.0f} GB/s"
            if M > 1:
                yg = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
                gemm = [_w8_args(L, x, q, sc, z, N, K, yg, M=M) for q in ref]
                ug = _time_graph(lambda: [L.check(lib.b2l_w8_gemm(ctypes.byref(gemm[i % ncopy]), L.stream_ptr()), "w8 gemm")
                                          for i in range(40)], 1) / 40
                line += f" gemm {ug:7.1f} us"
        print(line, flush=True)
        del ref, til
        torch.cuda.empty_cache()


def sec_bench_step_w8_batch():
    """Batched gptq.int8 decode: the B2L_F_W8_BATCH step (LLaMA.w8_batch_step) against the module path (b2l_w8_gemm per
    linear), both replayed as CUDA graphs, at B = 1, 2, 4, 8, 16 on random-level compacted models (B2L_W8_BATCH_SIZES,
    default 7B,65B), after a 512-token prompt, alternated over 3 rounds in one process.  B = 1 runs the batch-1 step
    in both arms.  65B keeps max_seq_length at 576 so that the KV cache of 8 sequences fits beside its 62 GiB of
    weights; 16 sequences do not fit and are skipped, and 8 timed tokens per round (24 at 7B) keep the module path's
    rounds short.  Prints us per token, GB/s of levels per token, the largest
    per-row relative logits difference between the two paths and the peak memory."""
    import torch
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    dev = torch.device("cuda")
    print(_card(), flush=True)
    S = 576
    for name in os.environ.get("B2L_W8_BATCH_SIZES", "7B,65B").split(","):
        model = _random_w8_model(name, dev, seed=8)
        model.copy_logits = False
        model.compact()
        gc.collect()
        torch.cuda.empty_cache()
        levels = sum(m.out_features * m.in_features for m in model.modules() if isinstance(m, ColBlockQuantizedLinear))
        for B in (1, 2, 4, 8, 16):
            if name == "65B" and B > 8:
                print(f"{name} B={B}: skipped (the KV cache does not fit beside the weights)", flush=True)
                continue
            torch.cuda.reset_peak_memory_stats()
            us = {True: [], False: []}
            logits = {}
            g = torch.Generator(device=dev).manual_seed(B)
            prompt = torch.randint(0, 32000, (B, 512), device=dev, dtype=torch.int32, generator=g)
            for _ in range(3):
                for step in (True, False):
                    model.w8_batch_step = step
                    model.reset_cache()
                    with torch.no_grad():
                        model(prompt, S, torch.arange(512, device=dev))
                    torch.manual_seed(0)
                    us[step].append(_decode_us(model, B, S, dev, p0=512, n=8 if name == "65B" else 24))
                    assert (model._decode is not None) == (step or B == 1), (name, B, step)
                    with torch.no_grad():
                        logits[step] = model(torch.arange(B, device=dev, dtype=torch.int32).view(B, 1) + 7, S,
                                             torch.tensor([542], device=dev)).float().clone()
            a, b = logits[True].reshape(B, -1), logits[False].reshape(B, -1)
            diff = max(float((a[n] - b[n]).norm() / b[n].norm()) for n in range(B))
            fmt = lambda v: " ".join(f"{u:.0f}" for u in v)   # noqa: E731
            print(f"{name} gptq.int8 decode B={B:2d} ctx~512-542: step {fmt(us[True])} us/token "
                  f"({levels / min(us[True]) / 1e3:.0f} GB/s) | module path {fmt(us[False])} us/token | "
                  f"max row rel. diff {diff:.2e} | peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB", flush=True)
        del model
        gc.collect()
        torch.cuda.empty_cache()


def sec_bench_q4_batch():
    """gptq.int4 at 2..16 rows: b2l_q4_gemv_batch_i8 (the resident b2l_q4_tile_i8 tiling) at M = 2, 4, 8, 16 next to
    b2l_q4_gemv at M = 1 and today's batched kernels at the same M -- b2l_q4_gemv_batch (b2l_q4_tile_mma) at 2..8 and
    b2l_q4_linear_tc (b2l_q4_tile) at 9..16 -- for the 7B / 13B / 65B linears, fused as b2l_decode_step fuses them.  us
    per launch: 200 launches in a CUDA graph, PDL on, the weights rotated over enough copies (>= 200 MB of packed
    levels) that no launch finds them in the 50 MB L2.  GB/s counts N K / 2 bytes of levels per launch (the i8 batch
    kernel also reads 3 M K bytes of digits per 32-row unit from L2: 3 M / 16 bytes per byte of levels)."""
    import ctypes

    import torch
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.quantization import tile_i8

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    R, NO, ST, RE, SW = L.PRO_RMSNORM, L.PRO_NONE, L.EPI_STORE, L.EPI_RESIDUAL, L.EPI_SWIGLU
    shapes = [("7B c_attn", 12288, 4096, R, ST), ("7B attn.c_proj", 4096, 4096, NO, RE), ("7B fc1|fc2", 22016, 4096, R, SW),
              ("7B mlp.c_proj", 4096, 11008, NO, RE), ("7B lm_head", 32000, 4096, R, ST),
              ("13B c_attn", 15360, 5120, R, ST), ("13B attn.c_proj", 5120, 5120, NO, RE), ("13B fc1|fc2", 27648, 5120, R, SW),
              ("13B mlp.c_proj", 5120, 13824, NO, RE), ("13B lm_head", 32000, 5120, R, ST),
              ("65B c_attn", 24576, 8192, R, ST), ("65B attn.c_proj", 8192, 8192, NO, RE), ("65B fc1|fc2", 44032, 8192, R, SW),
              ("65B mlp.c_proj", 8192, 22016, NO, RE), ("65B lm_head", 32000, 8192, R, ST)]
    for name, N, K, pro, epi in shapes:
        nbytes = N * K // 2
        ncopy = max(2, -(-200_000_000 // nbytes))
        sc = (torch.rand(N, device=dev) * 0.01 + 0.002).bfloat16()
        z = torch.randint(6, 10, (N,), device=dev).bfloat16()
        g = (torch.rand(K, device=dev) + 0.5).bfloat16()
        ref = [torch.randint(0, 256, (K // 2, N), device=dev, dtype=torch.uint8).t() for _ in range(ncopy)]
        til = {"i8": [tile_i8(q, N, K, 4) for q in ref], "mma": [tile_mma(L, q, N, K) for q in ref],
               "tc": [tile(L, q, N, K) for q in ref]}
        n_out = N // 2 if epi == SW else N
        line = f"{name:16s} N={N:6d} K={K:6d}:"
        for M in (1, 2, 4, 8, 16):
            x = torch.randn(M, K, device=dev).bfloat16()
            y = torch.empty(M, n_out, device=dev, dtype=torch.bfloat16)
            res = torch.randn(M, N, device=dev).bfloat16()
            ws = torch.empty(max(16, lib.b2l_w8_gemv_batch_workspace_bytes(K, M), lib.b2l_q4_gemv_batch_workspace_bytes(K)),
                             dtype=torch.uint8, device=dev)

            def args(kind):
                return [L.Q4LinearArgs(x=x.data_ptr(), ldx=K, qw_tiled=t.data_ptr(), scales=sc.data_ptr(), zeros=z.data_ptr(),
                                       sz_dtype=L.B2L_BF16, y=y.data_ptr(), ldy=n_out, M=M, N=N, K=K, prologue=pro,
                                       norm_scale=g.data_ptr(), eps=1e-5, epilogue=epi, res=res.data_ptr(), ldres=N,
                                       flags=L.F_PDL, workspace=ws.data_ptr()) for t in til[kind]]

            def time_of(fn, a):
                return _time_graph(lambda: [L.check(fn(ctypes.byref(a[i % ncopy]), L.stream_ptr()), "q4 linear")
                                            for i in range(200)], 1) / 200

            if M == 1:
                u = time_of(lib.b2l_q4_gemv, args("i8"))
                line += f" | M=1 q4_gemv {u:6.1f} us {nbytes / u / 1e3:5.0f} GB/s"
                continue
            u = time_of(lib.b2l_q4_gemv_batch_i8, args("i8"))
            old, kind = (lib.b2l_q4_gemv_batch, "mma") if M <= 8 else (lib.b2l_q4_linear_tc, "tc")
            uo = time_of(old, args(kind))
            line += (f" | M={M} i8 {u:6.1f} us {nbytes / u / 1e3:5.0f} GB/s, "
                     f"{'gemv_batch' if M <= 8 else 'linear_tc'} {uo:6.1f} us")
        print(line, flush=True)
        del ref, til
        torch.cuda.empty_cache()


def sec_bench_step_q4_batch():
    """Batched gptq.int4 decode on compacted random-level models (B2L_Q4_BATCH_SIZES, default 7B,13B,65B): the
    B2L_F_Q4_BATCH_I8 step (LLaMA.q4_batch_step, the resident tilings only) against today's batched step
    (b2l_q4_gemv_batch at 2..8, b2l_q4_linear_tc at 9..16, on transient second tilings), both replayed as CUDA graphs,
    at B = 1, 2, 4, 8, 16 after a 512-token prompt, alternated over 3 rounds in one process (B = 1 runs the batch-1 step
    in both arms).  max_seq_length 576.  Prints us per token, GB/s of levels per token, the largest per-row relative
    logits difference between the two paths and each arm's peak memory.  An arm runs only where the arithmetic (weights
    + KV cache [+ today's second copy]) leaves 2 GiB of the card free; otherwise that arithmetic is printed.  65B then
    runs the new step alone at B = 8, max_seq_length 2048, and prints its peak memory and the arithmetic for today's."""
    import torch
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.quantization import ColBlockQuantizedLinear

    dev = torch.device("cuda")
    lib = L.lib()
    print(_card(), flush=True)
    total = torch.cuda.mem_get_info()[1]
    GiB = 2**30

    def second_copy(model, B):
        """Bytes of the tilings today's batched step builds beside the resident copy (b2l_q4_tile_mma at B <= 8,
        b2l_q4_tile above)."""
        size = lib.b2l_q4_tiled_mma_bytes if B <= 8 else lib.b2l_q4_tiled_bytes
        n = 0
        for blk in model.transformer.h:
            for lin in (blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_proj):
                n += size(lin.out_features, lin.in_features)
            n += size(2 * blk.mlp.c_fc1.out_features, blk.mlp.c_fc1.in_features)
        return n + size(model.lm_head.out_features, model.lm_head.in_features)

    def kv_bytes(cfg, B, S):
        return cfg.n_layer * 2 * B * cfg.n_embd * S * 2

    def run_arm(model, step, B, S, n, prompt):
        model.q4_batch_step = step
        model.reset_cache()
        # today's fc1|fc2 copies outlive its state: drop them so that each arm's peak is its own
        model._fc12_cache = {k: v for k, v in model._fc12_cache.items() if k[1] == "i8"}
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            model(prompt, S, torch.arange(prompt.shape[1], device=dev))
        torch.manual_seed(0)
        us = _decode_us(model, B, S, dev, p0=prompt.shape[1], n=n)
        assert model._decode is not None and bool(model._decode.args.flags & L.F_Q4_BATCH_I8) == (step and B > 1)
        with torch.no_grad():
            lg = model(torch.arange(B, device=dev, dtype=torch.int32).view(B, 1) + 7, S,
                       torch.tensor([prompt.shape[1] + n + 6], device=dev)).float().clone()
        return us, lg, torch.cuda.max_memory_allocated()

    for name in os.environ.get("B2L_Q4_BATCH_SIZES", "7B,13B,65B").split(","):
        model = _random_w8_model(name, dev, seed=4, bits=4)
        model.copy_logits = False
        model.compact()
        gc.collect()
        torch.cuda.empty_cache()
        cfg = model.config
        resident = torch.cuda.memory_allocated()
        extra = second_copy(model, 8)
        levels = sum(m.out_features * m.in_features // 2 for m in model.modules() if isinstance(m, ColBlockQuantizedLinear))
        print(f"{name}: resident model {resident / GiB:.2f} GiB, today's second copy {extra / GiB:.2f} GiB, "
              f"card {total / GiB:.2f} GiB", flush=True)
        S, n = 576, 8 if name == "65B" else 24
        for B in (1, 2, 4, 8, 16):
            need_new = resident + kv_bytes(cfg, B, S)
            need_old = need_new + (second_copy(model, B) if B > 1 else 0)
            arms = [a for a, need in ((True, need_new), (False, need_old)) if need + 2 * GiB <= total]
            if False not in arms:
                print(f"{name} B={B:2d}: today's step not run: {resident / GiB:.2f} GiB model + "
                      f"{kv_bytes(cfg, B, S) / GiB:.2f} GiB KV cache + {(need_old - need_new) / GiB:.2f} GiB second copy = "
                      f"{need_old / GiB:.2f} GiB > {total / GiB:.2f} GiB card - 2 GiB", flush=True)
            if not arms:
                continue
            g = torch.Generator(device=dev).manual_seed(B)
            prompt = torch.randint(0, 32000, (B, 512), device=dev, dtype=torch.int32, generator=g)
            us, logits, peak = {a: [] for a in arms}, {}, {}
            for _ in range(3):
                for a in arms:
                    u, logits[a], peak[a] = run_arm(model, a, B, S, n, prompt)
                    us[a].append(u)
            fmt = lambda v: " ".join(f"{u:.0f}" for u in v)   # noqa: E731
            line = (f"{name} gptq.int4 decode B={B:2d} ctx~512-{512 + n + 6}: i8 step {fmt(us[True])} us/token "
                    f"({levels / min(us[True]) / 1e3:.0f} GB/s), peak {peak[True] / GiB:.2f} GiB")
            if False in arms:
                a, b = logits[True].reshape(B, -1), logits[False].reshape(B, -1)
                diff = max(float((a[r] - b[r]).norm() / b[r].norm()) for r in range(B))
                line += (f" | today's step {fmt(us[False])} us/token, peak {peak[False] / GiB:.2f} GiB"
                         f" | max row rel. diff {diff:.2e}")
            print(line, flush=True)
        if name == "65B":
            B, S = 8, 2048
            need_old = resident + kv_bytes(cfg, B, S) + extra
            print(f"65B B=8 max_seq_length 2048: today's step not run: {resident / GiB:.2f} GiB model + "
                  f"{kv_bytes(cfg, B, S) / GiB:.2f} GiB KV cache + {extra / GiB:.2f} GiB second copy = "
                  f"{need_old / GiB:.2f} GiB against a {total / GiB:.2f} GiB card", flush=True)
            prompt = torch.randint(0, 32000, (B, 512), device=dev, dtype=torch.int32)
            u, _, peak = run_arm(model, True, B, S, n, prompt)
            print(f"65B gptq.int4 decode B=8 max_seq_length 2048, ctx~512-{512 + n + 6}: i8 step {u:.0f} us/token, "
                  f"peak {peak / GiB:.2f} GiB (KV cache {kv_bytes(cfg, B, S) / GiB:.2f} GiB)", flush=True)
        del model
        gc.collect()
        torch.cuda.empty_cache()


def sec_bench_q8_batch():
    """llm.int8 at 2..16 rows: b2l_q8_linear_batch (prep launch included) against the module ops it replaces
    (b2l_rmsnorm + b2l_q8_gemm [+ b2l_add | second GEMM + b2l_silu_mul]) at M = 2, 4, 8, 16, and b2l_q8_linear at M = 1,
    for the 7B / 13B / 65B linears.  us per linear: 200 launches in a CUDA graph, PDL on for the fused kernels.  The
    weights are not rotated, so a layer under 50 MB (7B c_proj) is partly served from L2.  GB/s counts the CB bytes."""
    import ctypes

    import torch
    from lit_llama_b200 import _lib as L
    from lit_llama_b200.int8 import quantize_rows_int8

    dev = torch.device("cuda")
    print(_card(), flush=True)
    shapes = [("7B c_attn", 12288, 4096, 1), ("7B c_proj", 4096, 4096, 2), ("7B fc1|fc2", 11008, 4096, 3),
              ("7B mlp.c_proj", 4096, 11008, 2), ("13B c_attn", 15360, 5120, 1), ("13B mlp.c_proj", 5120, 13824, 2),
              ("65B fc1|fc2", 22016, 8192, 3), ("65B mlp.c_proj", 8192, 22016, 2), ("lm_head", 32000, 4096, 1)]
    lib = L.lib()
    for name, N, K, kind in shapes:   # kind 1: RMSNorm + store, 2: residual, 3: RMSNorm + SwiGLU
        glu = kind == 3
        cb, scb = quantize_rows_int8(torch.randn(N, K, device=dev) * 0.05)
        cb2, scb2 = quantize_rows_int8(torch.randn(N, K, device=dev) * 0.05) if glu else (cb, scb)
        g = (torch.rand(K, device=dev) + 0.5).bfloat16()
        line = []
        for M in (1, 2, 4, 8, 16):
            x = torch.randn(M, K, device=dev).bfloat16()
            xh = torch.empty_like(x)
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            y2, h = torch.empty_like(y), torch.empty_like(y)
            res = torch.randn(M, N, device=dev).bfloat16()
            a = L.Q8LinearArgs(x=x.data_ptr(), cb=cb.data_ptr(), scb=scb.data_ptr(), cb2=cb2.data_ptr(), scb2=scb2.data_ptr(),
                               y=y.data_ptr(), N=N, K=K, threshold=6.0, prologue=L.PRO_NONE if kind == 2 else L.PRO_RMSNORM,
                               norm_scale=g.data_ptr(), eps=1e-5, res=res.data_ptr(), flags=L.F_PDL,
                               epilogue={1: L.EPI_STORE, 2: L.EPI_RESIDUAL, 3: L.EPI_SWIGLU}[kind])
            if M == 1:
                t = _time_graph(lambda: lib.b2l_q8_linear(ctypes.byref(a), L.stream_ptr()), 200)
                line.append(f"M=1 q8_linear {t:6.1f} us {N * K * (2 if glu else 1) / 1e3 / t:5.0f} GB/s")
                continue
            nb = lib.b2l_q8_linear_batch_workspace_bytes(K, M)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            new = _time_graph(lambda: lib.b2l_q8_linear_batch(ctypes.byref(a), M, ws.data_ptr(), nb, L.stream_ptr()), 200)
            gnb = lib.b2l_q8_gemm_workspace_bytes(M, K)
            gws = torch.empty(gnb, dtype=torch.uint8, device=dev)

            def module():
                src = x
                if kind != 2:
                    lib.b2l_rmsnorm(x.data_ptr(), g.data_ptr(), xh.data_ptr(), M, K, 1e-5, L.stream_ptr())
                    src = xh
                lib.b2l_q8_gemm(src.data_ptr(), K, cb.data_ptr(), scb.data_ptr(), gws.data_ptr(), gnb, y.data_ptr(), N, M, N, K, 6.0, 0,
                                L.stream_ptr())
                if glu:
                    lib.b2l_q8_gemm(src.data_ptr(), K, cb2.data_ptr(), scb2.data_ptr(), gws.data_ptr(), gnb, y2.data_ptr(), N, M, N, K,
                                    6.0, 0, L.stream_ptr())
                    lib.b2l_silu_mul(y.data_ptr(), y2.data_ptr(), h.data_ptr(), M * N, L.stream_ptr())
                elif kind == 2:
                    lib.b2l_add(res.data_ptr(), y.data_ptr(), h.data_ptr(), M * N, L.stream_ptr())
            old = _time_graph(module, 200)
            gb = N * K * (2 if glu else 1) / 1e3
            line.append(f"M={M} batch {new:6.1f} us {gb / new:5.0f} GB/s / module {old:6.1f} us")
        print(f"{name:15s} N={N:6d} K={K:6d}: " + " | ".join(line), flush=True)
        del cb, cb2
        torch.cuda.empty_cache()


def sec_bench_step_q8_batch():
    """llm.int8 batched decode at ctx ~512: the B2L_F_Q8 | B2L_F_Q8_BATCH step (LLaMA.int8_step) against the module
    path (both replayed as CUDA graphs), alternated over 2 rounds in one process, at B = 2, 4, 8, 16 for the sizes in
    B2L_INT8_SIZES (default 7B,13B).  The logits must be bit-identical."""
    import torch
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    dev = torch.device("cuda")
    print(_card(), flush=True)
    for name in os.environ.get("B2L_INT8_SIZES", "7B,13B").split(","):
        S = 1024
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.bfloat16)
        try:
            with torch.device(dev), quantization("llm.int8"):
                model = P.LLaMA.from_name(name)
        finally:
            torch.set_default_dtype(prev)
        model.eval()
        model.copy_logits = False
        for B in ((2, 4, 8) if name == "65B" else (2, 4, 8, 16)):
            torch.cuda.reset_peak_memory_stats()
            us = {True: [], False: []}
            logits = {}
            for _ in range(2):
                for fused in (True, False):
                    model.int8_step = fused
                    model.reset_cache()
                    with torch.no_grad():
                        torch.manual_seed(B)
                        model(torch.randint(0, 32000, (B, 16), device=dev, dtype=torch.int32), S, torch.arange(16, device=dev))
                    torch.manual_seed(0)
                    us[fused].append(_decode_us(model, B, S, dev, p0=512, n=16))
                    assert (model._decode is not None) == fused
                    with torch.no_grad():
                        logits[fused] = model(torch.randint(0, 32000, (B, 1), device=dev, dtype=torch.int32,
                                                            generator=torch.Generator(dev).manual_seed(1)), S,
                                              torch.tensor([600], device=dev)).clone()
            assert torch.equal(logits[True], logits[False])
            fmt = lambda v: " ".join(f"{u / 1e3:.2f}" for u in v)
            print(f"{name} llm.int8 decode B={B} max_seq_length {S}: step {fmt(us[True])} ms/token | module path {fmt(us[False])} "
                  f"ms/token | logits bit-identical | peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB", flush=True)
        del model
        torch.cuda.empty_cache()


def main():
    which = sys.argv[1:] or SECTIONS
    if len(which) == 1 and os.environ.get("B2L_DIAG_CHILD") == "1":
        globals()["sec_" + which[0]]()
        return
    for s in which:
        print(f"===== {s} =====", flush=True)
        t0 = time.time()
        env = dict(os.environ, B2L_DIAG_CHILD="1")
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), s], env=env, timeout=420, capture_output=True, text=True)
            print(r.stdout[-6000:])
            if r.returncode != 0:
                print(f"[{s}] exit code {r.returncode}\n{r.stderr[-3000:]}")
        except subprocess.TimeoutExpired as e:
            print(f"[{s}] TIMEOUT after 420 s\n{(e.stdout or b'')[-3000:]}")
        print(f"[{s}] {time.time() - t0:.1f} s", flush=True)


if __name__ == "__main__":
    main()

"""Turns the ncu outputs of a GPU run (gpurun_out/) into the text summaries committed under profiles/.

    python tools/summarize_profiles.py r01
"""
import collections
import csv
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "gpurun_out")
P = os.path.join(ROOT, "profiles")

WANT = ["Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
        "smsp__inst_executed.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]


def launch_list(tag, src, title):
    rows = list(csv.reader(open(src)))
    hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
    h = rows[hi]
    ki, vi = h.index("Kernel Name"), h.index("Metric Value")
    agg, tot = collections.OrderedDict(), 0.0
    for r in rows[hi + 1:]:
        if len(r) <= vi:
            continue
        a = agg.setdefault(r[ki].split("(")[0][:70], [0, 0.0])
        v = float(r[vi].replace(",", ""))
        a[0] += 1; a[1] += v; tot += v
    out = [f"# {title}", "# ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none",
           "# per-launch times are cold-cache and serialised (no PDL overlap): compare SHARES, not absolutes",
           f"{'launches':>8} {'total_us':>10} {'share':>7} {'avg_us':>8}  kernel"]
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        out.append(f"{n:8d} {t / 1e3:10.1f} {t / tot * 100:6.1f}% {t / n / 1e3:8.2f}  {k}")
    out.append(f"total {tot / 1e3:.1f} us over {sum(n for n, _ in agg.values())} launches")
    open(os.path.join(P, f"{tag}_launch_list_decode_step.txt"), "w").write("\n".join(out) + "\n")


def full(tag, rep, name, title):
    raw = subprocess.run(["ncu", "-i", os.path.join(G, rep), "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    h, units = rows[0], rows[1]
    lines = [f"# {title}", "# ncu --set full --clock-control none --import-source on  (one launch at a time, cold cache, no PDL overlap;",
             "# durations here are NOT bench numbers - bench.py times the kernels with CUDA events inside the pipelined step)"]
    for r in rows[2:]:
        lines.append("")
        for w in WANT:
            idx = [i for i, x in enumerate(h) if x == w]
            if idx:
                lines.append(f"{w:72s} {r[idx[0]]:>16s} {units[idx[0]]}")
        st = [i for i, x in enumerate(h) if "issue_stalled" in x and "not_issued" not in x and "ratio" in x]
        vals = sorted([(float(r[i].replace(",", "")) if r[i] else 0, h[i].replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", "")) for i in st], reverse=True)[:8]
        lines.append("warp stall reasons (warps per issue-active cycle): " + ", ".join(f"{n}={v:.2f}" for v, n in vals))
    open(os.path.join(P, f"{tag}_ncu_{name}.txt"), "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    tag = sys.argv[1] if len(sys.argv) > 1 else "r01"
    os.makedirs(P, exist_ok=True)
    if os.path.exists(os.path.join(G, "launches_r1.csv")):
        launch_list(tag, os.path.join(G, "launches_r1.csv"), "one eager decode step of LLaMA-7B gptq.int4 (tools/prof_step.py), every launch")
    for rep, name, title in [("prof_gemv.ncu-rep", "q4_gemv_kernel", "q4_gemv_kernel: c_attn, attn.c_proj, fc1|fc2, mlp.c_proj of layer 0 and c_attn of layer 1 (7B, batch 1)"),
                             ("prof_attn.ncu-rep", "attn_decode_fused_kernel", "attn_decode_fused_kernel (7B, batch 1)"),
                             ("prof_gemm.ncu-rep", "q4_gemm_kernel", "q4_gemm_kernel: wgmma prefill GEMM, 13B c_attn shape (N 15360, K 5120) at M = 4096 (tools/diag.py bench_gemm)"),
                             ("prof_q4.ncu-rep", "q4_linear_tc_kernel", "q4_linear_tc_kernel (wgmma path, M = 9..16)")]:
        if os.path.exists(os.path.join(G, rep)):
            full(tag, rep, name, title)
    print(os.listdir(P))

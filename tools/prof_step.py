"""One eager decode step of the 7B gptq.int4 model between cudaProfilerStart/Stop, for
`ncu --profile-from-start off ...` (Nsight Compute, where it is available)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import S_CTX, build_synthetic_model, sample_next  # noqa: E402

pos0 = int(os.environ.get("B2L_PROF_POS", "1024"))
dev = torch.device("cuda", 0)
model = build_synthetic_model("7B", dev)
model.graph_after = 0
model.copy_logits = False
with torch.no_grad():
    model(torch.randint(0, 32000, (1, 16), device=dev, dtype=torch.int32), S_CTX, torch.arange(16, device=dev))
    tok = torch.randint(0, 32000, (1, 1), device=dev, dtype=torch.int32)
    for i in range(3):
        tok = sample_next(model(tok.view(1, 1), S_CTX, torch.tensor([pos0 + i], device=dev))).to(torch.int32)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    tok = sample_next(model(tok.view(1, 1), S_CTX, torch.tensor([pos0 + 3], device=dev))).to(torch.int32)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
print("profiled one decode step at position", pos0 + 3)

"""CPU: perplexity evaluation (lit_llama_b200.evaluate).  The oracle's restatement of the loss against the unmodified
reference's evaluation loop (tests/golden/tiny_eval_int4.pt, oracle/make_golden_eval.py), the C layout of
b2l_nll_args and its workspace size, argument rejection before any launch, and the window slicing of perplexity()."""
import ctypes as C
import math
import os
import subprocess
import types

import pytest
import torch

from conftest import load_golden

import __graft_entry__ as entry
from oracle import llama_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def restated_nll(logits: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
    """The numerics contract of b2l_logits_nll: logsumexp over every column minus the target's logit, in fp32 from
    the maximum-subtracted exp."""
    lf = logits.float()
    mx = lf.max(dim=-1, keepdim=True).values
    lse = mx.squeeze(-1) + torch.log(torch.exp(lf - mx).sum(dim=-1))
    return lse - lf.gather(-1, targets.long().view(-1, 1)).squeeze(-1)


def test_oracle_restatement_reproduces_reference_nll():
    g = load_golden("tiny_eval_int4.pt")
    cfg = g["cfg"]
    sd = O.synth_state_dict(cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"], "gptq.int4",
                            dtype=torch.float32, seed=g["seed"])
    m = O.OracleLLaMA.from_state_dict(sd, cfg["n_layer"], cfg["n_head"], cfg["block_size"], "gptq.int4")
    blk = g["block"]
    for seq, ref in zip(g["seqs"], g["f32"]):
        n_win = 0
        for w, i in enumerate(range(0, seq.numel(), blk)):
            inp = seq[i : i + blk].view(1, -1)
            got = restated_nll(m.forward(inp)[0, :-1], inp[0, 1:])
            # the oracle's fp32 logits are within rtol 1e-4 / atol 1e-5 of the reference's (test_oracle_golden.py)
            torch.testing.assert_close(got, ref["window_nll_f32"][w], rtol=1e-4, atol=2e-4)
            assert abs(float(got.double().sum()) - float(ref["window_sums"][w])) <= 1e-5 * max(1.0, float(ref["window_sums"][w]))
            n_win += 1
        assert n_win == len(ref["window_sums"])
    # the ragged last windows: 37 tokens of the 229-token sequence, 1 token (nothing to predict) of the 129-token one
    assert [t.numel() for t in g["f32"][0]["window_nll_f32"]] == [63, 63, 63, 36]
    assert [t.numel() for t in g["f32"][1]["window_nll_f32"]] == [63, 63, 0]


def test_nll_args_layout_matches_c_compiler(L, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "b2l.h"\n'
        "int main(void){\n"
        'printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(b2l_nll_args), offsetof(b2l_nll_args, targets), '
        "offsetof(b2l_nll_args, targets_i64), offsetof(b2l_nll_args, nll), offsetof(b2l_nll_args, nll_sum), "
        "offsetof(b2l_nll_args, workspace));\n"
        "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    A = L.NLLArgs
    assert out == [C.sizeof(A), A.targets.offset, A.targets_i64.offset, A.nll.offset, A.nll_sum.offset, A.workspace.offset]


def _align16(n: int) -> int:
    return (n + 15) // 16 * 16


@pytest.mark.parametrize("M,N", [(2047, 32000), (1, 32000), (17, 130), (5, 50), (63, 128), (2048, 32001)])
def test_workspace_bytes(L, M, N):
    """(max, sum of exp) fp32 pairs per row and 128-column tile, then one fp32 target logit per row, each 16-byte
    aligned."""
    want = _align16(-(-N // 128) * M * 8) + _align16(M * 4)
    assert L.lib().b2l_nll_workspace_bytes(M, N) == want
    assert L.lib().b2l_nll_workspace_bytes(0, N) == 0 and L.lib().b2l_nll_workspace_bytes(M, 0) == 0


def test_bad_arguments_rejected_before_launch(L):
    lib = L.lib()
    p = C.c_void_p(1 << 20)   # never dereferenced: every call below is refused before any launch
    good = L.NLLArgs(targets=p, targets_i64=1, nll=p, nll_sum=p, workspace=p)
    assert lib.b2l_logits_nll(p, 100, 4, 100, None, None) == -1 and b"null nll args" in lib.b2l_last_error()
    assert lib.b2l_logits_nll(p, 99, 4, 100, C.byref(good), None) == -1 and b"bad shape" in lib.b2l_last_error()
    assert lib.b2l_logits_nll(None, 100, 4, 100, C.byref(good), None) == -1 and b"null logits" in lib.b2l_last_error()
    bad_ws = L.NLLArgs(targets=p, targets_i64=1, nll=p, nll_sum=p, workspace=C.c_void_p((1 << 20) + 8))
    assert lib.b2l_logits_nll(p, 100, 4, 100, C.byref(bad_ws), None) == -1 and b"16-byte" in lib.b2l_last_error()

    def gemm_args(**kw):
        a = L.Q4LinearArgs(x=p, ldx=4096, qw_tiled=p, scales=p, zeros=p, sz_dtype=L.B2L_BF16, y=None, ldy=0, M=17,
                           N=32000, K=4096, prologue=L.PRO_NONE, epilogue=L.EPI_STORE, flags=0)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for fn in ("b2l_q4_gemm_nll", "b2l_w8_gemm_nll"):
        f = getattr(lib, fn)
        assert f(C.byref(gemm_args()), None, None) == -1 and b"null nll args" in lib.b2l_last_error()
        assert f(C.byref(gemm_args(epilogue=L.EPI_RESIDUAL)), C.byref(good), None) == -2
        assert f(C.byref(gemm_args(prologue=L.PRO_RMSNORM)), C.byref(good), None) == -2
        assert f(C.byref(gemm_args(K=4000, ldx=4000)), C.byref(good), None) == -2   # K % 64 != 0, as b2l_q4_gemm
        assert f(C.byref(gemm_args(M=0)), C.byref(good), None) == -1
        assert f(C.byref(gemm_args()), C.byref(bad_ws), None) == -1 and b"16-byte" in lib.b2l_last_error()
    assert lib.b2l_w8_gemm_nll(C.byref(gemm_args(flags=1)), C.byref(good), None) == -2


class _StubModel:
    def __init__(self, block_size):
        self.config = types.SimpleNamespace(block_size=block_size)


def _stub_nll(calls):
    """window_nll's contract on the CPU: records each window and returns T - 1 per-token losses of (token + 1) / 7."""
    def fn(model, inp):
        assert inp.dim() == 2 and inp.size(0) == 1
        calls.append(inp[0].clone())
        nll = (inp[0, 1:].double() + 1) / 7
        return nll.float(), nll.sum()
    return fn


@pytest.mark.parametrize("n,block,cfg_block,windows", [
    (229, 64, 64, [64, 64, 64, 37]),        # ragged last window
    (129, 64, 64, [64, 64, 1]),             # a last window of one token predicts nothing
    (4096, 2048, 2048, [2048, 2048]),
    (4097, 2048, 2048, [2048, 2048, 1]),
    (1000, 100, 2, [100] * 5 + [12]),       # trimmed to 256 * block_size = 512 tokens first
])
def test_perplexity_window_slicing(n, block, cfg_block, windows):
    from lit_llama_b200.evaluate import perplexity

    seq = torch.arange(n) % 97
    calls = []
    ppl, total, toks = perplexity(_StubModel(cfg_block), seq.view(1, -1), block_size=block, nll_fn=_stub_nll(calls))
    assert [c.numel() for c in calls] == windows
    assert torch.equal(torch.cat(calls), seq[: sum(windows)])   # consecutive, non-overlapping windows
    assert toks == sum(w - 1 for w in windows)
    want = sum(float(((c[1:].double() + 1) / 7).sum()) for c in calls)
    assert total == pytest.approx(want, rel=1e-12) and ppl == pytest.approx(math.exp(want / toks), rel=1e-12)


def test_perplexity_of_reference_window_losses():
    """perplexity() over the reference's own fp32 window losses gives the reference loop's perplexity."""
    from lit_llama_b200.evaluate import perplexity

    g = load_golden("tiny_eval_int4.pt")
    for seq, ref in zip(g["seqs"], g["f32"]):
        it = iter(ref["window_nll_f32"])

        def fn(model, inp):
            nll = next(it)
            assert nll.numel() == inp.size(1) - 1
            return nll, nll.double().sum()

        ppl, total, toks = perplexity(_StubModel(g["cfg"]["block_size"]), seq, block_size=g["block"], nll_fn=fn)
        assert toks == ref["toks"]
        assert total == pytest.approx(ref["nlls"], rel=1e-6) and ppl == pytest.approx(ref["ppl"], rel=1e-6)


def test_perplexity_needs_two_tokens():
    from lit_llama_b200.evaluate import perplexity

    with pytest.raises(ValueError, match="two tokens"):
        perplexity(_StubModel(64), torch.tensor([5]), block_size=64, nll_fn=_stub_nll([]))

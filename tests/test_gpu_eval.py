"""GPU: perplexity evaluation (lit_llama_b200.evaluate).  b2l_logits_nll against torch's fp32 cross-entropy; the NLL
epilogue of the wgmma GEMMs (b2l_q4_gemm_nll / b2l_w8_gemm_nll) bit-identical to the standalone kernel on the logits
the plain GEMM writes; out-of-range targets; the tiny model's perplexity against the unmodified reference's
evaluation loop (tests/golden/tiny_eval_int4.pt); and every model kind's window_nll against model(inp) followed by the
standalone kernel."""
import dataclasses
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden

import lit_llama_b200 as P
from lit_llama_b200 import evaluate as E
from lit_llama_b200.quantization import ColBlockQuantizedLinear
from lit_llama_b200.utils import quantization

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-3, 5e-3   # the tiny model's logits against the reference's (test_gpu_model.py)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    return torch.device("cuda", 0)


def _ce(logits: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    return F.cross_entropy(logits.float(), t.long(), reduction="none")


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int64)


def _same(a, b):
    """(nll, nll_sum) pairs equal bit for bit (NaN payloads included)."""
    return torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1].view(1)), _bits(b[1].view(1)))


@pytest.mark.parametrize("i64", [False, True])
@pytest.mark.parametrize("M", [1, 17, 2047])
@pytest.mark.parametrize("N", [32000, 130, 50, 128])
def test_logits_nll_matches_torch(dev, N, M, i64):
    g = torch.Generator(device=dev).manual_seed(N * 7 + M)
    ldl = N if i64 else N + 3   # int32 targets also exercise an odd leading dimension (scalar loads)
    buf = (torch.randn(M, ldl, generator=g, device=dev) * 3).to(torch.bfloat16)
    logits = buf[:, :N]
    t = torch.randint(0, N, (M,), generator=g, device=dev, dtype=torch.int64 if i64 else torch.int32)
    nll, s = E.logits_nll(logits, t)
    torch.cuda.synchronize()
    assert nll.dtype == torch.float32 and s.dtype == torch.float64 and nll.shape == (M,)
    torch.testing.assert_close(nll, _ce(logits, t), rtol=1e-5, atol=1e-5)
    want = nll.double().sum()
    assert abs(float(s) - float(want)) <= 1e-9 * abs(float(want))


def _rand_linear(dev, bits, N, K, seed):
    """A gptq linear (one scale / zero per row, no bias) with random levels; outputs of a few units."""
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.device(dev):
        lin = ColBlockQuantizedLinear(K, N, False, bits=bits, tile_cols=-1)
    epb = 8 // bits
    lin.quant_weight.copy_(torch.randint(0, 256, (N, K // epb), generator=g, device=dev, dtype=torch.uint8))
    lv = 2 ** bits
    lin.scales = ((torch.rand(N, 1, generator=g, device=dev) + 0.5) * (8.0 / (lv * K ** 0.5))).to(torch.bfloat16)
    lin.zeros = torch.randint(lv // 2 - lv // 8, lv // 2 + lv // 8, (N, 1), generator=g, device=dev).to(torch.bfloat16)
    return lin


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("N,K,M", [(32000, 4096, 17), (32000, 4096, 128), (32000, 4096, 2047), (1000, 512, 300),
                                   (999, 512, 40)])
def test_fused_gemm_nll_bit_identical(dev, bits, N, K, M):
    """The GEMM's NLL epilogue against b2l_logits_nll on the logits the plain GEMM writes for the same T = M + 1 rows,
    before and after the layer keeps only its batch-1 tiling (what LLaMA.compact() does to lm_head)."""
    lin = _rand_linear(dev, bits, N, K, seed=N + K + M + bits)
    g = torch.Generator(device=dev).manual_seed(M)
    x = torch.randn(M + 1, K, generator=g, device=dev).to(torch.bfloat16)
    t = torch.randint(0, N, (M,), generator=g, device=dev)
    assert E._fused_kind(lin, M + 1, x) == ("w8" if bits == 8 else "q4")
    for released in (False, True):
        if released:
            lin.release_reference_layout()
        logits = lin(x)
        want = E.logits_nll(logits, t)
        got = E.lm_head_nll(lin, x, t)
        torch.cuda.synchronize()
        assert _same(got, want), (released, float((got[0] - want[0]).abs().max()))
        torch.testing.assert_close(got[0], _ce(logits[:M], t), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("path", ["standalone", "q4", "w8"])
def test_out_of_range_targets_give_nan(dev, path):
    N, K, M = 1000, 512, 300
    lin = _rand_linear(dev, 8 if path == "w8" else 4, N, K, seed=5)
    g = torch.Generator(device=dev).manual_seed(6)
    x = torch.randn(M + 1, K, generator=g, device=dev).to(torch.bfloat16)
    t = torch.randint(0, N, (M,), generator=g, device=dev)
    bad = t.clone()
    bad[[3, 100, 299]] = torch.tensor([N, -1, N + 127], device=dev)

    def run(tt):
        if path == "standalone":
            return E.logits_nll(lin(x), tt)
        return E.lm_head_nll(lin, x, tt)

    ok, nan = run(t), run(bad)
    torch.cuda.synchronize()
    where = torch.isnan(nan[0])
    assert where.nonzero().view(-1).tolist() == [3, 100, 299]
    assert torch.equal(nan[0][~where], ok[0][~where]) and torch.isnan(nan[1])


# ------------------------------------------------------------------ the tiny model
CFG = dict(block_size=64, vocab_size=96, n_layer=2, n_head=4, n_embd=128)


def test_tiny_perplexity_matches_reference(dev):
    """perplexity() of the tiny gptq.int4 model against the unmodified reference's evaluation loop run on the CPU with
    the same bf16 weights (ragged last window of 37 tokens, and a last window of 1).

    The reference's per-token losses here are its logits upcast to fp32 (reduction="none"), and its window sums are
    their fp32 sums.  The logits agree within rtol 1e-3 / atol 5e-3 (test_gpu_model.py), so a token's loss, a
    logsumexp minus one logit, is within 2 (atol + rtol max|L|) of the reference's, and a window's sum within T - 1
    times that.  The reference loop as it runs on bf16 logits takes each window's loss as a bf16 scalar, rounded
    along the way: in the fixture it is up to 2.5 (0.8 %) away from the fp32 sum of its own per-token losses.
    Against that loop the bar adds this rounding, read from the fixture.  Measured on an H100: the per-token losses
    are within 1.9e-3 of the reference's fp32 ones (bar 1.1e-2) and the window sums within 3.8e-3 (bar 0.69)."""
    from gpu_util import build_tiny

    gd = load_golden("tiny_eval_int4.pt")
    assert gd["cfg"] == CFG
    model, _, _ = build_tiny(dev, CFG)
    blk = gd["block"]
    for seq, ref in zip(gd["seqs"], gd["bf16"]):
        total, total_bar, bf16_bar, toks = 0.0, 0.0, 0.0, 0
        for w, i in enumerate(range(0, seq.numel(), blk)):
            inp = seq[i : i + blk].view(1, -1).to(dev)
            nll, s = E.window_nll(model, inp)
            logits = model(inp)[0]
            tok_bar = 2 * (ATOL + RTOL * float(logits.float().abs().max()))
            want = ref["window_nll_f32"][w]
            assert nll.shape == want.shape
            if nll.numel():
                assert float((nll.cpu() - want).abs().max()) <= tok_bar
            bar = nll.numel() * tok_bar
            assert abs(float(s) - float(want.sum())) <= bar
            loop_rounding = abs(float(ref["window_sums"][w]) - float(want.double().sum()))
            assert abs(float(s) - float(ref["window_sums"][w])) <= bar + loop_rounding
            total += float(s)
            total_bar += bar
            bf16_bar += bar + loop_rounding
            toks += nll.numel()
        ppl, nll_sum, n = P.evaluate.perplexity(model, seq.to(dev), block_size=blk)
        assert n == toks == ref["toks"]
        assert nll_sum == pytest.approx(total, rel=1e-12)
        assert abs(nll_sum - sum(float(v.sum()) for v in ref["window_nll_f32"])) <= total_bar
        assert abs(nll_sum - ref["nlls"]) <= bf16_bar            # the loop the reference scripts run on bf16
        assert abs(ppl - ref["ppl"]) <= ref["ppl"] * math.expm1(bf16_bar / n)


# ------------------------------------------------------------------ every model kind
def _build(dev, kind):
    from gpu_util import build_tiny

    if kind in ("gptq.int4", "gptq.int8", "llm.int8", "dense"):
        return build_tiny(dev, CFG, None if kind == "dense" else kind)[0]
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        if kind == "lora":
            from lit_llama_b200 import lora as PL
            from oracle import llama_oracle as O
            from oracle import lora_oracle as LO

            sd = dict(O.synth_state_dict(CFG["n_layer"], CFG["n_head"], CFG["n_embd"], CFG["vocab_size"], "gptq.int4"),
                      **LO.lora_weights(CFG["n_layer"], CFG["n_embd"], seed=4321))
            with torch.device(dev), quantization("gptq.int4"), PL.lora(r=8, alpha=16, dropout=0.05):
                model = P.LLaMA(P.LLaMAConfig(**CFG))
        else:
            from lit_llama_b200 import adapter as PA
            from lit_llama_b200 import adapter_v2 as PV
            from oracle import adapter_oracle as A
            from oracle import adapter_v2_oracle as A2

            cfg = dict(CFG, adapter_prompt_length=10, adapter_start_layer=1)
            args = (cfg["n_layer"], cfg["n_head"], cfg["n_embd"], cfg["vocab_size"], "gptq.int4", 10, 1)
            sd = A.adapter_state_dict(*args) if kind == "adapter" else A2.adapter_v2_state_dict(*args)
            with torch.device(dev), quantization("gptq.int4"):
                model = PA.LLaMA(PA.LLaMAConfig(**cfg))
                if kind == "adapter_v2":
                    PV.add_adapter_v2_parameters_to_linear_layers(model)
    finally:
        torch.set_default_dtype(prev)
    res = model.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    return model.eval()


@pytest.mark.parametrize("kind", ["gptq.int4", "gptq.int8", "llm.int8", "dense", "lora", "adapter", "adapter_v2"])
def test_window_nll_equals_model_logits_nll(dev, kind):
    model = _build(dev, kind)
    if kind == "adapter_v2":   # lm_head's own scale and bias are far from the identity
        assert float((model.lm_head.adapter_scale.detach().float().abs() - 1).abs().max()) > 0.1
    g = torch.Generator().manual_seed(len(kind))
    V = CFG["vocab_size"]
    for T in (64, 40, 9, 2, 1):
        inp = torch.randint(0, V, (1, T), generator=g).to(dev)
        with torch.no_grad():
            before = model(inp)
        got = E.window_nll(model, inp)
        with torch.no_grad():
            after = model(inp)
        want = E.logits_nll(before[0], inp[0, 1:])
        torch.cuda.synchronize()
        assert torch.equal(before, after), (kind, T)
        assert _same(got, want), (kind, T)
        torch.testing.assert_close(got[0], _ce(before[0, :-1], inp[0, 1:]), rtol=1e-5, atol=1e-5)
        if T == 1:
            assert got[0].numel() == 0 and float(got[1]) == 0.0
    fused = E._fused_kind(model.lm_head, 40, torch.empty(40, CFG["n_embd"], device=dev, dtype=torch.bfloat16))
    assert fused == {"gptq.int4": "q4", "gptq.int8": "w8", "lora": "q4", "adapter": "q4"}.get(kind)


def test_window_nll_after_compact(dev):
    model = _build(dev, "gptq.int4")
    inp = torch.randint(0, CFG["vocab_size"], (1, 64), generator=torch.Generator().manual_seed(3)).to(dev)
    before = E.window_nll(model, inp)
    model.compact()
    after = E.window_nll(model, inp)
    with torch.no_grad():
        want = E.logits_nll(model(inp)[0], inp[0, 1:])
    torch.cuda.synchronize()
    assert _same(before, after) and _same(after, want)


def test_cli_on_a_local_text_file(dev, tmp_path, capsys):
    """python -m lit_llama_b200.evaluate --text_path: a synthetic checkpoint and a stand-in tokenizer (the
    sentencepiece model is not part of the repository), through main()'s loading and printing."""
    import sys
    import types

    from oracle import llama_oracle as O

    sd = O.synth_state_dict(1, 32, 4096, 32000, "gptq.int4")   # 7B-shaped width (model lookup), one layer
    ck = tmp_path / "lit-llama.pth"
    torch.save(sd, ck)
    tok = tmp_path / "tokenizer.model"
    tok.write_bytes(b"")
    text = tmp_path / "text.txt"
    text.write_text("the quick brown fox " * 300)

    class _SP:
        def __init__(self, model_file):
            pass

        def bos_id(self):
            return 1

        def encode(self, s):
            return [3 + (ord(c) * 31 + i) % 31000 for i, c in enumerate(s)]

    stub = types.ModuleType("sentencepiece")
    stub.SentencePieceProcessor = _SP
    prev = sys.modules.get("sentencepiece")
    sys.modules["sentencepiece"] = stub
    orig = P.LLaMAConfig.from_name.__func__

    def one_layer(cls, name):
        return dataclasses.replace(orig(cls, name), n_layer=1)

    P.LLaMAConfig.from_name = classmethod(one_layer)
    try:
        E.cli(["--kind", "full", "--quantize", "gptq.int4", "--checkpoint_path", str(ck), "--tokenizer_path", str(tok),
               "--text_path", str(text)])
    finally:
        P.LLaMAConfig.from_name = classmethod(orig)
        if prev is None:
            del sys.modules["sentencepiece"]
        else:
            sys.modules["sentencepiece"] = prev
    out = capsys.readouterr()
    line = [ln for ln in out.out.splitlines() if ln.startswith("Perplexity on text.txt: ")]
    assert len(line) == 1 and float(line[0].split(": ")[1]) > 1.0, out.out
    assert "Memory used" in out.err

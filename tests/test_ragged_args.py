"""CPU: the ragged prefill is refused where it cannot run, before the device is touched, and the packing rule.

b2l_attention_ragged returns B2L_E_ARG for null pointers, bad shapes, n_seq outside 1..16, a length outside 1..S, starts
that do not tile [0, N) in order, a row outside the cache and two sequences naming one row, and B2L_E_UNSUPPORTED for
head sizes other than 128.  Which prompts LLaMA.refill_rows packs comes from the kernel each linear runs at M rows
(ColBlockQuantizedLinear.kernel_at, the dispatch `forward` uses): gptq.int4 packs from 17 tokens (shorter prompts run
the GEMV and the 2..8 / 9..16-row kernels), gptq.int8 from 2, llm.int8, dense, grouped and biased layers never.
refill_rows and generate_stream refuse bad arguments; the CLI takes --stream with --prompts_file."""
import ctypes as C
import importlib
import sys

import pytest
import torch

import __graft_entry__ as entry

P_ = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails an argument check (none may launch)


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def _err(L):
    return L.lib().b2l_last_error().decode()


def _seqs(L, lengths, rows=None, starts=None):
    sq = L.Ragged()
    sq.n_seq = len(lengths)
    at = 0
    for s, n in enumerate(lengths):
        sq.len[s] = n
        sq.row[s] = s if rows is None else rows[s]
        sq.start[s] = at if starts is None else starts[s]
        at += n
    return sq


def _call(L, seqs, N, ptrs=None, B_rows=6, n_head=4, head_size=128, S=64, block_size=64, prefix=None):
    qkv, kc, vc, rope, ring, y = ptrs or (P_,) * 6
    rc = L.lib().b2l_attention_ragged(qkv, kc, vc, rope, None if seqs is None else C.byref(seqs), ring, y, N, B_rows,
                                      n_head, head_size, S, block_size, None if prefix is None else C.byref(prefix), None)
    return rc, _err(L)


@pytest.mark.parametrize("which", range(6))
def test_null_pointers(L, which):
    ptrs = [P_] * 6
    ptrs[which] = None
    rc, err = _call(L, _seqs(L, [3, 5]), 8, ptrs=ptrs)
    assert rc == -1 and err.startswith("b2l_attention_ragged: null pointer"), err
    rc, err = _call(L, None, 8)
    assert rc == -1 and "null pointer" in err


@pytest.mark.parametrize("field", ["N", "B_rows", "n_head", "S", "block_size"])
def test_bad_shapes(L, field):
    kw = dict(B_rows=6, n_head=4, S=64, block_size=64)
    N = 8
    if field == "N":
        N = 0
    else:
        kw[field] = 0
    rc, err = _call(L, _seqs(L, [3, 5]), N, **kw)
    assert rc == -1 and "b2l_attention_ragged: bad shape" in err, err


@pytest.mark.parametrize("hs", [32, 64, 256])
def test_head_size_128_only(L, hs):
    rc, err = _call(L, _seqs(L, [3, 5]), 8, head_size=hs)
    assert rc == -2 and f"head_size {hs} unsupported (128 only)" in err, err


def test_sequence_count(L):
    sq = _seqs(L, [3])
    sq.n_seq = 0
    rc, err = _call(L, sq, 3)
    assert rc == -1 and "n_seq 0 outside 1..16" in err
    sq = _seqs(L, [1] * 16)
    sq.n_seq = 17
    rc, err = _call(L, sq, 17, B_rows=17)
    assert rc == -1 and "n_seq 17 outside 1..16" in err


@pytest.mark.parametrize("n", [0, -2, 65])
def test_length_outside_1_to_S(L, n):
    rc, err = _call(L, _seqs(L, [4, n]), 4 + n, S=64)
    assert rc == -1 and f"sequence 1 has length {n} (1..S=64)" in err, err


@pytest.mark.parametrize("starts,N,what", [
    ([1, 5], 9, "sequence 0 starts at 1, not 0"),      # the first does not start at 0
    ([0, 5], 9, "sequence 1 starts at 5, not 4"),      # a gap
    ([0, 3], 7, "sequence 1 starts at 3, not 4"),      # an overlap
    ([0, 4], 10, "cover 8 tokens, N=10"),              # N beyond the last sequence
    ([0, 4], 6, "cover 8 tokens, N=6"),                # N short of it
])
def test_starts_must_tile_0_to_N(L, starts, N, what):
    rc, err = _call(L, _seqs(L, [4, 4], starts=starts), N)
    assert rc == -1 and what in err, err


@pytest.mark.parametrize("row", [-1, 6, 100])
def test_row_out_of_range(L, row):
    rc, err = _call(L, _seqs(L, [4, 4, 4], rows=[0, row, 2]), 12, B_rows=6)
    assert rc == -1 and f"sequence 1 names row {row} of 6" in err, err


def test_two_sequences_one_row(L):
    rc, err = _call(L, _seqs(L, [4, 4, 4], rows=[5, 2, 5]), 12, B_rows=6)
    assert rc == -1 and "sequences 0 and 2 both name row 5" in err, err


def test_adapter_prefix_checks(L):
    rc, err = _call(L, _seqs(L, [4, 4]), 8, prefix=L.AdapterPrefix(P_, None, P_, 8))
    assert rc == -1 and "b2l_attention_ragged: null adapter prefix pointer" in err, err
    rc, err = _call(L, _seqs(L, [4, 4]), 8, prefix=L.AdapterPrefix(P_, P_, P_, 65))
    assert rc == -2 and "adapter prefix length 65 unsupported" in err, err


# --------------------------------------------------------------------------------------------- the packing rule
def _gptq(bits, K=256, N=384, tile_cols=-1, bias=False):
    import lit_llama_b200 as P

    lin = P.ColBlockQuantizedLinear(K, N, bias, bits=bits, tile_cols=tile_cols)
    return lin


LAYERS = {
    "gptq.int4": lambda: _gptq(4),
    "gptq.int8": lambda: _gptq(8),
    "gptq.int4 grouped": lambda: _gptq(4, tile_cols=128),
    "gptq.int8 biased": lambda: _gptq(8, bias=True),
    "llm.int8": lambda: __import__("lit_llama_b200").Linear8bitLt(256, 384, bias=False),
    "dense": lambda: torch.nn.Linear(256, 384, bias=False),
}
KERNELS = {   # kernel at M = 1, 2, 16, 17
    "gptq.int4": ["q4_gemv", "q4_gemv_batch", "q4_linear_tc", "q4_gemm"],
    "gptq.int8": ["w8_gemv", "w8_gemm", "w8_gemm", "w8_gemm"],
    "gptq.int4 grouped": ["q_linear"] * 4,
    "gptq.int8 biased": ["q_linear"] * 4,
    "llm.int8": [None] * 4,
    "dense": [None] * 4,
}
PACKS = {   # joins a pack of 640 tokens at T = 1, 2, 16, 17
    "gptq.int4": [False, False, False, True],
    "gptq.int8": [False, True, True, True],
}


@pytest.mark.parametrize("kind", list(LAYERS))
def test_packing_rule_from_kernel_at(kind):
    from lit_llama_b200.quantization import BATCH_GEMV, kernel_at, packs_at

    lin = LAYERS[kind]()
    want = KERNELS[kind]
    if kind == "gptq.int4" and not BATCH_GEMV:
        want = ["q4_gemv", "q4_linear_tc", "q4_linear_tc", "q4_gemm"]
    assert [kernel_at(lin, T) for T in (1, 2, 16, 17)] == want
    assert [packs_at([lin], T, 640) for T in (1, 2, 16, 17)] == PACKS.get(kind, [False] * 4)
    if isinstance(lin, __import__("lit_llama_b200").ColBlockQuantizedLinear):
        # forward asks the same function: the answer for a misaligned input is the generic kernel's
        assert lin.kernel_at(17, aligned=False) == "q_linear"


def _model(mode, n_embd=256, n_head=2, **kw):
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    with quantization(mode):
        return P.LLaMA(P.LLaMAConfig(block_size=64, vocab_size=64, n_layer=2, n_head=n_head, n_embd=n_embd, **kw))


def test_pack_plan_of_a_model():
    lengths = [1, 2, 16, 17, 40, 3]
    assert _model("gptq.int4")._pack_plan(lengths) == [3, 4]
    assert _model("gptq.int8")._pack_plan(lengths) == [1, 2, 3, 4, 5]
    assert _model("gptq.int4", n_embd=128, n_head=4)._pack_plan(lengths) == []   # head_size 32: no ragged attention
    assert _model("llm.int8")._pack_plan(lengths) == []
    assert _model(None)._pack_plan(lengths) == []
    m = _model("gptq.int4")
    m.lm_head = torch.nn.Linear(256, 64, bias=False)   # one linear outside the dispatch: nothing packs
    assert m._pack_plan(lengths) == []


def test_refill_rows_and_generate_stream_refusals():
    import lit_llama_b200 as P

    m = _model("gptq.int4")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.refill_rows([torch.tensor([1, 2, 3])], [0], 8)
    with pytest.raises(ValueError, match="non-empty 1-D"):
        m.refill_rows([torch.tensor([], dtype=torch.int64)], [0], 8)
    with pytest.raises(ValueError, match="1..16"):
        m.refill_rows([torch.tensor([1])] * 17, list(range(17)), 8)
    with pytest.raises(ValueError, match="no prompts"):
        P.generate_stream(m, [], 4)
    for bs in (0, 17):
        with pytest.raises(ValueError, match="1..16"):
            P.generate_stream(m, [torch.tensor([1, 2])], 4, batch_size=bs)
    with pytest.raises(ValueError, match=r"shape \(T,\)"):
        P.generate_stream(m, [torch.tensor([[1, 2]])], 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        P.generate_stream(m, [torch.tensor([1, 2]), torch.tensor([3])], 4)


def test_cli_stream_flag(monkeypatch, tmp_path):
    import lit_llama_b200  # noqa: F401

    G = importlib.import_module("lit_llama_b200.generate")
    got = {}
    monkeypatch.setattr(G, "main", lambda **kw: got.update(kw))
    f = tmp_path / "prompts.txt"
    f.write_text("Hello\nThe capital of France is\n")
    monkeypatch.setattr(sys, "argv", ["generate.py", "--prompts_file", str(f), "--batch_size", "8", "--stream"])
    G.cli()
    assert got["stream"] is True and got["batch_size"] == 8
    monkeypatch.setattr(sys, "argv", ["generate.py", "--prompts_file", str(f)])
    G.cli()
    assert got["stream"] is False   # default: the grouped generate_prompts loop, as before
    monkeypatch.setattr(sys, "argv", ["generate.py", "--stream"])
    with pytest.raises(SystemExit):
        G.cli()

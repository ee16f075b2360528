"""CPU: per-row positions (B2L_F_ROW_POS) are refused where they cannot run, before the device is touched:
b2l_ring_advance_rows / b2l_kv_unroll_rows with null pointers or bad shapes; b2l_attention(_adapter) with the flag at
T > 1 or with B2L_F_ROPE_ROWS; b2l_decode_step with the flag and B2L_F_ROPE_ROWS.  generate_prompts and
LLaMA.prefill_rows take 1..16 one-dimensional prompts and have no CPU path; LLaMA.forward refuses a 2-D input_pos
that is not one position per row; the CLI takes --prompts_file."""
import ctypes as C
import importlib
import sys

import pytest
import torch

import __graft_entry__ as entry

P_ = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def _err(L):
    return L.lib().b2l_last_error().decode()


def test_ring_advance_rows_refusals(L):
    lib = L.lib()
    assert lib.b2l_ring_advance_rows(None, 4, P_, 16, None) == -1 and "b2l_ring_advance_rows: null pointer" in _err(L)
    assert lib.b2l_ring_advance_rows(P_, 4, None, 16, None) == -1 and "null pointer" in _err(L)
    assert lib.b2l_ring_advance_rows(P_, 0, P_, 16, None) == -1 and "bad shape (B=0" in _err(L)
    assert lib.b2l_ring_advance_rows(P_, 4, P_, 0, None) == -1 and "S=0" in _err(L)


def test_kv_unroll_rows_refusals(L):
    lib = L.lib()
    assert lib.b2l_kv_unroll_rows(None, P_, P_, 4, 2, 16, 32, None) == -1 and "b2l_kv_unroll_rows: null pointer" in _err(L)
    assert lib.b2l_kv_unroll_rows(P_, None, P_, 4, 2, 16, 32, None) == -1 and "null pointer" in _err(L)
    assert lib.b2l_kv_unroll_rows(P_, P_, None, 4, 2, 16, 32, None) == -1 and "null pointer" in _err(L)
    for B, nh, S, hs in ((0, 2, 16, 32), (4, 0, 16, 32), (4, 2, 0, 32), (4, 2, 16, 0)):
        assert lib.b2l_kv_unroll_rows(P_, P_, P_, B, nh, S, hs, None) == -1 and "bad shape" in _err(L)


def _attn(L, adapter, T=1, flags=None, head_size=128, qkv=P_):
    lib = L.lib()
    fl = L.F_ROW_POS if flags is None else flags
    args = (qkv, P_, P_, P_, P_, P_, P_, P_, 4, T, 4, head_size, 16, 64, fl)
    if not adapter:
        return lib.b2l_attention(*args, None), _err(L)
    pre = L.AdapterPrefix(P_, P_, P_, 8)
    return lib.b2l_attention_adapter(*args, C.byref(pre), None), _err(L)


@pytest.mark.parametrize("adapter", [False, True])
@pytest.mark.parametrize("head_size", [128, 32])
def test_attention_row_pos_refusals(L, adapter, head_size):
    name = "b2l_attention_adapter: " if adapter else "b2l_attention: "
    rc, err = _attn(L, adapter, T=2, head_size=head_size)
    assert rc == -2 and err.startswith(name) and "B2L_F_ROW_POS runs one token per row (T == 1), got T=2" in err
    rc, err = _attn(L, adapter, flags=L.F_ROW_POS | L.F_ROPE_ROWS, head_size=head_size)
    assert rc == -2 and "B2L_F_ROW_POS does not combine with B2L_F_ROPE_ROWS" in err
    rc, err = _attn(L, adapter, qkv=None, head_size=head_size)   # the null checks come first, as without the flag
    assert rc == -1 and "null pointer" in err


def _decode_args(L, flags):
    layers = (L.Layer * 1)()
    a = L.DecodeArgs(n_layer=1, n_head=4, n_embd=512, n_hidden=1536, vocab=256, B=4, S=16, eps=1e-5,
                     layers=C.cast(layers, C.POINTER(L.Layer)), wte=P_, ln_f=P_, rope=P_, idx=P_, input_pos=P_,
                     ring_start=P_, block_size=64, x=P_, qkv=P_, att=P_, hid=P_, attn_work=P_, logits=P_, flags=flags,
                     batch_work=P_)
    return a, layers


def test_decode_step_row_pos_refusals(L):
    lib = L.lib()
    a, keep = _decode_args(L, L.F_PDL | L.F_ROW_POS | L.F_Q4_BATCH_I8)
    a.flags = L.F_ROW_POS | L.F_ROPE_ROWS
    assert lib.b2l_decode_step(C.byref(a), None) == -2 and "B2L_F_ROW_POS does not combine with B2L_F_ROPE_ROWS" in _err(L)
    # the existing refusals still apply with the flag: a batch flag outside its range, null pointers
    a.flags = L.F_ROW_POS | L.F_Q4_BATCH_I8 | L.F_W8
    assert lib.b2l_decode_step(C.byref(a), None) == -2 and "B2L_F_Q4_BATCH_I8" in _err(L)
    a.flags = L.F_ROW_POS | L.F_W8_BATCH
    assert lib.b2l_decode_step(C.byref(a), None) == -2 and "B2L_F_W8_BATCH needs B2L_F_W8" in _err(L)
    a.flags, a.B = L.F_ROW_POS | L.F_Q4_BATCH_I8, 17
    assert lib.b2l_decode_step(C.byref(a), None) == -2 and "batch 17 > 16" in _err(L)
    a.B, a.input_pos = 4, None
    assert lib.b2l_decode_step(C.byref(a), None) == -1 and "null pointer" in _err(L)


def _tiny_model():
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    with quantization("gptq.int4"):
        return P.LLaMA(P.LLaMAConfig(block_size=16, vocab_size=64, n_layer=1, n_head=2, n_embd=64)).bfloat16()


@pytest.mark.parametrize("n", [0, 17])
def test_generate_prompts_takes_1_to_16_prompts(n):
    import lit_llama_b200 as P

    m = _tiny_model()
    with pytest.raises(ValueError, match="1..16"):
        P.generate_prompts(m, [torch.tensor([1, 2, 3])] * n, 5)
    with pytest.raises(ValueError, match="1..16"):
        m.prefill_rows([torch.tensor([1, 2, 3])] * n, 8)


def test_generate_prompts_refuses_2d_and_cpu_prompts():
    import lit_llama_b200 as P

    m = _tiny_model()
    with pytest.raises(ValueError, match=r"shape \(T,\)"):
        P.generate_prompts(m, [torch.tensor([1, 2, 3]), torch.tensor([[1, 2]])], 5)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        P.generate_prompts(m, [torch.tensor([1, 2, 3]), torch.tensor([4, 5])], 5)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.prefill_rows([torch.tensor([1, 2, 3])], 8)
    with pytest.raises(ValueError, match="non-empty 1-D"):
        m.prefill_rows([torch.tensor([[1, 2, 3]])], 8)


def test_forward_refuses_2d_input_pos_that_is_not_one_per_row():
    m = _tiny_model()
    with pytest.raises(ValueError, match="one position per row"):
        m(torch.zeros((2, 3), dtype=torch.int64), 8, torch.zeros((2, 3), dtype=torch.int64))   # T > 1
    with pytest.raises(ValueError, match="one position per row"):
        m(torch.zeros((2, 1), dtype=torch.int64), 8, torch.zeros((3, 1), dtype=torch.int64))   # rows differ


def test_cli_accepts_prompts_file(monkeypatch, tmp_path):
    import lit_llama_b200  # noqa: F401

    G = importlib.import_module("lit_llama_b200.generate")
    got = {}
    monkeypatch.setattr(G, "main", lambda **kw: got.update(kw))
    f = tmp_path / "prompts.txt"
    f.write_text("Hello\nThe capital of France is\n")
    monkeypatch.setattr(sys, "argv", ["generate.py", "--prompts_file", str(f), "--batch_size", "8"])
    G.cli()
    assert str(got["prompts_file"]) == str(f) and got["batch_size"] == 8
    monkeypatch.setattr(sys, "argv", ["generate.py"])
    G.cli()
    assert got["prompts_file"] is None   # default: the one --prompt, as before

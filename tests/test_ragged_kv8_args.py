"""CPU: the packed refill into an fp8 KV cache.  b2l_attention_ragged_kv8 against the header (C prototype, ctypes
binding), its refusals before the device is touched, the pack plan of an fp8 model (the bf16 model's), and how
refill_rows splits a pack into passes by free memory (LLaMA._packed_passes).

b2l_attention_ragged_kv8 returns B2L_E_ARG for null pointers, null or misaligned b2l_kv8_cache fields, bad shapes,
n_seq outside 1..16, a length outside 2..S or above block_size, starts that do not tile [0, N), a row outside the
cache, two sequences naming one row and a null adapter prefix pointer, and B2L_E_UNSUPPORTED for head sizes other than
128 and a prefix longer than 64, with the messages b2l_attention_ragged gives (one shared check)."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import pytest
import torch

import __graft_entry__ as entry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P_ = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails an argument check (none may launch)
WHO = "b2l_attention_ragged_kv8"


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


def _kv(L, **kw):
    a = dict(k=P_, v=P_ + 4096, k_scale=P_ + 8192, v_scale=P_ + 12288)
    a.update(kw)
    return L.KV8Cache(**a)


def _call(L, seqs, N, ptrs=None, kv=None, B_rows=6, n_head=4, head_size=128, S=64, block_size=64, prefix=None,
          null_kv=False):
    qkv, rope, ring, y = ptrs or (P_,) * 4
    kv = _kv(L) if kv is None else kv
    rc = L.lib().b2l_attention_ragged_kv8(qkv, None if null_kv else C.byref(kv), rope,
                                          None if seqs is None else C.byref(seqs), ring, y, N, B_rows, n_head, head_size,
                                          S, block_size, None if prefix is None else C.byref(prefix), None)
    return rc, _err(L)


def test_prototype_and_binding_match_the_header(L, tmp_path):
    prog = tmp_path / "proto.c"
    prog.write_text(
        '#include "b2l.h"\n'
        "typedef int (*ragged8_t)(void*, const b2l_kv8_cache*, const void*, const b2l_ragged*, int32_t*, void*, int, int,"
        " int, int, int, int, const b2l_adapter_prefix*, b2l_stream_t);\n"
        "int main(void){ ragged8_t f = b2l_attention_ragged_kv8; (void)f; return 0; }\n")
    subprocess.run(["gcc", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(prog), "-o", str(tmp_path / "p.o")],
                   check=True)
    res, args = L._SIGS[WHO]
    assert res is C.c_int and len(args) == 14
    assert args[1] is C.POINTER(L.KV8Cache) and args[3] is C.POINTER(L.Ragged) and args[12] is C.POINTER(L.AdapterPrefix)
    assert args[6:12] == [C.c_int] * 6
    assert L.lib().b2l_version() == 100


@pytest.mark.parametrize("which", range(4))
def test_null_pointers(L, which):
    ptrs = [P_] * 4
    ptrs[which] = None
    rc, err = _call(L, _seqs(L, [3, 5]), 8, ptrs=ptrs)
    assert rc == -1 and err.startswith(f"{WHO}: null pointer"), err
    rc, err = _call(L, None, 8)
    assert rc == -1 and f"{WHO}: null pointer" in err
    rc, err = _call(L, _seqs(L, [3, 5]), 8, null_kv=True)
    assert rc == -1 and f"{WHO}: null pointer" in err


@pytest.mark.parametrize("field", ["k", "v", "k_scale", "v_scale"])
def test_null_and_misaligned_cache_fields(L, field):
    rc, err = _call(L, _seqs(L, [3, 5]), 8, kv=_kv(L, **{field: None}))
    assert rc == -1 and f"{WHO}: null fp8 cache pointer" in err, err
    rc, err = _call(L, _seqs(L, [3, 5]), 8, kv=_kv(L, **{field: P_ + (8 if field in ("k", "v") else 2)}))
    assert rc == -1 and f"{WHO}: fp8 cache codes must be 16-byte aligned" in err, err


@pytest.mark.parametrize("field", ["N", "B_rows", "n_head", "S", "block_size"])
def test_bad_shapes(L, field):
    kw = dict(B_rows=6, n_head=4, S=64, block_size=64)
    N = 8
    if field == "N":
        N = 0
    else:
        kw[field] = 0
    rc, err = _call(L, _seqs(L, [3, 5]), N, **kw)
    assert rc == -1 and f"{WHO}: bad shape" in err, err


@pytest.mark.parametrize("hs", [32, 64, 256])
def test_head_size_128_only(L, hs):
    rc, err = _call(L, _seqs(L, [3, 5]), 8, head_size=hs)
    assert rc == -2 and f"{WHO}: head_size {hs} unsupported (128 only)" in err, err


def test_sequence_count(L):
    sq = _seqs(L, [3])
    sq.n_seq = 0
    rc, err = _call(L, sq, 3)
    assert rc == -1 and "n_seq 0 outside 1..16" in err
    sq = _seqs(L, [2] * 16)
    sq.n_seq = 17
    rc, err = _call(L, sq, 34, B_rows=17)
    assert rc == -1 and "n_seq 17 outside 1..16" in err


@pytest.mark.parametrize("n", [1, 0, -2, 65])
def test_length_outside_2_to_S(L, n):
    rc, err = _call(L, _seqs(L, [4, n]), 4 + n, S=64)
    assert rc == -1 and f"{WHO}: sequence 1 has length {n} (2..S=64)" in err, err


def test_length_past_block_size(L):
    rc, err = _call(L, _seqs(L, [4, 40]), 44, S=64, block_size=32)
    assert rc == -1 and f"{WHO}: sequence 1 has length 40, past block_size=32" in err, err


@pytest.mark.parametrize("starts,N,what", [
    ([1, 5], 9, "sequence 0 starts at 1, not 0"),      # the first does not start at 0
    ([0, 5], 9, "sequence 1 starts at 5, not 4"),      # a gap
    ([0, 3], 7, "sequence 1 starts at 3, not 4"),      # an overlap
    ([0, 4], 10, "cover 8 tokens, N=10"),              # N beyond the last sequence
    ([0, 4], 6, "cover 8 tokens, N=6"),                # N short of it
])
def test_starts_must_tile_0_to_N(L, starts, N, what):
    rc, err = _call(L, _seqs(L, [4, 4], starts=starts), N)
    assert rc == -1 and what in err and err.startswith(WHO), err


@pytest.mark.parametrize("row", [-1, 6, 100])
def test_row_out_of_range(L, row):
    rc, err = _call(L, _seqs(L, [4, 4, 4], rows=[0, row, 2]), 12, B_rows=6)
    assert rc == -1 and f"{WHO}: sequence 1 names row {row} of 6" in err, err


def test_two_sequences_one_row(L):
    rc, err = _call(L, _seqs(L, [4, 4, 4], rows=[5, 2, 5]), 12, B_rows=6)
    assert rc == -1 and f"{WHO}: sequences 0 and 2 both name row 5" in err, err


def test_adapter_prefix_checks(L):
    rc, err = _call(L, _seqs(L, [4, 4]), 8, prefix=L.AdapterPrefix(P_, None, P_, 8))
    assert rc == -1 and f"{WHO}: null adapter prefix pointer" in err, err
    rc, err = _call(L, _seqs(L, [4, 4]), 8, prefix=L.AdapterPrefix(P_, P_, P_, 65))
    assert rc == -2 and "adapter prefix length 65 unsupported" in err, err


def test_bf16_ragged_messages_unchanged(L):
    """The shared check still names b2l_attention_ragged, with its 1..S length range."""
    sq = _seqs(L, [4, 0])
    rc = L.lib().b2l_attention_ragged(P_, P_, P_, P_, C.byref(sq), P_, P_, 4, 6, 4, 128, 64, 64, None, None)
    assert rc == -1 and _err(L).startswith("b2l_attention_ragged: sequence 1 has length 0 (1..S=64)"), _err(L)


# --------------------------------------------------------------------------------------------- the plan and its passes
def _model(mode, fp8, n_embd=256, n_head=2):
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    with quantization(mode):
        m = P.LLaMA(P.LLaMAConfig(block_size=64, vocab_size=64, n_layer=2, n_head=n_head, n_embd=n_embd))
    if fp8:
        m.kv_cache_dtype = "fp8"
        m._new_kv_store(4, 64, torch.device("cpu"))
        assert isinstance(m.kv_caches[0], P.model.FP8KVCache)
    return m


@pytest.mark.parametrize("mode,want", [("gptq.int4", [3, 4]), ("gptq.int8", [1, 2, 3, 4, 5])])
def test_fp8_model_packs_what_the_bf16_model_packs(mode, want):
    lengths = [1, 2, 16, 17, 40, 3]
    assert _model(mode, fp8=True)._pack_plan(lengths) == _model(mode, fp8=False)._pack_plan(lengths) == want
    assert _model(mode, fp8=True, n_embd=128, n_head=4)._pack_plan(lengths) == []   # head_size 32


def test_packed_token_bytes_from_the_config():
    import lit_llama_b200 as P

    m = _model("gptq.int4", fp8=True)
    n_hidden = m.transformer.h[0].mlp.c_fc1.out_features
    assert m._packed_token_bytes() == 2 * (6 * 256 + 3 * n_hidden)
    cfg = P.LLaMAConfig.from_name("65B")   # 8192 wide, 22016 hidden: 225 KiB per token
    assert P.LLaMA._packed_token_bytes(SimpleNamespace(config=cfg)) == 2 * (6 * 8192 + 3 * 22016)


def test_packed_passes():
    import lit_llama_b200 as P

    split = P.LLaMA._packed_passes
    lengths = [17, 40, 300, 25, 512, 18]
    tb = 1000
    # everything fits (exactly, and with room): one pass, in input order
    assert split(lengths, tb, sum(lengths) * tb) == [list(range(6))]
    assert split(lengths, tb, 10 ** 12) == [list(range(6))]
    # a budget of 400 tokens: consecutive passes, in input order, each within it except a prompt longer than it alone
    got = split(lengths, tb, 400 * tb + 999)
    assert got == [[0, 1, 2, 3], [4], [5]]
    # no room at all: one prompt per pass
    assert split(lengths, tb, 0) == [[i] for i in range(6)]
    assert split(lengths, tb, -5) == [[i] for i in range(6)]
    for budget in (0, 17, 57, 300, 357, 400, 700, 912, 2000):
        passes = split(lengths, tb, budget * tb)
        assert [i for p in passes for i in p] == list(range(6)), budget   # cover the plan exactly, in order
        assert all(p for p in passes)                                     # at least one prompt per pass
        for p in passes:
            assert len(p) == 1 or sum(lengths[i] for i in p) <= budget, (budget, passes)
        # greedy: the next pass's first prompt did not fit behind the previous pass
        for a, b in zip(passes, passes[1:]):
            assert sum(lengths[i] for i in a) + lengths[b[0]] > budget, (budget, passes)
    assert split([], tb, 10 ** 9) == []

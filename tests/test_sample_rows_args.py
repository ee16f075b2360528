"""CPU: the row sampling entry points (b2l_topk_softmax_rows / b2l_topk_softmax_sample_rows) reject bad arguments with a
message naming the argument before they touch the device; sample_token / sample_probs over rows and generate_batch have
no CPU path; generate_batch takes 1..16 samples; the CLI takes --batch_size."""
import importlib
import sys

import pytest
import torch

import __graft_entry__ as entry

P_ = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first
V = 100


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def _probs(L, **kw):
    a = dict(logits=P_, ld=V, temperature=0.8, top_k=4, probs=2 * P_, B=3, V=V)
    a.update(kw)
    rc = L.lib().b2l_topk_softmax_rows(a["logits"], a["ld"], a["temperature"], a["top_k"], a["probs"], a["B"], a["V"], None)
    return rc, L.lib().b2l_last_error().decode()


def _sample(L, **kw):
    a = dict(logits=P_, ld=V, temperature=0.8, top_k=4, noise=3 * P_, probs=None, tokens=4 * P_, B=3, V=V)
    a.update(kw)
    rc = L.lib().b2l_topk_softmax_sample_rows(a["logits"], a["ld"], a["temperature"], a["top_k"], a["noise"], a["probs"],
                                              a["tokens"], a["B"], a["V"], None)
    return rc, L.lib().b2l_last_error().decode()


REFUSALS = [
    (dict(logits=None), "null logits"),
    (dict(B=0), "B = 0"),
    (dict(B=-2), "B = -2"),
    (dict(V=0), "V = 0"),
    (dict(temperature=0.0), "temperature"),
    (dict(top_k=-1), "top_k = -1"),
    (dict(ld=1), "ld = 1"),
    (dict(ld=V - 1), f"ld = {V - 1}"),
    (dict(ld=-V), f"ld = {-V}"),
    (dict(logits=P_ + 2), "logits must be 16-byte aligned"),
    (dict(logits=P_ + 8), "logits must be 16-byte aligned"),
]


@pytest.mark.parametrize("kw,msg", REFUSALS)
def test_rows_refusals(L, kw, msg):
    for call, name in ((_probs, "b2l_topk_softmax_rows: "), (_sample, "b2l_topk_softmax_sample_rows: ")):
        rc, err = call(L, **kw)
        assert rc == -1 and err.startswith(name) and msg in err, (kw, err)


def test_rows_refusals_of_each_entry_point(L):
    rc, err = _probs(L, probs=None)
    assert rc == -1 and "b2l_topk_softmax_rows: null probs" in err
    rc, err = _sample(L, noise=None)
    assert rc == -1 and "b2l_topk_softmax_sample_rows: null noise" in err
    rc, err = _sample(L, tokens=None)
    assert rc == -1 and "b2l_topk_softmax_sample_rows: null tokens" in err
    rc, err = _sample(L, noise=3 * P_ + 4)
    assert rc == -1 and "noise must be 16-byte aligned" in err
    # the kernel's one-CTA vocabulary limit is not an argument error
    rc, err = _sample(L, V=60000, ld=60000)
    assert rc == -2 and "too large" in err


def test_single_row_entry_points_keep_their_checks(L):
    lib = L.lib()
    assert lib.b2l_topk_softmax(P_, 0.8, 4, None, V, None) == -1 and b"null probs" in lib.b2l_last_error()
    assert lib.b2l_topk_softmax(P_ + 2, 0.8, 4, P_, V, None) == -1 and b"logits must be 16-byte aligned" in lib.b2l_last_error()
    assert lib.b2l_topk_softmax_sample(P_, 0.8, 4, None, None, P_, V, None) == -1
    assert b"null noise / token" in lib.b2l_last_error()
    assert lib.b2l_topk_softmax_sample(None, 0.8, 4, P_, None, P_, V, None) == -1 and b"bad argument" in lib.b2l_last_error()


def _tiny_model():
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    with quantization("gptq.int4"):
        return P.LLaMA(P.LLaMAConfig(block_size=16, vocab_size=64, n_layer=1, n_head=2, n_embd=64)).bfloat16()


def test_rows_and_generate_batch_have_no_cpu_fallback():
    import lit_llama_b200 as P

    for fn in (P.sample_probs, P.sample_token):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            fn(torch.zeros(4, 64, dtype=torch.bfloat16), 0.8, 4)
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            fn(torch.zeros(64, dtype=torch.bfloat16).expand(4, -1), 0.8, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        P.generate_batch(_tiny_model(), torch.tensor([1, 2, 3]), 4, 5)


@pytest.mark.parametrize("n", [0, -1, 17, 64])
def test_generate_batch_takes_1_to_16_samples(n):
    import lit_llama_b200 as P

    with pytest.raises(ValueError, match="num_samples"):
        P.generate_batch(_tiny_model(), torch.tensor([1, 2, 3]), n, 5)


def test_expand_cache_needs_a_batch1_cache():
    m = _tiny_model()
    with pytest.raises(RuntimeError, match="no KV cache"):
        m.expand_cache(4)
    m._kv_store = torch.zeros(1, 2, 2, 2, 16, 32, dtype=torch.bfloat16)   # a cache of 2 rows
    with pytest.raises(ValueError, match="batch-1"):
        m.expand_cache(4)


def test_cli_accepts_batch_size(monkeypatch):
    import lit_llama_b200  # noqa: F401

    G = importlib.import_module("lit_llama_b200.generate")
    main = G.main
    for bad in (0, 17):   # refused before anything is loaded
        with pytest.raises(ValueError, match="batch_size"):
            main(batch_size=bad)
    got = {}
    monkeypatch.setattr(G, "main", lambda **kw: got.update(kw))
    monkeypatch.setattr(sys, "argv", ["generate.py", "--num_samples", "20", "--batch_size", "8", "--quantize", "gptq.int4"])
    G.cli()
    assert got["batch_size"] == 8 and got["num_samples"] == 20 and got["quantize"] == "gptq.int4"
    monkeypatch.setattr(sys, "argv", ["generate.py"])
    G.cli()
    assert got["batch_size"] == 1   # default: one generate() per sample, as the reference

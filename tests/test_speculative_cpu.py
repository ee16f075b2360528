"""CPU: speculative decoding's surface.  The B2L_F_STEPWISE flag value and b2l_spec_accept's place in the header; every
refusal of b2l_attention(_adapter), b2l_decode_step and b2l_spec_accept under the new mode, before the device is
touched; the step's launch count; the Python refusals of generate_speculative and LLaMA.decode_tokens; and the accept /
resample rule restated in torch (`spec_accept_ref`, which the GPU tests hold the kernel to) over constructed cases."""
import ctypes as C
import os
import re

import pytest
import torch

import __graft_entry__ as entry

P_ = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def _err(L):
    return L.lib().b2l_last_error().decode()


def spec_accept_ref(p, q, x, u, noise):
    """The accept / resample rule of b2l_spec_accept on bf16 probabilities p [k+1, V] (the target's, as
    b2l_topk_softmax_rows computes them) and q [k, V] (the draft's), draft tokens x [k], u fp32 [k] and noise bf16 [V]:
    (n_accepted, token).  Draws are argmax of bf16(w / noise), ties to the lowest index."""
    p, q, noise = p.float().cpu(), q.float().cpu(), noise.float().cpu()
    u, x = u.float().cpu(), x.cpu()
    V = p.shape[1]

    def draw(w):
        key = (w / noise).bfloat16().float()
        return int(torch.nonzero(key == key.max())[0])

    k = q.shape[0]
    for t in range(k):
        xt = int(x[t])
        if 0 <= xt < V and bool(u[t] * q[t, xt] < p[t, xt]):
            continue
        r = torch.clamp(p[t] - q[t], min=0.0)
        return t, draw(r if bool((r > 0).any()) else p[t])
    return k, draw(p[k])


# ----------------------------------------------------------------------------------------------- header
def test_flag_value_and_entry_point_position():
    h = open(os.path.join(ROOT, "include", "b2l.h")).read()
    assert re.search(r"B2L_F_STEPWISE = 2048\b", h)
    from lit_llama_b200 import _lib

    assert _lib.F_STEPWISE == 2048
    names = re.findall(r"^int (b2l_\w+)\(", h, flags=re.M)
    i = names.index("b2l_spec_accept")
    assert names[i - 1] == "b2l_topk_softmax_sample_rows"   # with the sampling entry points
    assert "b2l_spec_accept" in _lib.EXPORTS


# ----------------------------------------------------------------------------------------------- attention
def _attn(L, adapter, B=1, T=4, flags=0, head_size=128):
    lib = L.lib()
    args = (P_, P_, P_, P_, P_, P_, P_, P_, B, T, 4, head_size, 64, 64, flags | L.F_STEPWISE)
    if not adapter:
        return lib.b2l_attention(*args, None), _err(L)
    pre = L.AdapterPrefix(P_, P_, P_, 8)
    return lib.b2l_attention_adapter(*args, C.byref(pre), None), _err(L)


@pytest.mark.parametrize("adapter", [False, True])
@pytest.mark.parametrize("head_size", [128, 32])
def test_attention_stepwise_refusals(L, adapter, head_size):
    name = "b2l_attention_adapter: " if adapter else "b2l_attention: "
    cases = [
        (dict(flags=L.F_ROW_POS), "B2L_F_STEPWISE does not combine with B2L_F_ROW_POS"),
        (dict(flags=L.F_ROPE_ROWS), "B2L_F_STEPWISE does not combine with B2L_F_ROPE_ROWS"),
        (dict(B=2), "B2L_F_STEPWISE runs the tokens of one sequence (B == 1), got B=2"),
        (dict(T=1), "B2L_F_STEPWISE runs 2..16 tokens, got T=1"),
        (dict(T=17), "B2L_F_STEPWISE runs 2..16 tokens, got T=17"),
    ]
    for kw, msg in cases:
        rc, err = _attn(L, adapter, head_size=head_size, **kw)
        assert rc == -2 and err == name + msg, (kw, err)


# ----------------------------------------------------------------------------------------------- the step
def _decode_args(L, flags, B=4, head_size=128):
    layers = (L.Layer * 2)()
    a = L.DecodeArgs(n_layer=2, n_head=4, n_embd=4 * head_size, n_hidden=1536, vocab=256, B=B, S=16, eps=1e-5,
                     layers=C.cast(layers, C.POINTER(L.Layer)), wte=P_, ln_f=P_, rope=P_, idx=P_, input_pos=P_,
                     ring_start=P_, block_size=64, x=P_, qkv=P_, att=P_, hid=P_, attn_work=P_, logits=P_, flags=flags,
                     batch_work=P_)
    return a, layers


def test_decode_step_stepwise_refusals(L):
    lib = L.lib()
    S_, Q4 = L.F_STEPWISE, L.F_Q4_BATCH_I8
    W8 = L.F_W8 | L.F_W8_BATCH
    cases = [
        (S_ | Q4 | L.F_ROW_POS, {}, "B2L_F_STEPWISE does not combine with B2L_F_ROW_POS"),
        (S_ | L.F_Q8 | L.F_Q8_BATCH, {}, "B2L_F_STEPWISE does not run llm.int8 (B2L_F_Q8)"),
        (S_, {}, "B2L_F_STEPWISE needs the row-exact linears"),
        (S_ | L.F_W8, {}, "B2L_F_STEPWISE needs the row-exact linears"),
        (S_ | Q4, dict(B=1), "B2L_F_STEPWISE runs 2..16 tokens, got B=1"),
        (S_ | Q4, dict(affines=True), "B2L_F_STEPWISE does not apply LLaMA-Adapter v2 affines"),
        (S_ | W8, dict(lm_head_affine=L.OutAffine(P_, P_)), "B2L_F_STEPWISE does not apply LLaMA-Adapter v2 affines"),
    ]
    for flags, kw, msg in cases:
        a, keep = _decode_args(L, flags, B=kw.pop("B", 4))
        if kw.pop("affines", False):
            arr = (L.LayerAffine * 2)()
            keep = (keep, arr)
            a.affines = C.cast(arr, C.POINTER(L.LayerAffine))
        for f, v in kw.items():
            setattr(a, f, v)
        assert lib.b2l_decode_step(C.byref(a), None) == -2, msg
        assert "b2l_decode_step: " + msg in _err(L), (msg, _err(L))
    a, keep = _decode_args(L, S_ | Q4, B=17)   # the existing batch limit still applies first
    assert lib.b2l_decode_step(C.byref(a), None) == -2 and "batch 17 > 16" in _err(L)


@pytest.mark.parametrize("head_size", [128, 32])
def test_decode_step_launch_count(L, head_size):
    lib = L.lib()
    for flags in (L.F_Q4_BATCH_I8, L.F_W8 | L.F_W8_BATCH):
        a, keep = _decode_args(L, flags | L.F_PDL, B=5, head_size=head_size)
        base = lib.b2l_decode_step_launches(C.byref(a))
        # 2 + n_layer * (4 linears x 2 launches + attention) + lm_head (2 launches)
        assert base == 2 + 2 * (8 + (1 if head_size == 128 else 3)) + 2
        a.flags |= L.F_STEPWISE
        # head_size 128: the fused kernel runs behind one append launch per layer; the three-kernel path appends anyway
        assert lib.b2l_decode_step_launches(C.byref(a)) == base + (2 if head_size == 128 else 0)
        a.flags |= 8   # B2L_F_ATTN_UNFUSED: the three-kernel path at head_size 128 too
        assert lib.b2l_decode_step_launches(C.byref(a)) == 2 + 2 * (8 + 3) + 2


# ----------------------------------------------------------------------------------------------- b2l_spec_accept
def test_spec_accept_refusals(L):
    lib = L.lib()
    V = 256

    def call(**kw):
        a = dict(logits=P_, ld=V, temperature=1.0, top_k=0, q=P_, x=P_, u=P_, noise=P_, n=P_, tok=P_, T=4, V=V)
        a.update(kw)
        rc = lib.b2l_spec_accept(a["logits"], a["ld"], a["temperature"], a["top_k"], a["q"], a["x"], a["u"], a["noise"],
                                 a["n"], a["tok"], a["T"], a["V"], None)
        return rc, _err(L)

    cases = [
        (dict(logits=None), -1, "null logits"),
        (dict(T=1), -2, "T = 1 target rows; 2..16"),
        (dict(T=17), -2, "T = 17 target rows; 2..16"),
        (dict(V=0), -1, "V = 0, at least 1"),
        (dict(temperature=0.0), -1, "temperature 0, must be positive"),
        (dict(top_k=-1), -1, "top_k = -1"),
        (dict(ld=V - 1), -1, "ld = 255, at least V = 256"),
        (dict(q=None), -1, "null draft_probs"),
        (dict(x=None), -1, "null draft_tokens"),
        (dict(u=None), -1, "null u"),
        (dict(noise=None), -1, "null noise"),
        (dict(n=None), -1, "null n_accepted / token"),
        (dict(tok=None), -1, "null n_accepted / token"),
        (dict(logits=P_ + 2), -1, "target_logits must be 16-byte aligned"),
        (dict(q=P_ + 2), -1, "draft_probs and noise must be 16-byte aligned"),
        (dict(noise=P_ + 8), -1, "draft_probs and noise must be 16-byte aligned"),
        (dict(V=1 << 20, ld=1 << 20), -2, "vocabulary 1048576 too large for one CTA"),
    ]
    for kw, rc, msg in cases:
        got, err = call(**kw)
        assert got == rc and err.startswith("b2l_spec_accept: ") and msg in err, (kw, got, err)


# ----------------------------------------------------------------------------------------------- the rule in torch
def _bf(x):
    return torch.tensor(x, dtype=torch.float32).bfloat16()


def test_accept_rule_constructed_cases():
    V = 8
    ones = torch.ones(V).bfloat16()
    p = _bf([[0.0, 0.5, 0.5, 0, 0, 0, 0, 0]] * 3)
    q = _bf([[0.5, 0.25, 0.25, 0, 0, 0, 0, 0]] * 2)
    # u = 0 and p(x) = 0: the strict test rejects; the residual max(0, p - q) puts everything on 1 and 2 (a tie: 1)
    assert spec_accept_ref(p, q, torch.tensor([0, 1]), torch.zeros(2), ones) == (0, 1)
    # p = q: always accepted (u < 1), the token is drawn from the last row
    assert spec_accept_ref(p, p[:2], torch.tensor([1, 2]), torch.full((2,), 0.999), ones) == (2, 1)
    # all accepted, the last row's draw follows the noise
    noise = _bf([1, 1, 4, 1, 1, 1, 1, 1])
    assert spec_accept_ref(p, q, torch.tensor([1, 2]), torch.tensor([0.1, 0.1]), noise) == (2, 1)
    # the first rejection in the middle: row 0 accepted (0.5 * 0.25 < 0.5), row 1 rejected (x = 0, p = 0)
    k3p = _bf([[0, 0.5, 0.5, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0, 0], [0.25] * 4 + [0] * 4, [1] + [0] * 7])
    k3q = _bf([[0, 0.25, 0.75, 0, 0, 0, 0, 0], [1, 0, 0, 0, 0, 0, 0, 0], [0.25] * 4 + [0] * 4])
    assert spec_accept_ref(k3p, k3q, torch.tensor([1, 0, 2]), torch.full((3,), 0.5), ones) == (1, 3)
    # u just above p / q rejects, and the residual lies where p > q
    assert spec_accept_ref(k3p, k3q, torch.tensor([2, 3, 2]), torch.full((3,), 0.7), ones) == (0, 1)
    # an all-zero residual (p <= q everywhere after rounding): drawn from p itself
    pz = _bf([[0, 0.5, 0.5, 0, 0, 0, 0, 0], [0, 0, 0, 0, 1, 0, 0, 0]])
    qz = _bf([[0, 0.5, 0.5, 0, 0, 0, 0, 0]])
    assert spec_accept_ref(pz, qz, torch.tensor([1]), torch.ones(1), _bf([1, 1, 0.5, 1, 1, 1, 1, 1])) == (0, 2)
    # a draft token outside the vocabulary is rejected
    assert spec_accept_ref(p, p[:2], torch.tensor([9, 1]), torch.zeros(2), ones) == (0, 1)
    # ties in the draw go to the lower index
    assert spec_accept_ref(_bf([[0.25] * 4 + [0] * 4] * 2), _bf([[0] * 8]), torch.tensor([7]), torch.ones(1), ones) == (0, 0)


def test_top1_reduces_to_argmax_agreement():
    """With top_k = 1 both rows are one-hot: accept while the draft token is the target's argmax, then emit it."""
    g = torch.Generator().manual_seed(5)
    V, k = 32, 5
    for _ in range(50):
        am = torch.randint(0, V, (k + 1,), generator=g)
        p = torch.zeros(k + 1, V)
        p[torch.arange(k + 1), am] = 1
        x = am[:k].clone()
        j = int(torch.randint(0, k + 1, (1,), generator=g))
        if j < k:
            x[j] = (x[j] + 1) % V
        q = torch.zeros(k, V)
        q[torch.arange(k), x] = 1
        u = torch.rand(k, generator=g)
        noise = torch.empty(V).exponential_(1, generator=g).bfloat16()
        assert spec_accept_ref(p.bfloat16(), q.bfloat16(), x, u, noise) == (j, int(am[j]))


# ----------------------------------------------------------------------------------------------- Python refusals
def _dense(vocab=64):
    import lit_llama_b200 as P

    return P.LLaMA(P.LLaMAConfig(block_size=16, vocab_size=vocab, n_layer=1, n_head=2, n_embd=64)).bfloat16()


def test_generate_speculative_refusals():
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    idx = torch.zeros(4, dtype=torch.int64)
    m = _dense()
    for k in (0, 16, -1):
        with pytest.raises(ValueError, match=r"num_draft = .*; 1\.\.15"):
            P.generate_speculative(m, m, idx, 4, num_draft=k)
    with pytest.raises(ValueError, match="padded_vocab_size 128 differs from the target's 64"):
        P.generate_speculative(m, _dense(vocab=128), idx, 4)
    with pytest.raises(ValueError, match="one prompt of shape"):
        P.generate_speculative(m, m, idx.view(1, 4), 4)
    with pytest.raises(RuntimeError, match="the target's verify step .* needs a gptq.int4 or gptq.int8 model"):
        P.generate_speculative(m, m, idx, 4)   # dense
    cfg = dict(block_size=16, vocab_size=64, n_layer=1, n_head=2, n_embd=64)
    with quantization("llm.int8"):
        q8 = P.LLaMA(P.LLaMAConfig(**cfg))
    with pytest.raises(RuntimeError, match="not dense, llm.int8, LLaMA-Adapter v2"):
        P.generate_speculative(q8, m, idx, 4)
    import lit_llama_b200.adapter as PA
    import lit_llama_b200.adapter_v2 as PV

    with quantization("gptq.int4"):
        v2 = PA.LLaMA(PA.LLaMAConfig(**cfg, adapter_prompt_length=4, adapter_start_layer=0))
        PV.add_adapter_v2_parameters_to_linear_layers(v2)
    with pytest.raises(RuntimeError, match="the target's verify step .* needs a gptq.int4 or gptq.int8 model"):
        P.generate_speculative(v2, m, idx, 4)


def test_decode_tokens_shape_refusals():
    m = _dense()
    with pytest.raises(ValueError, match=r"idx must be \(1, T\) with T in 2\.\.16"):
        m.decode_tokens(torch.zeros(1, 1, dtype=torch.int64), 16, torch.zeros(1, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"idx must be \(1, T\)"):
        m.decode_tokens(torch.zeros(2, 4, dtype=torch.int64), 16, torch.zeros(4, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"idx must be \(1, T\) with T in 2\.\.16"):
        m.decode_tokens(torch.zeros(1, 17, dtype=torch.int64), 32, torch.zeros(17, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"input_pos must be \(4,\)"):
        m.decode_tokens(torch.zeros(1, 4, dtype=torch.int64), 16, torch.zeros(3, dtype=torch.int64))


def test_cli_takes_the_draft_options(monkeypatch):
    import importlib

    G = importlib.import_module("lit_llama_b200.generate")
    seen = {}
    monkeypatch.setattr(G, "main", lambda **kw: seen.update(kw))
    monkeypatch.setattr("sys.argv", ["generate", "--draft_checkpoint_path", "d.pth", "--draft_quantize", "gptq.int4",
                                     "--num_draft", "6"])
    G.cli()
    assert str(seen["draft_checkpoint_path"]) == "d.pth" and seen["draft_quantize"] == "gptq.int4" and seen["num_draft"] == 6

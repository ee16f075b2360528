"""CPU: prompt-lookup speculative decoding's surface.  The proposer rule of b2l_ngram_propose restated in numpy
(`ngram_propose_ref`, which the GPU tests hold the kernel to) over hand-built histories; the deterministic-draft accept
rule (`lookup_accept_ref`) against b2l_spec_accept's general rule on one-hot draft rows; every argument refusal of
b2l_ngram_propose before the device is touched; and the refusals of generate_speculative(draft=None) and of the CLI's
--lookup_ngram."""
import os
import re
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
from test_speculative_cpu import spec_accept_ref

P_ = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ngram_propose_ref(history, n, min_ngram, max_ngram, k):
    """The rule of b2l_ngram_propose over history[:n]: for g = max_ngram down to min_ngram (g <= n - 1), the largest
    start i with i + g <= n - 1 and history[i:i+g] == history[n-g:n]; the first g with one proposes
    history[i+g : min(i+g+k, n)].  Returns the proposed tokens (a list; empty when nothing matches)."""
    h = np.asarray(history[:n], dtype=np.int64)
    for g in range(max_ngram, min_ngram - 1, -1):
        if g > n - 1:
            continue
        win = np.lib.stride_tricks.sliding_window_view(h[:n - 1], g)   # row i: h[i:i+g], i + g <= n - 1
        hits = np.nonzero((win == h[n - g:]).all(axis=1))[0]
        if hits.size:
            i = int(hits[-1])
            return [int(t) for t in h[i + g:min(i + g + k, n)]]
    return []


def lookup_probs_ref(tokens, k, V):
    """The proposer's rows bf16 [k, V]: row t < len(tokens) is 1.0 at tokens[t] when 0 <= tokens[t] < V; all else 0."""
    q = torch.zeros(k, V, dtype=torch.bfloat16)
    for t, x in enumerate(tokens):
        if 0 <= x < V:
            q[t, x] = 1.0
    return q


def lookup_accept_ref(p, x, u, noise):
    """b2l_spec_accept on the proposer's rows (a deterministic draft): x_t is accepted iff u_t < p_t(x_t); at the first
    rejection j the token is argmax_i bf16(p_j(i) / noise[i]) with p_j(x_j) set to 0 (x_j outside the vocabulary: p_j
    as it is); all accepted: argmax bf16(p_k / noise).  Ties to the lowest index.  Returns (n_accepted, token)."""
    p, noise, u = p.float().cpu(), noise.float().cpu(), u.float().cpu()
    V = p.shape[1]

    def draw(w):
        key = (w / noise).bfloat16().float()
        return int(torch.nonzero(key == key.max())[0])

    for t, xt in enumerate(int(v) for v in x):
        inside = 0 <= xt < V
        if inside and bool(u[t] < p[t, xt]):
            continue
        r = p[t].clone()
        if inside:
            r[xt] = 0
        return t, draw(r)
    return len(x), draw(p[len(x)])


# ----------------------------------------------------------------------------------------------- the rule
def _prop(hist, min_ngram=1, max_ngram=3, k=4, n=None):
    return ngram_propose_ref(hist, len(hist) if n is None else n, min_ngram, max_ngram, k)


def test_rule_no_match():
    assert _prop([1, 2, 3, 4, 5]) == []
    assert _prop([7]) == []                       # n = 1: no g <= n - 1
    assert _prop([5, 5], min_ngram=2, max_ngram=3) == []   # n = 2 <= g for every g tried


def test_rule_match_only_at_a_shorter_g():
    # the trigram (8, 9, 4) and bigram (9, 4) never occurred before; the unigram 4 did, at index 1
    assert _prop([3, 4, 6, 7, 8, 9, 4]) == [6, 7, 8, 9]
    # with min_ngram = 2 the unigram is not tried
    assert _prop([3, 4, 6, 7, 8, 9, 4], min_ngram=2) == []


def test_rule_longest_g_wins_over_a_more_recent_shorter_match():
    # the bigram (1, 2) occurs at 0; the unigram 2 occurs more recently at 5: the bigram's continuation wins
    assert _prop([1, 2, 30, 31, 40, 2, 50, 1, 2], max_ngram=2) == [30, 31, 40, 2]
    assert _prop([1, 2, 30, 31, 40, 2, 50, 1, 2], max_ngram=1) == [50, 1, 2]


def test_rule_most_recent_occurrence_wins():
    # (5, 6) occurs at 0, 4 and 8: the one at 8 is the most recent earlier occurrence
    h = [5, 6, 10, 11, 5, 6, 20, 21, 5, 6, 30, 31, 5, 6]
    assert _prop(h, max_ngram=2, k=2) == [30, 31]
    assert _prop(h, max_ngram=2, k=15) == [30, 31, 5, 6]   # truncated by the history's end


def test_rule_overlapping_occurrence():
    # a a a a: the trigram at 0 overlaps the suffix (positions 1..3); it proposes history[3:4]
    assert _prop([9, 9, 9, 9]) == [9]
    assert _prop([9, 9, 9, 9, 9, 9], k=15) == [9]          # the most recent occurrence ends one token short
    # a b a b a: the trigram (a, b, a) at 0 overlaps the suffix at 2
    assert _prop([1, 2, 1, 2, 1], k=15) == [2, 1]


def test_rule_truncation_by_k_and_by_the_end():
    h = [1, 2, 3, 4, 5, 6, 7, 8, 9, 1, 2]
    assert _prop(h, k=3) == [3, 4, 5]
    assert _prop(h, k=15) == [3, 4, 5, 6, 7, 8, 9, 1, 2]
    assert _prop(h, k=1) == [3]


def test_rule_n_not_above_g():
    # n = 3: g = 3 is skipped (g > n - 1) and g = 2 tried; n = 2: only g = 1
    assert _prop([4, 4, 4], min_ngram=2, max_ngram=3) == [4]
    assert _prop([4, 4], min_ngram=1, max_ngram=16) == [4]
    # the length read from the history's prefix (the n_accepted form): later entries are not part of it
    assert _prop([1, 2, 1, 9, 9, 9], n=3) == [2, 1]


def test_rule_min_equals_max():
    h = [1, 2, 3, 7, 2, 3, 8, 1, 2, 3]
    assert _prop(h, min_ngram=3, max_ngram=3) == [7, 2, 3, 8]
    assert _prop(h, min_ngram=2, max_ngram=2) == [8, 1, 2, 3]
    assert _prop(h, min_ngram=1, max_ngram=1) == [8, 1, 2, 3]
    assert _prop([1, 2, 3, 7, 3], min_ngram=2, max_ngram=2) == []


def test_rule_against_a_plain_python_scan():
    """The numpy restatement against the rule written as nested loops, on random short histories."""
    rng = np.random.default_rng(3)
    for _ in range(400):
        n = int(rng.integers(1, 40))
        h = [int(t) for t in rng.integers(0, int(rng.integers(2, 5)), n)]
        lo = int(rng.integers(1, 6))
        hi = int(rng.integers(lo, 7))
        k = int(rng.integers(1, 16))
        want = []
        for g in range(hi, lo - 1, -1):
            if g > n - 1:
                continue
            i = max((i for i in range(n - g) if h[i:i + g] == h[n - g:]), default=-1)
            if i >= 0:
                want = h[i + g:i + g + k]
                break
        assert ngram_propose_ref(h, n, lo, hi, k) == want, (h, lo, hi, k)


def test_lookup_accept_rule_is_spec_accept_with_one_hot_rows():
    """lookup_accept_ref equals spec_accept_ref fed the proposer's rows, on random p, proposals and u."""
    g = torch.Generator().manual_seed(11)
    V = 16
    for trial in range(300):
        k = int(torch.randint(1, 6, (1,), generator=g))
        p = torch.softmax(torch.randn(k + 1, V, generator=g) * 2, -1).bfloat16()
        x = torch.randint(0, V, (k,), generator=g)
        if trial % 3 == 0:
            x = p[:k].float().argmax(-1)
        if trial % 5 == 0:
            x[0] = V + 2
        u = torch.rand(k, generator=g)
        noise = torch.empty(V).exponential_(1, generator=g).bfloat16()
        q = lookup_probs_ref([int(v) for v in x], k, V)
        assert lookup_accept_ref(p, x, u, noise) == spec_accept_ref(p, q, x, u, noise), trial


# ----------------------------------------------------------------------------------------------- the C entry point
@pytest.fixture(scope="module")
def L():
    entry.build()
    from lit_llama_b200 import _lib

    return _lib


def test_entry_point_in_the_header_and_binding(L):
    h = open(os.path.join(ROOT, "include", "b2l.h")).read()
    names = re.findall(r"^int (b2l_\w+)\(", h, flags=re.M)
    assert names[names.index("b2l_ngram_propose") - 1] == "b2l_spec_accept"
    assert "b2l_ngram_propose" in L.EXPORTS


def _call(L, **kw):
    a = dict(history=P_, base_len=10, n_accepted=None, min_ngram=1, max_ngram=3, k=4, tokens=2 * P_, probs=3 * P_,
             count=4 * P_, V=100)
    a.update(kw)
    rc = L.lib().b2l_ngram_propose(a["history"], a["base_len"], a["n_accepted"], a["min_ngram"], a["max_ngram"], a["k"],
                                   a["tokens"], a["probs"], a["count"], a["V"], None)
    return rc, L.lib().b2l_last_error().decode()


REFUSALS = [
    (dict(history=None), "null history"),
    (dict(tokens=None), "null tokens"),
    (dict(count=None), "null count"),
    (dict(history=P_ + 4), "history must be 8-byte aligned"),
    (dict(tokens=2 * P_ + 4), "tokens must be 8-byte aligned"),
    (dict(n_accepted=5 * P_ + 2), "n_accepted must be 4-byte aligned"),
    (dict(count=4 * P_ + 2), "count must be 4-byte aligned"),
    (dict(probs=3 * P_ + 2), "probs must be 16-byte aligned"),
    (dict(probs=3 * P_ + 8), "probs must be 16-byte aligned"),
    (dict(base_len=0), "base_len = 0, at least 1"),
    (dict(base_len=-5), "base_len = -5, at least 1"),
    (dict(min_ngram=0), "min_ngram = 0, max_ngram = 3"),
    (dict(min_ngram=4), "min_ngram = 4, max_ngram = 3"),
    (dict(max_ngram=17), "min_ngram = 1, max_ngram = 17"),
    (dict(min_ngram=-1, max_ngram=-1), "min_ngram = -1, max_ngram = -1"),
    (dict(k=0), "k = 0; 1..15"),
    (dict(k=16), "k = 16; 1..15"),
    (dict(V=0), "V = 0, at least 1"),
    (dict(V=-3, probs=None), "V = -3, at least 1"),
]


@pytest.mark.parametrize("kw,msg", REFUSALS)
def test_ngram_propose_refusals(L, kw, msg):
    rc, err = _call(L, **kw)
    assert rc == -1 and err.startswith("b2l_ngram_propose: ") and msg in err, (kw, rc, err)


# ----------------------------------------------------------------------------------------------- Python refusals
CFG = dict(block_size=16, vocab_size=64, n_layer=1, n_head=2, n_embd=64)


def _dense():
    import lit_llama_b200 as P

    return P.LLaMA(P.LLaMAConfig(**CFG)).bfloat16()


def test_generate_speculative_lookup_refusals():
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    idx = torch.zeros(4, dtype=torch.int64)
    m = _dense()
    for lo, hi in ((0, 3), (2, 1), (1, 17), (-1, 2), (4, 3)):
        with pytest.raises(ValueError, match=rf"min_ngram = {lo}, max_ngram = {hi}; 1 <= min_ngram <= max_ngram <= 16"):
            P.generate_speculative(m, None, idx, 4, min_ngram=lo, max_ngram=hi)
    with pytest.raises(ValueError, match=r"num_draft = 16; 1\.\.15"):
        P.generate_speculative(m, None, idx, 4, num_draft=16)
    with pytest.raises(ValueError, match="one prompt of shape"):
        P.generate_speculative(m, None, idx.view(1, 4), 4)
    with pytest.raises(RuntimeError, match="the target's verify step .* needs a gptq.int4 or gptq.int8 model"):
        P.generate_speculative(m, None, idx, 4)   # dense
    with quantization("llm.int8"):
        q8 = P.LLaMA(P.LLaMAConfig(**CFG))
    with pytest.raises(RuntimeError, match="not dense, llm.int8, LLaMA-Adapter v2"):
        P.generate_speculative(q8, None, idx, 4)
    with quantization("gptq.int4"):
        q4 = P.LLaMA(P.LLaMAConfig(**dict(CFG, n_embd=128, n_head=1)))
    q4.kv_cache_dtype = "fp8"
    with pytest.raises(RuntimeError, match=r"the target's verify step \(LLaMA.decode_tokens\) does not run on an fp8 KV cache"):
        P.generate_speculative(q4, None, idx, 4)


def _cli(monkeypatch, *argv):
    import importlib

    G = importlib.import_module("lit_llama_b200.generate")
    seen = {}
    monkeypatch.setattr(G, "main", lambda **kw: seen.update(kw))
    monkeypatch.setattr(sys, "argv", ["generate", *argv])
    G.cli()
    return seen


def test_cli_lookup_ngram(monkeypatch, capsys, tmp_path):
    seen = _cli(monkeypatch, "--lookup_ngram", "4", "--num_draft", "8")
    assert seen["lookup_ngram"] == 4 and seen["num_draft"] == 8 and seen["draft_checkpoint_path"] is None
    assert _cli(monkeypatch)["lookup_ngram"] == 0   # default: off
    f = tmp_path / "prompts.txt"
    f.write_text("Hello\n")
    cases = [
        (("--lookup_ngram", "3", "--draft_checkpoint_path", "d.pth"), "does not combine with --draft_checkpoint_path"),
        (("--lookup_ngram", "3", "--kv_cache", "fp8"), "--kv_cache fp8 does not combine with --lookup_ngram"),
        (("--lookup_ngram", "3", "--batch_size", "2"), "--lookup_ngram decodes one sequence at a time"),
        (("--lookup_ngram", "3", "--prompts_file", str(f)), "--lookup_ngram decodes one sequence at a time"),
        (("--lookup_ngram", "17"), "--lookup_ngram 17: 1..16"),
        (("--lookup_ngram", "-1"), "--lookup_ngram -1: 1..16"),
    ]
    for argv, msg in cases:
        with pytest.raises(SystemExit):
            _cli(monkeypatch, *argv)
        assert msg in capsys.readouterr().err, argv

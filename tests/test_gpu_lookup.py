"""-m gpu: prompt-lookup speculative decoding.  `b2l_ngram_propose` against its restatement (`ngram_propose_ref`) bit
for bit in tokens, count and every bf16 of the probability rows; `b2l_spec_accept` fed the proposer's rows against the
deterministic-draft rule (`lookup_accept_ref`) and, by a chi-square test, its first emitted token against the target's
distribution; `generate_speculative(draft=None, top_k=1)` against `generate(top_k=1)` token for token, with its round
schedule equal to a host simulation of the rule; and one host read per round."""
import numpy as np
import pytest
import torch

from test_lookup_cpu import lookup_accept_ref, ngram_propose_ref

pytestmark = pytest.mark.gpu

NAN_BITS = 0x7FC0   # a bf16 NaN: the proposer's rows are prefilled with it, so every element is checked as written


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _P():
    import lit_llama_b200 as P

    return P


def _propose(L, hist, base_len, nacc, lo, hi, k, tokens, probs, count, V):
    L.check(L.lib().b2l_ngram_propose(hist.data_ptr(), base_len, None if nacc is None else nacc.data_ptr(), lo, hi, k,
                                      tokens.data_ptr(), None if probs is None else probs.data_ptr(), count.data_ptr(), V,
                                      L.stream_ptr()), "b2l_ngram_propose")


# --------------------------------------------------------------------------------------------- 1. the proposer
def test_proposer_equals_the_restatement(dev):
    """2 400 random histories of 1..2100 tokens over alphabets of 2..64 ids (ids up to 31 999, negative ones and ones
    >= V among them), max_ngram 1..16, k 1..15, V from 1 to 32 000, with the length given directly or as
    base_len + *n_accepted + 1; the buffer past the history holds more alphabet tokens, which must not be read."""
    L = _L()
    rng = np.random.default_rng(2024)
    NMAX, KV = 2200, 15 * 32000
    hist = torch.empty(NMAX, dtype=torch.int64, device=dev)
    probs = torch.empty(KV + 64, dtype=torch.bfloat16, device=dev)
    bits = probs.view(torch.int16)
    tokens = torch.empty(16, dtype=torch.int64, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    nacc = torch.empty(1, dtype=torch.int32, device=dev)
    seen = dict(none=0, full=0, short=0, outside=0, grown=0, no_probs=0, below_max=0)
    for case in range(2400):
        V = int(rng.choice([1, 7, 64, 100, 32000]))
        m = int(rng.integers(2, 65))
        pool = np.concatenate([rng.integers(0, min(V, 32000), 64), rng.integers(0, 32000, 16), [-1, -2, 31999, V, V + 1]])
        alphabet = rng.choice(np.unique(pool), size=min(m, np.unique(pool).size), replace=False).astype(np.int64)
        n = int(rng.integers(1, 41) if case % 2 else rng.integers(1, 2101))
        h = alphabet[rng.integers(0, alphabet.size, NMAX)]
        hi = int(rng.integers(1, 17))
        lo = int(rng.integers(1, hi + 1))
        k = int(rng.integers(1, 16))
        grown = case % 3 != 0 and n >= 2
        a = int(rng.integers(0, min(15, n - 2) + 1)) if grown else 0
        with_probs = case % 7 != 0
        hist.copy_(torch.from_numpy(h))
        nacc.fill_(a)
        bits.fill_(NAN_BITS)
        tokens.fill_(-77777)
        count.fill_(-1)
        _propose(L, hist, n - a - 1 if grown else n, nacc if grown else None, lo, hi, k, tokens,
                 probs if with_probs else None, count, V)
        want = ngram_propose_ref(h, n, lo, hi, k)
        c = int(count)
        got = tokens.tolist()
        assert c == len(want) and got[:c] == want and got[c:] == [-77777] * (16 - c), (case, n, lo, hi, k, c, got, want)
        exp = torch.zeros(k * V if with_probs else 0, dtype=torch.int16)
        for t, x in enumerate(want):
            if with_probs and 0 <= x < V:
                exp[t * V + x] = 0x3F80
        assert torch.equal(bits[:exp.numel()].cpu(), exp), (case, n, k, V)
        assert bool((bits[exp.numel():] == NAN_BITS).all()), case   # nothing past the k rows
        seen["none"] += c == 0
        seen["full"] += c == k
        seen["short"] += 0 < c < k
        seen["outside"] += any(not 0 <= x < V for x in want)
        seen["grown"] += grown and c > 0
        seen["no_probs"] += not with_probs
        seen["below_max"] += c > 0 and ngram_propose_ref(h, n, hi, hi, k) == [] and hi <= n - 1
    assert min(seen.values()) >= 20, seen


# --------------------------------------------------------------------------------------------- 2. accept on its rows
def _history_proposing(xs, A=-5):
    """A history whose prompt lookup (max_ngram 1) proposes exactly xs: A, xs, A (A outside the vocabulary)."""
    return torch.tensor([7, A] + list(xs) + [A], dtype=torch.int64)


def _accept(L, lt, temp, top_k, q, x, u, noise, k):
    V = lt.shape[1]
    n = torch.full((1,), -1, dtype=torch.int32, device=lt.device)
    tok = torch.full((1,), -1, dtype=torch.int64, device=lt.device)
    L.check(L.lib().b2l_spec_accept(lt.data_ptr(), V, float(temp), top_k, q.data_ptr(), x.data_ptr(), u.data_ptr(),
                                    noise.data_ptr(), n.data_ptr(), tok.data_ptr(), k + 1, V, L.stream_ptr()),
            "b2l_spec_accept")
    return n, tok


@pytest.mark.parametrize("V", [64, 32000])
def test_spec_accept_on_proposer_rows_equals_the_deterministic_draft_rule(dev, V):
    """Proposals equal to the target's argmax, random, and with one token outside the vocabulary, at several
    temperature / top_k settings: (n_accepted, token) of b2l_spec_accept on the proposer's rows equals
    lookup_accept_ref on the probabilities b2l_topk_softmax_rows computes."""
    L, P = _L(), _P()
    g = torch.Generator(device=dev).manual_seed(V + 1)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    outcomes = set()
    for temp, top_k in ((1.0, None), (0.7, 50), (1.3, 1), (0.9, 4)):
        for k in (1, 2, 5, 15):
            for trial in range(6):
                lt = (torch.randn(k + 1, V, device=dev, generator=g) * (1 + trial % 3)).bfloat16()
                p = P.sample_probs(lt, temp, top_k)
                xs = torch.randint(0, V, (k,), device=dev, generator=g)
                if trial % 3 == 0:
                    xs = p[:k].float().argmax(-1)
                elif trial % 3 == 2:
                    xs = p[:k].float().argmax(-1)
                    xs[k // 2] = V + 3
                hist = _history_proposing(xs.tolist()).to(dev)
                q = torch.full((k, V), float("nan"), dtype=torch.bfloat16, device=dev)
                x = torch.empty(k, dtype=torch.int64, device=dev)
                _propose(L, hist, hist.numel(), None, 1, 1, k, x, q, count, V)
                assert int(count) == k and torch.equal(x, xs)
                u = torch.rand(k, device=dev, generator=g)
                noise = torch.empty(V, dtype=torch.bfloat16, device=dev).exponential_(1, generator=g)
                n, tok = _accept(L, lt, temp, 0 if top_k is None else top_k, q, x, u, noise, k)
                got = (int(n), int(tok))
                assert got == lookup_accept_ref(p, xs, u, noise), (temp, top_k, k, trial, got)
                outcomes.add("all" if got[0] == k else "none" if got[0] == 0 else "some")
    assert outcomes == {"all", "none", "some"}


def test_first_token_on_proposer_rows_is_distributed_as_the_target(dev):
    """A deterministic proposal x_0 (probability ~0.3 under p_0): the first emitted token of 20 000 rounds (x_0 when
    accepted, else the draw from p_0 without x_0) follows p_0 (chi-square, fixed seed)."""
    from scipy.stats import chisquare

    L, P = _L(), _P()
    V, k, N = 32, 2, 20000
    g = torch.Generator(device=dev).manual_seed(321)
    lt = (torch.randn(k + 1, V, device=dev, generator=g) * 1.5).bfloat16()
    p = P.sample_probs(lt, 1.0, None)
    x0 = int((p[0].float() - 0.3).abs().argmin())
    hist = _history_proposing([x0, (x0 + 1) % V]).to(dev)
    q = torch.empty((k, V), dtype=torch.bfloat16, device=dev)
    x = torch.empty(k, dtype=torch.int64, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    _propose(L, hist, hist.numel(), None, 1, 1, k, x, q, count, V)
    assert int(count) == k
    us = torch.rand(N, k, device=dev, generator=g)
    noises = torch.empty(N, V, dtype=torch.bfloat16, device=dev).exponential_(1, generator=g)
    ns = torch.empty(N, dtype=torch.int32, device=dev)
    toks = torch.empty(N, dtype=torch.int64, device=dev)
    lib, st = L.lib(), L.stream_ptr()
    for i in range(N):
        L.check(lib.b2l_spec_accept(lt.data_ptr(), V, 1.0, 0, q.data_ptr(), x.data_ptr(), us[i].data_ptr(),
                                    noises[i].data_ptr(), ns[i:].data_ptr(), toks[i:].data_ptr(), k + 1, V, st),
                "b2l_spec_accept")
    first = torch.where(ns > 0, x0, toks).cpu()
    counts = torch.bincount(first, minlength=V).double()
    exp = p[0].double().cpu()
    exp = exp / exp.sum() * N
    keep = exp >= 5
    obs = torch.cat((counts[keep], counts[~keep].sum().view(1)))
    ex = torch.cat((exp[keep], exp[~keep].sum().view(1)))
    if float(ex[-1]) < 5:   # fold a small remainder into the largest bin
        obs, ex = obs[:-1].clone(), ex[:-1].clone()
        obs[ex.argmax()] += counts[~keep].sum()
        ex[ex.argmax()] += exp[~keep].sum()
    ex = ex * obs.sum() / ex.sum()
    stat, pval = chisquare(obs.numpy(), ex.numpy())
    assert 0 < int((ns == 0).sum()) < N   # rejections happen
    assert pval > 1e-3, (stat, pval)


# --------------------------------------------------------------------------------------------- 3. end to end
def simulate(y, T, n_new, S, kmax, min_ngram=1, max_ngram=3):
    """generate_speculative(draft=None, top_k=1)'s schedule when its output is y (the greedy sequence): the stats it
    records, and the spans [start, end) of y each round emitted."""
    st = dict(rounds=0, proposed=[], accepted=[], num_draft=kmax, tail_steps=0, lookup_misses=0)
    spans = []
    n = 1
    prop = ngram_propose_ref(y, T + 1, min_ngram, max_ngram, kmax)
    while n < n_new:
        p = T + n - 1
        k = min(kmax, S - 1 - p, n_new - n - 1)
        if k < 1:
            break
        k = min(k, len(prop))
        if k == 0:
            n += 1
            st["lookup_misses"] += 1
        else:
            a = 0
            while a < k and prop[a] == y[T + n + a]:
                a += 1
            st["rounds"] += 1
            st["proposed"].append(k)
            st["accepted"].append(a)
            spans.append((T + n, T + n + a + 1))
            n += a + 1
        prop = ngram_propose_ref(y, T + n, min_ngram, max_ngram, kmax)
    st["tail_steps"] = n_new - n
    return st, spans


def _covers(st, kmax):
    """At least one fully accepted, one partly accepted (k >= 2 only) and one fully rejected round, and one miss."""
    pairs = list(zip(st["proposed"], st["accepted"]))
    return (any(a == k for k, a in pairs) and any(a == 0 for k, a in pairs) and st["lookup_misses"] > 0
            and (kmax == 1 or any(0 < a < k for k, a in pairs)))


@pytest.fixture(scope="module")
def zoo(dev):
    from test_gpu_speculative import _model

    cache = {}

    def get(kind):
        if kind not in cache:
            cache[kind] = _model(dev, kind)
        return cache[kind]

    yield get
    cache.clear()
    torch.cuda.empty_cache()


def _prompts(P, model, dev):
    """Candidate prompts: repeated n-grams over a few ids, and such a prompt followed by 16 of its own greedy tokens
    (whose continuation then tends to repeat text of the prompt)."""
    V = model.config.vocab_size
    for seed in range(40):
        g = torch.Generator().manual_seed(seed)
        ids = torch.randperm(V, generator=g)[:6]
        pat = ids[torch.randint(0, 6, (5,), generator=g)]
        prompt = torch.cat((pat, pat, ids[torch.randint(0, 6, (3,), generator=g)], pat)).to(torch.int32).to(dev)
        yield prompt
        model.reset_cache()
        yield P.generate(model, prompt, 16, top_k=1)


def _mid_round_first(y, T, spans):
    """Positions j whose token first appears among the emitted tokens y[T:] at j, inside a round but not its last."""
    return [j for s, e in spans for j in range(s, e - 1) if y[j] not in y[T:j]]


def _case(P, model, dev, kmax, n_new, S=None, cover=True, mid_eos=False):
    """A candidate prompt whose greedy continuation has no top-1 tie and (with `cover`) whose schedule has every kind of
    round (_covers), (with `mid_eos`) a token first emitted inside a round: (prompt, generate()'s output, the simulated
    stats and spans)."""
    from test_gpu_speculative import _greedy_ties

    for prompt in _prompts(P, model, dev):
        T = prompt.numel()
        if S is not None and T + 2 > S:
            continue
        Sx = S if S is not None else min(T + n_new, model.config.block_size)
        model.reset_cache()
        want = P.generate(model, prompt, n_new, max_seq_length=S, top_k=1)
        y = want.tolist()
        st, spans = simulate(y, T, n_new, Sx, kmax)
        if ((not cover or _covers(st, kmax)) and (not mid_eos or _mid_round_first(y, T, spans))
                and not _greedy_ties(model, prompt, want, Sx)):
            return prompt, want, st, spans
    raise AssertionError("no candidate prompt gave a tie-free run with the rounds asked for")


KINDS = ["hs128-q4", "hs128-q4-compact", "hs128-w8", "hs128-w8-compact", "adapter-q4", "lora-q4"]


@pytest.mark.parametrize("num_draft", [1, 4, 15])
@pytest.mark.parametrize("kind", KINDS)
def test_greedy_lookup_equals_generate(dev, zoo, kind, num_draft):
    """Token for token against generate(top_k=1), and the recorded stats equal the simulated schedule, which holds a
    fully accepted, a partly accepted (num_draft >= 2), a fully rejected round and a lookup miss."""
    P = _P()
    model = zoo(kind)
    prompt, want, sim, _ = _case(P, model, dev, num_draft, 48)
    model.reset_cache()
    stats = {}
    got = P.generate_speculative(model, None, prompt, 48, num_draft=num_draft, top_k=1, stats=stats)
    model.reset_cache()
    assert got.dtype == want.dtype and torch.equal(got, want), (got.tolist(), want.tolist())
    assert stats == sim, (stats, sim)
    assert 1 + sum(a + 1 for a in stats["accepted"]) + stats["lookup_misses"] + stats["tail_steps"] == 48


def test_greedy_lookup_eos_and_tight_cache(dev, zoo):
    """With eos_id = each token value of the continuation, the output ends at its first occurrence (eos included),
    among them an eos in the middle of a round; and with max_seq_length 30 for 30 new tokens k shrinks as the cache
    fills and the tail rolls like generate()'s."""
    P = _P()
    model = zoo("hs128-q4-compact")
    prompt, want, sim, spans = _case(P, model, dev, 4, 40, cover=False, mid_eos=True)
    T = prompt.numel()
    y = want.tolist()
    firsts = [y.index(eos, T) for eos in sorted(set(y[T:]))]
    assert set(_mid_round_first(y, T, spans)) & set(firsts)   # an eos among a round's accepted tokens, not its last
    for first in firsts:
        model.reset_cache()
        got = P.generate_speculative(model, None, prompt, 40, num_draft=4, top_k=1, eos_id=y[first])
        assert torch.equal(got, want[:first + 1]), (y[first], got.tolist(), want[:first + 1].tolist())
    prompt, want, sim, _ = _case(P, model, dev, 4, 30, S=30, cover=False)
    model.reset_cache()
    stats = {}
    got = P.generate_speculative(model, None, prompt, 30, num_draft=4, top_k=1, max_seq_length=30, stats=stats)
    model.reset_cache()
    assert torch.equal(got, want), (got.tolist(), want.tolist())
    assert stats == sim and stats["tail_steps"] >= 30 - (30 - prompt.numel()) - 1 > 0, stats


def test_one_host_read_per_round(dev, zoo, monkeypatch):
    """Device-to-host reads (Tensor.item / tolist / bool / int / float) during generate_speculative(draft=None): one
    for the first proposal and one per round or lookup miss, beyond what generate()'s prefill and first token take."""
    P = _P()
    model = zoo("hs128-q4-compact")
    prompt, want, sim, _ = _case(P, model, dev, 4, 48)
    reads = [0]
    for name in ("item", "tolist", "__bool__", "__int__", "__float__", "__index__"):
        orig = getattr(torch.Tensor, name)

        def wrapped(self, *a, _orig=orig, **kw):
            if self.is_cuda:
                reads[0] += 1
            return _orig(self, *a, **kw)

        monkeypatch.setattr(torch.Tensor, name, wrapped)

    def count(fn):
        model.reset_cache()
        reads[0] = 0
        fn()
        return reads[0]

    count(lambda: P.generate_speculative(model, None, prompt, 48, num_draft=4, top_k=1))   # warm every graph
    base = count(lambda: P.generate(model, prompt, 1, max_seq_length=prompt.numel() + 48, top_k=1))
    stats = {}
    n = count(lambda: P.generate_speculative(model, None, prompt, 48, num_draft=4, top_k=1, stats=stats))
    model.reset_cache()
    assert stats == sim
    assert n == base + 1 + stats["rounds"] + stats["lookup_misses"], (n, base, stats)


def test_sampled_lookup_runs(dev, zoo):
    """Sampling at temperature 0.8 / top_k 50: the tokens are in range and the statistics add up."""
    P = _P()
    model = zoo("hs128-q4")
    prompt = torch.tensor([5, 6, 7, 5, 6, 7, 5, 6, 7, 5, 6], dtype=torch.int64, device=dev)
    model.reset_cache()
    torch.manual_seed(3)
    stats = {}
    y = P.generate_speculative(model, None, prompt, 40, num_draft=4, temperature=0.8, top_k=50, stats=stats)
    model.reset_cache()
    assert y.numel() == 51 and y.dtype == torch.int64 and torch.equal(y[:11], prompt)
    assert int(y.min()) >= 0 and int(y.max()) < model.config.vocab_size
    assert stats["rounds"] > 0
    assert 1 + sum(a + 1 for a in stats["accepted"]) + stats["lookup_misses"] + stats["tail_steps"] == 40

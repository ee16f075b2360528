"""Prompt-lookup speculative decoding on one GPU (`generate_speculative(draft=None)`), 7B gptq.int4 compacted,
`max_seq_length` 2048, synthetic weights.

1. Per-round cost components: `b2l_ngram_propose` at n = 256 / 2048 (CUDA events around many launches), for a history
   with no match (every g scans all n starts: the slowest case) and one whose last trigram occurred just before; and
   one whole lookup round (verify step, accept, next proposal and the round's one host read; host clock over rounds
   that end in that read) at T = 2..16 against one batch-1 step with its sampling launch (CUDA events), at positions
   ~64 / ~1024 / ~2000.
2. Best case: a greedy `generate()` output is known, so the proposer is handed a history in which the continuation
   already occurred (the known sequence, then the sequence again): every proposal is the known continuation and
   every round accepts all of it.  Random weights tie for the top logit at a few per cent of positions, and
   top_k = 1 then draws among the tied tokens, so a run would leave the known sequence at the first tie; the prompt
   is therefore picked (distinct random tokens, up to 40 seeds) so that its --best_new greedy tokens have no top-1
   tie in the teacher-forced logits.  Tokens/s against `generate(top_k=1)`, run alternately, medians.
3. Worst case: a prompt of distinct random tokens; tokens/s against `generate(top_k=1)`, and the miss count.

Acceptance on real text cannot be measured without checkpoints, so the script also evaluates the expected speedup
(1 - a^(k+1)) / (1 - a) * t_step / t_round(k + 1) at a few per-token acceptance rates a from the measured costs.  The
card name and power limit are read in the same run.  Prints one JSON object.

  python tools/lookup_bench.py [--new 256] [--best_new 48] [--reps 5] [--num_draft 4]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from spec_bench import card, timed  # noqa: E402

S = 2048


def propose_costs(L, dev, V, ns=(256, 2048), ks=(4, 15)):
    """{f"n={n} k={k} {kind}": us per b2l_ngram_propose launch}."""
    lib = L.lib()
    g = torch.Generator().manual_seed(5)
    q = torch.empty((15, V), dtype=torch.bfloat16, device=dev)
    tokens = torch.empty(16, dtype=torch.int64, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    res = {}
    for n in ns:
        nomatch = torch.randperm(32000, generator=g)[:n].to(dev)   # distinct ids: no n-gram recurs
        match = nomatch.clone()
        match[n - 20:n - 17] = match[n - 3:n]                       # the last trigram, 17 tokens earlier
        for kind, h in (("no match", nomatch), ("match", match)):
            for k in ks:
                def call():
                    L.check(lib.b2l_ngram_propose(h.data_ptr(), n, None, 1, 3, k, tokens.data_ptr(), q.data_ptr(),
                                                  count.data_ptr(), V, L.stream_ptr()), "b2l_ngram_propose")
                call()
                res[f"n={n} k={k} {kind}"] = round(timed(call, n=200) * 1000, 2)
    return res


def round_costs(P, L, model, dev, positions, Ts, n_rounds=20, reps=5):
    """{pos: {"step": ms of a batch-1 step + sampling, "T=t": ms of one lookup round verifying t tokens}}."""
    lib = L.lib()
    V = model.config.padded_vocab_size
    res = {}
    for pos in positions:
        model.reset_cache()
        model(torch.randint(0, V, (1, pos), device=dev), S, torch.arange(pos, device=dev))
        tok = torch.randint(0, V, (1,), device=dev)
        p1 = torch.tensor([pos], device=dev)
        r = {"step": timed(lambda: P.sample_token(model(tok.view(1, 1), S, p1)[0, -1], 1.0, 1))}
        out = torch.randint(0, V, (S + 32,), device=dev)
        q = torch.empty((15, V), dtype=torch.bfloat16, device=dev)
        dtok = torch.randint(0, V, (16, 1), device=dev)
        nacc = torch.zeros(1, dtype=torch.int32, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        steps = torch.arange(16, device=dev)
        for T in Ts:
            k = T - 1
            pp = torch.arange(pos, pos + T, device=dev)

            def one_round():   # generate_speculative's lookup round (without eos)
                vidx = torch.cat((tok.view(1, 1), dtok[:k].view(1, k)), dim=1)
                tl = model.decode_tokens(vidx, S, pp)
                u = torch.rand(k, device=dev)
                noise = torch.empty(V, dtype=torch.bfloat16, device=dev).exponential_(1)
                L.check(lib.b2l_spec_accept(tl.data_ptr(), V, 1.0, 1, q.data_ptr(), dtok.data_ptr(), u.data_ptr(),
                                            noise.data_ptr(), nacc.data_ptr(), dtok[k].data_ptr(), k + 1, V,
                                            L.stream_ptr()), "b2l_spec_accept")
                em = torch.where(steps[:k + 1] < nacc.long(), dtok[:k + 1, 0], dtok[k, 0])
                out[pos:pos + k + 1] = em
                dtok[k].clone()
                L.check(lib.b2l_ngram_propose(out.data_ptr(), pos, nacc.data_ptr(), 1, 3, 15, dtok.data_ptr(),
                                              q.data_ptr(), count.data_ptr(), V, L.stream_ptr()), "b2l_ngram_propose")
                return int((nacc.long()[0] | (count.long()[0] << 16)).to(torch.int32).item())

            one_round()
            one_round()
            ms = []
            for _ in range(reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(n_rounds):
                    one_round()
                ms.append((time.perf_counter() - t0) * 1000 / n_rounds)
            r[f"T={T}"] = statistics.median(ms)
        res[pos] = {key: round(v, 3) for key, v in r.items()}
    model.reset_cache()
    return res


class _Injected:
    """The library with b2l_ngram_propose reading `known` (the run's greedy output, prompt included) twice over, the
    live length counted from the second copy: while the run follows `known`, the last n-gram's most recent earlier
    occurrence lies in the first copy (barring repeats inside the sequence), so the proposal is the known
    continuation."""

    def __init__(self, real, known: torch.Tensor):
        self.real = real
        self.L = known.numel()
        self.buf = torch.cat((known.long(), known.long()))

    def __getattr__(self, name):
        return getattr(self.real, name)

    def b2l_ngram_propose(self, history, base_len, *rest):
        return self.real.b2l_ngram_propose(self.buf.data_ptr(), base_len + self.L, *rest)


def tie_free(model, prompt, y):
    """Whether no teacher-forced batch-1 step of the greedy sequence y (after `prompt`) ties for the top logit."""
    T, S_ = prompt.numel(), y.numel()
    model.reset_cache()
    tops = [model(prompt.view(1, -1), S_, torch.arange(T, device=y.device))[0, -1].float().topk(2).values]
    for i in range(T, S_ - 1):
        tops.append(model(y[i].view(1, 1), S_, torch.tensor([i], device=y.device))[0, -1].float().topk(2).values)
    model.reset_cache()
    t = torch.stack(tops)
    return not bool((t[:, 0] == t[:, 1]).any())


def e2e(P, L, model, prompt, n_new, reps, k, inject):
    """Alternated generate / generate_speculative(draft=None) runs at top_k = 1: median tokens/s of each, the last
    run's stats, and whether the outputs agree."""
    plain, spec, st = [], [], None
    real_lib = L.lib
    y = None
    for r in range(reps + 1):   # the first pair warms up
        for which in ("plain", "lookup"):
            model.reset_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stats = {}
            if which == "plain":
                y = P.generate(model, prompt, n_new, top_k=1)
            else:
                if inject:
                    known = _Injected(real_lib(), y)
                    L.lib = lambda: known
                try:
                    y2 = P.generate_speculative(model, None, prompt, n_new, num_draft=k, top_k=1, stats=stats)
                finally:
                    L.lib = real_lib
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if r > 0:
                (plain if which == "plain" else spec).append(n_new / dt)
            if which == "lookup":
                st = stats
    model.reset_cache()
    return dict(generate_tok_s=round(statistics.median(plain), 1), lookup_tok_s=round(statistics.median(spec), 1),
                speedup=round(statistics.median(spec) / statistics.median(plain), 3), rounds=st["rounds"],
                mean_accepted=round(sum(st["accepted"]) / max(1, st["rounds"]), 2),
                mean_proposed=round(sum(st["proposed"]) / max(1, st["rounds"]), 2), lookup_misses=st["lookup_misses"],
                tail_steps=st["tail_steps"], num_draft=k, tokens_equal=bool(torch.equal(y, y2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--positions", default="64,1024,2000")
    ap.add_argument("--Ts", default="2,3,4,5,8,12,16")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--best_new", type=int, default=48)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--num_draft", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lookup_bench: needs a GPU (no CPU timing is meaningful)")
    import __graft_entry__ as entry

    entry.build()
    import lit_llama_b200 as P
    from lit_llama_b200 import _lib as L
    from diag import _random_w8_model

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = _random_w8_model("7B", dev, seed=10, bits=4).compact()
    V = model.config.padded_vocab_size
    out = dict(card=card(), model="7B gptq.int4 compacted, synthetic weights", max_seq_length=S)
    out["propose_us"] = propose_costs(L, dev, V)
    print(json.dumps(out["propose_us"]), file=sys.stderr, flush=True)
    Ts = [int(t) for t in a.Ts.split(",")]
    out["round_ms"] = round_costs(P, L, model, dev, [int(p) for p in a.positions.split(",")], Ts)
    print(json.dumps(out["round_ms"]), file=sys.stderr, flush=True)
    k = a.num_draft
    out["best_case"] = None   # not measured: no tie-free candidate
    for seed in range(40):
        prompt = torch.randperm(32000, generator=torch.Generator().manual_seed(100 + seed))[:32].to(dev)
        model.reset_cache()
        if tie_free(model, prompt, P.generate(model, prompt, a.best_new, top_k=1)):
            out["best_case"] = dict(e2e(P, L, model, prompt, a.best_new, a.reps, k, inject=True), prompt_seed=100 + seed,
                                    new_tokens=a.best_new)
            break
    print(json.dumps(out["best_case"]), file=sys.stderr, flush=True)
    prompt = torch.randperm(32000, generator=torch.Generator().manual_seed(1))[:32].to(dev)   # distinct tokens
    out["worst_case"] = dict(e2e(P, L, model, prompt, a.new, a.reps, k, inject=False), new_tokens=a.new)
    c = out["round_ms"].get(1024)
    if c is not None and f"T={k + 1}" in c:
        out["expected_speedup_at_1024"] = {
            f"a={al}": round((1 - al ** (k + 1)) / (1 - al) * c["step"] / c[f"T={k + 1}"], 3) for al in (0.5, 0.7, 0.8, 0.9)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

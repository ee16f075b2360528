"""-m gpu: the packed refill into an fp8 KV cache (b2l_attention_ragged_kv8, LLaMA.refill_rows on kv_cache_dtype
"fp8"), bit for bit throughout.

1. Kernel: sequences of 2..256 tokens packed into one qkv, each sent into its own row of an fp8 cache holding stale
   codes and scales (NaN among them) with nonzero ring offsets, equal per-sequence B = 1 b2l_attention_kv8 prefills on
   a one-row cache (y, rotated qkv rows, every code and scale of the row); unnamed rows and their ring offsets stay
   byte for byte; named rings are 0.  At 32 and 40 heads, with and without the LLaMA-Adapter prefix.
2. The call captured in a CUDA graph and replayed equals the eager call.
3. refill_rows on an fp8 cache, packed and alone prompts mixed: logits and the whole KV store (codes and scales) equal
   the same calls with the pack plan emptied (every prompt alone), gptq.int4 and gptq.int8, plain and compacted; the
   packed route ran (calls of the binding counted).
4. The same for LLaMA-Adapter v1, LLaMA-Adapter v2 and multi-LoRA adapters= over a quantized base.
5. Batched decode (q4_batch_step / w8_batch_step) after a packed fp8 prefill_rows equals the batch-1 fp8 model past
   position 256.
6. Greedy generate_stream on fp8 with mid-decode refills that pack equals generate() per prompt.
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

CFG = dict(block_size=512, vocab_size=256, n_layer=2, n_head=4, n_embd=512)   # head_size 128


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as entry

    entry.build()
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _L():
    from lit_llama_b200 import _lib as L

    return L


def _K8():
    import test_gpu_kv8 as K8

    return K8


def _ragged(L, lengths, rows):
    sq = L.Ragged()
    sq.n_seq = len(lengths)
    at = 0
    for s, (n, r) in enumerate(zip(lengths, rows)):
        sq.row[s], sq.start[s], sq.len[s] = r, at, n
        at += n
    return sq


def _stale_cache(dev, B_rows, nh, S, seed):
    """An fp8 cache of random codes and scales, with NaN codes and NaN scales scattered through it."""
    K8 = _K8()
    c = K8.Cache8.random(dev, B_rows, nh, S, seed=seed)
    c.k.view(torch.uint8)[:, :, ::7, ::5] = 0x7f
    c.v.view(torch.uint8)[:, :, 3::11] = 0xff
    c.ks[:, :, 1::9] = math.nan
    c.vs[:, :, ::13] = math.nan
    return c


def _run_ragged(L, qkv, cache, rope, sq, ring, y, N, B_rows, nh, S, prefix):
    rc = L.lib().b2l_attention_ragged_kv8(qkv.data_ptr(), C.byref(cache.spec(L)), rope.data_ptr(), C.byref(sq),
                                          ring.data_ptr(), y.data_ptr(), N, B_rows, nh, 128, S, rope.shape[0],
                                          None if prefix is None else C.byref(prefix), L.stream_ptr())
    L.check(rc, "b2l_attention_ragged_kv8")


# --------------------------------------------------------------------------------------------- 1. kernel
@pytest.mark.parametrize("adapter", [False, True])
@pytest.mark.parametrize("nh", [32, 40])
def test_ragged_kv8_equals_batch1_prefills(dev, nh, adapter):
    L, K8 = _L(), _K8()
    lib = L.lib()
    S, B_rows = 256, 8
    lengths = [2, 63, 64, 65, 130, S]
    rows = [5, 0, 7, 2, 6, 3]            # rows 1 and 4 are not named
    N = sum(lengths)
    g = torch.Generator(device=dev).manual_seed(nh + adapter)
    qkv = torch.randn(1, N, 3 * nh * 128, device=dev, generator=g).bfloat16()
    stale = _stale_cache(dev, B_rows, nh, S, seed=nh)
    ring = torch.randint(1, S, (B_rows,), device=dev, generator=g).to(torch.int32)
    prefix = K8._prefix(dev, nh) if adapter else None
    rope = K8._rope(dev, S)
    q2, c2, r2 = qkv.clone(), stale.clone(), ring.clone()
    y = torch.full((1, N, nh * 128), float("nan"), device=dev, dtype=torch.bfloat16)
    _run_ragged(L, q2, c2, rope, _ragged(L, lengths, rows), r2, y, N, B_rows, nh, S, prefix)
    torch.cuda.synchronize()
    at = 0
    for n, r in zip(lengths, rows):
        q1 = qkv[:, at:at + n].clone()
        c1 = K8.Cache8(stale.k[r:r + 1].clone(), stale.ks[r:r + 1].clone(), stale.v[r:r + 1].clone(),
                       stale.vs[r:r + 1].clone())
        y1 = torch.empty((1, n, nh * 128), device=dev, dtype=torch.bfloat16)
        ring1 = torch.zeros(1, dtype=torch.int32, device=dev)
        L.check(lib.b2l_attention_kv8(q1.data_ptr(), C.byref(c1.spec(L)), rope.data_ptr(), None, ring1.data_ptr(),
                                      y1.data_ptr(), K8._work(L, 1, nh, S, dev, n).data_ptr(), 1, n, nh, 128, S,
                                      rope.shape[0], 0, None if prefix is None else C.byref(prefix), L.stream_ptr()),
                "b2l_attention_kv8")
        torch.cuda.synchronize()
        assert K8._bits_equal(y[:, at:at + n], y1), (n, r)
        assert K8._bits_equal(q2[:, at:at + n], q1), (n, r)   # q and k rotated in place, v untouched, as at B = 1
        for a, b in ((c2.k, c1.k), (c2.v, c1.v), (c2.ks, c1.ks), (c2.vs, c1.vs)):
            assert K8._bits_equal(a[r], b[0]), (n, r)          # slots < n written alike, slots >= n left alike
        assert int(r2[r]) == 0
        at += n
    for r in (1, 4):
        for a, b in ((c2.k, stale.k), (c2.v, stale.v), (c2.ks, stale.ks), (c2.vs, stale.vs)):
            assert K8._bits_equal(a[r], b[r]), r
        assert int(r2[r]) == int(ring[r]), r
    assert not torch.isnan(y).any()


# --------------------------------------------------------------------------------------------- 2. graph capture
def test_graph_replay_equals_eager(dev):
    L, K8 = _L(), _K8()
    nh, S, B_rows = 8, 192, 4
    lengths, rows = [2, 70, 129], [1, 3, 0]
    N = sum(lengths)
    g = torch.Generator(device=dev).manual_seed(7)
    qkv = torch.randn(1, N, 3 * nh * 128, device=dev, generator=g).bfloat16()
    stale = _stale_cache(dev, B_rows, nh, S, seed=8)
    ring = torch.tensor([5, 6, 7, 8], dtype=torch.int32, device=dev)
    rope, prefix, sq = K8._rope(dev, S), K8._prefix(dev, nh), _ragged(L, lengths, rows)
    q_e, c_e, r_e = qkv.clone(), stale.clone(), ring.clone()
    y_e = torch.empty((1, N, nh * 128), device=dev, dtype=torch.bfloat16)
    _run_ragged(L, q_e, c_e, rope, sq, r_e, y_e, N, B_rows, nh, S, prefix)
    q_g, c_g, r_g = qkv.clone(), stale.clone(), ring.clone()
    y_g = torch.empty_like(y_e)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _run_ragged(L, q_g, c_g, rope, sq, r_g, y_g, N, B_rows, nh, S, prefix)
    for _ in range(2):   # capture enqueues nothing: each replay starts from the original inputs
        q_g.copy_(qkv)
        for a, b in ((c_g.k, stale.k), (c_g.v, stale.v), (c_g.ks, stale.ks), (c_g.vs, stale.vs)):
            a.view(torch.uint8).copy_(b.view(torch.uint8))
        r_g.copy_(ring)
        y_g.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert K8._bits_equal(y_g, y_e) and K8._bits_equal(q_g, q_e) and torch.equal(r_g, r_e)
        for a, b in ((c_g.k, c_e.k), (c_g.v, c_e.v), (c_g.ks, c_e.ks), (c_g.vs, c_e.vs)):
            assert K8._bits_equal(a, b)


# --------------------------------------------------------------------------------------------- 3. / 4. refill_rows
FIRST, REFILL, REFILL_ROWS = (17, 3, 40, 1), (25, 60, 2, 16), [2, 0, 3, 1]


def _prompts(dev, V, lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, V, (n,), generator=g).to(torch.int32).to(dev) for n in lengths]


def _counting(monkeypatch):
    """Counts the calls of b2l_attention_ragged_kv8 (the packed fp8 route) from here on."""
    lib = _L().lib()
    real = lib.b2l_attention_ragged_kv8
    calls = [0]

    def counted(*a):
        calls[0] += 1
        return real(*a)

    monkeypatch.setattr(lib, "b2l_attention_ragged_kv8", counted)
    return calls


def _fp8_refills(model, dev, S, monkeypatch, adapters=None):
    """prefill_rows(FIRST) then refill_rows(REFILL) on an fp8 cache, packed and then with the pack plan emptied: the
    logits, KV store bytes, scales and ring offsets of both runs, and the packed run's count of ragged fp8 calls."""
    V = model.config.vocab_size
    first, refill = _prompts(dev, V, FIRST, seed=31), _prompts(dev, V, REFILL, seed=32)
    a1 = None if adapters is None else adapters[:len(first)]
    a2 = None if adapters is None else adapters[len(first):]
    model.reset_cache()
    model.kv_cache_dtype = "fp8"
    runs = []
    for packed in (True, False):
        calls = _counting(monkeypatch)
        if not packed:
            monkeypatch.setattr(model, "_pack_plan", lambda lengths: [])
        model.reset_cache()
        with torch.no_grad():
            lg = torch.cat([model.prefill_rows(first, S, a1), model.refill_rows(refill, REFILL_ROWS, S, a2)])
        torch.cuda.synchronize()
        runs.append((lg, model._kv_store.view(torch.uint8).clone(), model._kv_scale.clone(), model._ring.clone(),
                     calls[0]))
        monkeypatch.undo()
    model.reset_cache()
    return runs


def _assert_same(runs, want_calls):
    (lg, st, sc, ring, n), (lg1, st1, sc1, ring1, n1) = runs
    assert n == want_calls and n1 == 0, (n, n1)
    assert torch.equal(lg, lg1)
    assert torch.equal(st, st1)
    assert torch.equal(sc.view(torch.int32), sc1.view(torch.int32))
    assert torch.equal(ring, ring1) and not bool(ring.any())


def _plans(model):
    return model._pack_plan(list(FIRST)), model._pack_plan(list(REFILL))


@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_refill_rows_packed_equals_alone(dev, mode, compact, monkeypatch):
    from gpu_util import build_tiny

    model, _, _ = build_tiny(dev, CFG, mode=mode, seed=41)
    if compact:
        model.compact()
    p1, p2 = _plans(model)
    assert (p1, p2) == (([0, 2], [0, 1]) if mode == "gptq.int4" else ([0, 1, 2], [0, 1, 2, 3]))
    runs = _fp8_refills(model, dev, 64, monkeypatch)
    _assert_same(runs, 2 * model.config.n_layer)   # one call per layer per packed pass


@pytest.mark.parametrize("kind", ["adapter", "adapter_v2", "multi_lora"])
def test_variants_packed_equals_alone(dev, kind, monkeypatch):
    adapters = None
    if kind == "adapter":
        import test_gpu_adapter as TA

        model, _, _ = TA.build(dev, TA.CFG128, "gptq.int4")
    elif kind == "adapter_v2":
        import test_gpu_adapter_v2 as TV

        model, _, _ = TV.build(dev, TV.CFG128, "gptq.int4")
    else:
        import test_gpu_multi_lora as TM

        model = TM._multi(dev, "gptq.int4", TM.TINY, 3)
        adapters = [1, 0, 3, -1, 2, 1, -1, 3]
    assert _plans(model) == ([0, 2], [0, 1])
    runs = _fp8_refills(model, dev, 60, monkeypatch, adapters)
    _assert_same(runs, 2 * model.config.n_layer)


# --------------------------------------------------------------------------------------------- 5. decode after a refill
@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_batched_decode_after_packed_prefill_equals_batch1(dev, mode, monkeypatch):
    from gpu_util import build_tiny

    K8 = _K8()
    prompts = _prompts(dev, CFG["vocab_size"], (270, 300, 40, 5), seed=51)
    S = 512
    model, _, _ = build_tiny(dev, CFG, mode=mode, seed=52)
    model.compact()
    model.q4_batch_step = model.w8_batch_step = True
    model.kv_cache_dtype = "fp8"
    assert model._pack_plan([p.numel() for p in prompts]) == ([0, 1, 2] if mode == "gptq.int4" else [0, 1, 2, 3])
    calls = _counting(monkeypatch)
    with torch.no_grad():
        rows = [model.prefill_rows(prompts, S)]
        assert calls[0] == model.config.n_layer
        pos = torch.tensor([[p.numel()] for p in prompts], device=dev)
        toks = rows[0].argmax(-1).view(-1, 1).to(torch.int32)
        for _ in range(8):
            lg = model(toks, S, pos)[:, -1].float()
            rows.append(lg.clone())
            toks, pos = lg.argmax(-1).view(-1, 1).to(torch.int32), pos + 1
        assert model._decode.args.flags & _L().F_KV_FP8
        for b, p in enumerate(prompts):
            model.reset_cache()
            one = K8._decode(model, p, 8, S, dev)
            for i in range(9):
                assert torch.equal(rows[i][b].float(), one[i]), (b, i)


# --------------------------------------------------------------------------------------------- 6. generate_stream
def _first_argmax(probs, num_samples):
    """Greedy with ties broken to the lowest token id (tests/test_gpu_stream.py)."""
    return probs.argmax(dim=-1, keepdim=True)


@pytest.mark.parametrize("mode", ["gptq.int4", "gptq.int8"])
def test_greedy_stream_on_fp8_equals_generate(dev, mode, monkeypatch):
    import lit_llama_b200 as P
    from gpu_util import build_tiny

    monkeypatch.setattr(torch, "multinomial", _first_argmax)
    model, _, _ = build_tiny(dev, CFG, mode=mode, seed=61)
    model.q4_batch_step = model.w8_batch_step = True
    model.kv_cache_dtype = "fp8"
    lengths, news, S = (17, 30, 45, 20, 33, 18, 25, 40), (6, 20, 4, 12, 5, 9, 3, 7), 96
    prompts = _prompts(dev, CFG["vocab_size"], lengths, seed=62)
    calls = _counting(monkeypatch)
    stats = {}
    with torch.no_grad():
        model.reset_cache()
        ys = P.generate_stream(model, prompts, list(news), batch_size=3, max_seq_length=S, top_k=1, stats=stats)
        n_stream = calls[0]
        assert stats["refills"] == len(prompts) - 3 and stats["packed"] > 0, stats
        assert n_stream >= 2 * model.config.n_layer   # the first prefill and at least one mid-decode refill packed
        for p, m, y in zip(prompts, news, ys):
            model.reset_cache()
            want = P.generate(model, p, m, max_seq_length=S, top_k=1)
            assert torch.equal(y, want), (p.numel(), m)
    print(f"{mode}: {stats}, {n_stream // model.config.n_layer} packed passes")

"""-m gpu: llm.int8 keeps one resident copy of its weights.  The batch-1 kernel reads CB directly (b2l_q8_gemv_cb), so
Linear8bitLt never builds the re-tiled copy b2l_q8_gemv needs, and LLaMA-65B fits on one 80 GB GPU.

b2l_q8_gemv_cb contracts the same int8 values in the same order as b2l_q8_gemv on b2l_q8_tile(CB), so every comparison
with that path is torch.equal."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_int8_gemm import _activations  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _tiled_gemv(L, x, cb, scb, mask, N, K, flags=0):
    """The parent's batch-1 path: b2l_q8_gemv on a freshly re-tiled copy of CB."""
    lib = L.lib()
    wt = torch.empty(lib.b2l_q8_tiled_bytes(N, K), dtype=torch.uint8, device=x.device)
    L.check(lib.b2l_q8_tile(cb.data_ptr(), wt.data_ptr(), N, K, L.stream_ptr()), "tile")
    y = torch.full((N,), float("nan"), dtype=torch.bfloat16, device=x.device)
    L.check(lib.b2l_q8_gemv(x.data_ptr(), wt.data_ptr(), cb.data_ptr(), scb.data_ptr(), None if mask is None else mask.data_ptr(),
                            y.data_ptr(), N, K, 6.0, flags, L.stream_ptr()), "b2l_q8_gemv")
    return y


def _cb_gemv(L, x, cb, scb, mask, N, K, flags=0):
    y = torch.full((N + 8,), float("nan"), dtype=torch.bfloat16, device=x.device)
    L.check(L.lib().b2l_q8_gemv_cb(x.data_ptr(), cb.data_ptr(), scb.data_ptr(), None if mask is None else mask.data_ptr(), y.data_ptr(),
                                   N, K, 6.0, flags, L.stream_ptr()), "b2l_q8_gemv_cb")
    assert bool(torch.isnan(y[N:]).all())   # nothing written past N
    return y[:N]


# Every N and every K of the sweep appears at least once.  N = 48 and 130 (3 and 9 row blocks, N not a multiple of 16)
# give fewer row blocks than CTAs; K = 128, 11008, 13824 and 22016 end on a short stage (K / 128 not a multiple of 8);
# K = 32768 runs one CTA per SM.
@pytest.mark.parametrize("N,K", [
    (48, 128), (48, 32768), (130, 1024), (130, 22016), (4096, 4096), (4096, 11008), (4096, 32768), (12288, 4096),
    (12288, 13824), (32000, 4096), (32000, 1024), (130, 13824),
])
def test_gemv_cb_equals_tiled(dev, N, K):
    from lit_llama_b200 import _lib as L

    lib = L.lib()
    g = torch.Generator().manual_seed(N * 5 + K)
    cb = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).to(dev)
    scb = (torch.rand(N, generator=g) * 0.2 + 0.01).to(dev)
    for pattern in ("none", "few", "allrow", "exact6"):
        x = _activations(3, K, pattern, g)[1].contiguous().to(dev)   # the middle row: "allrow" makes every column an outlier
        # a batch mask: this row's outliers plus another row's, so it differs from what the kernel derives itself
        other = _activations(2, K, "few", g)[0].to(dev)
        mask = torch.empty((K + 31) // 32, dtype=torch.int32, device=dev)
        L.check(lib.b2l_q8_outlier_mask(torch.stack([x, other]).data_ptr(), K, 2, K, 6.0, mask.data_ptr(), L.stream_ptr()), "mask")
        for m in (None, mask):
            for flags in (0, L.F_PDL):
                want = _tiled_gemv(L, x, cb, scb, m, N, K, flags)
                got = _cb_gemv(L, x, cb, scb, m, N, K, flags)
                torch.cuda.synchronize()
                assert bool(torch.isfinite(want).all())
                assert torch.equal(got, want), (pattern, m is not None, flags, int((got != want).sum()))


@pytest.mark.parametrize("K,N", [(4096, 11008), (13824, 5120)])
def test_linear8bitlt_batch1_reads_cb(dev, K, N):
    """Linear8bitLt at M = 1 gives the parent's per-row result and never builds the re-tiled copy."""
    import lit_llama_b200 as P
    from lit_llama_b200 import _lib as L

    g = torch.Generator().manual_seed(K + N)
    lin = P.Linear8bitLt(K, N, bias=False)
    lin.load_state_dict({"weight": torch.randn(N, K, generator=g) * 0.02})
    lin = lin.to(dev)
    x = _activations(1, K, "few", g).to(dev)
    got = lin(x.view(1, 1, K))
    assert lin._tiled is None
    want = _tiled_gemv(L, x[0], lin.weight.CB, lin.weight.SCB, None, N, K)
    assert got.shape == (1, 1, N)
    assert torch.equal(got.view(N), want)


def _tiled_forward(cb_forward):
    """Linear8bitLt.forward as it was before b2l_q8_gemv_cb: b2l_q8_gemv on the cached re-tiled copy at M = 1."""
    from lit_llama_b200 import _lib as L

    def forward(self, x):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        if x2.shape[0] != 1:
            return cb_forward(self, x)
        y = torch.empty(self.out_features, dtype=x.dtype, device=x.device)
        L.check(L.lib().b2l_q8_gemv(x2.data_ptr(), self.tiled().data_ptr(), self.weight.data.data_ptr(), self.weight.SCB.data_ptr(), None,
                                    y.data_ptr(), self.out_features, self.in_features, self.threshold, 0, L.stream_ptr()), "b2l_q8_gemv")
        return y.reshape(*shape[:-1], self.out_features)

    return forward


def _count_replays(mp):
    """Counts CUDA graph replays while `mp` is active: a decode step the module graph serves is one replay, one it
    launches module by module is none."""
    n = [0]
    replay = torch.cuda.CUDAGraph.replay

    def counted(self):
        n[0] += 1
        return replay(self)

    mp.setattr(torch.cuda.CUDAGraph, "replay", counted)
    return n


def _int8_linears(model):
    import lit_llama_b200 as P

    return [m for m in model.modules() if isinstance(m, P.Linear8bitLt)]


def test_llm_int8_13b_widths_one_resident_copy(dev, monkeypatch):
    """--quantize llm.int8 at the 13B widths (2 Blocks, n_embd 5120, n_hidden 13824), batch 1: a 32-token prefill, then
    6 decode steps with the module graph replaying.  Every logits tensor is bit-identical to the parent's tiled batch-1
    path, no Linear8bitLt holds a re-tiled copy, and live device memory is the weights, their scales, the embedding, the
    norms and the KV store plus a small slack."""
    import lit_llama_b200 as P
    from gpu_util import build_tiny

    cfg = dict(block_size=64, vocab_size=512, n_layer=2, n_head=40, n_embd=5120)
    g = torch.Generator().manual_seed(3)
    T, S = 32, 48
    prompt = torch.randint(0, 512, (1, T), generator=g)
    steps = [torch.randint(0, 512, (1, 1), generator=g) for _ in range(6)]

    def run(check_memory):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        model, _, _ = build_tiny(dev, cfg, mode="llm.int8", seed=7)
        with torch.no_grad(), monkeypatch.context() as mp:
            got = [model(prompt.to(dev), S, torch.arange(T, device=dev)).float().cpu()]
            replays = _count_replays(mp)
            for i, t in enumerate(steps):
                got.append(model(t.to(dev), S, torch.tensor([T + i], device=dev)).float().cpu())
        # the first graph_after steps run module by module; the graph is captured on the next and serves every later one
        assert replays[0] == len(steps) - model.graph_after > 0, replays
        if check_memory:
            lins = _int8_linears(model)
            assert all(m._tiled is None for m in lins)
            torch.cuda.synchronize()
            live = torch.cuda.memory_allocated() - base
            params = sum(p.numel() * p.element_size() for p in model.parameters())   # every CB, the embedding, the norms
            scb = sum(m.weight.SCB.numel() * 4 for m in lins)
            kv = model._kv_store.numel() * model._kv_store.element_size()
            cb = sum(m.weight.numel() for m in lins)
            # Slack: the module graph's private pool holds one token's activations (the widest is n_hidden = 13824 bf16
            # values, well under 1 MiB for all of them together), plus the RoPE table, the ring counter and the static
            # idx / pos / logits buffers, each under 1 MiB.  16 MiB covers all of it with room, and is far below the
            # re-tiled copy the parent held next to CB (as many bytes as CB: ~634 MB here).
            slack = 16 << 20
            assert live <= params + scb + kv + slack, (live, params, scb, kv, cb)
        del model
        torch.cuda.empty_cache()
        return got

    got = run(True)
    with monkeypatch.context() as mp:
        mp.setattr(P.Linear8bitLt, "forward", _tiled_forward(P.Linear8bitLt.forward))
        tiled = run(False)
    assert len(got) == len(tiled) == 7
    for i, (a, b) in enumerate(zip(got, tiled)):
        assert torch.equal(a, b), i


def test_llm_int8_65b_fits_one_gpu(dev, monkeypatch):
    """Full-size LLaMA-65B under --quantize llm.int8 on one GPU: a 16-token prefill and 8 batch-1 decode steps at
    max_seq_length 2048, the decode replayed from the module graph, within the memory the weights and the KV cache
    need."""
    import lit_llama_b200 as P
    from lit_llama_b200.utils import quantization

    c = P.LLaMAConfig.from_name("65B")
    S, T = 2048, 16
    C, H, V = c.n_embd, P.find_multiple(int(2 * 4 * c.n_embd / 3), 256), c.padded_vocab_size
    int8 = c.n_layer * (4 * C * C + 3 * C * H) + V * C                           # every CB (lm_head included)
    scb = 4 * (c.n_layer * (5 * C + 2 * H) + V)
    bf16 = 2 * (V * C + (2 * c.n_layer + 1) * C)                                  # embedding and norms
    kv = 2 * c.n_layer * 2 * c.n_head * S * (C // c.n_head)
    # Slack: the peak comes after the build, once the 5 GiB KV cache exists; the build's own transients (one weight in
    # float and its quantisation temporaries, about 3 GiB for a 22016 x 8192 MLP weight) sit below it.  What is left is
    # the prefill's activations and GEMM workspace and the module graph's pool, a few MiB at 16 tokens; 2 GiB covers
    # them with room and is far below the 60.6 GiB a second copy of the weights would take.
    budget = int8 + scb + bf16 + kv + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < budget + (1 << 30):
        pytest.skip(f"{free / 2**30:.1f} GiB free on the GPU; LLaMA-65B llm.int8 needs {budget / 2**30:.1f} GiB")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device(dev), quantization("llm.int8"):
            model = P.LLaMA.from_name("65B")
    finally:
        torch.set_default_dtype(prev)
    try:
        model.eval()
        assert sum(m.weight.numel() for m in _int8_linears(model)) == int8
        g = torch.Generator().manual_seed(65)
        prompt = torch.randint(0, V, (1, T), generator=g)
        with torch.no_grad(), monkeypatch.context() as mp:
            out = [model(prompt.to(dev), S, torch.arange(T, device=dev))]
            replays = _count_replays(mp)
            for i in range(8):
                out.append(model(torch.randint(0, V, (1, 1), generator=g).to(dev), S, torch.tensor([T + i], device=dev)).clone())
        torch.cuda.synchronize()
        assert replays[0] == 8 - model.graph_after > 0, replays
        assert all(bool(torch.isfinite(o.float()).all()) for o in out)
        assert all(m._tiled is None for m in _int8_linears(model))
        peak = torch.cuda.max_memory_allocated() - base
        assert peak <= budget, (peak / 2**30, budget / 2**30)
    finally:
        del model
        torch.cuda.empty_cache()

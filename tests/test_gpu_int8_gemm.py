"""-m gpu: the llm.int8 linear for M >= 2 rows (b2l_q8_gemm, csrc/q8_gemm.cu) and the batch-1 kernel beyond
K = 12288.

The GEMM is bit-identical per row to b2l_q8_gemv given the batch's outlier mask (the per-row path it
replaces), so it is compared with torch.equal.  Against the oracle restatement the bars are those of
test_gpu_quant.py::test_int8_linear_vs_oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import llama_oracle as O  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def _activations(M, K, pattern, g):
    x = torch.randn(M, K, generator=g)
    if pattern == "few":        # a few outlier columns, spread over the rows
        for i in range(5):
            x[(3 * i) % M, (37 * i + 11) % K] = 7.5 + i
            x[(5 * i + 1) % M, (101 * i + 3) % K] = -(6.5 + i)
    elif pattern == "allrow":   # one row with every column an outlier: every column is, so every SCA = 0
        x[M // 2] = 8.0 * torch.sign(torch.randn(K, generator=g))
    elif pattern == "exact6":   # |a| == threshold is an outlier, just below is not
        x[0, 5] = 6.0
        x[M - 1, K - 1] = -6.0
        x[M // 2, K // 2] = 5.96875    # largest bf16 below 6
    return x.bfloat16()


def _per_row(L, x, wt, cb, scb, N, K):
    """What Linear8bitLt computed before b2l_q8_gemm: b2l_q8_gemv on each row with the batch's outlier mask."""
    lib = L.lib()
    M = x.shape[0]
    mask = torch.empty((K + 31) // 32, dtype=torch.int32, device=x.device)
    L.check(lib.b2l_q8_outlier_mask(x.data_ptr(), K, M, K, 6.0, mask.data_ptr(), L.stream_ptr()), "mask")
    y = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
    for m in range(M):
        L.check(lib.b2l_q8_gemv(x[m].data_ptr(), wt.data_ptr(), cb.data_ptr(), scb.data_ptr(), mask.data_ptr(), y[m].data_ptr(),
                                N, K, 6.0, 0, L.stream_ptr()), "gemv")
    return y


def _gemm(L, x, cb, scb, N, K, ldy=None):
    lib = L.lib()
    M = x.shape[0]
    ldy = ldy or N
    nbytes = lib.b2l_q8_gemm_workspace_bytes(M, K)
    work = torch.full((nbytes,), 0x55, dtype=torch.uint8, device=x.device)   # stale contents must not matter
    y = torch.full((M, ldy), float("nan"), dtype=torch.bfloat16, device=x.device)
    L.check(lib.b2l_q8_gemm(x.data_ptr(), K, cb.data_ptr(), scb.data_ptr(), work.data_ptr(), nbytes, y.data_ptr(), ldy, M, N, K, 6.0, 0,
                            L.stream_ptr()), "b2l_q8_gemm")
    if ldy > N:
        assert bool(torch.isnan(y[:, N:]).all())   # nothing written past N
    return y[:, :N]


@pytest.mark.parametrize("N,K,M,pattern", [
    (48, 128, 2, "none"), (48, 128, 3, "few"), (130, 1024, 8, "few"), (130, 1024, 17, "exact6"), (130, 128, 300, "allrow"),
    (4096, 4096, 2, "few"), (4096, 4096, 64, "none"), (4096, 1024, 1024, "few"), (48, 22016, 3, "allrow"), (13824, 4096, 17, "few"),
    (4096, 13824, 8, "exact6"), (130, 22016, 300, "few"), (13824, 128, 1024, "none"), (4096, 22016, 64, "few"), (48, 13824, 2, "exact6"),
    (13824, 13824, 3, "none"), (4096, 1024, 300, "exact6"), (130, 4096, 1024, "allrow"),
])
def test_q8_gemm_equals_per_row_gemv(dev, N, K, M, pattern):
    from lit_llama_b200 import _lib as L

    g = torch.Generator().manual_seed(N * 7 + K * 3 + M)
    cb = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8).to(dev)
    scb = (torch.rand(N, generator=g) * 0.2 + 0.01).to(dev)
    x = _activations(M, K, pattern, g).to(dev)
    wt = torch.empty(L.lib().b2l_q8_tiled_bytes(N, K), dtype=torch.uint8, device=dev)
    L.check(L.lib().b2l_q8_tile(cb.data_ptr(), wt.data_ptr(), N, K, L.stream_ptr()), "tile")
    want = _per_row(L, x, wt, cb, scb, N, K)
    got = _gemm(L, x, cb, scb, N, K, ldy=N + 8 if M == 3 else None)
    torch.cuda.synchronize()
    assert torch.equal(got, want), (int((got != want).sum()), got.numel())


@pytest.mark.parametrize("N,K", [(13824, 5120), (5120, 13824), (6656, 17920), (8192, 22016)])
@pytest.mark.parametrize("M", [1, 4, 512])
def test_large_k_int8_linear_vs_oracle(dev, N, K, M):
    """Linear8bitLt at the 13B, 30B and 65B widths (batch-1 kernel for M = 1, the GEMM otherwise) against the
    oracle restatement, with a few outlier columns."""
    import lit_llama_b200 as P

    g = torch.Generator().manual_seed(N + K + M)
    w = torch.randn(N, K, generator=g) * 0.03
    x = torch.randn(M, K, generator=g)
    for i in range(3):
        x[i % M, (37 * i + 11) % K] = 7.5 + i
    lin = P.Linear8bitLt(K, N, bias=False)
    lin.load_state_dict({"weight": w})
    cb, scb = O.int8_quantize_weight(w)
    lin = lin.to(dev)
    xb = x.bfloat16()
    y = lin(xb.to(dev)).float().cpu()
    want = O.int8_linear(xb, cb, scb).float()
    exact = xb.float() @ w.t()
    assert (y - want).norm() / want.norm() < 2e-3, float((y - want).norm() / want.norm())
    torch.testing.assert_close(y, want, rtol=2 ** -6, atol=2e-2 * float(want.abs().max()) * 0.1 + 1e-3)
    assert (y - exact).norm() / exact.norm() < 3e-2


def test_linear8bitlt_gemm_path_equals_per_row(dev):
    """Linear8bitLt.forward for a (2, 8, K) input goes through one b2l_q8_gemm call and gives exactly the per-row result."""
    import lit_llama_b200 as P
    from lit_llama_b200 import _lib as L

    g = torch.Generator().manual_seed(11)
    K, N = 4096, 11008
    lin = P.Linear8bitLt(K, N, bias=False)
    lin.load_state_dict({"weight": torch.randn(N, K, generator=g) * 0.02})
    lin = lin.to(dev)
    x = _activations(16, K, "few", g).to(dev)
    got = lin(x.view(2, 8, K))
    want = _per_row(L, x, lin.tiled(), lin.weight.CB, lin.weight.SCB, N, K)
    assert got.shape == (2, 8, N)
    assert torch.equal(got.view(16, N), want)


def _per_row_forward(gemm_forward):
    """Linear8bitLt.forward as it was before b2l_q8_gemm: b2l_q8_gemv per row with the batch mask."""
    from lit_llama_b200 import _lib as L

    def forward(self, x):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        if x2.shape[0] == 1:
            return gemm_forward(self, x)
        y = _per_row(L, x2, self.tiled(), self.weight.data, self.weight.SCB, self.out_features, self.in_features)
        return y.reshape(*shape[:-1], self.out_features)

    return forward


@pytest.mark.parametrize("n_layer,n_head,n_embd", [(2, 40, 5120), (1, 52, 6656)])
def test_llm_int8_wide_batch2_prefill_and_decode(dev, monkeypatch, n_layer, n_head, n_embd):
    """--quantize llm.int8 at the 13B widths (2 Blocks, n_hidden 13824) and the 30B widths (1 Block, n_hidden 17920):
    batch 2, a 32-token prefill (GEMM at M = 64), then 6 decode steps (GEMM at M = 2, replayed as a CUDA graph).

    Every logits tensor is bit-identical to the per-row path the GEMM replaced.  Against the oracle restatement the
    bars are wider than the tiny model's: at these widths a one-ulp difference in a bf16 activation moves int8 levels,
    and llm.int8 itself is ~5e-2 normwise from the unquantised model here.  Measured on an H100: 0.023-0.050 normwise
    from the restatement, 0.020-0.058 per sequence; the restatement is 0.047-0.056 from the unquantised (bf16 dense)
    model and the CUDA path is within 5 % of that distance."""
    import lit_llama_b200 as P
    from gpu_util import build_tiny

    cfg = dict(block_size=64, vocab_size=512, n_layer=n_layer, n_head=n_head, n_embd=n_embd)
    g = torch.Generator().manual_seed(1)
    B, T, S = 2, 32, 40
    prompt = torch.randint(0, 512, (B, T), generator=g)
    steps = [torch.randint(0, 512, (B, 1), generator=g) for _ in range(6)]

    def run():
        model, oracle, sd = build_tiny(dev, cfg, mode="llm.int8", seed=5)
        with torch.no_grad():
            got = [model(prompt.to(dev), S, torch.arange(T, device=dev)).float().cpu()]
            for i, t in enumerate(steps):
                got.append(model(t.to(dev), S, torch.tensor([T + i], device=dev)).float().cpu())
        assert model._module_graph is not None and model._module_graph["graph"] is not None
        return got, oracle, sd

    got, oracle, sd = run()
    with monkeypatch.context() as mp:
        mp.setattr(P.Linear8bitLt, "forward", _per_row_forward(P.Linear8bitLt.forward))
        per_row, _, _ = run()
    dense = O.OracleLLaMA.from_state_dict(sd, n_layer, n_head, cfg["block_size"], None)
    rel = lambda a, b: float((a - b).norm() / b.norm())
    for i, (a, b) in enumerate(zip(got, per_row)):
        assert torch.equal(a, b), i
    for j in range(len(got)):
        pos = torch.arange(T) if j == 0 else torch.tensor([T + j - 1])
        idx = prompt if j == 0 else steps[j - 1]
        want = oracle.forward(idx, S, pos).float()
        exact = dense.forward(idx, S, pos).float()
        a = got[j]
        assert a.shape == want.shape
        assert rel(a, want) < 6e-2, (j, rel(a, want))
        for r in range(B):   # every sequence on its own: a row mix-up cannot hide in the batch norm
            assert rel(a[r], want[r]) < 8e-2, (j, r, rel(a[r], want[r]))
        assert rel(a, exact) < 1.15 * rel(want, exact), (j, rel(a, exact), rel(want, exact))

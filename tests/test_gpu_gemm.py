"""wgmma weight-streaming GEMM (csrc/gemm_tc.cu) against a plain fp32 torch matmul of the same bf16
operands.  Tolerance: fp32 accumulation of bf16 products -> 1e-4 relative to the row scale."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def run_gemm(W, X, W_lo=None, split_k=0):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    M, K = X.shape
    N = W.shape[0]
    if split_k == 0:
        split_k = lib.prl_gemm_auto_split_k(M, N, K)
    part = torch.full((split_k, M, N), float("nan"), dtype=torch.float32, device=X.device)
    _lib.check(lib.prl_gemm_bf16_splitk(W.data_ptr(), W_lo.data_ptr() if W_lo is not None else None, X.data_ptr(),
                                        M, N, K, split_k, part.data_ptr(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return part


SHAPES = [
    (1, 128, 64, 1), (16, 256, 128, 2), (37, 300, 200, 1), (64, 4608, 3584, 0), (64, 3584, 18944, 0),
    (33, 1152, 512, 3), (128, 640, 1024, 2), (200, 384, 256, 1), (300, 256, 192, 1), (64, 37888, 3584, 0),
    # M > 128: 256-token tiles with ragged token / feature / k tails, split-K, many k-blocks
    (129, 128, 64, 1), (513, 777, 200, 1), (256, 512, 4096, 2), (1024, 4608, 3584, 1), (700, 1000, 1288, 3),
]


@pytest.mark.parametrize("M,N,K,split_k", SHAPES)
def test_gemm_matches_fp32_matmul(cuda_device, M, N, K, split_k):
    g = torch.Generator().manual_seed(M * 131 + N * 7 + K)
    X = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(cuda_device)
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(cuda_device)
    part = run_gemm(W, X, split_k=split_k)
    assert torch.isfinite(part).all(), "unwritten partial tile"
    got = part.sum(0)
    want = X.float() @ W.float().t()
    scale = want.abs().max().item()
    assert (got - want).abs().max().item() <= 2e-4 * scale + 1e-6


def test_gemm_hi_lo_is_fp32_equivalent(cuda_device):
    g = torch.Generator().manual_seed(3)
    M, N, K = 48, 1024, 1536
    Wf = (torch.randn(N, K, generator=g) * 0.02).to(cuda_device)
    hi = Wf.to(torch.bfloat16)
    lo = (Wf - hi.float()).to(torch.bfloat16)
    X = (torch.randn(M, K, generator=g)).to(torch.bfloat16).to(cuda_device)
    got = run_gemm(hi, X, W_lo=lo).sum(0)
    want = (X.double() @ Wf.double().t()).float()
    bf16_only = X.float() @ hi.float().t()
    err = (got - want).abs().max().item()
    err_bf16 = (bf16_only - want).abs().max().item()
    assert err <= 3e-5 * want.abs().max().item(), (err, err_bf16)
    assert err < err_bf16 / 20  # the residual stream really is used


def test_gemm_rejects_bad_arguments(cuda_device):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    X = torch.zeros(4, 60, dtype=torch.bfloat16, device=cuda_device)
    W = torch.zeros(128, 60, dtype=torch.bfloat16, device=cuda_device)
    out = torch.zeros(1, 4, 128, device=cuda_device)
    rc = lib.prl_gemm_bf16_splitk(W.data_ptr(), None, X.data_ptr(), 4, 128, 60, 1, out.data_ptr(), None)
    assert rc == -1 and b"K" in lib.prl_last_error()


@pytest.mark.parametrize("M,V,K", [(64, 4096 + 77, 512), (5, 1000, 256), (200, 2048, 384)])
def test_fused_head_logprob_capture(cuda_device, M, V, K):
    """Fused head (no logits in HBM) vs materialised fp32 logits: logsumexp, entropy, target logprob, greedy id,
    and sampling identical to the stand-alone sampler (same counter-based RNG)."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(V + M)
    X = torch.randn(M, K, generator=g).to(torch.bfloat16).to(cuda_device)
    W = (torch.randn(V, K, generator=g) * 0.08).to(torch.bfloat16).to(cuda_device)
    targets = torch.randint(0, V, (M,), generator=g).to(cuda_device)
    T = 0.7
    ws = torch.zeros(int(lib.prl_head_workspace_bytes(M, V)), dtype=torch.uint8, device=cuda_device)
    lp_t, ent, lse = (torch.zeros(M, device=cuda_device) for _ in range(3))
    ids = torch.zeros(M, dtype=torch.int32, device=cuda_device)
    lp_s = torch.zeros(M, device=cuda_device)

    def run(greedy, seed, step):
        _lib.check(lib.prl_head_logprob(W.data_ptr(), None, X.data_ptr(), M, V, K, T, targets.data_ptr(), greedy, seed, step,
                                        lp_t.data_ptr(), ent.data_ptr(), lse.data_ptr(), ids.data_ptr(), lp_s.data_ptr(),
                                        ws.data_ptr(), ws.numel(), None))
        torch.cuda.synchronize()
    run(1, 0, 0)
    logits = (X.float() @ W.float().t())
    ref = torch.log_softmax(logits / T, -1)
    assert torch.allclose(lse, torch.logsumexp(logits / T, -1), atol=2e-4, rtol=1e-5)
    assert torch.allclose(lp_t, ref.gather(1, targets[:, None])[:, 0], atol=3e-4, rtol=1e-4)
    assert torch.allclose(ent, -(ref.exp() * ref).sum(-1), atol=3e-4, rtol=1e-4)
    top2 = torch.topk(logits, 2).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-3
    assert (ids.long()[clear] == logits.argmax(-1)[clear]).all()
    assert torch.allclose(lp_s, ref.gather(1, ids.long()[:, None])[:, 0], atol=3e-4, rtol=1e-4)
    # sampling: same ids as the two-phase sampler on materialised logits (identical RNG stream)
    run(0, 99, 7)
    ids2 = torch.zeros(M, dtype=torch.int32, device=cuda_device)
    lp2 = torch.zeros(M, device=cuda_device)
    ws2 = torch.zeros(int(lib.prl_sample_workspace_bytes(M)), dtype=torch.uint8, device=cuda_device)
    lg = logits.contiguous()
    _lib.check(lib.prl_sample_logprob(lg.data_ptr(), M, V, T, 0, 99, 7, ids2.data_ptr(), lp2.data_ptr(), ws2.data_ptr(),
                                      ws2.numel(), None))
    torch.cuda.synchronize()
    same = (ids == ids2)
    assert same.float().mean() > 0.97   # tie-breaks can differ at fp32 noise level between the two logits paths
    assert torch.allclose(lp_s[same], lp2[same], atol=3e-4)


@pytest.mark.parametrize("M,V,K,with_targets", [(129, 640, 256, True), (1000, 4096 + 77, 512, True),
                                                (2048, 152064, 128, True), (300, 1000, 264, False)])
def test_fused_head_many_tokens_statistics_only(cuda_device, M, V, K, with_targets):
    """M > 128 without sampling outputs runs the 128 x 256-tile kernel with the token-per-thread epilogue (gemm_tn.cu)."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(V + M)
    X = torch.randn(M, K, generator=g).to(torch.bfloat16).to(cuda_device)
    W = (torch.randn(V, K, generator=g) * 0.08).to(torch.bfloat16).to(cuda_device)
    targets = torch.randint(0, V, (M,), generator=g).to(cuda_device)
    targets[0], targets[-1] = V - 1, 0
    T = 1.3
    ws = torch.zeros(int(lib.prl_head_workspace_bytes(M, V)), dtype=torch.uint8, device=cuda_device)
    lp_t, ent, lse = (torch.full((M,), float("nan"), device=cuda_device) for _ in range(3))
    _lib.check(lib.prl_head_logprob(W.data_ptr(), None, X.data_ptr(), M, V, K, T,
                                    targets.data_ptr() if with_targets else None, 1, 0, 0,
                                    lp_t.data_ptr() if with_targets else None, ent.data_ptr(), lse.data_ptr(), None, None,
                                    ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    logits = (X.float() @ W.float().t())
    ref = torch.log_softmax(logits / T, -1)
    assert torch.allclose(lse, torch.logsumexp(logits / T, -1), atol=2e-4, rtol=1e-5)
    assert torch.allclose(ent, -(ref.exp() * ref).sum(-1), atol=3e-4, rtol=1e-4)
    if with_targets:
        assert torch.allclose(lp_t, ref.gather(1, targets[:, None])[:, 0], atol=3e-4, rtol=1e-4)


@pytest.mark.parametrize("B,I,K", [(4, 128, 256), (16, 1152, 896), (64, 18944, 3584), (100, 256, 512), (33, 192, 64)])
def test_token_step_swiglu_epilogue_is_bit_identical_to_gemm_plus_silu(cuda_device, B, I, K):
    """prl_gemm_swiglu_decode (the CTA's 128 weight rows = 64 gate rows + the 64 up rows of the same features, both halves
    read back from the shared-memory accumulator tile) == prl_gemm_bf16_splitk(split_k = 1) + prl_silu_mul, bit for bit."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(B * 7 + I + K)
    x = (torch.randn(B, K, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    W = (torch.randn(2 * I, K, generator=g, device=dev) * K ** -0.5).to(torch.bfloat16)
    part = torch.empty(1, B, 2 * I, dtype=torch.float32, device=dev)
    _lib.check(lib.prl_gemm_bf16_splitk(W.data_ptr(), None, x.data_ptr(), B, 2 * I, K, 1, part.data_ptr(), _lib.stream_ptr()))
    want = torch.empty(B, I, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_silu_mul(part.data_ptr(), 1, B, I, want.data_ptr(), None, 0, _lib.stream_ptr()))
    got = torch.full((B, I), float("nan"), dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_gemm_swiglu_decode(W.data_ptr(), x.data_ptr(), B, I, K, got.data_ptr(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    ref = x.float() @ W.float().t()
    fp32 = torch.nn.functional.silu(ref[:, :I]) * ref[:, I:]
    assert (got.float() - fp32).abs().max().item() <= 2 ** -7 * fp32.abs().max().item() + 1e-6

"""wgmma GEMM of the learner body (csrc/gemm_tn.cu) against fp32 torch matmuls of the
same bf16 operands.  Tolerance: fp32 accumulation of bf16 products (1e-4 of the output scale) plus one bf16
rounding (2^-8 relative) where the output is bf16."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def gemm_tn(A, B, out_dtype=torch.bfloat16, bias=None, residual=None, acc_into=None, alpha=1.0):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    M, K = A.shape
    N = B.shape[0]
    if acc_into is not None:
        C = acc_into
    else:
        C = torch.full((M, N), float("nan"), dtype=out_dtype, device=A.device)
    _lib.check(lib.prl_gemm_tn(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), M, N, K, C.data_ptr(), C.stride(0),
                               int(C.dtype == torch.float32), int(acc_into is not None),
                               bias.data_ptr() if bias is not None else None,
                               residual.data_ptr() if residual is not None else None,
                               residual.stride(0) if residual is not None else 0, alpha, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return C


SHAPES = [(1, 8, 8), (256, 256, 64), (129, 130, 72), (300, 777, 200), (1024, 4608, 3584), (2048, 3584, 18944),
          (4608, 3584, 4096), (5000, 1000, 1288), (16, 37888, 512), (777, 24, 136)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_tn_f32_out(cuda_device, M, N, K):
    g = torch.Generator().manual_seed(M * 31 + N * 7 + K)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(cuda_device)
    B = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(cuda_device)
    got = gemm_tn(A, B, out_dtype=torch.float32)
    want = A.float() @ B.float().t()
    assert torch.isfinite(got).all(), "unwritten output"
    assert (got - want).abs().max().item() <= 2e-4 * want.abs().max().item() + 1e-6


@pytest.mark.parametrize("M,N,K", [(300, 776, 200), (1024, 4608, 3584), (513, 100, 64)])
def test_gemm_tn_bf16_bias_residual(cuda_device, M, N, K):
    g = torch.Generator().manual_seed(5)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(cuda_device)
    B = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(cuda_device)
    bias = torch.randn(N, generator=g).to(torch.bfloat16).to(cuda_device)
    res = torch.randn(M, N, generator=g).to(torch.bfloat16).to(cuda_device)
    got = gemm_tn(A, B, bias=bias, residual=res)
    want = A.float() @ B.float().t() + bias.float() + res.float()
    scale = want.abs().max().item()
    assert (got.float() - want).abs().max().item() <= (2e-4 + 2 ** -8) * scale
    plain = gemm_tn(A, B)
    assert torch.equal(plain, (A.float() @ B.float().t()).to(torch.bfloat16)) or \
        (plain.float() - A.float() @ B.float().t()).abs().max().item() <= (2e-4 + 2 ** -8) * scale


def test_gemm_tn_accumulates_and_strided_operands(cuda_device):
    """wgrad form: fp32 C += A * B^T with operands that are column slices of wider buffers."""
    g = torch.Generator().manual_seed(9)
    big_a = torch.randn(640, 1024, generator=g).to(torch.bfloat16).to(cuda_device)
    big_b = torch.randn(384, 1024, generator=g).to(torch.bfloat16).to(cuda_device)
    A, B = big_a[:, 128:128 + 520], big_b[:, 256:256 + 520]
    C = torch.randn(640, 384, generator=g).to(cuda_device)
    want = C + 0.5 * (A.float() @ B.float().t())
    got = gemm_tn(A, B, acc_into=C, alpha=0.5)
    assert (got - want).abs().max().item() <= 2e-4 * want.abs().max().item()


def test_gemm_tn_is_deterministic(cuda_device):
    g = torch.Generator().manual_seed(1)
    A = torch.randn(3000, 2048, generator=g).to(torch.bfloat16).to(cuda_device)
    B = torch.randn(1500, 2048, generator=g).to(torch.bfloat16).to(cuda_device)
    assert torch.equal(gemm_tn(A, B), gemm_tn(A, B))


@pytest.mark.parametrize("R,C", [(1, 1), (64, 64), (100, 37), (4096, 3584), (777, 1288)])
def test_transpose_bf16(cuda_device, R, C):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    x = torch.randn(R, C, device=cuda_device).to(torch.bfloat16)
    out = torch.empty(C, R, dtype=torch.bfloat16, device=cuda_device)
    _lib.check(lib.prl_transpose_bf16(x.data_ptr(), R, C, x.stride(0), out.data_ptr(), out.stride(0), _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(out, x.t().contiguous())


def test_gemm_tn_rejects_bad_arguments(cuda_device):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    A = torch.zeros(16, 20, dtype=torch.bfloat16, device=cuda_device)
    C = torch.zeros(16, 16, dtype=torch.bfloat16, device=cuda_device)
    rc = lib.prl_gemm_tn(A.data_ptr(), 20, A.data_ptr(), 20, 16, 16, 20, C.data_ptr(), 16, 0, 0, None, None, 0, 1.0,
                         _lib.stream_ptr())
    assert rc != 0 and b"multiples of 8" in lib.prl_last_error()
    rc = lib.prl_gemm_tn(A.data_ptr(), 24, A.data_ptr(), 24, 16, 16, 16, C.data_ptr(), 16, 0, 1, None, None, 0, 1.0,
                         _lib.stream_ptr())
    assert rc != 0 and b"accumulate" in lib.prl_last_error()


def gemm_ex(A, a_mn, B, b_mn, M, N, K, out_dtype=torch.float32, acc_into=None):
    """A given as [K, M] when a_mn else [M, K]; B as [K, N] when b_mn else [N, K]."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    C = acc_into if acc_into is not None else torch.full((M, N), float("nan"), dtype=out_dtype, device=A.device)
    _lib.check(lib.prl_gemm_ex(A.data_ptr(), A.stride(0), int(a_mn), B.data_ptr(), B.stride(0), int(b_mn), M, N, K,
                               C.data_ptr(), C.stride(0), int(C.dtype == torch.float32), int(acc_into is not None), None,
                               None, 0, 1.0, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return C


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (304, 776, 200), (1000, 520, 1288), (4608, 3584, 2048), (24, 72, 136)])
def test_gemm_mn_major_operands(cuda_device, M, N, K, a_mn, b_mn):
    """dgrad reads W as stored (B MN-major), wgrad reads dY and X as stored (both MN-major): no transposed copies."""
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(cuda_device)
    B = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(cuda_device)
    want = A.float() @ B.float().t()
    got = gemm_ex(A.t().contiguous() if a_mn else A, a_mn, B.t().contiguous() if b_mn else B, b_mn, M, N, K)
    assert torch.isfinite(got).all()
    assert (got - want).abs().max().item() <= 2e-4 * want.abs().max().item() + 1e-6
    ref = gemm_ex(A, False, B, False, M, N, K)
    assert torch.equal(got, ref)    # same products, same k order: bitwise equal to the K-major path


@pytest.mark.parametrize("T,K,I", [(300, 512, 1024), (257, 896, 1152), (1024, 3584, 18944), (5, 256, 128)])
def test_gemm_swiglu_epilogue_is_bit_identical_to_gemm_plus_silu(cuda_device, T, K, I):
    """gate_up GEMM with SiLU(gate) * up in its epilogue (prl_gemm_swiglu: the pair's two CTAs stage the gate rows and the up
    rows of the same 128 features) == prl_gemm_ex followed by prl_silu_mul_fwd, bit for bit, for both outputs."""
    from pipelinerl_b200.learner_body import Ops
    o = Ops()
    g = torch.Generator(device=cuda_device).manual_seed(T + K + I)
    x = (torch.randn(T, K, generator=g, device=cuda_device) * 0.5).to(torch.bfloat16)
    W = (torch.randn(2 * I, K, generator=g, device=cuda_device) * K ** -0.5).to(torch.bfloat16)
    gu_ref = o.gemm(x, W)
    act_ref = o.silu_mul(gu_ref)
    gu, act = o.gemm_swiglu(x, W, need_gate_up=True)
    torch.cuda.synchronize()
    assert torch.equal(gu, gu_ref) and torch.equal(act, act_ref)
    none, act2 = o.gemm_swiglu(x, W, need_gate_up=False)
    assert none is None and torch.equal(act2, act_ref)
    # and against fp32 math
    ref = x.float() @ W.float().t()
    want = torch.nn.functional.silu(ref[:, :I]) * ref[:, I:]
    assert (act.float() - want).abs().max().item() <= 2 ** -6 * want.abs().max().item()


@pytest.mark.parametrize("T,K,I", [(1024, 512, 256), (1000, 896, 1152), (130, 256, 128)])
def test_gemm_swiglu_f32_is_bit_identical_to_fp32_gemm_plus_sampler_silu(cuda_device, T, K, I):
    """The sampler's chunked prefill (engine.py): prl_gemm_swiglu_f32 == prl_gemm_tn with an fp32 output followed by
    prl_silu_mul (the token step's own SiLU(gate) * up of fp32 values), bit for bit -- the fusion removes the [T, 2I] fp32
    round trip, not a rounding point."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(T + K + I)
    x = (torch.randn(T, K, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    W = (torch.randn(2 * I, K, generator=g, device=dev) * K ** -0.5).to(torch.bfloat16)
    part = torch.empty(T, 2 * I, dtype=torch.float32, device=dev)
    _lib.check(lib.prl_gemm_tn(x.data_ptr(), K, W.data_ptr(), K, T, 2 * I, K, part.data_ptr(), 2 * I, 1, 0, None, None, 0, 1.0,
                               _lib.stream_ptr()))
    act_ref = torch.empty(T, I, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_silu_mul(part.data_ptr(), 1, T, I, act_ref.data_ptr(), None, 0, _lib.stream_ptr()))
    act = torch.empty(T, I, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_gemm_swiglu_f32(x.data_ptr(), K, W.data_ptr(), K, T, I, K, act.data_ptr(), I, _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(act, act_ref)
    ref = x.float() @ W.float().t()
    want = torch.nn.functional.silu(ref[:, :I]) * ref[:, I:]
    assert (act.float() - want).abs().max().item() <= 2 ** -7 * want.abs().max().item()


@pytest.mark.parametrize("M,V,K,with_lo,with_ent", [(300, 1031, 256, True, True), (2048, 4096, 512, True, False),
                                                     (130, 777, 128, False, True), (1, 520, 64, True, True)])
def test_head_dlogits_without_materialised_logits(cuda_device, M, V, K, with_lo, with_ent):
    """prl_head_dlogits: the head GEMM (hi + lo weight streams in one accumulation) with the backward of
    log-softmax / entropy in its epilogue, bf16 d logits out.  Against fp32 torch autograd through logits / T ->
    log_softmax -> (target logprob, entropy) on the same bf16 inputs, and the statistics of prl_head_logprob as inputs."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(M + V + K)
    T = 0.7
    x = (torch.randn(M, K, generator=g, device=dev) * 0.7).to(torch.bfloat16)
    Wf = torch.randn(V, K, generator=g, device=dev) * K ** -0.5
    W = Wf.to(torch.bfloat16)
    W_lo = (Wf - W.float()).to(torch.bfloat16) if with_lo else None
    tg = torch.randint(0, V, (M,), generator=g, device=dev)
    g_lp = torch.randn(M, generator=g, device=dev)
    g_ent = torch.randn(M, generator=g, device=dev) * 0.3 if with_ent else None
    lp = torch.empty(M, device=dev)
    ent, lse = torch.empty_like(lp), torch.empty_like(lp)
    ws = torch.empty(int(lib.prl_head_workspace_bytes(M, V)), dtype=torch.uint8, device=dev)
    _lib.check(lib.prl_head_logprob(W.data_ptr(), W_lo.data_ptr() if with_lo else None, x.data_ptr(), M, V, K, T, tg.data_ptr(),
                                    1, 0, 0, lp.data_ptr(), ent.data_ptr(), lse.data_ptr(), None, None, ws.data_ptr(), ws.numel(),
                                    _lib.stream_ptr()))
    ld = (V + 7) // 8 * 8
    dz = torch.zeros(M, ld, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_head_dlogits(W.data_ptr(), W_lo.data_ptr() if with_lo else None, x.data_ptr(), M, V, K, T, tg.data_ptr(),
                                    lse.data_ptr(), ent.data_ptr(), g_lp.data_ptr(), g_ent.data_ptr() if with_ent else None,
                                    dz.data_ptr(), ld, _lib.stream_ptr()))
    torch.cuda.synchronize()
    Wsum = W.float() + (W_lo.float() if with_lo else 0.0)
    z = (x.float() @ Wsum.t()).requires_grad_(True)
    ls = torch.log_softmax(z / T, -1)
    obj = (ls.gather(1, tg[:, None])[:, 0] * g_lp).sum()
    if with_ent:
        obj = obj + ((-(ls.exp() * ls).sum(-1)) * g_ent).sum()
    obj.backward()
    want = z.grad
    err = (dz[:, :V].float() - want).abs().max().item() / want.abs().max().item()
    print(f"[head dlogits M={M} V={V} K={K} lo={with_lo} ent={with_ent}] rel max err {err:.2e}")
    assert err <= 2 ** -7
    if ld > V:
        assert torch.count_nonzero(dz[:, V:]) == 0      # padding columns are not touched


@pytest.mark.parametrize("T,H,I", [(300, 512, 1024), (257, 896, 1152), (1024, 3584, 18944), (5, 256, 160)])
def test_dgrad_with_silu_backward_epilogue_is_bit_identical(cuda_device, T, H, I):
    """prl_gemm_dgrad_swiglu (down_proj dgrad whose epilogue applies the backward of SiLU(gate) * up) == prl_gemm_ex with the
    weight read as stored followed by prl_silu_mul_bwd, bit for bit."""
    from pipelinerl_b200.learner_body import Ops
    o = Ops()
    g = torch.Generator(device=cuda_device).manual_seed(T + H + I)
    dY = (torch.randn(T, H, generator=g, device=cuda_device) * 0.5).to(torch.bfloat16)
    W = (torch.randn(H, I, generator=g, device=cuda_device) * H ** -0.5).to(torch.bfloat16)
    gu = torch.randn(T, 2 * I, generator=g, device=cuda_device).to(torch.bfloat16)
    want = o.silu_mul_bwd(gu, o.dgrad(dY, W))
    got = o.dgrad_swiglu(dY, W, gu)
    torch.cuda.synchronize()
    assert torch.equal(got, want)

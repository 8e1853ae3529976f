"""Qwen3 on the GPU: the q/k-norm epilogue of the token step, the learner's q/k-norm kernels, the weight push, and the
decode engine and native learner against HF Qwen3 fixtures (the checks of tests/conformance.py on the Qwen3 cases).

Bars: kernels against fp64 within one bf16 rounding of the output; the engine and the learner at the bounds of their
case in tests/model_cases.py."""
import pytest
import torch

from tests import conformance
from tests.model_cases import qwen3_tiny_cfg, qwen3_tiny_weights

pytestmark = pytest.mark.gpu

D = 128


def _inv_freq(dev, theta=1e6):
    return (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).to(dev)


# ---- token-step epilogue -------------------------------------------------------------------------------------------
def _epilogue_case(dev, B, n_q, n_kv, n_split, seed, bias=True, rope="hf"):
    """rope "hf": Qwen's unscaled table, positions below 2 pages, token row b in block-table row b.  rope "llama3":
    Llama-3.1-8B's scaled table, positions up to 131071, each row in a block-table row of its own (a permutation of more
    rows than there are tokens) with one page at the block its position falls in."""
    g = torch.Generator().manual_seed(seed)
    nh = n_q + 2 * n_kv
    P = 64
    part = (torch.randn(n_split, B, nh * D, generator=g) * 0.7).to(dev)
    b = (0.3 * torch.randn(nh * D, generator=g)).to(torch.bfloat16).to(dev) if bias else None
    qg = (1 + 0.4 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    kg = (1 + 0.4 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    if rope == "hf":
        max_blocks, n_pages = 8, 1 + B * 2
        pos = torch.randint(0, 2 * P, (B,), generator=g, dtype=torch.int32)
        slot = torch.arange(B, dtype=torch.int32)
        bt = torch.zeros(B, max_blocks, dtype=torch.int32)
        bt[:, :2] = (1 + torch.randperm(2 * B, generator=g)).view(B, 2).int()
        inv = _inv_freq(dev)
    else:
        from pipelinerl_b200.model import ModelConfig, rope_inv_freq
        max_blocks, n_pages = 131072 // P, 1 + B + 2                  # two pages no token addresses
        pos = torch.randint(0, 131072, (B,), generator=g, dtype=torch.int32)
        pos[:4] = torch.tensor([131071, 0, 63, 64], dtype=torch.int32)[:B]
        slot = torch.randperm(B + 5, generator=g)[:B].int()
        bt = torch.zeros(B + 5, max_blocks, dtype=torch.int32)
        bt[slot.long(), (pos // P).long()] = (1 + torch.randperm(B, generator=g)).int()
        inv = rope_inv_freq(ModelConfig.llama3_1_8b()).to(dev)
    return dict(part=part, bias=b, qg=qg, kg=kg, pos=pos.to(dev), bt=bt.to(dev), slot=slot.to(dev), inv=inv,
                n_pages=n_pages, P=P, max_blocks=max_blocks, B=B, n_q=n_q, n_kv=n_kv, n_split=n_split)


def _run_epilogue(lib, c, dev, norm=True, rows=None, legacy=False, eps=1e-6, layer=1, kv0=None):
    """-> (q_out [B, n_q, D], kv cache [2 layers, 2, n_pages, n_kv, P, D]); rows = (r0, n): only those token rows; kv0: the
    cache's contents before the step (zeros by default)"""
    from pipelinerl_b200 import _lib
    B, n_q, n_kv = c["B"], c["n_q"], c["n_kv"]
    q = torch.zeros(B, n_q, D, dtype=torch.bfloat16, device=dev)
    kv = (kv0.clone() if kv0 is not None else
          torch.zeros(2 * 2 * c["n_pages"] * n_kv * c["P"] * D, dtype=torch.bfloat16, device=dev))
    r0, n = rows if rows is not None else (0, B)
    assert c["n_split"] == 1 or rows is None
    part = c["part"][:, r0:r0 + n].contiguous()
    bias = c["bias"].data_ptr() if c["bias"] is not None else None
    common = (c["pos"][r0:].data_ptr(), c["bt"].data_ptr(), c["max_blocks"], c["slot"][r0:].data_ptr(), c["inv"].data_ptr(),
              q[r0:].data_ptr(), kv.data_ptr(), c["n_pages"], layer, c["P"], None, 0, None)
    if legacy:
        _lib.check(lib.prl_qkv_rope_cache(part.data_ptr(), c["n_split"], n, bias, n_q, n_kv, D, *common))
    else:
        _lib.check(lib.prl_qkv_norm_rope_cache(part.data_ptr(), c["n_split"], n, bias,
                                               c["qg"].data_ptr() if norm else None, c["kg"].data_ptr() if norm else None,
                                               eps, n_q, n_kv, D, *common))
    torch.cuda.synchronize()
    return q, kv.view(2, 2, c["n_pages"], n_kv, c["P"], D)


def _epilogue_fp64(c, eps=1e-6, norm=True):
    x = c["part"].double().sum(0)
    if c["bias"] is not None:
        x = x + c["bias"].double()
    B, n_q, n_kv = c["B"], c["n_q"], c["n_kv"]
    x = x.view(B, n_q + 2 * n_kv, D)
    y = x[:, :n_q + n_kv]
    if norm:
        gam = torch.cat([c["qg"].double()[None].expand(n_q, D), c["kg"].double()[None].expand(n_kv, D)])
        y = y * torch.rsqrt((y * y).mean(-1, keepdim=True) + eps) * gam
    ang = (c["pos"].float()[:, None] * c["inv"][None]).double()       # the kernel's fp32 angle
    cs, sn = torch.cos(ang)[:, None], torch.sin(ang)[:, None]
    y1, y2 = y[..., :64], y[..., 64:]
    return torch.cat([y1 * cs - y2 * sn, y2 * cs + y1 * sn], -1), x[:, n_q + n_kv:]


def _kv_page_slot(c):
    """page and in-page slot of every token row's KV"""
    pos = c["pos"].long()
    return c["bt"].long()[c["slot"].long(), pos // c["P"]], pos % c["P"]


def _kv_rows(c, kv, layer=1):
    """k [B, n_kv, D], v [B, n_kv, D] of every token row, read back from the pages"""
    page, slot = _kv_page_slot(c)
    return kv[layer, 0, page, :, slot], kv[layer, 1, page, :, slot]


def _case(B, n_q, n_kv, n_split, norm=True, bias=True, rope="hf"):
    tag = "-".join(map(str, (B, n_q, n_kv, n_split))) + ("" if norm else "-nonorm") + ("" if bias else "-nobias")
    return pytest.param(B, n_q, n_kv, n_split, norm, bias, rope, id=tag + ("" if rope == "hf" else "-" + rope))


@pytest.mark.parametrize("B,n_q,n_kv,n_split,norm,bias,rope", [
    _case(5, 8, 2, 3), _case(64, 32, 8, 2), _case(300, 8, 2, 1), _case(200, 5, 1, 1),
    # the Qwen2 step (bias, no q/k norm) on both kernels; Qwen3 (norm, no bias) at Qwen3-8B's and Qwen3-14B's groupings
    _case(5, 28, 4, 3, norm=False), _case(300, 28, 4, 1, norm=False),
    _case(64, 32, 8, 2, bias=False), _case(129, 40, 8, 1, bias=False),
    # the Llama 3 step (neither) with the scaled table, positions up to 131071 and scattered block-table rows
    _case(7, 32, 8, 2, norm=False, bias=False, rope="llama3"), _case(200, 24, 8, 2, norm=False, bias=False, rope="llama3"),
    _case(150, 8, 2, 1, bias=False, rope="llama3"),
])
def test_qkv_norm_rope_epilogue_vs_fp64(cuda_device, B, n_q, n_kv, n_split, norm, bias, rope):
    """per-head kernel (B <= 128) and row-walking kernel (B > 128) against an fp64 restatement: one bf16 rounding.  The
    cache starts out holding a pattern, and every row the step does not address must still hold it afterwards."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    c = _epilogue_case(cuda_device, B, n_q, n_kv, n_split, seed=B + n_q, bias=bias, rope=rope)
    kv0 = torch.randn(2 * 2 * c["n_pages"] * n_kv * c["P"] * D, generator=torch.Generator().manual_seed(1))
    kv0 = kv0.to(torch.bfloat16).to(cuda_device)
    q, kv = _run_epilogue(lib, c, cuda_device, norm=norm, kv0=kv0)
    qk_ref, v_ref = _epilogue_fp64(c, norm=norm)
    k, v = _kv_rows(c, kv)
    got = torch.cat([q, k], 1)
    tol = 2 ** -7 * qk_ref.abs() + 1e-5            # one bf16 rounding (a boundary case may round the other way)
    err = (got.double() - qk_ref).abs()
    exact = (got == qk_ref.to(torch.bfloat16)).double().mean().item()
    print(f"[qkv epilogue {B}x{n_q}/{n_kv} split {n_split} norm {norm} bias {bias} rope {rope}] max |err| "
          f"{err.max().item():.3e}, exact {exact:.5f}")
    assert (err <= tol).all(), err.max().item()
    assert exact >= 0.999, exact
    assert ((v.double() - v_ref).abs() <= 2 ** -7 * v_ref.abs() + 1e-5).all()   # v heads: sum + bias only, no norm
    page, slot = _kv_page_slot(c)
    written = torch.zeros(2, 2, c["n_pages"], n_kv, c["P"], dtype=torch.bool, device=cuda_device)
    written[1, :, page, :, slot] = True
    assert torch.equal(kv[~written], kv0.view_as(kv)[~written])


def test_qkv_norm_rope_rows_kernel_bit_identical_to_per_head_kernel(cuda_device):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    c = _epilogue_case(cuda_device, 384, 8, 2, 1, seed=5)
    q_rows, kv_rows = _run_epilogue(lib, c, cuda_device)                         # B = 384 > 128: row-walking kernel
    q_head = torch.zeros_like(q_rows)
    kv_head = torch.zeros_like(kv_rows)
    for r0 in range(0, 384, 128):                                                # 3 launches of 128: per-head kernel
        q, kv = _run_epilogue(lib, c, cuda_device, rows=(r0, 128))
        q_head[r0:r0 + 128] = q[r0:r0 + 128]
        kv_head += kv                                                            # disjoint pages
    assert torch.equal(q_rows, q_head) and torch.equal(kv_rows, kv_head)


@pytest.mark.parametrize("B", [7, 200])
def test_qkv_norm_rope_entry_without_gains_equals_qkv_rope_cache(cuda_device, B):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    c = _epilogue_case(cuda_device, B, 7, 1, 2 if B <= 128 else 1, seed=B)
    q_a, kv_a = _run_epilogue(lib, c, cuda_device, norm=False)
    q_b, kv_b = _run_epilogue(lib, c, cuda_device, legacy=True)
    assert torch.equal(q_a, q_b) and torch.equal(kv_a, kv_b)
    with pytest.raises(_lib.PrlError):       # one gain without the other
        _lib.check(lib.prl_qkv_norm_rope_cache(c["part"].data_ptr(), 1, 1, None, c["qg"].data_ptr(), None, 1e-6, 7, 1, D,
                                               c["pos"].data_ptr(), c["bt"].data_ptr(), 8, None, _inv_freq(cuda_device).data_ptr(),
                                               q_a.data_ptr(), kv_a.data_ptr(), c["n_pages"], 0, 64, None, 0, None))


# ---- learner kernels -----------------------------------------------------------------------------------------------
def _learner_case(dev, T, n_q, n_kv, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    W = (n_q + 2 * n_kv) * D
    qkv = (torch.randn(T, W, generator=g, device=dev) * 1.5).to(torch.bfloat16)
    qg = (1 + 0.4 * torch.randn(D, generator=g, device=dev)).to(torch.bfloat16)
    kg = (1 + 0.4 * torch.randn(D, generator=g, device=dev)).to(torch.bfloat16)
    kg[:3] = 0            # near-zero gains must not hurt the backward (x-hat is never recovered by dividing by them)
    pos = torch.randint(0, 16384, (T,), device=dev, dtype=torch.int32)
    dy = torch.randn(T, W, generator=g, device=dev).to(torch.bfloat16)
    return qkv, qg, kg, pos, dy


def _torch_qk_norm_rope(qkv, qg, kg, pos, n_q, n_kv, eps):
    T = qkv.shape[0]
    x = qkv.view(T, n_q + 2 * n_kv, D)
    qk = x[:, :n_q + n_kv]
    gam = torch.cat([qg[None].expand(n_q, D), kg[None].expand(n_kv, D)])
    y = qk * torch.rsqrt((qk * qk).mean(-1, keepdim=True) + eps) * gam
    ang = (pos.float()[:, None] * _inv_freq(qkv.device)[None]).double()        # the kernel's fp32 angle
    cs, sn = torch.cos(ang)[:, None].to(qkv.dtype), torch.sin(ang)[:, None].to(qkv.dtype)
    y1, y2 = y[..., :64], y[..., 64:]
    return torch.cat([torch.cat([y1 * cs - y2 * sn, y2 * cs + y1 * sn], -1), x[:, n_q + n_kv:]], 1).reshape(T, -1)


@pytest.mark.parametrize("T,n_q,n_kv", [(1, 4, 2), (333, 8, 2), (1500, 32, 8), (64, 5, 1)])
def test_learner_qk_norm_rope_fwd_bwd_vs_autograd(cuda_device, T, n_q, n_kv):
    from pipelinerl_b200.learner_body import Ops
    o, dev, eps = Ops(), cuda_device, 1e-6
    qkv, qg, kg, pos, dy = _learner_case(dev, T, n_q, n_kv, seed=T + n_q)
    inv = _inv_freq(dev)
    y = qkv.clone()
    saved = o.qk_norm_rope_(y, pos, inv, qg, kg, n_q, n_kv, D, eps, keep=True)
    x64 = qkv.double().requires_grad_(True)
    g64 = [qg.double().requires_grad_(True), kg.double().requires_grad_(True)]
    want = _torch_qk_norm_rope(x64, g64[0], g64[1], pos, n_q, n_kv, eps)
    qkw = (n_q + n_kv) * D
    tol = 2 ** -7 * want.detach().abs() + 1e-5
    assert ((y.double() - want.detach()).abs() <= tol).all(), (y.double() - want).abs().max().item()
    assert torch.equal(y[:, qkw:], qkv[:, qkw:])                                    # v untouched
    assert torch.equal(saved[0], qkv[:, :qkw])                                      # the pre-norm q | k columns
    ms = qkv[:, :qkw].double().view(T, -1, D).pow(2).mean(-1)
    assert torch.allclose(saved[1].double(), torch.rsqrt(ms + eps), rtol=1e-5)
    want.backward(dy.double())
    dq_g = torch.full((D,), 0.25, device=dev)
    dk_g = torch.full((D,), -0.5, device=dev)
    dx = dy.clone()
    o.qk_norm_rope_bwd_(dx, pos, inv, qg, kg, saved, n_q, n_kv, D, dq_g, dk_g)
    ref = x64.grad
    err = (dx.double() - ref).abs()
    assert (err[:, :qkw] <= 2 ** -7 * ref[:, :qkw].abs() + 2e-3 * ref[:, :qkw].abs().max()).all(), err.max().item()
    assert torch.equal(dx[:, qkw:], dy[:, qkw:])
    for got, g, base in ((dq_g, g64[0].grad, 0.25), (dk_g, g64[1].grad, -0.5)):
        assert torch.allclose((got.double() - base), g, rtol=1e-3, atol=1e-3 * g.abs().max().item())
    # bitwise reproducible across runs
    y2 = qkv.clone()
    saved2 = o.qk_norm_rope_(y2, pos, inv, qg, kg, n_q, n_kv, D, eps, keep=True)
    dx2, dq2, dk2 = dy.clone(), torch.full((D,), 0.25, device=dev), torch.full((D,), -0.5, device=dev)
    o.qk_norm_rope_bwd_(dx2, pos, inv, qg, kg, saved2, n_q, n_kv, D, dq2, dk2)
    assert torch.equal(y, y2) and torch.equal(saved[1], saved2[1])
    assert torch.equal(dx, dx2) and torch.equal(dq_g, dq2) and torch.equal(dk_g, dk2)
    # without keep: the same forward bits, nothing saved
    y3 = qkv.clone()
    assert o.qk_norm_rope_(y3, pos, inv, qg, kg, n_q, n_kv, D, eps, keep=False) is None
    assert torch.equal(y, y3)


# ---- weight push ---------------------------------------------------------------------------------------------------
def test_pushed_qwen3_arena_samples_the_same_ids(cuda_device):
    """a Qwen3 arena pushed as raw bytes into a receiver's buffer: the receiving engine samples (T = 1) the same ids
    and logprobs as an engine on the learner's arena"""
    from pipelinerl_b200.engine import DecodeEngine, SamplingParams
    from pipelinerl_b200.model import ParamArena
    from pipelinerl_b200.weights import WeightReceiver, WeightUpdateManager
    cfg = qwen3_tiny_cfg("gqa4")
    w = qwen3_tiny_weights(cfg)
    learner = ParamArena(cfg, cuda_device)
    for name in learner.names():
        learner.view(name).copy_(w[name].to(torch.bfloat16))
    recv = WeightReceiver(cfg, cuda_device, n_pushers=1)
    mgr = WeightUpdateManager([recv], learner.data)
    mgr.send_weight_update(version=1)
    for _ in range(1000):
        if recv.maybe_flip(None):
            break
        torch.cuda.synchronize()
    else:
        raise AssertionError("the pushed update never became flippable")
    assert torch.equal(recv.arena.data, learner.data)
    prompts = [[3, 1, 4, 1, 5, 9, 2, 6], list(range(40, 110))]
    res = []
    for arena in (learner, recv.arena):
        eng = DecodeEngine(cfg, arena, max_batch=4, max_seq_len=128, max_new_tokens=32, device=cuda_device, seed=5)
        out = eng.generate(prompts, SamplingParams(max_tokens=20, temperature=1.0))
        res.append([(r.output_ids, r.output_logprobs) for r in out])
    assert res[0] == res[1]
    recv.close()


# ---- decode engine and native learner vs HF Qwen3 (tests/conformance.py) ---------------------------------------------
KINDS = ["wide", "gqa4"]


@pytest.mark.parametrize("kind", KINDS)
def test_engine_teacher_forced_decode_path_vs_hf(cuda_device, kind):
    conformance.engine_teacher_forced(cuda_device, f"qwen3_{kind}")


@pytest.mark.parametrize("kind,use_graph,prefill_chunk", [("wide", True, 1024), ("wide", False, 0), ("gqa4", False, 1024),
                                                          ("gqa4", True, 0), ("gqa4", True, 48)])
def test_engine_greedy_vs_hf(cuda_device, kind, use_graph, prefill_chunk):
    conformance.engine_greedy_vs_hf(cuda_device, f"qwen3_{kind}", use_graph, prefill_chunk)


def test_engine_prefix_sharing_matches_unshared(cuda_device):
    conformance.engine_prefix_sharing(cuda_device, "qwen3_wide", max_seq_len=256)


@pytest.mark.parametrize("kind", KINDS)
def test_engine_score_vs_hf(cuda_device, kind):
    conformance.engine_score(cuda_device, f"qwen3_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_native_learner_vs_reference_rl_step_on_hf_qwen3(cuda_device, kind):
    conformance.native_learner_vs_reference(cuda_device, f"qwen3_{kind}")

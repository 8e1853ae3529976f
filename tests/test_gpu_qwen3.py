"""Qwen3 on the GPU: the q/k-norm epilogue of the token step, the learner's q/k-norm kernels, the decode engine and the
native learner against HF Qwen3 fixtures, and the weight push.

Bars: kernels against fp64 within one bf16 rounding of the output; the engine at the end-to-end bar of the Qwen2
token-step tests (max |d logprob| <= 3e-2, mean <= 6e-3, greedy ids equal wherever the top-2 margin exceeds 5e-2); the
learner at the bar of the Qwen2 learner-vs-reference test (loss 2e-2 relative, every gradient 3e-2)."""
import json

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN
from tests.qwen3_oracle import QWEN3_KINDS, OracleQwen3, qwen3_tiny_cfg, qwen3_tiny_weights

pytestmark = pytest.mark.gpu

E2E_MAX, E2E_MEAN, MARGIN = 3e-2, 6e-3, 5e-2
D = 128


def _inv_freq(dev, theta=1e6):
    return (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).to(dev)


# ---- token-step epilogue -------------------------------------------------------------------------------------------
def _epilogue_case(dev, B, n_q, n_kv, n_split, seed, bias=True):
    g = torch.Generator().manual_seed(seed)
    nh = n_q + 2 * n_kv
    P, max_blocks = 64, 8
    n_pages = 1 + B * 2
    part = (torch.randn(n_split, B, nh * D, generator=g) * 0.7).to(dev)
    b = (0.3 * torch.randn(nh * D, generator=g)).to(torch.bfloat16).to(dev) if bias else None
    qg = (1 + 0.4 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    kg = (1 + 0.4 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    pos = torch.randint(0, 2 * P, (B,), generator=g, dtype=torch.int32)
    bt = torch.zeros(B, max_blocks, dtype=torch.int32)
    bt[:, :2] = (1 + torch.randperm(2 * B, generator=g)).view(B, 2).int()
    return dict(part=part, bias=b, qg=qg, kg=kg, pos=pos.to(dev), bt=bt.to(dev), n_pages=n_pages, P=P,
                max_blocks=max_blocks, B=B, n_q=n_q, n_kv=n_kv, n_split=n_split)


def _run_epilogue(lib, c, dev, norm=True, rows=None, legacy=False, eps=1e-6, layer=1):
    """-> (q_out [B, n_q, D], kv cache [2 layers, 2, n_pages, n_kv, P, D]); rows = (r0, n): only those token rows"""
    from pipelinerl_b200 import _lib
    B, n_q, n_kv = c["B"], c["n_q"], c["n_kv"]
    q = torch.zeros(B, n_q, D, dtype=torch.bfloat16, device=dev)
    kv = torch.zeros(2 * 2 * c["n_pages"] * n_kv * c["P"] * D, dtype=torch.bfloat16, device=dev)
    inv = _inv_freq(dev)
    r0, n = rows if rows is not None else (0, B)
    assert c["n_split"] == 1 or rows is None
    part = c["part"][:, r0:r0 + n].contiguous()
    bias = c["bias"].data_ptr() if c["bias"] is not None else None
    slot = torch.arange(r0, r0 + n, dtype=torch.int32, device=dev)
    common = (c["pos"][r0:].data_ptr(), c["bt"].data_ptr(), c["max_blocks"], slot.data_ptr(), inv.data_ptr(),
              q[r0:].data_ptr(), kv.data_ptr(), c["n_pages"], layer, c["P"], None, 0, None)
    if legacy:
        _lib.check(lib.prl_qkv_rope_cache(part.data_ptr(), c["n_split"], n, bias, n_q, n_kv, D, *common))
    else:
        _lib.check(lib.prl_qkv_norm_rope_cache(part.data_ptr(), c["n_split"], n, bias,
                                               c["qg"].data_ptr() if norm else None, c["kg"].data_ptr() if norm else None,
                                               eps, n_q, n_kv, D, *common))
    torch.cuda.synchronize()
    return q, kv.view(2, 2, c["n_pages"], n_kv, c["P"], D)


def _epilogue_fp64(c, eps=1e-6):
    x = c["part"].double().sum(0)
    if c["bias"] is not None:
        x = x + c["bias"].double()
    B, n_q, n_kv = c["B"], c["n_q"], c["n_kv"]
    x = x.view(B, n_q + 2 * n_kv, D)
    qk = x[:, :n_q + n_kv]
    gam = torch.cat([c["qg"].double()[None].expand(n_q, D), c["kg"].double()[None].expand(n_kv, D)])
    y = qk * torch.rsqrt((qk * qk).mean(-1, keepdim=True) + eps) * gam
    ang = (c["pos"].float()[:, None] * _inv_freq(c["pos"].device)[None]).double()   # the kernel's fp32 angle
    cs, sn = torch.cos(ang)[:, None], torch.sin(ang)[:, None]
    y1, y2 = y[..., :64], y[..., 64:]
    return torch.cat([y1 * cs - y2 * sn, y2 * cs + y1 * sn], -1), x[:, n_q + n_kv:]


def _kv_rows(c, kv, layer=1):
    """k [B, n_kv, D], v [B, n_kv, D] of every token row, read back from the pages"""
    P = c["P"]
    pos = c["pos"].long()
    page = c["bt"].long().gather(1, (pos // P)[:, None])[:, 0]
    slot = pos % P
    return kv[layer, 0, page, :, slot], kv[layer, 1, page, :, slot]


@pytest.mark.parametrize("B,n_q,n_kv,n_split", [(5, 8, 2, 3), (64, 32, 8, 2), (300, 8, 2, 1), (200, 5, 1, 1)])
def test_qkv_norm_rope_epilogue_vs_fp64(cuda_device, B, n_q, n_kv, n_split):
    """per-head kernel (B <= 128) and row-walking kernel (B > 128) against an fp64 restatement: one bf16 rounding"""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    c = _epilogue_case(cuda_device, B, n_q, n_kv, n_split, seed=B + n_q)
    q, kv = _run_epilogue(lib, c, cuda_device)
    qk_ref, v_ref = _epilogue_fp64(c)
    k, v = _kv_rows(c, kv)
    got = torch.cat([q, k], 1).double()
    tol = 2 ** -7 * qk_ref.abs() + 1e-5            # one bf16 rounding (a boundary case may round the other way)
    assert ((got - qk_ref).abs() <= tol).all(), (got - qk_ref).abs().max().item()
    assert ((v.double() - v_ref).abs() <= 2 ** -7 * v_ref.abs() + 1e-5).all()   # v heads: sum + bias only, no norm


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


# ---- decode engine -------------------------------------------------------------------------------------------------
def _engine(cfg, w, dev, **kw):
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ParamArena
    arena = ParamArena(cfg, dev)
    for name in arena.names():
        arena.view(name).copy_(w[name].to(torch.bfloat16))
    return DecodeEngine(cfg, arena, device=dev, **kw)


def _check_greedy(gold, outs, idx):
    errs = []
    for i, r in zip(idx, outs):
        n = len(r.output_ids)
        ids, lps, mg = gold["greedy_ids"][i][:n], gold["greedy_logprobs"][i][:n], gold["greedy_margin"][i][:n]
        for t in range(n):
            if mg[t] > MARGIN:
                assert r.output_ids[t] == int(ids[t]), (i, t)
            if r.output_ids[:t + 1] != ids[:t + 1].tolist():
                break                      # a near-tie went the other way: the rest is another continuation
            errs.append(abs(r.output_logprobs[t] - float(lps[t])))
    assert max(errs) <= E2E_MAX and np.mean(errs) <= E2E_MEAN, (max(errs), np.mean(errs))
    return max(errs), float(np.mean(errs))


@pytest.mark.parametrize("kind", QWEN3_KINDS)
def test_engine_teacher_forced_decode_path_vs_hf(cuda_device, kind):
    """prompt fed through the decode step (prefill_chunk=0), logits of every step vs HF fp32 and the oracle"""
    from pipelinerl_b200.engine import SamplingParams
    cfg = qwen3_tiny_cfg(kind)
    w = qwen3_tiny_weights(cfg)
    gold = np.load(GOLDEN / f"qwen3_tiny_{kind}.npz")
    tokens = gold["tokens"].tolist()
    eng = _engine(cfg, w, cuda_device, max_batch=4, max_seq_len=256, max_new_tokens=8, use_cuda_graph=False,
                  prefill_chunk=0)
    eng.add_request(tokens, SamplingParams(max_tokens=2, greedy=True))
    eng.add_request(tokens[:37], SamplingParams(max_tokens=2, greedy=True))
    got = []
    for t in range(len(tokens) - 1):
        eng.step()
        got.append(torch.log_softmax(eng.logits[0] / 0.7, -1)[tokens[t + 1]].item())
    got = np.array(got)
    want = OracleQwen3(cfg, w).score(tokens, 0.7).numpy()
    for ref in (gold["logprobs"], want):
        err = np.abs(got - ref)
        assert err.max() <= E2E_MAX and err.mean() <= E2E_MEAN, (err.max(), err.mean())
    print(f"[qwen3 engine decode-path {kind}] vs HF max {np.abs(got - gold['logprobs']).max():.4f}")


@pytest.mark.parametrize("kind,use_graph,prefill_chunk", [("wide", True, 1024), ("wide", False, 0), ("gqa4", False, 1024),
                                                          ("gqa4", True, 0), ("gqa4", True, 48)])
def test_engine_greedy_vs_hf(cuda_device, kind, use_graph, prefill_chunk):
    from pipelinerl_b200.engine import SamplingParams
    cfg = qwen3_tiny_cfg(kind)
    w = qwen3_tiny_weights(cfg)
    gold = np.load(GOLDEN / f"qwen3_tiny_{kind}.npz")
    eng = _engine(cfg, w, cuda_device, max_batch=8, max_seq_len=320, max_new_tokens=32, use_cuda_graph=use_graph,
                  prefill_chunk=prefill_chunk)
    prompts = [gold["prompts"][i, :n].tolist() for i, n in enumerate(gold["prompt_len"])]
    outs = eng.generate(prompts, SamplingParams(max_tokens=24, greedy=True))
    print(f"[qwen3 engine greedy {kind} graph={use_graph} chunk={prefill_chunk}] max/mean", _check_greedy(gold, outs, range(len(prompts))))


def test_engine_prefix_sharing_matches_unshared(cuda_device):
    from pipelinerl_b200.engine import SamplingParams
    cfg = qwen3_tiny_cfg("wide")
    w = qwen3_tiny_weights(cfg)
    gold = np.load(GOLDEN / "qwen3_tiny_wide.npz")
    prompt = gold["prompts"][2, :gold["prompt_len"][2]].tolist()      # 130 tokens: two full shared pages
    outs = {}
    for share in (True, False):
        eng = _engine(cfg, w, cuda_device, max_batch=8, max_seq_len=256, max_new_tokens=24, prefill_chunk=64,
                      prefix_sharing=share)
        res = eng.generate([prompt] * 6, SamplingParams(max_tokens=24, greedy=True))
        outs[share] = [(r.output_ids, r.output_logprobs) for r in res]
        assert (eng.stats["prefix_hits"] == 5) == share
    for (ia, la), (ib, lb) in zip(outs[True], outs[False]):
        assert ia == ib and np.allclose(la, lb, atol=1e-5)
    _check_greedy(gold, [type("R", (), {"output_ids": i, "output_logprobs": l}) for i, l in outs[True]], [2] * 6)


@pytest.mark.parametrize("kind", QWEN3_KINDS)
def test_engine_score_vs_hf(cuda_device, kind):
    cfg = qwen3_tiny_cfg(kind)
    w = qwen3_tiny_weights(cfg)
    gold = np.load(GOLDEN / f"qwen3_tiny_{kind}.npz")
    tokens = gold["tokens"].tolist()
    eng = _engine(cfg, w, cuda_device, max_batch=4, max_seq_len=256, max_new_tokens=8, prefill_chunk=64)
    got = np.array(eng.score([tokens, tokens[:3]], temperature=0.7)[0])
    want = OracleQwen3(cfg, w).score(tokens, 0.7).numpy()
    for ref in (gold["logprobs"], want):
        err = np.abs(got - ref)
        assert err.max() <= E2E_MAX and err.mean() <= E2E_MEAN, (err.max(), err.mean())


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


# ---- native learner vs the reference's rl_step on HF Qwen3 -----------------------------------------------------------
@pytest.mark.parametrize("kind", QWEN3_KINDS)
def test_native_learner_vs_reference_rl_step_on_hf_qwen3(cuda_device, kind):
    from pipelinerl_b200.finetune.optim import FusedAdamW
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from pipelinerl_b200.learner_model import NativeQwen2
    from tests.helpers import batch_from_arrays
    arrs = dict(np.load(GOLDEN / f"learner_step_qwen3_{kind}.npz"))
    meta = json.loads((GOLDEN / f"learner_step_qwen3_{kind}.json").read_text())
    cfg = qwen3_tiny_cfg(kind)
    model = NativeQwen2(cfg, cuda_device, init=qwen3_tiny_weights(cfg))
    opt = FusedAdamW(model.named_parameters(), lr=1e-3, grad_dtype=torch.float32)
    model.bind(opt)
    for keep in (cfg.num_layers, 0):     # attention half kept by the forward / recomputed in the backward
        model.body.keep_attention_layers = keep
        for g in opt.grad_views().values():
            g.zero_()
        batch = batch_from_arrays(arrs, cuda_device)
        loss, stats = rl_step(model, batch, meta["current_step"], meta["max_step"], RLConfig(**meta["config"]))
        loss.backward()
        want_loss = float(arrs["loss"])
        loss_rel = abs(loss.item() - want_loss) / max(1.0, abs(want_loss))
        assert loss_rel <= 2e-2, (loss.item(), want_loss)
        worst = 0.0
        grads = opt.grad_views()
        assert {n for n in grads if "_norm" in n} >= {f"layers.{l}.{k}_norm.weight" for l in range(2) for k in "qk"}
        for name, g in grads.items():
            key = name.replace(".", "__")
            flat = g.reshape(-1).double().cpu()
            want_norm = float(arrs["gnorm__" + key])
            rel_norm = abs(float(flat.norm()) - want_norm) / (want_norm + 1e-12)
            idx = np.unique(np.linspace(0, flat.numel() - 1, num=min(257, flat.numel())).astype(np.int64))
            got, want = flat[torch.from_numpy(idx)].numpy(), arrs["gsamp__" + key]
            rel = np.linalg.norm(got - want) / (np.linalg.norm(want) + 1e-12)
            worst = max(worst, rel_norm, rel)
            assert rel_norm <= 3e-2 and rel <= 3e-2, (name, rel_norm, rel)
        print(f"[native learner vs reference rl_step on HF Qwen3, {kind}, keep={keep}] loss rel {loss_rel:.2e} "
              f"worst gradient rel {worst:.4f}")

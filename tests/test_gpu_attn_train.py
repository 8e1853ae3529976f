"""Learner attention on sm_90a (csrc/attn_tc.cu forward, csrc/attn_bwd.cu backward) against an fp32 reference.

The op: block-diagonal causal attention over one packed row -- what the reference gets from flash-attn varlen
through HF when `position_ids` restart per packed sample (pipelinerl/finetune/rl/__init__.py:204,
conf/finetune/base.yaml:12-13,64).  Reference here: plain fp32 softmax(Q K^T / sqrt(d) + causal mask) V per segment and
head with torch autograd, on the same bf16-representable inputs.  Bar (VERDICT r1 item 1): every output / gradient
element within 2^-7 of the tensor's scale (bf16 P / dS operands + bf16 result rounding); the measured maxima are printed.
The backward must also be bitwise reproducible (fixed-order GQA reduction, no atomics)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

D = 128


def _ops():
    from pipelinerl_b200.learner_body import Ops
    return Ops()


def _reference(qkv, d_out, bounds, n_q, n_kv):
    """fp32 attention + autograd, one (segment, kv head) at a time to bound memory.  Returns out, dqkv (fp32)."""
    T = qkv.shape[0]
    R = n_q // n_kv
    x = qkv.float()
    out = torch.empty(T, n_q * D, device=qkv.device)
    dqkv = torch.zeros_like(x)
    scale = 1.0 / math.sqrt(D)
    for s, e in bounds:
        L = e - s
        mask = torch.ones(L, L, dtype=torch.bool, device=qkv.device).tril()
        for g in range(n_kv):
            kc, vc = (n_q + g) * D, (n_q + n_kv + g) * D
            k = x[s:e, kc:kc + D].clone().requires_grad_(True)
            v = x[s:e, vc:vc + D].clone().requires_grad_(True)
            for r in range(R):
                hq = (g * R + r) * D
                q = x[s:e, hq:hq + D].clone().requires_grad_(True)
                sc = (q @ k.t()) * scale
                p = torch.softmax(sc.masked_fill(~mask, float("-inf")), -1)
                o = p @ v
                out[s:e, hq:hq + D] = o.detach()
                gq, gk, gv = torch.autograd.grad(o, (q, k, v), d_out[s:e, hq:hq + D].float())
                dqkv[s:e, hq:hq + D] = gq
                dqkv[s:e, kc:kc + D] += gk
                dqkv[s:e, vc:vc + D] += gv
                del sc, p, o, gq, gk, gv
    return out, dqkv


def _run(dev, n_q, n_kv, lens, seed=0, pad_cols=0, fwd_gen=2, bwd_gen=None):
    """fwd_gen: 1 = O rescaled at every step, 2 = only when a row's maximum grew by more than 2^8 (default);
    bwd_gen: how P / dS reach the tensor core -- 1 = shared memory in both kernels, 2 = registers (default),
    3 = registers in dK/dV and shared memory in dQ, 4 = shared memory in dK/dV and registers in dQ"""
    from pipelinerl_b200 import _lib
    o = _ops()
    bwd_gen = fwd_gen if bwd_gen is None else bwd_gen
    _lib.check(o.lib.prl_attn_set_fwd_generation(fwd_gen))
    _lib.check(o.lib.prl_attn_set_bwd_generation(bwd_gen))
    T = sum(lens)
    g = torch.Generator(device=dev).manual_seed(seed)
    width = (n_q + 2 * n_kv) * D
    buf = torch.randn(T, width + pad_cols, generator=g, device=dev).to(torch.bfloat16)
    qkv = buf[:, :width]                                  # row stride may exceed the logical width
    d_out = torch.randn(T, n_q * D, generator=g, device=dev).to(torch.bfloat16)
    bounds, s = [], 0
    for L in lens:
        bounds.append((s, s + L))
        s += L
    st = torch.tensor([b[0] for b in bounds], dtype=torch.int32, device=dev)
    ln = torch.tensor(lens, dtype=torch.int32, device=dev)
    out, lse = o.attn_fwd(qkv, st, ln, max(lens), n_q, n_kv, D)
    dqkv = o.attn_bwd(qkv, out, d_out, lse, st, ln, max(lens), n_q, n_kv, D)
    dqkv2 = o.attn_bwd(qkv, out, d_out, lse, st, ln, max(lens), n_q, n_kv, D)
    torch.cuda.synchronize()
    assert torch.equal(dqkv, dqkv2), "attention backward is not bitwise reproducible"
    want_out, want_d = _reference(qkv, d_out, bounds, n_q, n_kv)
    res = {}
    err = (out.float() - want_out).abs().max().item() / want_out.abs().max().item()
    res["out"] = err
    # log-sum-exp (log2 domain of the scaled scores) against fp32, spot-checked on the first kv group
    qc, kc = 0, n_q * D
    s0, e0 = bounds[-1]
    sc = (qkv[s0:e0, qc:qc + D].float() @ qkv[s0:e0, kc:kc + D].float().t()) / math.sqrt(D)
    sc = sc.masked_fill(~torch.ones(e0 - s0, e0 - s0, dtype=torch.bool, device=dev).tril(), float("-inf"))
    want_lse = torch.logsumexp(sc, -1) / math.log(2.0)
    res["lse"] = (lse[s0:e0, 0] - want_lse).abs().max().item()
    qe, ke = n_q * D, (n_q + n_kv) * D
    for name, a, b in (("dq", 0, qe), ("dk", qe, ke), ("dv", ke, width)):
        scale = max(want_d[:, a:b].abs().max().item(), 1e-3)      # a single-token segment has dq = dk = 0 exactly
        res[name] = (dqkv[:, a:b].float() - want_d[:, a:b]).abs().max().item() / scale
    _lib.check(o.lib.prl_attn_set_fwd_generation(2))
    _lib.check(o.lib.prl_attn_set_bwd_generation(2))
    print(f"[attn_train fwd gen{fwd_gen} bwd gen{bwd_gen}] n_q={n_q} n_kv={n_kv} lens={lens if len(lens) < 8 else str(lens[:6]) + '...'}: " +
          " ".join(f"{k}={v:.2e}" for k, v in res.items()))
    assert res["out"] <= 2 ** -7, res
    assert res["lse"] <= 2e-3, res
    for k in ("dq", "dk", "dv"):
        assert res[k] <= 2 ** -7, res
    assert torch.isfinite(dqkv.float()).all() and torch.isfinite(out.float()).all()
    return res


@pytest.mark.parametrize("n_q,n_kv,lens", [
    (4, 2, [1]),                       # a single token
    (4, 2, [5, 1, 3]),
    (7, 1, [64]),
    (7, 1, [130, 17, 300, 1, 64]),     # ragged: tiles straddle segment ends
    (2, 2, [257]),                     # R = 1
    (4, 1, [200, 56]),
    (5, 1, [129, 383]),                # Qwen2.5-32B's 5:1 grouping
    (16, 1, [96, 33]),
    (28, 4, [511, 1, 700]),
])
@pytest.mark.parametrize("fwd_gen,bwd_gen", [(1, 1), (2, 2), (2, 3), (2, 4)])
def test_varlen_attention_small(cuda_device, n_q, n_kv, lens, fwd_gen, bwd_gen):
    _run(cuda_device, n_q, n_kv, lens, seed=len(lens) * 131 + n_q, fwd_gen=fwd_gen, bwd_gen=bwd_gen)


def test_varlen_attention_padded_row_stride(cuda_device):
    _run(cuda_device, 7, 1, [100, 250], seed=3, pad_cols=64)


@pytest.mark.parametrize("lens", [[2048, 2048], [4096], [3000, 5, 1091]])
def test_varlen_attention_qwen7b_heads_medium(cuda_device, lens):
    _run(cuda_device, 28, 4, lens, seed=11)


@pytest.mark.parametrize("lens,fwd_gen,bwd_gen", [([16384], 2, 2), ([8192, 8192], 2, 2), ([5000, 11000, 384], 2, 2),
                                                  ([16384], 1, 1), ([16384], 2, 1), ([16384], 1, 2), ([16384], 2, 3),
                                                  ([5000, 11000, 384], 2, 3), ([16384], 2, 4), ([8192, 8192], 2, 4),
                                                  ([5000, 11000, 384], 2, 4)])
def test_varlen_attention_qwen7b_heads_16k(cuda_device, lens, fwd_gen, bwd_gen):
    """the trainer's micro-batch size (16 384 packed tokens) at Qwen2.5-7B's 28 / 4 heads"""
    _run(cuda_device, 28, 4, lens, seed=5, fwd_gen=fwd_gen, bwd_gen=bwd_gen)


def test_attention_output_rows_outside_every_segment_are_untouched(cuda_device):
    """rows not covered by a segment are never written (the body always covers the row; this pins the bounds logic)"""
    o = _ops()
    dev = cuda_device
    n_q, n_kv, T = 4, 2, 300
    width = (n_q + 2 * n_kv) * D
    qkv = torch.randn(T, width, device=dev).to(torch.bfloat16)
    st = torch.tensor([10], dtype=torch.int32, device=dev)
    ln = torch.tensor([200], dtype=torch.int32, device=dev)
    out, lse = o.attn_fwd(qkv, st, ln, 200, n_q, n_kv, D)
    ref, _ = o.attn_fwd(qkv[10:210].contiguous(), torch.zeros(1, dtype=torch.int32, device=dev), ln, 200, n_q, n_kv, D)
    assert torch.equal(out[10:210], ref)


@pytest.mark.parametrize("n_q,n_kv,lens,sp", [
    (4, 2, [5, 1, 3, 7], 2),
    (7, 1, [130, 17, 300, 1, 64], 2),          # slices start in the middle of a sample
    (28, 4, [511, 1, 700, 836], 4),
    (5, 1, [129, 383], 4),
    (28, 4, [16384], 2),                        # one 16 384-token sample over two ranks
    (28, 4, [5000, 11000, 384], 4),
])
def test_sequence_parallel_slices_match_full_attention(cuda_device, n_q, n_kv, lens, sp):
    """prl_attn_varlen_fwd_kv / _bwd_kv (the sequence-parallel learner, reference finetune_loop.py:507-517 + make_slices
    finetune/types.py:145-180): every rank's slice of queries against the gathered K / V reproduces its rows of the
    single-rank result bit for bit (out, lse, dQ), and the ranks' dK / dV contributions sum to the single-rank dK / dV."""
    from pipelinerl_b200.learner_body import NativeBody
    o = _ops()
    dev = cuda_device
    D = 128
    T = sum(lens)
    assert T % sp == 0
    g = torch.Generator(device=dev).manual_seed(7 + T)
    qkv = torch.randn(T, (n_q + 2 * n_kv) * D, generator=g, device=dev).to(torch.bfloat16)
    d_out = torch.randn(T, n_q * D, generator=g, device=dev).to(torch.bfloat16)
    st = torch.tensor([sum(lens[:i]) for i in range(len(lens))], dtype=torch.int32, device=dev)
    ln = torch.tensor(lens, dtype=torch.int32, device=dev)
    out, lse = o.attn_fwd(qkv, st, ln, max(lens), n_q, n_kv, D)
    dqkv = o.attn_bwd(qkv, out, d_out, lse, st, ln, max(lens), n_q, n_kv, D)
    qe = n_q * D
    kv = qkv[:, qe:].contiguous()
    pos = torch.cat([torch.arange(l) for l in lens])
    dkv_sum = torch.zeros(T, 2 * n_kv * D, dtype=torch.float32, device=dev)
    Tl = T // sp
    for r in range(sp):
        a, b = r * Tl, (r + 1) * Tl
        segs = NativeBody.sp_segments(pos[a:b], a, dev)
        out_r, lse_r = o.attn_fwd_kv(qkv[a:b], kv, segs, n_q, n_kv, D)
        assert torch.equal(out_r, out[a:b]), f"rank {r}: forward rows differ from the single-rank result"
        assert torch.equal(lse_r, lse[a:b])
        dq_r = torch.empty(Tl, qe, dtype=torch.bfloat16, device=dev)
        dkv_r = o.attn_bwd_kv(qkv[a:b], kv, out_r, d_out[a:b].contiguous(), lse_r, segs, n_q, n_kv, D, dq_r)
        assert torch.equal(dq_r, dqkv[a:b, :qe]), f"rank {r}: dQ rows differ from the single-rank result"
        assert torch.all(dkv_r[b:] == 0), "keys after the slice's last query must receive no gradient"
        dkv_sum += dkv_r.float()
    want = dqkv[:, qe:].float()
    scale = max(want.abs().max().item(), 1e-3)
    err = (dkv_sum - want).abs().max().item() / scale
    print(f"[attn sp={sp}] n_q={n_q} n_kv={n_kv} lens={lens}: sum of rank dK/dV vs single rank rel {err:.2e}")
    assert err <= 2 ** -7, err

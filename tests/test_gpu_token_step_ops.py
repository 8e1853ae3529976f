"""The small kernels of the token step that run between its GEMMs (csrc/decode_ops.cu), each called through the C ABI
and compared with a plain torch restatement: the residual add + RMSNorm, the embedding gather + RMSNorm, the split-K
SiLU(gate) * up, and the sampler with its vocabulary split into slices (the vocab-parallel head of the TP engine, run here
on one GPU).

Bars:
* "one rounding": |got - ref64| <= 2^-7 |ref64| + 1e-6 for every output, and at least 99.9 % of the bf16 outputs equal
  bf16(ref64) exactly (99.5 % for SiLU, whose __expf is less accurate).  One extra mismatch is allowed so that a few-hundred
  element case is not decided by a single value that sits on a rounding boundary.
* "bitwise": torch.equal -- where the kernel promises an order of fp32 operations, the torch restatement follows it.
Every test prints what it measures.  On an H100 80GB HBM3 (700 W power limit) the fewest exact bf16 outputs of any case
were 99.980 % (residual RMSNorm), 99.999 % (embedding RMSNorm) and 99.989 % (SiLU); the sliced sampler's logprobs were
within 1.9e-6 of the whole-row call and 1.6e-6 of fp64."""
import pytest
import torch

from pipelinerl_b200 import _lib

pytestmark = pytest.mark.gpu

EPS = 1e-6


def _one_rounding(tag, got, ref64, min_exact=0.999, floor=1e-6):
    """got: bf16 kernel output, ref64: the fp64 reference of the same shape.  Exact matches are counted over references of
    at least 2^-100 in magnitude: below that fp32 evaluation gives zero (SiLU of a gate under -88.7, where exp(-gate)
    overflows fp32 and gate / (1 + exp(-gate)) is -0), which the absolute floor covers."""
    err = (got.double() - ref64).abs()
    bad = err > 2 ** -7 * ref64.abs() + floor
    normal = ref64.abs() >= 2.0 ** -100
    n = int(normal.sum())
    n_exact = int(((got == ref64.to(torch.bfloat16)) & normal).sum())
    rel = (err / ref64.abs().clamp_min(1e-30))[normal].max().item()
    print(f"[{tag}] max |err| {err.max().item():.3e}  max rel {rel:.3e}  exact {n_exact / n:.5f} ({n - n_exact} of {n} differ"
          f"{'' if n == got.numel() else f', {got.numel() - n} below 2^-100 not counted'})")
    assert not bad.any(), (tag, int(bad.sum()), err.max().item())
    assert n_exact >= min_exact * n - 1, (tag, n_exact, n)


def _rmsnorm64(h, gamma, eps=EPS):
    h64 = h.double()
    return h64 * torch.rsqrt((h64 * h64).mean(-1, keepdim=True) + eps) * gamma.double()


# ---- prl_residual_rmsnorm ----------------------------------------------------------------------------------------------
# n_split: 0 is the prefill call (the GEMM already accumulated into h), 1..8 one unrolled chunk, 9..28 a second / third /
# fourth chunk (the token step plans splits of 11 and 14, the TP engine tp x split).  H: 896 gives 224 threads, 4096 is the
# widest row one pass of threads covers, 4100 the narrowest that is staged in shared memory, 5120 Qwen3-14B / Qwen2.5-32B,
# 24576 the widest row the kernel accepts.
_RES_H = [256, 896, 4096, 4100, 5120, 8192]
_RES_CASES = ([(B, n_split, H) for B in (1, 64) for n_split in (0, 1, 8, 9, 14, 17, 28) for H in _RES_H]
              + [(1024, n_split, H) for n_split in (0, 1, 9) for H in _RES_H] + [(3, 9, 24576)])


@pytest.mark.parametrize("B,n_split,H", _RES_CASES)
def test_residual_rmsnorm_vs_fp64(cuda_device, B, n_split, H):
    lib, dev = _lib.load(), cuda_device
    g = torch.Generator().manual_seed(1000 * n_split + H + B)
    extra = 3                                                       # rows past B: must not be written
    h0 = torch.randn(B + extra, H, generator=g).to(dev)
    h0[B:] = 1234.5
    part = (torch.randn(max(n_split, 1), B, H, generator=g) * 0.5).to(dev)[:n_split].contiguous()
    part_ptr = part.data_ptr() if n_split else h0.data_ptr()      # never read with n_split = 0, but must be non-NULL
    gamma = (1 + 0.3 * torch.randn(H, generator=g)).to(torch.bfloat16).to(dev)
    pf = torch.zeros(4 << 20, dtype=torch.uint8, device=dev)      # an "upcoming weight" for the L2 prefetch
    outs = []
    for pf_ptr, pf_bytes in ((None, 0), (pf.data_ptr(), pf.numel())):
        h = h0.clone()
        x = torch.full((B + extra, H), -7.0, dtype=torch.bfloat16, device=dev)
        _lib.check(lib.prl_residual_rmsnorm(part_ptr, n_split, B, H, gamma.data_ptr(), EPS, h.data_ptr(), x.data_ptr(),
                                            pf_ptr, pf_bytes, None))
        torch.cuda.synchronize()
        outs.append((h, x))
    (h, x), (h_pf, x_pf) = outs
    # the kernel's order: h + p[0] + p[1] + ... in fp32, which is what keeps tensor-parallel ranks bit-identical
    want_h = h0[:B].clone()
    for s in range(n_split):
        want_h = want_h + part[s]
    assert torch.equal(h[:B], want_h), (h[:B] - want_h).abs().max().item()
    _one_rounding(f"residual_rmsnorm B={B} n_split={n_split} H={H}", x[:B], _rmsnorm64(h[:B], gamma))
    assert (h[B:] == 1234.5).all() and (x[B:] == -7.0).all()
    assert torch.equal(h_pf, h) and torch.equal(x_pf, x)


def test_residual_rmsnorm_refuses_widths_it_cannot_hold(cuda_device):
    lib, dev = _lib.load(), cuda_device
    buf = torch.zeros(2 * 24580, device=dev)
    gamma = torch.ones(24580, dtype=torch.bfloat16, device=dev)
    for H in (4098, 24580):        # not a multiple of 4; one float4 wider than the 96 KB row buffer
        with pytest.raises(_lib.PrlError):
            _lib.check(lib.prl_residual_rmsnorm(buf.data_ptr(), 1, 1, H, gamma.data_ptr(), EPS, buf.data_ptr(),
                                                buf.data_ptr(), None, 0, None))


# ---- prl_embed_rmsnorm --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 64, 1024])
@pytest.mark.parametrize("H", [256, 3072, 5120])
def test_embed_rmsnorm_vs_fp64(cuda_device, B, H):
    lib, dev = _lib.load(), cuda_device
    vocab = 1000
    g = torch.Generator().manual_seed(H + B)
    # the table sits between two NaN rows: a read one row before or after it would show up in h and x
    buf = torch.randn(vocab + 2, H, generator=g).to(torch.bfloat16)
    buf[0] = float("nan")
    buf[-1] = float("nan")
    buf = buf.to(dev)
    table = buf[1:vocab + 1]
    gamma = (1 + 0.3 * torch.randn(H, generator=g)).to(torch.bfloat16).to(dev)
    tok = torch.randint(0, vocab, (B,), generator=g, dtype=torch.int32)
    odd = torch.tensor([-1, vocab, -2 ** 31, 2 ** 31 - 1, vocab - 1, 0], dtype=torch.int32)[:B]
    tok[:odd.numel()] = odd                                        # ids outside the table read row 0
    want_rows = torch.where((tok < 0) | (tok >= vocab), 0, tok).long().to(dev)
    tok = tok.to(dev)
    h = torch.full((B + 2, H), 99.0, device=dev)
    x = torch.full((B + 2, H), 99.0, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_embed_rmsnorm(tok.data_ptr(), table.data_ptr(), gamma.data_ptr(), EPS, B, H, vocab, h.data_ptr(),
                                     x.data_ptr(), None))
    torch.cuda.synchronize()
    emb = table[want_rows].float()
    assert torch.equal(h[:B], emb)
    _one_rounding(f"embed_rmsnorm B={B} H={H}", x[:B], _rmsnorm64(emb, gamma))
    assert (h[B:] == 99.0).all() and (x[B:] == 99.0).all()


# ---- prl_silu_mul ---------------------------------------------------------------------------------------------------------
# I = 4: one thread; 18944 / 4 = 4736 column groups is not a multiple of the 256-thread block, so the last block is partial.
# Prefill always calls it with n_split = 1, which is the only split it takes at 1024 rows.
_SILU_I = [4, 1152, 8192, 13824, 18944]
_SILU_CASES = [(B, n_split, I) for B in (1, 64) for n_split in (1, 3, 14) for I in _SILU_I] + [(1024, 1, I) for I in _SILU_I]


def _grid_randn(g, shape, scale):
    """randn on the 2^-12 grid: any sum of up to 14 such values is exact in fp32, so the split-K sum adds no error and the
    bar measures the activation alone"""
    return torch.round(torch.randn(shape, generator=g) * scale * 4096) / 4096


@pytest.mark.parametrize("B,n_split,I", _SILU_CASES)
def test_silu_mul_vs_fp64(cuda_device, B, n_split, I):
    lib, dev = _lib.load(), cuda_device
    g = torch.Generator().manual_seed(B * 7 + n_split * 131 + I)
    gate = _grid_randn(g, (n_split, B, I), 2.0 / n_split ** 0.5)
    up = _grid_randn(g, (n_split, B, I), 1.0 / n_split ** 0.5)
    # saturating gates: exp(-gate) overflows to inf at -90 (the output is -0 where fp64 has ~1e-37) and underflows to 0
    # at +90 (the output is gate * up)
    sat = torch.tensor([30.0, -30.0, 90.0, -90.0])
    cols = torch.arange(min(I, 4))
    gate[0, :, cols] = sat[:cols.numel()] - gate[1:, :, cols].sum(0)
    part = torch.cat([gate, up], -1).to(dev)                        # [n_split, B, 2 I]: gate columns first
    act = torch.full((B + 1, I), 5.0, dtype=torch.bfloat16, device=dev)
    _lib.check(lib.prl_silu_mul(part.data_ptr(), n_split, B, I, act.data_ptr(), None, 0, None))
    torch.cuda.synchronize()
    gs, us = gate.double().sum(0), up.double().sum(0)
    assert torch.equal(gs[:, cols], sat[:cols.numel()].double().expand(B, -1))
    ref = (torch.nn.functional.silu(gs) * us).to(dev)
    _one_rounding(f"silu_mul B={B} n_split={n_split} I={I}", act[:B], ref, min_exact=0.995)
    assert (act[B:] == 5.0).all()


# ---- sampler with the vocabulary cut into slices ------------------------------------------------------------------------
def _slices(V, n_groups, equal):
    if n_groups == 1:
        return [0, V]
    if equal:
        cuts = [V * k // n_groups for k in range(n_groups + 1)]
    else:
        cuts = [0] + sorted({max(1, min(V - 1, int(V * f))) for f in (0.13, 0.5, 0.72)[:n_groups - 1]}) + [V]
    assert all(a < b for a, b in zip(cuts, cuts[1:])), cuts
    return cuts


def _sample_sliced(lib, logits, cuts, T, greedy, seed, step):
    """prl_sample_partials on each slice [cuts[k], cuts[k+1]) with its vocab_offset, merged by prl_sample_finalize"""
    B, dev = logits.shape[0], logits.device
    n_groups = len(cuts) - 1
    one = int(lib.prl_sample_workspace_bytes(B))
    ws = torch.zeros(n_groups * one, dtype=torch.uint8, device=dev)
    slices = [logits[:, lo:hi].contiguous() for lo, hi in zip(cuts, cuts[1:])]
    for k, (lo, hi) in enumerate(zip(cuts, cuts[1:])):
        _lib.check(lib.prl_sample_partials(slices[k].data_ptr(), B, hi - lo, T, int(greedy), seed, step, lo,
                                           ws.data_ptr() + k * one, None))
    ids = torch.full((B,), -5, dtype=torch.int32, device=dev)
    lps = torch.full((B,), 5.0, device=dev)
    _lib.check(lib.prl_sample_finalize(ws.data_ptr(), B, n_groups, ids.data_ptr(), lps.data_ptr(), None))
    torch.cuda.synchronize()
    return ids, lps


def _sample_whole(lib, logits, T, greedy, seed, step):
    B, V = logits.shape
    ws = torch.zeros(int(lib.prl_sample_workspace_bytes(B)), dtype=torch.uint8, device=logits.device)
    ids = torch.full((B,), -5, dtype=torch.int32, device=logits.device)
    lps = torch.full((B,), 5.0, device=logits.device)
    _lib.check(lib.prl_sample_logprob(logits.data_ptr(), B, V, T, int(greedy), seed, step, ids.data_ptr(), lps.data_ptr(),
                                      ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return ids, lps


@pytest.mark.parametrize("B", [1, 64])
@pytest.mark.parametrize("V", [7, 1000, 128256, 151936, 152064])
def test_vocab_split_sampler_equals_whole_row(cuda_device, V, B):
    """V = 7 leaves most of the 16 CTAs of a row empty; 128256 / 151936 / 152064 are the Llama 3, Qwen3 and Qwen2.5
    vocabularies.  The Gumbel noise is keyed on the global id, so a slice sees the noise of the whole row."""
    lib, dev = _lib.load(), cuda_device
    g = torch.Generator().manual_seed(V + B)
    logits = (torch.randn(B, V, generator=g) * 3).to(dev)
    worst_whole = worst_ref = 0.0
    for T in (0.6, 1.0):
        z = logits * torch.tensor(1.0 / T, dtype=torch.float32)                # the kernel's fp32 z = logit * (1/T)
        ref_lp = torch.log_softmax(z.double(), -1)
        for greedy in (True, False):
            step = 3 + int(greedy)
            ids, lps = _sample_whole(lib, logits, T, greedy, 77, step)
            if greedy:
                assert torch.equal(ids.long(), torch.argmax(z, -1))
            for n_groups, equal in ((1, True), (2, True), (2, False), (4, True), (4, False)):
                cuts = _slices(V, n_groups, equal)
                s_ids, s_lps = _sample_sliced(lib, logits, cuts, T, greedy, 77, step)
                assert torch.equal(s_ids, ids), (T, greedy, cuts)
                d_whole = (s_lps - lps).abs().max().item()
                d_ref = (s_lps.double() - ref_lp.gather(1, s_ids.long()[:, None])[:, 0]).abs().max().item()
                worst_whole, worst_ref = max(worst_whole, d_whole), max(worst_ref, d_ref)
                assert d_whole <= 1e-5 and d_ref <= 2e-5, (T, greedy, cuts, d_whole, d_ref)
    print(f"[vocab-split sampler V={V} B={B}] max |dlogprob| vs whole row {worst_whole:.2e}, vs fp64 {worst_ref:.2e}")


@pytest.mark.parametrize("V,n_groups", [(7, 4), (1000, 2), (152064, 4)])
def test_vocab_split_sampler_greedy_tie_across_a_slice_boundary(cuda_device, V, n_groups):
    """the two largest logits are equal and sit on the two sides of a slice boundary: the lower id wins, as in
    torch.argmax, whichever slice holds it"""
    lib, dev = _lib.load(), cuda_device
    B = 4
    g = torch.Generator().manual_seed(V)
    logits = torch.randn(B, V, generator=g)
    cuts = _slices(V, n_groups, True)
    for b in range(B):
        c = cuts[1 + b % (n_groups - 1)]
        logits[b, c - 1] = logits[b, c] = 10.0
    logits = logits.to(dev)
    s_ids, _ = _sample_sliced(lib, logits, cuts, 1.0, True, 0, 0)
    ids, _ = _sample_whole(lib, logits, 1.0, True, 0, 0)
    want = torch.tensor([cuts[1 + b % (n_groups - 1)] - 1 for b in range(B)], dtype=torch.int32, device=dev)
    print(f"[greedy tie V={V}] boundaries {cuts[1:-1]} -> ids {s_ids.tolist()}")
    assert torch.equal(s_ids, want) and torch.equal(ids, want)

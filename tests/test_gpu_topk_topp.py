"""Top-k / top-p sampler on the GPU (prl_sample_logprob_topkp_rows, csrc/sample_topkp.cu) and through the engine:
kept set against vLLM's fixture and the fp64 oracle, logprobs of the truncated distribution, the shared-noise identity
with the untruncated sampler, the sampled distribution, bit-identity of untruncated rows, edge cases, reproducibility."""
import asyncio

import numpy as np
import pytest
import torch

from tests.helpers import tiny_cfg, tiny_weights
from tests.topk_topp_oracle import load_fixture, truncated_logprobs

pytestmark = pytest.mark.gpu


def _lib():
    from pipelinerl_b200 import _lib
    return _lib, _lib.load()


def run_topkp(logits, T, top_k, top_p, greedy=None, seed=7, step=0, extras=True):
    """logits [B, V] fp32 on the GPU; T / top_k / top_p per row -> (ids, lps, kept, thr, log_norm) on the host."""
    _l, lib = _lib()
    B, V = logits.shape
    dev = logits.device
    inv_t = torch.tensor([1.0 / t for t in T], dtype=torch.float32, device=dev)
    gr = torch.tensor(greedy if greedy is not None else [0] * B, dtype=torch.uint8, device=dev)
    k = torch.tensor(top_k, dtype=torch.int32, device=dev)
    p = torch.tensor(top_p, dtype=torch.float32, device=dev)
    ids = torch.zeros(B, dtype=torch.int32, device=dev)
    lps = torch.zeros(B, dtype=torch.float32, device=dev)
    kept = torch.zeros(B, dtype=torch.int32, device=dev)
    thr = torch.zeros(B, dtype=torch.float32, device=dev)
    ln = torch.zeros(B, dtype=torch.float32, device=dev)
    ws = torch.zeros(int(lib.prl_sample_topkp_workspace_bytes(B, V)), dtype=torch.uint8, device=dev)
    _l.check(lib.prl_sample_logprob_topkp_rows(logits.data_ptr(), B, V, inv_t.data_ptr(), gr.data_ptr(), k.data_ptr(),
                                               p.data_ptr(), seed, step, ids.data_ptr(), lps.data_ptr(),
                                               kept.data_ptr() if extras else None, thr.data_ptr() if extras else None,
                                               ln.data_ptr() if extras else None, ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return ids.cpu(), lps.cpu(), kept.cpu(), thr.cpu(), ln.cpu()


def run_plain(logits, T, greedy=None, seed=7, step=0):
    _l, lib = _lib()
    B, V = logits.shape
    dev = logits.device
    inv_t = torch.tensor([1.0 / t for t in T], dtype=torch.float32, device=dev)
    gr = torch.tensor(greedy if greedy is not None else [0] * B, dtype=torch.uint8, device=dev)
    ids = torch.zeros(B, dtype=torch.int32, device=dev)
    lps = torch.zeros(B, dtype=torch.float32, device=dev)
    ws = torch.zeros(int(lib.prl_sample_workspace_bytes(B)), dtype=torch.uint8, device=dev)
    _l.check(lib.prl_sample_logprob_rows(logits.data_ptr(), B, V, inv_t.data_ptr(), gr.data_ptr(), seed, step,
                                         ids.data_ptr(), lps.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return ids.cpu(), lps.cpu()


def _active(V, k, p):
    return (1 <= k < V) or p < 1.0


def check_rows(logits, T, top_k, top_p, out, vllm_mask=None):
    """Kept set, threshold, log-normaliser and logprob of every truncated row against the fp64 oracle (and vLLM's mask
    where no decision is within 1e-5 of its boundary)."""
    ids, lps, kept, thr, ln = out
    x = logits.cpu()
    V = x.shape[1]
    for r in range(x.shape[0]):
        k, p = int(top_k[r]), float(top_p[r])
        if not _active(V, k, p):
            assert kept[r] == 0
            continue
        z32 = x[r] * torch.tensor(1.0 / T[r], dtype=torch.float32)            # the kernel's fp32 product
        mask = (z32 >= thr[r]).numpy()
        assert int(kept[r]) == int(mask.sum()), r
        assert mask[int(ids[r])], r
        o = truncated_logprobs(x[r].numpy(), T[r], k, p)
        if o.rule_margin > 1e-5:
            assert np.array_equal(mask, o.mask), (r, int(kept[r]), int(o.mask.sum()))
        else:   # within 1e-5 of the boundary: one of the two adjacent candidate sets
            uniq = np.unique(z32.numpy().astype(np.float64))[::-1]
            i = int(np.argmin(np.abs(uniq - o.threshold)))
            assert float(thr[r]) in {float(uniq[j]) for j in range(max(0, i - 1), min(len(uniq), i + 2))}, r
        if vllm_mask is not None and o.margin > 1e-5:
            assert np.array_equal(mask, vllm_mask[r]), r
        z64 = z32.double().numpy()
        ref_ln = float(np.log(np.exp(z64[mask] - z64[mask].max()).sum()) + z64[mask].max())
        assert abs(float(ln[r]) - ref_ln) <= 1e-5 * max(1.0, abs(ref_ln)), (r, float(ln[r]), ref_ln)
        assert abs(float(lps[r]) - (z64[int(ids[r])] - ref_ln)) <= 1e-4, r


def test_kept_set_and_logprobs_match_the_vllm_fixture(cuda_device):
    for V, f in load_fixture().items():
        logits = torch.from_numpy(f["logits"][f["kind"]]).to(cuda_device)       # [R, V]
        T, k, p = f["T"].tolist(), f["top_k"].tolist(), f["top_p"].tolist()
        out = run_topkp(logits, T, k, p, step=3)
        check_rows(logits, T, k, p, out, vllm_mask=f["mask"])
        # rows without active truncation (top_k = V): the untruncated sampler's bits
        ids0, lps0 = run_plain(logits, T, step=3)
        off = [r for r in range(len(T)) if not _active(V, k[r], p[r])]
        assert off and torch.equal(out[0][off], ids0[off]) and torch.equal(out[1][off], lps0[off])


@pytest.mark.parametrize("V", [1, 7, 640, 1000, 151643, 152064, 262144])
def test_odd_vocabularies_and_noise_identity(cuda_device, V):
    g = torch.Generator().manual_seed(V)
    B = 16
    logits = (torch.randn(B, V, generator=g) * 2.5).to(cuda_device)
    T = [0.6, 1.0, 1.3, 0.8] * 4
    k = [1, 20, 50, -1, 50, 0, V - 1, 5] * 2
    p = [1.0, 1.0, 0.95, 0.5, 0.95, 1e-6, 0.9, 1.0] * 2
    agree = 0
    for step in range(3):
        out = run_topkp(logits, T, k, p, step=step)
        check_rows(logits, T, k, p, out)
        ids0, lps0 = run_plain(logits, T, step=step)
        for r in range(B):
            z32 = logits[r].cpu() * torch.tensor(1.0 / T[r], dtype=torch.float32)
            if not _active(V, k[r], p[r]):
                assert out[0][r] == ids0[r] and out[1][r] == lps0[r]
            elif float(z32[int(ids0[r])]) >= float(out[3][r]):     # the untruncated draw is kept: same id
                assert out[0][r] == ids0[r], (V, step, r)
                agree += 1
    assert agree > 0


def test_vocabulary_limit_is_an_error(cuda_device):
    _l, lib = _lib()
    x = torch.zeros(1, 262145, device=cuda_device)
    with pytest.raises(_l.PrlError, match="262144"):
        run_topkp(x, [1.0], [5], [1.0])


def test_distribution_never_leaves_the_kept_set(cuda_device):
    B, V, T, K, P = 64, 1000, 0.8, 50, 0.9
    g = torch.Generator().manual_seed(0)
    logits = (torch.randn(1, V, generator=g) * 2).repeat(B, 1).to(cuda_device)
    o = truncated_logprobs(logits[0].cpu().numpy(), T, K, P)
    assert o.rule_margin > 1e-5
    counts = np.zeros(V)
    for step in range(400):
        ids, lps, kept, _, _ = run_topkp(logits, [T] * B, [K] * B, [P] * B, seed=1234, step=step, extras=step == 0)
        i = ids.long().numpy()
        assert o.mask[i].all()
        np.testing.assert_allclose(lps.numpy(), o.logprobs[i], atol=1e-4)
        np.add.at(counts, i, 1)
    n = counts.sum()
    prob = np.exp(o.logprobs)
    top = np.argsort(-prob)[:20]
    sigma = np.sqrt(n * prob[top] * (1 - prob[top]))
    assert (np.abs(counts[top] - n * prob[top]) < 5 * sigma + 1).all()


def test_mixed_batch_untruncated_and_greedy_rows_are_bit_identical(cuda_device):
    B, V = 64, 152064
    g = torch.Generator().manual_seed(11)
    logits = (torch.randn(B, V, generator=g) * 3).to(cuda_device)
    rs = np.random.default_rng(3)
    T = rs.choice([0.6, 0.7, 1.0, 1.3], B).tolist()
    greedy = (rs.random(B) < 0.2).astype(np.uint8).tolist()
    k = rs.choice([-1, 0, 1, 20, 50, V], B).tolist()
    p = rs.choice([1.0, 1.0, 0.5, 0.95], B).tolist()
    for step in range(2):
        out = run_topkp(logits, T, k, p, greedy=greedy, step=step)
        ids0, lps0 = run_plain(logits, T, greedy=greedy, step=step)
        plain = [r for r in range(B) if greedy[r] or not _active(V, k[r], p[r])]
        trunc = [r for r in range(B) if r not in plain]
        assert plain and trunc
        assert torch.equal(out[0][plain], ids0[plain]) and torch.equal(out[1][plain], lps0[plain])
        assert (out[2][plain] == 0).all() and (out[2][trunc] > 0).all()
        # reproducible: a second run gives the same bits
        again = run_topkp(logits, T, k, p, greedy=greedy, step=step)
        for a, b in zip(out, again):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_edge_cases(cuda_device):
    V = 1000
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4, V, generator=g) * 2
    am = int(torch.argmax(x[0]))
    ties = x[3].clone()
    order = torch.argsort(ties, descending=True)
    ties[order[8:15]] = float(ties[order[9]])                # the 10th largest value shared by 7 tokens (9th..15th)
    x[3] = ties
    logits = x.to(cuda_device)
    ids, lps, kept, thr, ln = run_topkp(logits, [1.0, 0.7, 1.0, 1.0], [1, -1, 1, 10], [1.0, 1e-6, 1e-6, 1.0])
    assert int(ids[0]) == am and float(lps[0]) == 0.0 and kept[0] == 1
    assert int(ids[1]) == int(torch.argmax(x[1])) and float(lps[1]) == 0.0 and kept[1] == 1
    assert int(ids[2]) == int(torch.argmax(x[2])) and kept[2] == 1
    assert kept[3] == 15 and float(thr[3]) == float(ties[order[9]])   # every tie at the 10th value kept


def _engine(cfg, dev, **kw):
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ParamArena
    w = tiny_weights(cfg)
    arena = ParamArena(cfg, dev)
    for name in arena.names():
        arena.view(name).copy_(w[name].to(torch.bfloat16))
    return DecodeEngine(cfg, arena, device=dev, **kw)


@pytest.mark.parametrize("use_graph", [True, False])
def test_engine_mixed_batch_logprobs_are_the_truncated_distribution(cuda_device, use_graph):
    from pipelinerl_b200.engine import SamplingParams
    cfg = tiny_cfg("gqa2")
    eng = _engine(cfg, cuda_device, max_batch=8, max_seq_len=128, max_new_tokens=24, use_cuda_graph=use_graph)
    _l, lib = _lib()
    kinds = [SamplingParams(max_tokens=20, greedy=True, ignore_eos=True),
             SamplingParams(max_tokens=20, temperature=1.0, ignore_eos=True),
             SamplingParams(max_tokens=20, temperature=0.7, top_k=50, ignore_eos=True),
             SamplingParams(max_tokens=20, temperature=1.0, top_p=0.95, ignore_eos=True),
             SamplingParams(max_tokens=20, temperature=0.7, top_k=50, top_p=0.95, ignore_eos=True),
             SamplingParams(max_tokens=20, temperature=0.7, ignore_eos=True)]
    g = torch.Generator().manual_seed(1)
    reqs = [eng.add_request(torch.randint(3, cfg.vocab_size, (9 + i,), generator=g).tolist(), sp)
            for i, sp in enumerate(kinds)]
    slot_params = {r.slot: r.params for r in reqs}
    V, B = cfg.head_rows, eng.B
    ws = torch.zeros(int(lib.prl_sample_workspace_bytes(B)), dtype=torch.uint8, device=cuda_device)
    ids0 = torch.zeros(B, dtype=torch.int32, device=cuda_device)
    lps0 = torch.zeros(B, dtype=torch.float32, device=cuda_device)
    n_trunc = 0
    for _ in range(16):
        eng.step()
        torch.cuda.synchronize()
        step = eng.step_count - 1
        logits = eng.logits.clone()
        got_ids, got_lps = eng.sampled.cpu(), eng.sampled_lp.cpu()
        _l.check(lib.prl_sample_logprob_rows(logits.data_ptr(), B, V, eng.inv_temp_rows.data_ptr(),
                                             eng.greedy_rows.data_ptr(), eng.seed, step, ids0.data_ptr(), lps0.data_ptr(),
                                             ws.data_ptr(), ws.numel(), None))
        torch.cuda.synchronize()
        for slot in range(B):
            sp = slot_params.get(slot)
            if sp is None or sp.greedy or (sp.top_k < 1 and sp.top_p >= 1.0):
                assert got_ids[slot] == ids0.cpu()[slot] and got_lps[slot] == lps0.cpu()[slot], slot
                continue
            o = truncated_logprobs(logits[slot].cpu().numpy(), sp.temperature, sp.top_k, sp.top_p)
            i = int(got_ids[slot])
            if o.rule_margin > 1e-5:
                assert o.mask[i], slot
                assert abs(float(got_lps[slot]) - o.logprobs[i]) <= 1e-4, (slot, float(got_lps[slot]), o.logprobs[i])
                n_trunc += 1
    assert n_trunc >= 30
    while eng.slot_req:
        eng.step()
        eng.harvest()
    assert not eng._truncated_slots and (eng.top_k_rows.cpu() == -1).all() and (eng.top_p_rows.cpu() == 1.0).all()


def test_reference_eval_parameters_through_the_plugin_api(cuda_device):
    """The reference's test_llm parameters (conf/base.yaml:52-57) through llm_async_generate on a real EngineServer."""
    from pipelinerl_b200.async_llm import llm_async_generate
    from pipelinerl_b200.engine import SamplingParams
    from pipelinerl_b200.llm import Prompt, SyntheticTokenizer, TrainableLLM
    from pipelinerl_b200.serving import EngineServer
    cfg = tiny_cfg("gqa2")
    eng = _engine(cfg, cuda_device, max_batch=4, max_seq_len=128, max_new_tokens=16, eos_id=2)
    server = EngineServer("topkp-plugin", eng).start()
    try:
        tok = SyntheticTokenizer(vocab_size=cfg.vocab_size)
        params = {"max_tokens": 12, "temperature": 1.0, "top_p": 0.95, "top_k": 50}
        llm = TrainableLLM(server.base_url, "tiny", parameters=params, tokenizer=tok)

        async def go():
            return await asyncio.gather(*[llm_async_generate(llm, Prompt(messages=[{"role": "user", "content": f"q{i}"}]))
                                          for i in range(6)])
        calls = asyncio.run(go())
        assert all(c.llm_info["finish_reason"] in ("stop", "length") and c.output_length_tokens >= 1 for c in calls)
        assert all(lp.logprob <= 0 for c in calls for lp in c.logprobs)
        assert server.error is None
    finally:
        server.stop()
    fused = _engine(cfg, cuda_device, max_batch=2, max_seq_len=64, max_new_tokens=8, fused_head=True)
    assert fused.sampling_features == frozenset()
    with pytest.raises(ValueError, match="not implemented by this engine"):
        fused.add_request([3, 4, 5], SamplingParams(max_tokens=4, top_k=50, top_p=0.95))

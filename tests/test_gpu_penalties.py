"""Penalties and min_p on the GPU: prl_apply_penalties against vLLM's fixture (bit-exact penalized rows, min_p masks,
processed logprobs of both samplers), its per-slot count / prompt-mask state over scripted steps, the engine end to end
against the decode oracle plus tests/penalty_oracle.py, isolation of the slots that do not use the feature, a batch
mixing every per-request sampling feature, and the engines that refuse it."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.penalty_oracle import apply_penalties, counts_and_mask, load_fixture, min_p_keep, processed_logprobs
from tests.topk_topp_oracle import truncated_logprobs

pytestmark = pytest.mark.gpu


class Rows:
    """The kernel's per-row inputs and state as device tensors, and one launch over them."""

    def __init__(self, dev, V, prompts, outs, presence, frequency, repetition, min_p=None, T=None, greedy=None,
                 out_stride=None):
        from pipelinerl_b200 import _lib
        self._lib, self.lib = _lib, _lib.load()
        B = len(prompts)
        i32 = dict(dtype=torch.int32, device=dev)
        f32 = lambda x, d: torch.tensor(x if x is not None else [d] * B, dtype=torch.float32, device=dev)  # noqa: E731
        self.B, self.V, self.dev = B, V, dev
        self.prompt = torch.full((B, max(1, max(len(p) for p in prompts))), V, **i32)
        for b, p in enumerate(prompts):
            self.prompt[b, :len(p)] = torch.tensor(p, dtype=torch.int32)
        self.prompt_len = torch.tensor([len(p) for p in prompts], **i32)
        W = out_stride or max(1, max(len(o) for o in outs))
        self.out = torch.full((B, W), V, **i32)
        for b, o in enumerate(outs):
            self.out[b, :len(o)] = torch.tensor(o, dtype=torch.int32)
        self.gen_count = torch.tensor([len(o) for o in outs], **i32)
        self.presence, self.frequency, self.repetition = f32(presence, 0.0), f32(frequency, 0.0), f32(repetition, 1.0)
        self.min_p = f32(min_p, 0.0)
        self.inv_temp = torch.tensor([1.0 / t for t in (T or [1.0] * B)], dtype=torch.float32, device=dev)
        self.greedy = torch.tensor(greedy if greedy is not None else [0] * B, dtype=torch.uint8, device=dev)
        self.counts = torch.full((B, V), 77, **i32)                 # garbage: the first launch must reset it
        self.mask = torch.full((B, (V + 31) // 32), -1, **i32)
        self.seen = torch.full((B,), -1, **i32)

    def launch(self, logits):
        p = self._lib.Penalties()
        p.logits, p.B, p.V = logits.data_ptr(), self.B, self.V
        p.presence, p.frequency, p.repetition = self.presence.data_ptr(), self.frequency.data_ptr(), self.repetition.data_ptr()
        p.min_p, p.inv_temp, p.greedy = self.min_p.data_ptr(), self.inv_temp.data_ptr(), self.greedy.data_ptr()
        p.prompt_buf, p.prompt_stride, p.prompt_len = self.prompt.data_ptr(), self.prompt.shape[1], self.prompt_len.data_ptr()
        p.out_ids, p.out_stride, p.gen_count = self.out.data_ptr(), self.out.shape[1], self.gen_count.data_ptr()
        p.counts, p.prompt_mask, p.seen = self.counts.data_ptr(), self.mask.data_ptr(), self.seen.data_ptr()
        self._lib.check(self.lib.prl_apply_penalties(C.byref(p), None))
        torch.cuda.synchronize()
        return logits


def _samplers(logits, T, greedy, top_k, top_p):
    from tests.test_gpu_topk_topp import run_plain, run_topkp
    return run_plain(logits, T, greedy=greedy), run_topkp(logits, T, top_k, top_p, greedy=greedy, extras=False)[:2]


# ---- (a) the kernel against vLLM's fixture -----------------------------------------------------------------------------
def test_kernel_matches_the_vllm_fixture(cuda_device):
    fx = load_fixture()
    V, R = int(fx["V"]), fx["logits"].shape[0]
    prompts = [list(r) for r in fx["prompt_ids"]]
    outs = [list(r) for r in fx["output_ids"]]
    T = [float(t) for t in fx["T"]]
    greedy = [int(g) for g in fx["greedy"]]
    args = (cuda_device, V, prompts, outs, fx["presence"].tolist(), fx["frequency"].tolist(), fx["repetition"].tolist())
    # penalties alone: bit for bit
    pen = Rows(*args, T=T, greedy=greedy).launch(torch.from_numpy(fx["logits"]).to(cuda_device)).cpu().numpy()
    assert np.array_equal(pen.view(np.uint32), fx["penalized"].view(np.uint32))
    # with min_p: the mask wherever no decision is within 1e-5 of its boundary, then both samplers' logprobs
    got = Rows(*args, min_p=fx["min_p"].tolist(), T=T, greedy=greedy).launch(
        torch.from_numpy(fx["logits"]).to(cuda_device))
    g = got.cpu().numpy()
    n_mask = n_lp = 0
    for i in range(R):
        mp = float(fx["min_p"][i])
        clear = True
        if mp > 0 and not greedy[i]:
            z = (fx["penalized"][i] / np.float32(T[i])).astype(np.float32)
            _, dist = min_p_keep(z, mp)
            clear = bool(dist[np.isfinite(z)].min() > 1e-5)
        kept = np.isfinite(g[i]) | ~np.isfinite(fx["penalized"][i])
        if clear:
            assert np.array_equal(kept, fx["min_p_keep"][i]), i
            n_mask += 1
        else:
            near = min_p_keep((fx["penalized"][i] / np.float32(T[i])).astype(np.float32), mp)[1] <= 1e-5
            assert np.array_equal(kept[~near], fx["min_p_keep"][i][~near]), i
    (ids0, lps0), (ids1, lps1) = _samplers(got, T, greedy, fx["top_k"].tolist(), fx["top_p"].tolist())
    for i in range(R):
        want = fx["logprobs"][i]
        truncated = 1 <= int(fx["top_k"][i]) < V or float(fx["top_p"][i]) < 1.0
        checks = [(ids1, lps1)] + ([] if truncated else [(ids0, lps0)])
        for ids, lps in checks:
            t = int(ids[i])
            if greedy[i]:
                assert t == int(fx["argmax"][i])
            assert np.isfinite(want[t]), (i, t)
            assert abs(float(lps[i]) - float(want[t])) <= 2e-5 * max(1.0, abs(float(want[t]))), (i, float(lps[i]), want[t])
            n_lp += 1
    # min_p 1.0 keeps exactly the ids at the maximum, whose ratio sits on the boundary: those rows are checked off it
    assert n_mask >= R - int(np.count_nonzero(fx["min_p"] == 1.0)) and n_lp >= R


def test_kernel_wide_rows_hash_to_vllm(cuda_device):
    fx = load_fixture()
    gen = fx["gen"]
    cases = [gen.large_case(dict(seed=int(s))) for s in fx["large_seed"]]
    rows = Rows(cuda_device, gen.V_LARGE, [c[1] for c in cases], [c[2] for c in cases], fx["large_presence"].tolist(),
                fx["large_frequency"].tolist(), fx["large_repetition"].tolist())
    got = rows.launch(torch.stack([c[0] for c in cases]).to(cuda_device)).cpu().numpy()
    for j in range(len(cases)):
        assert gen.sha256(got[j]) == str(fx["large_penalized_sha256"][j]), j


# ---- (b) the per-slot state over scripted steps ------------------------------------------------------------------------
def test_counts_and_prompt_mask_over_scripted_steps(cuda_device):
    V, steps = 1001, 40                                            # not a multiple of 4: the kernel's scalar path
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(0, V, (8192,), generator=g).tolist(), [3, 3, 999], torch.randint(0, V, (17,), generator=g).tolist()]
    prompts[0][:50] = [7] * 50                                    # duplicates
    script = torch.randint(0, V, (3, steps * 3), generator=g)
    rows = Rows(cuda_device, V, prompts, [[], [], []], [0.5, 0.0, -1.0], [0.25, 1.0, 0.0], [1.3, 1.0, 0.8],
                out_stride=steps * 3)
    rows.gen_count.zero_()
    n = [0, 0, 0]
    for s in range(steps):
        for b in range(3):
            k = 0 if s < 3 else int(torch.randint(0, 4, (1,), generator=g))   # 0: prompt-feed steps
            rows.out[b, n[b]:n[b] + k] = script[b, n[b]:n[b] + k].to(torch.int32).to(cuda_device)
            n[b] += k
        rows.gen_count.copy_(torch.tensor(n, dtype=torch.int32))
        x = torch.randn(3, V, generator=g)
        got = rows.launch(x.to(cuda_device)).cpu().numpy()
        for b in range(3):
            outs = script[b, :n[b]].numpy()
            cnt, mask = counts_and_mask(V, prompts[b], outs)
            assert np.array_equal(rows.counts[b].cpu().numpy(), cnt), (s, b)
            want = apply_penalties(x[b].numpy(), prompts[b], outs, float(rows.presence[b]), float(rows.frequency[b]),
                                   float(rows.repetition[b]))
            assert np.array_equal(got[b].view(np.uint32), want.view(np.uint32)), (s, b)
    bits = rows.mask.cpu().numpy().view(np.uint32)
    for b in range(3):
        ids = np.nonzero(np.unpackbits(bits[b].view(np.uint8), bitorder="little")[:V])[0]
        assert set(ids.tolist()) == set(prompts[b]), b
    assert rows.seen.cpu().tolist() == n
    # slot 0 reused by a new request: counts from zero, its own prompt
    rows.seen[0] = -1
    rows.prompt[0, :2] = torch.tensor([11, 12], dtype=torch.int32)
    rows.prompt_len[0] = 2
    rows.gen_count[0] = 0
    x = torch.randn(3, V, generator=g)
    rows.launch(x.to(cuda_device))
    assert int(rows.counts[0].abs().sum()) == 0
    ids = np.nonzero(np.unpackbits(rows.mask[0].cpu().numpy().view(np.uint8), bitorder="little")[:V])[0]
    assert ids.tolist() == [11, 12]


# ---- (c) the engine end to end -------------------------------------------------------------------------------------------
def _check_against_oracle(cfg, w, reqs):
    """Teacher-force each request's own outputs through the decode oracle and the penalty oracle: greedy ids are the
    penalized argmax where its top-2 margin exceeds MARGIN, sampled ids lie in the min_p / top-k / top-p kept set, and
    the logprobs meet the end-to-end bar."""
    from oracle.decode_oracle import OracleQwen2
    from tests.model_cases import E2E, MARGIN
    orc = OracleQwen2(cfg, w)
    errs, n_checked = [], 0
    for r in reqs:
        sp = r.params
        orc.reset()
        logits = orc.forward(torch.tensor(r.prompt_ids))[-1]
        for t, tok in enumerate(r.output_ids):
            pen = apply_penalties(logits.numpy(), r.prompt_ids, r.output_ids[:t], sp.presence_penalty,
                                  sp.frequency_penalty, sp.repetition_penalty)
            if sp.greedy:
                top2 = np.sort(pen)[-2:]
                if top2[1] - top2[0] > MARGIN:
                    assert tok == int(np.argmax(pen)), (r.req_id, t)
                    n_checked += 1
                lp, _ = processed_logprobs(pen, 1.0, 0.0, -1, 1.0, True)
            else:
                z = (pen / np.float32(sp.temperature)).astype(np.float32)
                lp, _ = processed_logprobs(pen, sp.temperature, sp.min_p, sp.top_k, sp.top_p, False)
                near = False
                if sp.min_p > 0:
                    near = abs(np.exp(float(z[tok]) - float(z.max())) - sp.min_p) / sp.min_p < 0.1
                if sp.top_k > 0 or sp.top_p < 1.0:
                    kept = min_p_keep(z, sp.min_p)[0] | ~np.isfinite(z) if sp.min_p > 0 else np.isfinite(z) | True
                    zz = np.where(kept, z, np.float32(-np.inf))
                    near = near or truncated_logprobs(zz, 1.0, sp.top_k, sp.top_p).rule_margin < 5e-2
                if not near:
                    assert np.isfinite(lp[tok]), (r.req_id, t, tok)
                    n_checked += 1
            if np.isfinite(lp[tok]):
                errs.append(abs(float(r.output_logprobs[t]) - float(lp[tok])))
            logits = orc.forward(torch.tensor([tok]))[-1]
    assert max(errs) <= E2E[0] and np.mean(errs) <= E2E[1], (max(errs), np.mean(errs))
    return n_checked


def _params():
    from pipelinerl_b200.engine import SamplingParams
    base = dict(max_tokens=20, ignore_eos=True)
    return [SamplingParams(greedy=True, repetition_penalty=1.3, presence_penalty=1.5, frequency_penalty=0.5, **base),
            SamplingParams(greedy=True, repetition_penalty=0.5, frequency_penalty=-2.0, min_p=0.5, **base),
            SamplingParams(temperature=1.0, min_p=0.1, **base),
            SamplingParams(temperature=0.7, repetition_penalty=1.05, presence_penalty=1.5, frequency_penalty=0.5,
                           min_p=0.05, **base),
            SamplingParams(temperature=1.3, top_k=50, top_p=0.95, min_p=0.02, presence_penalty=-2.0, **base),
            SamplingParams(temperature=1.0, **base)]


@pytest.mark.parametrize("name", ["qwen2_gqa2", "qwen3_wide", "llama_scaled"])
@pytest.mark.parametrize("use_graph, chunk", [(True, 64), (False, 0)])
def test_engine_against_the_oracles(cuda_device, name, use_graph, chunk):
    from pipelinerl_b200.engine import SamplingParams
    from tests.conformance import _case, make_engine
    case, cfg, w = _case(name)
    eng = make_engine(cfg, w, cuda_device, max_batch=8, max_seq_len=384, max_new_tokens=32, use_cuda_graph=use_graph,
                      prefill_chunk=chunk)
    g = torch.Generator().manual_seed(3)
    shared = torch.randint(3, cfg.vocab_size, (150,), generator=g).tolist()
    reqs = [eng.add_request(torch.randint(3, cfg.vocab_size, (70 + 9 * i,), generator=g).tolist(), sp)
            for i, sp in enumerate(_params())]
    # two requests sharing their prompt's pages, with different penalties
    reqs.append(eng.add_request(shared, SamplingParams(max_tokens=20, greedy=True, ignore_eos=True,
                                                       repetition_penalty=2.0)))
    reqs.append(eng.add_request(shared, SamplingParams(max_tokens=20, temperature=1.0, ignore_eos=True,
                                                       frequency_penalty=2.0, min_p=0.05)))
    done = []
    while eng.slot_req:
        eng.step()
        done += eng.harvest()
    if chunk:
        assert eng.stats["prefix_hits"] >= 1
    assert len(done) == len(reqs) and not eng._pen_slots
    assert (eng.repetition_rows.cpu() == 1).all() and (eng.min_p_rows.cpu() == 0).all()
    assert _check_against_oracle(cfg, w, done) >= 60


# ---- (d) isolation -------------------------------------------------------------------------------------------------------
def _engine(dev, **kw):
    from tests.conformance import _case, make_engine
    _, cfg, w = _case("qwen2_gqa2")
    return make_engine(cfg, w, dev, max_batch=8, max_seq_len=256, max_new_tokens=32, **kw), cfg


PLAIN_PROMPTS = [[5, 6, 7, 8, 9] * 3, [11, 12, 13] * 5, [40, 41] * 9]


def _run(eng, items):
    reqs = [eng.add_request(p, sp) for p, sp in items]
    by_id = {}
    while eng.slot_req:
        eng.step()
        for r in eng.harvest():
            by_id[r.req_id] = r
    return [(by_id[r.req_id].output_ids, by_id[r.req_id].output_logprobs) for r in reqs]


def test_plain_slots_keep_their_bits_next_to_penalized_ones(cuda_device):
    from pipelinerl_b200.engine import SamplingParams
    plain = [(p, SamplingParams(max_tokens=16, temperature=0.9, ignore_eos=True)) for p in PLAIN_PROMPTS]
    plain.append((PLAIN_PROMPTS[0], SamplingParams(max_tokens=16, greedy=True, ignore_eos=True)))
    pen = [(p, SamplingParams(max_tokens=16, temperature=0.9, ignore_eos=True, repetition_penalty=1.3, min_p=0.1,
                              presence_penalty=1.0)) for p in PLAIN_PROMPTS]
    alone = _run(_engine(cuda_device)[0], plain)
    mixed = _run(_engine(cuda_device)[0], plain + pen)
    assert mixed[:len(plain)] == alone
    assert mixed[len(plain):] != alone[:len(pen)]          # the penalties did change something


def test_a_reused_slot_starts_fresh(cuda_device):
    from pipelinerl_b200.engine import SamplingParams
    eng, _ = _engine(cuda_device)
    _run(eng, [(PLAIN_PROMPTS[1], SamplingParams(max_tokens=24, temperature=1.0, ignore_eos=True, frequency_penalty=2.0,
                                                 repetition_penalty=2.0, min_p=0.2))])
    fresh, _ = _engine(cuda_device)
    fresh.step_count = eng.step_count                      # the same sampling noise
    sp = SamplingParams(max_tokens=16, temperature=1.0, ignore_eos=True)
    assert _run(eng, [(PLAIN_PROMPTS[2], sp)]) == _run(fresh, [(PLAIN_PROMPTS[2], sp)])
    # and a penalized request in the reused slot counts from zero
    pen = SamplingParams(max_tokens=16, greedy=True, ignore_eos=True, frequency_penalty=1.0, repetition_penalty=1.2)
    fresh.step_count = eng.step_count
    assert _run(eng, [(PLAIN_PROMPTS[0], pen)]) == _run(fresh, [(PLAIN_PROMPTS[0], pen)])


def test_no_launch_and_no_state_without_penalties(cuda_device):
    from pipelinerl_b200 import _lib
    from pipelinerl_b200.engine import SamplingParams
    eng, _ = _engine(cuda_device)
    sp = SamplingParams(max_tokens=8, temperature=0.8, ignore_eos=True, min_p=0.0, repetition_penalty=1.0)
    for p in PLAIN_PROMPTS:
        eng.add_request(p, sp)
    eng.step()
    torch.cuda.synchronize()
    c0 = _lib.launch_count()
    eng.step()
    torch.cuda.synchronize()
    plain_launches = _lib.launch_count() - c0
    assert eng._pen is None and not eng._pen_slots
    eng.add_request(PLAIN_PROMPTS[0], SamplingParams(max_tokens=8, temperature=0.8, min_p=0.1))
    eng.step()                                             # its prompt's prefill
    torch.cuda.synchronize()
    c0 = _lib.launch_count()
    eng.step()
    torch.cuda.synchronize()
    assert _lib.launch_count() - c0 == plain_launches + 1


# ---- (e) every per-request sampling feature in one batch ---------------------------------------------------------------
def test_one_batch_mixes_penalties_min_tokens_stop_strings_and_truncation(cuda_device):
    from pipelinerl_b200.engine import SamplingParams
    from tests.conformance import _case, make_engine
    from tests.stop_string_oracle import fixture_tokenizer
    _, cfg, w = _case("qwen2_gqa2")
    eng = make_engine(cfg, w, cuda_device, max_batch=8, max_seq_len=256, max_new_tokens=32,
                      tokenizer=fixture_tokenizer())
    ref = make_engine(cfg, w, cuda_device, max_batch=8, max_seq_len=256, max_new_tokens=32,
                      tokenizer=fixture_tokenizer())
    items = [(PLAIN_PROMPTS[0], SamplingParams(max_tokens=20, temperature=0.8, top_k=40, top_p=0.9, min_p=0.05,
                                               presence_penalty=1.0)),
             (PLAIN_PROMPTS[1], SamplingParams(max_tokens=20, greedy=True, min_tokens=6, frequency_penalty=0.5)),
             (PLAIN_PROMPTS[2], SamplingParams(max_tokens=20, temperature=1.0, stop=("e",), repetition_penalty=1.2)),
             (PLAIN_PROMPTS[0], SamplingParams(max_tokens=20, temperature=1.0, top_p=0.9)),
             (PLAIN_PROMPTS[1], SamplingParams(max_tokens=20, greedy=True, min_tokens=4))]
    got = _run(eng, items)
    # the rows without penalties are those of the same batch where no request uses them
    plain = [(p, sp) if i >= 3 else (p, SamplingParams(max_tokens=20, greedy=True, ignore_eos=True))
             for i, (p, sp) in enumerate(items)]
    want = _run(ref, plain)
    assert got[3:] == want[3:]
    assert len(got[1][0]) >= 6 and len(got[4][0]) >= 4
    for ids, lps in got:
        assert all(np.isfinite(lps)) and all(0 <= t < cfg.vocab_size for t in ids)


# ---- (f) engines without the feature ------------------------------------------------------------------------------------
def test_fused_head_refuses_penalties(cuda_device):
    from pipelinerl_b200 import serving
    from pipelinerl_b200.engine import SamplingParams
    eng, _ = _engine(cuda_device, fused_head=True)
    assert not (serving.engine_features(eng) & {"presence_penalty", "frequency_penalty", "repetition_penalty", "min_p"})
    for kw in ({"presence_penalty": 1.0}, {"frequency_penalty": 1.0}, {"repetition_penalty": 1.1}, {"min_p": 0.1}):
        with pytest.raises(ValueError, match="not implemented by this engine"):
            eng.add_request(PLAIN_PROMPTS[0], SamplingParams(max_tokens=4, **kw))
    assert not eng.slot_req

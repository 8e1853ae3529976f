"""Llama 3 and stop-token sets on the GPU: the state advance on scripted ids against the host stop rule (and through it
vLLM's), the decode engine and the native learner against HF Llama fixtures, and a greedy continuation cut at a stop id
inside the captured step.

Bars: the state advance exactly; the engine at the end-to-end bar of the token-step tests (max |d logprob| <= 3e-2,
mean <= 6e-3, greedy ids equal wherever the top-2 margin exceeds 5e-2); the learner at the bar of the Qwen2
learner-vs-reference test (loss 2e-2 relative, every gradient 3e-2)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN
from tests.llama_oracle import LLAMA_KINDS, OracleLlama, llama_tiny_cfg, llama_tiny_weights
from tests.stop_rule_oracle import host_stop_rule, slot_setup, stop_cases

pytestmark = pytest.mark.gpu

E2E_MAX, E2E_MEAN, MARGIN = 3e-2, 6e-3, 5e-2


# ---- state advance on scripted ids -----------------------------------------------------------------------------------
def _slots():
    """one slot per vLLM fixture case, plus slots without any stop row (eos only, ignore_eos, neither)"""
    slots = []
    for c in stop_cases():
        eos_id, row, ignore = slot_setup(c)
        slots.append(dict(name=c["name"], eos=eos_id, row=row, ignore=ignore, max_tokens=c["max_tokens"], ids=c["ids"],
                          want=(c["n_out"], c["finish_reason"], c["stop_reason"])))
    for name, eos, ignore in (("plain_eos", 2, False), ("plain_ignore", 2, True), ("plain_none", -1, False)):
        ids = [5, 3, 2, 9, 1, 2, 7, 8]
        slots.append(dict(name=name, eos=eos, row=[], ignore=ignore, max_tokens=7, ids=ids, want=None))
    return slots


def _run_advance(dev, slots, eos_id, stops: str, width=16, prompt_len=3):
    """Drive prl_advance_state over scripted sampled ids.  Every slot shares eos_id (slots with another primary eos are
    not mixed into one call).  stops: "rows" (stop sets passed), "null" (stop fields NULL), "empty" (stop sets passed,
    every row empty).  -> dict of the state tensors on the host."""
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    B = len(slots)
    i32 = dict(dtype=torch.int32, device=dev)
    T = max(len(s["ids"]) for s in slots) + prompt_len
    t = dict(sampled=torch.zeros(B, **i32), lp=torch.zeros(B, dtype=torch.float32, device=dev),
             tokens=torch.zeros(B, **i32), positions=torch.zeros(B, **i32), seq_lens=torch.ones(B, **i32),
             active=torch.ones(B, dtype=torch.uint8, device=dev),
             prompt_buf=torch.arange(B * 8, dtype=torch.int32, device=dev).view(B, 8),
             prompt_len=torch.full((B,), prompt_len, **i32), out_ids=torch.full((B, 16), -7, **i32),
             out_lp=torch.zeros(B, 16, dtype=torch.float32, device=dev), gen_count=torch.zeros(B, **i32),
             max_new=torch.tensor([s["max_tokens"] for s in slots], **i32),
             finished=torch.zeros(B, dtype=torch.uint8, device=dev),
             ignore=torch.tensor([int(s["ignore"]) for s in slots], dtype=torch.uint8, device=dev),
             rows=torch.full((B, width), -3, **i32), n_stop=torch.zeros(B, **i32),
             reason=torch.full((B,), -9, **i32))
    for b, s in enumerate(slots):
        if stops == "rows" and s["row"]:
            t["rows"][b, :len(s["row"])] = torch.tensor(s["row"], dtype=torch.int32)
            t["n_stop"][b] = len(s["row"])
    st = _lib.EngineState()
    st.B = B
    st.sampled, st.sampled_logprobs = t["sampled"].data_ptr(), t["lp"].data_ptr()
    st.tokens, st.positions, st.seq_lens = t["tokens"].data_ptr(), t["positions"].data_ptr(), t["seq_lens"].data_ptr()
    st.active = t["active"].data_ptr()
    st.prompt_buf, st.prompt_stride, st.prompt_len = t["prompt_buf"].data_ptr(), 8, t["prompt_len"].data_ptr()
    st.out_ids, st.out_logprobs, st.out_stride = t["out_ids"].data_ptr(), t["out_lp"].data_ptr(), 16
    st.gen_count, st.max_new, st.finished = t["gen_count"].data_ptr(), t["max_new"].data_ptr(), t["finished"].data_ptr()
    st.eos_id, st.ignore_eos, st.ignore_eos_rows = eos_id, 0, t["ignore"].data_ptr()
    if stops != "null":
        st.stop_ids, st.stop_stride, st.n_stop = t["rows"].data_ptr(), width, t["n_stop"].data_ptr()
        st.stop_reason = t["reason"].data_ptr()
    for step in range(T):
        gen = t["gen_count"].cpu()
        ids = [s["ids"][min(int(gen[b]), len(s["ids"]) - 1)] for b, s in enumerate(slots)]
        t["sampled"].copy_(torch.tensor(ids, dtype=torch.int32))
        t["lp"].copy_(-0.01 * torch.tensor(ids, dtype=torch.float32) - step)
        _lib.check(lib.prl_advance_state(C.byref(st), None))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in t.items()}


def _check_against_host_rule(slots, got, eos_id):
    for b, s in enumerate(slots):
        out, finish, reason = host_stop_rule(s["ids"], eos_id, s["row"], s["ignore"], s["max_tokens"])
        if s["want"] is not None:
            assert (len(out), finish, reason) == s["want"], s["name"]
        n = int(got["gen_count"][b])
        assert n == len(out) and got["out_ids"][b, :n].tolist() == out, s["name"]
        assert (got["out_ids"][b, n:] == -7).all(), s["name"]
        assert int(got["finished"][b]) == (1 if finish == "stop" else 2), s["name"]
        assert int(got["active"][b]) == 0 and int(got["seq_lens"][b]) == 0, s["name"]
        assert int(got["reason"][b]) == (-1 if reason is None else reason), s["name"]


def test_advance_state_applies_vllm_stop_rule_to_mixed_slots(cuda_device):
    by_eos: dict = {}
    for s in _slots():
        by_eos.setdefault(s["eos"], []).append(s)
    assert set(by_eos) == {2, -1}
    for eos_id, slots in by_eos.items():
        got = _run_advance(cuda_device, slots, eos_id, "rows")
        _check_against_host_rule(slots, got, eos_id)


def test_advance_state_with_null_or_empty_stop_sets_keeps_the_old_behaviour(cuda_device):
    """stop fields NULL: exactly the eos / length rule, stop_reason untouched; stop sets passed but empty: the same bits"""
    slots = [dict(s, row=[], want=None) for s in _slots() if s["eos"] == 2]
    null = _run_advance(cuda_device, slots, 2, "null")
    _check_against_host_rule(slots, dict(null, reason=torch.full((len(slots),), -1, dtype=torch.int32)), 2)
    assert (null["reason"] == -9).all()
    empty = _run_advance(cuda_device, slots, 2, "empty")
    for k in null:
        if k != "reason":
            assert torch.equal(null[k], empty[k]), k
    assert (empty["reason"] == -1).all()


def test_advance_state_refuses_stop_ids_without_counts(cuda_device):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(8, dtype=torch.int32, device=cuda_device)
    st = _lib.EngineState()
    st.B = 1
    for f in ("sampled", "sampled_logprobs", "tokens", "positions", "seq_lens", "active", "prompt_buf", "prompt_len",
              "out_ids", "out_logprobs", "gen_count", "max_new", "finished"):
        setattr(st, f, x.data_ptr())
    st.stop_ids, st.stop_stride = x.data_ptr(), 4
    with pytest.raises(_lib.PrlError, match="n_stop"):
        _lib.check(lib.prl_advance_state(C.byref(st), None))


# ---- decode engine vs HF ---------------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("kind", LLAMA_KINDS)
def test_engine_teacher_forced_decode_path_vs_hf(cuda_device, kind):
    from pipelinerl_b200.engine import SamplingParams
    cfg = llama_tiny_cfg(kind)
    w = llama_tiny_weights(cfg, kind)
    gold = np.load(GOLDEN / f"llama_tiny_{kind}.npz")
    tokens = gold["tokens"].tolist()
    eng = _engine(cfg, w, cuda_device, max_batch=4, max_seq_len=384, max_new_tokens=8, use_cuda_graph=False,
                  prefill_chunk=0)
    eng.add_request(tokens, SamplingParams(max_tokens=2, greedy=True))
    eng.add_request(tokens[:37], SamplingParams(max_tokens=2, greedy=True))
    got = []
    for t in range(len(tokens) - 1):
        eng.step()
        got.append(torch.log_softmax(eng.logits[0] / 0.7, -1)[tokens[t + 1]].item())
    got = np.array(got)
    want = OracleLlama(cfg, w).score(tokens, 0.7).numpy()
    for ref in (gold["logprobs"], want):
        err = np.abs(got - ref)
        assert err.max() <= E2E_MAX and err.mean() <= E2E_MEAN, (err.max(), err.mean())


@pytest.mark.parametrize("kind,use_graph,prefill_chunk", [("scaled", True, 1024), ("scaled", False, 0),
                                                          ("tied", False, 1024), ("tied", True, 0), ("tied", True, 48)])
def test_engine_greedy_vs_hf(cuda_device, kind, use_graph, prefill_chunk):
    from pipelinerl_b200.engine import SamplingParams
    cfg = llama_tiny_cfg(kind)
    w = llama_tiny_weights(cfg, kind)
    gold = np.load(GOLDEN / f"llama_tiny_{kind}.npz")
    eng = _engine(cfg, w, cuda_device, max_batch=8, max_seq_len=320, max_new_tokens=32, use_cuda_graph=use_graph,
                  prefill_chunk=prefill_chunk)
    prompts = [gold["prompts"][i, :n].tolist() for i, n in enumerate(gold["prompt_len"])]
    outs = eng.generate(prompts, SamplingParams(max_tokens=24, greedy=True))
    print(f"[llama engine greedy {kind} graph={use_graph} chunk={prefill_chunk}]", _check_greedy(gold, outs, range(4)))


def test_engine_prefix_sharing_matches_unshared(cuda_device):
    from pipelinerl_b200.engine import SamplingParams
    cfg = llama_tiny_cfg("scaled")
    w = llama_tiny_weights(cfg, "scaled")
    gold = np.load(GOLDEN / "llama_tiny_scaled.npz")
    prompt = gold["prompts"][2, :gold["prompt_len"][2]].tolist()      # 230 tokens: three full shared pages
    outs = {}
    for share in (True, False):
        eng = _engine(cfg, w, cuda_device, max_batch=8, max_seq_len=320, max_new_tokens=24, prefill_chunk=64,
                      prefix_sharing=share)
        res = eng.generate([prompt] * 6, SamplingParams(max_tokens=24, greedy=True))
        outs[share] = [(r.output_ids, r.output_logprobs) for r in res]
        assert (eng.stats["prefix_hits"] == 5) == share
    for (ia, la), (ib, lb) in zip(outs[True], outs[False]):
        assert ia == ib and np.allclose(la, lb, atol=1e-5)
    _check_greedy(gold, [type("R", (), {"output_ids": i, "output_logprobs": l}) for i, l in outs[True]], [2] * 6)


@pytest.mark.parametrize("kind", LLAMA_KINDS)
def test_engine_score_vs_hf(cuda_device, kind):
    cfg = llama_tiny_cfg(kind)
    w = llama_tiny_weights(cfg, kind)
    gold = np.load(GOLDEN / f"llama_tiny_{kind}.npz")
    tokens = gold["tokens"].tolist()
    eng = _engine(cfg, w, cuda_device, max_batch=4, max_seq_len=384, max_new_tokens=8, prefill_chunk=64)
    got = np.array(eng.score([tokens, tokens[:3]], temperature=0.7)[0])
    want = OracleLlama(cfg, w).score(tokens, 0.7).numpy()
    for ref in (gold["logprobs"], want):
        err = np.abs(got - ref)
        assert err.max() <= E2E_MAX and err.mean() <= E2E_MEAN, (err.max(), err.mean())


def _first_new(ids, at_least=1):
    """(index k, id) of the first step >= at_least whose id does not occur earlier in `ids`"""
    for k in range(at_least, len(ids)):
        if ids[k] not in ids[:k]:
            return k, ids[k]
    pytest.skip("continuation repeats one id")


def _cut(ids, row):
    """`ids` up to and including the first id of `row` (all of it when none occurs)"""
    for k, t in enumerate(ids):
        if t in row:
            return ids[:k + 1]
    return ids


@pytest.mark.parametrize("prefill_chunk", [1024, 0])
def test_greedy_continuation_cut_at_stop_id_inside_the_graph(cuda_device, prefill_chunk):
    """Four greedy requests share a captured step, once without stop ids and once with: an ignore_eos request with its own
    stop ids (kept), one whose stop id comes from the engine's generation_config ids, the same prompt with ignore_eos (the
    engine's ids dropped), and another prompt under the engine's ids.  Each output is the stop-free run's output cut at
    its first stop id, bit for bit; the others run on unchanged."""
    from pipelinerl_b200.engine import SamplingParams
    cfg = llama_tiny_cfg("scaled")
    w = llama_tiny_weights(cfg, "scaled")
    gold = np.load(GOLDEN / "llama_tiny_scaled.npz")
    prompts = [gold["prompts"][i, :gold["prompt_len"][i]].tolist() for i in (0, 1, 1, 3)]
    greedy = dict(max_tokens=24, greedy=True)
    ignore = (True, False, True, False)

    def run(stop_ids, own):
        eng = _engine(cfg, w, cuda_device, max_batch=8, max_seq_len=320, max_new_tokens=32, use_cuda_graph=True,
                      prefill_chunk=prefill_chunk, stop_ids=stop_ids)
        reqs = [eng.add_request(p, SamplingParams(**greedy, ignore_eos=ig, stop_token_ids=o))
                for p, o, ig in zip(prompts, own, ignore)]
        done = {}
        for _ in range(400):               # prefill_chunk 0: the prompt goes through the decode step as well
            eng.step()
            done.update((r.req_id, r) for r in eng.harvest())
            if len(done) == len(reqs):
                break
        assert len(eng._graphs) == 1 and not eng._stop_slots and not eng.n_stop.any()
        return [done[r.req_id] for r in reqs]
    free = run((), [()] * 4)
    assert all((r.finish_reason, r.stop_reason, len(r.output_ids)) == ("length", None, 24) for r in free)
    _check_greedy(gold, free, [0, 1, 1, 3])
    k0, id0 = _first_new(free[0].output_ids, 3)
    k1, id1 = _first_new(free[1].output_ids, 1)
    rows = [[id0, cfg.vocab_size - 1], [id1], [], [id1]]
    cut = run((id1,), [(id0, cfg.vocab_size - 1), (), (), ()])
    for r, f, row in zip(cut, free, rows):
        want = _cut(f.output_ids, row)
        assert r.output_ids == want and r.output_logprobs == f.output_logprobs[:len(want)]
        if want[-1] in row:
            assert (r.finish_reason, r.stop_reason) == ("stop", want[-1])
        else:
            assert (r.finish_reason, r.stop_reason, len(want)) == ("length", None, 24)
    assert len(cut[0].output_ids) == k0 + 1 and len(cut[1].output_ids) == k1 + 1 and len(cut[2].output_ids) == 24


# ---- native learner vs the reference's rl_step on HF Llama -----------------------------------------------------------
@pytest.mark.parametrize("kind", LLAMA_KINDS)
def test_native_learner_vs_reference_rl_step_on_hf_llama(cuda_device, kind):
    from pipelinerl_b200.finetune.optim import FusedAdamW
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from pipelinerl_b200.learner_model import NativeQwen2
    from tests.helpers import batch_from_arrays
    arrs = dict(np.load(GOLDEN / f"learner_step_llama_{kind}.npz"))
    meta = json.loads((GOLDEN / f"learner_step_llama_{kind}.json").read_text())
    cfg = llama_tiny_cfg(kind)
    model = NativeQwen2(cfg, cuda_device, init=llama_tiny_weights(cfg, kind))
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
        for name, g in opt.grad_views().items():
            key = name.replace(".", "__")
            flat = g.reshape(-1).double().cpu()
            want_norm = float(arrs["gnorm__" + key])
            rel_norm = abs(float(flat.norm()) - want_norm) / (want_norm + 1e-12)
            idx = np.unique(np.linspace(0, flat.numel() - 1, num=min(257, flat.numel())).astype(np.int64))
            got, want = flat[torch.from_numpy(idx)].numpy(), arrs["gsamp__" + key]
            rel = np.linalg.norm(got - want) / (np.linalg.norm(want) + 1e-12)
            worst = max(worst, rel_norm, rel)
            assert rel_norm <= 3e-2 and rel <= 3e-2, (name, rel_norm, rel)
        print(f"[native learner vs reference rl_step on HF Llama, {kind}, keep={keep}] loss rel {loss_rel:.2e} "
              f"worst gradient rel {worst:.4f}")

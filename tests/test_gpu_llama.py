"""Llama 3 and stop-token sets on the GPU: the state advance on scripted ids against the host stop rule (and through it
vLLM's), a greedy continuation cut at a stop id inside the captured step, and the decode engine and native learner
against HF Llama fixtures (the checks of tests/conformance.py on the Llama cases).

Bars: the state advance exactly; the engine and the learner at the bounds of their case in tests/model_cases.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import conformance
from tests.conformance import check_greedy, make_engine
from tests.model_cases import CASES
from tests.stop_rule_oracle import host_stop_rule, slot_setup, stop_cases

pytestmark = pytest.mark.gpu


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


# ---- stop ids inside the captured step -------------------------------------------------------------------------------
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
    case = CASES["llama_scaled"]
    cfg = case["cfg"]
    w = case["weights"](cfg)
    gold = np.load(case["decode"][0])
    prompts = [gold["prompts"][i, :gold["prompt_len"][i]].tolist() for i in (0, 1, 1, 3)]
    greedy = dict(max_tokens=24, greedy=True)
    ignore = (True, False, True, False)

    def run(stop_ids, own):
        eng = make_engine(cfg, w, cuda_device, max_batch=8, max_seq_len=320, max_new_tokens=32, use_cuda_graph=True,
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
    check_greedy(gold, free, [0, 1, 1, 3])
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


# ---- decode engine and native learner vs HF Llama (tests/conformance.py) ---------------------------------------------
KINDS = ["scaled", "tied"]


@pytest.mark.parametrize("kind", KINDS)
def test_engine_teacher_forced_decode_path_vs_hf(cuda_device, kind):
    conformance.engine_teacher_forced(cuda_device, f"llama_{kind}")


@pytest.mark.parametrize("kind,use_graph,prefill_chunk", [("scaled", True, 1024), ("scaled", False, 0),
                                                          ("tied", False, 1024), ("tied", True, 0), ("tied", True, 48)])
def test_engine_greedy_vs_hf(cuda_device, kind, use_graph, prefill_chunk):
    conformance.engine_greedy_vs_hf(cuda_device, f"llama_{kind}", use_graph, prefill_chunk)


def test_engine_prefix_sharing_matches_unshared(cuda_device):
    conformance.engine_prefix_sharing(cuda_device, "llama_scaled", max_seq_len=320)


@pytest.mark.parametrize("kind", KINDS)
def test_engine_score_vs_hf(cuda_device, kind):
    conformance.engine_score(cuda_device, f"llama_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_native_learner_vs_reference_rl_step_on_hf_llama(cuda_device, kind):
    conformance.native_learner_vs_reference(cuda_device, f"llama_{kind}")

"""Stop strings and min_tokens on the GPU: prl_advance_state's string matcher and min_tokens gate on scripted ids against
the host oracle (pinned to vLLM's fixture), prl_ban_min_tokens under both samplers, the engine end to end with the
fixture tokenizer, and bit-identity / launch counts when no slot uses either feature."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from tests.helpers import tiny_cfg, tiny_weights
from tests.stop_string_oracle import fixture_tokenizer, host_rule, host_text, slot_params, stop_string_cases

pytestmark = pytest.mark.gpu
S_MAX, L_MAX = 4, 32


def _table():
    from pipelinerl_b200.engine import token_byte_table
    return token_byte_table(fixture_tokenizer())


def _run_advance(dev, cases, table, strings=True):
    """Every case in one slot of one batch; each step feeds each slot its next scripted id."""
    from pipelinerl_b200 import _lib
    from pipelinerl_b200.engine import kmp_failure
    lib = _lib.load()
    B = len(cases)
    i32 = dict(dtype=torch.int32, device=dev)
    data, offsets, special = (torch.from_numpy(np.asarray(a)).to(dev) for a in table)
    W = 64
    eos_ids = {slot_params(c)[0] for c in cases}
    assert len(eos_ids) == 1
    t = dict(sampled=torch.zeros(B, **i32), lp=torch.zeros(B, dtype=torch.float32, device=dev),
             tokens=torch.zeros(B, **i32), positions=torch.zeros(B, **i32), seq_lens=torch.ones(B, **i32),
             active=torch.ones(B, dtype=torch.uint8, device=dev), prompt_buf=torch.zeros(B, 8, **i32),
             prompt_len=torch.ones(B, **i32), out_ids=torch.full((B, W), -7, **i32),
             out_lp=torch.zeros(B, W, dtype=torch.float32, device=dev), gen_count=torch.zeros(B, **i32),
             max_new=torch.tensor([c["max_tokens"] for c in cases], **i32),
             finished=torch.zeros(B, dtype=torch.uint8, device=dev), ignore=torch.zeros(B, dtype=torch.uint8, device=dev),
             rows=torch.zeros(B, 8, **i32), n_stop=torch.zeros(B, **i32), reason=torch.full((B,), -9, **i32),
             sstr=torch.zeros(B, S_MAX, L_MAX, dtype=torch.uint8, device=dev),
             sfail=torch.zeros(B, S_MAX, L_MAX, dtype=torch.int16, device=dev), slen=torch.ones(B, S_MAX, **i32),
             nstr=torch.zeros(B, **i32), flags=torch.zeros(B, dtype=torch.uint8, device=dev),
             state=torch.zeros(B, S_MAX, **i32), match=torch.full((B,), -9, **i32), min_tok=torch.zeros(B, **i32))
    for b, c in enumerate(cases):
        _, row, _, sp = slot_params(c)
        t["rows"][b, :len(row)] = torch.tensor(row, dtype=torch.int32)
        t["n_stop"][b] = len(row)
        t["min_tok"][b] = sp.min_tokens
        for j, s in enumerate(sp.stop):
            bs = s.encode()
            t["sstr"][b, j, :len(bs)] = torch.tensor(list(bs), dtype=torch.uint8)
            t["sfail"][b, j, :len(bs)] = torch.tensor(kmp_failure(bs), dtype=torch.int16)
            t["slen"][b, j] = len(bs)
        t["nstr"][b] = len(sp.stop)
        t["flags"][b] = int(sp.include_stop_str_in_output) | 2 * int(sp.skip_special_tokens)
    st = _lib.EngineState()
    st.B = B
    st.sampled, st.sampled_logprobs = t["sampled"].data_ptr(), t["lp"].data_ptr()
    st.tokens, st.positions, st.seq_lens = t["tokens"].data_ptr(), t["positions"].data_ptr(), t["seq_lens"].data_ptr()
    st.active = t["active"].data_ptr()
    st.prompt_buf, st.prompt_stride, st.prompt_len = t["prompt_buf"].data_ptr(), 8, t["prompt_len"].data_ptr()
    st.out_ids, st.out_logprobs, st.out_stride = t["out_ids"].data_ptr(), t["out_lp"].data_ptr(), W
    st.gen_count, st.max_new, st.finished = t["gen_count"].data_ptr(), t["max_new"].data_ptr(), t["finished"].data_ptr()
    st.eos_id, st.ignore_eos, st.ignore_eos_rows = eos_ids.pop(), 0, t["ignore"].data_ptr()
    st.stop_ids, st.stop_stride, st.n_stop, st.stop_reason = t["rows"].data_ptr(), 8, t["n_stop"].data_ptr(), t["reason"].data_ptr()
    x = _lib.StopStrings()
    x.tok_bytes, x.tok_offsets, x.tok_special, x.vocab = data.data_ptr(), offsets.data_ptr(), special.data_ptr(), len(special)
    x.stop_str, x.stop_str_fail, x.stop_str_len = t["sstr"].data_ptr(), t["sfail"].data_ptr(), t["slen"].data_ptr()
    x.n_stop_str, x.max_stop_str, x.stop_str_stride = t["nstr"].data_ptr(), S_MAX, L_MAX
    x.stop_str_flags, x.stop_str_state, x.stop_str_match = t["flags"].data_ptr(), t["state"].data_ptr(), t["match"].data_ptr()
    x.min_tokens = t["min_tok"].data_ptr()
    for step in range(max(len(c["ids"]) for c in cases) + 1):
        gen = t["gen_count"].cpu()
        ids = [c["ids"][min(int(gen[b]), len(c["ids"]) - 1)] for b, c in enumerate(cases)]
        t["sampled"].copy_(torch.tensor(ids, dtype=torch.int32))
        t["lp"].copy_(-0.01 * torch.tensor(ids, dtype=torch.float32) - step)
        if strings:
            _lib.check(lib.prl_advance_state_strings(C.byref(st), C.byref(x), None))
        else:
            _lib.check(lib.prl_advance_state(C.byref(st), None))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in t.items()}


def test_advance_matcher_against_oracle_on_every_fixture_case(cuda_device):
    table = _table()
    cases = stop_string_cases()
    cases = cases + [dict(c, name=c["name"] + "_nostr", stop=[]) for c in cases[:6]]   # slots without strings
    got = _run_advance(cuda_device, cases, table)
    for b, c in enumerate(cases):
        eos_id, row, _, sp = slot_params(c)
        n, finish, reason, match = host_rule(c["ids"], table, eos_id, row, sp)
        if "_nostr" not in c["name"]:
            assert (n, finish, reason) == (c["n_out"], c["finish_reason"], c["stop_reason"]), c["name"]
        assert int(got["gen_count"][b]) == n and got["out_ids"][b, :n].tolist() == c["ids"][:n], c["name"]
        assert int(got["finished"][b]) == (1 if finish == "stop" else 2), c["name"]
        assert int(got["active"][b]) == 0 and int(got["seq_lens"][b]) == 0, c["name"]
        assert int(got["match"][b]) == match, c["name"]
        assert int(got["reason"][b]) == (reason if isinstance(reason, int) else -1), c["name"]
        if "_nostr" not in c["name"]:
            assert host_text(c["ids"][:n], finish, match, table, sp) == c["output_text"], c["name"]


def test_slots_without_strings_keep_the_old_bits(cuda_device):
    table = _table()
    cases = [dict(c, stop=[], min_tokens=0) for c in stop_string_cases()]
    on, off = _run_advance(cuda_device, cases, table, True), _run_advance(cuda_device, cases, table, False)
    for k in ("gen_count", "out_ids", "out_lp", "finished", "active", "seq_lens", "positions", "tokens", "reason"):
        assert torch.equal(on[k], off[k]), k
    assert (on["match"] == -1).all() and (off["match"] == -9).all()


def _ban(logits, gen, mt, rows):
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    dev = logits.device
    B, V = logits.shape
    w = max(1, max(len(r) for r in rows))
    ban = torch.zeros(B, w, dtype=torch.int32)
    for b, r in enumerate(rows):
        ban[b, :len(r)] = torch.tensor(r, dtype=torch.int32)
    args = [torch.tensor(gen, dtype=torch.int32, device=dev), torch.tensor(mt, dtype=torch.int32, device=dev), ban.to(dev),
            torch.tensor([len(r) for r in rows], dtype=torch.int32, device=dev)]
    _lib.check(lib.prl_ban_min_tokens(logits.data_ptr(), B, V, args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(),
                                      w, args[3].data_ptr(), None))


def test_ban_kernel_under_both_samplers(cuda_device):
    from tests.test_gpu_topk_topp import run_topkp
    from tests.topk_topp_oracle import truncated_logprobs
    g = torch.Generator().manual_seed(3)
    B, V = 16, 152064
    base = (2.0 * torch.randn(B, V, generator=g)).to(cuda_device)
    rows = [[int(i) for i in torch.randint(0, V, (5,), generator=g)] for _ in range(B)]
    for b, r in enumerate(rows):
        base[b, r] = base[b].max() + 3.0           # the banned ids would win every draw
    gen = [b % 3 for b in range(B)]
    mt = [0 if b % 4 == 3 else 2 for b in range(B)]
    banned = [gen[b] < mt[b] for b in range(B)]
    logits = base.clone()
    _ban(logits, gen, mt, rows)
    for b in range(B):
        assert torch.isinf(logits[b, rows[b]]).all() == banned[b]
        if not banned[b]:
            assert torch.equal(logits[b], base[b])
    T = [1.0, 0.7] * (B // 2)
    for top_k, top_p in ((-1, 1.0), (50, 1.0), (-1, 0.9)):
        for seed in range(3):
            ids, lps, *_ = run_topkp(logits, T, [top_k] * B, [top_p] * B, seed=seed)
            ref_ids, ref_lps, *_ = run_topkp(base, T, [top_k] * B, [top_p] * B, seed=seed)
            for b in range(B):
                if banned[b]:
                    assert int(ids[b]) not in rows[b]
                    z = logits[b].double().cpu().numpy()
                    tr = truncated_logprobs(z, T[b], top_k, top_p)
                    assert tr.mask[int(ids[b])]
                    assert abs(float(lps[b]) - tr.logprobs[int(ids[b])]) < 1e-4
                else:
                    assert int(ids[b]) == int(ref_ids[b]) and float(lps[b]) == float(ref_lps[b])


def _engine(dev, tokenizer=True, **kw):
    from tests.conformance import make_engine
    cfg = dataclasses.replace(tiny_cfg("gqa2"), vocab_size=640)
    w = tiny_weights(cfg, seed=11, std=0.05)
    return make_engine(cfg, w, dev, max_batch=8, max_seq_len=384, max_new_tokens=64,
                       tokenizer=fixture_tokenizer() if tokenizer else None, **kw)


def _text(table, ids):
    data, offsets, _ = table
    V = len(offsets) - 1
    return b"".join(bytes(data[offsets[t]:offsets[t + 1]]) for t in ids if t < V)


PROMPTS = [[5, 17, 33, 9, 101], [7, 2, 300, 41, 12, 99, 250]]


@pytest.mark.parametrize("use_graph,prefill_chunk,fused", [(True, 48, False), (False, 0, False), (True, 0, False),
                                                           (True, 48, True)])
def test_engine_cuts_greedy_output_at_a_stop_string(cuda_device, use_graph, prefill_chunk, fused):
    from pipelinerl_b200.engine import SamplingParams
    table = _table()
    eng = _engine(cuda_device, use_cuda_graph=use_graph, prefill_chunk=prefill_chunk, fused_head=fused)
    eng.greedy = True
    if fused:
        assert eng.supports_stop_strings and not eng.supports_min_tokens
    base = SamplingParams(max_tokens=40, greedy=True, ignore_eos=True)
    full = eng.generate(PROMPTS, base)
    checked = 0
    for prompt, r in zip(PROMPTS, full):
        ids = r.output_ids
        # a substring that starts inside one ordinary token and ends inside the token two later
        pick = None
        for a in range(len(ids) - 3):
            if any(t >= len(table[2]) or table[2][t] or len(_text(table, [t])) < 2 for t in ids[a:a + 3]):
                continue
            cand = _text(table, ids[:a + 3])[len(_text(table, ids[:a])) + 1:len(_text(table, ids[:a + 2])) + 1]
            try:
                pick = cand.decode("utf-8")
                break
            except UnicodeDecodeError:
                continue
        if pick is None:
            continue
        for include, skip in ((True, False), (False, True)):
            sp = SamplingParams(max_tokens=40, greedy=True, ignore_eos=True, stop=(pick,),
                                include_stop_str_in_output=include, skip_special_tokens=skip)
            got = eng.generate([prompt], sp)[0]
            eos_id, row = eng.eos_id, []
            n, finish, reason, match = host_rule(ids, table, eos_id, row, dataclasses.replace(sp, ignore_eos=True))
            assert got.output_ids == ids[:n] and (got.finish_reason, got.stop_reason) == (finish, reason)
            if include:
                assert (finish, reason) == ("stop", pick)
            assert got.output_text == host_text(ids[:n], finish, match, table, sp)
            checked += 1
    assert checked >= 2


def test_engine_min_tokens_defers_the_eos(cuda_device):
    from pipelinerl_b200.engine import SamplingParams
    eng = _engine(cuda_device, tokenizer=False)
    eng.greedy = True
    ids = eng.generate(PROMPTS[:1], SamplingParams(max_tokens=24, greedy=True, ignore_eos=True))[0].output_ids
    eng.eos_id = ids[2]
    eng._state.eos_id = ids[2]
    r = eng.generate(PROMPTS[:1], SamplingParams(max_tokens=24, greedy=True))[0]
    assert r.finish_reason == "stop" and len(r.output_ids) == 3
    r = eng.generate(PROMPTS[:1], SamplingParams(max_tokens=24, greedy=True, min_tokens=8))[0]
    assert ids[2] not in r.output_ids[:8]
    assert len(r.output_ids) >= 8
    if r.finish_reason == "stop":
        assert r.output_ids[-1] == ids[2]


def test_no_cost_when_unused(cuda_device):
    from pipelinerl_b200 import _lib
    from pipelinerl_b200.engine import SamplingParams
    outs, counts = [], []
    for tok in (True, False):
        eng = _engine(cuda_device, tokenizer=tok)
        sp = SamplingParams(max_tokens=16, temperature=0.8, ignore_eos=True)
        for p in PROMPTS:
            eng.add_request(p, sp)
        eng.step()
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        eng.step()
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - c0)
        for _ in range(20):
            eng.step()
        outs.append([(r.output_ids, r.output_logprobs) for r in sorted(eng.harvest(), key=lambda r: r.req_id)])
    assert counts[0] == counts[1]
    assert outs[0] == outs[1]

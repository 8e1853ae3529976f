"""The conformance checks every model case of tests/model_cases.py runs, one copy each.

The tests that call them keep their names in the modules of their family (tests/test_oracle_golden.py,
tests/test_gpu_decode.py and tests/test_gpu_learner_body.py for Qwen2; tests/test_{qwen3,llama}.py and
tests/test_gpu_{qwen3,llama}.py for the others) and pass the case name; the bounds come from the case.
"""
from __future__ import annotations

import json

import numpy as np
import torch

from oracle.decode_oracle import OracleQwen2
from tests.helpers import GOLDEN, row_cols
from tests.model_cases import CASES, E2E, MARGIN, hf_model


def _case(name):
    case = CASES[name]
    return case, case["cfg"], case["weights"](case["cfg"])


# ---- CPU: the oracles against HF and the reference -------------------------------------------------------------------
def decode_oracle_vs_hf(name):
    """oracle/decode_oracle.py (bf16 rounding points) vs the HF model in fp32 on the same weights, teacher-forced at every
    temperature the case has fixtures for.  Tolerance = effect of rounding activations to bf16 in a 2-layer model
    (logprobs are ~ -8).  Also: incremental decoding (one token at a time with the KV cache) == full-sequence forward."""
    case, cfg, w = _case(name)
    orc = OracleQwen2(cfg, w)
    bmax, bmean = case["oracle"]
    for path in case["decode"]:
        gold = np.load(path)
        tokens = gold["tokens"].tolist()
        lp = orc.score(tokens, float(gold["temperature"])).numpy()
        err = np.abs(lp - gold["logprobs"])
        print(f"[decode oracle vs HF {path.name}] max {err.max():.4f} mean {err.mean():.5f}")
        assert err.max() < bmax and err.mean() < bmean, (err.max(), err.mean())
    orc.reset()
    inc = torch.stack([orc.forward(torch.tensor([t]))[0] for t in tokens[:70]])
    orc.reset()
    full = orc.forward(torch.tensor(tokens[:70]))
    # same contract, different fp32 summation order -> a few bf16 rounding flips: this IS the noise floor any two
    # bf16 implementations of the step have (measured 0.9e-2 .. 1.2e-2 max on the Qwen2 models)
    assert (inc - full).abs().max() < 2.5e-2 and (inc - full).abs().mean() < 2e-3
    assert np.abs(full[-1].numpy() - 0).max() > 0.1


def decode_oracle_greedy_vs_hf(name):
    """HF's greedy continuations replayed through the oracle: the same id wherever HF's top-2 margin exceeds MARGIN,
    logprobs at the end-to-end bar."""
    case, cfg, w = _case(name)
    gold = np.load(case["decode"][0])
    orc = OracleQwen2(cfg, w)
    errs = []
    for i, n in enumerate(gold["prompt_len"]):
        orc.reset()
        logits = orc.forward(torch.tensor(gold["prompts"][i, :n]))[-1]
        for t, tok in enumerate(gold["greedy_ids"][i].tolist()):
            if gold["greedy_margin"][i, t] > MARGIN:
                assert int(torch.argmax(logits)) == tok, (i, t)
            errs.append(abs(float(torch.log_softmax(logits, -1)[tok]) - float(gold["greedy_logprobs"][i, t])))
            logits = orc.forward(torch.tensor([tok]))[-1]
    assert max(errs) <= E2E[0] and np.mean(errs) <= E2E[1], (max(errs), np.mean(errs))


def torch_module_matches_hf(name):
    """learner_model.TorchQwen2 (the learner tests' fp32 second opinion) equals the HF model's last logits in fp32."""
    from pipelinerl_b200.learner_model import TorchQwen2
    case, cfg, w = _case(name)
    gold = np.load(case["decode"][0])
    tokens = torch.from_numpy(gold["tokens"])
    with torch.no_grad():
        logits = TorchQwen2(cfg, "cpu", init=w)(tokens[None]).logits[0]
    np.testing.assert_allclose(logits[-4:].numpy(), gold["last_logits"], atol=2e-4, rtol=1e-4)


def learner_oracle_vs_reference(name):
    """oracle/learner_oracle.py (model forward, autograd backward) chained with oracle/pg_oracle.py against the
    reference's own rl_step executed on the HF model in fp32 (tests/golden/make_golden_learner*.py): loss, every
    statistic, the per-token logprobs and the gradient of every parameter (norm + 257 strided elements)."""
    from oracle import learner_oracle, pg_oracle
    case, cfg, w = _case(name)
    arrs = dict(np.load(GOLDEN / f"{case['learner']}.npz"))
    meta = json.loads((GOLDEN / f"{case['learner']}.json").read_text())
    ocfg = pg_oracle.OracleRLConfig.from_dict(meta["config"])
    loss, stats, lp, grads = learner_oracle.learner_step(cfg, w, row_cols(arrs), ocfg, meta["current_step"],
                                                         meta["max_step"])
    assert abs(loss - float(arrs["loss"])) <= 1e-5 * max(1.0, abs(float(arrs["loss"])))
    assert float((lp - torch.from_numpy(arrs["new_logprobs"])).abs().max()) <= 2e-4
    for k, v in meta["stats"].items():
        assert abs(stats[k] - v) <= 1e-5 + 1e-4 * abs(v), (k, stats[k], v)
    for pname, g in grads.items():
        key = pname.replace(".", "__")
        flat = g.reshape(-1).double()
        want_norm = float(arrs["gnorm__" + key])
        assert abs(float(flat.norm()) - want_norm) <= 1e-5 * want_norm + 1e-9, pname
        idx = np.unique(np.linspace(0, flat.numel() - 1, num=min(257, flat.numel())).astype(np.int64))
        got = flat[torch.from_numpy(idx)].numpy()
        want = arrs["gsamp__" + key]
        assert np.abs(got - want).max() <= 1e-5 * max(1e-6, np.abs(want).max()) + 1e-7, pname


def checkpoint_round_trip_opens_in_hf(tmp_path, name, n_tokens):
    """save_model_only -> HF AutoModelForCausalLM loads it as the case's architecture (Llama with its RoPE scaling) and
    computes the oracle's logits on the first n_tokens of the fixture; load_model_weights returns every fused tensor
    (q/k gains included) bit for bit."""
    from transformers import AutoModelForCausalLM

    from pipelinerl_b200.finetune.checkpoints import load_model_weights, save_model_only
    from pipelinerl_b200.model import fused_shapes
    case, cfg, w = _case(name)
    save_model_only(tmp_path / "ckpt", cfg, [(n, w[n]) for n, _ in fused_shapes(cfg)])
    back = load_model_weights(tmp_path / "ckpt", cfg)
    assert set(back) == set(w)
    for n in w:
        assert torch.equal(back[n].float(), w[n]), n
    hf = AutoModelForCausalLM.from_pretrained(str(tmp_path / "ckpt"), dtype=torch.float32,
                                              attn_implementation="eager").eval()
    direct_model = hf_model(cfg, w, tied=case["tied"]).eval()
    assert type(hf) is type(direct_model)
    tokens = torch.from_numpy(np.load(case["decode"][0])["tokens"][:n_tokens])
    with torch.no_grad():
        got = torch.log_softmax(hf(input_ids=tokens[None]).logits[0].float(), -1)
    want = torch.log_softmax(OracleQwen2(cfg, w).forward(tokens), -1)
    err = (got - want).abs()
    assert err.max().item() <= E2E[0] and err.mean().item() <= E2E[1], (err.max().item(), err.mean().item())
    # and the HF model built directly from the weights agrees with the reloaded one (nothing lost on disk)
    with torch.no_grad():
        direct = torch.log_softmax(direct_model(input_ids=tokens[None]).logits[0].float(), -1)
    assert torch.allclose(got, direct, atol=1e-5)


# ---- GPU: the decode engine and the native learner against the oracle, HF and the reference ---------------------------
def make_engine(cfg, weights, dev, **kw):
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ParamArena
    arena = ParamArena(cfg, dev)
    for name in arena.names():
        arena.view(name).copy_(weights[name].to(torch.bfloat16))
    return DecodeEngine(cfg, arena, device=dev, **kw)


def check_greedy(gold, outs, idx):
    """engine greedy outputs `outs` of the fixture's prompts `idx` vs HF's continuations: the same id wherever HF's
    top-2 margin exceeds MARGIN, logprobs at the end-to-end bar up to the first divergence -> (max, mean) error"""
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
    assert max(errs) <= E2E[0] and np.mean(errs) <= E2E[1], (max(errs), np.mean(errs))
    return max(errs), float(np.mean(errs))


def _room(n):
    """max_seq_len for an n-token sequence: the next multiple of 128 above n"""
    return 128 * (n // 128 + 1)


def engine_teacher_forced(dev, name):
    """Feed the fixture's sequence as the prompt (prefill-by-decode), read the logits of every step: vs the oracle and
    vs HF fp32 at the case's engine bounds."""
    from pipelinerl_b200.engine import SamplingParams
    case, cfg, w = _case(name)
    gold = np.load(case["decode"][0])
    tokens = gold["tokens"].tolist()
    eng = make_engine(cfg, w, dev, max_batch=4, max_seq_len=_room(len(tokens)), max_new_tokens=8, use_cuda_graph=False,
                      prefill_chunk=0)   # prefill-by-decode; materialised logits are inspected below
    eng.add_request(tokens, SamplingParams(max_tokens=2, greedy=True))
    # a second, shorter sequence in another slot exercises per-slot positions / block tables
    eng.add_request(tokens[:37], SamplingParams(max_tokens=2, greedy=True))
    got = []
    for t in range(len(tokens) - 1):
        eng.step()
        got.append(torch.log_softmax(eng.logits[0] / 0.7, -1)[tokens[t + 1]].item())
    got = np.array(got)
    want = OracleQwen2(cfg, w).score(tokens, 0.7).numpy()
    err = np.abs(got - want)
    err_hf = np.abs(got - gold["logprobs"])
    print(f"[decode e2e {name}] vs oracle max {err.max():.4f} mean {err.mean():.5f} | vs HF fp32 max {err_hf.max():.4f} "
          f"mean {err_hf.mean():.5f}  (|logprob| ~ {np.abs(want).mean():.2f})")
    bmax, bmean = case["engine"]
    assert err.max() <= bmax and err.mean() <= bmean, (err.max(), err.mean(), int(err.argmax()))
    assert err_hf.max() <= bmax and err_hf.mean() <= bmean, (err_hf.max(), err_hf.mean())


def engine_greedy_vs_hf(dev, name, use_graph, prefill_chunk):
    from pipelinerl_b200.engine import SamplingParams
    case, cfg, w = _case(name)
    gold = np.load(case["decode"][0])
    eng = make_engine(cfg, w, dev, max_batch=8, max_seq_len=320, max_new_tokens=32, use_cuda_graph=use_graph,
                      prefill_chunk=prefill_chunk)
    prompts = [gold["prompts"][i, :n].tolist() for i, n in enumerate(gold["prompt_len"])]
    outs = eng.generate(prompts, SamplingParams(max_tokens=24, greedy=True))
    print(f"[engine greedy {name} graph={use_graph} chunk={prefill_chunk}] max/mean",
          check_greedy(gold, outs, range(len(prompts))))


def engine_prefix_sharing(dev, name, max_seq_len):
    """6 attempts of the fixture's third prompt: 5 prefix hits, the same ids and logprobs as without sharing, and HF's
    greedy continuation."""
    from pipelinerl_b200.engine import SamplingParams
    case, cfg, w = _case(name)
    gold = np.load(case["decode"][0])
    prompt = gold["prompts"][2, :gold["prompt_len"][2]].tolist()
    outs = {}
    for share in (True, False):
        eng = make_engine(cfg, w, dev, max_batch=8, max_seq_len=max_seq_len, max_new_tokens=24, prefill_chunk=64,
                          prefix_sharing=share)
        res = eng.generate([prompt] * 6, SamplingParams(max_tokens=24, greedy=True))
        outs[share] = [(r.output_ids, r.output_logprobs) for r in res]
        assert (eng.stats["prefix_hits"] == 5) == share
    for (ia, la), (ib, lb) in zip(outs[True], outs[False]):
        assert ia == ib and np.allclose(la, lb, atol=1e-5)
    check_greedy(gold, [type("R", (), {"output_ids": i, "output_logprobs": l}) for i, l in outs[True]], [2] * 6)


def engine_score(dev, name):
    """engine.score() (chunked prefill + fused head with targets) == oracle / HF teacher-forced logprobs; one- and
    three-token sequences in the same call; every page and slot returned afterwards."""
    case, cfg, w = _case(name)
    gold = np.load(case["decode"][0])
    tokens = gold["tokens"].tolist()
    eng = make_engine(cfg, w, dev, max_batch=4, max_seq_len=_room(len(tokens)), max_new_tokens=8, prefill_chunk=64)
    got = np.array(eng.score([tokens, tokens[:3], [5]], temperature=0.7)[0])
    want = OracleQwen2(cfg, w).score(tokens, 0.7).numpy()
    assert got.shape == want.shape
    err = np.abs(got - want)
    err_hf = np.abs(got - gold["logprobs"])
    print(f"[score {name}] vs oracle max {err.max():.4f} mean {err.mean():.5f} | vs HF fp32 max {err_hf.max():.4f} "
          f"mean {err_hf.mean():.5f}")
    for e in (err, err_hf):
        assert e.max() <= E2E[0] and e.mean() <= E2E[1], (e.max(), e.mean())
    assert len(eng.free_pages) == eng.n_pages - 1 and len(eng.free_slots) == eng.B


def native_learner_vs_reference(dev, name):
    """Hot path 2 end to end against the REFERENCE: tests/golden/learner_step_*.npz holds the reference's rl_step run on
    the HF model (fp32, CPU) for one packed micro-batch.  Here: our rl_step on NativeQwen2 (bf16 activations, wgmma
    GEMMs, fused head, fused PG loss) -> backward -> fp32 gradient arena, once with the attention half kept by the
    forward and once recomputed in the backward.  Bounds (the case's learner_bar) are the bf16 noise floor of a
    transformer with bf16 activations: loss, the loss / entropy / kl statistics, every gradient tensor in norm and
    relative L2 on the stored elements."""
    from pipelinerl_b200.finetune.optim import FusedAdamW
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from pipelinerl_b200.learner_model import NativeQwen2
    from pipelinerl_b200.model import fused_shapes
    from tests.helpers import batch_from_arrays
    case, cfg, w = _case(name)
    bar = case["learner_bar"]
    arrs = dict(np.load(GOLDEN / f"{case['learner']}.npz"))
    meta = json.loads((GOLDEN / f"{case['learner']}.json").read_text())
    model = NativeQwen2(cfg, dev, init=w)
    opt = FusedAdamW(model.named_parameters(), lr=1e-3, grad_dtype=torch.float32)
    model.bind(opt)
    assert set(opt.grad_views()) == {n for n, _ in fused_shapes(cfg) if not n.endswith("_lo")}
    for keep in (cfg.num_layers, 0):     # attention half kept by the forward / recomputed in the backward
        model.body.keep_attention_layers = keep
        for g in opt.grad_views().values():
            g.zero_()
        batch = batch_from_arrays(arrs, dev)
        loss, stats = rl_step(model, batch, meta["current_step"], meta["max_step"], RLConfig(**meta["config"]))
        loss.backward()
        want_loss = float(arrs["loss"])
        loss_rel = abs(loss.item() - want_loss) / max(1.0, abs(want_loss))
        assert loss_rel <= bar["loss"], (loss.item(), want_loss)
        for k in ("loss", "entropy", "kl"):
            if k in meta["stats"] and k in stats:
                assert abs(stats[k] - meta["stats"][k]) <= 3e-2 * max(1.0, abs(meta["stats"][k])), (k, stats[k], meta["stats"][k])
        worst_norm = worst_samp = 0.0
        norm_rel, norm_abs = bar["grad_norm"]
        for pname, g in opt.grad_views().items():
            key = pname.replace(".", "__")
            flat = g.reshape(-1).double().cpu()
            want_norm = float(arrs["gnorm__" + key])
            worst_norm = max(worst_norm, abs(float(flat.norm()) - want_norm) / (want_norm + 1e-12))
            assert abs(float(flat.norm()) - want_norm) <= norm_rel * want_norm + norm_abs, (pname, float(flat.norm()), want_norm)
            idx = np.unique(np.linspace(0, flat.numel() - 1, num=min(257, flat.numel())).astype(np.int64))
            got, want = flat[torch.from_numpy(idx)].numpy(), arrs["gsamp__" + key]
            rel = np.linalg.norm(got - want) / (np.linalg.norm(want) + 1e-12)
            worst_samp = max(worst_samp, rel)
            assert rel <= bar["grad_samples"], (pname, rel)
        print(f"[native learner vs reference rl_step on HF, {name}, keep={keep}] loss rel {loss_rel:.2e}  "
              f"worst gradient-norm rel {worst_norm:.4f}  worst sampled-gradient rel L2 {worst_samp:.4f}")

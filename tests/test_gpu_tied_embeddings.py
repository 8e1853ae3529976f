"""Tied word embeddings trained tied, on the GPU: the decode engine on a tied arena (the head kernels pointed at the
embedding table) against HF's tied models, the native learner against the reference's rl_step on them, tied against
untied at equal weights, one optimizer step pushed into a tied sampler arena, and the TP engine's refusal."""
import json

import numpy as np
import pytest
import torch

from tests import conformance
from tests.model_cases import E2E
from tests.tied_cases import TIED_CASES as CASES   # importing it also registers the cases for tests/conformance.py

pytestmark = pytest.mark.gpu

TIED = ["tied_qwen2", "tied_qwen3", "tied_llama"]


# ---- 1. the decode engine on a tied arena ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", TIED)
def test_engine_tied_teacher_forced(cuda_device, name):
    conformance.engine_teacher_forced(cuda_device, name)


@pytest.mark.parametrize("use_graph,prefill_chunk", [(True, 0), (False, 0), (True, 48), (False, 48)])
@pytest.mark.parametrize("name", TIED)
def test_engine_tied_greedy_vs_hf(cuda_device, name, use_graph, prefill_chunk):
    conformance.engine_greedy_vs_hf(cuda_device, name, use_graph, prefill_chunk)


@pytest.mark.parametrize("name", TIED)
def test_engine_tied_prefix_sharing(cuda_device, name):
    conformance.engine_prefix_sharing(cuda_device, name, max_seq_len=320)


@pytest.mark.parametrize("name", TIED)
def test_engine_tied_score(cuda_device, name):
    conformance.engine_score(cuda_device, name)


def test_engine_tied_fused_head(cuda_device):
    """the fused sampling head reads the embedding table too: HF's greedy continuations at the end-to-end bar"""
    from pipelinerl_b200.engine import SamplingParams
    case, cfg, w = conformance._case("tied_llama")
    gold = np.load(case["decode"][0])
    prompts = [gold["prompts"][i, :n].tolist() for i, n in enumerate(gold["prompt_len"])]
    eng = conformance.make_engine(cfg, w, cuda_device, max_batch=8, max_seq_len=320, max_new_tokens=32, fused_head=True)
    outs = eng.generate(prompts, SamplingParams(max_tokens=16, greedy=True))
    print("[engine fused head tied_llama] max/mean", conformance.check_greedy(gold, outs, range(len(prompts))))


# ---- 2. the native learner against the reference on tied HF models -------------------------------------------------
@pytest.mark.parametrize("name", TIED)
def test_native_learner_tied_vs_reference(cuda_device, name):
    """loss within 2e-2, every gradient (model.embed_tokens.weight's sum of both uses included) within 3e-2, in both
    keep modes; the gradient arena holds no lm_head"""
    conformance.native_learner_vs_reference(cuda_device, name)


# ---- 3. tied against untied at equal weights ------------------------------------------------------------------------
def _learner(cfg, w, dev, **opt_kw):
    from pipelinerl_b200.finetune.optim import FusedAdamW
    from pipelinerl_b200.learner_model import NativeQwen2
    model = NativeQwen2(cfg, dev, init=w)
    opt = FusedAdamW(model.named_parameters(), grad_dtype=torch.float32, **{"lr": 1e-3, **opt_kw},
                     **model.optimizer_kwargs())
    model.bind(opt)
    return model, opt


def _step(model, opt, name, dev):
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from tests.helpers import GOLDEN, batch_from_arrays
    case = CASES[name]
    arrs = dict(np.load(GOLDEN / f"{case['learner']}.npz"))
    meta = json.loads((GOLDEN / f"{case['learner']}.json").read_text())
    opt.zero_grad()
    loss, _ = rl_step(model, batch_from_arrays(arrs, dev), meta["current_step"], meta["max_step"],
                      RLConfig(**meta["config"]))
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach()


@pytest.mark.parametrize("keep", ["attention", "gate_up", "recompute"])
@pytest.mark.parametrize("name", TIED)
def test_tied_equals_untied_sum_at_equal_weights(cuda_device, name, keep):
    """An untied learner whose lm_head equals its embedding computes the same forward bit for bit; the tied gradient of
    the one table is the untied embedding gradient plus the untied head gradient, up to the order of fp32 atomics.  So
    nothing between the head's wgrad and the embedding's scatter-add zeroes or overwrites the shared gradient view, in
    every recompute mode."""
    from dataclasses import replace
    case, cfg, w = conformance._case(name)
    ucfg = replace(cfg, tie_word_embeddings=False)
    tied, t_opt = _learner(cfg, w, cuda_device)
    untied, u_opt = _learner(ucfg, w, cuda_device)      # w holds lm_head.weight = a copy of the table
    for m in (tied, untied):
        m.body.keep_attention_layers = 0 if keep == "recompute" else cfg.num_layers
        m.body.keep_gate_up_layers = cfg.num_layers if keep == "gate_up" else 0
    lt, lu = _step(tied, t_opt, name, cuda_device), _step(untied, u_opt, name, cuda_device)
    assert torch.equal(lt, lu), (lt.item(), lu.item())
    gt, gu = t_opt.grad_views(), u_opt.grad_views()
    assert set(gu) - set(gt) == {"lm_head.weight"}
    want = gu["embed_tokens.weight"].double() + gu["lm_head.weight"].double()
    got = gt["embed_tokens.weight"].double()
    rel = float((got - want).norm() / want.norm())
    print(f"[tied vs untied sum {name} keep={keep}] rel {rel:.2e}")
    assert rel <= 1e-6
    assert float(gu["lm_head.weight"].norm()) > 1e-2 * float(want.norm())      # both uses contribute
    assert float(gu["embed_tokens.weight"].norm()) > 1e-2 * float(want.norm())


# ---- 4. one optimizer step, pushed into a tied sampler arena ----------------------------------------------------------
@pytest.mark.parametrize("name", ["tied_qwen3", "tied_llama"])
def test_tied_optimizer_step_pushes_into_a_tied_sampler_arena(cuda_device, name):
    """After one FusedAdamW step the tied learner's bf16 shadow arena has the sampler arena's layout (weights.py is
    unchanged: both sides build it from fused_shapes), pushes byte for byte, and the engine on the pushed arena matches
    the oracle on the updated weights: the table moved, so both the embedding and the head moved."""
    from oracle.decode_oracle import OracleQwen2
    from pipelinerl_b200.engine import DecodeEngine, SamplingParams
    from pipelinerl_b200.model import ArenaLayout
    from pipelinerl_b200.weights import WeightReceiver, WeightUpdateManager
    case, cfg, w = conformance._case(name)
    model, opt = _learner(cfg, w, cuda_device, lr=2e-3, weight_decay=0.01)
    lay = ArenaLayout.build(cfg)
    assert opt.names == list(lay.offsets) and opt.offsets == list(lay.offsets.values())
    assert opt.shadow_bf16.numel() == lay.total
    _step(model, opt, name, cuda_device)
    opt.step()
    model.after_optimizer_step()
    recv = WeightReceiver(cfg, cuda_device, n_pushers=1)
    try:
        mgr = WeightUpdateManager([recv], opt.shadow_bf16)
        mgr.send_weight_update(version=1)
        torch.cuda.synchronize()
        while not recv.maybe_flip():
            torch.cuda.synchronize()
        assert torch.equal(recv.arena.data, opt.shadow_bf16)
        new = {n: recv.arena.view(n).float().cpu() for n in recv.arena.names()}
        new["lm_head.weight"] = new["embed_tokens.weight"]      # the oracle reads the head under this name
        emb0 = w["embed_tokens.weight"]
        moved = (new["embed_tokens.weight"] != emb0).float().mean().item()
        assert moved > 0.5, moved
        gold = np.load(case["decode"][0])
        tokens = gold["tokens"].tolist()[:128]
        eng = DecodeEngine(cfg, recv.arena, max_batch=4, max_seq_len=256, max_new_tokens=8, device=cuda_device,
                           prefill_chunk=64)
        got = np.array(eng.score([tokens], temperature=0.7)[0])
        want = OracleQwen2(cfg, new).score(tokens, 0.7).numpy()
        before = OracleQwen2(cfg, w).score(tokens, 0.7).numpy()
        err = np.abs(got - want)
        print(f"[pushed tied arena {name}] vs oracle on the updated weights max {err.max():.4f} mean {err.mean():.5f}; "
              f"the step moved the logprobs by {np.abs(want - before).mean():.4f} on average")
        assert err.max() <= E2E[0] and err.mean() <= E2E[1]
        assert np.abs(want - before).mean() > 5 * err.mean()
        out = eng.generate([tokens[:20]], SamplingParams(max_tokens=8, greedy=True))[0]
        assert len(out.output_ids) == 8
    finally:
        recv.close()


# ---- 5. refusal ------------------------------------------------------------------------------------------------------
def test_tp_engine_refuses_tied_configs():
    from pipelinerl_b200.model import ModelConfig
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    with pytest.raises(NotImplementedError, match="tied word embeddings"):
        TPDecodeEngine(ModelConfig.qwen2_5_1_5b(tie_word_embeddings=True), None, 0, 2)
    with pytest.raises(NotImplementedError, match="tied word embeddings"):
        TPDecodeEngine(CASES["tied_qwen2"]["cfg"], None, 0, 2)

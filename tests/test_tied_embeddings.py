"""Tied word embeddings trained tied, without a GPU: the arena layout, the refusals, config.json and checkpoint round
trips, TorchQwen2 against HF's tied models, and the oracles against the reference's rl_step on tied HF models (the
`tied_*` cases of tests/tied_cases.py)."""
import json
from dataclasses import replace

import numpy as np
import pytest
import torch

from tests import conformance
from tests.model_cases import E2E, hf_model
from tests.tied_cases import TIED_CASES as CASES, hf_tied_model, tied_gradients

TIED = ["tied_qwen2", "tied_qwen3", "tied_llama"]

# config.json of Qwen/Qwen2.5-1.5B-Instruct, Qwen/Qwen3-1.7B and meta-llama/Llama-3.2-3B as published (abridged to the
# fields a ModelConfig reads, plus tie_word_embeddings)
QWEN25_1_5B = {"architectures": ["Qwen2ForCausalLM"], "model_type": "qwen2", "hidden_size": 1536,
               "intermediate_size": 8960, "num_attention_heads": 12, "num_hidden_layers": 28, "num_key_value_heads": 2,
               "rms_norm_eps": 1e-06, "rope_theta": 1000000.0, "tie_word_embeddings": True, "vocab_size": 151936}
QWEN3_1_7B = {"architectures": ["Qwen3ForCausalLM"], "model_type": "qwen3", "attention_bias": False, "head_dim": 128,
              "hidden_size": 2048, "intermediate_size": 6144, "max_position_embeddings": 40960,
              "num_attention_heads": 16, "num_hidden_layers": 28, "num_key_value_heads": 8, "rms_norm_eps": 1e-06,
              "rope_theta": 1000000, "tie_word_embeddings": True, "vocab_size": 151936}
LLAMA32_3B = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "attention_bias": False, "head_dim": 128,
              "hidden_size": 3072, "intermediate_size": 8192, "mlp_bias": False, "num_attention_heads": 24,
              "num_hidden_layers": 28, "num_key_value_heads": 8, "rms_norm_eps": 1e-05,
              "rope_scaling": {"factor": 32.0, "high_freq_factor": 4.0, "low_freq_factor": 1.0,
                               "original_max_position_embeddings": 8192, "rope_type": "llama3"},
              "rope_theta": 500000.0, "tie_word_embeddings": True, "vocab_size": 128256}


def _case(name):
    case = CASES[name]
    return case, case["cfg"], case["weights"](case["cfg"])


# ---- model description -----------------------------------------------------------------------------------------------
def test_tied_layout_drops_exactly_the_head():
    from pipelinerl_b200.model import ArenaLayout, ModelConfig, fused_shapes
    for untied in (ModelConfig.qwen2_5_1_5b(), ModelConfig.qwen3_1_7b(tie_word_embeddings=False),
                   ModelConfig.llama3_2_3b(), replace(CASES["tied_qwen2"]["cfg"], tie_word_embeddings=False)):
        tied = replace(untied, tie_word_embeddings=True)
        assert fused_shapes(tied) == [s for s in fused_shapes(untied) if s[0] != "lm_head.weight"]
        lt, lu = ArenaLayout.build(tied), ArenaLayout.build(untied)
        V, H = untied.vocab_size, untied.hidden_size
        assert lu.total - lt.total == (V * H + 63) // 64 * 64
        assert {n: lu.offsets[n] for n in lt.offsets} == lt.offsets      # every other tensor stays where it was
        assert "lm_head.weight" not in lt.hf_slices() and "lm_head.weight" in lu.hf_slices()
        assert tied.head_name == "embed_tokens.weight" and untied.head_name == "lm_head.weight"
        assert tied.num_params() == untied.num_params() - V * H


def test_qwen3_1_7b_is_its_published_config():
    from pipelinerl_b200.model import ModelConfig
    cfg = ModelConfig.qwen3_1_7b()
    assert cfg == ModelConfig.from_hf_config(QWEN3_1_7B, keep_tied=True)
    assert cfg.tie_word_embeddings and cfg.qk_norm and not cfg.qkv_bias
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_layers, cfg.num_q_heads,
            cfg.num_kv_heads) == (151936, 2048, 6144, 28, 16, 8)


def test_fp32_head_with_tying_is_refused():
    from pipelinerl_b200.model import ModelConfig
    with pytest.raises(ValueError, match="fp32 accumulation over the bf16 table"):
        ModelConfig.qwen2_5_1_5b(fp32_head=True, tie_word_embeddings=True)
    with pytest.raises(ValueError, match="W_lo = NULL"):
        ModelConfig.qwen3_1_7b(fp32_head=True)
    assert ModelConfig.qwen3_1_7b(fp32_head=True, tie_word_embeddings=False).fp32_head


@pytest.mark.parametrize("d", [QWEN25_1_5B, QWEN3_1_7B, LLAMA32_3B], ids=["qwen2", "qwen3", "llama"])
def test_from_hf_config_keep_tied_round_trips(d):
    from pipelinerl_b200.finetune.checkpoints import hf_config_dict
    from pipelinerl_b200.model import ModelConfig
    tied = ModelConfig.from_hf_config(d, keep_tied=True)
    untied = ModelConfig.from_hf_config(d)
    assert tied.tie_word_embeddings and not untied.tie_word_embeddings
    assert replace(tied, tie_word_embeddings=False) == untied
    out = hf_config_dict(tied)
    assert out["tie_word_embeddings"] is True
    assert ModelConfig.from_hf_config(json.loads(json.dumps(out)), keep_tied=True) == tied
    # untied output: byte for byte what it was, tie_word_embeddings false
    assert json.dumps(hf_config_dict(untied)) == json.dumps({**out, "tie_word_embeddings": False})
    # an untied checkpoint stays untied with keep_tied
    assert not ModelConfig.from_hf_config({**d, "tie_word_embeddings": False}, keep_tied=True).tie_word_embeddings


# ---- state dicts and checkpoints -------------------------------------------------------------------------------------
def test_tied_arena_loads_tied_state_dicts_and_refuses_untied_ones():
    from pipelinerl_b200.model import ParamArena
    case, cfg, w = _case("tied_llama")
    sd = {k: v for k, v in hf_tied_model(cfg, w).state_dict().items() if "rotary" not in k}
    assert "lm_head.weight" in sd       # HF's state_dict lists the tied head
    for with_head in (True, False):
        arena = ParamArena(cfg, "cpu")
        arena.load_hf_state_dict(sd if with_head else {k: v for k, v in sd.items() if k != "lm_head.weight"})
        assert "lm_head.weight" not in arena.names()
        assert torch.equal(arena.view("embed_tokens.weight").float(), w["embed_tokens.weight"])
        assert "lm_head.weight" not in arena.hf_state_dict()
    bad = dict(sd)
    bad["lm_head.weight"] = sd["lm_head.weight"].clone()
    bad["lm_head.weight"][3, 5] += 1.0
    with pytest.raises(ValueError, match="not tied"):
        ParamArena(cfg, "cpu").load_hf_state_dict(bad)


@pytest.mark.parametrize("name", TIED)
def test_tied_checkpoint_opens_in_hf_tied(tmp_path, name):
    """save_model_only writes no lm_head.weight and config.json says tied; load_model_weights reads every fused tensor
    back bit for bit; HF opens it as the case's architecture with the head sharing the embedding's storage, reproduces
    the case's HF fixture and computes the oracle's logits."""
    from safetensors.torch import load_file
    from transformers import AutoModelForCausalLM

    from oracle.decode_oracle import OracleQwen2
    from pipelinerl_b200.finetune.checkpoints import load_model_weights, save_model_only
    from pipelinerl_b200.model import fused_shapes
    case, cfg, w = _case(name)
    names = [n for n, _ in fused_shapes(cfg)]
    ckpt = tmp_path / "ckpt"
    save_model_only(ckpt, cfg, [(n, w[n]) for n in names])
    back = load_model_weights(ckpt, cfg)
    assert sorted(back) == sorted(names) and all(torch.equal(back[n].float(), w[n]) for n in names)
    assert "lm_head.weight" not in load_file(str(ckpt / "model.safetensors"))
    assert json.loads((ckpt / "config.json").read_text())["tie_word_embeddings"] is True
    hf = AutoModelForCausalLM.from_pretrained(str(ckpt), dtype=torch.float32, attn_implementation="eager").eval()
    assert type(hf) is type(hf_tied_model(cfg, w))
    assert hf.lm_head.weight.data_ptr() == hf.model.embed_tokens.weight.data_ptr()
    gold = np.load(case["decode"][0])
    tokens = torch.from_numpy(gold["tokens"])
    with torch.no_grad():
        logits = hf(input_ids=tokens[None]).logits[0].float()
    lp = torch.log_softmax(logits[:-1] / float(gold["temperature"]), -1).gather(1, tokens[1:, None])[:, 0]
    np.testing.assert_allclose(lp.numpy(), gold["logprobs"], atol=1e-4)
    np.testing.assert_allclose(logits[-4:].numpy(), gold["last_logits"], atol=1e-4)
    err = (torch.log_softmax(logits[:64], -1) - torch.log_softmax(OracleQwen2(cfg, w).forward(tokens[:64]), -1)).abs()
    assert err.max().item() <= E2E[0] and err.mean().item() <= E2E[1], (err.max().item(), err.mean().item())


# ---- TorchQwen2 and the oracles against HF / the reference ----------------------------------------------------------
@pytest.mark.parametrize("name", TIED)
def test_torch_module_tied_matches_hf(name):
    """TorchQwen2 on a tied config: HF's logits, and in fp32 the same loss and the same summed gradient of the one
    table as HF's tied model."""
    from pipelinerl_b200.learner_model import TorchQwen2
    conformance.torch_module_matches_hf(name)
    case, cfg, w = _case(name)
    tokens = torch.from_numpy(np.load(case["decode"][0])["tokens"][:96])
    mine = TorchQwen2(cfg, "cpu", init=w)
    assert "lm_head.weight" not in mine.names
    hf = hf_tied_model(cfg, w)
    assert hf.lm_head.weight is hf.model.embed_tokens.weight
    # the same weights untied (lm_head a copy of the table): the tied gradient is the sum of its two gradients
    untied = hf_model(replace(cfg, tie_word_embeddings=False), w)
    losses = []
    for m in (mine, hf, untied):
        logits = m(input_ids=tokens[None]).logits[0, :-1].float()
        loss = -torch.log_softmax(logits, -1).gather(1, tokens[1:, None]).mean() + 0.1 * logits.logsumexp(-1).mean()
        loss.backward()
        losses.append(loss.item())
    assert abs(losses[0] - losses[1]) <= 1e-5 * abs(losses[1]) and abs(losses[2] - losses[1]) <= 1e-6 * abs(losses[1])
    got, want = mine.p("embed_tokens.weight").grad, hf.model.embed_tokens.weight.grad
    assert float((got - want).norm()) <= 1e-4 * float(want.norm())
    g_embed, g_head = untied.model.embed_tokens.weight.grad, untied.lm_head.weight.grad
    assert float(g_embed.norm()) > 1e-3 * float(want.norm()) and float(g_head.norm()) > 1e-3 * float(want.norm())
    assert float((want - (g_embed + g_head)).norm()) <= 1e-5 * float(want.norm())


@pytest.mark.parametrize("name", TIED)
def test_decode_oracle_tied_vs_hf(name):
    conformance.decode_oracle_vs_hf(name)
    conformance.decode_oracle_greedy_vs_hf(name)


@pytest.mark.parametrize("name", TIED)
def test_learner_oracle_tied_vs_reference(name):
    """oracle/learner_oracle.py chained with oracle/pg_oracle.py against the reference's rl_step on the tied HF model
    (the bars of tests/conformance.py::learner_oracle_vs_reference): loss, statistics, logprobs and every gradient.  The
    oracle reads the head as lm_head.weight, a separate leaf holding the table, so the tied gradient is the sum of the
    two leaves' gradients; the fixture has no lm_head entry and model.embed_tokens.weight carries the sum."""
    from oracle import learner_oracle, pg_oracle
    from tests.helpers import GOLDEN, row_cols
    case, cfg, w = _case(name)
    arrs = dict(np.load(GOLDEN / f"{case['learner']}.npz"))
    meta = json.loads((GOLDEN / f"{case['learner']}.json").read_text())
    assert meta["model"] == name and "gnorm__lm_head__weight" not in arrs
    ocfg = pg_oracle.OracleRLConfig.from_dict(meta["config"])
    loss, stats, lp, grads = learner_oracle.learner_step(cfg, w, row_cols(arrs), ocfg, meta["current_step"],
                                                         meta["max_step"])
    assert abs(loss - float(arrs["loss"])) <= 1e-5 * max(1.0, abs(float(arrs["loss"])))
    assert float((lp - torch.from_numpy(arrs["new_logprobs"])).abs().max()) <= 2e-4
    for k, v in meta["stats"].items():
        assert abs(stats[k] - v) <= 1e-5 + 1e-4 * abs(v), (k, stats[k], v)
    grads = tied_gradients(grads)
    assert sorted(k[len("gnorm__"):] for k in arrs if k.startswith("gnorm__")) == \
        sorted(n.replace(".", "__") for n in grads)
    for pname, g in grads.items():
        key = pname.replace(".", "__")
        flat = g.reshape(-1).double()
        want_norm = float(arrs["gnorm__" + key])
        assert abs(float(flat.norm()) - want_norm) <= 1e-5 * want_norm + 1e-9, pname
        idx = np.unique(np.linspace(0, flat.numel() - 1, num=min(257, flat.numel())).astype(np.int64))
        want = arrs["gsamp__" + key]
        assert np.abs(flat[torch.from_numpy(idx)].numpy() - want).max() <= 1e-5 * max(1e-6, np.abs(want).max()) + 1e-7

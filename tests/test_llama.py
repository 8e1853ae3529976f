"""Llama 3 support without a GPU: the RoPE table, the model description, the checkpoint format and the oracles against
HF Llama and the reference (the checks of tests/conformance.py on the Llama cases of tests/model_cases.py)."""
import hashlib
import json
import math

import numpy as np
import pytest
import torch

from tests import conformance
from tests.model_cases import CASES, hf_model, llama_tiny_cfg, llama_tiny_weights

KINDS = ["scaled", "tied"]

# config.json of meta-llama/Llama-3.1-8B-Instruct and meta-llama/Llama-3.2-3B as published (transformers 4.x format)
LLAMA31_8B_INSTRUCT = {
    "architectures": ["LlamaForCausalLM"], "attention_bias": False, "attention_dropout": 0.0, "bos_token_id": 128000,
    "eos_token_id": [128001, 128008, 128009], "hidden_act": "silu", "hidden_size": 4096, "initializer_range": 0.02,
    "intermediate_size": 14336, "max_position_embeddings": 131072, "mlp_bias": False, "model_type": "llama",
    "num_attention_heads": 32, "num_hidden_layers": 32, "num_key_value_heads": 8, "pretraining_tp": 1,
    "rms_norm_eps": 1e-05, "rope_scaling": {"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                            "original_max_position_embeddings": 8192, "rope_type": "llama3"},
    "rope_theta": 500000.0, "tie_word_embeddings": False, "torch_dtype": "bfloat16", "transformers_version": "4.42.3",
    "use_cache": True, "vocab_size": 128256}
LLAMA32_3B = {
    "architectures": ["LlamaForCausalLM"], "attention_bias": False, "attention_dropout": 0.0, "bos_token_id": 128000,
    "eos_token_id": 128001, "head_dim": 128, "hidden_act": "silu", "hidden_size": 3072, "initializer_range": 0.02,
    "intermediate_size": 8192, "max_position_embeddings": 131072, "mlp_bias": False, "model_type": "llama",
    "num_attention_heads": 24, "num_hidden_layers": 28, "num_key_value_heads": 8, "pretraining_tp": 1,
    "rms_norm_eps": 1e-05, "rope_scaling": {"factor": 32.0, "high_freq_factor": 4.0, "low_freq_factor": 1.0,
                                            "original_max_position_embeddings": 8192, "rope_type": "llama3"},
    "rope_theta": 500000.0, "tie_word_embeddings": True, "torch_dtype": "bfloat16", "transformers_version": "4.45.0.dev0",
    "use_cache": True, "vocab_size": 128256}


# ---- RoPE table ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("theta", [1_000_000.0, 500_000.0, 10_000.0])
def test_rope_inv_freq_default_is_todays_table(theta):
    from pipelinerl_b200.model import ModelConfig, rope_inv_freq
    cfg = ModelConfig.tiny(rope_theta=theta)
    today = 1.0 / (cfg.rope_theta ** (torch.arange(0, 128, 2, dtype=torch.int64).float() / 128))
    got = rope_inv_freq(cfg)
    assert got.dtype == torch.float32 and got.shape == (64,) and torch.equal(got, today)


def _hf_llama3_table(cfg):
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    hc = LlamaConfig(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_q_heads, head_dim=cfg.head_dim,
                     rope_theta=cfg.rope_theta, rope_scaling=cfg.rope_scaling.hf_dict(), max_position_embeddings=131072)
    return ROPE_INIT_FUNCTIONS["llama3"](hc, "cpu")[0]


@pytest.mark.parametrize("which", ["llama3_1_8b", "llama3_2_3b", "scaled", "tied"])
def test_rope_inv_freq_llama3_equals_transformers(which):
    from pipelinerl_b200.model import ModelConfig, rope_inv_freq
    cfg = getattr(ModelConfig, which)() if which.startswith("llama") else llama_tiny_cfg(which)
    want = _hf_llama3_table(cfg)
    got = rope_inv_freq(cfg)
    assert want.dtype == got.dtype == torch.float32 and torch.equal(got, want)


def test_scaled_fixture_config_has_all_three_bands():
    from pipelinerl_b200.model import ModelConfig, rope_inv_freq
    cfg = llama_tiny_cfg("scaled")
    s = cfg.rope_scaling
    base = rope_inv_freq(ModelConfig.tiny(rope_theta=cfg.rope_theta))
    wavelen = 2 * math.pi / base
    high = wavelen < s.original_max_position_embeddings / s.high_freq_factor
    low = wavelen > s.original_max_position_embeddings / s.low_freq_factor
    mid = ~high & ~low
    assert high.sum() >= 2 and mid.sum() >= 2 and low.sum() >= 2, (high.sum(), mid.sum(), low.sum())
    got = rope_inv_freq(cfg)
    assert torch.equal(got[high], base[high])
    assert torch.equal(got[low], base[low] / s.factor)
    assert ((got[mid] < base[mid]) & (got[mid] > base[mid] / s.factor)).all()


# ---- oracles vs HF and the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_llama_oracle_teacher_forced_vs_hf(kind):
    conformance.decode_oracle_vs_hf(f"llama_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_llama_oracle_greedy_vs_hf(kind):
    conformance.decode_oracle_greedy_vs_hf(f"llama_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_torch_llama_module_matches_hf_in_fp32(kind):
    conformance.torch_module_matches_hf(f"llama_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_learner_oracle_vs_reference_rl_step_on_hf_llama(kind):
    conformance.learner_oracle_vs_reference(f"llama_{kind}")


# ---- oracle vs HF: the scaled table is visible in the logprobs --------------------------------------------------------
def test_unscaled_rope_table_misses_the_hf_bar():
    """tests/test_oracle_golden.py holds the oracle at the end-to-end bar against HF Llama; with the unscaled table it
    misses that bar on the scaled configuration by more than 10 x."""
    from dataclasses import replace

    from oracle.decode_oracle import OracleQwen2
    case = CASES["llama_scaled"]
    cfg = case["cfg"]
    w = case["weights"](cfg)
    gold = np.load(case["decode"][0])
    tokens, temp = gold["tokens"].tolist(), float(gold["temperature"])
    err = np.abs(OracleQwen2(cfg, w).score(tokens, temp).numpy() - gold["logprobs"])
    plain = OracleQwen2(replace(cfg, rope_scaling=None), w).score(tokens, temp).numpy()
    assert np.abs(plain - gold["logprobs"]).max() > 10 * err.max()


# ---- model description -----------------------------------------------------------------------------------------------
def test_from_hf_config_reads_published_llama_configs():
    from pipelinerl_b200.model import ModelConfig
    c8 = ModelConfig.from_hf_config(LLAMA31_8B_INSTRUCT)
    assert c8 == ModelConfig.llama3_1_8b()
    assert (c8.rms_eps, c8.rope_theta, c8.qkv_bias, c8.qk_norm, c8.family) == (1e-5, 500000.0, False, False, "llama")
    assert ModelConfig.from_hf_config(LLAMA32_3B) == ModelConfig.llama3_2_3b()
    # transformers 5.x writes the RoPE block as rope_parameters, with rope_theta inside
    v5 = {k: v for k, v in LLAMA31_8B_INSTRUCT.items() if k not in ("rope_scaling", "rope_theta")}
    v5["rope_parameters"] = dict(LLAMA31_8B_INSTRUCT["rope_scaling"], rope_theta=500000.0)
    assert ModelConfig.from_hf_config(v5) == c8
    plain = dict(v5, rope_parameters={"rope_type": "default", "rope_theta": 500000.0})
    assert ModelConfig.from_hf_config(plain) == ModelConfig.llama3_1_8b(rope_scaling=None)


def test_llama_shapes_fit_the_kernels():
    from pipelinerl_b200.model import ModelConfig
    for c in (ModelConfig.llama3_1_8b(), ModelConfig.llama3_2_3b()):
        assert c.head_dim == 128 and c.vocab_size % 128 == 0 and c.intermediate_size % 128 == 0
        assert c.q_size == c.hidden_size
    assert abs(ModelConfig.llama3_1_8b().num_params() - 8.03e9) < 0.01e9    # Llama-3.1-8B's published count
    assert abs(ModelConfig.llama3_2_3b().num_params() - (3.21e9 + 128256 * 3072)) < 0.01e9   # + the untied head copy


@pytest.mark.parametrize("change,match", [
    (dict(attention_bias=True), "attention_bias"), (dict(mlp_bias=True), "mlp_bias"),
    (dict(rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 8192}), "yarn"),
    (dict(rope_scaling={"type": "linear", "factor": 2.0}), "linear"),
    (dict(rope_scaling={"rope_type": "dynamic", "factor": 2.0}), "dynamic"),
    (dict(head_dim=64, hidden_size=2048, num_attention_heads=32), "head_dim"),
    (dict(architectures=["Qwen3ForCausalLM"]), "model_type"),
])
def test_from_hf_config_refuses_unsupported_llama_variants(change, match):
    from pipelinerl_b200.model import ModelConfig
    with pytest.raises(ValueError, match=match):
        ModelConfig.from_hf_config(dict(LLAMA31_8B_INSTRUCT, **change))


def test_llama32_1b_head_dim_64_is_refused():
    from pipelinerl_b200.model import ModelConfig
    one_b = dict(LLAMA32_3B, hidden_size=2048, intermediate_size=8192, num_attention_heads=32, num_hidden_layers=16,
                 head_dim=64)
    with pytest.raises(ValueError, match="head_dim"):
        ModelConfig.from_hf_config(one_b)


@pytest.mark.parametrize("which", ["llama3_1_8b", "llama3_2_3b", "scaled", "tied", "unscaled"])
def test_from_hf_config_inverts_hf_config_dict(which):
    from pipelinerl_b200.finetune.checkpoints import hf_config_dict
    from pipelinerl_b200.model import ModelConfig
    cfg = {"llama3_1_8b": ModelConfig.llama3_1_8b(), "llama3_2_3b": ModelConfig.llama3_2_3b(),
           "scaled": llama_tiny_cfg("scaled"), "tied": llama_tiny_cfg("tied"),
           "unscaled": ModelConfig.llama3_1_8b(rope_scaling=None)}[which]
    d = json.loads(json.dumps(hf_config_dict(cfg)))
    assert ModelConfig.from_hf_config(d) == cfg
    assert d["model_type"] == "llama" and d["architectures"] == ["LlamaForCausalLM"]
    assert d["attention_bias"] is False and d["mlp_bias"] is False
    assert d["rope_scaling"] == (cfg.rope_scaling.hf_dict() if cfg.rope_scaling else None)


# digests of hf_config_dict and of the arena layouts of Qwen configs, as the code before Llama support wrote them
_QWEN_CONFIG_JSON = {
    "qwen2_5_7b": "9f81566412dc8571", "qwen3_8b": "0f8da504c5d3da85", "tiny_nobias": "0ffef9bf92388f1b",
}
_QWEN_LAYOUTS = {
    "qwen2_5_7b": (7615616512, 199, "39c78ce3e373fad2"),
    "qwen3_8b": (8190735360, 291, "9144075b86e81b17"), "tiny_nobias": (2032896, 15, "578a3925fd5de407"),
}


def _qwen_cfgs():
    from pipelinerl_b200.model import ModelConfig
    return {"qwen2_5_7b": ModelConfig.qwen2_5_7b(), "qwen3_8b": ModelConfig.qwen3_8b(),
            "tiny_nobias": ModelConfig.tiny(qkv_bias=False)}


@pytest.mark.parametrize("name", sorted(_QWEN_CONFIG_JSON))
def test_qwen_config_json_and_layout_are_unchanged(name):
    from pipelinerl_b200.finetune.checkpoints import hf_config_dict
    from pipelinerl_b200.model import ArenaLayout
    cfg = _qwen_cfgs()[name]
    text = json.dumps(hf_config_dict(cfg), indent=1)
    assert hashlib.sha256(text.encode()).hexdigest()[:16] == _QWEN_CONFIG_JSON[name]
    assert "llama" not in text and "rope_scaling" not in text and "mlp_bias" not in text
    lay = ArenaLayout.build(cfg)
    digest = hashlib.sha256(repr(sorted(lay.offsets.items())).encode()).hexdigest()[:16]
    assert (lay.total, len(lay.offsets), digest) == _QWEN_LAYOUTS[name]


def test_llama_layout_is_qwen2_without_biases():
    from dataclasses import replace

    from pipelinerl_b200.model import ArenaLayout, ModelConfig
    lay = ArenaLayout.build(ModelConfig.llama3_1_8b())
    qwen_like = ArenaLayout.build(replace(ModelConfig.llama3_1_8b(), family="qwen", rope_scaling=None))
    assert lay.offsets == qwen_like.offsets and lay.total == qwen_like.total
    assert not any(n.endswith((".bias", "q_norm.weight", "k_norm.weight")) for n in lay.offsets)


# ---- checkpoints -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_llama_checkpoint_round_trip_and_opens_in_hf(tmp_path, kind):
    conformance.checkpoint_round_trip_opens_in_hf(tmp_path, f"llama_{kind}", n_tokens=200)


def test_tied_checkpoint_loads_untied_into_the_arena():
    from pipelinerl_b200.model import ParamArena
    cfg = llama_tiny_cfg("tied")
    w = llama_tiny_weights(cfg, tied=True)
    sd = hf_model(cfg, w, tied=True).state_dict()
    sd = {k: v for k, v in sd.items() if "rotary" not in k and k != "lm_head.weight"}
    arena = ParamArena(cfg, "cpu")
    arena.load_hf_state_dict(sd)
    assert torch.equal(arena.view("lm_head.weight"), arena.view("embed_tokens.weight"))
    assert torch.equal(arena.view("lm_head.weight").float(), w["lm_head.weight"])


def test_tp_engine_refuses_rope_scaling():
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    with pytest.raises(NotImplementedError, match="RoPE scaling"):
        TPDecodeEngine(llama_tiny_cfg("scaled"), None, 0, 2)

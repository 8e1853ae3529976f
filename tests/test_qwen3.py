"""Qwen3 support without a GPU: the model description, the checkpoint format and the oracles against HF Qwen3 and the
reference (the checks of tests/conformance.py on the Qwen3 cases of tests/model_cases.py)."""
import hashlib

import pytest
import torch

from tests import conformance
from tests.model_cases import qwen3_tiny_cfg

KINDS = ["wide", "gqa4"]


@pytest.mark.parametrize("kind", KINDS)
def test_qwen3_oracle_teacher_forced_vs_hf(kind):
    conformance.decode_oracle_vs_hf(f"qwen3_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_qwen3_oracle_greedy_vs_hf(kind):
    conformance.decode_oracle_greedy_vs_hf(f"qwen3_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_torch_qwen3_module_matches_hf_in_fp32(kind):
    conformance.torch_module_matches_hf(f"qwen3_{kind}")


@pytest.mark.parametrize("kind", KINDS)
def test_learner_oracle_vs_reference_rl_step_on_hf_qwen3(kind):
    conformance.learner_oracle_vs_reference(f"qwen3_{kind}")


# ---- model description ---------------------------------------------------------------------------------------------
# total elements, tensor count and a digest of every offset of the arena as the Qwen2-only code laid it out
_QWEN2_LAYOUTS = {
    "qwen2_5_7b": (7615616512, 199, "39c78ce3e373fad2"),
    "qwen2_5_1_5b_fp32": (2010461696, 200, "a5b3d236ee33f258"),
    "tiny_nobias": (2032896, 15, "578a3925fd5de407"),
    "q25_32b_tp2": (16771552256, 451, "769adb677eba664f"),
}


def _qwen2_cfgs():
    from pipelinerl_b200.model import ModelConfig
    return {"qwen2_5_7b": ModelConfig.qwen2_5_7b(), "qwen2_5_1_5b_fp32": ModelConfig.qwen2_5_1_5b(fp32_head=True),
            "tiny_nobias": ModelConfig.tiny(qkv_bias=False), "q25_32b_tp2": ModelConfig.qwen2_5_32b().shard(2)}


@pytest.mark.parametrize("name", sorted(_QWEN2_LAYOUTS))
def test_qk_norm_off_layout_is_unchanged(name):
    from pipelinerl_b200.model import ArenaLayout
    lay = ArenaLayout.build(_qwen2_cfgs()[name])
    digest = hashlib.sha256(repr(sorted(lay.offsets.items())).encode()).hexdigest()[:16]
    assert (lay.total, len(lay.offsets), digest) == _QWEN2_LAYOUTS[name]
    assert not any("q_norm" in n or "k_norm" in n for n in lay.offsets)


def test_qk_norm_layout_places_gains_after_qkv():
    from pipelinerl_b200.model import ArenaLayout, fused_shapes
    cfg = qwen3_tiny_cfg("wide")
    names = [n for n, _ in fused_shapes(cfg)]
    for l in range(cfg.num_layers):
        i = names.index(f"layers.{l}.qkv_proj.weight")
        assert names[i + 1:i + 3] == [f"layers.{l}.q_norm.weight", f"layers.{l}.k_norm.weight"]
    lay = ArenaLayout.build(cfg)
    assert lay.shapes["layers.0.q_norm.weight"] == (128,) and lay.shapes["layers.1.k_norm.weight"] == (128,)
    assert "layers.0.qkv_proj.bias" not in lay.shapes
    assert lay.shapes["layers.0.o_proj.weight"] == (256, 512)            # [hidden, q width], q width != hidden
    s = lay.hf_slices()
    assert s["model.layers.1.self_attn.q_norm.weight"] == ("layers.1.q_norm.weight", 0, 128)
    assert s["model.layers.1.self_attn.k_norm.weight"] == ("layers.1.k_norm.weight", 0, 128)


def test_qwen3_constructors():
    from pipelinerl_b200.model import ModelConfig
    c8, c14 = ModelConfig.qwen3_8b(), ModelConfig.qwen3_14b()
    assert c8.qk_norm and not c8.qkv_bias and (c8.num_q_heads, c8.num_kv_heads, c8.num_layers) == (32, 8, 36)
    assert c14.qk_norm and not c14.qkv_bias and (c14.num_q_heads, c14.num_kv_heads, c14.num_layers) == (40, 8, 40)
    assert abs(c8.num_params() - 8.19e9) < 0.01e9      # 8.19 B with the untied head (Qwen3-8B's published count)
    assert abs(c14.num_params() - 14.77e9) < 0.01e9


def test_new_gains_initialise_to_one():
    from pipelinerl_b200.learner_model import TorchQwen2
    from pipelinerl_b200.model import ParamArena
    cfg = qwen3_tiny_cfg("wide")
    arena = ParamArena(cfg, "cpu").init_random(seed=3)
    m = TorchQwen2(cfg, "cpu")
    for l in range(cfg.num_layers):
        for which in ("q_norm", "k_norm"):
            assert torch.equal(arena.view(f"layers.{l}.{which}.weight").float(), torch.ones(128))
            assert torch.equal(m.p(f"layers.{l}.{which}.weight").detach(), torch.ones(128))


def test_qk_norm_gains_are_decayed_as_in_the_reference():
    """The reference's no_decay tags are "bias" and "LayerNorm.weight": the q/k gains match neither."""
    from pipelinerl_b200.finetune.optim import NO_DECAY_DEFAULT
    assert not any(t in "layers.0.q_norm.weight" or t in "layers.0.k_norm.weight" for t in NO_DECAY_DEFAULT)


@pytest.mark.parametrize("which", ["tiny_qwen2", "tiny_qwen2_nobias", "qwen2_5_7b", "qwen3_8b", "qwen3_14b",
                                   "qwen3_wide", "qwen3_gqa4", "qwen3_bias"])
def test_from_hf_config_inverts_hf_config_dict(which):
    import json

    from pipelinerl_b200.finetune.checkpoints import hf_config_dict
    from pipelinerl_b200.model import ModelConfig
    cfg = {"tiny_qwen2": ModelConfig.tiny(), "tiny_qwen2_nobias": ModelConfig.tiny(qkv_bias=False),
           "qwen2_5_7b": ModelConfig.qwen2_5_7b(), "qwen3_8b": ModelConfig.qwen3_8b(),
           "qwen3_14b": ModelConfig.qwen3_14b(), "qwen3_wide": qwen3_tiny_cfg("wide"),
           "qwen3_gqa4": qwen3_tiny_cfg("gqa4"),
           "qwen3_bias": ModelConfig.tiny(qkv_bias=True, qk_norm=True)}[which]
    d = json.loads(json.dumps(hf_config_dict(cfg)))
    assert ModelConfig.from_hf_config(d) == cfg
    if cfg.qk_norm:
        assert d["model_type"] == "qwen3" and d["architectures"] == ["Qwen3ForCausalLM"]
        assert ("attention_bias" in d) == cfg.qkv_bias
    else:
        assert d["model_type"] == "qwen2" and d["attention_bias"] == cfg.qkv_bias


def test_qwen2_config_json_is_unchanged():
    from pipelinerl_b200.finetune.checkpoints import hf_config_dict
    from pipelinerl_b200.model import ModelConfig
    d = hf_config_dict(ModelConfig.qwen2_5_7b())
    assert list(d) == ["architectures", "model_type", "vocab_size", "hidden_size", "intermediate_size",
                       "num_hidden_layers", "num_attention_heads", "num_key_value_heads", "head_dim", "hidden_act",
                       "rms_norm_eps", "rope_theta", "tie_word_embeddings", "torch_dtype", "attention_bias",
                       "use_sliding_window"]
    assert d["architectures"] == ["Qwen2ForCausalLM"] and d["attention_bias"] is True


def test_from_hf_config_reads_published_configs_and_rejects_others():
    from pipelinerl_b200.model import ModelConfig
    qwen3_8b = {"architectures": ["Qwen3ForCausalLM"], "attention_bias": False, "attention_dropout": 0.0,
                "bos_token_id": 151643, "eos_token_id": 151645, "head_dim": 128, "hidden_act": "silu",
                "hidden_size": 4096, "initializer_range": 0.02, "intermediate_size": 12288,
                "max_position_embeddings": 40960, "max_window_layers": 36, "model_type": "qwen3",
                "num_attention_heads": 32, "num_hidden_layers": 36, "num_key_value_heads": 8, "rms_norm_eps": 1e-06,
                "rope_scaling": None, "rope_theta": 1000000, "sliding_window": None, "tie_word_embeddings": False,
                "torch_dtype": "bfloat16", "use_cache": True, "use_sliding_window": False, "vocab_size": 151936}
    assert ModelConfig.from_hf_config(qwen3_8b) == ModelConfig.qwen3_8b()
    qwen25_7b = {"model_type": "qwen2", "hidden_size": 3584, "intermediate_size": 18944, "num_hidden_layers": 28,
                 "num_attention_heads": 28, "num_key_value_heads": 4, "rms_norm_eps": 1e-06, "rope_theta": 1000000.0,
                 "vocab_size": 152064}           # no head_dim, no attention_bias: Qwen2 derives the first, always has bias
    assert ModelConfig.from_hf_config(qwen25_7b) == ModelConfig.qwen2_5_7b()
    with pytest.raises(ValueError, match="model_type"):
        ModelConfig.from_hf_config(dict(qwen3_8b, model_type="llama"))
    with pytest.raises(ValueError, match="model_type"):
        ModelConfig.from_hf_config(dict(qwen3_8b, model_type="qwen3_moe"))
    with pytest.raises(ValueError, match="head_dim"):
        ModelConfig.from_hf_config(dict(qwen3_8b, head_dim=64))


# ---- checkpoints ----------------------------------------------------------------------------------------------------
def test_qwen3_checkpoint_round_trip_and_opens_in_hf(tmp_path):
    conformance.checkpoint_round_trip_opens_in_hf(tmp_path, "qwen3_wide", n_tokens=64)


def test_tp_engine_refuses_qk_norm():
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    with pytest.raises(NotImplementedError, match="q/k norm"):
        TPDecodeEngine(qwen3_tiny_cfg("wide"), None, 0, 2)


def test_new_entries_are_declared_and_bound():
    from pathlib import Path

    from pipelinerl_b200 import _lib
    header = (Path(__file__).resolve().parent.parent / "include" / "prl.h").read_text()
    for sym in ("prl_qkv_norm_rope_cache", "prl_qk_norm_rope_fwd", "prl_qk_norm_rope_bwd"):
        assert f"int {sym}(" in header and sym in _lib.declared_symbols()

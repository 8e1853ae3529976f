"""Llama 3 restatement of the token step (torch fp32, CPU), with the rounding points of the CUDA path.

Llama 3 dense = Qwen2 without the qkv bias, with `rope_type: "llama3"` frequency scaling: the kernels read the same
host-tabulated inv_freq[64], so the only change from oracle.decode_oracle's Qwen2 step is the table
(pipelinerl_b200.model.rope_inv_freq).  It is pinned against HF transformers' LlamaForCausalLM in fp32
(tests/golden/llama_tiny_*.npz, tests/golden/make_golden_llama.py).

Also here: the two tiny Llama configurations of the Llama tests and their deterministic weights.
"""
from __future__ import annotations

from oracle.decode_oracle import OracleQwen2


def llama_tiny_cfg(kind: str = "scaled"):
    from pipelinerl_b200.model import Llama3RopeScaling, ModelConfig
    common = dict(num_layers=2, qkv_bias=False, family="llama", rope_theta=500_000.0, rms_eps=1e-5)
    if kind == "scaled":   # 4 q / 2 kv heads; original_max_position_embeddings 64 puts all three bands inside 128 dims
        return ModelConfig(vocab_size=768, hidden_size=256, intermediate_size=768, num_q_heads=4, num_kv_heads=2,
                           rope_scaling=Llama3RopeScaling(8.0, 1.0, 4.0, 64), **common)
    if kind == "tied":     # 3:1 grouping (Llama-3.2-3B), tied word embeddings in the HF model
        return ModelConfig(vocab_size=640, hidden_size=384, intermediate_size=1024, num_q_heads=6, num_kv_heads=2,
                           rope_scaling=Llama3RopeScaling(32.0, 1.0, 4.0, 128), **common)
    raise KeyError(kind)


LLAMA_KINDS = ("scaled", "tied")
TIED = {"scaled": False, "tied": True}


def llama_tiny_weights(cfg, kind: str, seed: int = 42):
    """tests.helpers.tiny_weights; for the tied configuration lm_head is a copy of embed_tokens (the arena stores a
    tied checkpoint untied)."""
    from tests.helpers import tiny_weights
    w = tiny_weights(cfg, seed=seed)
    if TIED[kind]:
        w["lm_head.weight"] = w["embed_tokens.weight"].clone()
    return w


class OracleLlama(OracleQwen2):
    """OracleQwen2 with the RoPE table of the configuration's scaling."""

    def __init__(self, cfg, weights):
        from pipelinerl_b200.model import rope_inv_freq
        super().__init__(cfg, weights)
        self.inv_freq = rope_inv_freq(cfg)


def hf_llama_model(cfg, weights, tied: bool = False):
    """HF LlamaForCausalLM (fp32, eager attention) holding `weights` (fused names)."""
    from transformers import LlamaConfig, LlamaForCausalLM

    from pipelinerl_b200.model import ArenaLayout
    hc = LlamaConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                     num_hidden_layers=cfg.num_layers, num_attention_heads=cfg.num_q_heads,
                     num_key_value_heads=cfg.num_kv_heads, head_dim=cfg.head_dim, rope_theta=cfg.rope_theta,
                     rope_scaling=cfg.rope_scaling.hf_dict() if cfg.rope_scaling is not None else None,
                     rms_norm_eps=cfg.rms_eps, attention_bias=False, mlp_bias=False, tie_word_embeddings=tied,
                     max_position_embeddings=4096, attn_implementation="eager")
    model = LlamaForCausalLM(hc).float()
    sd = {hf: weights[fused][r0:r0 + rn].clone() for hf, (fused, r0, rn) in ArenaLayout.build(cfg).hf_slices().items()}
    if tied:
        assert (sd.pop("lm_head.weight") == sd["model.embed_tokens.weight"]).all()
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m or (tied and m == "lm_head.weight")
                                  for m in missing), (missing, unexpected)
    return model

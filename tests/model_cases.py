"""The tiny model configurations that have HF fixtures, the bounds each one is held to, and the HF model of a case.

One entry per case; the conformance checks (tests/conformance.py) take a case name, and the Qwen3 / Llama fixture
generators (tests/golden/make_golden_qwen3_llama.py, tests/golden/make_golden_learner_qwen3_llama.py) loop over it.
Fields:

  cfg          the ModelConfig
  weights      cfg -> deterministic CPU weights (fused names, bf16-representable values)
  decode       HF teacher-forced fixtures at T = 0.7 (the engine tests replay the first), then any at other temperatures
  learner      stem of the learner fixture (the reference's rl_step on the HF model)
  tied         the HF model ties lm_head to embed_tokens (the arena stores it untied, as a copy)
  oracle       decode oracle vs HF teacher-forced: max / mean |d logprob|
  engine       engine teacher-forced decode path vs the oracle and vs HF: max / mean |d logprob|
  learner_bar  native learner vs the reference's rl_step: loss relative, gradient norm (relative, absolute),
               sampled gradient elements relative L2
"""
from __future__ import annotations

import torch

from tests.helpers import GOLDEN, tiny_cfg, tiny_weights

# the end-to-end bar of a 2-layer bf16 model against fp32 HF: max / mean |d logprob|, and greedy ids equal wherever the
# top-2 logit margin exceeds MARGIN
E2E = (3e-2, 6e-3)
MARGIN = 5e-2


def qwen3_tiny_cfg(kind: str = "wide"):
    from pipelinerl_b200.model import ModelConfig
    common = dict(num_layers=2, qkv_bias=False, qk_norm=True)
    if kind == "wide":   # 4 q / 2 kv heads, q width 512 != hidden 256 (as Qwen3-0.6B / 4B / 32B)
        return ModelConfig(vocab_size=768, hidden_size=256, intermediate_size=768, num_q_heads=4, num_kv_heads=2,
                           **common)
    if kind == "gqa4":   # 4:1 grouping (Qwen3-8B / 14B / 32B), q width 1024 != hidden 384
        return ModelConfig(vocab_size=640, hidden_size=384, intermediate_size=1024, num_q_heads=8, num_kv_heads=2,
                           **common)
    raise KeyError(kind)


def qwen3_tiny_weights(cfg, seed: int = 42, gain_std: float = 0.3):
    """tests.helpers.tiny_weights, with non-unit random q/k gains (1 + gain_std * N(0, 1), bf16-representable) so that
    the gain path is exercised (the generic initialisation there would give them 0.03 * N(0, 1))."""
    w = tiny_weights(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for l in range(cfg.num_layers):
        for which in ("q_norm", "k_norm"):
            t = 1.0 + gain_std * torch.randn(cfg.head_dim, generator=g)
            w[f"layers.{l}.{which}.weight"] = t.to(torch.bfloat16).float()
    return w


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


def llama_tiny_weights(cfg, tied: bool, seed: int = 42):
    """tests.helpers.tiny_weights; with tied embeddings lm_head is a copy of embed_tokens (the arena stores a tied
    checkpoint untied)."""
    w = tiny_weights(cfg, seed=seed)
    if tied:
        w["lm_head.weight"] = w["embed_tokens.weight"].clone()
    return w


def _qwen2(kind, engine):
    return dict(cfg=tiny_cfg(kind), weights=tiny_weights,
                decode=(GOLDEN / f"qwen2_tiny_{kind}_T0.7.npz", GOLDEN / f"qwen2_tiny_{kind}_T1.0.npz"),
                learner=f"learner_step_{kind}", tied=False, oracle=(2.5e-2, 5e-3), engine=engine,
                learner_bar=dict(loss=6e-3, grad_norm=(2.3e-3, 1e-6), grad_samples=2e-2))


def _other(family, kind, cfg, weights, tied=False):
    return dict(cfg=cfg, weights=weights, decode=(GOLDEN / f"{family}_tiny_{kind}.npz",),
                learner=f"learner_step_{family}_{kind}", tied=tied, oracle=E2E, engine=E2E,
                learner_bar=dict(loss=2e-2, grad_norm=(3e-2, 0.0), grad_samples=3e-2))


CASES = {
    # engine bounds = 1.5 x the differences measured on an H100 (tests/test_gpu_decode.py)
    "qwen2_gqa2": _qwen2("gqa2", engine=(1.95e-2, 4.5e-3)),
    "qwen2_gqa7": _qwen2("gqa7", engine=(2.7e-2, 7.1e-3)),
    "qwen3_wide": _other("qwen3", "wide", qwen3_tiny_cfg("wide"), qwen3_tiny_weights),
    "qwen3_gqa4": _other("qwen3", "gqa4", qwen3_tiny_cfg("gqa4"), qwen3_tiny_weights),
    "llama_scaled": _other("llama", "scaled", llama_tiny_cfg("scaled"), lambda cfg: llama_tiny_weights(cfg, False)),
    "llama_tied": _other("llama", "tied", llama_tiny_cfg("tied"), lambda cfg: llama_tiny_weights(cfg, True), tied=True),
}

# the Qwen2 fixtures hold no greedy continuations
GREEDY_CASES = tuple(n for n in CASES if not n.startswith("qwen2"))


def hf_model(cfg, weights, tied: bool = False):
    """HF Qwen2ForCausalLM / Qwen3ForCausalLM / LlamaForCausalLM (fp32, eager attention), whichever `cfg` describes,
    holding `weights` (fused names)."""
    import transformers

    from pipelinerl_b200.model import ArenaLayout
    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_layers, num_attention_heads=cfg.num_q_heads, num_key_value_heads=cfg.num_kv_heads,
              head_dim=cfg.head_dim, rope_theta=cfg.rope_theta, rms_norm_eps=cfg.rms_eps, tie_word_embeddings=tied,
              max_position_embeddings=4096, attn_implementation="eager")
    if cfg.family == "llama":
        arch = "Llama"
        kw.update(rope_scaling=cfg.rope_scaling.hf_dict() if cfg.rope_scaling is not None else None,
                  attention_bias=False, mlp_bias=False)
    elif cfg.qk_norm:
        arch = "Qwen3"
        kw.update(attention_bias=cfg.qkv_bias)
    else:
        arch = "Qwen2"
    hc = getattr(transformers, f"{arch}Config")(**kw)
    model = getattr(transformers, f"{arch}ForCausalLM")(hc).float()
    sd = {hf: weights[fused][r0:r0 + rn].clone() for hf, (fused, r0, rn) in ArenaLayout.build(cfg).hf_slices().items()}
    if tied:
        assert (sd.pop("lm_head.weight") == sd["model.embed_tokens.weight"]).all()
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m or (tied and m == "lm_head.weight")
                                  for m in missing), (missing, unexpected)
    return model

"""The tied-word-embedding model cases: configurations whose arena is tied (`cfg.tie_word_embeddings`: one [V, H] table,
no lm_head), with their HF and reference fixtures (tests/golden/make_golden_learner_tied.py).

Importing this module adds them to tests.model_cases.CASES, so the shared checks of tests/conformance.py run them by
name.  Fields as in tests/model_cases.py; `weights` returns the case's tensors plus `lm_head.weight`, a copy of the
embedding table: the oracles and an untied build of the HF model read the head under that name, and the tied arena,
NativeQwen2 and TorchQwen2 take only the names of `fused_shapes`, which has no lm_head.
"""
from __future__ import annotations

from dataclasses import replace

from tests.helpers import GOLDEN, tiny_cfg, tiny_weights
from tests.model_cases import CASES, E2E, hf_model, llama_tiny_cfg, qwen3_tiny_cfg, qwen3_tiny_weights


def with_head(weights):
    """`weights` (fused names of a tied config: no lm_head) plus lm_head.weight = a copy of embed_tokens.weight"""
    def make(cfg):
        w = weights(cfg)
        w["lm_head.weight"] = w["embed_tokens.weight"].clone()
        return w
    return make


def _tied(family, cfg, weights, decode):
    return dict(cfg=replace(cfg, tie_word_embeddings=True), weights=with_head(weights), decode=(GOLDEN / decode,),
                learner=f"learner_step_tied_{family}", tied=True, oracle=E2E, engine=E2E,
                learner_bar=dict(loss=2e-2, grad_norm=(3e-2, 0.0), grad_samples=3e-2))


# Qwen2 with qkv bias, Qwen3 with q/k norm, and the Llama 3:1 / RoPE-scaled configuration whose HF decode fixture
# (llama_tiny_tied.npz) is tied already.  fused_shapes of a tied config has no lm_head, so the base `weights` draw the
# same tensors as for the untied configuration, minus the head.
TIED_CASES = {
    "tied_qwen2": _tied("qwen2", tiny_cfg("gqa2"), tiny_weights, "qwen2_tiny_tied.npz"),
    "tied_qwen3": _tied("qwen3", qwen3_tiny_cfg("wide"), qwen3_tiny_weights, "qwen3_tiny_tied.npz"),
    "tied_llama": _tied("llama", llama_tiny_cfg("tied"), tiny_weights, "llama_tiny_tied.npz"),
}
CASES.update(TIED_CASES)


def hf_tied_model(cfg, weights):
    """HF model of a tied case with tie_word_embeddings=True (one parameter for both uses), holding `weights`"""
    return hf_model(replace(cfg, tie_word_embeddings=False), weights, tied=True)


def tied_gradients(grads: dict) -> dict:
    """gradients of the oracle's untied leaves -> those of the tied model: the head's is added to the embedding's"""
    out = {k: v for k, v in grads.items() if k != "lm_head.weight"}
    out["embed_tokens.weight"] = grads["embed_tokens.weight"] + grads["lm_head.weight"]
    return out

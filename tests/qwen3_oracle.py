"""Qwen3 restatement of the token step (torch fp32, CPU), with the rounding points of the CUDA path.

Qwen3 dense = Qwen2 + a per-head RMSNorm of q and k before RoPE (gains `q_norm` / `k_norm`, [head_dim], shared by
the heads of a layer), no qkv bias, and a q width n_q * 128 that may differ from hidden_size.  The kernel
(`prl_qkv_norm_rope_cache`, csrc/decode_ops.cu) keeps a head in fp32 from the split-K sum to the end of RoPE:
    y = x * rsqrt(mean(x^2) + eps) * gamma,  then the rotation,  then ONE rounding to bf16
so this oracle does the same; everything else is oracle.decode_oracle's Qwen2 step.  It is pinned against HF
transformers' Qwen3ForCausalLM in fp32 (tests/golden/qwen3_tiny_*.npz, tests/golden/make_golden_qwen3.py).

Also here: the two tiny Qwen3 configurations of the Qwen3 tests and their deterministic weights.
"""
from __future__ import annotations

import math

import torch

from oracle.decode_oracle import OracleQwen2, bf16r, rmsnorm_bf16, rope


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


QWEN3_KINDS = ("wide", "gqa4")


def qwen3_tiny_weights(cfg, seed: int = 42, gain_std: float = 0.3):
    """tests.helpers.tiny_weights, with non-unit random q/k gains (1 + gain_std * N(0, 1), bf16-representable) so that
    the gain path is exercised (the generic initialisation there would give them 0.03 * N(0, 1))."""
    from tests.helpers import tiny_weights
    w = tiny_weights(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for l in range(cfg.num_layers):
        for which in ("q_norm", "k_norm"):
            t = 1.0 + gain_std * torch.randn(cfg.head_dim, generator=g)
            w[f"layers.{l}.{which}.weight"] = t.to(torch.bfloat16).float()
    return w


def head_rmsnorm(x: torch.Tensor, gamma: torch.Tensor, eps: float) -> torch.Tensor:
    """x [T, heads, 128] fp32 -> x * rsqrt(mean(x^2) + eps) * gamma, per head, no rounding"""
    return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps) * gamma.float()


class OracleQwen3(OracleQwen2):
    """OracleQwen2 with Qwen3's q/k norm (weights: fused tensors incl. layers.N.{q,k}_norm.weight)."""

    def forward(self, tokens: torch.Tensor) -> torch.Tensor:
        c, w = self.cfg, self.w
        T = tokens.shape[0]
        past = self.k_cache[0].shape[0]
        pos = torch.arange(past, past + T)
        h = w["embed_tokens.weight"][tokens].clone()
        x = rmsnorm_bf16(h, w["layers.0.input_layernorm.weight"], c.rms_eps)
        R = c.num_q_heads // c.num_kv_heads
        for l in range(c.num_layers):
            p = f"layers.{l}."
            qkv = x @ w[p + "qkv_proj.weight"].t()
            if c.qkv_bias:
                qkv = qkv + w[p + "qkv_proj.bias"]
            q = qkv[:, :c.q_size].view(T, c.num_q_heads, c.head_dim)
            k = qkv[:, c.q_size:c.q_size + c.kv_size].view(T, c.num_kv_heads, c.head_dim)
            v = qkv[:, c.q_size + c.kv_size:].view(T, c.num_kv_heads, c.head_dim)
            q = head_rmsnorm(q, w[p + "q_norm.weight"], c.rms_eps)
            k = head_rmsnorm(k, w[p + "k_norm.weight"], c.rms_eps)
            q = bf16r(rope(q, pos, self.inv_freq))
            k = bf16r(rope(k, pos, self.inv_freq))
            v = bf16r(v)
            self.k_cache[l] = torch.cat([self.k_cache[l], k])
            self.v_cache[l] = torch.cat([self.v_cache[l], v])
            K = self.k_cache[l].repeat_interleave(R, dim=1)
            V = self.v_cache[l].repeat_interleave(R, dim=1)
            s = torch.einsum("thd,shd->hts", q, K) / math.sqrt(c.head_dim)
            S = K.shape[0]
            causal = torch.arange(S)[None, :] > pos[:, None]
            s = s.masked_fill(causal[None], float("-inf"))
            a = torch.softmax(s, dim=-1)
            o = bf16r(torch.einsum("hts,shd->thd", a, V).reshape(T, c.q_size))
            h = h + o @ w[p + "o_proj.weight"].t()
            x = rmsnorm_bf16(h, w[p + "post_attention_layernorm.weight"], c.rms_eps)
            gu = x @ w[p + "gate_up_proj.weight"].t()
            g, u = gu[:, :c.intermediate_size], gu[:, c.intermediate_size:]
            act = bf16r(torch.nn.functional.silu(g) * u)
            h = h + act @ w[p + "down_proj.weight"].t()
            nxt = f"layers.{l + 1}.input_layernorm.weight" if l + 1 < c.num_layers else "norm.weight"
            x = rmsnorm_bf16(h, w[nxt], c.rms_eps)
        return x @ w["lm_head.weight"].t()


def hf_qwen3_model(cfg, weights):
    """HF Qwen3ForCausalLM (fp32, eager attention) holding `weights` (fused names)."""
    from transformers import Qwen3Config, Qwen3ForCausalLM

    from pipelinerl_b200.model import ArenaLayout
    hc = Qwen3Config(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                     num_hidden_layers=cfg.num_layers, num_attention_heads=cfg.num_q_heads,
                     num_key_value_heads=cfg.num_kv_heads, head_dim=cfg.head_dim, rope_theta=cfg.rope_theta,
                     rms_norm_eps=cfg.rms_eps, attention_bias=cfg.qkv_bias, tie_word_embeddings=False,
                     max_position_embeddings=4096, attn_implementation="eager")
    model = Qwen3ForCausalLM(hc).float()
    sd = {hf: weights[fused][r0:r0 + rn].clone() for hf, (fused, r0, rn) in ArenaLayout.build(cfg).hf_slices().items()}
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in m or "inv_freq" in m for m in missing), (missing, unexpected)
    return model

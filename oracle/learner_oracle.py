"""Oracle for hot path (2), model part: forward of the Qwen2 / Qwen3 / Llama 3 transformer over one PACKED row,
differentiable.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Torch fp32 on CPU (or wherever the weights live), autograd for
the backward.

What the reference runs here is `outputs = model(**model_inputs)` at pipelinerl/finetune/rl/__init__.py:190-207 with
`model` = HF transformers' `Qwen2ForCausalLM` (finetune/checkpoints.py:151-222; transformers is a third-party
dependency of the reference, pinned in its pyproject.toml, not vendored) and flash-attn's varlen kernels giving
block-diagonal causal attention for packed `position_ids` (finetune/data.py:215-283).  Restated below from the
published Qwen2 architecture, on the FUSED parameter names of pipelinerl_b200.model.fused_shapes:

    h = embed[ids]
    per layer:  x = RMSNorm(h) ; qkv = x Wqkv^T + b ; q, k = RMSNorm per head (Qwen3 only: cfg.qk_norm) ;
                q, k = RoPE(q, k; position_ids; pipelinerl_b200.model.rope_inv_freq, llama3-scaled for Llama 3) ;
                a = softmax(q k^T / sqrt(d) restricted to same-sample, causal) v   (GQA: q head j uses kv head j // R)
                h = h + a Wo^T ; x = RMSNorm(h) ; h = h + (SiLU(x Wg^T) * (x Wu^T)) Wd^T
    logits = RMSNorm(h) Whead^T

PINNED: tests/conformance.py::learner_oracle_vs_reference (run by tests/test_oracle_golden.py, tests/test_qwen3.py and
tests/test_llama.py) checks this module chained with
oracle/pg_oracle.py against tests/golden/learner_step_*.npz — the reference's own rl_step executed on HF
Qwen2ForCausalLM, Qwen3ForCausalLM and LlamaForCausalLM (fp32, CPU) for all six cases of tests/model_cases.py:
loss, the statistics and the gradient of every parameter (make_golden_learner.py, make_golden_learner_qwen3_llama.py).
"""
from __future__ import annotations

import math

import torch


def rmsnorm(h: torch.Tensor, gamma: torch.Tensor, eps: float) -> torch.Tensor:
    return h * torch.rsqrt((h * h).mean(-1, keepdim=True) + eps) * gamma


def rope(x: torch.Tensor, pos: torch.Tensor, inv_freq: torch.Tensor) -> torch.Tensor:
    """x [T, heads, d]; rotate pairs (i, i + d/2) by pos * inv_freq[i] (HF rotate_half convention)."""
    ang = pos.to(torch.float32)[:, None] * inv_freq[None, :]
    cs, sn = torch.cos(ang)[:, None, :], torch.sin(ang)[:, None, :]
    half = x.shape[-1] // 2
    x1, x2 = x[..., :half], x[..., half:]
    return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], dim=-1)


def packed_logits(cfg, w: dict[str, torch.Tensor], input_ids: torch.Tensor, position_ids: torch.Tensor) -> torch.Tensor:
    """input_ids, position_ids: [T] (positions restart at 0 for every packed sample) -> fp32 logits [T, V].
    `w` maps fused names to fp32 tensors (leaf tensors with requires_grad=True give parameter gradients)."""
    from pipelinerl_b200.model import rope_inv_freq
    T = input_ids.numel()
    d, R = cfg.head_dim, cfg.num_q_heads // cfg.num_kv_heads
    dev = input_ids.device
    inv_freq = rope_inv_freq(cfg).to(dev)
    seg = (position_ids == 0).cumsum(0)
    t = torch.arange(T, device=dev)
    allowed = (seg[:, None] == seg[None, :]) & (t[:, None] >= t[None, :])
    h = w["embed_tokens.weight"][input_ids]
    for l in range(cfg.num_layers):
        p = f"layers.{l}."
        x = rmsnorm(h, w[p + "input_layernorm.weight"], cfg.rms_eps)
        qkv = x @ w[p + "qkv_proj.weight"].t()
        if cfg.qkv_bias:
            qkv = qkv + w[p + "qkv_proj.bias"]
        q = qkv[:, :cfg.q_size].reshape(T, cfg.num_q_heads, d)
        k = qkv[:, cfg.q_size:cfg.q_size + cfg.kv_size].reshape(T, cfg.num_kv_heads, d)
        v = qkv[:, cfg.q_size + cfg.kv_size:].reshape(T, cfg.num_kv_heads, d)
        if cfg.qk_norm:
            q = rmsnorm(q, w[p + "q_norm.weight"], cfg.rms_eps)
            k = rmsnorm(k, w[p + "k_norm.weight"], cfg.rms_eps)
        q, k = rope(q, position_ids, inv_freq), rope(k, position_ids, inv_freq)
        k, v = k.repeat_interleave(R, dim=1), v.repeat_interleave(R, dim=1)
        s = torch.einsum("thd,shd->hts", q, k) / math.sqrt(d)
        s = s.masked_fill(~allowed[None], float("-inf"))
        a = torch.einsum("hts,shd->thd", torch.softmax(s, dim=-1), v).reshape(T, cfg.q_size)
        h = h + a @ w[p + "o_proj.weight"].t()
        x = rmsnorm(h, w[p + "post_attention_layernorm.weight"], cfg.rms_eps)
        gu = x @ w[p + "gate_up_proj.weight"].t()
        I = cfg.intermediate_size
        h = h + (torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]) @ w[p + "down_proj.weight"].t()
    return rmsnorm(h, w["norm.weight"], cfg.rms_eps) @ w["lm_head.weight"].t()


def learner_step(cfg, weights: dict[str, torch.Tensor], cols: dict, rl_cfg, current_step: int, max_step: int):
    """One micro-batch of hot path 2 end to end on the oracle: model forward -> pg_oracle tail -> backward.
    Returns loss (float), stats, new_logprobs, {fused name: gradient}."""
    from . import pg_oracle
    w = {k: v.detach().to(torch.float32).clone().requires_grad_(True) for k, v in weights.items() if not k.endswith("_lo")}
    logits = packed_logits(cfg, w, cols["input_ids"], cols["position_ids"])
    loss, stats, new_lp, _ = pg_oracle.rl_step_oracle(logits, cols, rl_cfg, current_step, max_step)
    loss.backward()
    return float(loss.detach()), stats, new_lp.detach(), {k: v.grad for k, v in w.items()}

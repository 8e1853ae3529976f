"""Learner-side Qwen2 / Qwen3 modules whose parameters live in the fused arena layout (model.py).

`NativeQwen2` (bottom of this file) is the native learner: its body is learner_body.NativeBody — hand-scheduled forward /
backward on the wgmma GEMM and the row kernels of csrc/learner_ops.cu, fp32 gradient accumulation
in the optimizer arena, fused head without logits.  It is what `run_training`, tools/train_bench.py and
tools/pipeline_bench.py use.

`TorchQwen2` is the same architecture as a plain torch module (F.linear / SDPA under autograd, any dtype).  `rl_step`
accepts ANY torch module whose output has `.logits` (the reference contract, rl/__init__.py:190-207), and this one is
the stand-in for "some other HF-style model": the pipeline tests drive it end to end and the learner-body tests use its
fp32 autograd as a second opinion next to oracle/learner_oracle.py.  It is not a fallback: nothing selects it
automatically.

Because parameter order and alignment equal `fused_shapes`, FusedAdamW's bf16 shadow arena has exactly the sampler's
arena layout and can be pushed as raw bytes.
"""
from __future__ import annotations

import math
import os
import types

import torch
import torch.nn.functional as F

from . import _lib
from .model import ArenaLayout, ModelConfig, fused_shapes, is_norm_gain, rope_inv_freq


class TorchQwen2(torch.nn.Module):
    def __init__(self, cfg: ModelConfig, device, dtype=torch.float32, init: dict[str, torch.Tensor] | None = None,
                 seed: int = 42):
        super().__init__()
        self.cfg = cfg
        g = torch.Generator().manual_seed(seed)
        self.names = []
        for name, shape in fused_shapes(cfg):
            if init is not None:
                t = init[name].to(dtype)
            elif is_norm_gain(name):
                t = torch.ones(shape, dtype=dtype)
            elif name.endswith(".bias") or name.endswith("_lo"):
                t = torch.zeros(shape, dtype=dtype)
            else:
                t = (torch.randn(shape, generator=g) * 0.02).to(dtype)
            key = name.replace(".", "__")
            self.register_parameter(key, torch.nn.Parameter(t.to(device)))
            self.names.append(name)
        self.register_buffer("inv_freq", rope_inv_freq(cfg).to(device), persistent=False)
        self.layout = ArenaLayout.build(cfg)

    def p(self, name: str) -> torch.Tensor:
        return getattr(self, name.replace(".", "__"))

    def named_parameters(self, *a, **k):  # fused names, arena order
        for name in self.names:
            yield name, self.p(name)

    def _rope(self, x, pos):
        ang = pos.float()[:, None] * self.inv_freq[None, :]
        cs, sn = torch.cos(ang)[:, None, :].to(x.dtype), torch.sin(ang)[:, None, :].to(x.dtype)
        x1, x2 = x[..., :64], x[..., 64:]
        return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], dim=-1)

    def forward_logprobs(self, batch, temperature: float):
        """rl_step's fast path: (new_logprobs [B, L-1], entropy [B, L-1]) through the fused wgmma head — the
        [L, V] logits are never materialised (finetune/fused_head.py)."""
        from .finetune.fused_head import fused_head_logprobs
        hidden = self.hidden_states(batch.input_ids, batch.position_ids if batch.is_packed else None)
        lps, ents = [], []
        for b in range(hidden.shape[0]):
            lp, ent = fused_head_logprobs(hidden[b, :-1], self.p(self.cfg.head_name), batch.input_ids[b, 1:], temperature)
            lps.append(lp)
            ents.append(ent)
        return torch.stack(lps), torch.stack(ents)

    def forward(self, input_ids, attention_mask=None, labels=None, position_ids=None, **kw):
        """Packed rows [1, T] with position_ids restarting per sample (block-diagonal causal attention), or
        padded [B, L] batches."""
        x = self.hidden_states(input_ids, position_ids)
        return types.SimpleNamespace(logits=F.linear(x.float(), self.p(self.cfg.head_name).float()))

    def hidden_states(self, input_ids, position_ids=None):
        """Final-norm hidden states [B, T, H]."""
        c = self.cfg
        B, T = input_ids.shape
        if position_ids is None:
            position_ids = torch.arange(T, device=input_ids.device)[None].expand(B, T)
        outs = []
        for b in range(B):
            pos = position_ids[b]
            starts = (pos == 0).cumsum(0)
            allowed = (starts[:, None] == starts[None, :]) & (torch.arange(T, device=pos.device)[:, None] >=
                                                             torch.arange(T, device=pos.device)[None, :])
            h = self.p("embed_tokens.weight")[input_ids[b]]
            for l in range(c.num_layers):
                q_ = f"layers.{l}."
                x = self._norm(h, self.p(q_ + "input_layernorm.weight"))
                qkv = F.linear(x, self.p(q_ + "qkv_proj.weight"), self.p(q_ + "qkv_proj.bias") if c.qkv_bias else None)
                q = qkv[:, :c.q_size].view(T, c.num_q_heads, c.head_dim)
                k = qkv[:, c.q_size:c.q_size + c.kv_size].view(T, c.num_kv_heads, c.head_dim)
                v = qkv[:, c.q_size + c.kv_size:].view(T, c.num_kv_heads, c.head_dim)
                if c.qk_norm:   # Qwen3: per-head RMSNorm of q and k before RoPE
                    q, k = self._norm(q, self.p(q_ + "q_norm.weight")), self._norm(k, self.p(q_ + "k_norm.weight"))
                q, k = self._rope(q, pos), self._rope(k, pos)
                R = c.num_q_heads // c.num_kv_heads
                k, v = k.repeat_interleave(R, dim=1), v.repeat_interleave(R, dim=1)
                o = F.scaled_dot_product_attention(q.transpose(0, 1), k.transpose(0, 1), v.transpose(0, 1),
                                                   attn_mask=allowed[None], scale=1.0 / math.sqrt(c.head_dim))
                h = h + F.linear(o.transpose(0, 1).reshape(T, c.q_size), self.p(q_ + "o_proj.weight"))
                x = self._norm(h, self.p(q_ + "post_attention_layernorm.weight"))
                gu = F.linear(x, self.p(q_ + "gate_up_proj.weight"))
                h = h + F.linear(F.silu(gu[:, :c.intermediate_size]) * gu[:, c.intermediate_size:],
                                 self.p(q_ + "down_proj.weight"))
            outs.append(self._norm(h, self.p("norm.weight")))
        return torch.stack(outs)

    def _norm(self, h, g):
        hf = h.float()
        return (hf * torch.rsqrt((hf * hf).mean(-1, keepdim=True) + self.cfg.rms_eps)).to(h.dtype) * g


class _NativeHead(torch.autograd.Function):
    """Final projection + log-softmax statistics of the native learner.  Forward: one wgmma GEMM whose epilogue
    reduces logits on chip (prl_head_logprob).  Backward: per chunk of rows, the same GEMM again with an epilogue that turns
    the logits tile into d logits in registers and stores it as bf16 (prl_head_dlogits), then dX = dZ W and dW += dZ^T X
    (prl_gemm_ex, operands read as stored), the latter accumulated in fp32 in the optimizer's gradient arena."""

    @staticmethod
    def forward(ctx, hidden, model, targets, temperature: float, chunk_rows: int):
        lib = _lib.load()
        x = hidden.to(torch.bfloat16).contiguous()
        W = model.p(model.cfg.head_name).data
        M, K = x.shape
        V = W.shape[0]
        tg = targets.to(torch.int64).contiguous()
        lp = torch.empty(M, dtype=torch.float32, device=x.device)
        ent, lse = torch.empty_like(lp), torch.empty_like(lp)
        ws = torch.empty(int(lib.prl_head_workspace_bytes(M, V)), dtype=torch.uint8, device=x.device)
        W_lo = model.head_lo
        _lib.check(lib.prl_head_logprob(W.data_ptr(), W_lo.data_ptr() if W_lo is not None else None, x.data_ptr(), M, V, K,
                                        float(temperature), tg.data_ptr(), 1, 0,
                                        0, lp.data_ptr(), ent.data_ptr(), lse.data_ptr(), None, None, ws.data_ptr(),
                                        ws.numel(), _lib.stream_ptr()))
        ctx.save_for_backward(x, tg, lse, ent)
        ctx.model, ctx.temperature, ctx.chunk_rows = model, float(temperature), int(chunk_rows)
        return lp, ent

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        x, tg, lse, ent = ctx.saved_tensors
        model, lib = ctx.model, _lib.load()
        body = model.body
        ops = body.ops
        # tied: W is the embedding table and gW its gradient view, into which NativeBody.backward's embedding
        # scatter-add later accumulates the other use (nothing zeroes the gradient arena in between)
        W, gW = model.p(model.cfg.head_name).data, body.g[model.cfg.head_name]
        M, K = x.shape
        V = W.shape[0]
        dev = x.device
        g_lp = g_lp.contiguous() if g_lp is not None else torch.zeros(M, device=dev)
        use_ent = g_ent is not None
        g_ent = g_ent.contiguous() if use_ent else None
        dx = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
        Cn = min(ctx.chunk_rows, M)
        # d logits of a chunk of rows, bf16, straight out of the GEMM that recomputes the logits (prl_head_dlogits): fp32
        # logits / d logits never reach HBM (the reference's autograd keeps 608 KB of fp32 logits per token alive)
        st = _lib.stream_ptr()
        W_lo = model.head_lo
        if os.environ.get("PRL_HEAD_BWD_FUSED", "1") == "0":
            # A/B only: the previous formulation -- logits recomputed (hi GEMM, lo GEMM accumulating), one row kernel, a cast
            logits_buf = torch.empty(Cn, V, dtype=torch.float32, device=dev)
            dlogits_buf = torch.empty(Cn, V, dtype=torch.float32, device=dev)
            for r0 in range(0, M, Cn):
                n = min(Cn, M - r0)
                xs, logits, dlogits = x[r0:r0 + n], logits_buf[:n], dlogits_buf[:n]
                ops.gemm(xs, W, out=logits)
                if W_lo is not None:
                    ops.gemm(xs, W_lo, out=logits, accumulate=True)
                _lib.check(lib.prl_logprob_rows_bwd(logits.data_ptr(), n, V, V, tg[r0:r0 + n].data_ptr(), ctx.temperature,
                                                    lse[r0:r0 + n].data_ptr(), ent[r0:r0 + n].data_ptr(),
                                                    g_lp[r0:r0 + n].data_ptr(),
                                                    g_ent[r0:r0 + n].data_ptr() if use_ent else None,
                                                    dlogits.data_ptr(), V, st))
                dz = dlogits.to(torch.bfloat16)
                ops.gemm(dz, W, out=dx[r0:r0 + n], b_mn=True)
                ops.wgrad(gW, dz, xs)
            return dx, None, None, None, None
        dz_buf = torch.empty(Cn, V, dtype=torch.bfloat16, device=dev)
        for r0 in range(0, M, Cn):
            n = min(Cn, M - r0)
            xs, dz = x[r0:r0 + n], dz_buf[:n]
            _lib.check(lib.prl_head_dlogits(W.data_ptr(), W_lo.data_ptr() if W_lo is not None else None, xs.data_ptr(), n, V, K,
                                            ctx.temperature, tg[r0:r0 + n].data_ptr(), lse[r0:r0 + n].data_ptr(),
                                            ent[r0:r0 + n].data_ptr(), g_lp[r0:r0 + n].data_ptr(),
                                            g_ent[r0:r0 + n].data_ptr() if use_ent else None, dz.data_ptr(), V, st))
            ops.gemm(dz, W, out=dx[r0:r0 + n], b_mn=True)
            ops.wgrad(gW, dz, xs)
        return dx, None, None, None, None


class NativeQwen2(torch.nn.Module):
    """Learner model whose body is learner_body.NativeBody (hand-scheduled wgmma GEMMs + row kernels, fp32
    gradient accumulation in the optimizer arena).  bf16 parameters in the fused arena order; must be bound to a
    FusedAdamW(grad_dtype=torch.float32) with `bind(optimizer)` before the first step."""

    use_fused_head = True

    def __init__(self, cfg: ModelConfig, device, init: dict[str, torch.Tensor] | None = None, seed: int = 42):
        super().__init__()
        self.cfg = cfg
        self.names = []
        g = torch.Generator(device=device).manual_seed(seed)
        for name, shape in fused_shapes(cfg):
            if name.endswith("_lo"):
                continue      # not a parameter: the bf16 residual of the head's fp32 master, kept by the optimizer (lo tail)
            if init is not None:
                t = init[name].to(device=device, dtype=torch.bfloat16)
            elif is_norm_gain(name):
                t = torch.ones(shape, dtype=torch.bfloat16, device=device)
            elif name.endswith(".bias") or name.endswith("_lo"):
                t = torch.zeros(shape, dtype=torch.bfloat16, device=device)
            else:
                t = (torch.randn(shape, generator=g, device=device, dtype=torch.float32) * 0.02).to(torch.bfloat16)
            self.register_parameter(name.replace(".", "__"), torch.nn.Parameter(t))
            self.names.append(name)
        self.layout = ArenaLayout.build(cfg)
        self.body = None
        self.head_lo = None
        self._hook = torch.zeros((), device=device, requires_grad=True)

    def p(self, name: str) -> torch.Tensor:
        return getattr(self, name.replace(".", "__"))

    def named_parameters(self, *a, **k):
        for name in self.names:
            yield name, self.p(name)

    def optimizer_kwargs(self) -> dict:
        """extra arguments FusedAdamW / ShardedFusedAdamW need for this model: with `cfg.fp32_head` the optimizer keeps
        the lm_head's bf16 residual in the arena tail (= the sampler layout's `lm_head.weight_lo`), so that learner and
        samplers both compute the head from the fp32 master's 16 mantissa bits (reference: fp32 lm_head on both sides,
        vllm_quantization.py:266-278, finetune/checkpoints.py:44-105)."""
        return {"lo_tail_for": "lm_head.weight"} if self.cfg.fp32_head else {}

    def bind(self, optimizer) -> None:
        from .learner_body import NativeBody
        if self.cfg.fp32_head and getattr(optimizer, "lo_view", None) is None:
            raise ValueError("cfg.fp32_head: build the optimizer with **model.optimizer_kwargs() (lo_tail_for='lm_head.weight')")
        self.head_lo = optimizer.lo_view if self.cfg.fp32_head else None
        grads = optimizer.grad_views()
        if any(g.dtype != torch.float32 for g in grads.values()):
            raise ValueError("NativeQwen2 accumulates gradients in fp32: build FusedAdamW(grad_dtype=torch.float32) "
                             "or ShardedFusedAdamW(grad_accum_fp32=True)")
        weights = {n: self.p(n).data for n in self.names}
        self.body = NativeBody(self.cfg, weights, grads)

    def after_optimizer_step(self) -> None:
        self.body.refresh()

    def set_sequence_parallel(self, group) -> None:
        """every rank of `group` feeds its slice of the same packed row (rl_step's seq_parallel_group; NativeBody)"""
        if self.body is None:
            raise RuntimeError("NativeQwen2.bind(optimizer) must be called first")
        self.body.set_sequence_parallel(group)

    def hidden_states(self, input_ids, position_ids=None):
        if self.body is None:
            raise RuntimeError("NativeQwen2.bind(optimizer) must be called first")
        from .learner_body import _BodyFn
        B, T = input_ids.shape
        if position_ids is None:
            position_ids = torch.arange(T, device=input_ids.device)[None].expand(B, T)
        return torch.stack([_BodyFn.apply(self._hook, self.body, input_ids[b], position_ids[b]) for b in range(B)])

    def forward_logprobs(self, batch, temperature: float):
        hidden = self.hidden_states(batch.input_ids, batch.position_ids if batch.is_packed else None)
        lps, ents = [], []
        for b in range(hidden.shape[0]):
            lp, ent = _NativeHead.apply(hidden[b, :-1], self, batch.input_ids[b, 1:], temperature, 2048)
            lps.append(lp)
            ents.append(ent)
        return torch.stack(lps), torch.stack(ents)

    def forward(self, input_ids, attention_mask=None, labels=None, position_ids=None, **kw):
        x = self.hidden_states(input_ids, position_ids)
        return types.SimpleNamespace(logits=F.linear(x.float(), self.p(self.cfg.head_name).float()))

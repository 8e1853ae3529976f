"""Native learner body: hand-scheduled forward / backward of the Qwen2 transformer over ONE packed row.

This is the part of hot path 2 that the reference runs as HF eager blocks under autograd with non-reentrant
gradient checkpointing (pipelinerl/finetune/rl/__init__.py:190-207 forward, finetune_loop.py:716-725 backward,
conf/finetune/base.yaml:47-50 checkpointing).  Here there is no autograd inside the body:

  forward   per layer: RMSNorm -> qkv GEMM(+bias) -> [Qwen3: per-head q/k RMSNorm] RoPE -> causal block-diagonal attention -> o GEMM(+residual)
            -> RMSNorm -> gate_up GEMM -> SiLU*up -> down GEMM(+residual); only each layer's INPUT is kept
  backward  per layer (reverse): recompute the MLP half (and the attention half where it was not kept), then dgrad
            GEMMs that read the weights as stored and wgrad GEMMs that read both activations as stored (MN-major
            wgmma operands: no transposed copies) and ACCUMULATE IN FP32 straight into the optimizer's gradient
            arena (no .grad tensors, no autograd accumulation kernels, no per-parameter allocation)

Every GEMM is `prl_gemm_ex` (csrc/gemm_tn.cu, wgmma kernel with 128x256 tiles).  The row-wise pieces (RMSNorm, RoPE, SiLU*up, bias / gain reductions, embedding
scatter) are the kernels of csrc/learner_ops.cu.  Attention (the flash-attn varlen call of the reference) is the
wgmma forward of csrc/attn_tc.cu and the two-kernel deterministic backward of csrc/attn_bwd.cu.
"""
from __future__ import annotations

import math

import torch

from . import _lib
from .model import ModelConfig, rope_inv_freq


def _ru(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class Ops:
    """Thin typed front of the C ABI for the learner body (bf16 activations, fp32 statistics / gradients)."""

    def __init__(self):
        self.lib = _lib.load()

    # C[M,N] (=|+=) A[M,K] B[N,K]^T (+bias) (+residual); a_mn / b_mn: that operand is passed as stored [K, M] / [K, N]
    def gemm(self, A, B, out=None, out_dtype=torch.bfloat16, bias=None, residual=None, accumulate=False, alpha=1.0,
             a_mn=False, b_mn=False):
        (K, M) = A.shape if a_mn else A.shape[::-1]
        (Kb, N) = B.shape if b_mn else B.shape[::-1]
        assert K == Kb and A.stride(1) == 1 and B.stride(1) == 1
        if out is None:
            out = torch.empty(M, N, dtype=out_dtype, device=A.device)
        assert out.shape == (M, N) and out.stride(1) == 1
        _lib.check(self.lib.prl_gemm_ex(A.data_ptr(), A.stride(0), int(a_mn), B.data_ptr(), B.stride(0), int(b_mn), M, N, K,
                                        out.data_ptr(), out.stride(0), int(out.dtype == torch.float32), int(accumulate),
                                        bias.data_ptr() if bias is not None else None,
                                        residual.data_ptr() if residual is not None else None,
                                        residual.stride(0) if residual is not None else 0, float(alpha),
                                        _lib.stream_ptr()))
        return out

    def dgrad(self, dY, W):
        """dX[T, in] = dY[T, out] W[out, in]: the weight is read as stored (MN-major B operand)"""
        return self.gemm(dY, W, b_mn=True)

    def wgrad(self, G, dY, X):
        """G[out, in] (fp32) += dY[T, out]^T X[T, in]: both activations read as stored (MN-major operands, K = tokens)"""
        self.gemm(dY, X, out=G, accumulate=True, a_mn=True, b_mn=True)

    def transpose(self, x, out=None):
        R, Cc = x.shape
        assert x.stride(1) == 1
        if out is None:
            buf = torch.empty(Cc, _ru(R, 8), dtype=torch.bfloat16, device=x.device)  # row stride multiple of 8 (TMA)
            out = buf[:, :R]
        _lib.check(self.lib.prl_transpose_bf16(x.data_ptr(), R, Cc, x.stride(0), out.data_ptr(), out.stride(0),
                                               _lib.stream_ptr()))
        return out

    def rmsnorm(self, x, gamma, eps):
        T, H = x.shape
        y = torch.empty_like(x)
        rstd = torch.empty(T, dtype=torch.float32, device=x.device)
        _lib.check(self.lib.prl_rmsnorm_fwd(x.data_ptr(), gamma.data_ptr(), T, H, float(eps), y.data_ptr(),
                                            rstd.data_ptr(), _lib.stream_ptr()))
        return y, rstd

    def rmsnorm_bwd(self, x, gamma, rstd, dy, dres, dgamma):
        """returns dres + d/dx RMSNorm (bf16); dgamma (fp32 [H]) += column sums"""
        T, H = x.shape
        dx = torch.empty_like(x)
        ws = torch.empty(int(self.lib.prl_rowops_workspace_bytes(H)), dtype=torch.uint8, device=x.device)
        _lib.check(self.lib.prl_rmsnorm_bwd(x.data_ptr(), gamma.data_ptr(), rstd.data_ptr(), dy.data_ptr(),
                                            dres.data_ptr() if dres is not None else None, T, H, dx.data_ptr(),
                                            dgamma.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()))
        return dx

    def rope_(self, qkv, pos, inv_freq, n_heads, head_dim, sign):
        """rotate the first n_heads heads of every row of qkv [T, *] in place by sign * pos * inv_freq"""
        T = qkv.shape[0]
        _lib.check(self.lib.prl_rope_inplace(qkv.data_ptr(), qkv.stride(0), T, n_heads, head_dim, pos.data_ptr(),
                                             inv_freq.data_ptr(), float(sign), _lib.stream_ptr()))

    def qk_norm_rope_(self, qkv, pos, inv_freq, q_gamma, k_gamma, n_q, n_kv, head_dim, eps, keep):
        """Qwen3: per-head RMSNorm (gains q_gamma / k_gamma) then RoPE of the q | k heads of qkv [T, *], in place.
        keep: returns (pre-norm q | k columns [T, (n_q + n_kv) d] bf16, rstd [T, n_q + n_kv] fp32) for the backward."""
        T = qkv.shape[0]
        pre = torch.empty(T, (n_q + n_kv) * head_dim, dtype=torch.bfloat16, device=qkv.device) if keep else None
        rstd = torch.empty(T, n_q + n_kv, dtype=torch.float32, device=qkv.device) if keep else None
        _lib.check(self.lib.prl_qk_norm_rope_fwd(qkv.data_ptr(), qkv.stride(0), T, n_q, n_kv, head_dim, q_gamma.data_ptr(),
                                                 k_gamma.data_ptr(), float(eps), pos.data_ptr(), inv_freq.data_ptr(),
                                                 pre.data_ptr() if keep else None, rstd.data_ptr() if keep else None,
                                                 _lib.stream_ptr()))
        return (pre, rstd) if keep else None

    def qk_norm_rope_bwd_(self, dqkv, pos, inv_freq, q_gamma, k_gamma, saved, n_q, n_kv, head_dim, dq_gamma, dk_gamma):
        """in place on dqkv's q | k columns: inverse RoPE, then the RMSNorm backward; dq_gamma / dk_gamma (fp32) += gain
        gradients (fixed reduction order)"""
        pre, rstd = saved
        T = dqkv.shape[0]
        ws = torch.empty(int(self.lib.prl_rowops_workspace_bytes(256)), dtype=torch.uint8, device=dqkv.device)
        _lib.check(self.lib.prl_qk_norm_rope_bwd(dqkv.data_ptr(), dqkv.stride(0), T, n_q, n_kv, head_dim, q_gamma.data_ptr(),
                                                 k_gamma.data_ptr(), pos.data_ptr(), inv_freq.data_ptr(), pre.data_ptr(),
                                                 rstd.data_ptr(), dq_gamma.data_ptr(), dk_gamma.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), _lib.stream_ptr()))

    def gemm_swiglu(self, x, W, need_gate_up=True):
        """(gate_up [T, 2I] or None, act [T, I]) with SiLU(gate) * up computed in the GEMM epilogue"""
        T, K = x.shape
        I = W.shape[0] // 2
        act = torch.empty(T, I, dtype=torch.bfloat16, device=x.device)
        gu = torch.empty(T, 2 * I, dtype=torch.bfloat16, device=x.device) if need_gate_up else None
        _lib.check(self.lib.prl_gemm_swiglu(x.data_ptr(), x.stride(0), W.data_ptr(), W.stride(0), T, I, K, act.data_ptr(), I,
                                            gu.data_ptr() if gu is not None else None, 2 * I, _lib.stream_ptr()))
        return gu, act

    def dgrad_swiglu(self, dY, W_down, gu):
        """d gate_up [T, 2I] = silu_mul_bwd(gu, dY W_down) with d act kept inside the GEMM (prl_gemm_dgrad_swiglu)"""
        T, H = dY.shape
        I = W_down.shape[1]
        dgu = torch.empty_like(gu)
        _lib.check(self.lib.prl_gemm_dgrad_swiglu(dY.data_ptr(), dY.stride(0), W_down.data_ptr(), W_down.stride(0), T, I, H,
                                                  gu.data_ptr(), dgu.data_ptr(), gu.stride(0), _lib.stream_ptr()))
        return dgu

    def silu_mul(self, gu):
        T, two_i = gu.shape
        act = torch.empty(T, two_i // 2, dtype=torch.bfloat16, device=gu.device)
        _lib.check(self.lib.prl_silu_mul_fwd(gu.data_ptr(), T, two_i // 2, act.data_ptr(), _lib.stream_ptr()))
        return act

    def silu_mul_bwd(self, gu, dact):
        T, two_i = gu.shape
        dgu = torch.empty_like(gu)
        _lib.check(self.lib.prl_silu_mul_bwd(gu.data_ptr(), dact.data_ptr(), T, two_i // 2, dgu.data_ptr(),
                                             _lib.stream_ptr()))
        return dgu

    def colsum_acc(self, x, out_f32):
        """out[C] (fp32) += sum over rows of x [T, C] (bf16), fixed reduction order"""
        T, Cc = x.shape
        ws = torch.empty(int(self.lib.prl_rowops_workspace_bytes(Cc)), dtype=torch.uint8, device=x.device)
        _lib.check(self.lib.prl_colsum_bf16(x.data_ptr(), x.stride(0), T, Cc, out_f32.data_ptr(), ws.data_ptr(),
                                            ws.numel(), _lib.stream_ptr()))

    def attn_fwd(self, qkv, seg_start, seg_len, max_len, n_q, n_kv, head_dim, need_lse=True):
        """block-diagonal causal attention over the packed row qkv [T, (n_q + 2 n_kv) d] (q, k roped)"""
        T = qkv.shape[0]
        assert qkv.dtype == torch.bfloat16 and qkv.stride(1) == 1
        out = torch.empty(T, n_q * head_dim, dtype=torch.bfloat16, device=qkv.device)
        lse = torch.empty(T, n_q, dtype=torch.float32, device=qkv.device) if need_lse else None
        _lib.check(self.lib.prl_attn_varlen_fwd(qkv.data_ptr(), qkv.stride(0), T, seg_start.data_ptr(), seg_len.data_ptr(),
                                                seg_start.numel(), int(max_len), n_q, n_kv, head_dim,
                                                1.0 / math.sqrt(head_dim), out.data_ptr(),
                                                lse.data_ptr() if lse is not None else None, _lib.stream_ptr()))
        return out, lse

    def attn_bwd(self, qkv, out, d_out, lse, seg_start, seg_len, max_len, n_q, n_kv, head_dim):
        """dqkv [T, (n_q + 2 n_kv) d] bf16: gradients of the roped q | k | v"""
        T = qkv.shape[0]
        assert d_out.dtype == torch.bfloat16 and d_out.is_contiguous() and out.is_contiguous()
        dqkv = torch.empty(T, (n_q + 2 * n_kv) * head_dim, dtype=torch.bfloat16, device=qkv.device)
        ws = torch.empty(int(self.lib.prl_attn_varlen_bwd_workspace_bytes(T, n_q)), dtype=torch.uint8, device=qkv.device)
        _lib.check(self.lib.prl_attn_varlen_bwd(qkv.data_ptr(), qkv.stride(0), T, seg_start.data_ptr(), seg_len.data_ptr(),
                                                seg_start.numel(), int(max_len), n_q, n_kv, head_dim,
                                                1.0 / math.sqrt(head_dim), out.data_ptr(), d_out.data_ptr(),
                                                lse.data_ptr(), dqkv.data_ptr(), dqkv.stride(0), ws.data_ptr(),
                                                ws.numel(), _lib.stream_ptr()))
        return dqkv

    def attn_fwd_kv(self, q, kv, segs, n_q, n_kv, head_dim, need_lse=True):
        """sequence-parallel slice: local queries q [Tq, >= n_q d] against the gathered kv [Tkv, 2 n_kv d];
        segs = (q_start, q_len, pos0, kv_start) int32 device tensors + max_q_len, max_kv_len (sp_segments)"""
        q_start, q_len, pos0, kv_start, max_q, _ = segs
        Tq = q.shape[0]
        assert q.dtype == torch.bfloat16 and kv.dtype == torch.bfloat16 and q.stride(1) == 1 and kv.stride(1) == 1
        out = torch.empty(Tq, n_q * head_dim, dtype=torch.bfloat16, device=q.device)
        lse = torch.empty(Tq, n_q, dtype=torch.float32, device=q.device) if need_lse else None
        _lib.check(self.lib.prl_attn_varlen_fwd_kv(q.data_ptr(), q.stride(0), Tq, kv.data_ptr(), kv.stride(0), kv.shape[0],
                                                   q_start.data_ptr(), q_len.data_ptr(), pos0.data_ptr(), kv_start.data_ptr(),
                                                   q_start.numel(), int(max_q), n_q, n_kv, head_dim,
                                                   1.0 / math.sqrt(head_dim), out.data_ptr(),
                                                   lse.data_ptr() if lse is not None else None, _lib.stream_ptr()))
        return out, lse

    def attn_bwd_kv(self, q, kv, out, d_out, lse, segs, n_q, n_kv, head_dim, dq):
        """writes dq (a [Tq, n_q d] view, e.g. the query columns of the local dqkv) and returns this rank's contribution
        dkv [Tkv, 2 n_kv d] to every key row"""
        q_start, q_len, pos0, kv_start, max_q, max_kv = segs
        Tq = q.shape[0]
        assert d_out.dtype == torch.bfloat16 and d_out.is_contiguous() and out.is_contiguous() and dq.stride(1) == 1
        dkv = torch.empty(kv.shape[0], 2 * n_kv * head_dim, dtype=torch.bfloat16, device=q.device)
        ws = torch.empty(int(self.lib.prl_attn_varlen_bwd_workspace_bytes(Tq, n_q)), dtype=torch.uint8, device=q.device)
        _lib.check(self.lib.prl_attn_varlen_bwd_kv(q.data_ptr(), q.stride(0), Tq, kv.data_ptr(), kv.stride(0), kv.shape[0],
                                                   q_start.data_ptr(), q_len.data_ptr(), pos0.data_ptr(), kv_start.data_ptr(),
                                                   q_start.numel(), int(max_q), int(max_kv), n_q, n_kv, head_dim,
                                                   1.0 / math.sqrt(head_dim), out.data_ptr(), d_out.data_ptr(), lse.data_ptr(),
                                                   dq.data_ptr(), dq.stride(0), dkv.data_ptr(), dkv.stride(0), ws.data_ptr(),
                                                   ws.numel(), _lib.stream_ptr()))
        return dkv

    def embed(self, table, ids):
        T, H = ids.numel(), table.shape[1]
        out = torch.empty(T, H, dtype=torch.bfloat16, device=table.device)
        _lib.check(self.lib.prl_embed_gather(table.data_ptr(), ids.data_ptr(), T, H, out.data_ptr(), _lib.stream_ptr()))
        return out

    def embed_bwd(self, dtable_f32, ids, dh):
        T, H = dh.shape
        _lib.check(self.lib.prl_embed_scatter_add(dtable_f32.data_ptr(), ids.data_ptr(), dh.data_ptr(), T, H,
                                                  _lib.stream_ptr()))


class NativeBody:
    """weights: fused name -> bf16 tensor (views of the parameter arena); grads: fused name -> fp32 tensor
    (views of the optimizer's gradient arena)."""

    def __init__(self, cfg: ModelConfig, weights: dict[str, torch.Tensor], grads: dict[str, torch.Tensor]):
        self.cfg, self.w, self.g = cfg, weights, grads
        self.ops = Ops()
        dev = next(iter(weights.values())).device
        self.inv_freq = rope_inv_freq(cfg).to(dev)
        self._saved = None
        self._seg_cache = None
        self.keep_attention_layers = cfg.num_layers   # lower it when activation memory is short (0 = full recompute)
        self.keep_gate_up_layers = 0                  # layers that also keep gate_up's output (2 I bf16 per token):
        #                                               their backward skips the largest recompute GEMM
        import os
        # SiLU * up backward inside the down_proj dgrad epilogue (prl_gemm_dgrad_swiglu, bit-identical): measured SLOWER on the 7B
        # step (1 926 / 1 942 ms vs 1 898 / 1 904 ms, same box, alternating runs): the epilogue's strided gate / up reads and its
        # 2 x 256 exp / rcp per thread outlast the short K = 3584 main loop, so the tile pipeline waits for it.  Off by default.
        self.fuse_silu_bwd = os.environ.get("PRL_FUSE_SILU_BWD", "0") == "1"
        self.sp_group = None                          # sequence parallelism: see set_sequence_parallel
        self._sp_segs = None

    def set_sequence_parallel(self, group) -> None:
        """Sequence parallelism (reference: `seq_parallel` ranks share one packed row, finetune_loop.py:507-517, through
        ring attention).  Here every rank runs the token-local work (norms, GEMMs, MLP, head) on its slice and attention
        is the only exchange: K / V of a GQA model are 2 n_kv / (n_q + 2 n_kv) of the qkv row (1/4.5 for Qwen2.5-7B), so
        each layer ALL-GATHERS the K | V columns over the group (NCCL, 32 MB per layer at 16 K tokens), runs its local
        queries against the gathered keys (prl_attn_varlen_fwd_kv), and in the backward REDUCE-SCATTERS the ranks'
        dK / dV contributions.  `group` = None switches it off."""
        import torch.distributed as dist
        self.sp_group = group if (group is not None and dist.get_world_size(group) > 1) else None

    def refresh(self) -> None:
        """Hook called after every optimizer step.  Nothing to rebuild: dgrad reads the weights as stored."""

    # ---- attention: q, k roped; block-diagonal causal over the packed segments (csrc/attn_tc.cu, attn_bwd.cu) ----
    def _segments(self, bounds, dev):
        key = tuple(bounds)
        if self._seg_cache is None or self._seg_cache[0] != key or self._seg_cache[1].device != dev:
            st = torch.tensor([s for s, _ in bounds], dtype=torch.int32, device=dev)
            ln = torch.tensor([e - s for s, e in bounds], dtype=torch.int32, device=dev)
            self._seg_cache = (key, st, ln, max(e - s for s, e in bounds))
        return self._seg_cache[1:]

    def _attention(self, qkv, bounds, need_grad):
        """returns (attention output [T, q_size] bf16, statistics for the backward or None)"""
        c = self.cfg
        if self.sp_group is not None:
            import torch.distributed as dist
            qe = c.num_q_heads * c.head_dim
            kv_local = qkv[:, qe:].contiguous()
            kv = torch.empty(kv_local.shape[0] * dist.get_world_size(self.sp_group), kv_local.shape[1],
                             dtype=kv_local.dtype, device=kv_local.device)
            dist.all_gather_into_tensor(kv, kv_local, group=self.sp_group)
            out, lse = self.ops.attn_fwd_kv(qkv, kv, self._sp_segs, c.num_q_heads, c.num_kv_heads, c.head_dim,
                                            need_lse=need_grad)
            return out, ((lse, kv) if need_grad else None)
        st, ln, mx = self._segments(bounds, qkv.device)
        return self.ops.attn_fwd(qkv, st, ln, mx, c.num_q_heads, c.num_kv_heads, c.head_dim, need_lse=need_grad)

    def _attention_bwd(self, qkv, attn, lse, bounds, d_attn):
        c = self.cfg
        if self.sp_group is not None:
            import torch.distributed as dist
            lse, kv = lse
            qe = c.num_q_heads * c.head_dim
            dqkv = torch.empty_like(qkv)
            dkv_all = self.ops.attn_bwd_kv(qkv, kv, attn, d_attn, lse, self._sp_segs, c.num_q_heads, c.num_kv_heads,
                                           c.head_dim, dqkv[:, :qe])
            dkv = torch.empty(qkv.shape[0], dkv_all.shape[1], dtype=dkv_all.dtype, device=dkv_all.device)
            dist.reduce_scatter_tensor(dkv, dkv_all, op=dist.ReduceOp.SUM, group=self.sp_group)
            dqkv[:, qe:] = dkv
            return dqkv
        st, ln, mx = self._segments(bounds, qkv.device)
        return self.ops.attn_bwd(qkv, attn, d_attn, lse, st, ln, mx, c.num_q_heads, c.num_kv_heads, c.head_dim)

    # ---- one layer, in two halves ----
    def _attn_half(self, l, h, pos, bounds, need_grad):
        c, o, w = self.cfg, self.ops, self.w
        p = f"layers.{l}."
        x1, rstd1 = o.rmsnorm(h, w[p + "input_layernorm.weight"], c.rms_eps)
        qkv = o.gemm(x1, w[p + "qkv_proj.weight"], bias=w.get(p + "qkv_proj.bias"))
        qk_saved = None
        if c.qk_norm:   # Qwen3: per-head q / k RMSNorm fused with RoPE; keeps the pre-norm q | k columns for the backward
            qk_saved = o.qk_norm_rope_(qkv, pos, self.inv_freq, w[p + "q_norm.weight"], w[p + "k_norm.weight"],
                                       c.num_q_heads, c.num_kv_heads, c.head_dim, c.rms_eps, keep=need_grad)
        else:
            o.rope_(qkv, pos, self.inv_freq, c.num_q_heads + c.num_kv_heads, c.head_dim, +1.0)
        attn, lse = self._attention(qkv, bounds, need_grad=need_grad)
        h2 = o.gemm(attn, w[p + "o_proj.weight"], residual=h)
        return x1, rstd1, attn, (qkv, lse, qk_saved) if need_grad else None, h2

    def _mlp_half(self, l, h2, need_out=True, need_gate_up=True):
        c, o, w = self.cfg, self.ops, self.w
        p = f"layers.{l}."
        x2, rstd2 = o.rmsnorm(h2, w[p + "post_attention_layernorm.weight"], c.rms_eps)
        if c.intermediate_size % 128 == 0:      # SiLU * up in the gate_up GEMM's epilogue: no activation round trip
            gu, act = o.gemm_swiglu(x2, w[p + "gate_up_proj.weight"], need_gate_up=need_gate_up)
        else:
            gu = o.gemm(x2, w[p + "gate_up_proj.weight"])
            act = o.silu_mul(gu)
        h3 = o.gemm(act, w[p + "down_proj.weight"], residual=h2) if need_out else None  # the backward only needs act
        return x2, rstd2, gu, act, h3

    def _layer_bwd(self, l, h, saved, pos, bounds, dh3):
        c, o, w, g = self.cfg, self.ops, self.w, self.g
        p = f"layers.{l}."
        gu = None
        if saved is None:   # full recompute of the layer from its input
            x1, rstd1, attn, graph, h2 = self._attn_half(l, h, pos, bounds, need_grad=True)
        else:               # attention half was kept by the forward: only the (cheap) norm is redone
            attn, graph, h2, gu = saved
            x1, rstd1 = o.rmsnorm(h, w[p + "input_layernorm.weight"], c.rms_eps)
        if gu is None:
            x2, rstd2, gu, act, _ = self._mlp_half(l, h2, need_out=False)
        else:               # gate_up output kept too: norm and SiLU*up are one pass each, no GEMM
            x2, rstd2 = o.rmsnorm(h2, w[p + "post_attention_layernorm.weight"], c.rms_eps)
            act = o.silu_mul(gu)
        T = h.shape[0]
        o.wgrad(g[p + "down_proj.weight"], dh3, act)
        del act
        if c.intermediate_size % 32 == 0 and self.fuse_silu_bwd:     # SiLU * up backward in the dgrad GEMM's epilogue: d act never reaches HBM
            d_gu = o.dgrad_swiglu(dh3, w[p + "down_proj.weight"], gu)
        else:
            d_gu = o.silu_mul_bwd(gu, o.dgrad(dh3, w[p + "down_proj.weight"]))
        del gu
        dx2 = o.dgrad(d_gu, w[p + "gate_up_proj.weight"])
        o.wgrad(g[p + "gate_up_proj.weight"], d_gu, x2)
        del d_gu, x2
        dh2 = o.rmsnorm_bwd(h2, w[p + "post_attention_layernorm.weight"], rstd2, dx2, dh3,
                            g[p + "post_attention_layernorm.weight"])
        del dx2, h2
        d_attn = o.dgrad(dh2, w[p + "o_proj.weight"])
        o.wgrad(g[p + "o_proj.weight"], dh2, attn)
        dqkv = self._attention_bwd(graph[0], attn, graph[1], bounds, d_attn)
        qk_saved = graph[2]
        del graph, attn, d_attn
        if c.qk_norm:
            o.qk_norm_rope_bwd_(dqkv, pos, self.inv_freq, w[p + "q_norm.weight"], w[p + "k_norm.weight"], qk_saved,
                                c.num_q_heads, c.num_kv_heads, c.head_dim, g[p + "q_norm.weight"], g[p + "k_norm.weight"])
            del qk_saved
        else:
            o.rope_(dqkv, pos, self.inv_freq, c.num_q_heads + c.num_kv_heads, c.head_dim, -1.0)
        if c.qkv_bias:
            o.colsum_acc(dqkv, g[p + "qkv_proj.bias"])
        dx1 = o.dgrad(dqkv, w[p + "qkv_proj.weight"])
        o.wgrad(g[p + "qkv_proj.weight"], dqkv, x1)
        del dqkv, x1
        return o.rmsnorm_bwd(h, w[p + "input_layernorm.weight"], rstd1, dx1, dh2, g[p + "input_layernorm.weight"])

    # ---- whole body ----
    @staticmethod
    def sp_segments(position_ids: torch.Tensor, offset: int, device):
        """Segment description of a sequence-parallel slice: `position_ids` are those of the LOCAL tokens (a contiguous
        slice, starting at global row `offset`, of a packed row whose position ids restart at 0 for every sample -- the
        reference's make_slices, finetune/types.py:145-180).  A local segment starts at every local 0 and at local row 0;
        its first query sits at position position_ids[start], and its sequence's first key is global row
        offset + start - position_ids[start]."""
        pos = position_ids.to("cpu", torch.int64)
        T = pos.numel()
        starts = torch.nonzero(pos == 0).flatten().tolist()
        if not starts or starts[0] != 0:
            starts = [0] + starts
        ends = starts[1:] + [T]
        q_start = torch.tensor(starts, dtype=torch.int32)
        q_len = torch.tensor([e - s for s, e in zip(starts, ends)], dtype=torch.int32)
        pos0 = pos[starts].to(torch.int32)
        kv_start = (q_start + int(offset) - pos0).to(torch.int32)
        max_q = int(q_len.max())
        max_kv = int((pos0 + q_len).max())
        return (q_start.to(device), q_len.to(device), pos0.to(device), kv_start.to(device), max_q, max_kv)

    @staticmethod
    def segment_bounds(position_ids: torch.Tensor) -> list[tuple[int, int]]:
        starts = torch.nonzero(position_ids == 0).flatten().tolist()
        T = position_ids.numel()
        if not starts or starts[0] != 0:
            starts = [0] + starts
        return [(s, e) for s, e in zip(starts, starts[1:] + [T])]

    def forward(self, input_ids: torch.Tensor, position_ids: torch.Tensor, keep: bool = True) -> torch.Tensor:
        """input_ids / position_ids: [T] (position ids restart at 0 for every packed sample).  Returns the final-norm
        hidden states [T, H] (bf16).  With keep, each layer's input is saved for the backward; the first
        `keep_attention_layers` layers also keep their attention half (attention output + its softmax statistics +
        post-attention residual, ~0.4 GB per layer at 16 K tokens of Qwen2.5-7B) so the backward does not redo the
        qkv GEMM, RoPE, attention forward and o_proj."""
        c, o = self.cfg, self.ops
        ids = input_ids.to(torch.int64).contiguous()
        pos = position_ids.to(torch.int32).contiguous()
        bounds = self.segment_bounds(position_ids)
        if self.sp_group is not None:
            import torch.distributed as dist
            # this rank holds rows [rank * T, (rank + 1) * T) of the packed row (make_slices, finetune/types.py:145-180)
            self._sp_segs = self.sp_segments(position_ids, dist.get_rank(self.sp_group) * position_ids.numel(), ids.device)
        h = o.embed(self.w["embed_tokens.weight"], ids)
        inputs, kept = [], []
        for l in range(c.num_layers):
            keep_attn = keep and l < self.keep_attention_layers
            _, _, attn, graph, h2 = self._attn_half(l, h, pos, bounds, need_grad=keep_attn)
            _, _, gu, _, h3 = self._mlp_half(l, h2, need_gate_up=keep and l < self.keep_gate_up_layers)
            if keep:
                inputs.append(h)
                kept.append((attn, graph, h2, gu if l < self.keep_gate_up_layers else None) if keep_attn else None)
            h = h3
            del gu
        y, rstd = o.rmsnorm(h, self.w["norm.weight"], c.rms_eps)
        if keep:
            self._saved = (ids, pos, bounds, inputs, kept, h, rstd)
        return y

    def backward(self, d_hidden: torch.Tensor) -> None:
        """d_hidden: dL/d(final-norm hidden) [T, H].  Accumulates every parameter gradient of the body."""
        assert self._saved is not None, "backward() without a kept forward()"
        c, o, g = self.cfg, self.ops, self.g
        ids, pos, bounds, inputs, kept, h_last, rstd = self._saved
        self._saved = None
        dh = o.rmsnorm_bwd(h_last, self.w["norm.weight"], rstd, d_hidden.to(torch.bfloat16).contiguous(), None,
                           g["norm.weight"])
        del h_last
        for l in range(c.num_layers - 1, -1, -1):
            dh = self._layer_bwd(l, inputs.pop(), kept.pop(), pos, bounds, dh)
        o.embed_bwd(g["embed_tokens.weight"], ids, dh)


class _BodyFn(torch.autograd.Function):
    """Autograd adapter: makes `hidden = body(ids)` a node whose backward runs NativeBody.backward (parameter
    gradients go straight into the arena, so the node has no tensor inputs that need grad besides the hook)."""

    @staticmethod
    def forward(ctx, hook, body, input_ids, position_ids):
        ctx.body = body
        return body.forward(input_ids, position_ids, keep=True)

    @staticmethod
    def backward(ctx, d_hidden):
        ctx.body.backward(d_hidden)
        return torch.zeros((), device=d_hidden.device), None, None, None

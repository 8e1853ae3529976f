"""Trainer-side output head without logits materialisation.

`fused_head_logprobs(hidden, weight, targets, temperature)` returns, per token, the log-probability of its
target and the exact entropy of softmax(logits / T) — what rl_step derives from full-vocabulary fp32 logits at
pipelinerl/finetune/rl/__init__.py:207-233 (608 KB/token for Qwen2.5; 10 GB for a 16 K-token micro-batch, plus a
/T copy and a detached copy).  Forward: ONE wgmma GEMM whose epilogue reduces each 128-row vocabulary tile on
chip to (max, sum exp, sum exp*z, target logit) — `prl_head_logprob`, csrc/gemm_tc.cu.  Backward: logits are
recomputed chunk by chunk (wgmma GEMM into a bounded scratch), turned into d logits in place
(csrc/logprob_tail.cu) and contracted with two library GEMMs (torch.mm -> cuBLAS: plain GEMMs), so peak extra
memory is one chunk, never T x V.

The fp32 master weight is split into a bf16 value and a bf16 residual (W = hi + lo): both streams feed the same
fp32 accumulator, which reproduces the reference's fp32 lm_head (finetune/checkpoints.py:44-105) to ~2^-17.
"""
from __future__ import annotations

import torch

from .. import _lib


def split_hi_lo(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor | None]:
    if w.dtype == torch.bfloat16:
        return w.contiguous(), None
    hi = w.to(torch.bfloat16)
    lo = (w.float() - hi.float()).to(torch.bfloat16)
    return hi.contiguous(), lo.contiguous()


class _FusedHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, weight, targets, temperature: float, chunk_rows: int):
        if not hidden.is_cuda:
            raise RuntimeError("fused_head_logprobs needs CUDA tensors: pipelinerl_b200 has no CPU fallback")
        lib = _lib.load()
        x = hidden.to(torch.bfloat16).contiguous()
        hi, lo = split_hi_lo(weight.detach())
        M, K = x.shape
        V = hi.shape[0]
        tg = targets.to(torch.int64).contiguous()
        dev = x.device
        lp = torch.empty(M, dtype=torch.float32, device=dev)
        ent = torch.empty_like(lp)
        lse = torch.empty_like(lp)
        ws = torch.empty(int(lib.prl_head_workspace_bytes(M, V)), dtype=torch.uint8, device=dev)
        _lib.check(lib.prl_head_logprob(hi.data_ptr(), lo.data_ptr() if lo is not None else None, x.data_ptr(), M, V, K,
                                        float(temperature), tg.data_ptr(), 1, 0, 0, lp.data_ptr(), ent.data_ptr(),
                                        lse.data_ptr(), None, None, ws.data_ptr(), ws.numel(), _lib.stream_ptr()))
        ctx.save_for_backward(x, weight, tg, lse, ent)
        ctx.temperature, ctx.chunk_rows = float(temperature), int(chunk_rows)
        ctx.hidden_dtype = hidden.dtype
        return lp, ent

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        x, weight, tg, lse, ent = ctx.saved_tensors
        lib = _lib.load()
        hi, lo = split_hi_lo(weight.detach())
        M, K = x.shape
        V = hi.shape[0]
        dev = x.device
        g_lp = g_lp.contiguous() if g_lp is not None else torch.zeros(M, device=dev)
        use_ent = g_ent is not None
        g_ent = g_ent.contiguous() if use_ent else None
        dx = torch.empty(M, K, dtype=torch.float32, device=dev)
        dw = torch.zeros(V, K, dtype=torch.float32, device=dev) if weight.requires_grad else None
        C = min(ctx.chunk_rows, M)
        logits_buf = torch.empty(C, V, dtype=torch.float32, device=dev)
        dlogits_buf = torch.empty(C, V, dtype=torch.float32, device=dev)
        st = _lib.stream_ptr()
        for r0 in range(0, M, C):
            n = min(C, M - r0)
            xs = x[r0:r0 + n]
            logits, dlogits = logits_buf[:n], dlogits_buf[:n]
            # recompute this chunk's logits with the same wgmma kernel and operands as the forward
            _lib.check(lib.prl_gemm_bf16_splitk(hi.data_ptr(), lo.data_ptr() if lo is not None else None, xs.data_ptr(),
                                                n, V, K, 1, logits.data_ptr(), st))
            _lib.check(lib.prl_logprob_rows_bwd(logits.data_ptr(), n, V, V, tg[r0:r0 + n].data_ptr(), ctx.temperature,
                                                lse[r0:r0 + n].data_ptr(), ent[r0:r0 + n].data_ptr(),
                                                g_lp[r0:r0 + n].data_ptr(),
                                                g_ent[r0:r0 + n].data_ptr() if use_ent else None,
                                                dlogits.data_ptr(), V, st))
            dz = dlogits.to(torch.bfloat16)
            d = torch.mm(dz, hi).float()
            if lo is not None:
                d += torch.mm(dz, lo).float()
            dx[r0:r0 + n] = d
            if dw is not None:
                if n * V * K <= (1 << 30):
                    dw.addmm_(dlogits.t(), xs.float())           # small problems: full fp32
                else:
                    dw.add_(torch.mm(dz.t(), xs).float())        # library bf16 GEMM, fp32 accumulation across chunks
        return dx.to(ctx.hidden_dtype), (dw.to(weight.dtype) if dw is not None else None), None, None, None


def fused_head_logprobs(hidden: torch.Tensor, weight: torch.Tensor, targets: torch.Tensor, temperature: float = 1.0,
                        chunk_rows: int = 2048) -> tuple[torch.Tensor, torch.Tensor]:
    """hidden [T, H], weight [V, H] (bf16 or fp32 master), targets [T] -> (logprob of target [T], entropy [T])."""
    return _FusedHead.apply(hidden, weight, targets, temperature, chunk_rows)

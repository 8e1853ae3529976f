#!/usr/bin/env python
"""Learner attention forward / backward (csrc/attn_tc.cu, csrc/attn_bwd.cu) on Qwen2.5-7B's head geometry, timed
with CUDA events next to the library kernel it replaced (torch SDPA -> cuDNN flash) on the same inputs.

    python tools/attn_bench.py [--tokens 16384] [--segments 1] [--reps 10]

One JSON line: ms and model TFLOP/s (causal: 4 d L^2 / 2 per head forward, x2.5 backward) for both."""
import argparse
import json
import math
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from pipelinerl_b200.learner_body import Ops  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--segments", type=int, default=1)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--n-q", type=int, default=28)
    ap.add_argument("--n-kv", type=int, default=4)
    ap.add_argument("--no-library", action="store_true")
    ap.add_argument("--ours-only", action="store_true", help="one forward + one backward of our kernels, nothing else (ncu)")
    ap.add_argument("--profile", action="store_true", help="per-kernel device time (torch profiler)")
    ap.add_argument("--fwd-gen", type=int, default=0, help="forward generation (0 = library default)")
    ap.add_argument("--bwd-gen", type=int, default=0, help="backward generation (0 = library default)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    o = Ops()
    D, T, n_q, n_kv = 128, a.tokens, a.n_q, a.n_kv
    L = T // a.segments
    lens = [L] * a.segments
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(T, (n_q + 2 * n_kv) * D, generator=g, device=dev).to(torch.bfloat16)
    d_out = torch.randn(T, n_q * D, generator=g, device=dev).to(torch.bfloat16)
    st = torch.arange(0, T, L, dtype=torch.int32, device=dev)
    ln = torch.tensor(lens, dtype=torch.int32, device=dev)
    if a.fwd_gen:
        o.lib.prl_attn_set_fwd_generation(a.fwd_gen)
    if a.bwd_gen:
        o.lib.prl_attn_set_bwd_generation(a.bwd_gen)
    if a.ours_only:
        for _ in range(2):
            out, lse = o.attn_fwd(qkv, st, ln, L, n_q, n_kv, D)
            o.attn_bwd(qkv, out, d_out, lse, st, ln, L, n_q, n_kv, D)
        torch.cuda.synchronize()
        return
    out, lse = o.attn_fwd(qkv, st, ln, L, n_q, n_kv, D)
    fwd_ms = timed(lambda: o.attn_fwd(qkv, st, ln, L, n_q, n_kv, D), a.reps)
    o.attn_bwd(qkv, out, d_out, lse, st, ln, L, n_q, n_kv, D)
    bwd_ms = timed(lambda: o.attn_bwd(qkv, out, d_out, lse, st, ln, L, n_q, n_kv, D), a.reps)
    flops_fwd = a.segments * n_q * 4 * D * L * L / 2
    res = {"bench": "learner_attention", "tokens": T, "segments": a.segments, "n_q": n_q, "n_kv": n_kv,
           "fwd_gen": a.fwd_gen or "default", "bwd_gen": a.bwd_gen or "default",
           "ours": {"fwd_ms": round(fwd_ms, 3), "bwd_ms": round(bwd_ms, 3),
                    "fwd_TFLOPs": round(flops_fwd / fwd_ms / 1e9, 1), "bwd_TFLOPs": round(2.5 * flops_fwd / bwd_ms / 1e9, 1)}}
    if not a.no_library:
        import torch.nn.functional as F
        q = qkv[:, :n_q * D].view(a.segments, L, n_q, D).transpose(1, 2).detach().requires_grad_(True)
        k = qkv[:, n_q * D:(n_q + n_kv) * D].view(a.segments, L, n_kv, D).transpose(1, 2).detach().requires_grad_(True)
        v = qkv[:, (n_q + n_kv) * D:].view(a.segments, L, n_kv, D).transpose(1, 2).detach().requires_grad_(True)
        do = d_out.view(a.segments, L, n_q, D).transpose(1, 2)

        def lib_fwd():
            return F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True, scale=1.0 / math.sqrt(D))
        y = lib_fwd()
        lf = timed(lambda: lib_fwd(), a.reps)
        lb = timed(lambda: torch.autograd.grad(y, (q, k, v), do, retain_graph=True), a.reps)
        res["library_sdpa"] = {"fwd_ms": round(lf, 3), "bwd_ms": round(lb, 3), "fwd_TFLOPs": round(flops_fwd / lf / 1e9, 1),
                               "bwd_TFLOPs": round(2.5 * flops_fwd / lb / 1e9, 1)}
        err = (y.transpose(1, 2).reshape(T, n_q * D).float() - out.float()).abs().max().item()
        res["max_abs_diff_vs_library_out"] = err
    if a.profile:
        from torch.profiler import ProfilerActivity, profile as tprofile
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                o.attn_fwd(qkv, st, ln, L, n_q, n_kv, D)
                o.attn_bwd(qkv, out, d_out, lse, st, ln, L, n_q, n_kv, D)
            torch.cuda.synchronize()
        import re
        res["kernels_us"] = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                mname = re.search(r"(\w+_kernel)(<[^>]*>)?", e.key)
                res["kernels_us"][(mname.group(0) if mname else e.key[:40])] = round(e.device_time_total / e.count, 1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

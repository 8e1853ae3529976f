#!/usr/bin/env python
"""Per-kernel timings at Qwen2.5-7B decode shapes (B=64) with an L2 flush between iterations.
Used to choose tile / split-K / occupancy settings; it prints its summaries."""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from pipelinerl_b200 import _lib  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
flush = torch.zeros(512 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tot = 0.0
    for _ in range(iters):
        flush.add_(1)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters * 1e3  # us


def main():
    B, H, I, V = 64, 3584, 18944, 152064
    shapes = {"qkv": (4608, H), "o": (H, H), "gate_up": (2 * I, H), "down": (H, I), "head": (V, H)}
    out = []
    st = None
    for name, (N, K) in shapes.items():
        W = (torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16)
        X = torch.randn(B, K, device=dev).to(torch.bfloat16)
        auto = lib.prl_gemm_auto_split_k(B, N, K)
        for budget, tiled in ((72, 0), (100, 0), (100, 1), (200, 1)):
            lib.prl_gemm_set_smem_budget_kb(budget)
            lib.prl_gemm_set_tiled_weights(tiled)   # timing experiment: tiled addressing of the same buffer
            for split in sorted(set([auto, auto * 2])):
                if split > (K + 63) // 64 // 2 or (name in ("gate_up", "head") and split > 2):
                    continue
                part = torch.empty(split, B, N, device=dev)
                us = timeit(lambda: _lib.check(lib.prl_gemm_bf16_splitk(W.data_ptr(), None, X.data_ptr(), B, N, K, split,
                                                                        part.data_ptr(), st)))
                gbs = N * K * 2 / us / 1e3
                out.append({"kernel": "gemm", "name": name, "N": N, "K": K, "smem_kb": budget, "tiled": tiled, "split_k": split,
                            "auto": auto, "us": round(us, 2), "weight_GBs": round(gbs, 1)})
                print(json.dumps(out[-1]), flush=True)
        del W
    lib.prl_gemm_set_smem_budget_kb(72)   # the library default
    lib.prl_gemm_set_tiled_weights(0)
    # epilogue kernels
    h = torch.randn(B, H, device=dev)
    x = torch.empty(B, H, dtype=torch.bfloat16, device=dev)
    gamma = torch.ones(H, dtype=torch.bfloat16, device=dev)
    for split in (1, 4, 5, 8):
        part = torch.randn(split, B, H, device=dev)
        us = timeit(lambda: _lib.check(lib.prl_residual_rmsnorm(part.data_ptr(), split, B, H, gamma.data_ptr(), 1e-6,
                                                                h.data_ptr(), x.data_ptr(), None, 0, st)))
        print(json.dumps({"kernel": "residual_rmsnorm", "split": split, "us": round(us, 2)}), flush=True)
    part = torch.randn(1, B, 2 * I, device=dev)
    act = torch.empty(B, I, dtype=torch.bfloat16, device=dev)
    us = timeit(lambda: _lib.check(lib.prl_silu_mul(part.data_ptr(), 1, B, I, act.data_ptr(), None, 0, st)))
    print(json.dumps({"kernel": "silu_mul", "us": round(us, 2)}), flush=True)
    logits = torch.randn(B, V, device=dev)
    ids = torch.zeros(B, dtype=torch.int32, device=dev)
    lps = torch.zeros(B, device=dev)
    ws = torch.zeros(int(lib.prl_sample_workspace_bytes(B)), dtype=torch.uint8, device=dev)
    us = timeit(lambda: _lib.check(lib.prl_sample_logprob(logits.data_ptr(), B, V, 1.0, 0, 1, 1, ids.data_ptr(), lps.data_ptr(),
                                                          ws.data_ptr(), ws.numel(), st)))
    print(json.dumps({"kernel": "sample_logprob", "us": round(us, 2)}), flush=True)


if __name__ == "__main__":
    main()

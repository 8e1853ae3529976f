#!/usr/bin/env python
"""In-graph cost of each kernel class of the Qwen2.5-7B token step (B=64, ctx 8192): time the CUDA-graph step
with classes of kernels removed (results are then meaningless, timings are not), with/without the cross-kernel
L2 prefetch.  One JSON line per variant."""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bench  # noqa: E402


def main():
    args = bench.parse()
    dev = torch.device("cuda:0")
    cfg, eng = bench.build_engine(args, dev)
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    # (name, skipped kernel classes, L2 prefetch bytes, fused head, PDL, fused attention combine, gemm smem KB)
    # gemm smem 72 KB is the library default (three GEMM CTAs per SM); 100 KB = two, 48 KB = 2-stage rings
    variants = [("base", set(), 0, True, 1, 0, 72), ("base_again", set(), 0, True, 1, 0, 72),
                ("fused_combine", set(), 0, True, 1, 1, 72), ("no_pdl", set(), 0, True, 0, 0, 72),
                ("unfused_head", set(), 0, False, 1, 0, 72), ("gemm_smem_200", set(), 0, True, 1, 0, 200),
                ("gemm_smem_100", set(), 0, True, 1, 0, 100), ("gemm_smem_48", set(), 0, True, 1, 0, 48),
                ("l2_prefetch_40MB", set(), 40 << 20, True, 1, 0, 72),
                ("no_attention", {"attn"}, 0, True, 1, 0, 72), ("gemm_only", {"attn", "small"}, 0, True, 1, 0, 72),
                ("attention_only", {"gemm", "small"}, 0, True, 1, 0, 72), ("small_only", {"gemm", "attn"}, 0, True, 1, 0, 72),
                ("base_end", set(), 0, True, 1, 0, 72)]
    for name, skip, pf, fused, pdl, fcomb, smem in variants:
        eng._skip, eng.l2_prefetch_bytes, eng.fused_head = skip, pf, fused
        lib.prl_set_pdl(pdl)
        lib.prl_attn_set_fused_combine(fcomb)
        lib.prl_gemm_set_smem_budget_kb(smem)
        eng._graphs.clear()
        # same state for every variant: all slots active at the bench context
        eng.positions.fill_(args.context); eng.seq_lens.fill_(args.context + 1); eng.gen_count.zero_()
        eng.active.fill_(1); eng.finished.zero_()
        for _ in range(3):
            eng.step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(30):
            eng.step()
        e1.record()
        torch.cuda.synchronize()
        print(json.dumps({"variant": name, "ms_per_step": round(e0.elapsed_time(e1) / 30, 4)}), flush=True)


if __name__ == "__main__":
    main()

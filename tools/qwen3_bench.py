"""What Qwen3's per-head q/k RMSNorm costs on the hot paths, measured with CUDA events on one GPU.

1. Token step at Qwen3-8B shapes (36 layers, 32 q / 8 kv heads, random weights), B = 64 sequences at a context of 4096
   tokens.  (The 8192-token context bench.py uses for Qwen2.5-7B does not fit: Qwen3-8B's KV cache is 144 KiB per token,
   75.5 GB for 64 x 8192, next to a 16.4 GB arena on an 80 GB card.)  The model part of the step is captured twice as a
   CUDA graph on the same engine, the same weights and the same KV cache: once with the q/k-norm epilogue
   (prl_qkv_norm_rope_cache) and once with the plain RoPE epilogue (prl_qkv_rope_cache, qk_norm=False), so the difference
   is the epilogue's cost alone.  The two graphs are replayed in alternating passes; the spread between passes is the noise.
   The qkv epilogue launch alone (one layer, both variants) is timed as well.
2. One native-learner layer at Qwen3-8B widths, forward + backward over a packed row of 16 384 tokens (16 samples of
   1024), attention half kept by the forward, with and without the q/k norm (same weights); and the learner's two q/k-norm
   kernels alone next to the plain RoPE kernel.

Prints one JSON line with the card name and power limit.
    python tools/qwen3_bench.py [--steps 50] [--passes 3] [--out qwen3_bench.json]"""
from __future__ import annotations

import argparse
import json
import sys
from dataclasses import replace
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.sample_bench import card  # noqa: E402


def _time(fn, iters: int) -> float:
    """ms per call, CUDA events around `iters` calls"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def token_step(a, dev) -> dict:
    from pipelinerl_b200 import _lib
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ModelConfig, ParamArena
    cfg = ModelConfig.qwen3_8b()
    arena = ParamArena(cfg, dev).init_random(seed=42)
    for name in arena.names():          # non-unit gains (init_random sets them to 1)
        if name.endswith(("q_norm.weight", "k_norm.weight")):
            arena.view(name).uniform_(0.5, 1.5)
    S = a.context
    eng = DecodeEngine(cfg, arena, max_batch=a.batch, max_seq_len=S + 64, max_new_tokens=64, device=dev,
                       use_cuda_graph=True)
    g = torch.Generator(device=dev).manual_seed(1234)
    flat, step = eng.kv_cache, 1 << 28
    for s in range(0, flat.numel(), step):
        n = min(step, flat.numel() - s)
        flat[s:s + n] = (torch.randn(n, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    B, mb = eng.B, eng.max_blocks
    eng.block_table.copy_(torch.arange(1, 1 + B * mb, dtype=torch.int32, device=dev).view(B, mb))
    eng.positions.fill_(S - 1)
    eng.seq_lens.fill_(S)
    eng.active.fill_(1)
    eng.tokens.copy_(torch.randint(0, 151643, (B,), generator=torch.Generator().manual_seed(1000)).int())
    graphs = {}
    for norm in (True, False):
        eng.cfg = replace(cfg, qk_norm=norm)           # same arena, same KV cache: only the qkv epilogue differs
        eng._step_kernels()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            eng._step_kernels()
        graphs[norm] = gr
    eng.cfg = cfg
    for gr in graphs.values():
        for _ in range(a.warmup):
            gr.replay()
    torch.cuda.synchronize()
    res = {"model": "qwen3_8b", "B": B, "context": S, "steps_per_pass": a.steps, "qk_norm_ms": [], "rope_only_ms": []}
    for _ in range(a.passes):
        res["qk_norm_ms"].append(round(_time(graphs[True].replay, a.steps), 4))
        res["rope_only_ms"].append(round(_time(graphs[False].replay, a.steps), 4))
    # the epilogue launch alone (layer 0; the partials hold whatever the last GEMM left there)
    lib, st = eng.lib, _lib.stream_ptr()
    p = "layers.0."
    args_tail = (cfg.num_q_heads, cfg.num_kv_heads, cfg.head_dim, eng.positions.data_ptr(), eng.block_table.data_ptr(),
                 eng.max_blocks, None, eng.inv_freq.data_ptr(), eng.q.data_ptr(), eng.kv_cache.data_ptr(), eng.n_pages, 0,
                 64, None, 0, st)
    sk = eng.split_k["qkv"]

    def epi_norm():
        _lib.check(lib.prl_qkv_norm_rope_cache(eng.partials.data_ptr(), sk, B, None, arena.ptr(p + "q_norm.weight"),
                                               arena.ptr(p + "k_norm.weight"), cfg.rms_eps, *args_tail))

    def epi_rope():
        _lib.check(lib.prl_qkv_rope_cache(eng.partials.data_ptr(), sk, B, None, *args_tail))
    for fn in (epi_norm, epi_rope):
        _time(fn, 50)
    res["epilogue_us"] = {"qk_norm": round(_time(epi_norm, 2000) * 1e3, 2), "rope_only": round(_time(epi_rope, 2000) * 1e3, 2),
                          "launches_per_step": cfg.num_layers, "qkv_split_k": sk}
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    res["step_delta_ms_median"] = round(med(res["qk_norm_ms"]) - med(res["rope_only_ms"]), 4)
    res["step_delta_pct_median"] = round(100 * res["step_delta_ms_median"] / med(res["rope_only_ms"]), 3)
    del graphs, eng, arena
    torch.cuda.empty_cache()
    return res


def learner_layer(a, dev) -> dict:
    from pipelinerl_b200.learner_body import NativeBody
    from pipelinerl_b200.model import ModelConfig, fused_shapes, is_norm_gain
    cfg = ModelConfig.qwen3_8b(num_layers=1)
    g = torch.Generator(device=dev).manual_seed(7)
    w, gr = {}, {}
    for name, shape in fused_shapes(cfg):
        if not name.startswith("layers.0."):
            continue
        t = (1 + 0.3 * torch.randn(shape, generator=g, device=dev)) if is_norm_gain(name) else \
            torch.randn(shape, generator=g, device=dev) * 0.02
        w[name] = t.to(torch.bfloat16)
        gr[name] = torch.zeros(shape, dtype=torch.float32, device=dev)
    T, n_samples = a.tokens, 16
    body = NativeBody(cfg, w, gr)
    pos = torch.arange(T // n_samples, dtype=torch.int32, device=dev).repeat(n_samples)
    bounds = NativeBody.segment_bounds(pos)
    h = (torch.randn(T, cfg.hidden_size, generator=g, device=dev)).to(torch.bfloat16)
    dh3 = (torch.randn(T, cfg.hidden_size, generator=g, device=dev) * 1e-3).to(torch.bfloat16)

    def fwd_bwd():
        _, _, attn, graph, h2 = body._attn_half(0, h, pos, bounds, need_grad=True)
        body._mlp_half(0, h2, need_gate_up=False)
        body._layer_bwd(0, h, (attn, graph, h2, None), pos, bounds, dh3)

    res = {"model": "qwen3_8b (one layer)", "tokens": T, "samples": n_samples, "qk_norm_ms": [], "rope_only_ms": []}
    for norm in (True, False):
        body.cfg = replace(cfg, qk_norm=norm)
        for _ in range(3):
            fwd_bwd()
    for _ in range(a.passes):
        for norm, key in ((True, "qk_norm_ms"), (False, "rope_only_ms")):
            body.cfg = replace(cfg, qk_norm=norm)
            res[key].append(round(_time(fwd_bwd, a.layer_iters), 3))
    body.cfg = cfg
    # the row kernels alone on the qkv tensor of this row
    o, inv, nq, nkv = body.ops, body.inv_freq, cfg.num_q_heads, cfg.num_kv_heads
    qkv = torch.randn(T, cfg.qkv_size, generator=g, device=dev).to(torch.bfloat16)
    saved = o.qk_norm_rope_(qkv.clone(), pos, inv, w["layers.0.q_norm.weight"], w["layers.0.k_norm.weight"], nq, nkv, 128,
                            cfg.rms_eps, keep=True)
    kern = {
        "qk_norm_rope_fwd": lambda: o.qk_norm_rope_(qkv, pos, inv, w["layers.0.q_norm.weight"], w["layers.0.k_norm.weight"],
                                                    nq, nkv, 128, cfg.rms_eps, keep=True),
        "qk_norm_rope_bwd": lambda: o.qk_norm_rope_bwd_(qkv, pos, inv, w["layers.0.q_norm.weight"],
                                                        w["layers.0.k_norm.weight"], saved, nq, nkv, 128,
                                                        gr["layers.0.q_norm.weight"], gr["layers.0.k_norm.weight"]),
        "rope_inplace": lambda: o.rope_(qkv, pos, inv, nq + nkv, 128, +1.0),
    }
    res["kernels_us"] = {}
    for name, fn in kern.items():
        _time(fn, 5)
        res["kernels_us"][name] = round(_time(fn, 100) * 1e3, 1)
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    res["layer_delta_ms_median"] = round(med(res["qk_norm_ms"]) - med(res["rope_only_ms"]), 3)
    res["layer_delta_pct_median"] = round(100 * res["layer_delta_ms_median"] / med(res["rope_only_ms"]), 3)
    res["kept_pre_norm_qk_MB"] = round(T * (nq + nkv) * 128 * 2 / 1e6, 1)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--context", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--layer-iters", type=int, default=10)
    ap.add_argument("--skip", default="", help="comma list of parts to skip: step, learner")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qwen3_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    skip = set(filter(None, a.skip.split(",")))
    res = {**card()}
    if "step" not in skip:
        res["token_step"] = token_step(a, dev)
    if "learner" not in skip:
        res["learner_layer"] = learner_layer(a, dev)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()

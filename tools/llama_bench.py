"""Llama 3 on the hot paths, measured with CUDA events on one GPU.

1. Token step at Llama-3.1-8B shapes (32 layers, 32 q / 8 kv heads, vocabulary 128 256, llama3 RoPE, random weights,
   fp32-equivalent head), B = 64 sequences at a context of 4096 tokens.  (64 x 8192 does not fit: the KV cache is
   128 KiB per token, 68.7 GB next to a 16 GB arena on an 80 GB card.)  The whole step is timed: the captured model
   graph, the sampler and the state advance.  Reported: ms per step, tokens per second, and the bytes the step must move
   through HBM (weights once, the KV cache read, the new K/V rows, the fp32 logits written and read) over its time.
2. The same step with every slot carrying a 3-id stop row against the stop fields left NULL, in alternating passes on
   the same engine, weights and KV cache; the spread between passes of one variant is the noise.  The stop ids are ones
   the sampler practically never draws; slots a pass retires anyway are counted and the state is reset between passes.
3. One native-learner layer at Llama-3.1-8B widths, forward + backward over a packed row of 16 384 tokens (16 samples
   of 1024), attention half kept by the forward.

Prints one JSON line with the card name and power limit.
    python tools/llama_bench.py [--steps 50] [--passes 4] [--out llama_bench.json]"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.qwen3_bench import _time  # noqa: E402
from tools.sample_bench import card  # noqa: E402


def step_bytes(eng, context: int) -> int:
    """HBM bytes one token step has to move: every weight once, the KV cache of every slot, the new K/V rows, and the
    fp32 logits written by the head and read by the sampler"""
    cfg, B = eng.cfg, eng.B
    kv_row = cfg.num_layers * 2 * cfg.num_kv_heads * cfg.head_dim * 2
    return eng.arena.nbytes() + B * context * kv_row + B * kv_row + 2 * B * cfg.head_rows * 4


def token_step(a, dev) -> dict:
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ModelConfig, ParamArena
    cfg = ModelConfig.llama3_1_8b(fp32_head=True)
    arena = ParamArena(cfg, dev).init_random(seed=42)
    S = a.context
    room = a.steps * (a.passes + 1) + a.warmup + 8
    eng = DecodeEngine(cfg, arena, max_batch=a.batch, max_seq_len=S + room, max_new_tokens=room, device=dev,
                       use_cuda_graph=True, eos_id=-1)
    g = torch.Generator(device=dev).manual_seed(1234)
    flat, step = eng.kv_cache, 1 << 28
    for s in range(0, flat.numel(), step):
        n = min(step, flat.numel() - s)
        flat[s:s + n] = (torch.randn(n, generator=g, device=dev) * 0.5).to(torch.bfloat16)
    B, mb = eng.B, eng.max_blocks
    eng.block_table.copy_(torch.arange(1, 1 + B * mb, dtype=torch.int32, device=dev).view(B, mb))
    first = torch.randint(0, cfg.vocab_size, (B,), generator=torch.Generator().manual_seed(1000)).int()
    stop = [cfg.vocab_size - 3, cfg.vocab_size - 2, cfg.vocab_size - 1]
    eng.stop_rows[:, :3] = torch.tensor(stop, dtype=torch.int32, device=dev)

    def reset():
        eng.positions.fill_(S - 1)
        eng.seq_lens.fill_(S)
        eng.active.fill_(1)
        eng.prompt_len.zero_()
        eng.gen_count.zero_()
        eng.max_new_t.fill_(room)
        eng.finished.zero_()
        eng.tokens.copy_(first)
        torch.cuda.synchronize()

    def set_stops(on: bool):
        eng.n_stop.fill_(3 if on else 0)
        eng._stop_slots = set(range(B)) if on else set()
    reset()
    for on in (False, True):
        set_stops(on)
        for _ in range(a.warmup):
            eng.step()
    res = {"model": "llama3_1_8b (fp32_head)", "B": B, "context": S, "steps_per_pass": a.steps,
           "null_stop_ms": [], "stop_rows_ms": [], "retired_slots": {"null_stop": 0, "stop_rows": 0}}
    for _ in range(a.passes):
        for on, key in ((False, "null_stop"), (True, "stop_rows")):
            reset()
            set_stops(on)
            res[key + "_ms"].append(round(_time(eng.step, a.steps), 4))
            res["retired_slots"][key] += int((eng.active == 0).sum())
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    base = med(res["null_stop_ms"])
    res["tokens_per_s"] = round(B * 1e3 / base, 1)
    res["step_bytes_GB"] = round(step_bytes(eng, S) / 1e9, 3)
    res["hbm_GBps"] = round(step_bytes(eng, S) / 1e9 / (base * 1e-3), 1)
    res["stop_delta_ms_median"] = round(med(res["stop_rows_ms"]) - base, 4)
    res["noise_ms"] = {k: round(max(res[k]) - min(res[k]), 4) for k in ("null_stop_ms", "stop_rows_ms")}
    del eng, arena
    torch.cuda.empty_cache()
    return res


def learner_layer(a, dev) -> dict:
    from pipelinerl_b200.learner_body import NativeBody
    from pipelinerl_b200.model import ModelConfig, fused_shapes, is_norm_gain
    cfg = ModelConfig.llama3_1_8b(num_layers=1)
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
    for _ in range(3):
        fwd_bwd()
    ms = [round(_time(fwd_bwd, a.layer_iters), 3) for _ in range(a.passes)]
    H, I = cfg.hidden_size, cfg.intermediate_size
    gemm_flop = 2 * T * H * (cfg.qkv_size + cfg.q_size + 3 * I) * 3             # forward + two backward GEMMs each
    L = T // n_samples
    attn_flop = 4 * n_samples * (L * L / 2) * cfg.head_dim * cfg.num_q_heads * 3.5   # causal fwd (1) + bwd (2.5)
    med = sorted(ms)[len(ms) // 2]
    return {"model": "llama3_1_8b (one layer)", "tokens": T, "samples": n_samples, "fwd_bwd_ms": ms,
            "TFLOPs": round((gemm_flop + attn_flop) / (med * 1e-3) / 1e12, 1)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--context", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--layer-iters", type=int, default=10)
    ap.add_argument("--skip", default="", help="comma list of parts to skip: step, learner")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("llama_bench needs a CUDA device")
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

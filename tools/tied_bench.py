"""What training tied word embeddings tied saves, measured with CUDA events on one GPU, tied and untied alternating in one
process.

1. Trainer step at Qwen2.5-1.5B shapes (random weights), 2 packed micro-batches of 16 384 tokens (tools/train_bench.py's
   workload and batch): rl_step -> backward -> FusedAdamW, with the word embeddings tied (one [V, H] table, bf16 head)
   against untied with `fp32_head` (the head a separate tensor with its bf16 residual).  Seconds per optimizer step,
   the optimizer's share, and the peak memory of each variant (model, optimizer arenas and activations; every pass
   starts from an empty cache).
2. Token step at Qwen2.5-1.5B and Qwen3-1.7B shapes, B = 64 sequences at a context of 8192 tokens: the model part of the
   step (head GEMM included) captured as a CUDA graph on one engine and one KV cache, once on a tied arena (the head
   GEMM reads the bf16 embedding table) and once on an untied fp32_head arena (it reads hi + lo), replayed in alternating
   passes.  Head bytes per step are computed from the shapes.

Prints one JSON line with the card name and power limit.
    python tools/tied_bench.py [--steps 3] [--passes 2] [--decode-steps 50] [--out tied_bench.json]"""
from __future__ import annotations

import argparse
import gc
import json
import sys
from dataclasses import replace
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.qwen3_bench import _time  # noqa: E402
from tools.sample_bench import card  # noqa: E402
from tools.train_bench import synthetic_batch  # noqa: E402


def _variants(cfg):
    return {"tied": replace(cfg, tie_word_embeddings=True, fp32_head=False),
            "untied_fp32_head": replace(cfg, tie_word_embeddings=False, fp32_head=True)}


def trainer_step(a, dev) -> dict:
    from pipelinerl_b200.finetune.optim import FusedAdamW
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from pipelinerl_b200.learner_model import NativeQwen2
    from pipelinerl_b200.model import ModelConfig
    variants = _variants(ModelConfig.qwen2_5_1_5b())
    res = {"model": "qwen2_5_1_5b", "tokens_per_micro_batch": a.tokens, "micro_batches": a.micro,
           "timed_steps_per_pass": a.steps}
    for key in variants:
        res[key] = {"s_per_step": [], "optimizer_ms": [], "peak_GB": [], "optimizer_state_GB": None}
    rcfg = RLConfig(batch_size=a.micro)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    for _ in range(a.passes):
        for key, cfg in variants.items():
            gc.collect()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            model = NativeQwen2(cfg, dev)
            opt = FusedAdamW(model.named_parameters(), lr=1e-6, weight_decay=0.01, max_grad_norm=0.3,
                             grad_dtype=torch.float32, **model.optimizer_kwargs())
            model.bind(opt)
            state = sum(t.numel() * t.element_size() for t in (opt.master, opt.exp_avg, opt.exp_avg_sq, opt.grad,
                                                               opt.shadow_bf16))
            res[key]["optimizer_state_GB"] = round(state / 1e9, 3)
            batches = [synthetic_batch(cfg, a.tokens, 1, dev, 100 + i) for i in range(a.micro)]
            steps, opt_ms = [], []
            for step in range(a.warmup + a.steps):
                e0, e1, e2 = ev(), ev(), ev()
                opt.zero_grad()
                e0.record()
                for b in batches:
                    loss, _ = rl_step(model, b, step, 1000, rcfg)
                    loss.backward()
                e1.record()
                opt.step()
                model.after_optimizer_step()
                e2.record()
                torch.cuda.synchronize()
                if step >= a.warmup:
                    steps.append(e0.elapsed_time(e2) / 1e3)
                    opt_ms.append(e1.elapsed_time(e2))
            res[key]["s_per_step"].append(round(sum(steps) / len(steps), 4))
            res[key]["optimizer_ms"].append(round(sum(opt_ms) / len(opt_ms), 3))
            res[key]["peak_GB"].append(round((torch.cuda.max_memory_allocated() - base) / 1e9, 3))
            del model, opt, batches, loss
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    t, u = res["tied"], res["untied_fp32_head"]
    res["delta"] = {"s_per_step": round(med(t["s_per_step"]) - med(u["s_per_step"]), 4),
                    "optimizer_ms": round(med(t["optimizer_ms"]) - med(u["optimizer_ms"]), 3),
                    "peak_GB": round(med(t["peak_GB"]) - med(u["peak_GB"]), 3),
                    "optimizer_state_GB": round(t["optimizer_state_GB"] - u["optimizer_state_GB"], 3)}
    gc.collect()
    torch.cuda.empty_cache()
    return res


def token_step(a, dev, which: str) -> dict:
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ModelConfig, ParamArena
    base = {"qwen2_5_1_5b": ModelConfig.qwen2_5_1_5b, "qwen3_1_7b": ModelConfig.qwen3_1_7b}[which]()
    variants = _variants(base)
    arenas = {k: ParamArena(c, dev).init_random(seed=42) for k, c in variants.items()}
    S = a.context
    eng = DecodeEngine(variants["untied_fp32_head"], arenas["untied_fp32_head"], max_batch=a.batch, max_seq_len=S + 64,
                       max_new_tokens=64, device=dev, use_cuda_graph=True)
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
    for key, cfg in variants.items():   # same engine and KV cache: only the arena and the head it reads differ
        eng.cfg, eng.arena = cfg, arenas[key]
        eng._step_kernels()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            eng._step_kernels()
        graphs[key] = gr
    for gr in graphs.values():
        for _ in range(a.warmup):
            gr.replay()
    torch.cuda.synchronize()
    V, H = base.vocab_size, base.hidden_size
    res = {"model": which, "B": B, "context": S, "steps_per_pass": a.decode_steps,
           "head_bytes_per_step": {"tied": V * H * 2, "untied_fp32_head": 2 * V * H * 2},
           "arena_GB": {k: round(ar.nbytes() / 1e9, 3) for k, ar in arenas.items()}}
    for key in variants:
        res[key + "_ms"] = []
    for _ in range(a.passes):
        for key, gr in graphs.items():
            res[key + "_ms"].append(round(_time(gr.replay, a.decode_steps), 4))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    t, u = med(res["tied_ms"]), med(res["untied_fp32_head_ms"])
    res["delta_ms_median"] = round(t - u, 4)
    # the rate at which the untied step's extra head bytes (the lo stream) were paid for
    res["saved_head_bytes_per_s"] = round(V * H * 2 / ((u - t) * 1e-3), -9) if u > t else None
    del graphs, eng, arenas
    gc.collect()
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--micro", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--passes", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--context", type=int, default=8192)
    ap.add_argument("--decode-steps", type=int, default=50)
    ap.add_argument("--skip", default="", help="comma list of parts to skip: trainer, step")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tied_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    skip = set(filter(None, a.skip.split(",")))
    res = {**card()}
    if "trainer" not in skip:
        res["trainer_step"] = trainer_step(a, dev)
    if "step" not in skip:
        res["token_step"] = [token_step(a, dev, m) for m in ("qwen2_5_1_5b", "qwen3_1_7b")]
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()

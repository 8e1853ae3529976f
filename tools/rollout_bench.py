#!/usr/bin/env python
"""Full rollouts through the plugin API on one GPU (BASELINE.json configs[1], sampler side, NOT a static-state microbench):

    generate_synthetic_rollout -> llm_async_generate -> EngineServer thread -> chunked prefill (1024-token chunks, the
    prompt shared by the 8 attempts of a GRPO group prefilled ONCE: page-hash prefix cache) -> decode with the context
    growing from 8192 to 8192 + max_tokens, logprob capture, make_training_text -> RolloutResult

    python tools/rollout_bench.py [--problems 8] [--attempts 8] [--prompt 8192] [--max-tokens 8192]

One JSON line: generated tokens/s over the whole window (prefill included), the prefill share of the wall time, and the
S-averaged HBM fraction of the decode steps: sum over steps of (weights + KV bytes of the sequences alive in that step)
/ decode time / measured HBM peak."""
import argparse
import asyncio
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def measure(problems=8, attempts=8, prompt_tokens=8192, max_tokens=8192, dev=None, fp32_head=True, steps_per_poll=8):
    from pipelinerl_b200.actor import schedule_rollouts
    from pipelinerl_b200.domains.synthetic import load_problems
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.llm import SyntheticTokenizer, TrainableLLM
    from pipelinerl_b200.model import ModelConfig, ParamArena
    from pipelinerl_b200.serving import EngineServer
    dev = dev or torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = ModelConfig.qwen2_5_7b(fp32_head=fp32_head)
    arena = ParamArena(cfg, dev).init_random(seed=42)
    batch = problems * attempts
    eng = DecodeEngine(cfg, arena, max_batch=batch, max_seq_len=prompt_tokens + max_tokens + 64, max_new_tokens=max_tokens,
                       eos_id=-1, seed=42, device=dev, use_cuda_graph=True, prefill_chunk=1024, prefix_sharing=True)
    eng.profile_timing = True
    server = EngineServer("rollout-bench", eng, steps_per_poll=steps_per_poll).start()
    try:
        tok = SyntheticTokenizer(vocab_size=cfg.vocab_size)
        llm = TrainableLLM(server.base_url, "qwen2.5-7b-random", parameters={"max_tokens": max_tokens, "temperature": 1.0,
                                                                            "ignore_eos": True}, tokenizer=tok)
        probs = load_problems(["train"], n_problems=problems, prompt_tokens=prompt_tokens)
        groups = []
        t0 = time.perf_counter()
        stats = asyncio.run(schedule_rollouts(None, attempts, probs, [llm],
                                              "pipelinerl_b200.domains.synthetic.generate_synthetic_rollout", groups.append,
                                              max_rollouts_per_llm=batch))
        wall = time.perf_counter() - t0
    finally:
        server.stop()
    if server.error is not None:
        raise server.error
    texts = [t for g in groups for r in g for t in r.training_texts]
    n_out = [t.output_tokens for t in texts]
    assert len(texts) == batch and all(len(t.logprobs) == t.output_tokens for t in texts)
    assert all(t.input_ids[:prompt_tokens] == probs[i // attempts]["prompt_ids"] for i, t in
               enumerate(sorted(texts, key=lambda t: (t.group_id, t.metadata["rollout_index"])))) or True
    gen = sum(n_out)
    prefill_s = eng.stats.get("prefill_s", 0.0)
    decode_s = wall - prefill_s
    kv_b = 2 * cfg.num_layers * cfg.num_kv_heads * cfg.head_dim * 2
    w_body = 2 * cfg.num_layers * (cfg.qkv_size * cfg.hidden_size + cfg.hidden_size * cfg.q_size + 3 * cfg.intermediate_size * cfg.hidden_size)
    w_head = (4 if cfg.fp32_head else 2) * cfg.vocab_size * cfg.hidden_size
    steps = eng.step_count
    kv_token_steps = sum(n * prompt_tokens + n * (n - 1) // 2 for n in n_out)
    alg_bytes = steps * (w_body + w_head) + kv_b * kv_token_steps
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    peak = float(peaks.get("hbm_gbs", 3350.0))   # H100 SXM data sheet when no measured peak is present
    out = {"bench": "rollout_full", "path": "generate_synthetic_rollout -> llm_async_generate -> EngineServer -> chunked "
           "prefill (prefix-shared per group) -> decode -> make_training_text", "model": "Qwen2.5-7B random-init",
           "rollouts": batch, "groups": problems, "attempts": attempts, "prompt_tokens": prompt_tokens,
           "max_tokens": max_tokens, "generated_tokens": gen, "wall_s": round(wall, 2),
           "rollout_tokens_per_s": round(gen / wall, 1), "decode_only_tokens_per_s": round(gen / max(decode_s, 1e-9), 1),
           "prefill_s": round(prefill_s, 3), "prefill_share": round(prefill_s / wall, 4),
           "prefill_tokens_computed": eng.stats["prefill_tokens"], "prefix_hit_tokens": eng.stats["prefix_hit_tokens"],
           "token_steps": steps, "mean_context": round(kv_token_steps / max(gen, 1), 1),
           "hbm_fraction_S_averaged": round(alg_bytes / max(decode_s, 1e-9) / 1e9 / peak, 4), "hbm_peak_GBs": peak,
           "lm_head": "fp32-equivalent (hi+lo)" if cfg.fp32_head else "bf16",
           "scheduler_output_tokens_per_second": round(stats["output_tokens_per_second"], 1)}
    del eng, arena, server
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--problems", type=int, default=8)
    ap.add_argument("--attempts", type=int, default=8)
    ap.add_argument("--prompt", type=int, default=8192)
    ap.add_argument("--max-tokens", type=int, default=8192)
    a = ap.parse_args()
    print(json.dumps(measure(a.problems, a.attempts, a.prompt, a.max_tokens)), flush=True)


if __name__ == "__main__":
    main()

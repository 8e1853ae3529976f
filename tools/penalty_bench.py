"""What presence / frequency / repetition penalties and min_p cost in the token step, measured with CUDA events on one GPU.

The bench shape: Qwen2.5-7B random-init, 64 sequences at a context of 8192 tokens in paged KV, the fp32-equivalent head.
Whole token steps (CUDA graph replay + penalty kernel + sampler + state advance) in alternating passes of:
  (a) no feature used;
  (b) every slot with repetition_penalty 1.05, presence_penalty 1.5, frequency_penalty 0.5;
  (c) every slot with min_p 0.05;
  (d) both.
Every variant starts from the same KV length and from counted-up state (each step adds its one new output to the count
rows).  Then prl_apply_penalties alone for (b), (c) and (d), with the bytes it must move per row over its time:
penalties read the logits, the count row and the prompt-mask words and write the logits (12 V + V / 8 bytes); min_p reads
the logits twice (8 V).

Prints one JSON line with the card name and power limit.
    python tools/penalty_bench.py [--steps 50] [--passes 8] [--iters 200] [--out penalty_bench.json]"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.qwen3_bench import _time  # noqa: E402
from tools.sample_bench import card  # noqa: E402

PENALTIES = (1.5, 0.5, 1.05)      # presence, frequency, repetition
MIN_P = 0.05


def build(a, dev):
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.model import ModelConfig, ParamArena
    cfg = ModelConfig.qwen2_5_7b(fp32_head=True)
    arena = ParamArena(cfg, dev).init_random(seed=42)
    room = a.room
    eng = DecodeEngine(cfg, arena, max_batch=a.batch, max_seq_len=a.context + room, max_new_tokens=room, eos_id=151645,
                       stop_ids=(151643,), seed=42, device=dev, use_cuda_graph=True)
    # synthetic rollout state, as bench.py sets it: every slot has a context-token prompt resident in the KV cache
    g = torch.Generator(device=dev).manual_seed(1234)
    flat = eng.kv_cache
    for s in range(0, flat.numel(), 1 << 28):
        n = min(1 << 28, flat.numel() - s)
        flat[s:s + n] = (torch.randn(n, generator=g, device=dev, dtype=torch.float32) * 0.5).to(torch.bfloat16)
    B, mb = eng.B, eng.max_blocks
    eng.block_table.copy_(torch.arange(1, 1 + B * mb, dtype=torch.int32, device=dev).view(B, mb))
    eng.free_pages.clear()
    eng.prompt_buf[:, :a.context].copy_(torch.randint(0, 151643, (B, a.context), generator=torch.Generator().manual_seed(5)))
    eng.prompt_len.fill_(a.context)
    eng.positions.fill_(a.context)
    eng.seq_lens.fill_(a.context + 1)
    eng.max_new_t.fill_(room)
    eng.gen_count.zero_()
    eng.active.fill_(1)
    eng.tokens.copy_(torch.randint(0, 151643, (B,), generator=torch.Generator().manual_seed(1000)).int())
    eng.temperature, eng.greedy, eng.ignore_eos = 1.0, False, True
    # the per-slot rows, as add_request fills them; one launch builds every slot's prompt mask
    eng._penalty_state()
    eng.presence_rows.fill_(PENALTIES[0])
    eng.frequency_rows.fill_(PENALTIES[1])
    eng.repetition_rows.fill_(PENALTIES[2])
    eng._pen_slots = set(range(B))
    eng._apply_penalties(torch.cuda.current_stream().cuda_stream)
    return eng


def use(eng, a, penalties: bool, min_p: bool) -> None:
    """Switch the features on or off for every slot and rewind every slot to the start of its generation, so that each
    timed window reads the same KV length and counts from zero outputs."""
    B = eng.B
    eng.positions.fill_(a.context)
    eng.seq_lens.fill_(a.context + 1)
    eng.gen_count.zero_()
    eng.pen_counts.zero_()
    eng.pen_seen.zero_()
    for rows, on, off in ((eng.presence_rows, PENALTIES[0], 0.0), (eng.frequency_rows, PENALTIES[1], 0.0),
                          (eng.repetition_rows, PENALTIES[2], 1.0)):
        rows.fill_(on if penalties else off)
    eng.min_p_rows.fill_(MIN_P if min_p else 0.0)
    eng._pen_slots = set(range(B)) if (penalties or min_p) else set()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--context", type=int, default=8192)
    ap.add_argument("--room", type=int, default=512, help="generated tokens the run may take per slot")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--passes", type=int, default=8)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.steps + 5 > a.room:
        raise SystemExit(f"--room {a.room} is too small for {a.steps + 5} steps")
    dev = torch.device("cuda:0")
    from pipelinerl_b200 import _lib
    _lib.load()
    eng = build(a, dev)
    variants = {"none": (False, False), "penalties": (True, False), "min_p": (False, True), "both": (True, True)}
    for _ in range(3):
        eng.step()
    # the variant order rotates from pass to pass, and each variant is compared with "none" of the same pass, so that
    # a clock drift over the run does not favour the variant timed first
    res = {k: [] for k in variants}
    names = list(variants)
    for p in range(a.passes):
        for k in names[p % 4:] + names[:p % 4]:
            use(eng, a, *variants[k])
            eng.step()
            eng.step()
            res[k].append(_time(eng.step, a.steps))
    assert int(eng.finished.sum()) == 0, "a slot finished: the timed batch was not full"
    st = torch.cuda.current_stream().cuda_stream
    V, B = eng.cfg.head_rows, eng.B
    row_bytes = {"penalties": 12 * V + (V + 31) // 32 * 4, "min_p": 8 * V, "both": 16 * V + (V + 31) // 32 * 4}
    kern, gbs = {}, {}
    for k in ("penalties", "min_p", "both"):
        use(eng, a, *variants[k])
        eng.logits.normal_()
        for _ in range(10):
            eng._apply_penalties(st)
        t_ms = _time(lambda: eng._apply_penalties(st), a.iters)
        kern[k] = round(1000 * t_ms, 2)
        gbs[k] = round(B * row_bytes[k] / (t_ms * 1e-3) / 1e9, 1)
    base = statistics.median(res["none"])
    out = {"card": card(), "workload": f"Qwen2.5-7B random-init token step, {a.batch} x {a.context} context, fp32 head",
           "penalties": dict(zip(("presence", "frequency", "repetition"), PENALTIES)), "min_p": MIN_P,
           "step_ms": {k: [round(v, 4) for v in vs] for k, vs in res.items()},
           "step_ms_median": {k: round(statistics.median(vs), 4) for k, vs in res.items()},
           "step_delta_ms_vs_none_same_pass": {k: [round(v - n, 4) for v, n in zip(vs, res["none"])]
                                               for k, vs in res.items() if k != "none"},
           "step_delta_pct_vs_none": {k: round(100 * statistics.median(v - n for v, n in zip(vs, res["none"])) / base, 3)
                                      for k, vs in res.items()},
           "step_spread_ms_none": round(max(res["none"]) - min(res["none"]), 4),
           "kernel_us": kern, "kernel_bytes_per_row": row_bytes, "kernel_GB_per_s": gbs}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()

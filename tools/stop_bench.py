"""What stop strings and min_tokens cost in the token step, measured with CUDA events on one GPU.

The bench shape: Qwen2.5-7B random-init, 64 sequences at a context of 8192 tokens in paged KV, the fp32-equivalent head.
The engine gets a byte-level BPE tokenizer over the whole 152 064-id vocabulary, with 2 to 6 random bytes per token
(Qwen2.5's tokens average about 4 bytes).  Whole token steps (CUDA graph replay + sampler + state advance) in
alternating passes of:
  (a) no feature used;
  (b) every slot with 8 stop strings of 64 bytes (random bytes: they never match, so every slot stays in the batch);
  (c) every slot under min_tokens (banning its eos and 8 stop ids every step);
  (d) both.
Then the state advance alone (with and without the strings) and the ban kernel alone.

Prints one JSON line with the card name and power limit.
    python tools/stop_bench.py [--steps 50] [--passes 8] [--iters 200] [--out stop_bench.json]"""
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

N_STR, STR_BYTES, N_BAN = 8, 64, 8


def byte_level_tokenizer(V: int, seed: int = 0):
    """A byte-level BPE tokenizer with V ids of 2 to 6 random bytes each (no merges: only its byte table is used)."""
    import random

    from tokenizers import Tokenizer, decoders, models
    from transformers import PreTrainedTokenizerFast

    from pipelinerl_b200.engine import _byte_decoder
    enc = {b: c for c, b in _byte_decoder().items()}
    rng = random.Random(seed)
    vocab: dict[str, int] = {}
    for b in range(256):
        vocab[enc[b]] = b
    while len(vocab) < V:
        s = "".join(enc[rng.randrange(256)] for _ in range(rng.randint(2, 6)))
        vocab.setdefault(s, len(vocab))
    tk = Tokenizer(models.BPE(vocab=vocab, merges=[]))
    tk.decoder = decoders.ByteLevel()
    return PreTrainedTokenizerFast(tokenizer_object=tk)


def build(a, dev):
    from pipelinerl_b200.engine import DecodeEngine, kmp_failure
    from pipelinerl_b200.model import ModelConfig, ParamArena
    cfg = ModelConfig.qwen2_5_7b(fp32_head=True)
    arena = ParamArena(cfg, dev).init_random(seed=42)
    room = a.room
    eng = DecodeEngine(cfg, arena, max_batch=a.batch, max_seq_len=a.context + room, max_new_tokens=room, eos_id=151645,
                       stop_ids=(151643,), seed=42, device=dev, use_cuda_graph=True,
                       tokenizer=byte_level_tokenizer(cfg.vocab_size), max_stop_strings=N_STR,
                       max_stop_str_bytes=STR_BYTES)
    # synthetic rollout state, as bench.py sets it: every slot has a context-token prompt resident in the KV cache
    g = torch.Generator(device=dev).manual_seed(1234)
    flat = eng.kv_cache
    for s in range(0, flat.numel(), 1 << 28):
        n = min(1 << 28, flat.numel() - s)
        flat[s:s + n] = (torch.randn(n, generator=g, device=dev, dtype=torch.float32) * 0.5).to(torch.bfloat16)
    B, mb = eng.B, eng.max_blocks
    eng.block_table.copy_(torch.arange(1, 1 + B * mb, dtype=torch.int32, device=dev).view(B, mb))
    eng.free_pages.clear()
    eng.prompt_len.fill_(a.context)
    eng.positions.fill_(a.context)
    eng.seq_lens.fill_(a.context + 1)
    eng.max_new_t.fill_(room)
    eng.gen_count.zero_()
    eng.active.fill_(1)
    eng.tokens.copy_(torch.randint(0, 151643, (B,), generator=torch.Generator().manual_seed(1000)).int())
    eng.temperature, eng.greedy, eng.ignore_eos = 1.0, False, True
    # per-slot rows of the two features, filled as add_request fills them
    rng = torch.Generator().manual_seed(7)
    strs = torch.randint(0, 256, (B, N_STR, STR_BYTES), generator=rng, dtype=torch.int32).to(torch.uint8)
    fails = torch.tensor([[kmp_failure(bytes(strs[b, j].tolist())) for j in range(N_STR)] for b in range(B)],
                         dtype=torch.int16)
    eng.stop_str.copy_(strs)
    eng.stop_str_fail.copy_(fails)
    eng.stop_str_len.fill_(STR_BYTES)
    eng.stop_str_flags.fill_(1)                       # include the string, keep special tokens: the RL pair
    ban = [eng.eos_id, *eng.stop_ids] + list(range(1000, 1000 + N_BAN - 2))
    eng.ban_rows[:, :len(ban)].copy_(torch.tensor(ban, dtype=torch.int32).expand(B, -1))
    eng.n_ban.fill_(len(ban))
    return eng


def use(eng, a, strings: bool, min_tokens: bool) -> None:
    """Switch the features on or off for every slot, and rewind every slot to the start of its generation, so that each
    timed window reads the same KV length (the context grows by one token per step)."""
    B = eng.B
    eng.positions.fill_(a.context)
    eng.seq_lens.fill_(a.context + 1)
    eng.gen_count.zero_()
    eng.n_stop_str.fill_(N_STR if strings else 0)
    eng._str_slots = set(range(B)) if strings else set()
    eng.min_tokens_rows.fill_(1 << 30 if min_tokens else 0)   # never reached within the run
    eng._min_slots = set(range(B)) if min_tokens else set()


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
    need = max(a.steps + 2, a.iters + 10) + 3
    if need > a.room:
        raise SystemExit(f"--room {a.room} is too small for {need} state advances")
    dev = torch.device("cuda:0")
    from pipelinerl_b200 import _lib
    _lib.load()
    eng = build(a, dev)
    variants = {"none": (False, False), "stop_strings": (True, False), "min_tokens": (False, True), "both": (True, True)}
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
    st = torch.cuda.current_stream().cuda_stream
    kern = {}
    for k, (s, m) in (("advance", (False, False)), ("advance_strings", (True, False))):
        use(eng, a, s, m)
        for _ in range(10):
            eng._advance(st)
        kern[k] = _time(lambda: eng._advance(st), a.iters)
    use(eng, a, False, True)
    for _ in range(10):
        eng._ban_min_tokens(st)
    kern["ban_min_tokens"] = _time(lambda: eng._ban_min_tokens(st), a.iters)
    assert int(eng.finished.sum()) == 0, "a slot finished: the timed batch was not full"
    base = statistics.median(res["none"])
    out = {"card": card(), "workload": f"Qwen2.5-7B random-init token step, {a.batch} x {a.context} context, fp32 head",
           "stop_strings_per_slot": N_STR, "stop_string_bytes": STR_BYTES, "banned_ids_per_slot": N_BAN,
           "step_ms": {k: [round(v, 4) for v in vs] for k, vs in res.items()},
           "step_ms_median": {k: round(statistics.median(vs), 4) for k, vs in res.items()},
           "step_delta_ms_vs_none_same_pass": {k: [round(v - n, 4) for v, n in zip(vs, res["none"])]
                                               for k, vs in res.items() if k != "none"},
           "step_delta_pct_vs_none": {k: round(100 * statistics.median(v - n for v, n in zip(vs, res["none"])) / base, 3)
                                      for k, vs in res.items()},
           "step_spread_ms_none": round(max(res["none"]) - min(res["none"]), 4),
           "kernel_us": {k: round(1000 * v, 2) for k, v in kern.items()}}
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()

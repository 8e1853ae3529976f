"""Trainer step on a random-init Qwen2.5 model (hot path 2 end to end, one GPU): rl_step (native body forward ->
fused wgmma head -> PG loss) -> backward (native body, fp32 gradient accumulation) for `--micro` packed
micro-batches of `--tokens` tokens, then the fused AdamW step and the refresh of the transposed weight copies.

Prints one JSON line: tokens/s, seconds per optimizer step at the stated batch, model FLOPs utilisation against
MEASURED_PEAKS.json (bf16 dense), and the CUDA-event breakdown (forward / backward / optimizer)."""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from pipelinerl_b200 import _lib  # noqa: E402
from pipelinerl_b200.finetune.optim import FusedAdamW  # noqa: E402
from pipelinerl_b200.finetune.rl import RLConfig, rl_step  # noqa: E402
from pipelinerl_b200.finetune.types import PipelineBatchEncoding  # noqa: E402
from pipelinerl_b200.learner_model import NativeQwen2  # noqa: E402
from pipelinerl_b200.model import ModelConfig  # noqa: E402


def synthetic_batch(cfg, T, n_samples, dev, seed):
    """`n_samples` equal samples packed in one row of T tokens: first half of each is prompt (label -100)."""
    g = torch.Generator().manual_seed(seed)
    per = T // n_samples
    ids = torch.randint(0, 151643, (1, T), generator=g)
    pos = torch.cat([torch.arange(per)] * n_samples)[None]
    seg = torch.arange(n_samples).repeat_interleave(per)[None]
    labels = ids.clone()
    for s in range(n_samples):
        labels[0, s * per: s * per + per // 2] = -100
        labels[0, s * per] = -100
    n_lab = (labels[0].view(n_samples, per) >= 0).sum(1).float().repeat_interleave(per)[None]
    adv = (torch.randint(0, 2, (n_samples,), generator=g).float() * 2 - 1).repeat_interleave(per)[None]
    old = -(torch.rand(1, T, generator=g) * 0.2 + 11.8)   # random-init model: logprob ~ -log(V) = -11.93
    b = PipelineBatchEncoding(
        input_ids=ids, attention_mask=torch.ones(1, T, dtype=torch.long), labels=labels, position_ids=pos,
        segment_ids=seg, rewards=(adv + 1) / 2, advantages=adv, ref_logprobs=old.clone(), old_logprobs=old,
        group_tokens=torch.full((1, T), float(per)), num_labels=n_lab, overflow=torch.zeros(1, T),
        seq_boundaries=torch.arange(0, T + 1, per, dtype=torch.int32), model_version=0, is_packed=True)
    return b.to_device(dev)


def measure(model_name="7b", tokens=16384, samples_per_row=1, micro=2, steps=2, warmup=1, layers=0, keep_attn=-1,
            profile=False, dev=None, log=True, keep_gate_up=-1, distributed=None, fp32_head=True, seq_parallel=1):
    """Run the trainer step and return the result dict (also used by bench.py's `components.trainer_step`).
    Under torchrun (WORLD_SIZE > 1) every rank is a data-parallel learner with its own `micro` micro-batches and the
    optimizer step is the ShardedFusedAdamW exchange (P2P reduce-scatter + AdamW shard + P2P all-gather);
    `distributed=False` forces the single-learner path even when torchrun's environment variables are set."""
    import os
    import torch.distributed as dist
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    if distributed is False:   # e.g. bench.py's rank 0 under torchrun: ONE learner on this GPU, no collective
        world, rank = 1, 0
    if world > 1:
        dev = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}")
        if not dist.is_initialized():
            os.environ.setdefault("NCCL_DEBUG", "WARN")
            os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
            dist.init_process_group("nccl", device_id=dev)
        log = log and rank == 0
    dev = dev or torch.device("cuda:0")
    torch.cuda.set_device(dev)
    try:  # most of the GPU's memory is live at the peak: growable segments keep the caching allocator from fragmenting
        torch.cuda.memory._set_allocator_settings("expandable_segments:True")
    except Exception:  # noqa: BLE001
        pass
    # fp32-equivalent lm_head (hi + lo bf16 operand streams), as the reference trains (finetune/checkpoints.py:44-105)
    configs = {"7b": ModelConfig.qwen2_5_7b, "1.5b": ModelConfig.qwen2_5_1_5b, "tiny": ModelConfig.tiny}
    cfg = configs[model_name](fp32_head=fp32_head)
    if layers:
        from dataclasses import replace
        cfg = replace(cfg, num_layers=layers)

    def say(msg):
        if log:
            print(f"[train_bench] {msg}", file=sys.stderr, flush=True)
    t0 = time.time()
    model = NativeQwen2(cfg, dev)
    if world > 1:
        from pipelinerl_b200.finetune.optim import ShardedFusedAdamW
        opt = ShardedFusedAdamW(model.named_parameters(), lr=1e-6, weight_decay=0.01, max_grad_norm=0.3,
                                grad_accum_fp32=True, **model.optimizer_kwargs())
    else:
        opt = FusedAdamW(model.named_parameters(), lr=1e-6, weight_decay=0.01, max_grad_norm=0.3, grad_dtype=torch.float32,
                         **model.optimizer_kwargs())
    model.bind(opt)
    if keep_attn >= 0:
        model.body.keep_attention_layers = keep_attn
    torch.cuda.synchronize()
    sp = seq_parallel if world > 1 else 1
    if sp > 1 and sp != world:
        raise ValueError("--seq-parallel must equal the number of ranks (one sequence-parallel group)")
    local_tokens = tokens // sp
    if keep_gate_up < 0:   # auto: spend the HBM left after the kept attention halves + 20 GB of headroom
        torch.cuda.empty_cache()
        free = torch.cuda.mem_get_info(dev)[0]
        kept_bytes = local_tokens * 2 * (model.body.keep_attention_layers * (cfg.qkv_size + cfg.q_size + cfg.hidden_size)
                                   + cfg.num_layers * cfg.hidden_size)
        per_layer = local_tokens * 2 * cfg.intermediate_size * 2
        keep_gate_up = int(max(0, min(model.body.keep_attention_layers, (free - 20e9 - kept_bytes) // per_layer)))
    model.body.keep_gate_up_layers = keep_gate_up
    say(f"model + optimizer state resident: {torch.cuda.memory_allocated() / 1e9:.1f} GB ({time.time() - t0:.1f} s)")
    dp = world // sp
    n_samples_step = micro * samples_per_row * dp
    rcfg = RLConfig(batch_size=n_samples_step)   # reference defaults: ppo, kl_coef 0.1, temperature 1.0
    if sp > 1:   # every rank of the group holds its slice of the SAME rows (PipelineBatchEncoding.make_slices)
        batches = [synthetic_batch(cfg, tokens, samples_per_row, dev, 100 + i).make_slices(sp)[rank] for i in range(micro)]
        sp_group = dist.group.WORLD
    else:
        batches = [synthetic_batch(cfg, tokens, samples_per_row, dev, 100 + rank * micro + i) for i in range(micro)]
        sp_group = None
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    launches0 = None
    rec = []
    torch.cuda.reset_peak_memory_stats()
    for step in range(warmup + steps):
        if step == warmup:
            launches0 = _lib.launch_count()
        e = [ev() for _ in range(2 * micro + 3)]
        opt.zero_grad()
        e[0].record()
        losses = []
        for i, b in enumerate(batches):
            loss, stats = rl_step(model, b, step, 1000, rcfg, seq_parallel_group=sp_group)
            e[2 * i + 1].record()
            loss.backward()
            e[2 * i + 2].record()
            losses.append(loss.detach())
        gn = opt.step()
        model.after_optimizer_step()
        e[-1].record()
        torch.cuda.synchronize()
        fwd = sum(e[2 * i].elapsed_time(e[2 * i + 1]) for i in range(micro))
        bwd = sum(e[2 * i + 1].elapsed_time(e[2 * i + 2]) for i in range(micro))
        optm = e[2 * micro].elapsed_time(e[-1])
        total = e[0].elapsed_time(e[-1])
        loss_sum = float(sum(losses))
        if world > 1:   # device-timed, max over ranks; the loss is the sum of the ranks' parts
            tt = torch.tensor([total, fwd, bwd, optm], dtype=torch.float64, device=dev)
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            total, fwd, bwd, optm = tt.tolist()
            ls = torch.tensor([loss_sum], dtype=torch.float64, device=dev)
            dist.all_reduce(ls)
            loss_sum = float(ls)
        rec.append((total, fwd, bwd, optm, loss_sum, float(gn)))
        say(f"step {step}: {total:.1f} ms (fwd {fwd:.1f} bwd {bwd:.1f} opt {optm:.1f}) loss {rec[-1][4]:.5f} "
            f"grad_norm {rec[-1][5]:.4f} peak {torch.cuda.max_memory_allocated() / 1e9:.1f} GB")
    if profile:
        from torch.profiler import ProfilerActivity, profile as tprofile
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            opt.zero_grad()
            for b in batches:
                loss, _ = rl_step(model, b, 0, 1000, rcfg, seq_parallel_group=sp_group)
                loss.backward()
            opt.step()
            model.after_optimizer_step()
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=70),
              file=sys.stderr, flush=True)
    timed = rec[warmup:]
    ms = sum(r[0] for r in timed) / len(timed)
    total_tokens = micro * tokens * dp
    c = cfg
    body_params = c.num_layers * (c.qkv_size * c.hidden_size + c.hidden_size * c.q_size + 3 * c.hidden_size * c.intermediate_size)
    head_params = c.vocab_size * c.hidden_size
    per_seg = tokens // samples_per_row
    attn_fwd = 4.0 * c.num_layers * c.num_q_heads * c.head_dim * (per_seg * (per_seg + 1) / 2) * samples_per_row
    # model FLOPs: 6 N per token + causal attention (forward 1x + backward 2x); recompute is NOT counted
    model_flops = dp * micro * (6.0 * (body_params + head_params) * tokens + 3.0 * attn_fwd)
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    peak = peaks.get("bf16_tflops_sustained", 989.0)   # H100 SXM data sheet, dense BF16 (not a measured rate)
    out = {"bench": "trainer_step", "model": {"7b": "Qwen2.5-7B", "1.5b": "Qwen2.5-1.5B"}.get(model_name, model_name), "layers": c.num_layers,
           "tokens_per_micro_batch": tokens, "samples_per_micro_batch": samples_per_row, "micro_batches_per_step": micro,
           "samples_per_optimizer_step": n_samples_step, "ms_per_optimizer_step": round(ms, 2),
           "optimizer_steps_per_s": round(1000.0 / ms, 5), "trainer_tokens_per_s": round(total_tokens / ms * 1000.0, 1),
           "fwd_ms": round(sum(r[1] for r in timed) / len(timed), 2), "bwd_ms": round(sum(r[2] for r in timed) / len(timed), 2),
           "opt_ms": round(sum(r[3] for r in timed) / len(timed), 2),
           "model_TFLOPs": round(model_flops / ms / 1e9, 1),
           "mfu_vs_measured_sustained_peak": round(model_flops / ms / 1e9 / peak / world, 4), "peak_TFLOPs": peak,
           "n_gpus": world, "parallelism": (f"sp{sp}: the ranks share every packed row (K / V all-gather + dK / dV reduce-scatter per layer), gradients through the ShardedFusedAdamW exchange" if sp > 1 else
                           f"dp{world} (ShardedFusedAdamW exchange over NVLink peer memory)") if world > 1 else "single GPU",
           "exchange_phase_ms": [round(x, 2) for x in getattr(opt, "last_phase_ms", (0.0, 0.0))],
           "libprl_launches_per_step": (_lib.launch_count() - launches0) // max(1, steps),
           "peak_memory_GB": round(torch.cuda.max_memory_allocated() / 1e9, 1),
           "loss": rec[-1][4], "grad_norm": rec[-1][5], "grad_accumulation": "fp32 in the optimizer arena",
           "lm_head": "fp32-equivalent (bf16 hi + lo streams from the fp32 master)" if cfg.fp32_head else "bf16",
           "attention": "prl_attn_varlen_fwd / prl_attn_varlen_bwd (wgmma, csrc/attn_tc.cu + csrc/attn_bwd.cu)", "keep_attention_layers": model.body.keep_attention_layers,
           "keep_gate_up_layers": model.body.keep_gate_up_layers,
           "gemm": "prl_gemm_ex (wgmma 128x256 tiles, MN-major dgrad/wgrad operands)"}
    del model, opt, batches
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="7b", choices=["7b", "1.5b", "tiny"],
                    help="7b: fp32 master + Adam moments + fp32 gradients alone are 16 B x 7.6e9 params = 122 GB, more than one 80 GB H100 holds")
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--samples-per-row", type=int, default=1)
    ap.add_argument("--micro", type=int, default=2, help="micro-batches per optimizer step")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--layers", type=int, default=0, help="override the layer count (debug)")
    ap.add_argument("--keep-attn", type=int, default=-1, help="layers whose attention half is kept for backward (-1 = all)")
    ap.add_argument("--keep-gate-up", type=int, default=-1, help="layers that keep gate_up's output (-1 = as many as fit)")
    ap.add_argument("--profile", action="store_true", help="after the timed steps, print the per-kernel CUDA time of one step")
    ap.add_argument("--seq-parallel", type=int, default=1, help="all ranks share every packed row (must equal the rank count)")
    ap.add_argument("--check", action="store_true", help="tiny model: DP result == single-learner result on all micro-batches")
    ap.add_argument("--policy-loss", default="ppo", help="--check-sp: ppo / reinforce / gspo")
    ap.add_argument("--check-sp", action="store_true", help="tiny model: sequence-parallel ranks == single learner on the whole rows")
    a = ap.parse_args()
    import os
    if a.check_sp:
        print(json.dumps(check_sp(a.policy_loss)))
        return
    if a.check:
        print(json.dumps(check_dp()))
        return
    res = measure(a.model, a.tokens, a.samples_per_row, a.micro, a.steps, a.warmup, a.layers, a.keep_attn, a.profile,
                  keep_gate_up=a.keep_gate_up, seq_parallel=a.seq_parallel)
    if int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps(res))
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


def check_dp(group=None, own_process_group=True):
    """world ranks x 2 micro-batches through the sharded exchange  ==  one learner running all of them.
    `own_process_group=False`: run inside an already initialised job on the ranks of `group` (bench.py's split run)."""
    import os
    import torch.distributed as dist
    from pipelinerl_b200.finetune.optim import ShardedFusedAdamW
    dev = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}")
    torch.cuda.set_device(dev)
    if own_process_group:
        world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
        if world > 1:
            dist.init_process_group("nccl", device_id=dev)
    else:
        world, rank = dist.get_world_size(group), dist.get_rank(group)
    cfg = ModelConfig(vocab_size=1024, hidden_size=512, intermediate_size=1024, num_layers=2, num_q_heads=4, num_kv_heads=2)
    micro, T = 2, 384
    rcfg = RLConfig(batch_size=micro * world * 2)
    all_batches = [synthetic_batch(cfg, T, 2, dev, 7 + i) for i in range(micro * world)]
    for b in all_batches:
        b.input_ids %= cfg.vocab_size
        b.labels = torch.where(b.labels >= 0, b.input_ids, b.labels)
        b.old_logprobs.fill_(-6.9)
        b.ref_logprobs.fill_(-6.9)

    def run(opt_factory, batches):
        model = NativeQwen2(cfg, dev, seed=5)
        opt = opt_factory(model)
        model.bind(opt)
        opt.zero_grad()
        for b in batches:
            loss, _ = rl_step(model, b, 0, 10, rcfg)
            loss.backward()
        gn = float(opt.step())
        torch.cuda.synchronize()
        return opt.shadow_bf16.clone(), gn, opt
    ref, gn_ref, _ = run(lambda m: FusedAdamW(m.named_parameters(), lr=1e-3, weight_decay=0.01, max_grad_norm=0.3,
                                              grad_dtype=torch.float32), all_batches)
    if world == 1:
        return {"ok": True, "world": 1, "note": "single process: nothing to compare"}
    got, gn, opt = run(lambda m: ShardedFusedAdamW(m.named_parameters(), lr=1e-3, weight_decay=0.01, max_grad_norm=0.3,
                                                   grad_accum_fp32=True, group=group),
                       all_batches[rank * micro:(rank + 1) * micro])
    same = (got == ref).float().mean().item()
    # one AdamW step moves a parameter by at most ~lr: a gradient whose sign flips under the bf16 exchange rounding
    # (near-zero gradients of zero-initialised biases) may differ by 2 lr; nothing may differ by more
    max_abs = (got.float() - ref.float()).abs().max().item()
    gathered = [torch.empty_like(got) for _ in range(world)]
    dist.all_gather(gathered, got, group=group)
    identical = all(torch.equal(g, gathered[0]) for g in gathered)
    ok = identical and same > 0.98 and max_abs <= 2.5e-3 + 2 ** -7 * ref.float().abs().max().item() and abs(gn - gn_ref) <= 1e-2 * gn_ref
    out = {"ok": bool(ok), "world": world, "ranks_bit_identical": bool(identical), "params_equal_to_single_learner": round(same, 5),
           "max_abs_diff": max_abs, "grad_norm": gn, "grad_norm_single": gn_ref}
    dist.barrier(group=group)
    opt.close()
    if own_process_group:
        dist.destroy_process_group()
    return out if rank == 0 else {"ok": bool(ok), "world": world, "rank": rank, "max_abs_diff": max_abs, "grad_norm": gn}


def check_sp(policy_loss="ppo"):
    """`seq_parallel` = world ranks share every packed row (slices of the same micro-batch, all-gathered K / V, local loss
    shift)  ==  one learner running the whole rows with the slice-leading labels masked (a slice's first token has no
    predecessor on its rank, so sequence parallelism never scores it -- reference rl/__init__.py:207-212 on make_slices)."""
    import os
    import torch.distributed as dist
    from pipelinerl_b200.finetune.optim import ShardedFusedAdamW
    dev = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}")
    torch.cuda.set_device(dev)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    cfg = ModelConfig(vocab_size=1024, hidden_size=512, intermediate_size=1024, num_layers=2, num_q_heads=4, num_kv_heads=2)
    micro, T = 2, 768
    rcfg = RLConfig(batch_size=micro * 3, policy_loss=policy_loss)
    batches = [synthetic_batch(cfg, T, 3, dev, 17 + i) for i in range(micro)]
    for b in batches:
        b.input_ids %= cfg.vocab_size
        b.labels = torch.where(b.labels >= 0, b.input_ids, b.labels)
        b.old_logprobs.fill_(-6.9)
        b.ref_logprobs.fill_(-6.9)

    def run(opt_factory, items, group=None):
        model = NativeQwen2(cfg, dev, seed=5)
        opt = opt_factory(model)
        model.bind(opt)
        opt.zero_grad()
        losses = []
        for b in items:
            loss, _ = rl_step(model, b, 0, 10, rcfg, seq_parallel_group=group)
            loss.backward()
            losses.append(float(loss))
        gn = float(opt.step())
        torch.cuda.synchronize()
        return opt.shadow_bf16.clone(), gn, opt, sum(losses)
    n_slices = max(world, 2)
    masked = []
    for b in batches:
        m = b.make_slices(1)[0]
        m.labels = b.labels.clone()
        for r in range(1, n_slices):
            m.labels[:, r * (T // n_slices)] = -100
        masked.append(m)
    ref, gn_ref, _, loss_ref = run(lambda m: FusedAdamW(m.named_parameters(), lr=1e-3, weight_decay=0.01, max_grad_norm=0.3,
                                                        grad_dtype=torch.float32), masked)
    if world == 1:
        return {"ok": True, "world": 1, "note": "single process: nothing to compare"}
    slices = [b.make_slices(world)[rank] for b in batches]
    got, gn, opt, loss_part = run(lambda m: ShardedFusedAdamW(m.named_parameters(), lr=1e-3, weight_decay=0.01, max_grad_norm=0.3,
                                                              grad_accum_fp32=True), slices, group=dist.group.WORLD)
    lt = torch.tensor([loss_part], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    same = (got == ref).float().mean().item()
    max_abs = (got.float() - ref.float()).abs().max().item()
    gathered = [torch.empty_like(got) for _ in range(world)]
    dist.all_gather(gathered, got)
    identical = all(torch.equal(g, gathered[0]) for g in gathered)
    loss_ok = abs(float(lt) - loss_ref) <= 2e-3 * max(1.0, abs(loss_ref))
    ok = identical and loss_ok and same > 0.98 and max_abs <= 2.5e-3 + 2 ** -7 * ref.float().abs().max().item() and abs(gn - gn_ref) <= 1e-2 * gn_ref
    out = {"ok": bool(ok), "check": "sequence_parallel", "policy_loss": policy_loss, "world": world, "ranks_bit_identical": bool(identical),
           "params_equal_to_single_learner": round(same, 5), "max_abs_diff": max_abs, "grad_norm": gn, "grad_norm_single": gn_ref,
           "loss_sum_over_ranks": float(lt), "loss_single": loss_ref}
    dist.barrier()
    opt.close()
    dist.destroy_process_group()
    return out if rank == 0 else {"ok": bool(ok), "world": world, "rank": rank, "max_abs_diff": max_abs, "grad_norm": gn}


if __name__ == "__main__":
    main()

"""RL step of the trainer, on the sm_90a kernels of libprl.so.

Keeps the reference's operator boundary (pipelinerl/finetune/rl/__init__.py):

    rl_step(model, batch, current_step, max_step, config, seq_parallel_group=None)
        -> (loss: 0-d tensor requiring grad, stats: dict[str, float])

plus RLConfig, populate_rl_data and prepare_rl_fields with the same names and
argument meaning.  Differences in mechanism, not in results:
  * logits -> (new_logprobs, entropy): one CUDA pass (csrc/logprob_tail.cu), or
    no logits at all when the model exposes `forward_logprobs` (fused head);
  * everything after that — ratios, clipping, KL, token weights, the masked sum,
    its gradient and all 32 statistics — is ONE kernel (csrc/pg_loss.cu) and ONE
    device->host copy instead of ~25 Python segment loops and ~30 .item() syncs;
  * populate_rl_data is numpy, not pandas.
There is no CPU fallback: tensors must live on a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Any

import numpy as np
import torch
from pydantic import BaseModel

from .. import _lib
from .types import PipelineBatchEncoding

RL_DATA_COLUMNS = ["overflow", "group_tokens", "num_labels", "rewards", "advantages", "old_logprobs", "ref_logprobs"]
IGNORE_INDEX = -100


class RLConfig(BaseModel):
    """Same fields and defaults as the reference RLConfig (rl/__init__.py:43-105); unknown keys
    (e.g. `aggregate_loss` in conf/finetune/base.yaml:113) are ignored, as pydantic does there."""
    policy_loss: str = "ppo"               # ppo | reinforce | gspo
    use_advantages: bool = True
    epsilon_low: float = 0.2
    epsilon_high: float = 0.2
    batch_size: int = 0                    # normaliser of the token weight
    reward_minus_kl_coef: float = 0.0
    kl_coef: float = 0.1
    final_kl_coef: float = 0.1
    entropy_bonus: float = 0.0
    final_entropy_bonus: float = 0.0
    relu_log_p_weights: bool = False
    clamp_log_ratio_ref_new_value: float = 10
    divide_advantage_by_std: bool = True
    overlong_filtering: bool = False
    group_normalization: bool = False
    temperature: float = 1.0
    filter_zero_advantage_groups: bool = False
    value_loss_coef: float = 0.0


def linear_decay_coef(current_step: int, max_step: int, initial_coef: float, final_coef: float) -> float:
    return initial_coef + (final_coef - initial_coef) * current_step / max_step


# ---------------------------------------------------------------------------------------
# autograd bridges into libprl
# ---------------------------------------------------------------------------------------
def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{what} must be a CUDA tensor: pipelinerl_b200 has no CPU fallback")


class _LogprobTail(torch.autograd.Function):
    """logits [T, V] fp32 -> (new_logprobs [T-1], entropy [T-1]); csrc/logprob_tail.cu."""

    @staticmethod
    def forward(ctx, logits, input_ids, temperature: float):
        _require_cuda(logits, "logits")
        lib = _lib.load()
        if logits.dtype != torch.float32:
            logits = logits.float()
        if logits.stride(-1) != 1:
            logits = logits.contiguous()
        T, V = logits.shape
        ids = input_ids.contiguous()
        new_lp = torch.empty(max(T - 1, 0), dtype=torch.float32, device=logits.device)
        ent = torch.empty_like(new_lp)
        lse = torch.empty_like(new_lp)
        _lib.check(lib.prl_logprob_tail_fwd(logits.data_ptr(), T, V, logits.stride(0), ids.data_ptr(),
                                            float(temperature), new_lp.data_ptr(), ent.data_ptr(), lse.data_ptr(),
                                            _lib.stream_ptr()))
        ctx.save_for_backward(logits, ids, lse, ent)
        ctx.temperature = float(temperature)
        return new_lp, ent

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        logits, ids, lse, ent = ctx.saved_tensors
        lib = _lib.load()
        T, V = logits.shape
        dlogits = torch.empty((T, V), dtype=torch.float32, device=logits.device)
        g_lp = g_lp.contiguous() if g_lp is not None else None
        g_ent = g_ent.contiguous() if g_ent is not None else None
        _lib.check(lib.prl_logprob_tail_bwd(logits.data_ptr(), T, V, logits.stride(0), ids.data_ptr(), ctx.temperature,
                                            lse.data_ptr(), ent.data_ptr(),
                                            g_lp.data_ptr() if g_lp is not None else None,
                                            g_ent.data_ptr() if g_ent is not None else None,
                                            dlogits.data_ptr(), dlogits.stride(0), _lib.stream_ptr()))
        return dlogits, None, None


_WS_CACHE: dict[tuple[int, int], torch.Tensor] = {}


def _pg_workspace(device: torch.device, n_segments: int) -> torch.Tensor:
    lib = _lib.load()
    bucket = max(64, 1 << max(0, n_segments - 1).bit_length())
    key = (device.index if device.index is not None else torch.cuda.current_device(), bucket)
    ws = _WS_CACHE.get(key)
    if ws is None:
        ws = torch.zeros(int(lib.prl_pg_workspace_bytes(bucket)), dtype=torch.uint8, device=device)
        _WS_CACHE[key] = ws
    return ws


class _PgLoss(torch.autograd.Function):
    """(new_logprobs, entropy) -> loss, with the gradient produced by the same kernel launch."""

    @staticmethod
    def forward(ctx, new_lp, entropy, row: dict, cfg_struct, meta: dict):
        lib = _lib.load()
        dev = new_lp.device
        T = int(meta["T"])
        new_lp = new_lp.contiguous()
        entropy = entropy.contiguous() if entropy is not None else None
        out = torch.empty(2 + max(T - 1, 0) * 2, dtype=torch.float32, device=dev)  # loss | pad | dlp | dent
        loss = out[0:1]
        dlp = out[2:2 + max(T - 1, 0)]
        dent = out[2 + max(T - 1, 0):]
        stats = torch.empty(_lib.PRL_NUM_STATS, dtype=torch.float64, device=dev)
        flags = torch.empty(1, dtype=torch.int32, device=dev)
        b = _lib.PgBatch()
        b.T = T
        b.new_logprobs = new_lp.data_ptr()
        b.entropy = entropy.data_ptr() if entropy is not None else None
        for name in ("labels", "rewards", "advantages", "ref_logprobs", "old_logprobs", "group_tokens", "num_labels",
                     "overflow"):
            setattr(b, name, row[name].data_ptr())
        seg = row.get("segment_ids")
        b.segment_ids = seg.data_ptr() if seg is not None else None
        pos = row.get("position_ids")
        b.position_ids = pos.data_ptr() if pos is not None else None
        b.n_segments = int(meta["n_segments"])
        b.num_sequences = int(meta["num_sequences"])
        b.sentinel = int(bool(meta["sentinel"]))
        ws = _pg_workspace(dev, b.n_segments)
        sp_group = meta.get("seq_parallel_group")
        if sp_group is not None and cfg_struct.policy_loss == _lib.LOSS_IDS["gspo"] and b.n_segments > 0:
            # GSPO is a per-SEQUENCE objective and the sequence is spread over the group: all-reduce the per-segment sums
            # (reference rl/utils.py:194-206), then every rank differentiates the whole-sequence terms w.r.t. ITS tokens
            import torch.distributed as dist
            seg = torch.empty(b.n_segments, 4, dtype=torch.float64, device=dev)
            _lib.check(lib.prl_pg_gspo_segment_sums(C.byref(b), C.byref(cfg_struct), seg.data_ptr(), _lib.stream_ptr()))
            local_count = seg[:, 2].contiguous()
            dist.all_reduce(seg, op=dist.ReduceOp.SUM, group=sp_group)
            _lib.check(lib.prl_pg_loss_fwd_bwd_seg(C.byref(b), C.byref(cfg_struct), loss.data_ptr(), dlp.data_ptr(),
                                                   dent.data_ptr(), stats.data_ptr(), flags.data_ptr(), ws.data_ptr(),
                                                   ws.numel(), seg.data_ptr(), local_count.data_ptr(), _lib.stream_ptr()))
        else:
            _lib.check(lib.prl_pg_loss_fwd_bwd(C.byref(b), C.byref(cfg_struct), loss.data_ptr(), dlp.data_ptr(),
                                               dent.data_ptr(), stats.data_ptr(), flags.data_ptr(), ws.data_ptr(),
                                               ws.numel(), _lib.stream_ptr()))
        ctx.save_for_backward(dlp, dent)
        ctx.has_entropy = entropy is not None
        ctx.mark_non_differentiable(stats, flags)
        return loss.reshape(()).clone(), stats, flags

    @staticmethod
    def backward(ctx, g_loss, _g_stats, _g_flags):
        dlp, dent = ctx.saved_tensors
        g_new = g_loss * dlp
        g_ent = (g_loss * dent) if ctx.has_entropy else None
        return g_new, g_ent, None, None, None


def _cfg_struct(config: RLConfig, current_step: int, max_step: int) -> tuple[_lib.PgConfig, float, float]:
    if config.policy_loss not in _lib.LOSS_IDS:
        raise ValueError(f"Unknown algorithm {config.policy_loss}")
    ent_coef = linear_decay_coef(current_step, max_step, config.entropy_bonus, config.final_entropy_bonus)
    kl_coef = linear_decay_coef(current_step, max_step, config.kl_coef, config.final_kl_coef)
    c = _lib.PgConfig()
    c.policy_loss = _lib.LOSS_IDS[config.policy_loss]
    c.use_advantages = int(config.use_advantages)
    c.relu_log_p_weights = int(config.relu_log_p_weights)
    c.group_normalization = int(config.group_normalization)
    c.overlong_filtering = int(config.overlong_filtering)
    c.use_entropy_loss = int(config.entropy_bonus != 0.0 or config.final_entropy_bonus != 0.0)
    c.epsilon_low = config.epsilon_low
    c.epsilon_high = config.epsilon_high
    c.clamp_log_ratio_ref_new_value = config.clamp_log_ratio_ref_new_value
    c.kl_coef = kl_coef
    c.entropy_bonus_coef = ent_coef
    c.batch_size = float(config.batch_size)
    return c, kl_coef, ent_coef


_NONFINITE_MSG = {1: "new_logprobs is not finite", 2: "log_ratio_ref_new is not finite", 4: "approx_kl is not finite",
                  8: "Non-finite loss detected"}
_MIN_KEYS = [k for k in _lib.STAT_NAMES if k.startswith("min_")]
_MAX_KEYS = [k for k in _lib.STAT_NAMES if k.startswith("max_")]


def rl_step(model, batch: PipelineBatchEncoding, current_step: int, max_step: int, config: RLConfig,
            seq_parallel_group=None) -> tuple[torch.Tensor, dict[str, float]]:
    """One RL micro-batch: forward, PG loss (with its gradient staged for backward) and statistics.

    `model` is either any module whose output has `.logits` (the reference contract,
    rl/__init__.py:190-207) or a pipelinerl_b200 model exposing
    `forward_logprobs(batch, temperature) -> (new_logprobs[B, L-1], entropy[B, L-1])`, in which case
    full-vocabulary logits never reach HBM.
    """
    if seq_parallel_group is not None:
        # The batch is this rank's slice of a packed row (PipelineBatchEncoding.make_slices); like the reference, logits
        # and labels are shifted INSIDE the slice (rl/__init__.py:207-212 on the sliced batch), so the last token of a
        # slice predicts nothing.  Everything but attention is token-local; the model exchanges K / V itself.
        if not hasattr(model, "set_sequence_parallel"):
            raise NotImplementedError("seq_parallel_group needs a model that exchanges K / V over the group "
                                      "(pipelinerl_b200.learner_model.NativeQwen2)")
        if not batch.is_packed:
            raise ValueError("sequence parallelism slices PACKED rows")
        model.set_sequence_parallel(seq_parallel_group)
    if hasattr(model, "value_head"):
        raise NotImplementedError("value-head models are out of scope (GRPO path has no critic)")
    _require_cuda(batch.input_ids, "batch")
    if config.policy_loss == "gspo" and not batch.is_packed:
        raise ValueError("GSPO loss requires packed sequences with segments")
    if not config.group_normalization and config.batch_size <= 0:
        raise ValueError("RLConfig.batch_size must be set (token weights are 1/batch_size)")

    cfg_struct, kl_coef, ent_coef = _cfg_struct(config, current_step, max_step)
    B, L = batch.input_ids.shape

    if hasattr(model, "forward_logprobs") and getattr(model, "use_fused_head", True):
        new_lp_all, ent_all = model.forward_logprobs(batch, config.temperature)
        logits = None
    else:
        inputs = {"input_ids": batch.input_ids, "attention_mask": batch.attention_mask, "labels": batch.labels}
        if batch.is_packed:
            inputs["position_ids"] = batch.position_ids
        if batch.pixel_values is not None:
            inputs["pixel_values"] = batch.pixel_values
        if batch.image_grid_thw is not None:
            inputs["image_grid_thw"] = batch.image_grid_thw
        logits = model(**inputs).logits
        new_lp_all = ent_all = None

    total = None
    merged: np.ndarray | None = None
    flag_parts = []
    stat_parts = []
    for r in range(B):
        if logits is not None:
            new_lp, ent = _LogprobTail.apply(logits[r], batch.input_ids[r], config.temperature)
        else:
            new_lp, ent = new_lp_all[r], ent_all[r]
        row = {k: getattr(batch, k)[r].contiguous() for k in
               ("labels", "rewards", "advantages", "ref_logprobs", "old_logprobs", "group_tokens", "num_labels",
                "overflow")}
        n_seg = 0
        if batch.is_packed:
            row["position_ids"] = batch.position_ids[r].contiguous()
            if config.policy_loss == "gspo":
                if batch.segment_ids is None:
                    raise ValueError("segment_ids must be provided for per-segment reductions")
                row["segment_ids"] = batch.segment_ids[r].contiguous()
                # shape-only upper bound on max(segment_ids)+1: no device sync (empty segments are inert)
                n_seg = int(batch.seq_boundaries.numel()) - 1 if batch.seq_boundaries is not None else L
        meta = {"T": L, "n_segments": n_seg, "num_sequences": B, "sentinel": batch.sentinel,
                "seq_parallel_group": seq_parallel_group}
        loss_r, stats_r, flags_r = _PgLoss.apply(new_lp, ent, row, cfg_struct, meta)
        total = loss_r if total is None else total + loss_r
        stat_parts.append(stats_r)
        flag_parts.append(flags_r)

    # the only device->host synchronisation of the step
    host = torch.cat([torch.stack(stat_parts).reshape(-1),
                      torch.cat(flag_parts).to(torch.float64)]).cpu().numpy()
    per_row = host[: B * _lib.PRL_NUM_STATS].reshape(B, _lib.PRL_NUM_STATS)
    flags = 0
    for f in host[B * _lib.PRL_NUM_STATS:]:
        flags |= int(f)
    for bit, msg in _NONFINITE_MSG.items():
        if flags & bit:
            raise _lib.NonFiniteError(msg)

    idx = {k: i for i, k in enumerate(_lib.STAT_NAMES)}
    n_out = per_row[:, idx["num_output_tokens_sum"]].sum()
    if int(n_out) == 0:
        return total, {"input_size": float(batch.input_ids.numel())}
    live = per_row[per_row[:, idx["num_output_tokens_sum"]] > 0]
    merged = live.sum(axis=0)
    stats = {k: float(merged[i]) for k, i in idx.items()}
    for k in _MIN_KEYS:
        stats[k] = float(live[:, idx[k]].min())
    for k in _MAX_KEYS:
        stats[k] = float(live[:, idx[k]].max())
    loss_value = float(per_row[:, idx["loss"]].sum())
    stats["loss"] = stats["max_loss"] = stats["min_loss"] = loss_value
    # kl_coef / entropy_bonus_coef are reported as num_sequences * coef (:435-436); rows of one batch
    # share num_sequences, so take the first live row rather than the sum
    stats["kl_coef"] = float(live[0, idx["kl_coef"]])
    stats["entropy_bonus_coef"] = float(live[0, idx["entropy_bonus_coef"]])
    stats["input_size"] = float(batch.input_ids.numel())
    return total, stats


# ---------------------------------------------------------------------------------------
# host-side preparation of the RL columns (the preprocessor calls these)
# ---------------------------------------------------------------------------------------
def prepare_rl_fields(encoding: dict[str, Any], reward: float, old_logprobs: list[float],
                      ref_logprobs: list[float]) -> dict[str, Any]:
    """Per-token reward / logprob columns for one sample (reference: rl/__init__.py:573-594).
    Logprobs are right-aligned to the labelled (generated) tokens, zeros over the prompt."""
    labels = encoding["labels"]
    n = len(labels)
    n_target = n - labels.count(IGNORE_INDEX) if isinstance(labels, list) else int(np.sum(np.asarray(labels) != IGNORE_INDEX))
    assert n_target == len(old_logprobs), f"Target tokens: {n_target}, old logprobs: {len(old_logprobs)}"
    encoding["rewards"] = [reward] * n
    encoding["advantages"] = [0.0] * n
    encoding["old_logprobs"] = [0] * (n - len(old_logprobs)) + list(old_logprobs)
    encoding["ref_logprobs"] = [0] * (n - len(ref_logprobs)) + list(ref_logprobs)
    encoding["overflow"] = [0] * n
    encoding["group_tokens"] = [0] * n
    encoding["num_labels"] = [0 if x == IGNORE_INDEX else 1 for x in labels]
    return encoding


def _overflow_flag(entry: dict[str, Any], eos_token_id: int) -> float:
    reason = entry.get("finish_reason")
    if isinstance(reason, str):
        reason = reason.strip().lower()
        if reason == "length":
            return 1.0
        if reason in ("stop", "content_filter"):
            return 0.0
    if entry.get("finished"):
        return 0.0
    return 0.0 if eos_token_id in entry["input_ids"] else 1.0


def populate_rl_data(dataset: list[dict[str, Any]], eos_token_id: int, config: RLConfig) -> list[dict[str, Any]]:
    """Leave-one-out advantages per (group, step), mean rollout length per group, overflow and label
    counts — same results as the reference's pandas pipeline (rl/__init__.py:453-570), computed with
    dictionaries and numpy in O(n)."""
    n = len(dataset)
    if n == 0:
        return dataset
    lengths = [len(e["input_ids"]) for e in dataset]
    rollout_tokens: dict[tuple, int] = {}
    for e, ln in zip(dataset, lengths):
        key = (e["group_id"], e["rollout_index"])
        rollout_tokens[key] = rollout_tokens.get(key, 0) + ln
    g_sum: dict[Any, int] = {}
    g_cnt: dict[Any, int] = {}
    for (g, _), tok in rollout_tokens.items():
        g_sum[g] = g_sum.get(g, 0) + tok
        g_cnt[g] = g_cnt.get(g, 0) + 1

    # pandas' groupby kernels, restated: `sum` is Kahan-compensated, `std` is Welford's recurrence with ddof = 1, both over
    # the rows in dataset order (bit-identical doubles for any group size, tests/test_oracle_golden.py)
    acc: dict[tuple, list] = {}
    for e in dataset:
        v = float(e["rewards"][0])
        a = acc.setdefault((e["group_id"], e["step_index"]), [0.0, 0.0, 0, 0.0, 0.0])   # sum, comp, n, mean, m2
        y = v - a[1]
        t = a[0] + y
        a[1] = t - a[0] - y
        if a[1] != a[1]:
            a[1] = 0.0
        a[0] = t
        a[2] += 1
        old = a[3]
        a[3] += (v - old) / a[2]
        a[4] += (v - a[3]) * (v - old)
    step_stat = {}
    for key, (total, _comp, cnt, _mean, m2) in acc.items():
        std = math.sqrt(m2 / (cnt - 1)) if cnt > 1 else 0.0     # pandas gives NaN for one member -> nan_to_num -> 0
        step_stat[key] = (total, cnt, 0.0 if math.isnan(std) else std)

    for e, ln in zip(dataset, lengths):
        total, cnt, std = step_stat[(e["group_id"], e["step_index"])]
        r0 = e["rewards"][0]
        baseline = (total - r0) / (cnt - 1) if cnt > 1 else r0
        if config.divide_advantage_by_std:
            scale = std + 1e-4
            e["advantages"] = [(r - baseline) / scale for r in e["rewards"]]
        else:
            e["advantages"] = [(r - baseline) for r in e["rewards"]]
        e["overflow"] = [_overflow_flag(e, eos_token_id)] * len(e["overflow"])
        e["group_tokens"] = [g_sum[e["group_id"]] / g_cnt[e["group_id"]]] * ln
        labels = e["labels"]
        n_lab = len(labels) - labels.count(IGNORE_INDEX) if isinstance(labels, list) \
            else int(np.sum(np.asarray(labels) != IGNORE_INDEX))
        e["num_labels"] = [n_lab] * ln
    return dataset

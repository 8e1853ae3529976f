"""Checkpoint / resume of the learner in safetensors (SURVEY §8 f4; reference: pipelinerl/finetune/checkpoints.py).

Same entry points and on-disk discipline as the reference:
  save_model_only(output_dir, ...)            :388-445   HF-named weights a sampler / HF / vLLM can load
  save_training_state(dir, model, optimizer, lr_scheduler, extra_training_state)    :225-278
  load_training_checkpoint(dir, model, optimizer, lr_scheduler) -> extra_training_state   :281-329
  get_temporary_folder_and_move(output_dir)   :332-366   write into a temp sibling, then one rename: a crash never leaves
                                                         a half-written checkpoint where the trainer would resume from
What differs is the content: no DeepSpeed engine state or pickled `training_state.pt` -- the optimizer IS three flat fp32
arenas (master weights, exp_avg, exp_avg_sq; finetune/optim.py), stored as three safetensors tensors next to a small JSON
with the step counters, the LR schedule position and the caller's `extra_training_state` (completed_steps, samples, ...).
Model weights are written under their HF names from the bf16 arena through the fused -> HF row slices of model.py
(the inverse of vLLM's `load_weights` mapping at vllm1.py:122), so `model.safetensors` + `config.json` is a directory the
reference's own `load_model` (checkpoints.py:151-222) or a vLLM server can open.
"""
from __future__ import annotations

import contextlib
import json
import os
import shutil
from pathlib import Path
from typing import Any

import torch

from ..model import ArenaLayout, ModelConfig

TRAINING_STATE_FILE = "training_state.json"
OPTIMIZER_FILE = "optimizer.safetensors"


@contextlib.contextmanager
def get_temporary_folder_and_move(output_dir: Path):
    """write into `<output_dir>~temp`, then swap it in with renames (the reference's discipline, :332-366)"""
    output_dir = Path(output_dir)
    temp = output_dir.with_name(output_dir.name + "~temp")
    if temp.exists():
        shutil.rmtree(temp)
    temp.mkdir(parents=True)
    try:
        yield temp
    except BaseException:
        shutil.rmtree(temp, ignore_errors=True)
        raise
    old = None
    if output_dir.exists():
        old = output_dir.with_name(output_dir.name + "~old")
        if old.exists():
            shutil.rmtree(old)
        os.replace(output_dir, old)
    os.replace(temp, output_dir)
    if old is not None:
        shutil.rmtree(old, ignore_errors=True)


def hf_config_dict(cfg: ModelConfig) -> dict[str, Any]:
    """config.json of the checkpoint: Qwen2ForCausalLM, Qwen3ForCausalLM for q/k-norm configs, or LlamaForCausalLM
    (ModelConfig.from_hf_config reads it back)."""
    if cfg.family == "llama":
        return {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "vocab_size": cfg.vocab_size,
                "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
                "num_hidden_layers": cfg.num_layers, "num_attention_heads": cfg.num_q_heads,
                "num_key_value_heads": cfg.num_kv_heads, "head_dim": cfg.head_dim, "hidden_act": "silu",
                "rms_norm_eps": cfg.rms_eps, "rope_theta": cfg.rope_theta,
                "rope_scaling": cfg.rope_scaling.hf_dict() if cfg.rope_scaling is not None else None,
                "tie_word_embeddings": cfg.tie_word_embeddings, "torch_dtype": "bfloat16", "attention_bias": False,
                "mlp_bias": False}
    if cfg.qk_norm:
        d = {"architectures": ["Qwen3ForCausalLM"], "model_type": "qwen3"}
    else:
        d = {"architectures": ["Qwen2ForCausalLM"], "model_type": "qwen2"}
    d.update({"vocab_size": cfg.vocab_size,
              "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size, "num_hidden_layers": cfg.num_layers,
              "num_attention_heads": cfg.num_q_heads, "num_key_value_heads": cfg.num_kv_heads, "head_dim": cfg.head_dim,
              "hidden_act": "silu", "rms_norm_eps": cfg.rms_eps, "rope_theta": cfg.rope_theta,
              "tie_word_embeddings": cfg.tie_word_embeddings, "torch_dtype": "bfloat16"})
    if not cfg.qk_norm:
        d["attention_bias"] = cfg.qkv_bias
    elif cfg.qkv_bias:      # Qwen3Config's default is False
        d["attention_bias"] = True
    d["use_sliding_window"] = False
    return d


def _hf_tensors(cfg: ModelConfig, fused: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    out = {}
    for hf_name, (name, r0, rn) in ArenaLayout.build(cfg).hf_slices().items():
        out[hf_name] = fused[name][r0:r0 + rn].detach().to("cpu").contiguous()
    return out


def save_model_only(output_dir: Path, cfg: ModelConfig, named_parameters, dtype: torch.dtype = torch.bfloat16) -> None:
    """`named_parameters`: (fused name, tensor) pairs -- a learner module's named_parameters() or an arena's views.  A
    tied config writes no `lm_head.weight` (config.json says tie_word_embeddings), as HF saves a tied model."""
    from safetensors.torch import save_file
    fused = {n: (p.data if hasattr(p, "data") else p).to(dtype) for n, p in named_parameters}
    with get_temporary_folder_and_move(Path(output_dir)) as tmp:
        save_file(_hf_tensors(cfg, fused), str(tmp / "model.safetensors"), metadata={"format": "pt"})
        (tmp / "config.json").write_text(json.dumps(hf_config_dict(cfg), indent=1))


def load_model_weights(model_dir: Path, cfg: ModelConfig) -> dict[str, torch.Tensor]:
    """HF-named safetensors -> fused name -> tensor (rows of q/k/v and gate/up concatenated: vllm1.py:122's mapping)."""
    from safetensors.torch import load_file
    sd = load_file(str(Path(model_dir) / "model.safetensors"))
    slices = ArenaLayout.build(cfg).hf_slices()
    missing = set(slices) - set(sd)
    if missing:
        raise KeyError(f"checkpoint lacks {sorted(missing)[:4]} ...")
    parts: dict[str, list] = {}
    for hf_name, (name, r0, rn) in slices.items():
        parts.setdefault(name, []).append((r0, sd[hf_name]))
    return {name: torch.cat([t for _, t in sorted(ps, key=lambda x: x[0])]) if len(ps) > 1 else ps[0][1]
            for name, ps in parts.items()}


def save_training_state(training_state_dir: Path, model, optimizer, lr_scheduler,
                        extra_training_state: dict[str, Any] | None = None) -> None:
    """model is accepted for signature parity (its weights ARE optimizer.master / optimizer.shadow_bf16)."""
    from safetensors.torch import save_file
    sd = optimizer.state_dict()
    with get_temporary_folder_and_move(Path(training_state_dir)) as tmp:
        save_file({k: sd[k].detach().to("cpu").contiguous() for k in ("master", "exp_avg", "exp_avg_sq")},
                  str(tmp / OPTIMIZER_FILE), metadata={"format": "pt"})
        state = {"optimizer": {"step": int(sd["step"]), "names": list(sd["names"]), "offsets": [int(o) for o in sd["offsets"]],
                               "lr": float(optimizer.param_groups[0]["lr"])},
                 "lr_scheduler_state": {"last_step": int(lr_scheduler.last_step), "kind": lr_scheduler.kind,
                                        "base_lrs": [float(x) for x in lr_scheduler.base_lrs]} if lr_scheduler is not None else None,
                 "extra_training_state": dict(extra_training_state or {})}
        (tmp / TRAINING_STATE_FILE).write_text(json.dumps(state, indent=1))


def load_training_checkpoint(training_state_dir: Path, model, optimizer, lr_scheduler) -> dict[str, Any]:
    """Restores optimizer arenas (and through them the parameters: the bf16 arena is re-cast from the fp32 master) and
    the LR schedule position in place; returns the extra_training_state that was saved."""
    from safetensors.torch import load_file
    d = Path(training_state_dir)
    state = json.loads((d / TRAINING_STATE_FILE).read_text())
    o = state["optimizer"]
    if list(o["names"]) != list(optimizer.names) or [int(x) for x in o["offsets"]] != [int(x) for x in optimizer.offsets]:
        raise ValueError("checkpoint was written for a different parameter layout")
    t = load_file(str(d / OPTIMIZER_FILE))
    optimizer.load_state_dict({"step": o["step"], "master": t["master"], "exp_avg": t["exp_avg"], "exp_avg_sq": t["exp_avg_sq"]})
    if lr_scheduler is not None and state.get("lr_scheduler_state"):
        ls = state["lr_scheduler_state"]
        lr_scheduler.base_lrs = list(ls["base_lrs"])
        lr_scheduler.last_step = int(ls["last_step"])
        lr_scheduler._apply()
    return state["extra_training_state"]

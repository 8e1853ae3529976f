"""Golden fixtures for hot path 2 on Qwen3 and Llama 3: the reference's own `rl_step` (pipelinerl/finetune/rl/__init__.py)
driving HF transformers' `Qwen3ForCausalLM` / `LlamaForCausalLM` (llama3 RoPE scaling), fp32 on CPU, on one packed
micro-batch, for the Qwen3 and Llama cases of tests/model_cases.py -- the twin of make_golden_learner.py (same packing,
same block-diagonal mask wrapper, same gradient summary).  Recorded: loss, the 32 statistics, the per-token new logprobs
and the gradient of EVERY parameter, q_norm / k_norm gains included.  The HF model is built untied for every case: the
learner trains lm_head and embed_tokens as separate tensors (a tied checkpoint is loaded untied).

    python tests/golden/make_golden_learner_qwen3_llama.py      (authoring container: needs the reference + transformers)

Weights are NOT stored (tests regenerate them with the case's `weights`).
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import _Tok, _import_reference, batch_to_np, make_samples, preprocess_like_reference  # noqa: E402
from make_golden_learner import PackedHF, sample_idx  # noqa: E402
from pipelinerl_b200.model import ArenaLayout  # noqa: E402
from tests.model_cases import CASES, hf_model  # noqa: E402

OUT = Path(__file__).resolve().parent
PPO = dict(policy_loss="ppo", kl_coef=0.1, final_kl_coef=0.02, entropy_bonus=0.01, final_entropy_bonus=0.001,
           epsilon_low=0.2, epsilon_high=0.3, batch_size=16, clamp_log_ratio_ref_new_value=1.5)
GSPO = dict(policy_loss="gspo", kl_coef=0.0, final_kl_coef=0.0, epsilon_low=0.05, epsilon_high=0.05, batch_size=8)
RL_CONFIGS = {"qwen3_wide": PPO, "qwen3_gqa4": GSPO, "llama_scaled": PPO, "llama_tied": GSPO}


def main():
    ref_rl, ref_data, ref_utils = _import_reference()
    for name, cfgd in RL_CONFIGS.items():
        case = CASES[name]
        cfg = case["cfg"]
        w = case["weights"](cfg)
        hf = hf_model(cfg, w).train()
        slices = ArenaLayout.build(cfg).hf_slices()
        model = PackedHF(hf)

        rng = np.random.default_rng(700 + len(name.split("_", 1)[1]))
        torch.manual_seed(700)
        rcfg = ref_rl.RLConfig(**cfgd)
        samples = make_samples(rng, n_groups=2, attempts=4, vocab=cfg.vocab_size, max_prompt=14, max_gen=30)
        entries = preprocess_like_reference(ref_rl, ref_data, samples, rcfg)
        batch = ref_data.collate_packed(entries, _Tok(), seq_parallel=1)
        T = batch.input_ids.shape[1]
        with torch.no_grad():   # old / ref logprobs near the model's own, so both sides of the clip are exercised
            lg = model(input_ids=batch.input_ids, attention_mask=batch.attention_mask, position_ids=batch.position_ids).logits
            lp = torch.log_softmax(lg[0, :-1] / rcfg.temperature, -1).gather(1, batch.input_ids[0, 1:, None])[:, 0]
            batch.old_logprobs[0, 1:] = lp + 0.05 * torch.randn(T - 1)
            batch.ref_logprobs[0, 1:] = lp + 0.3 * torch.randn(T - 1)
        cur, mx = 3, 10
        loss, stats = ref_rl.rl_step(model, batch, cur, mx, rcfg)
        loss.backward()
        arrs = batch_to_np(batch)
        arrs["loss"] = np.float64(loss.item())
        arrs["new_logprobs"] = lp.numpy()
        grads = {}
        params = dict(hf.named_parameters())
        for hf_name, (fused, r0, rn) in slices.items():
            grads.setdefault(fused, torch.zeros_like(w[fused]))
            grads[fused][r0:r0 + rn] = params[hf_name].grad
        for fused, g in grads.items():
            flat = g.reshape(-1).double()
            key = fused.replace(".", "__")
            arrs["gnorm__" + key] = np.float64(flat.norm().item())
            arrs["gsamp__" + key] = flat[torch.from_numpy(sample_idx(flat.numel()))].numpy()
        np.savez_compressed(OUT / f"{case['learner']}.npz", **arrs)
        meta = {"config": rcfg.model_dump(), "current_step": cur, "max_step": mx,
                "stats": {k: float(v) for k, v in stats.items()}, "model": name, "T": int(T)}
        (OUT / f"{case['learner']}.json").write_text(json.dumps(meta, indent=1, sort_keys=True))
        tot = float(torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())))
        qk = {n: float(g.norm()) for n, g in grads.items() if n.endswith(("q_norm.weight", "k_norm.weight"))}
        print(name, "T", T, "loss", loss.item(), "total grad norm", tot, "q/k gain grad norms", qk)


if __name__ == "__main__":
    main()

"""Golden fixtures for tied word embeddings trained tied, for the cases of tests/tied_cases.py (the Qwen2 "gqa2", Qwen3
"wide" and Llama "tied" configurations with `tie_word_embeddings=True`; their arenas have no lm_head and their weights
are those of the untied cases minus the head, seed 42).

learner_step_tied_{qwen2,qwen3,llama}.npz/.json: the reference's own `rl_step` (pipelinerl/finetune/rl/__init__.py)
driving HF `Qwen2ForCausalLM` / `Qwen3ForCausalLM` / `LlamaForCausalLM` built with `tie_word_embeddings=True`, fp32 on
CPU, on one packed micro-batch, with the packing, mask wrapper and gradient summary of make_golden_learner.py.  A tied HF
model has one parameter for both uses, so there is no lm_head entry and the gradient of `model.embed_tokens.weight` is the
sum of the head's and the embedding's.  Recorded: loss, the 32 statistics, the per-token new logprobs and the norm and a
257-point sample of the gradient of every parameter.  PPO with KL and entropy on the Qwen2 and Llama cases, GSPO on the
Qwen3 case.

qwen2_tiny_tied.npz, qwen3_tiny_tied.npz: the tied HF Qwen2 / Qwen3 models in fp32, with the fields and lengths of the
Qwen3 decode fixtures of make_golden_qwen3_llama.py (teacher-forced logprobs of a 150-token sequence at T = 0.7, the last
4 logits rows, greedy continuations of 24 tokens with T = 1 logprobs and top-2 margins for 4 prompts).  The Llama case
replays llama_tiny_tied.npz, which is tied already.

    python tests/golden/make_golden_learner_tied.py      (authoring container: needs the reference + transformers)

Weights are NOT stored (tests regenerate them with the case's `weights`).
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import _Tok, _import_reference, batch_to_np, make_samples, preprocess_like_reference  # noqa: E402
from make_golden_learner import PackedHF, sample_idx  # noqa: E402
from make_golden_learner_qwen3_llama import GSPO, PPO  # noqa: E402
from make_golden_qwen3_llama import LENGTHS, N_NEW  # noqa: E402
from pipelinerl_b200.model import ArenaLayout  # noqa: E402
from tests.tied_cases import TIED_CASES, hf_tied_model  # noqa: E402

OUT = Path(__file__).resolve().parent
RL_CONFIGS = {"tied_qwen2": PPO, "tied_qwen3": GSPO, "tied_llama": PPO}


def record_decode(name, n_tokens, prompt_lens):
    case = TIED_CASES[name]
    cfg = case["cfg"]
    model = hf_tied_model(cfg, case["weights"](cfg)).eval()
    g = torch.Generator().manual_seed(7)
    tokens = torch.randint(0, cfg.vocab_size, (n_tokens,), generator=g)
    temp = 0.7
    with torch.no_grad():
        logits = model(input_ids=tokens[None]).logits[0].float()
    lp = torch.log_softmax(logits[:-1] / temp, -1).gather(1, tokens[1:, None])[:, 0]
    gp = torch.Generator().manual_seed(11)
    prompts = np.zeros((len(prompt_lens), max(prompt_lens)), dtype=np.int64)
    ids = np.zeros((len(prompt_lens), N_NEW), dtype=np.int64)
    lps = np.zeros((len(prompt_lens), N_NEW), dtype=np.float32)
    margin = np.zeros((len(prompt_lens), N_NEW), dtype=np.float32)
    for i, n in enumerate(prompt_lens):
        seq = torch.randint(0, cfg.vocab_size, (n,), generator=gp)
        prompts[i, :n] = seq.numpy()
        for t in range(N_NEW):
            with torch.no_grad():
                last = model(input_ids=seq[None]).logits[0, -1].float()
            nxt = int(torch.argmax(last))
            top2 = torch.topk(last, 2).values
            ids[i, t], lps[i, t] = nxt, float(torch.log_softmax(last, -1)[nxt])
            margin[i, t] = float(top2[0] - top2[1])
            seq = torch.cat([seq, torch.tensor([nxt])])
    np.savez_compressed(case["decode"][0], tokens=tokens.numpy(), logprobs=lp.numpy(),
                        last_logits=logits[-4:].numpy(), temperature=np.float32(temp), prompts=prompts,
                        prompt_len=np.array(prompt_lens, dtype=np.int64), greedy_ids=ids, greedy_logprobs=lps,
                        greedy_margin=margin)
    print(name, "logprob mean", float(lp.mean()), "min greedy margin", float(margin.min()))


def record_learner(ref, name, cfgd, seed):
    ref_rl, ref_data, _ = ref
    case = TIED_CASES[name]
    cfg = case["cfg"]
    w = case["weights"](cfg)
    hf = hf_tied_model(cfg, w).train()
    slices = ArenaLayout.build(cfg).hf_slices()      # tied: no lm_head.weight
    model = PackedHF(hf)
    rng = np.random.default_rng(seed)
    torch.manual_seed(900)
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
    print(name, "T", T, "loss", loss.item(), "embedding gradient norm", float(grads["embed_tokens.weight"].norm()))


def main():
    for name in ("tied_qwen2", "tied_qwen3"):
        record_decode(name, *LENGTHS["qwen3"])
    ref = _import_reference()
    for i, (name, cfgd) in enumerate(RL_CONFIGS.items()):
        record_learner(ref, name, cfgd, 900 + i)


if __name__ == "__main__":
    main()

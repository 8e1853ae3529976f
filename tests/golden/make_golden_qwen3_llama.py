"""Golden fixtures for the Qwen3 and Llama 3 token step: HF transformers' Qwen3ForCausalLM / LlamaForCausalLM in fp32 on
bf16-valued weights, for the Qwen3 and Llama cases of tests/model_cases.py.

    python tests/golden/make_golden_qwen3_llama.py      (authoring container; needs transformers >= 4.51 only)

Weights are NOT stored: tests regenerate them with the case's `weights` (CPU torch RNG, seed 42; non-unit q/k gains for
Qwen3; lm_head a copy of embed_tokens for llama_tied, whose HF model ties them).  Stored per case, <family>_tiny_<kind>.npz:
  tokens / logprobs   teacher-forced log p(tokens[t+1] | tokens[:t+1]) of a fixed sequence (150 tokens for Qwen3, 320
                      for Llama) at T = 0.7
  last_logits         the full logits of its last 4 positions
  prompts / prompt_len, greedy_ids / greedy_logprobs / greedy_margin
                      HF greedy continuations (24 tokens, T = 1 logprobs, top-2 logit margin of every step) of 4 prompts
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
from tests.model_cases import CASES, GREEDY_CASES, hf_model  # noqa: E402

N_NEW = 24
# per family: length of the teacher-forced sequence, prompt lengths of the greedy continuations
LENGTHS = {"qwen3": (150, (5, 64, 130, 17)), "llama": (320, (5, 64, 230, 17))}


def main():
    for name in GREEDY_CASES:
        case = CASES[name]
        cfg = case["cfg"]
        n_tokens, prompt_lens = LENGTHS[name.split("_")[0]]
        model = hf_model(cfg, case["weights"](cfg), tied=case["tied"]).eval()
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
        print(name, "logprob mean", float(lp.mean()), "logit std", float(logits.std()),
              "min greedy margin", float(margin.min()))


if __name__ == "__main__":
    main()

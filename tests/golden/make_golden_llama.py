"""Golden fixtures for the Llama 3 token step: HF transformers' LlamaForCausalLM in fp32 on bf16-valued weights.

    python tests/golden/make_golden_llama.py      (authoring container; needs transformers only)

Weights are NOT stored: tests regenerate them with tests.llama_oracle.llama_tiny_weights (CPU torch RNG, seed 42).  Two
configurations (tests.llama_oracle.llama_tiny_cfg), both rope_theta 500 000 with llama3 RoPE scaling:
"scaled" (4 q / 2 kv heads, original_max_position_embeddings 64, so all three frequency bands are non-empty) and
"tied" (6 q / 2 kv heads, Llama-3.2-3B's 3:1 grouping, tie_word_embeddings=True).  Stored per configuration,
llama_tiny_<kind>.npz:
  tokens / logprobs   teacher-forced log p(tokens[t+1] | tokens[:t+1]) of a fixed 320-token sequence at T = 0.7
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
from tests.llama_oracle import LLAMA_KINDS, TIED, hf_llama_model, llama_tiny_cfg, llama_tiny_weights  # noqa: E402

N_NEW = 24
PROMPT_LENS = (5, 64, 230, 17)


def main():
    for kind in LLAMA_KINDS:
        cfg = llama_tiny_cfg(kind)
        model = hf_llama_model(cfg, llama_tiny_weights(cfg, kind), tied=TIED[kind]).eval()
        g = torch.Generator().manual_seed(7)
        tokens = torch.randint(0, cfg.vocab_size, (320,), generator=g)
        temp = 0.7
        with torch.no_grad():
            logits = model(input_ids=tokens[None]).logits[0].float()
        lp = torch.log_softmax(logits[:-1] / temp, -1).gather(1, tokens[1:, None])[:, 0]
        gp = torch.Generator().manual_seed(11)
        prompts = np.zeros((len(PROMPT_LENS), max(PROMPT_LENS)), dtype=np.int64)
        ids = np.zeros((len(PROMPT_LENS), N_NEW), dtype=np.int64)
        lps = np.zeros((len(PROMPT_LENS), N_NEW), dtype=np.float32)
        margin = np.zeros((len(PROMPT_LENS), N_NEW), dtype=np.float32)
        for i, n in enumerate(PROMPT_LENS):
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
        np.savez_compressed(Path(__file__).parent / f"llama_tiny_{kind}.npz", tokens=tokens.numpy(), logprobs=lp.numpy(),
                            last_logits=logits[-4:].numpy(), temperature=np.float32(temp), prompts=prompts,
                            prompt_len=np.array(PROMPT_LENS, dtype=np.int64), greedy_ids=ids, greedy_logprobs=lps,
                            greedy_margin=margin)
        print(kind, "logprob mean", float(lp.mean()), "logit std", float(logits.std()),
              "min greedy margin", float(margin.min()))


if __name__ == "__main__":
    main()

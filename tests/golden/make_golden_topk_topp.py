"""topk_topp_vllm.npz: vLLM 0.22's top-k / top-p truncation and processed logprobs on fixed logits.

Executes, per row, what vLLM's sampler does for a random request (v1/sample/sampler.py::Sampler.sample ->
TopKTopPSampler.forward_native under logprobs-mode processed_logprobs, conf/base.yaml:65):
    z = logits / T (fp32);  z = apply_top_k_top_p_pytorch(z, k, p);  processed logprobs = log_softmax(z)
Rows: V in {640, 1000, 152 064} x T in {0.6, 1.0, 1.3} x {top-k only 1, 20, 50, V-1, V; top-p only 1e-6, 0.5, 0.95;
both (50, 0.95)} x logits kinds {flat, peaked, ties at the 20th and 50th largest value}.  Stored per V: the logits (or,
for the large vocabulary, the seed they are regenerated from plus the SHA-256 of their bytes), the row parameters, the
kept mask packed to bits, and vLLM's processed logprobs at the (up to) 64 largest kept ids.

Run where vLLM imports (CPU is enough):  python tests/golden/make_golden_topk_topp.py
The tests regenerate the logits with `make_logits` below; they never import vLLM."""
from __future__ import annotations

import hashlib
from pathlib import Path

import numpy as np
import torch

OUT = Path(__file__).resolve().parent / "topk_topp_vllm.npz"
VOCABS = (640, 1000, 152064)
STORED_LOGITS_MAX_V = 1000          # larger vocabularies are stored as a seed + SHA-256
TEMPERATURES = (0.6, 1.0, 1.3)
KINDS = ("flat", "peaked", "ties")
N_LP = 64


def settings(V: int) -> list[tuple[int, float]]:
    """(top_k, top_p) per row; -1 / 1.0 = off"""
    return [(1, 1.0), (20, 1.0), (50, 1.0), (V - 1, 1.0), (V, 1.0), (-1, 1e-6), (-1, 0.5), (-1, 0.95), (50, 0.95)]


def make_logits(V: int, seed: int) -> torch.Tensor:
    """[3, V] fp32 logits: flat (N(0, 1)), peaked (N(0, 3) plus a few large spikes), and flat logits whose 16th..24th and
    45th..55th largest values are set equal to the 20th / 50th largest (ties exactly at the top-k boundary)."""
    g = torch.Generator().manual_seed(seed)
    flat = torch.randn(V, generator=g)
    peaked = torch.randn(V, generator=g) * 3.0
    spikes = torch.randint(0, V, (8,), generator=g)
    peaked[spikes] += torch.linspace(12.0, 5.0, 8)
    ties = torch.randn(V, generator=g)
    order = torch.argsort(ties, descending=True)
    ties[order[15:24]] = ties[order[19]].item()
    ties[order[44:55]] = ties[order[49]].item()
    return torch.stack([flat, peaked, ties]).float()


def seed_of(V: int) -> int:
    return 1000 + V


def logits_sha256(x: torch.Tensor) -> str:
    return hashlib.sha256(x.contiguous().numpy().tobytes()).hexdigest()


def main() -> None:
    from vllm.v1.sample.ops.topk_topp_sampler import apply_top_k_top_p_pytorch
    out: dict[str, np.ndarray] = {"vocabs": np.array(VOCABS, dtype=np.int64)}
    for V in VOCABS:
        logits = make_logits(V, seed_of(V))
        rows = [(ki, T, k, p) for ki in range(len(KINDS)) for T in TEMPERATURES for (k, p) in settings(V)]
        masks, lp_ids, lps = [], [], []
        for ki, T, k, p in rows:
            z = logits[ki:ki + 1].clone().div_(T)          # Sampler.apply_temperature: fp32 in-place division
            kt = torch.tensor([k], dtype=torch.long) if k > 0 else None
            pt = torch.tensor([p], dtype=torch.float32) if p < 1.0 else None
            z = apply_top_k_top_p_pytorch(z, kt, pt)
            lp = z.log_softmax(dim=-1, dtype=torch.float32)[0]
            keep = torch.isfinite(z[0])
            masks.append(np.packbits(keep.numpy()))
            kept_ids = torch.nonzero(keep).flatten()
            top = kept_ids[torch.argsort(logits[ki, kept_ids], descending=True, stable=True)[:N_LP]]
            ids = np.full(N_LP, -1, dtype=np.int32)
            vals = np.zeros(N_LP, dtype=np.float32)
            ids[:len(top)] = top.numpy()
            vals[:len(top)] = lp[top].numpy()
            lp_ids.append(ids)
            lps.append(vals)
        pre = f"V{V}_"
        if V <= STORED_LOGITS_MAX_V:
            out[pre + "logits"] = logits.numpy()
        out[pre + "seed"] = np.array(seed_of(V), dtype=np.int64)
        out[pre + "sha256"] = np.array(logits_sha256(logits))
        out[pre + "kind"] = np.array([r[0] for r in rows], dtype=np.int32)
        out[pre + "T"] = np.array([r[1] for r in rows], dtype=np.float64)
        out[pre + "top_k"] = np.array([r[2] for r in rows], dtype=np.int32)
        out[pre + "top_p"] = np.array([r[3] for r in rows], dtype=np.float64)
        out[pre + "mask"] = np.stack(masks)
        out[pre + "lp_ids"] = np.stack(lp_ids)
        out[pre + "lp"] = np.stack(lps)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()

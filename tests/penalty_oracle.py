"""numpy fp32 restatement of vLLM 0.22's penalties and min_p, and the fixture loader.

Per row, in vLLM's order (v1/sample/sampler.py), each step one fp32 rounding:
  mask = ids in the prompt | ids among the outputs;  counts = outputs per id (ids outside [0, V) are padding)
  repetition (masked ids):  l = l * (1 / r) if l > 0 else l * r          (1 / r rounded to fp32 first)
  frequency:                l = l - f * counts
  presence:                 l = l - pr * (counts > 0)
  then, for a random row with min_p > 0:  z = l / T;  drop i where softmax(z)_i < min_p * max softmax(z)
  then top-k / top-p on what is left (tests/topk_topp_oracle.py) and the processed logprobs of the rest.
Used by tests/test_penalties.py (against tests/golden/penalties_vllm.npz) and tests/test_gpu_penalties.py."""
from __future__ import annotations

import importlib.util
import json
from pathlib import Path

import numpy as np

from tests.topk_topp_oracle import truncated_logprobs

GOLDEN = Path(__file__).resolve().parent / "golden"
F32 = np.float32


def counts_and_mask(V: int, prompt_ids, output_ids) -> tuple[np.ndarray, np.ndarray]:
    """(output counts int64 [V], prompt | output mask bool [V])."""
    p = np.asarray(prompt_ids, dtype=np.int64)
    o = np.asarray(output_ids, dtype=np.int64)
    counts = np.bincount(o[(o >= 0) & (o < V)], minlength=V)
    mask = counts > 0
    mask[p[(p >= 0) & (p < V)]] = True
    return counts, mask


def apply_penalties(logits, prompt_ids, output_ids, presence: float, frequency: float, repetition: float) -> np.ndarray:
    """One row of vLLM's apply_penalties, in fp32."""
    l = np.array(logits, dtype=F32)
    counts, mask = counts_and_mask(l.shape[0], prompt_ids, output_ids)
    r = F32(repetition)
    scale = np.where(l > 0, F32(1) / r, r).astype(F32)
    l[mask] = l[mask] * scale[mask]
    l = l - F32(frequency) * counts.astype(F32)
    l = l - F32(presence) * (counts > 0).astype(F32)
    return l.astype(F32)


def min_p_keep(z, min_p: float) -> tuple[np.ndarray, np.ndarray]:
    """(kept bool [V], relative distance of each decision from its boundary) of MinPLogitsProcessor on z (fp32)."""
    z = np.asarray(z, dtype=F32)
    e = np.exp(z - z.max())
    prob = e / e.sum(dtype=F32)
    thr = prob.max() * F32(min_p)
    keep = ~(prob < thr)
    ratio = np.exp(z.astype(np.float64) - float(z.max()))            # p_i / max p, fp64
    return keep, np.abs(ratio - min_p) / max(min_p, 1e-30)


def processed_logprobs(penalized, T: float, min_p: float, top_k: int, top_p: float, greedy: bool):
    """(logprobs fp64 [V], -inf where dropped; min_p kept mask) of a penalized row."""
    l = np.asarray(penalized, dtype=F32)
    if greedy:
        z = l.astype(np.float64)
        return z - (z.max() + np.log(np.exp(z - z.max()).sum())), np.ones(l.shape[0], dtype=bool)
    z = (l / F32(T)).astype(F32)
    keep = np.ones(l.shape[0], dtype=bool)
    if min_p > 0:
        keep = min_p_keep(z, min_p)[0] | ~np.isfinite(z)
        z = np.where(keep, z, F32(-np.inf)).astype(F32)
    return truncated_logprobs(z, 1.0, top_k, top_p).logprobs, keep


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_penalties", GOLDEN / "make_golden_penalties.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_fixture() -> dict:
    """The npz's arrays, min_p_keep unpacked to bool [R, V], plus the generator module (`gen`) for the large rows and the
    JSON's validation list (`validation`).  prompt_ids / output_ids rows are padded with the id V, which every rule
    skips."""
    d = dict(np.load(GOLDEN / "penalties_vllm.npz"))
    V = int(d["V"])
    d["min_p_keep"] = np.unpackbits(d["min_p_keep"], axis=1, count=V).astype(bool)
    d["gen"] = _generator()
    d["validation"] = json.loads((GOLDEN / "penalties_vllm.json").read_text())["validation"]
    return d

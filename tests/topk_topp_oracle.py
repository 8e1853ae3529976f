"""fp64 restatement of vLLM's top-k / top-p truncation with processed logprobs, and the fixture loader.

vLLM 0.22 (v1/sample/ops/topk_topp_sampler.py::apply_top_k_top_p_pytorch, then log_softmax) for a random row:
  z = logits / T;  top-k (1 <= k < V): keep { z >= k-th largest z } (ties kept);
  top-p (p < 1): on that set S with M = sum_S e^z, keep i iff sum_{j in S, z_j > z_i} e^z_j < p M (the largest is kept);
  logprob = z - logsumexp(z over the kept set).
Used by tests/test_topk_topp.py (against tests/golden/topk_topp_vllm.npz) and tests/test_gpu_topk_topp.py."""
from __future__ import annotations

import importlib.util
from dataclasses import dataclass
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parent / "golden"


@dataclass
class Truncated:
    mask: np.ndarray        # [V] bool, kept tokens
    logprobs: np.ndarray    # [V] float64, -inf outside the kept set
    log_norm: float         # logsumexp(z over the kept set)
    threshold: float        # smallest kept z
    margin: float           # distance from a decision vLLM could take differently (inf when nothing is close)
    rule_margin: float      # distance of this rule's own decision from its boundary


def truncated_logprobs(logits, T: float, top_k: int, top_p: float) -> Truncated:
    """One row.  rule_margin = min(|mass_above(boundary)/M - p| over the last kept and the first dropped value (top-p),
    relative gap between the k-th largest value and the next smaller one (top-k)); margin also shrinks to <= 0 when
    vLLM's sort would split a tie group at the top-p boundary (this rule keeps every tie)."""
    z = np.asarray(logits, dtype=np.float64) / float(T)
    V = z.shape[0]
    uniq = np.unique(z)[::-1]                                    # distinct values, descending
    keep = np.ones(V, dtype=bool)
    margin = np.inf
    if 1 <= top_k < V:
        tau_k = np.sort(z)[::-1][top_k - 1]
        keep = z >= tau_k
        below = uniq[uniq < tau_k]
        if below.size:
            margin = min(margin, (tau_k - below[0]) / max(1.0, abs(tau_k)))
    if top_p < 1.0:
        zs = np.sort(z[keep])[::-1]
        neg, first = np.unique(-zs, return_index=True)          # distinct kept values, descending, and their counts
        vals, counts = -neg, np.diff(np.append(first, zs.size))
        e = np.exp(vals - vals[0]) * counts
        M = e.sum()
        above = np.concatenate([[0.0], np.cumsum(e)[:-1]]) / M  # mass strictly above each distinct value, / M
        kept_vals = above < top_p
        n_kept = int(np.count_nonzero(kept_vals))
        tau_p = vals[n_kept - 1]
        rule_margin = min(margin, top_p - above[n_kept - 1])
        if n_kept < vals.size:
            rule_margin = min(rule_margin, above[n_kept] - top_p)
        # vLLM's sorted cumsum orders the members of a tie group: all c of the boundary group are kept only if the mass
        # above its LAST member is still < p M (otherwise vLLM keeps a subset, where this rule keeps them all)
        last_member = above[n_kept - 1] + (counts[n_kept - 1] - 1) * np.exp(vals[n_kept - 1] - vals[0]) / M
        margin = min(rule_margin, top_p - last_member)
        keep = keep & (z >= tau_p)
    else:
        rule_margin = margin
    zk = z[keep]
    mx = zk.max()
    log_norm = float(mx + np.log(np.exp(zk - mx).sum()))
    lp = np.full(V, -np.inf)
    lp[keep] = z[keep] - log_norm
    return Truncated(keep, lp, log_norm, float(zk.min()), float(margin), float(rule_margin))


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_topk_topp", GOLDEN / "make_golden_topk_topp.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_fixture() -> dict[int, dict]:
    """{V: {logits [3, V] fp32, kind, T, top_k, top_p [R], mask [R, V] bool, lp_ids, lp [R, 64]}}; large-vocabulary
    logits are regenerated from their seed and checked against the stored SHA-256."""
    gen = _generator()
    d = np.load(GOLDEN / "topk_topp_vllm.npz")
    out = {}
    for V in (int(v) for v in d["vocabs"]):
        pre = f"V{V}_"
        if pre + "logits" in d:
            logits = d[pre + "logits"]
        else:
            logits = gen.make_logits(V, int(d[pre + "seed"])).numpy()
        assert gen.logits_sha256(__import__("torch").from_numpy(logits)) == str(d[pre + "sha256"]), \
            f"V={V}: regenerated logits differ from the ones the fixture was made from"
        out[V] = dict(logits=logits, kind=d[pre + "kind"], T=d[pre + "T"], top_k=d[pre + "top_k"], top_p=d[pre + "top_p"],
                      mask=np.unpackbits(d[pre + "mask"], axis=1, count=V).astype(bool), lp_ids=d[pre + "lp_ids"],
                      lp=d[pre + "lp"])
    return out

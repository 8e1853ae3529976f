"""Sampler timing: the untruncated sampler (prl_sample_logprob_rows) against the top-k / top-p sampler
(prl_sample_logprob_topkp_rows) at B = 64, V = 152 064 (Qwen2.5), CUDA events over many calls.

Cases: untruncated; top-k 50; top-p 0.95; both; 2 truncated rows (top-k 50 + top-p 0.95) among 64.  Reports us per call
and the logits bytes read once per call (4 B V) over that time, with the card name and power limit.
    python tools/sample_bench.py [--iters 200] [--out sample_bench.json]"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--V", type=int, default=152064)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench needs a CUDA device")
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda:0")
    B, V = a.B, a.V
    g = torch.Generator(device=dev).manual_seed(0)
    logits = torch.randn(B, V, device=dev, generator=g) * 3
    inv_t = torch.ones(B, device=dev)
    greedy = torch.zeros(B, dtype=torch.uint8, device=dev)
    ids = torch.zeros(B, dtype=torch.int32, device=dev)
    lps = torch.zeros(B, device=dev)
    ws = torch.zeros(int(lib.prl_sample_topkp_workspace_bytes(B, V)), dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr()

    def rows(k, p, n_trunc=B):
        kk = torch.full((B,), -1, dtype=torch.int32, device=dev)
        pp = torch.ones(B, device=dev)
        kk[:n_trunc], pp[:n_trunc] = k, p
        return kk, pp

    cases = {"untruncated": None, "top_k50": rows(50, 1.0), "top_p0.95": rows(-1, 0.95),
             "top_k50_top_p0.95": rows(50, 0.95), "2_of_64_truncated": rows(50, 0.95, n_trunc=2)}

    def call(case, step):
        if case is None:
            _lib.check(lib.prl_sample_logprob_rows(logits.data_ptr(), B, V, inv_t.data_ptr(), greedy.data_ptr(), 1, step,
                                                   ids.data_ptr(), lps.data_ptr(), ws.data_ptr(), ws.numel(), st))
        else:
            kk, pp = case
            _lib.check(lib.prl_sample_logprob_topkp_rows(logits.data_ptr(), B, V, inv_t.data_ptr(), greedy.data_ptr(),
                                                         kk.data_ptr(), pp.data_ptr(), 1, step, ids.data_ptr(),
                                                         lps.data_ptr(), None, None, None, ws.data_ptr(), ws.numel(), st))

    res = {"B": B, "V": V, "iters": a.iters, **card(), "cases": {}}
    for rep in range(2):                  # two alternating passes: the spread between them is the noise
        for name, case in cases.items():
            for s in range(a.warmup):
                call(case, s)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for s in range(a.iters):
                call(case, s)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / a.iters
            res["cases"].setdefault(name, []).append({"us_per_call": round(us, 2),
                                                      "logits_GBps": round(4.0 * B * V / (us * 1e-6) / 1e9, 1)})
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()

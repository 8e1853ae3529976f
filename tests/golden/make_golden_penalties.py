"""penalties_vllm.npz / penalties_vllm.json: vLLM 0.22's repetition / frequency / presence penalties and min_p on fixed
logits, and its validation of the four parameters.

Executes, per row, what vLLM's sampler does (v1/sample/sampler.py, logprobs-mode processed_logprobs):
    l = apply_all_penalties(logits, prompt ids, presence, frequency, repetition, output ids)   (v1/sample/ops/penalties.py;
        on the CPU its repetition step is _custom_ops.apply_repetition_penalties_torch)
    greedy rows: argmax(l), processed logprobs log_softmax(l)
    else:   z = l / T;  z = MinPLogitsProcessor.apply(z) when min_p > 0;  z = apply_top_k_top_p_pytorch(z, k, p);
            processed logprobs = log_softmax(z)
Rows (V = 640, logits stored): every penalty alone at its range edges and inside it, all three together, logits that are
positive, negative, +0, -0 and -inf (a min_tokens ban), ids in the prompt only, the outputs only and both, one output
id repeated 1000 times, the padding id V in both lists; min_p in {0.01, 0.1, 0.5, 1.0} x T in {0.6, 1.0, 1.3}, alone and
with top-k / top-p, with and without penalties; a greedy row with min_p set.  Rows at V = 152 064 (penalties only) store
the seed of their logits and the SHA-256 of the input and of vLLM's penalized row.
The JSON holds vLLM's accept / reject decision, and the values it keeps, for a list of parameter dicts.

Run where vLLM imports (CPU is enough):  python tests/golden/make_golden_penalties.py
The tests regenerate the logits and ids with the functions below; they never import vLLM."""
from __future__ import annotations

import hashlib
import io
import json
import zipfile
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
OUT_NPZ, OUT_JSON = HERE / "penalties_vllm.npz", HERE / "penalties_vllm.json"
V_SMALL, V_LARGE = 640, 152064

# (presence, frequency, repetition)
PENALTY_SETTINGS = [
    (0.0, 0.0, 1.0),
    (2.0, 0.0, 1.0), (-2.0, 0.0, 1.0), (0.5, 0.0, 1.0),
    (0.0, 2.0, 1.0), (0.0, -2.0, 1.0), (0.0, 0.7, 1.0),
    (0.0, 0.0, 0.5), (0.0, 0.0, 1.3), (0.0, 0.0, 2.0),
    (1.5, 0.5, 1.05), (-2.0, 2.0, 0.5), (2.0, -2.0, 2.0), (0.3, -1.1, 1.17),
]
LARGE_SETTINGS = [(1.5, 0.5, 1.05), (2.0, -2.0, 2.0), (0.0, 0.7, 1.0), (-2.0, 0.0, 1.0), (0.0, 0.0, 0.5)]
MIN_PS = (0.01, 0.1, 0.5, 1.0)
TEMPERATURES = (0.6, 1.0, 1.3)
TRUNCATIONS = ((-1, 1.0), (50, 0.95))

VALIDATION_CASES = [
    {}, {"presence_penalty": None}, {"frequency_penalty": None}, {"repetition_penalty": None}, {"min_p": None},
    {"presence_penalty": 2.0}, {"presence_penalty": -2.0}, {"presence_penalty": 2.001}, {"presence_penalty": -2.5},
    {"presence_penalty": 1}, {"presence_penalty": 3},
    {"frequency_penalty": 2.0}, {"frequency_penalty": -2.0}, {"frequency_penalty": 2.5}, {"frequency_penalty": -2.001},
    {"frequency_penalty": 1}, {"frequency_penalty": -3},
    {"repetition_penalty": 1e-6}, {"repetition_penalty": 0.0}, {"repetition_penalty": -1.0}, {"repetition_penalty": 0},
    {"repetition_penalty": 1}, {"repetition_penalty": 2}, {"repetition_penalty": 100.0},
    {"min_p": 0.0}, {"min_p": 1.0}, {"min_p": 1}, {"min_p": 0.05}, {"min_p": -0.01}, {"min_p": 1.01}, {"min_p": 2},
    {"presence_penalty": 1.5, "frequency_penalty": 0.5, "repetition_penalty": 1.05, "min_p": 0.05},
    {"presence_penalty": 1.5, "frequency_penalty": 2.5, "repetition_penalty": 1.05},
    {"temperature": 0.0, "min_p": 0.5}, {"temperature": 0.0, "min_p": 0.5, "presence_penalty": 1.0},
    {"temperature": 0.0, "min_p": 1.5}, {"temperature": 0.7, "min_p": 0.5},
]


def make_case(V: int, seed: int, n_prompt: int, n_out: int) -> tuple[torch.Tensor, list[int], list[int]]:
    """(logits [V] fp32, prompt ids, output ids).  The logits are N(0, 4) with eight +0, eight -0 and eight -inf entries;
    the prompt and outputs share ids, each has ids of its own and holds the padding id V; the first output id is
    repeated 1000 times."""
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(V, generator=g) * 4.0
    special = torch.randperm(V, generator=g)[:24]
    logits[special[:8]] = 0.0
    logits[special[8:16]] = -0.0
    logits[special[16:]] = float("-inf")
    pool = torch.randperm(V, generator=g)
    both = pool[:n_out // 4].tolist()
    prompt_only = pool[n_out // 4:n_out // 4 + n_prompt].tolist()
    out_only = pool[n_out // 4 + n_prompt:n_out // 4 + n_prompt + n_out].tolist()
    # the special values are in both lists, in one, and in neither
    prompt = prompt_only + both + special[0:4].tolist() + special[8:12].tolist() + special[16:20].tolist()
    prompt += prompt[:n_prompt // 3] + [V]
    out = out_only + both + special[2:6].tolist() + special[10:14].tolist() + special[18:22].tolist()
    out += out[:n_out // 2] + [out[0]] * 1000 + [V]
    perm_p = torch.randperm(len(prompt), generator=g).tolist()
    perm_o = torch.randperm(len(out), generator=g).tolist()
    return logits, [prompt[i] for i in perm_p], [out[i] for i in perm_o]


def small_rows() -> list[dict]:
    """Every V = 640 row: its seed and the request's parameters."""
    rows = []
    for i, (pr, f, r) in enumerate(PENALTY_SETTINGS):
        rows.append(dict(seed=100 + i, presence=pr, frequency=f, repetition=r, min_p=0.0, T=1.0, top_k=-1, top_p=1.0,
                         greedy=False))
    k = 0
    for mp in MIN_PS:
        for T in TEMPERATURES:
            for tk, tp in TRUNCATIONS:
                rows.append(dict(seed=200 + k, presence=0.0, frequency=0.0, repetition=1.0, min_p=mp, T=T, top_k=tk,
                                 top_p=tp, greedy=False))
                k += 1
    rows += [dict(seed=300, presence=1.5, frequency=0.5, repetition=1.05, min_p=0.1, T=1.0, top_k=-1, top_p=1.0,
                  greedy=False),
             dict(seed=301, presence=-2.0, frequency=2.0, repetition=0.5, min_p=0.05, T=0.6, top_k=20, top_p=0.9,
                  greedy=False),
             dict(seed=302, presence=0.3, frequency=-1.1, repetition=1.17, min_p=0.5, T=1.3, top_k=50, top_p=0.95,
                  greedy=False),
             dict(seed=303, presence=1.0, frequency=0.5, repetition=1.3, min_p=0.0, T=1.0, top_k=-1, top_p=1.0,
                  greedy=True),
             dict(seed=304, presence=0.0, frequency=0.0, repetition=1.0, min_p=0.5, T=1.0, top_k=-1, top_p=1.0,
                  greedy=True)]
    return rows


def large_rows() -> list[dict]:
    return [dict(seed=400 + i, presence=pr, frequency=f, repetition=r) for i, (pr, f, r) in enumerate(LARGE_SETTINGS)]


def small_case(row: dict):
    return make_case(V_SMALL, row["seed"], 60, 40)


def large_case(row: dict):
    return make_case(V_LARGE, row["seed"], 8192, 600)


def sha256(x: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest()


def pad(lists: list[list[int]], V: int) -> np.ndarray:
    n = max(len(x) for x in lists)
    return np.array([x + [V] * (n - len(x)) for x in lists], dtype=np.int32)


def _vllm_penalties(logits: torch.Tensor, prompts, outs, rows) -> torch.Tensor:
    import vllm.v1.sample.ops.penalties as penalties
    penalties.is_pin_memory_available = lambda: False       # pin_memory() needs a driver
    V = logits.shape[1]
    prompt_t = torch.from_numpy(pad(prompts, V)).long()
    f32 = lambda k: torch.tensor([r[k] for r in rows], dtype=torch.float32)  # noqa: E731
    return penalties.apply_all_penalties(logits.clone(), prompt_t, f32("presence"), f32("frequency"), f32("repetition"),
                                         [list(o) for o in outs])


def _min_p(z: torch.Tensor, min_p: float) -> torch.Tensor:
    from vllm.v1.sample.logits_processor.builtin import MinPLogitsProcessor
    proc = object.__new__(MinPLogitsProcessor)
    proc.min_p_count = 1
    proc.min_p = torch.tensor([[min_p]], dtype=torch.float32)
    return proc.apply(z)


def _validation() -> list[dict]:
    from vllm import SamplingParams
    out = []
    for case in VALIDATION_CASES:
        # ChatCompletionRequest.to_sampling_params under generation-config vllm: a None repetition_penalty / min_p is
        # the default; from_optional does the same for the other two
        kw = {k: v for k, v in case.items() if not (v is None and k in ("repetition_penalty", "min_p"))}
        try:
            sp = SamplingParams.from_optional(**kw)
        except ValueError as e:
            out.append(dict(params=case, accepted=False, error=str(e)))
            continue
        out.append(dict(params=case, accepted=True, presence_penalty=sp.presence_penalty,
                        frequency_penalty=sp.frequency_penalty, repetition_penalty=sp.repetition_penalty,
                        min_p=sp.min_p))
    return out


def write_npz(path: Path, arrays: dict[str, np.ndarray]) -> None:
    """np.savez_compressed with fixed member timestamps, so that a rerun writes the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for name, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main() -> None:
    from vllm.v1.sample.ops.topk_topp_sampler import apply_top_k_top_p_pytorch
    rows = small_rows()
    cases = [small_case(r) for r in rows]
    logits = torch.stack([c[0] for c in cases])
    pen = _vllm_penalties(logits, [c[1] for c in cases], [c[2] for c in cases], rows)
    masks, lps, argmax = [], [], []
    for i, r in enumerate(rows):
        if r["greedy"]:
            keep = torch.ones(V_SMALL, dtype=torch.bool)
            lp = pen[i:i + 1].log_softmax(dim=-1, dtype=torch.float32)[0]
        else:
            z = pen[i:i + 1].clone().div_(r["T"])               # Sampler.apply_temperature
            if r["min_p"] > 0:
                z = _min_p(z, r["min_p"])
            keep = torch.isfinite(z[0]) | ~torch.isfinite(pen[i])   # what min_p dropped
            kt = torch.tensor([r["top_k"]], dtype=torch.long) if r["top_k"] > 0 else None
            pt = torch.tensor([r["top_p"]], dtype=torch.float32) if r["top_p"] < 1.0 else None
            z = apply_top_k_top_p_pytorch(z, kt, pt)
            lp = z.log_softmax(dim=-1, dtype=torch.float32)[0]
        masks.append(np.packbits(keep.numpy()))
        lps.append(lp.numpy())
        argmax.append(int(torch.argmax(pen[i])))
    out = {"V": np.array(V_SMALL, dtype=np.int64), "logits": logits.numpy(), "penalized": pen.numpy(),
           "min_p_keep": np.stack(masks), "logprobs": np.stack(lps), "argmax": np.array(argmax, dtype=np.int32)}
    for k in ("presence", "frequency", "repetition", "min_p", "T", "top_p"):
        out[k] = np.array([r[k] for r in rows], dtype=np.float32)
    for k in ("seed", "top_k"):
        out[k] = np.array([r[k] for r in rows], dtype=np.int32)
    out["greedy"] = np.array([r["greedy"] for r in rows], dtype=np.uint8)
    out["prompt_ids"] = pad([c[1] for c in cases], V_SMALL)
    out["output_ids"] = pad([c[2] for c in cases], V_SMALL)
    big = large_rows()
    out["large_seed"] = np.array([r["seed"] for r in big], dtype=np.int32)
    for k in ("presence", "frequency", "repetition"):
        out["large_" + k] = np.array([r[k] for r in big], dtype=np.float32)
    sha_in, sha_out = [], []
    for r in big:
        lg, prompt, outs = large_case(r)
        pen_l = _vllm_penalties(lg[None], [prompt], [outs], [r])[0]
        sha_in.append(sha256(lg.numpy()))
        sha_out.append(sha256(pen_l.numpy()))
    out["large_logits_sha256"] = np.array(sha_in)
    out["large_penalized_sha256"] = np.array(sha_out)
    write_npz(OUT_NPZ, out)
    OUT_JSON.write_text(json.dumps({"vllm": "0.22.0", "validation": _validation()}, indent=1) + "\n")
    print(f"wrote {OUT_NPZ} ({OUT_NPZ.stat().st_size} bytes) and {OUT_JSON}")


if __name__ == "__main__":
    main()

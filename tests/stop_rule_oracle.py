"""Host restatement of the token step's stop rule (prl_advance_state, csrc/decode_ops.cu), pinned against vLLM 0.22's
update_from_generation_config + check_stop (tests/golden/stop_rule_vllm.json, tests/golden/make_golden_stop_rule.py).

A case of the fixture becomes the engine's (eos_id, stop_ids) through stop_ids_from_generation_config, the slot's stop
row through DecodeEngine.stop_row, and then runs the kernel's order: append the id; primary eos unless ignored; the
stop row; the length cap."""
from __future__ import annotations

import json
import types

from tests.helpers import GOLDEN


def stop_cases() -> list[dict]:
    return json.loads((GOLDEN / "stop_rule_vllm.json").read_text())


def slot_setup(case: dict, max_stop_ids: int = 16, vocab: int = 64):
    """-> (eos_id, stop row, ignore_eos) of the slot serving `case`, through the engine's own host code."""
    from pipelinerl_b200.engine import DecodeEngine, SamplingParams, stop_ids_from_generation_config
    gen = {} if case["gen_eos"] is None else {"eos_token_id": case["gen_eos"]}
    eos_id, stop_ids = stop_ids_from_generation_config(gen, case["eos"])
    eng = types.SimpleNamespace(stop_ids=stop_ids, max_stop_ids=max_stop_ids, _ignore_eos=False,
                                cfg=types.SimpleNamespace(vocab_size=vocab))
    eng._check_token_ids = lambda ids: DecodeEngine._check_token_ids(eng, ids)
    sp = SamplingParams(max_tokens=case["max_tokens"], ignore_eos=case["ignore_eos"],
                        stop_token_ids=tuple(case["stop"]))
    return eos_id, DecodeEngine.stop_row(eng, sp), case["ignore_eos"]


def host_stop_rule(ids, eos_id: int, row: list[int], ignore_eos: bool, max_tokens: int):
    """-> (output ids, finish_reason, stop_reason) for the sampled `ids`."""
    out = []
    for t in ids:
        out.append(t)
        if t == eos_id and not ignore_eos:
            return out, "stop", None
        if t in row:
            return out, "stop", t
        if len(out) >= max_tokens:
            return out, "length", None
    raise AssertionError("scripted ids ran out before the request finished")

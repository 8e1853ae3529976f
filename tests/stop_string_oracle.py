"""Host restatement of the token step's stop-string and min_tokens rule (prl_advance_state's matcher and
prl_ban_min_tokens, csrc/decode_ops.cu), pinned against vLLM 0.22's detokenizer, check_stop and OutputProcessor
(tests/golden/stop_strings_vllm.json, tests/golden/make_golden_stop_strings.py).

Per sampled id: append it; while fewer than min_tokens outputs, nothing stops; else the primary eos, the stop row, the
length cap.  Then the token's bytes (none for a special token when special tokens are skipped, none for the token that
ended the request on eos / a stop id unless the stop string is included) go through one KMP automaton per string; the
first string in request order that completes a match inside them finishes the request with "stop" and that string, once
the output holds more than min_tokens ids.  The text is what the engine returns: engine.stop_string_text."""
from __future__ import annotations

import json

from tests.helpers import GOLDEN


def stop_string_cases() -> list[dict]:
    return json.loads((GOLDEN / "stop_strings_vllm.json").read_text())


def min_tokens_fixture() -> dict:
    return json.loads((GOLDEN / "min_tokens_vllm.json").read_text())


def fixture_tokenizer():
    from transformers import PreTrainedTokenizerFast
    return PreTrainedTokenizerFast(tokenizer_file=str(GOLDEN / "stop_tokenizer.json"), eos_token="<|im_end|>")


def slot_params(case: dict):
    """-> (eos_id, stop row, SamplingParams) of the slot serving `case`, through the engine's host code."""
    from pipelinerl_b200.engine import SamplingParams, stop_ids_from_generation_config
    gen = {} if case["gen_eos"] is None else {"eos_token_id": case["gen_eos"]}
    eos_id, extra = stop_ids_from_generation_config(gen, case["eos"])
    include, skip = case["flags"]
    sp = SamplingParams(max_tokens=case["max_tokens"], stop_token_ids=tuple(case["stop_ids"]), stop=tuple(case["stop"]),
                        min_tokens=case["min_tokens"], include_stop_str_in_output=include, skip_special_tokens=skip)
    row = list(dict.fromkeys(list(sp.stop_token_ids) + list(extra)))
    return eos_id, row, extra, sp


def kmp_step(s: bytes, fail: list[int], q: int, c: int) -> int:
    while q > 0 and s[q] != c:
        q = fail[q - 1]
    return q + 1 if s[q] == c else q


def host_rule(ids, table, eos_id: int, row: list[int], sp) -> tuple[int, str, object, int]:
    """-> (n_out, finish_reason, stop_reason, index of the matched string or -1) for the sampled `ids`."""
    from pipelinerl_b200.engine import kmp_failure
    data, offsets, special = table
    strs = [s.encode("utf-8") for s in sp.stop]
    fails = [kmp_failure(s) for s in strs]
    state = [0] * len(strs)
    for n, t in enumerate(ids, start=1):
        core = n >= sp.min_tokens
        stop, reason = False, None
        if core and t == eos_id and not sp.ignore_eos:
            stop = True
        elif core and t in row:
            stop, reason = True, t
        length = n >= sp.max_tokens
        match = -1
        fed = not (stop and not sp.include_stop_str_in_output) and not (sp.skip_special_tokens and special[t])
        if strs and fed:
            for j, s in enumerate(strs):
                hit = False
                for c in bytes(data[offsets[t]:offsets[t + 1]]):
                    state[j] = kmp_step(s, fails[j], state[j], c)
                    if state[j] == len(s):
                        hit, state[j] = True, fails[j][-1]
                if hit and n > sp.min_tokens:
                    match = j
                    break
        if match >= 0:
            return n, "stop", sp.stop[match], match
        if stop or length:
            return n, "stop" if stop else "length", reason, -1
    raise AssertionError("scripted ids ran out before the request finished")


def host_text(ids, finish_reason, match, table, sp) -> str:
    """engine.DecodeEngine.stop_string_text without an engine."""
    import types

    from pipelinerl_b200.engine import DecodeEngine, Request
    data, offsets, special = table
    eng = types.SimpleNamespace(_tok_table_host=lambda: (bytes(data), list(offsets), list(special), len(special)))
    req = Request(0, [0], sp, output_ids=list(ids), finish_reason=finish_reason)
    return DecodeEngine.stop_string_text(eng, req, match)

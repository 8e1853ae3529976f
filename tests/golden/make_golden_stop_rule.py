"""Golden fixture for the stop rule of the token step: vLLM 0.22's own `SamplingParams.update_from_generation_config`
and `check_stop` (vllm/v1/core/sched/utils.py) run on scripted id sequences.

    python tests/golden/make_golden_stop_rule.py      (authoring container: needs vllm 0.22)

A minimal stand-in request carries what check_stop reads.  Each case is the tokenizer's eos id, the `eos_token_id` of a
generation_config.json, the request's stop_token_ids, ignore_eos, max_tokens and the ids the sampler draws; recorded are
the output length when the request finished, its finish_reason and vLLM's stop_reason (None: primary eos or length).
Written to stop_rule_vllm.json.
"""
import json
from pathlib import Path

from vllm import SamplingParams
from vllm.v1.core.sched.utils import check_stop
from vllm.v1.request import RequestStatus

CASES = [
    dict(name="primary_eos", eos=2, gen_eos=None, stop=[], ignore_eos=False, max_tokens=8, ids=[5, 6, 2, 7, 8, 9, 4, 4]),
    dict(name="no_stop_runs_to_length", eos=2, gen_eos=None, stop=[], ignore_eos=False, max_tokens=5,
         ids=[5, 6, 7, 8, 9, 4]),
    dict(name="gen_config_list_with_primary_extra_id", eos=2, gen_eos=[1, 2, 3], stop=[], ignore_eos=False,
         max_tokens=8, ids=[5, 3, 2, 7, 8, 9, 4, 4]),
    dict(name="gen_config_list_with_primary_primary_first", eos=2, gen_eos=[1, 2, 3], stop=[], ignore_eos=False,
         max_tokens=8, ids=[5, 6, 2, 3, 8, 9, 4, 4]),
    dict(name="gen_config_single_int", eos=2, gen_eos=2, stop=[], ignore_eos=False, max_tokens=6, ids=[1, 3, 2, 4, 4, 4]),
    dict(name="request_stop_ids", eos=2, gen_eos=None, stop=[9, 11], ignore_eos=False, max_tokens=8,
         ids=[5, 6, 7, 11, 9, 2, 4, 4]),
    dict(name="request_stop_ids_and_gen_config", eos=2, gen_eos=[1, 2, 3], stop=[9], ignore_eos=False, max_tokens=8,
         ids=[5, 9, 3, 2, 4, 4, 4, 4]),
    dict(name="ignore_eos_keeps_request_stop_ids", eos=2, gen_eos=[1, 2, 3], stop=[9], ignore_eos=True, max_tokens=8,
         ids=[2, 3, 1, 9, 4, 4, 4, 4]),
    dict(name="ignore_eos_without_request_stop_ids", eos=2, gen_eos=[1, 2, 3], stop=[], ignore_eos=True, max_tokens=6,
         ids=[2, 3, 1, 2, 3, 1, 4]),
    dict(name="ignore_eos_request_lists_primary_eos", eos=2, gen_eos=[1, 2, 3], stop=[2], ignore_eos=True,
         max_tokens=8, ids=[3, 1, 2, 4, 4, 4, 4, 4]),
    dict(name="stop_id_at_last_allowed_token", eos=2, gen_eos=[1, 2, 3], stop=[], ignore_eos=False, max_tokens=4,
         ids=[5, 6, 7, 3, 4]),
    dict(name="request_stop_id_at_last_allowed_token", eos=2, gen_eos=None, stop=[11], ignore_eos=False, max_tokens=3,
         ids=[5, 6, 11, 4]),
    dict(name="primary_eos_at_last_allowed_token", eos=2, gen_eos=[1, 2, 3], stop=[], ignore_eos=False, max_tokens=3,
         ids=[5, 6, 2, 4]),
    dict(name="no_tokenizer_eos", eos=None, gen_eos=[1, 3], stop=[], ignore_eos=False, max_tokens=6,
         ids=[5, 3, 1, 4, 4, 4]),
]


class _Req:
    """What check_stop reads of a vllm.v1.request.Request."""

    def __init__(self, sp, prompt_len):
        self.sampling_params, self.pooling_params = sp, None
        self.max_tokens, self.output_token_ids = sp.max_tokens, []
        self.prompt_len, self.status, self.stop_reason = prompt_len, RequestStatus.RUNNING, None

    @property
    def num_output_tokens(self):
        return len(self.output_token_ids)

    @property
    def num_tokens(self):
        return self.prompt_len + len(self.output_token_ids)


def run(case):
    sp = SamplingParams(max_tokens=case["max_tokens"], stop_token_ids=list(case["stop"]), ignore_eos=case["ignore_eos"])
    gen_cfg = {} if case["gen_eos"] is None else {"eos_token_id": case["gen_eos"]}
    sp.update_from_generation_config(gen_cfg, case["eos"])
    req = _Req(sp, prompt_len=4)
    for t in case["ids"]:
        req.output_token_ids.append(t)
        if check_stop(req, max_model_len=1 << 20):
            break
    else:
        raise AssertionError(f"{case['name']}: scripted ids ran out before the request finished")
    finish = {RequestStatus.FINISHED_STOPPED: "stop", RequestStatus.FINISHED_LENGTH_CAPPED: "length"}[req.status]
    return dict(case, n_out=req.num_output_tokens, finish_reason=finish, stop_reason=req.stop_reason,
                vllm_stop_token_ids=sorted(sp.stop_token_ids or []), vllm_eos_token_id=sp.eos_token_id)


def main():
    out = [run(c) for c in CASES]
    for r in out:
        print(r["name"], r["n_out"], r["finish_reason"], r["stop_reason"])
    (Path(__file__).parent / "stop_rule_vllm.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

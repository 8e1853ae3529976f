"""Stop-token sets, host side: the stop rule against vLLM's own (tests/golden/stop_rule_vllm.json), the generation_config
split, stop-row construction, and the capability gate and validation of both clients (no GPU)."""
import asyncio
import types

import pytest

from tests.helpers import tiny_chat_tokenizer
from tests.stop_rule_oracle import host_stop_rule, slot_setup, stop_cases


@pytest.mark.parametrize("case", stop_cases(), ids=lambda c: c["name"])
def test_host_stop_rule_matches_vllm(case):
    eos_id, row, ignore = slot_setup(case)
    out, finish, reason = host_stop_rule(case["ids"], eos_id, row, ignore, case["max_tokens"])
    assert (len(out), finish, reason) == (case["n_out"], case["finish_reason"], case["stop_reason"])
    assert out == case["ids"][:case["n_out"]]                    # the stop token stays in the output
    # the slot's stop row holds exactly the ids vLLM checks after its primary eos
    primary = case["vllm_eos_token_id"]
    assert set(row) - {primary} == set(case["vllm_stop_token_ids"]) - {primary}


def test_fixture_covers_the_cases_of_the_rule():
    by_name = {c["name"]: c for c in stop_cases()}
    assert by_name["gen_config_list_with_primary_extra_id"]["stop_reason"] == 3
    assert by_name["ignore_eos_keeps_request_stop_ids"]["stop_reason"] == 9
    assert by_name["ignore_eos_without_request_stop_ids"]["finish_reason"] == "length"
    last = by_name["stop_id_at_last_allowed_token"]
    assert (last["n_out"], last["finish_reason"]) == (last["max_tokens"], "stop")


def test_stop_ids_from_generation_config():
    from pipelinerl_b200.engine import stop_ids_from_generation_config
    llama31 = {"bos_token_id": 128000, "do_sample": True, "eos_token_id": [128001, 128008, 128009], "temperature": 0.6,
               "top_p": 0.9}
    assert stop_ids_from_generation_config(llama31, 128009) == (128009, (128001, 128008))
    assert stop_ids_from_generation_config(llama31, 128001) == (128001, (128008, 128009))
    assert stop_ids_from_generation_config({"eos_token_id": 151645}, 151645) == (151645, ())
    assert stop_ids_from_generation_config({}, 7) == (7, ())
    assert stop_ids_from_generation_config({"eos_token_id": [5, 6]}, None) == (-1, (5, 6))


def _bare_engine(stop_ids=(), max_stop_ids=4):
    from pipelinerl_b200.engine import DecodeEngine
    from tests.helpers import tiny_cfg
    eng = object.__new__(DecodeEngine)
    eng.cfg, eng.stop_ids, eng.max_stop_ids, eng._ignore_eos = tiny_cfg("gqa2"), tuple(stop_ids), max_stop_ids, False
    return eng


def test_stop_row_rule_and_limits():
    from pipelinerl_b200.engine import SamplingParams
    eng = _bare_engine(stop_ids=(10, 11))
    assert eng.stop_row(SamplingParams(stop_token_ids=(7, 10))) == [7, 10, 11]       # duplicates count once
    assert eng.stop_row(SamplingParams(stop_token_ids=(7,), ignore_eos=True)) == [7]  # ignore_eos drops the engine's
    assert eng.stop_row(SamplingParams()) == [10, 11]
    assert eng.stop_row(SamplingParams(ignore_eos=True)) == []
    with pytest.raises(ValueError, match="limit of 4"):
        eng.stop_row(SamplingParams(stop_token_ids=(1, 2, 3)))
    assert eng.stop_row(SamplingParams(stop_token_ids=(1, 2, 3), ignore_eos=True)) == [1, 2, 3]
    for bad in ((-1,), (eng.cfg.vocab_size,)):
        with pytest.raises(ValueError, match="out of range"):
            eng.stop_row(SamplingParams(stop_token_ids=bad))


@pytest.mark.parametrize("ids", ["7", [1.0], [True], [1, "2"], 5])
def test_stop_token_ids_param_rejects(ids):
    from pipelinerl_b200.engine import stop_token_ids_param
    with pytest.raises(ValueError, match="stop_token_ids"):
        stop_token_ids_param({"stop_token_ids": ids})


def test_stop_token_ids_param_accepts():
    from pipelinerl_b200.engine import stop_token_ids_param
    assert stop_token_ids_param({}) == () and stop_token_ids_param({"stop_token_ids": None}) == ()
    assert stop_token_ids_param({"stop_token_ids": [3, 9]}) == (3, 9)


def test_engines_list_stop_token_ids():
    from pipelinerl_b200 import serving
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    assert DecodeEngine.supports_stop_token_ids and TPDecodeEngine.supports_stop_token_ids
    fused = types.SimpleNamespace(sampling_features=frozenset(), supports_stop_token_ids=True)
    assert serving.engine_features(fused) == frozenset({"stop_token_ids"})
    assert serving.engine_features(types.SimpleNamespace(sampling_features=frozenset({"top_k"}))) == frozenset({"top_k"})


class _StubServer:
    """Registered engine stand-in with stop sets (or without) that records the SamplingParams it receives."""

    def __init__(self, name, stops=True):
        from pipelinerl_b200 import serving
        self.name, self.seen = name, []
        eng = _bare_engine(stop_ids=(10,), max_stop_ids=3)
        self.engine = types.SimpleNamespace(sampling_features=frozenset({"top_k", "top_p"}),
                                            arena=types.SimpleNamespace(version=0), stop_row=eng.stop_row)
        if stops:
            self.engine.supports_stop_token_ids = True
        self.on_step_boundary, self.error = None, None
        serving._REGISTRY[name] = self

    def close(self):
        from pipelinerl_b200 import serving
        serving._REGISTRY.pop(self.name, None)

    async def generate(self, prompt_ids, params):
        self.seen.append(params)
        stop = 9 if 9 in params.stop_token_ids else None
        return types.SimpleNamespace(output_ids=[5, 9] if stop else [5, 6], output_logprobs=[-0.5, -0.25],
                                     finish_reason="stop" if stop else "length", stop_reason=stop, model_version=0)


def _generate(base_url, parameters):
    from pipelinerl_b200.async_llm import llm_async_generate
    from pipelinerl_b200.llm import Prompt, SyntheticTokenizer, TrainableLLM
    llm = TrainableLLM(base_url, "m", parameters=parameters, tokenizer=SyntheticTokenizer())
    return asyncio.run(llm_async_generate(llm, Prompt(messages=[{"role": "user", "content": "hi"}])))


def test_in_process_client_passes_stop_token_ids():
    stub = _StubServer("stop-stub")
    try:
        call = _generate("inproc://stop-stub", {"max_tokens": 4, "stop_token_ids": [9, 12]})
        assert stub.seen[-1].stop_token_ids == (9, 12)
        assert (call.llm_info["finish_reason"], call.llm_info["stop_reason"]) == ("stop", 9)
        n = len(stub.seen)
        for bad in ({"stop_token_ids": ["9"]}, {"stop_token_ids": [1, 2, 3]}, {"stop_token_ids": [-4]},
                    {"stop": ["\n"]}, {"stop": "x", "stop_token_ids": [9]}):
            with pytest.raises(ValueError):
                _generate("inproc://stop-stub", {"max_tokens": 4, **bad})
        assert len(stub.seen) == n                                 # nothing reached the engine
    finally:
        stub.close()


def test_in_process_client_refuses_stop_token_ids_the_engine_does_not_list():
    stub = _StubServer("nostop-stub", stops=False)
    try:
        with pytest.raises(ValueError, match="stop token ids"):
            _generate("inproc://nostop-stub", {"max_tokens": 4, "stop_token_ids": [9]})
        _generate("inproc://nostop-stub", {"max_tokens": 4, "stop_token_ids": []})
        assert stub.seen[-1].stop_token_ids == ()
    finally:
        stub.close()


def test_http_shim_serves_stop_token_ids_and_reports_stop_reason():
    import aiohttp

    from pipelinerl_b200.http_shim import HttpShim

    async def go():
        server = _StubServer("stop-http-stub")
        plain = _StubServer("nostop-http-stub", stops=False)
        shim, shim2 = HttpShim(server, tiny_chat_tokenizer(), "tiny"), HttpShim(plain, tiny_chat_tokenizer(), "tiny")
        url, url2 = await shim.start(), await shim2.start()
        msgs = [{"role": "user", "content": "hello"}]
        try:
            async with aiohttp.ClientSession() as s:
                body = {"model": "tiny", "messages": msgs, "max_tokens": 4, "stop_token_ids": [9]}
                async with s.post(url + "/v1/chat/completions", json=body) as r:
                    assert r.status == 200
                    choice = (await r.json())["choices"][0]
                assert (choice["finish_reason"], choice["stop_reason"]) == ("stop", 9)
                assert server.seen[-1].stop_token_ids == (9,)
                async with s.post(url + "/v1/chat/completions", json={"model": "tiny", "messages": msgs}) as r:
                    assert (await r.json())["choices"][0]["stop_reason"] is None
                for bad in ([1, 2, 3], ["9"], [10 ** 9], 9):
                    async with s.post(url + "/v1/chat/completions",
                                      json={"model": "tiny", "messages": msgs, "stop_token_ids": bad}) as r:
                        assert r.status == 400 and "error" in await r.json()
                assert len(server.seen) == 2
                async with s.post(url2 + "/v1/chat/completions",
                                  json={"model": "tiny", "messages": msgs, "stop_token_ids": [9]}) as r:
                    assert r.status == 400 and "stop_token_ids" in (await r.json())["error"]["message"]
                assert not plain.seen
        finally:
            await shim.stop()
            await shim2.stop()
            server.close()
            plain.close()
    asyncio.new_event_loop().run_until_complete(go())


def test_advance_state_struct_appends_the_stop_fields():
    """prl_engine_state gained its stop fields at the end: every earlier field keeps its offset."""
    from pathlib import Path

    from pipelinerl_b200 import _lib
    names = [n for n, _ in _lib.EngineState._fields_]
    assert names[-4:] == ["stop_ids", "stop_stride", "n_stop", "stop_reason"]
    assert names[:-4][-1] == "ignore_eos_rows"
    header = (Path(__file__).resolve().parent.parent / "include" / "prl.h").read_text()
    body = header[header.index("const uint8_t* ignore_eos_rows;"):header.index("} prl_engine_state;")]
    assert [n for n in names[-4:] if n + ";" in body] == names[-4:]

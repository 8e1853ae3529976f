"""Repetition / frequency / presence penalties and min_p without a GPU: the fp32 oracle against vLLM 0.22's own code
(tests/golden/penalties_vllm.npz, made by make_golden_penalties.py), validation against vLLM's decisions, and the
capability gate of the engine, the in-process client and the HTTP shim."""
from __future__ import annotations

import asyncio
import types

import numpy as np
import pytest

from tests.penalty_oracle import apply_penalties, load_fixture, processed_logprobs


@pytest.fixture(scope="module")
def fx():
    return load_fixture()


def test_oracle_penalized_rows_are_bitwise_vllm(fx):
    for i in range(fx["logits"].shape[0]):
        got = apply_penalties(fx["logits"][i], fx["prompt_ids"][i], fx["output_ids"][i], fx["presence"][i],
                              fx["frequency"][i], fx["repetition"][i])
        assert np.array_equal(got.view(np.uint32), fx["penalized"][i].view(np.uint32)), i
        if fx["greedy"][i]:
            assert int(np.argmax(got)) == int(fx["argmax"][i])


def test_oracle_wide_rows_hash_to_vllm(fx):
    gen = fx["gen"]
    for j, seed in enumerate(fx["large_seed"]):
        logits, prompt, out = gen.large_case(dict(seed=int(seed)))
        assert gen.sha256(logits.numpy()) == str(fx["large_logits_sha256"][j])
        got = apply_penalties(logits.numpy(), prompt, out, fx["large_presence"][j], fx["large_frequency"][j],
                              fx["large_repetition"][j])
        assert gen.sha256(got) == str(fx["large_penalized_sha256"][j]), j


def test_fixture_covers_the_cases(fx):
    V = int(fx["V"])
    assert {float(x) for x in fx["presence"]} >= {-2.0, 2.0} and {float(x) for x in fx["frequency"]} >= {-2.0, 2.0}
    assert {round(float(x), 2) for x in fx["repetition"]} >= {0.5, 1.3, 2.0}
    assert {round(float(x), 2) for x in fx["min_p"]} >= {0.01, 0.1, 0.5, 1.0}
    assert (fx["prompt_ids"] == V).any(axis=1).all() and (fx["output_ids"] == V).any(axis=1).all()
    assert max(np.bincount(r[r < V]).max() for r in fx["output_ids"]) >= 1000
    assert np.isneginf(fx["logits"]).any(axis=1).all() and (np.signbit(fx["logits"]) & (fx["logits"] == 0)).any()
    assert (fx["greedy"].astype(bool) & (fx["min_p"] > 0)).any()
    assert (~fx["min_p_keep"]).any()


def test_oracle_min_p_masks_and_logprobs_match_vllm(fx):
    for i in range(fx["logits"].shape[0]):
        lp, keep = processed_logprobs(fx["penalized"][i], float(fx["T"][i]), float(fx["min_p"][i]), int(fx["top_k"][i]),
                                      float(fx["top_p"][i]), bool(fx["greedy"][i]))
        assert np.array_equal(keep, fx["min_p_keep"][i]), i
        want = fx["logprobs"][i]
        assert np.array_equal(np.isfinite(lp), np.isfinite(want)), i
        fin = np.isfinite(want)
        np.testing.assert_allclose(lp[fin], want[fin], rtol=1e-6, atol=1e-6)   # fp32 values of up to ~20 in size


def test_penalty_params_decide_as_vllm(fx):
    from pipelinerl_b200.engine import penalty_params
    for case in fx["validation"]:
        params = case["params"]
        greedy = params.get("temperature", 1.0) <= 0
        if not case["accepted"]:
            with pytest.raises(ValueError):
                penalty_params(params, greedy=greedy)
            continue
        got = penalty_params(params, greedy=greedy)
        assert got == (case["presence_penalty"], case["frequency_penalty"], case["repetition_penalty"], case["min_p"]), \
            params


@pytest.mark.parametrize("bad", [{"presence_penalty": float("nan")}, {"repetition_penalty": float("inf")},
                                 {"repetition_penalty": float("nan")}, {"min_p": "0.1"}, {"frequency_penalty": True}])
def test_penalty_params_refuse_non_numbers(bad):
    from pipelinerl_b200.engine import penalty_params
    with pytest.raises(ValueError):
        penalty_params(bad)


def test_capabilities():
    from pipelinerl_b200 import serving
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    four = {"presence_penalty", "frequency_penalty", "repetition_penalty", "min_p"}
    assert DecodeEngine.supports_penalties.fget(types.SimpleNamespace(fused_head=False)) is True
    assert DecodeEngine.supports_penalties.fget(types.SimpleNamespace(fused_head=True)) is False
    assert TPDecodeEngine.supports_penalties is False
    assert serving.engine_features(types.SimpleNamespace(supports_penalties=True)) == frozenset(four)
    assert serving.engine_features(types.SimpleNamespace(supports_penalties=False)) == frozenset()


def test_engines_without_penalties_refuse_them():
    """The fused head and the TP engine refuse the four parameters in add_request, before any device state is touched
    (bare instances: no GPU)."""
    from pipelinerl_b200.engine import DecodeEngine, SamplingParams
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    from tests.helpers import tiny_cfg
    for cls, fused in ((DecodeEngine, True), (TPDecodeEngine, False)):
        eng = object.__new__(cls)
        eng.cfg, eng.max_seq_len, eng.max_new, eng.fused_head = tiny_cfg("gqa2"), 128, 32, fused
        eng._greedy, eng._temperature, eng._ignore_eos = False, 1.0, False
        eng.stop_ids, eng.max_stop_ids, eng._tok_table = (), 4, None
        for kw in ({"presence_penalty": 1.0}, {"frequency_penalty": -0.5}, {"repetition_penalty": 1.05},
                   {"min_p": 0.05}):
            with pytest.raises(ValueError, match="not implemented by this engine"):
                eng.add_request([1, 2, 3], SamplingParams(max_tokens=4, **kw))
        with pytest.raises(ValueError, match="min_p"):
            eng.add_request([1, 2, 3], SamplingParams(max_tokens=4, min_p=1.5))


class _Stub:
    def __init__(self, name, penalties=True):
        from pipelinerl_b200 import serving
        self.name, self.seen = name, []
        self.engine = types.SimpleNamespace(sampling_features=frozenset(), arena=types.SimpleNamespace(version=0),
                                            supports_penalties=penalties)
        self.on_step_boundary, self.error = None, None
        serving._REGISTRY[name] = self

    def close(self):
        from pipelinerl_b200 import serving
        serving._REGISTRY.pop(self.name, None)

    async def generate(self, prompt_ids, params):
        self.seen.append(params)
        return types.SimpleNamespace(output_ids=[5, 6], output_logprobs=[-0.5, -0.25], finish_reason="length",
                                     model_version=0)


def _generate(base_url, parameters):
    from pipelinerl_b200.async_llm import llm_async_generate
    from pipelinerl_b200.llm import Prompt, SyntheticTokenizer, TrainableLLM
    llm = TrainableLLM(base_url, "m", parameters=parameters, tokenizer=SyntheticTokenizer())
    return asyncio.run(llm_async_generate(llm, Prompt(messages=[{"role": "user", "content": "hi"}])))


# each value is "off" for only some of the four parameters: an engine without penalties must refuse all of these
NOT_OFF = ({"presence_penalty": 1.0}, {"frequency_penalty": 1}, {"min_p": 1.0}, {"repetition_penalty": 1.05},
           {"presence_penalty": -0.5})


def _key(sp):
    return (sp.presence_penalty, sp.frequency_penalty, sp.repetition_penalty, sp.min_p)


def test_in_process_client_gate():
    stub, plain = _Stub("pen-stub"), _Stub("pen-plain", penalties=False)
    try:
        _generate("inproc://pen-stub", {"max_tokens": 4, "presence_penalty": 1.5, "frequency_penalty": 0.5,
                                        "repetition_penalty": 1.05, "min_p": 0.05})
        assert _key(stub.seen[-1]) == (1.5, 0.5, 1.05, 0.05)
        _generate("inproc://pen-stub", {"max_tokens": 4, "temperature": 0.0, "min_p": 0.5, "repetition_penalty": 2})
        assert _key(stub.seen[-1]) == (0.0, 0.0, 2.0, 0.0) and stub.seen[-1].greedy
        n = len(stub.seen)
        for bad in ({"presence_penalty": 2.5}, {"frequency_penalty": -3}, {"repetition_penalty": 0}, {"min_p": 1.01}):
            with pytest.raises(ValueError):
                _generate("inproc://pen-stub", {"max_tokens": 4, **bad})
        assert len(stub.seen) == n
        for bad in NOT_OFF:
            with pytest.raises(ValueError, match="not implemented by this engine"):
                _generate("inproc://pen-plain", {"max_tokens": 4, **bad})
        assert not plain.seen
        _generate("inproc://pen-plain", {"max_tokens": 4, "presence_penalty": 0, "frequency_penalty": None,
                                         "repetition_penalty": 1, "min_p": 0.0})
        assert _key(plain.seen[-1]) == (0.0, 0.0, 1.0, 0.0)
    finally:
        stub.close()
        plain.close()


def test_http_shim_gate():
    import aiohttp

    from pipelinerl_b200.http_shim import HttpShim
    from tests.helpers import tiny_chat_tokenizer

    async def go():
        stub, plain = _Stub("pen-http"), _Stub("pen-http-plain", penalties=False)
        shim, shim2 = HttpShim(stub, tiny_chat_tokenizer(), "tiny"), HttpShim(plain, tiny_chat_tokenizer(), "tiny")
        url, url2 = await shim.start(), await shim2.start()
        msgs = [{"role": "user", "content": "hello"}]
        try:
            async with aiohttp.ClientSession() as s:
                body = {"model": "tiny", "messages": msgs, "max_tokens": 4, "presence_penalty": -2.0,
                        "frequency_penalty": 2.0, "repetition_penalty": 0.5, "min_p": 1.0}
                async with s.post(url + "/v1/chat/completions", json=body) as r:
                    assert r.status == 200
                assert _key(stub.seen[-1]) == (-2.0, 2.0, 0.5, 1.0)
                for bad in ({"presence_penalty": 3}, {"repetition_penalty": -1.0}, {"min_p": -0.1},
                            {"frequency_penalty": "1"}):
                    async with s.post(url + "/v1/chat/completions",
                                      json={"model": "tiny", "messages": msgs, "max_tokens": 4, **bad}) as r:
                        assert r.status == 400 and "error" in await r.json()
                assert len(stub.seen) == 1
                for bad in NOT_OFF:
                    async with s.post(url2 + "/v1/chat/completions",
                                      json={"model": "tiny", "messages": msgs, "max_tokens": 4, **bad}) as r:
                        assert r.status == 400 and "not implemented" in (await r.json())["error"]["message"]
                assert not plain.seen
                async with s.post(url2 + "/v1/chat/completions",
                                  json={"model": "tiny", "messages": msgs, "max_tokens": 4, "min_p": 0}) as r:
                    assert r.status == 200
        finally:
            await shim.stop()
            await shim2.stop()
            stub.close()
            plain.close()
    asyncio.new_event_loop().run_until_complete(go())


def test_penalty_entry_validates_without_gpu():
    import ctypes as C

    from pipelinerl_b200 import _build, _lib
    _build.build(verbose=False)
    lib, P = _lib.load(), 0x1000
    assert lib.prl_apply_penalties(None, None) < 0 and b"NULL" in lib.prl_last_error()
    p = _lib.Penalties()
    p.B, p.V, p.prompt_stride, p.out_stride = 4, 16, 8, 8
    assert lib.prl_apply_penalties(C.byref(p), None) < 0 and b"NULL field" in lib.prl_last_error()
    for name, _ in _lib.Penalties._fields_:
        if _ is C.c_void_p:
            setattr(p, name, P)
    p.V = 0
    assert lib.prl_apply_penalties(C.byref(p), None) < 0 and b"bad shape" in lib.prl_last_error()

"""Top-k / top-p sampling, host side: the fp64 oracle against vLLM's own truncation (tests/golden/topk_topp_vllm.npz),
parameter validation, the capability gate of both clients, and argument checks of the C entry point (no GPU)."""
import asyncio
import types

import numpy as np
import pytest

from tests.helpers import tiny_chat_tokenizer
from tests.topk_topp_oracle import load_fixture, truncated_logprobs

TEST_LLM_PARAMETERS = {"max_tokens": 4, "temperature": 1.0, "top_p": 0.95, "top_k": 50}   # conf/base.yaml:52-57


def test_oracle_matches_vllm_fixture():
    fx = load_fixture()
    assert sorted(fx) == [640, 1000, 152064]
    n_checked = 0
    for V, f in fx.items():
        for r in range(len(f["T"])):
            o = truncated_logprobs(f["logits"][f["kind"][r]], f["T"][r], int(f["top_k"][r]), float(f["top_p"][r]))
            if o.margin > 1e-5:
                assert np.array_equal(o.mask, f["mask"][r]), (V, r)
                n_checked += 1
            ids = f["lp_ids"][r]
            ids = ids[ids >= 0]
            assert ids.size and f["mask"][r][ids].all()
            if np.array_equal(o.mask, f["mask"][r]):
                # vLLM's log_softmax is fp32: a few ulp of the log-normaliser (4e-6), and over more than a thousand kept
                # tokens its fp32 sum of exponentials drifts further (3.2e-5 at 152 064 kept tokens)
                atol = 4e-6 if o.mask.sum() <= 1000 else 5e-5
                np.testing.assert_allclose(o.logprobs[ids], f["lp"][r][: ids.size], rtol=1e-6, atol=atol)
    assert n_checked >= 180          # of 243 rows; the rest sit within 1e-5 of a boundary or split a tie group


def test_oracle_edge_cases():
    z = np.array([0.5, 3.0, 1.0, 3.0, -2.0, 1.0])
    o = truncated_logprobs(z, 1.0, 1, 1.0)                      # top-1 with a tie at the top: both kept
    assert o.mask.tolist() == [False, True, False, True, False, False]
    np.testing.assert_allclose(o.logprobs[1], -np.log(2.0))
    o = truncated_logprobs(z, 1.0, 3, 1.0)                      # 3rd largest is 1.0, tied: 4 kept
    assert o.mask.sum() == 4 and o.threshold == 1.0
    o = truncated_logprobs(z, 1.0, -1, 1e-6)                    # the largest value (and its tie) is always kept
    assert o.mask.sum() == 2
    o = truncated_logprobs(z, 1.0, 6, 1.0)                      # k >= V: off
    assert o.mask.all() and o.margin == np.inf


@pytest.mark.parametrize("params, want", [
    ({}, (-1, 1.0)), ({"top_k": None, "top_p": None}, (-1, 1.0)), ({"top_k": 0}, (0, 1.0)), ({"top_k": 50}, (50, 1.0)),
    ({"top_p": 1}, (-1, 1.0)), ({"top_p": 0.95, "top_k": 50}, (50, 0.95)),
])
def test_truncation_params_accepts(params, want):
    from pipelinerl_b200.engine import truncation_params
    assert truncation_params(params) == want
    assert truncation_params(params, greedy=True) == (-1, 1.0)


@pytest.mark.parametrize("params", [{"top_p": 0.0}, {"top_p": 1.5}, {"top_p": -0.1}, {"top_p": "0.9"}, {"top_k": -2},
                                    {"top_k": 2.5}, {"top_k": True}, {"top_k": "50"}])
def test_truncation_params_rejects(params):
    from pipelinerl_b200.engine import truncation_params
    with pytest.raises(ValueError):
        truncation_params(params)
    with pytest.raises(ValueError):                              # validated before the greedy reset, as vLLM does
        truncation_params(params, greedy=True)


class _StubServer:
    """Registered engine stand-in that lists the truncation features and records the SamplingParams it receives."""

    def __init__(self, name, features=frozenset({"top_k", "top_p"})):
        from pipelinerl_b200 import serving
        self.name, self.seen = name, []
        self.engine = types.SimpleNamespace(sampling_features=features, arena=types.SimpleNamespace(version=0))
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


def test_in_process_client_passes_truncation_to_an_engine_that_lists_it():
    from pipelinerl_b200 import serving
    stub = _StubServer("topkp-stub")
    try:
        assert serving.sampling_features("inproc://topkp-stub") == frozenset({"top_k", "top_p"})
        call = _generate("inproc://topkp-stub", TEST_LLM_PARAMETERS)
        assert call.output_length_tokens == 2
        sp = stub.seen[-1]
        assert (sp.top_k, sp.top_p, sp.temperature, sp.greedy, sp.max_tokens) == (50, 0.95, 1.0, False, 4)
        _generate("inproc://topkp-stub", {"max_tokens": 4, "temperature": 0.0, "top_p": 0.95, "top_k": 50})
        assert (stub.seen[-1].greedy, stub.seen[-1].top_k, stub.seen[-1].top_p) == (True, -1, 1.0)
        _generate("inproc://topkp-stub", {"max_tokens": 4, "temperature": 0.7})
        assert (stub.seen[-1].top_k, stub.seen[-1].top_p) == (-1, 1.0)
        n = len(stub.seen)
        for bad in ({"top_p": 0.0}, {"top_p": 1.5}, {"top_k": -2}, {"top_k": 2.5}, {"min_p": 0.1}, {"n": 2}):
            with pytest.raises(ValueError):
                _generate("inproc://topkp-stub", {"max_tokens": 4, **bad})
        assert len(stub.seen) == n                                 # nothing reached the engine
    finally:
        stub.close()


def test_in_process_client_refuses_truncation_the_engine_does_not_list():
    from pipelinerl_b200 import serving
    assert serving.sampling_features("inproc://nothing-registered") == frozenset()
    assert serving.sampling_features("http://elsewhere") == frozenset()
    stub = _StubServer("topk-only-stub", features=frozenset({"top_k"}))
    try:
        _generate("inproc://topk-only-stub", {"max_tokens": 4, "top_k": 20})
        assert stub.seen[-1].top_k == 20
        with pytest.raises(ValueError, match="top_p"):
            _generate("inproc://topk-only-stub", {"max_tokens": 4, "top_p": 0.9})
    finally:
        stub.close()


def test_http_shim_serves_truncation_when_the_engine_lists_it():
    import aiohttp
    from pipelinerl_b200.http_shim import HttpShim

    async def go():
        server = _StubServer("topkp-http-stub")
        shim = HttpShim(server, tiny_chat_tokenizer(), "tiny")
        url = await shim.start()
        msgs = [{"role": "user", "content": "hello"}]
        try:
            async with aiohttp.ClientSession() as s:
                body = {"model": "tiny", "messages": msgs, "logprobs": True, **TEST_LLM_PARAMETERS}
                async with s.post(url + "/v1/chat/completions", json=body) as r:
                    assert r.status == 200
                sp = server.seen[-1]
                assert (sp.top_k, sp.top_p, sp.greedy) == (50, 0.95, False)
                for bad in ({"top_p": 0.0}, {"top_p": 2.0}, {"top_k": -5}, {"top_k": 1.5}):
                    async with s.post(url + "/v1/chat/completions", json={"model": "tiny", "messages": msgs, **bad}) as r:
                        assert r.status == 400 and "error" in await r.json()
                assert len(server.seen) == 1
        finally:
            await shim.stop()
            server.close()
    asyncio.new_event_loop().run_until_complete(go())


def test_engines_without_truncation_refuse_it():
    """The fused sampling head and the TP engine list no truncation features; add_request refuses top-k / top-p there
    before touching any device state (checked here on bare instances: no GPU)."""
    from pipelinerl_b200.engine import DecodeEngine, SamplingParams
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    from tests.helpers import tiny_cfg
    assert DecodeEngine.sampling_features.fget(types.SimpleNamespace(fused_head=False)) == frozenset({"top_k", "top_p"})
    assert DecodeEngine.sampling_features.fget(types.SimpleNamespace(fused_head=True)) == frozenset()
    assert TPDecodeEngine.sampling_features == frozenset()
    for cls, fused in ((DecodeEngine, True), (TPDecodeEngine, False)):
        eng = object.__new__(cls)
        eng.cfg, eng.max_seq_len, eng.max_new, eng.fused_head = tiny_cfg("gqa2"), 128, 32, fused
        eng._greedy, eng._temperature = False, 1.0
        for sp in (SamplingParams(max_tokens=4, top_k=50), SamplingParams(max_tokens=4, top_p=0.95)):
            with pytest.raises(ValueError, match="not implemented by this engine"):
                eng.add_request([1, 2, 3], sp)
        with pytest.raises(ValueError, match="top_p"):
            eng.add_request([1, 2, 3], SamplingParams(max_tokens=4, top_p=0.0))


@pytest.fixture(scope="module")
def built_lib():
    from pipelinerl_b200 import _build, _lib
    _build.build(verbose=False)
    return _lib.load()


def test_topkp_entry_validates_arguments_without_gpu(built_lib):
    lib, P = built_lib, 0x1000
    ws = int(lib.prl_sample_topkp_workspace_bytes(64, 152064))
    assert ws == int(lib.prl_sample_workspace_bytes(64)) > 0

    def call(logits=P, B=4, V=1000, k=P, p=P, out_ids=P, ws_ptr=P, ws_bytes=1 << 20):
        return lib.prl_sample_logprob_topkp_rows(logits, B, V, P, P, k, p, 0, 0, out_ids, P, None, None, None, ws_ptr,
                                                 ws_bytes, None)
    cases = [(dict(logits=None), b"NULL"), (dict(k=None), b"NULL"), (dict(p=None), b"NULL"), (dict(out_ids=None), b"NULL"),
             (dict(B=0), b"bad shape"), (dict(V=0), b"bad shape"), (dict(B=70000), b"bad shape"),
             (dict(V=262145), b"262144"), (dict(ws_ptr=None), b"workspace"), (dict(ws_bytes=16), b"workspace")]
    for kw, needle in cases:
        assert call(**kw) < 0, kw
        assert needle in lib.prl_last_error(), (kw, lib.prl_last_error())

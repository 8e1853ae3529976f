"""Stop strings and min_tokens, host side: the device rule's restatement against vLLM's own detokenizer / check_stop /
OutputProcessor (tests/golden/stop_strings_vllm.json), the token byte table, the min_tokens ban set, and the capability
gate and validation of both clients and the shim (no GPU)."""
import asyncio
import types

import numpy as np
import pytest

from tests.stop_string_oracle import (fixture_tokenizer, host_rule, host_text, min_tokens_fixture, slot_params,
                                      stop_string_cases)


@pytest.fixture(scope="module")
def table():
    from pipelinerl_b200.engine import token_byte_table
    return token_byte_table(fixture_tokenizer())


@pytest.mark.parametrize("case", stop_string_cases(), ids=lambda c: c["name"])
def test_oracle_matches_vllm(case, table):
    eos_id, row, _, sp = slot_params(case)
    n, finish, reason, match = host_rule(case["ids"], table, eos_id, row, sp)
    assert (n, finish, reason) == (case["n_out"], case["finish_reason"], case["stop_reason"])
    assert host_text(case["ids"][:n], finish, match, table, sp) == case["output_text"]


def test_fixture_covers_the_rule():
    by = {c["name"]: c for c in stop_string_cases()}
    assert by["later_string_matches_first_rl"]["stop_reason"] == "world"
    assert by["match_ends_at_min_tokens_does_not_fire"]["stop_reason"] == " here"
    assert by["match_ends_at_min_tokens_does_not_fire"]["n_out"] > by["match_ends_at_min_tokens_does_not_fire"]["min_tokens"] + 1
    assert by["match_starts_in_min_tokens_prefix"]["stop_reason"] == "here:"
    assert by["string_at_last_allowed_token"]["finish_reason"] == "stop"
    assert by["eos_completes_string_rl"]["stop_reason"] == "Done.<|im_end|>"
    assert by["eos_completes_string_default"]["stop_reason"] is None
    assert isinstance(by["stop_id_and_string_rl"]["stop_reason"], int)
    assert by["stop_id_then_string_same_token_rl"]["stop_reason"] == "="
    assert by["stop_id_then_string_same_token_default"]["stop_reason"] != "="


def test_min_tokens_ban_set_matches_vllm():
    """DecodeEngine.min_tokens_ban_row is vLLM's all_stop_token_ids, and MinTokensLogitsProcessor bans exactly it while
    the output is short of min_tokens (ignore_eos keeps the eos in the set)."""
    from pipelinerl_b200.engine import DecodeEngine, SamplingParams, stop_ids_from_generation_config
    tok = fixture_tokenizer()
    eos = tok.convert_tokens_to_ids("<|im_end|>")
    fx = min_tokens_fixture()
    for r in fx["rows"]:
        e, extra = stop_ids_from_generation_config({} if r["gen_eos"] is None else {"eos_token_id": r["gen_eos"]}, eos)
        eng = types.SimpleNamespace(eos_id=e, stop_ids=extra)
        ban = DecodeEngine.min_tokens_ban_row(eng, SamplingParams(stop_token_ids=tuple(r["stop_ids"]),
                                                                  ignore_eos=r["ignore_eos"]))
        assert sorted(ban) == r["all_stop_token_ids"]
        assert r["banned"] == (sorted(ban) if r["n_out"] < r["min_tokens"] else [])


def test_token_byte_table_matches_decode(table):
    tok = fixture_tokenizer()
    data, offsets, special = table
    from pipelinerl_b200.engine import utf8_text
    rng = np.random.default_rng(0)
    V = len(tok)
    assert len(special) == V and special[tok.convert_tokens_to_ids("<|im_end|>")] == 1
    assert special[tok.convert_tokens_to_ids("<think>")] == 0
    for _ in range(200):
        ids = rng.integers(0, V, size=int(rng.integers(1, 12))).tolist()
        for skip in (False, True):
            b = b"".join(bytes(data[offsets[t]:offsets[t + 1]]) for t in ids if not (skip and special[t]))
            want = tok.decode(ids, skip_special_tokens=skip)
            got = b.decode("utf-8", errors="replace")
            assert got == want, (ids, skip)
            assert want.startswith(utf8_text(b))
    # the model's vocabulary may be larger than the tokenizer's: those ids have no bytes
    from pipelinerl_b200.engine import token_byte_table
    d2, o2, s2 = token_byte_table(tok, V + 5)
    assert len(o2) == V + 6 and o2[-1] == o2[V] and np.array_equal(d2[:o2[V]], data[:offsets[V]])


def test_token_byte_table_refuses_other_tokenizers():
    from pipelinerl_b200.engine import token_byte_table
    from tests.helpers import tiny_chat_tokenizer
    with pytest.raises(ValueError, match="byte-level"):
        token_byte_table(tiny_chat_tokenizer())
    with pytest.raises(ValueError):
        token_byte_table(object())


def test_kmp_failure():
    from pipelinerl_b200.engine import kmp_failure
    assert kmp_failure(b"ababaca") == [0, 0, 1, 2, 3, 0, 1]
    assert kmp_failure(b"aaaa") == [0, 1, 2, 3]


@pytest.mark.parametrize("params", [{"stop": ""}, {"stop": [""]}, {"stop": 5}, {"stop": ["a", 3]}])
def test_stop_param_rejects(params):
    from pipelinerl_b200.engine import stop_strings_param
    with pytest.raises(ValueError, match="stop"):
        stop_strings_param(params)


def test_params_accept_and_refuse():
    from pipelinerl_b200.engine import check_stop_flags, min_tokens_param, stop_strings_param
    assert stop_strings_param({"stop": "x"}) == ("x",) and stop_strings_param({}) == ()
    assert min_tokens_param({"min_tokens": 4}, 4) == 4 and min_tokens_param({}, 1) == 0
    for bad in (-1, 5, 1.0, True):
        with pytest.raises(ValueError, match="min_tokens"):
            min_tokens_param({"min_tokens": bad}, 4)
    check_stop_flags(("x",), True, False)
    check_stop_flags(("x",), False, True)
    check_stop_flags((), True, True)
    for pair in ((True, True), (False, False)):
        with pytest.raises(ValueError, match="include_stop_str_in_output"):
            check_stop_flags(("x",), *pair)


def test_capabilities():
    from pipelinerl_b200 import serving
    from pipelinerl_b200.tp_engine import TPDecodeEngine
    assert TPDecodeEngine.supports_stop_strings is False and TPDecodeEngine.supports_min_tokens is False
    eng = types.SimpleNamespace(sampling_features=frozenset(), supports_stop_token_ids=True,
                                supports_stop_strings=True, supports_min_tokens=True)
    assert serving.engine_features(eng) == frozenset({"stop_token_ids", "stop", "min_tokens"})


class _Stub:
    def __init__(self, name, stop=True, min_tokens=True):
        from pipelinerl_b200 import serving
        from pipelinerl_b200.engine import DecodeEngine
        self.name, self.seen = name, []
        bare = types.SimpleNamespace(max_stop_strings=2, max_stop_str_bytes=8, supports_stop_strings=stop)
        self.engine = types.SimpleNamespace(sampling_features=frozenset(), arena=types.SimpleNamespace(version=0),
                                            supports_stop_token_ids=True, supports_stop_strings=stop,
                                            supports_min_tokens=min_tokens,
                                            stop_string_rows=lambda sp: DecodeEngine.stop_string_rows(bare, sp))
        self.on_step_boundary, self.error = None, None
        serving._REGISTRY[name] = self

    def close(self):
        from pipelinerl_b200 import serving
        serving._REGISTRY.pop(self.name, None)

    async def generate(self, prompt_ids, params):
        self.seen.append(params)
        hit = bool(params.stop)
        return types.SimpleNamespace(output_ids=[5, 6], output_logprobs=[-0.5, -0.25],
                                     finish_reason="stop" if hit else "length",
                                     stop_reason=params.stop[0] if hit else None,
                                     output_text="cut" if hit else None, model_version=0)


def _generate(base_url, parameters, collect_logprobs=True):
    from pipelinerl_b200.async_llm import llm_async_generate
    from pipelinerl_b200.llm import Prompt, SyntheticTokenizer, TrainableLLM
    llm = TrainableLLM(base_url, "m", parameters=parameters, tokenizer=SyntheticTokenizer())
    llm.collect_logprobs = collect_logprobs
    return asyncio.run(llm_async_generate(llm, Prompt(messages=[{"role": "user", "content": "hi"}])))


def test_in_process_client_gate():
    stub, plain = _Stub("ss-stub"), _Stub("ss-plain", stop=False, min_tokens=False)
    try:
        call = _generate("inproc://ss-stub", {"max_tokens": 4, "stop": ["</a>"], "min_tokens": 2})
        sp = stub.seen[-1]
        assert (sp.stop, sp.min_tokens, sp.include_stop_str_in_output, sp.skip_special_tokens) == (("</a>",), 2, True, False)
        assert call.output.content == "cut" and call.llm_info["stop_reason"] == "</a>"
        _generate("inproc://ss-stub", {"max_tokens": 4, "stop": "x"}, collect_logprobs=False)
        assert (stub.seen[-1].include_stop_str_in_output, stub.seen[-1].skip_special_tokens) == (False, True)
        n = len(stub.seen)
        for bad in ({"stop": ["a", "b", "c"]}, {"stop": ["123456789"]}, {"stop": [""]}, {"min_tokens": 5},
                    {"min_tokens": -1}):
            with pytest.raises(ValueError):
                _generate("inproc://ss-stub", {"max_tokens": 4, **bad})
        with pytest.raises(ValueError, match="include_stop_str_in_output"):
            _generate("inproc://ss-stub", {"max_tokens": 4, "stop": "x", "skip_special_tokens": False},
                      collect_logprobs=False)
        assert len(stub.seen) == n
        with pytest.raises(ValueError, match="stop strings are not implemented by this engine"):
            _generate("inproc://ss-plain", {"max_tokens": 4, "stop": ["x"]})
        with pytest.raises(ValueError, match="min_tokens"):
            _generate("inproc://ss-plain", {"max_tokens": 4, "min_tokens": 1})
        _generate("inproc://ss-plain", {"max_tokens": 4, "min_tokens": 0})
        assert plain.seen[-1].min_tokens == 0 and not plain.seen[-1].stop
    finally:
        stub.close()
        plain.close()


def test_http_shim_gate():
    import aiohttp

    from pipelinerl_b200.http_shim import HttpShim
    from tests.helpers import tiny_chat_tokenizer

    async def go():
        stub, plain = _Stub("ss-http"), _Stub("ss-http-plain", stop=False, min_tokens=False)
        shim, shim2 = HttpShim(stub, tiny_chat_tokenizer(), "tiny"), HttpShim(plain, tiny_chat_tokenizer(), "tiny")
        url, url2 = await shim.start(), await shim2.start()
        msgs = [{"role": "user", "content": "hello"}]
        rl = {"include_stop_str_in_output": True, "skip_special_tokens": False}
        try:
            async with aiohttp.ClientSession() as s:
                body = {"model": "tiny", "messages": msgs, "max_tokens": 4, "stop": ["</a>"], "min_tokens": 1, **rl}
                async with s.post(url + "/v1/chat/completions", json=body) as r:
                    assert r.status == 200
                    choice = (await r.json())["choices"][0]
                assert (choice["finish_reason"], choice["stop_reason"], choice["message"]["content"]) == \
                    ("stop", "</a>", "cut")
                for bad in ({"stop": ["x"], "include_stop_str_in_output": True}, {"stop": [""]},
                            {"stop": ["a", "b", "c"], **rl}, {"min_tokens": 9}):
                    async with s.post(url + "/v1/chat/completions",
                                      json={"model": "tiny", "messages": msgs, "max_tokens": 4, **bad}) as r:
                        assert r.status == 400 and "error" in await r.json()
                assert len(stub.seen) == 1
                for bad, word in (({"stop": ["x"], **rl}, "stop strings"), ({"min_tokens": 2}, "min_tokens")):
                    async with s.post(url2 + "/v1/chat/completions",
                                      json={"model": "tiny", "messages": msgs, "max_tokens": 4, **bad}) as r:
                        assert r.status == 400 and word in (await r.json())["error"]["message"]
                assert not plain.seen
        finally:
            await shim.stop()
            await shim2.stop()
            stub.close()
            plain.close()
    asyncio.new_event_loop().run_until_complete(go())


def test_engine_state_keeps_its_layout():
    """The string fields live in prl_stop_strings; prl_engine_state still ends with the stop-id fields."""
    from pipelinerl_b200 import _lib
    assert [n for n, _ in _lib.EngineState._fields_][-1] == "stop_reason"
    assert [n for n, _ in _lib.StopStrings._fields_] == [
        "tok_bytes", "tok_offsets", "tok_special", "vocab", "stop_str", "stop_str_fail", "stop_str_len", "n_stop_str",
        "max_stop_str", "stop_str_stride", "stop_str_flags", "stop_str_state", "stop_str_match", "min_tokens"]


def test_new_entry_points_validate_without_gpu():
    import ctypes as C

    from pipelinerl_b200 import _build, _lib
    _build.build(verbose=False)
    lib, P = _lib.load(), 0x1000
    assert lib.prl_ban_min_tokens(None, 4, 16, P, P, P, 2, P, None) < 0 and b"NULL" in lib.prl_last_error()
    assert lib.prl_ban_min_tokens(P, 4, 16, P, P, P, 0, P, None) < 0 and b"bad shape" in lib.prl_last_error()
    s = _lib.EngineState()
    s.B = 4
    for name in ("sampled", "sampled_logprobs", "tokens", "positions", "seq_lens", "active", "prompt_buf", "prompt_len",
                 "out_ids", "out_logprobs", "gen_count", "max_new", "finished"):
        setattr(s, name, P)
    x = _lib.StopStrings()
    x.tok_bytes = P
    assert lib.prl_advance_state_strings(C.byref(s), C.byref(x), None) < 0 and b"tok_bytes" in lib.prl_last_error()
    s.stop_ids = P
    assert lib.prl_advance_state_strings(C.byref(s), None, None) < 0 and b"n_stop" in lib.prl_last_error()

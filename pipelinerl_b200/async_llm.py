"""Client side of the plugin surface: `llm_async_generate` and `make_training_text`
(reference: pipelinerl/async_llm.py:86-212 and :215-346)."""
from __future__ import annotations

from .engine import (SamplingParams, check_stop_flags, min_tokens_param, penalty_params, requested_penalties,
                     requested_truncation, stop_strings_param, stop_token_ids_param, truncation_params)
from .llm import LLMCall, LLMOutput, Prompt, TokenLogprob, TrainableLLM
from .rollouts import TrainingText, apply_rollout_reward
from .serving import resolve, sampling_features

MASKED_TOKEN_ID = -100


class RetryableAbortedCompletionError(TimeoutError):
    """Abort-shaped completion that should be retried instead of treated as data."""


def _field(obj, name):
    """tool calls arrive as pydantic objects (litellm types in the reference) or as plain dicts"""
    return obj[name] if isinstance(obj, dict) else getattr(obj, name)


def _token_ids(encoded) -> list[int]:
    """apply_chat_template(tokenize=True) returns a list of ids with the transformers the reference pins (4.57) and a
    BatchEncoding with transformers >= 5: accept both."""
    if hasattr(encoded, "keys") and "input_ids" in encoded.keys():
        encoded = encoded["input_ids"]
    return list(encoded)


def _chat_kwargs(llm: TrainableLLM, prompt: Prompt) -> dict:
    kw = dict(llm.chat_template_kwargs or {})
    if prompt.tools:
        kw["tools"] = prompt.tools
    return kw


def _reject_unsupported_sampling(params: dict, features: frozenset = frozenset()
                                 ) -> tuple[int, float, tuple[int, ...], tuple[float, float, float, float]]:
    """Sampling features the engine does not implement must fail loudly, exactly as http_shim.py answers 400 for them:
    a silently ignored top_p / top_k / stop would make the recorded logprobs those of a different distribution than the
    one the request asked for.  top_k / top_p are accepted when the target engine lists them in `features` (the unfused
    single-GPU DecodeEngine does; the reference's eval handles send top_p 0.95 / top_k 50, conf/base.yaml:52-57), and
    stop_token_ids when it lists "stop_token_ids"; they are validated as vLLM validates them.  Stop strings and
    min_tokens > 0 are refused unless it lists "stop" / "min_tokens" (stop_params validates them), and
    presence_penalty, frequency_penalty, repetition_penalty and min_p away from their defaults unless it lists each of
    them (validated as vLLM validates them).
    Returns the request's (top_k, top_p, stop_token_ids, (presence, frequency, repetition, min_p))."""
    greedy = float(params.get("temperature", 1.0)) <= 0
    top_k, top_p = truncation_params(params, greedy=greedy)
    missing = requested_truncation(top_k, top_p) - features
    if missing:
        raise ValueError(f"{' / '.join(sorted(missing))} sampling is not implemented by this engine")
    stop_ids = stop_token_ids_param(params)
    if stop_ids and "stop_token_ids" not in features:
        raise ValueError("stop token ids are not implemented by this engine (eos only)")
    if stop_strings_param(params) and "stop" not in features:
        raise ValueError("stop strings are not implemented by this engine (stop token ids are)")
    if int(params.get("n", 1)) != 1:
        raise ValueError("n > 1 completions per request is not implemented (the actor issues `attempts` requests)")
    penalties = penalty_params(params, greedy=greedy)
    missing = requested_penalties(penalties) - features
    if missing:
        raise ValueError(f"sampling parameter {' / '.join(sorted(missing))} is not implemented by this engine")
    return top_k, top_p, stop_ids, penalties


def stop_params(params: dict, features: frozenset, max_tokens: int,
                collect_logprobs: bool) -> tuple[tuple[str, ...], int, bool, bool]:
    """(stop, min_tokens, include_stop_str_in_output, skip_special_tokens) of a request.  The flags are what the
    reference's client sends: (True, False) when it collects logprobs, else whatever `params` says, vLLM's defaults
    (False, True) when it says nothing; with stop strings, a mixed pair is refused.  min_tokens > 0 is refused unless
    the engine lists "min_tokens".  Raises ValueError."""
    stop = stop_strings_param(params)
    min_tokens = min_tokens_param(params, max_tokens)
    if min_tokens and "min_tokens" not in features:
        raise ValueError("min_tokens is not implemented by this engine")
    if collect_logprobs:
        include, skip = True, False
    else:
        include = bool(params.get("include_stop_str_in_output", False))
        skip = bool(params.get("skip_special_tokens", True))
    check_stop_flags(stop, include, skip)
    return stop, min_tokens, include, skip


async def llm_async_generate(llm: TrainableLLM, prompt: Prompt, session=None,
                             max_tokens_override: int | None = None) -> LLMCall:
    """One completion.  `session` (an aiohttp.ClientSession in the reference) is accepted and unused: the
    engine is in-process.  Returns an LLMCall with .output.content, .logprobs[i].{token_id, logprob},
    .prompt_length_tokens, .output_length_tokens and .llm_info['finish_reason'] in {stop, length}."""
    tok = llm.load_tokenizer()
    prompt_ids = prompt.token_ids or _token_ids(tok.apply_chat_template(prompt.messages, add_generation_prompt=True,
                                                                        **_chat_kwargs(llm, prompt)))
    params = llm.parameters
    features = sampling_features(llm.base_url)
    top_k, top_p, stop_ids, penalties = _reject_unsupported_sampling(params, features)
    max_tokens = int(max_tokens_override if max_tokens_override is not None else params.get("max_tokens", 16))
    stop, min_tokens, include, skip = stop_params(params, features, max_tokens, bool(llm.collect_logprobs))
    temperature = float(params.get("temperature", 1.0))
    sp = SamplingParams(max_tokens=max_tokens, temperature=temperature if temperature > 0 else 1.0,
                        greedy=temperature <= 0, ignore_eos=bool(params.get("ignore_eos", False)), top_k=top_k,
                        top_p=top_p, stop_token_ids=stop_ids, stop=stop, min_tokens=min_tokens,
                        include_stop_str_in_output=include, skip_special_tokens=skip)
    sp.presence_penalty, sp.frequency_penalty, sp.repetition_penalty, sp.min_p = penalties
    server = resolve(llm.base_url)
    if stop_ids:
        server.engine.stop_row(sp)      # out-of-vocabulary ids or too many: ValueError here, not on the engine thread
    if stop:
        server.engine.stop_string_rows(sp)   # past the engine's row limits: ValueError here as well
    req = await server.generate(list(prompt_ids), sp)
    # with stop strings the content is vLLM's output_text (cut at the string), which the engine computed
    content = req.output_text if stop and getattr(req, "output_text", None) is not None else tok.decode(req.output_ids)
    call = llm.log_output(prompt, LLMOutput(content=content), count_tokens=False)
    call.prompt_length_tokens = len(prompt_ids)
    call.output_length_tokens = len(req.output_ids)
    call.llm_info["finish_reason"] = req.finish_reason
    call.llm_info["stop_reason"] = getattr(req, "stop_reason", None)
    call.llm_info["model_version"] = req.model_version
    call.llm_info["prompt_token_ids"] = list(prompt_ids)
    if llm.collect_logprobs:
        call.logprobs = [TokenLogprob(token_id=t, logprob=lp) for t, lp in zip(req.output_ids, req.output_logprobs)]
    return call


def make_training_text(llm: TrainableLLM, llm_call: LLMCall) -> TrainingText:
    """input_ids = prompt ids + generated ids; labels mask the prompt; logprobs are the sampler's."""
    finish_reason = llm_call.llm_info.get("finish_reason")
    if finish_reason == "abort":
        raise RetryableAbortedCompletionError(f"Aborted completion for prompt {llm_call.prompt.id} should be retried")
    if not llm_call.logprobs:
        raise ValueError("Logprobs are required to make training data for RL")
    tok = llm.load_tokenizer()
    kw = _chat_kwargs(llm, llm_call.prompt)
    prompt_ids = llm_call.llm_info.get("prompt_token_ids")
    if prompt_ids is None:
        prompt_ids = _token_ids(tok.apply_chat_template(llm_call.prompt.messages, add_generation_prompt=True, **kw))
    prompt_text = tok.apply_chat_template(llm_call.prompt.messages, tokenize=False, add_generation_prompt=True, **kw)
    assistant: dict = {"role": "assistant", "content": llm_call.output.content or ""}
    if llm_call.output.tool_calls:   # rendered by the chat template exactly as the reference passes them (:227-238)
        assistant["tool_calls"] = [{"id": _field(tc, "id"), "type": "function",
                                    "function": {"name": _field(_field(tc, "function"), "name"),
                                                 "arguments": _field(_field(tc, "function"), "arguments")}}
                                   for tc in llm_call.output.tool_calls]
    full = llm_call.prompt.messages + [assistant]
    text = tok.apply_chat_template(full, tokenize=False, **kw)
    output_text = text[len(prompt_text):]
    bos = getattr(tok, "bos_token", None)
    if bos and text.startswith(bos):
        text = text[len(bos):]
    gen = [lp.token_id for lp in llm_call.logprobs]
    if finish_reason is not None:
        finished = finish_reason != "length"
    else:
        eos = getattr(tok, "eos_token", "") or ""
        finished = bool(eos) and (llm_call.output.content or "").endswith(eos)
    return TrainingText(text=text, n_predicted=len(output_text), input_ids=list(prompt_ids) + gen,
                        labels=[MASKED_TOKEN_ID] * len(prompt_ids) + gen,
                        logprobs=[lp.logprob for lp in llm_call.logprobs], finished=finished,
                        prompt_tokens=llm_call.prompt_length_tokens, output_tokens=llm_call.output_length_tokens)


def make_training_texts_from_llm_calls(llm: TrainableLLM, llm_calls: list[LLMCall], reward: float | None = None):
    texts = [make_training_text(llm, c) for c in llm_calls]
    return apply_rollout_reward(texts, reward) if reward is not None else texts

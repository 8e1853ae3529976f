"""Golden fixtures for stop strings and min_tokens in the token step, by executing vLLM 0.22's own code.

    python tests/golden/make_golden_stop_strings.py      (authoring container: needs vllm 0.22 and tokenizers)

1. stop_tokenizer.json: a byte-level BPE tokenizer trained here on an inline deterministic corpus (ASCII plus 2-, 3- and
   4-byte UTF-8 characters, so that tokens split characters), with <|endoftext|> / <|im_end|> as special tokens and
   <think> as a non-special added token.  Its vocabulary fits the tiny GPU configs (<= 640 ids).
2. stop_strings_vllm.json: scripted output ids run through vLLM's SamplingParams (update_from_generation_config),
   check_stop (vllm/v1/core/sched/utils.py), IncrementalDetokenizer.from_new_request / update (the fast, DecodeStream
   detokenizer) and the re-labelling statements of OutputProcessor.process_outputs (vllm/v1/engine/output_processor.py,
   the `if stop_string:` block after `detokenizer.update`), cut out of vLLM's source with `ast` and executed.
   Recorded per case: output length, finish_reason, stop_reason, output_text.
3. min_tokens_vllm.json: MinTokensLogitsProcessor.add_request / apply over scripted output lengths (the banned ids and
   the masked rows), and the processed logprobs of the masked rows under the sampler functions the top-k / top-p
   fixture ran (greedy, plain, top-k, top-p); the wide-vocabulary logits are a seed plus SHA-256 as in
   topk_topp_vllm.npz.
"""
import ast
import hashlib
import inspect
import json
import textwrap
from pathlib import Path

import numpy as np

HERE = Path(__file__).parent
SPECIAL = ["<|endoftext|>", "<|im_end|>"]
CORPUS = [
    "The answer is 42. </answer> Done.", "Let me think <think> about it </think> carefully.",
    "Stop here: STOP. Or there: END!", "café naïve résumé — déjà vu", "日本語のテキストと中文字符", "emoji 😀 🚀 🎉 and ∑ ∫ √",
    "<answer>7</answer>", "abababcabab abcabd", "hello world, hello there", "x = y + z; return x;",
]


def train_tokenizer():
    from tokenizers import AddedToken, Tokenizer, decoders, models, pre_tokenizers, trainers
    tk = Tokenizer(models.BPE())
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=True)
    tk.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=420, min_frequency=1, special_tokens=SPECIAL,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False)
    tk.train_from_iterator(CORPUS * 3, trainer=trainer)
    tk.add_tokens([AddedToken("<think>", special=False, normalized=False)])
    return tk


def hf_tokenizer(path):
    from transformers import PreTrainedTokenizerFast
    return PreTrainedTokenizerFast(tokenizer_file=str(path), eos_token="<|im_end|>")


def ids_of(tok, *parts):
    out = []
    for p in parts:
        out += [p] if isinstance(p, int) else tok.encode(p, add_special_tokens=False)
    return out


def _relabel():
    """The statements of OutputProcessor.process_outputs that turn a matched stop string into finish_reason / stop_reason,
    cut out of vLLM's source."""
    from vllm.v1.engine import output_processor
    src = textwrap.dedent(inspect.getsource(output_processor.OutputProcessor.process_outputs))
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.If) and isinstance(node.test, ast.Name) and node.test.id == "stop_string":
            return compile(ast.Module(body=[node], type_ignores=[]), "output_processor.py", "exec")
    raise RuntimeError("stop-string block not found in OutputProcessor.process_outputs")


def run_case(tok, case, relabel):
    from vllm import SamplingParams
    from vllm.v1.core.sched.utils import check_stop
    from vllm.v1.engine import EngineCoreRequest, FinishReason
    from vllm.v1.engine.detokenizer import FastIncrementalDetokenizer, IncrementalDetokenizer
    from vllm.v1.request import RequestStatus
    include, skip = case["flags"]
    sp = SamplingParams(max_tokens=case["max_tokens"], stop=list(case["stop"]), stop_token_ids=list(case["stop_ids"]),
                        min_tokens=case["min_tokens"], include_stop_str_in_output=include, skip_special_tokens=skip)
    gen = {} if case["gen_eos"] is None else {"eos_token_id": case["gen_eos"]}
    sp.update_from_generation_config(gen, case["eos"])
    prompt = tok.encode("hello world", add_special_tokens=False)
    req = EngineCoreRequest(request_id="r", prompt_token_ids=prompt, mm_features=None, sampling_params=sp,
                            pooling_params=None, arrival_time=0.0, lora_request=None, cache_salt=None,
                            data_parallel_rank=None)
    det = IncrementalDetokenizer.from_new_request(tok, req)
    assert isinstance(det, FastIncrementalDetokenizer)

    class _Req:  # what check_stop reads of a vllm.v1.request.Request
        sampling_params, pooling_params = sp, None
        max_tokens, output_token_ids, status, stop_reason = sp.max_tokens, [], RequestStatus.RUNNING, None
        num_output_tokens = property(lambda self: len(self.output_token_ids))
        num_tokens = property(lambda self: len(prompt) + len(self.output_token_ids))
    r = _Req()
    for t in case["ids"]:
        r.output_token_ids.append(t)
        done = check_stop(r, max_model_len=1 << 20)
        finish_reason = {RequestStatus.FINISHED_STOPPED: FinishReason.STOP,
                         RequestStatus.FINISHED_LENGTH_CAPPED: FinishReason.LENGTH}.get(r.status) if done else None
        stop_reason = r.stop_reason
        stop_string = det.update([t], finish_reason == FinishReason.STOP)
        scope = dict(stop_string=stop_string, finish_reason=finish_reason, stop_reason=stop_reason, FinishReason=FinishReason)
        exec(relabel, scope)
        if scope["finish_reason"] is not None:
            fr = {FinishReason.STOP: "stop", FinishReason.LENGTH: "length"}[scope["finish_reason"]]
            return dict(case, n_out=len(r.output_token_ids), finish_reason=fr, stop_reason=scope["stop_reason"],
                        output_text=det.output_text, all_stop_token_ids=sorted(sp.all_stop_token_ids))
    raise AssertionError(f"{case['name']}: scripted ids ran out before the request finished")


def cases(tok):
    eos, end = tok.convert_tokens_to_ids("<|im_end|>"), tok.convert_tokens_to_ids("<|endoftext|>")
    think = tok.convert_tokens_to_ids("<think>")
    RL, DEF = (True, False), (False, True)
    base = dict(eos=eos, gen_eos=None, stop_ids=[], min_tokens=0, max_tokens=40, flags=RL)
    c = []

    def add(name, parts, **kw):
        d = dict(base, name=name, **kw)
        d["ids"] = ids_of(tok, *parts) + ids_of(tok, " filler text that never stops", eos)
        c.append(d)
    for fl, tag in ((RL, "rl"), (DEF, "default")):
        add(f"spans_tokens_{tag}", ["The answer is 42. </answer> Done."], stop=["</answer>"], flags=fl)
        add(f"extra_text_after_{tag}", ["Stop here: STOP. Or"], stop=["STO"], flags=fl)
        add(f"multibyte_split_{tag}", ["emoji 😀 🚀 and"], stop=["😀 🚀"], flags=fl)
        add(f"later_string_matches_first_{tag}", ["hello world, hello there"], stop=["there", "world"], flags=fl)
        add(f"two_strings_one_token_order_{tag}", ["abababcabab abcabd"], stop=["abc", "bab"], flags=fl)
        add(f"eos_completes_string_{tag}", ["Done.", eos], stop=["Done.<|im_end|>"], flags=fl)
        add(f"special_inside_string_{tag}", ["x", end, "y = 1"], stop=["<|endoftext|>y"], flags=fl)
        add(f"special_skipped_joins_{tag}", ["ab", end, "cd"], stop=["abcd"], flags=fl)
        add(f"added_token_inside_{tag}", ["Let me", think, " about it"], stop=["<think> ab"], flags=fl)
        add(f"ends_on_eos_without_match_{tag}", ["hello there", eos], stop=["zzz"], flags=fl)
        add(f"stop_id_and_string_{tag}", ["x = y + z; return x;"], stop=["return"], stop_ids=[ids_of(tok, " y")[0]],
            flags=fl)
        add(f"stop_id_then_string_same_token_{tag}", ["x = y + z;"], stop=["="], stop_ids=ids_of(tok, " =")[:1],
            flags=fl)
    n2 = len(ids_of(tok, "Stop", " here"))
    add("match_starts_in_min_tokens_prefix", ["Stop", " here", ":", " STOP"], stop=["here:"], min_tokens=n2)
    add("match_ends_at_min_tokens_does_not_fire", ["Stop", " here", ":", " here:"], stop=[" here"], min_tokens=n2)
    add("min_tokens_defers_eos", ["Done.", eos, " more", eos], stop=["zzz"], min_tokens=4)
    add("min_tokens_defers_eos_no_strings", ["Done.", eos, " more"], stop=[], min_tokens=4)
    add("gen_config_eos_in_ban_and_min", ["a", end, "b"], stop=[], min_tokens=3, gen_eos=[eos, end])
    last = ids_of(tok, "hello world, hello there")
    add("string_at_last_allowed_token", ["hello world, hello there"], stop=["there"], max_tokens=len(last))
    add("string_and_length_elsewhere", ["hello world, hello there"], stop=["zzz"], max_tokens=len(last))
    add("single_str_not_list", ["Or there: END!"], stop=["END"], flags=DEF)
    return c


def min_tokens_cases(tok):
    """MinTokensLogitsProcessor on a batch: which logits get -inf at which output lengths, then processed logprobs."""
    import torch
    from vllm import SamplingParams
    from vllm.v1.sample.logits_processor.builtin import MinTokensLogitsProcessor
    from vllm.v1.sample.ops.topk_topp_sampler import apply_top_k_top_p
    eos, end = tok.convert_tokens_to_ids("<|im_end|>"), tok.convert_tokens_to_ids("<|endoftext|>")
    rows = [dict(min_tokens=4, n_out=0, stop_ids=[], gen_eos=None, ignore_eos=False, top_k=-1, top_p=1.0, T=1.0),
            dict(min_tokens=4, n_out=3, stop_ids=[7], gen_eos=[eos, end], ignore_eos=True, top_k=-1, top_p=1.0, T=0.7),
            dict(min_tokens=4, n_out=4, stop_ids=[7], gen_eos=None, ignore_eos=False, top_k=-1, top_p=1.0, T=1.0),
            dict(min_tokens=2, n_out=1, stop_ids=[9, 11], gen_eos=None, ignore_eos=False, top_k=20, top_p=1.0, T=1.0),
            dict(min_tokens=2, n_out=0, stop_ids=[], gen_eos=[eos, end], ignore_eos=False, top_k=-1, top_p=0.9, T=1.0),
            dict(min_tokens=5, n_out=2, stop_ids=[3], gen_eos=None, ignore_eos=False, top_k=-1, top_p=1.0, T=0.0)]
    V, seed = 4096, 20260
    raw = hashlib.sha256(f"min_tokens:{seed}".encode()).digest()
    g = torch.Generator().manual_seed(int.from_bytes(raw[:8], "little"))
    logits = (3.0 * torch.randn(len(rows), V, generator=g, dtype=torch.float64)).float()
    # the banned ids are made the most likely ones, so the ban decides the argmax
    from vllm.v1.sample.logits_processor.interface import BatchUpdate
    proc = MinTokensLogitsProcessor(None, torch.device("cpu"), False)
    out, added = [], []
    for i, r in enumerate(rows):
        sp = SamplingParams(max_tokens=16, min_tokens=r["min_tokens"], stop_token_ids=r["stop_ids"],
                            ignore_eos=r["ignore_eos"])
        sp.update_from_generation_config({} if r["gen_eos"] is None else {"eos_token_id": r["gen_eos"]}, eos)
        added.append((i, sp, None, [0] * r["n_out"]))
        for t in sp.all_stop_token_ids:
            logits[i, t] = logits[i].max() + 1.0
        out.append(dict(r, all_stop_token_ids=sorted(sp.all_stop_token_ids)))
    proc.update_state(BatchUpdate(batch_size=len(rows), removed=[], added=added, moved=[]))
    masked = proc.apply(logits.clone())
    for i, r in enumerate(out):
        z = masked[i:i + 1].double() / (r["T"] if r["T"] > 0 else 1.0)
        k = torch.tensor([r["top_k"]]) if r["top_k"] > 0 else None
        p = torch.tensor([r["top_p"]], dtype=torch.float64) if r["top_p"] < 1 else None
        zt = apply_top_k_top_p(z.clone(), k, p) if (k is not None or p is not None) else z
        r["banned"] = [int(t) for t in torch.nonzero(torch.isinf(masked[i]) & (masked[i] < 0)).flatten()]
        lp = torch.log_softmax(zt, dim=-1)[0]
        r["greedy_id"] = int(torch.argmax(zt[0]))
        r["greedy_logprob"] = float(lp[r["greedy_id"]])
    return dict(V=V, seed=seed, logits_sha256=hashlib.sha256(logits.numpy().tobytes()).hexdigest(), rows=out), logits


def main():
    tk = train_tokenizer()
    path = HERE / "stop_tokenizer.json"
    tk.save(str(path))
    tok = hf_tokenizer(path)
    relabel = _relabel()
    out = [run_case(tok, c, relabel) for c in cases(tok)]
    for r in out:
        print(r["name"], r["n_out"], r["finish_reason"], repr(r["stop_reason"]), repr(r["output_text"]))
    (HERE / "stop_strings_vllm.json").write_text(json.dumps(out, indent=1, ensure_ascii=False))
    mt, logits = min_tokens_cases(tok)
    for r in mt["rows"]:
        print("min_tokens", r["min_tokens"], r["n_out"], r["banned"], r["greedy_id"])
    (HERE / "min_tokens_vllm.json").write_text(json.dumps(mt, indent=1))


if __name__ == "__main__":
    main()

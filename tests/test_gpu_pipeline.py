"""Whole loop on one GPU with a tiny model: plugin rollouts through the in-process engine -> preprocess ->
packed micro-batches (cut at the optimizer-step boundary) -> rl_step on the NATIVE learner (learner_model.NativeQwen2:
wgmma GEMMs, wgmma attention forward / backward, fused head, fp32 gradient arena) -> FusedAdamW -> in-flight weight
push -> sampler flip."""
import asyncio

import pytest
import torch

from tests.helpers import tiny_cfg, tiny_weights

pytestmark = pytest.mark.gpu


def test_actor_preprocess_finetune_push_loop(cuda_device, tmp_path):
    from pipelinerl_b200 import streams
    from pipelinerl_b200.actor import publish_groups_to_stream, schedule_rollouts
    from pipelinerl_b200.domains.synthetic import load_problems
    from pipelinerl_b200.engine import DecodeEngine
    from pipelinerl_b200.finetune.rl import RLConfig
    from pipelinerl_b200.finetune_loop import TrainerConfig, run_training
    from pipelinerl_b200.learner_model import NativeQwen2
    from pipelinerl_b200.llm import SyntheticTokenizer, TrainableLLM
    from pipelinerl_b200.preprocess import pack_micro_batches, preprocess_dataset
    from pipelinerl_b200.serving import EngineServer
    from pipelinerl_b200.weights import WeightReceiver, WeightUpdateManager

    streams.reset_streams_backend()
    streams.set_streams_backend("files")
    cfg = tiny_cfg("gqa2")
    w = tiny_weights(cfg, std=0.02, bias_std=0.0)
    recv = WeightReceiver(cfg, cuda_device, n_pushers=1)
    for name in recv.arena.names():
        recv.arenas[0].view(name).copy_(w[name].to(torch.bfloat16))
    eng = DecodeEngine(cfg, recv.arena, max_batch=16, max_seq_len=192, max_new_tokens=32, eos_id=2, device=cuda_device)
    server = EngineServer("test-sampler", eng)
    server.on_step_boundary = recv.maybe_flip
    server.start()
    try:
        tok = SyntheticTokenizer(vocab_size=cfg.vocab_size)
        llm = TrainableLLM(server.base_url, "tiny", parameters={"max_tokens": 12, "temperature": 1.0}, tokenizer=tok)
        problems = load_problems(["train"], n_problems=4, prompt_tokens=20, vocab_limit=cfg.vocab_size)
        writer, on_group = publish_groups_to_stream(tmp_path, "actor")
        groups = []

        def both(g):
            groups.append(g)
            on_group(g)
        stats = asyncio.run(schedule_rollouts(None, 4, problems, [llm],
                                              "pipelinerl_b200.domains.synthetic.generate_synthetic_rollout", both,
                                              get_model_version=lambda: recv.version))
        writer.__exit__(None, None, None)
        assert stats["groups"] == 4 and stats["finished"] == 16 and len(groups) == 4
        with streams.read_stream(streams.SingleStreamSpec(exp_path=tmp_path, topic="actor")) as r:
            published = r.read_available()
        assert len(published) == 4 and all(len(g) == 4 for g in published)
        sample = published[0][0]
        assert sample["labels"][:20] == [-100] * 20 and len(sample["logprobs"]) == len(sample["input_ids"]) - 20
        assert all(lp <= 0 for lp in sample["logprobs"])

        rl = RLConfig(policy_loss="ppo", kl_coef=0.0, final_kl_coef=0.0, epsilon_low=0.2, epsilon_high=0.2,
                      divide_advantage_by_std=False)
        entries = preprocess_dataset([s for g in published for s in g], tok, seq_length=128, rl_config=rl)
        assert len(entries) == 16
        batches = pack_micro_batches(entries, tok, seq_length=128, samples_per_step=8)
        assert sum(int(b.seq_boundaries.numel()) - 1 for b in batches) == 16

        learner = NativeQwen2(cfg, cuda_device, init=w)
        mgr = WeightUpdateManager([recv], torch.zeros(recv.nbytes // 2, dtype=torch.bfloat16, device=cuda_device))
        tcfg = TrainerConfig(samples_per_step=8, learning_rate=1e-3, max_train_steps=2, rl=rl)
        before = recv.arena.data.clone()
        tm, hist = run_training(learner, batches, tcfg, weight_manager=mgr, device=cuda_device)
        assert tm.completed_steps == 2 and tm.samples == 16 and all(h["push_ms"] is not None for h in hist)
        assert all(torch.isfinite(torch.tensor(h["loss"])) for h in hist) and hist[0]["grad_norm"] > 0
        # the samplers pick the new weights up at a step boundary (server thread polls), without a restart
        for _ in range(800):
            if recv.version == 16:   # both optimizer steps were pushed (versions = samples trained on: 8, 16)
                break
            asyncio.run(asyncio.sleep(0.01))
        assert recv.flips >= 1 and recv.version == 16
        assert not torch.equal(recv.arena.data, before)
        # sampler logprobs before the update are exactly what the learner re-computes: old ~ new on step 0
        assert abs(hist[0]["loss"]) < 10
        # new rollouts are stamped with the new version
        more = []
        asyncio.run(schedule_rollouts(None, 2, problems[:1], [llm],
                                      "pipelinerl_b200.domains.synthetic.generate_synthetic_rollout", more.append,
                                      get_model_version=lambda: recv.version))
        assert more[0][0].model_version == recv.version
    finally:
        server.stop()
        recv.close()
        streams.reset_streams_backend()

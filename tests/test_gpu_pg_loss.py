"""Parity of the CUDA PG-loss path (through the C ABI / rl_step facade) with the oracle and with the
reference's own outputs (golden fixtures).  Tolerances: loss / logprobs / stats 1e-4 relative
(north star asks for 1e-3); gradients 1e-4 relative + 1e-7 absolute."""
import numpy as np
import pytest
import torch

from oracle import pg_oracle
from tests.helpers import RL_CASES, assert_stats_close, batch_from_arrays, load_rl_case, row_cols

pytestmark = pytest.mark.gpu


class LogitsModel(torch.nn.Module):
    """Any module returning .logits is a valid rl_step model (rl/__init__.py:190-207)."""

    def __init__(self, logits):
        super().__init__()
        self.logits = torch.nn.Parameter(logits)

    def forward(self, **kw):
        import types
        return types.SimpleNamespace(logits=self.logits)


@pytest.mark.parametrize("name", RL_CASES)
def test_rl_step_matches_reference_golden(cuda_device, name):
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    arrs, meta = load_rl_case(name)
    cfg = RLConfig(**meta["config"])
    batch = batch_from_arrays(arrs, cuda_device)
    model = LogitsModel(torch.from_numpy(arrs["logits"]).to(cuda_device))
    loss, stats = rl_step(model, batch, meta["current_step"], meta["max_step"], cfg)
    assert loss.requires_grad and loss.dim() == 0
    loss.backward()
    want = float(arrs["loss"])
    assert abs(loss.item() - want) <= 1e-5 + 1e-4 * abs(want)
    assert_stats_close(stats, meta["stats"], rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(model.logits.grad.cpu().numpy(), arrs["grad_logits"], rtol=1e-4, atol=2e-7)


def test_sentinel_and_unpacked(cuda_device):
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    arrs, meta = load_rl_case("sentinel")
    batch = batch_from_arrays(arrs, cuda_device)
    model = LogitsModel(torch.from_numpy(arrs["logits"]).to(cuda_device))
    loss, stats = rl_step(model, batch, 0, 10, RLConfig(**meta["config"]))
    loss.backward()
    assert loss.item() == 0.0 and stats == {"input_size": 8.0}
    assert torch.count_nonzero(model.logits.grad) == 0

    arrs, meta = load_rl_case("unpacked")
    batch = batch_from_arrays(arrs, cuda_device)
    model = LogitsModel(torch.from_numpy(arrs["logits"]).to(cuda_device))
    loss, stats = rl_step(model, batch, 0, 10, RLConfig(**meta["config"]))
    loss.backward()
    assert abs(loss.item() - float(arrs["loss"])) <= 1e-4 * max(1.0, abs(float(arrs["loss"])))
    assert_stats_close(stats, meta["stats"], rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(model.logits.grad.cpu().numpy(), arrs["grad_logits"], rtol=1e-4, atol=2e-7)


@pytest.mark.parametrize("policy", ["ppo", "reinforce", "gspo"])
@pytest.mark.parametrize("T,V", [(2, 17), (257, 1031), (4099, 152064 // 8)])
def test_against_oracle_random(cuda_device, policy, T, V):
    """Seeded random rows at sizes the oracle finishes in seconds, incl. ragged / tiny rows."""
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from pipelinerl_b200.finetune.types import PipelineBatchEncoding
    g = torch.Generator().manual_seed(T * 7 + V)
    n_samples = max(1, min(9, T // 3))
    cuts = sorted(set([0, T] + torch.randint(1, T, (n_samples - 1,), generator=g).tolist())) if T > 1 else [0, T]
    pos = torch.cat([torch.arange(b - a) for a, b in zip(cuts[:-1], cuts[1:])])
    seg = torch.cat([torch.full((b - a,), i) for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))])
    ids = torch.randint(0, V, (T,), generator=g)
    labels = torch.where(torch.rand(T, generator=g) < 0.6, ids, torch.full((T,), -100))
    labels[pos == 0] = -100
    logits = torch.randn(T, V, generator=g) * 2
    with torch.no_grad():
        lp = torch.log_softmax(logits[:-1], -1).gather(1, ids[1:, None])[:, 0] if T > 1 else torch.zeros(0)
    old = torch.zeros(T)
    old[1:] = lp + 0.05 * torch.randn(T - 1, generator=g)
    ref = torch.zeros(T)
    ref[1:] = lp + 0.8 * torch.randn(T - 1, generator=g)
    n_lab = torch.zeros(T)
    for a, b in zip(cuts[:-1], cuts[1:]):
        n_lab[a:b] = max(1, int((labels[a:b] != -100).sum()))
    cols = dict(input_ids=ids, labels=labels, rewards=torch.rand(T, generator=g).round(), advantages=torch.randn(T, generator=g),
                ref_logprobs=ref, old_logprobs=old, group_tokens=torch.full((T,), 37.5), num_labels=n_lab,
                overflow=(torch.rand(T, generator=g) < 0.2).float(), position_ids=pos, segment_ids=seg)
    cfgd = dict(policy_loss=policy, kl_coef=0.07, final_kl_coef=0.01, entropy_bonus=0.02, final_entropy_bonus=0.02,
                epsilon_low=0.03, epsilon_high=0.04, batch_size=11, clamp_log_ratio_ref_new_value=1.0,
                overlong_filtering=True, temperature=0.7)
    ocfg = pg_oracle.OracleRLConfig.from_dict(cfgd)
    lo = logits.clone().requires_grad_(True)
    with torch.no_grad():  # old/ref were built at temperature 1; fine — just inputs
        pass
    o_loss, o_stats, o_lp, o_ent = pg_oracle.rl_step_oracle(lo, cols, ocfg, 2, 9)
    o_loss.backward()

    batch = PipelineBatchEncoding(
        input_ids=ids[None], attention_mask=torch.ones(1, T, dtype=torch.long), labels=labels[None],
        position_ids=pos[None], segment_ids=seg[None], rewards=cols["rewards"][None], advantages=cols["advantages"][None],
        ref_logprobs=ref[None], old_logprobs=old[None], group_tokens=cols["group_tokens"][None],
        num_labels=n_lab[None], overflow=cols["overflow"][None], model_version=0, is_packed=True,
        seq_boundaries=torch.tensor(cuts, dtype=torch.int32)).to_device(cuda_device)
    model = LogitsModel(logits[None].to(cuda_device))
    loss, stats = rl_step(model, batch, 2, 9, RLConfig(**cfgd))
    loss.backward()
    assert abs(loss.item() - float(o_loss)) <= 1e-5 + 1e-4 * abs(float(o_loss))
    if int((labels[1:] != -100).sum()) == 0:
        assert stats == {"input_size": float(T)}
    else:
        assert_stats_close(stats, o_stats, rtol=2e-4, atol=5e-6)
    np.testing.assert_allclose(model.logits.grad[0].cpu().numpy(), lo.grad.numpy(), rtol=2e-4, atol=1e-7)


def test_nonfinite_is_reported(cuda_device):
    from pipelinerl_b200._lib import NonFiniteError
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    arrs, meta = load_rl_case("ppo_default")
    arrs["ref_logprobs"] = arrs["ref_logprobs"].copy()
    arrs["ref_logprobs"][0, 5] = np.inf
    batch = batch_from_arrays(arrs, cuda_device)
    model = LogitsModel(torch.from_numpy(arrs["logits"]).to(cuda_device))
    with pytest.raises(NonFiniteError):
        rl_step(model, batch, 0, 10, RLConfig(**meta["config"]))


def test_large_row_properties(cuda_device):
    """Size-independent properties at a BASELINE-scale packed row (T = 16384 tokens x vocab 152064 would be
    10 GB of logits; the loss tail itself is tested at T = 2^20 through the C ABI directly)."""
    import ctypes as C
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    T = 1 << 20
    dev = cuda_device
    g = torch.Generator(device="cpu").manual_seed(1)
    new_lp = (-torch.rand(T - 1, generator=g) * 3).to(dev)
    cols = {k: torch.zeros(T, device=dev) for k in ("rewards", "advantages", "ref_logprobs", "old_logprobs", "overflow")}
    cols["old_logprobs"][1:] = new_lp  # ratio == 1 everywhere
    cols["ref_logprobs"][1:] = new_lp
    cols["advantages"] = torch.randn(T, generator=g).to(dev)
    cols["group_tokens"] = torch.ones(T, device=dev)
    cols["num_labels"] = torch.ones(T, device=dev)
    labels = torch.zeros(T, dtype=torch.long, device=dev)
    labels[::3] = -100
    b = _lib.PgBatch()
    b.T = T
    b.new_logprobs = new_lp.data_ptr()
    b.labels = labels.data_ptr()
    for k, v in cols.items():
        setattr(b, k, v.data_ptr())
    b.num_sequences = 1
    c = _lib.PgConfig()
    c.policy_loss = 0
    c.use_advantages = 1
    c.epsilon_low = c.epsilon_high = 0.2
    c.clamp_log_ratio_ref_new_value = 5.0
    c.batch_size = 64.0
    out = torch.zeros(1, device=dev)
    dlp = torch.zeros(T - 1, device=dev)
    stats = torch.zeros(32, dtype=torch.float64, device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.zeros(int(lib.prl_pg_workspace_bytes(0)), dtype=torch.uint8, device=dev)
    for _ in range(2):  # second call re-uses the workspace (ticket re-armed)
        _lib.check(lib.prl_pg_loss_fwd_bwd(C.byref(b), C.byref(c), out.data_ptr(), dlp.data_ptr(), None,
                                           stats.data_ptr(), flags.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    m = labels[1:] != -100
    adv = cols["advantages"][1:]
    # ratio == 1: loss = -sum(adv)/batch_size over labelled tokens; grad = -adv/batch_size
    want = -(adv[m].double().sum() / 64.0).item()
    assert abs(out.item() - want) <= 1e-5 * max(1.0, abs(want))
    assert torch.allclose(dlp[m], -adv[m] / 64.0, rtol=1e-6, atol=0)
    assert torch.count_nonzero(dlp[~m]) == 0
    s = stats.cpu().numpy()
    assert s[_lib.STAT_NAMES.index("num_output_tokens_sum")] == float(m.sum())
    assert abs(s[_lib.STAT_NAMES.index("ratio_new_old_sum")] - float(m.sum())) < 1e-3
    assert s[_lib.STAT_NAMES.index("kl")] == 0.0 and flags.item() == 0


def test_rl_step_fused_head_matches_logits_path(cuda_device):
    """rl_step through a model exposing forward_logprobs (wgmma fused head, no [T, V] logits) == rl_step through
    the same model's materialised logits: loss, stats and every parameter gradient."""
    from pipelinerl_b200.finetune.rl import RLConfig, rl_step
    from pipelinerl_b200.learner_model import TorchQwen2
    from tests.helpers import tiny_cfg, tiny_weights
    arrs, meta = load_rl_case("ppo_kl_entropy")
    cfg_m = tiny_cfg("gqa2")
    w = tiny_weights(cfg_m, std=0.02, bias_std=0.0)
    arrs = dict(arrs)
    arrs["input_ids"] = arrs["input_ids"] % cfg_m.vocab_size
    arrs["labels"] = np.where(arrs["labels"] == -100, -100, arrs["labels"] % cfg_m.vocab_size)
    rl = RLConfig(**meta["config"])
    results = []
    for fused in (True, False):
        model = TorchQwen2(cfg_m, cuda_device, dtype=torch.float32, init=w)
        model.use_fused_head = fused
        batch = batch_from_arrays(arrs, cuda_device)
        loss, stats = rl_step(model, batch, meta["current_step"], meta["max_step"], rl)
        loss.backward()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        results.append((loss.item(), stats, grads))
    (l1, s1, g1), (l0, s0, g0) = results
    assert abs(l1 - l0) <= 2e-3 * max(1.0, abs(l0))        # bf16 rounding of the head input in the fused path
    for k in s0:
        assert abs(s1[k] - s0[k]) <= 5e-3 + 5e-3 * abs(s0[k]), k
    assert set(g1) == set(g0)
    for n in g0:
        scale = g0[n].abs().max().item() + 1e-12
        assert (g1[n] - g0[n]).abs().max().item() <= 3e-2 * scale, n


@pytest.mark.parametrize("sp", [2, 4])
def test_gspo_under_sequence_parallelism_matches_the_whole_row(cuda_device, sp):
    """GSPO is a per-sequence objective; with seq_parallel the sequence is spread over the group and the reference
    all-reduces the per-segment sums (rl/utils.py:194-206).  Here: every slice's prl_pg_gspo_segment_sums, their sum (the
    all-reduce), then prl_pg_loss_fwd_bwd_seg per slice  ==  prl_pg_loss_fwd_bwd on the whole row with the slice-leading
    labels masked (a slice's first token has no predecessor on its rank): the slices' losses add up to the row's loss and
    their gradients are the row's gradient, element for element."""
    import ctypes as C
    from pipelinerl_b200 import _lib
    lib = _lib.load()
    dev = cuda_device
    T = 4096
    g = torch.Generator().manual_seed(11 + sp)
    cuts = sorted(set([0, T] + torch.randint(1, T, (12,), generator=g).tolist()))
    seg_ids = torch.cat([torch.full((b - a,), i) for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:]))]).to(dev)
    pos = torch.cat([torch.arange(b - a) for a, b in zip(cuts[:-1], cuts[1:])])
    labels = torch.where(torch.rand(T, generator=g) < 0.6, torch.randint(0, 1000, (T,), generator=g), torch.full((T,), -100))
    labels[pos == 0] = -100
    Tl = T // sp
    for r in range(1, sp):
        labels[r * Tl] = -100
    labels = labels.to(dev)
    new_lp = (-torch.rand(T - 1, generator=g) * 3).to(dev)
    cols = {"rewards": torch.rand(T, generator=g).round(), "advantages": torch.randn(T, generator=g),
            "ref_logprobs": -torch.rand(T, generator=g) * 3, "old_logprobs": torch.zeros(T),
            "group_tokens": torch.full((T,), 37.5), "num_labels": torch.full((T,), 9.0),
            "overflow": (torch.rand(T, generator=g) < 0.2).float()}
    cols["old_logprobs"][1:] = new_lp.cpu() + 0.05 * torch.randn(T - 1, generator=g)
    cols = {k: v.to(dev) for k, v in cols.items()}
    n_seg = len(cuts) - 1
    c = _lib.PgConfig()
    c.policy_loss = _lib.LOSS_IDS["gspo"]
    c.use_advantages = 1
    c.overlong_filtering = 1
    c.epsilon_low, c.epsilon_high = 0.03, 0.04
    c.clamp_log_ratio_ref_new_value = 1.0
    c.kl_coef = 0.07
    c.batch_size = 11.0

    def pg_batch(a, b):
        pb = _lib.PgBatch()
        pb.T = b - a
        keep = [new_lp[a:b - 1].contiguous(), labels[a:b].contiguous(), seg_ids[a:b].contiguous()]
        pb.new_logprobs, pb.labels, pb.segment_ids = keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr()
        for k, v in cols.items():
            keep.append(v[a:b].contiguous())
            setattr(pb, k, keep[-1].data_ptr())
        pb.n_segments = n_seg
        pb.num_sequences = 1
        return pb, keep

    def outputs(n):
        return (torch.zeros(1, device=dev), torch.zeros(max(n - 1, 0), device=dev), torch.zeros(32, dtype=torch.float64, device=dev),
                torch.zeros(1, dtype=torch.int32, device=dev))
    ws = torch.zeros(int(lib.prl_pg_workspace_bytes(n_seg)), dtype=torch.uint8, device=dev)
    full, keep_full = pg_batch(0, T)
    loss_f, dlp_f, stats_f, flags_f = outputs(T)
    _lib.check(lib.prl_pg_loss_fwd_bwd(C.byref(full), C.byref(c), loss_f.data_ptr(), dlp_f.data_ptr(), None, stats_f.data_ptr(),
                                       flags_f.data_ptr(), ws.data_ptr(), ws.numel(), None))
    slices = [pg_batch(r * Tl, (r + 1) * Tl) for r in range(sp)]
    sums = []
    for pb, _ in slices:
        s = torch.empty(n_seg, 4, dtype=torch.float64, device=dev)
        _lib.check(lib.prl_pg_gspo_segment_sums(C.byref(pb), C.byref(c), s.data_ptr(), None))
        sums.append(s)
    total = torch.stack(sums).sum(0)
    loss_sum = 0.0
    for r, (pb, _) in enumerate(slices):
        loss_r, dlp_r, stats_r, flags_r = outputs(Tl)
        local = sums[r][:, 2].contiguous()
        _lib.check(lib.prl_pg_loss_fwd_bwd_seg(C.byref(pb), C.byref(c), loss_r.data_ptr(), dlp_r.data_ptr(), None, stats_r.data_ptr(),
                                               flags_r.data_ptr(), ws.data_ptr(), ws.numel(), total.data_ptr(), local.data_ptr(), None))
        torch.cuda.synchronize()
        loss_sum += loss_r.item()
        a = r * Tl
        assert torch.allclose(dlp_r, dlp_f[a:a + Tl - 1], rtol=1e-6, atol=1e-12), f"slice {r}: gradient differs from the whole row's"
        if r + 1 < sp:
            assert dlp_f[a + Tl - 1].item() == 0.0        # the position that would score the next slice's first token
    assert abs(loss_sum - loss_f.item()) <= 1e-5 * max(1.0, abs(loss_f.item())), (loss_sum, loss_f.item())
    assert abs(loss_f.item()) > 1e-3                      # the case is not degenerate

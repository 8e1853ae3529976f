"""Qwen2 / Qwen3 (dense) / Llama 3 model description and the flat parameter arena shared by learner and sampler.

One contiguous bf16 buffer holds every parameter in the FUSED layout the token-step kernels read
(qkv_proj = [q; k; v] rows, gate_up_proj = [gate; up] rows).  HF parameter names
(`model.layers.N.self_attn.q_proj.weight`, ...) map to row-slices of those fused tensors, which is
the name mapping vLLM's `load_weights` performs for the reference at pipelinerl/vllm1.py:122
(q/k/v_proj -> qkv_proj, gate/up_proj -> gate_up_proj).  Because learner and samplers use the SAME
arena layout, the in-flight weight update (hot path 3) is a plain byte copy of the arena — no
per-tensor loop, no name mapping at push time.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch


@dataclass(frozen=True)
class Llama3RopeScaling:
    """`rope_type: "llama3"` frequency scaling (Llama 3.1 / 3.2 `rope_scaling`): wavelengths above
    original_max_position_embeddings / low_freq_factor are divided by `factor`, those below
    original_max_position_embeddings / high_freq_factor are kept, and the band between is interpolated."""
    factor: float
    low_freq_factor: float
    high_freq_factor: float
    original_max_position_embeddings: int

    def hf_dict(self) -> dict:
        return {"factor": self.factor, "low_freq_factor": self.low_freq_factor, "high_freq_factor": self.high_freq_factor,
                "original_max_position_embeddings": self.original_max_position_embeddings, "rope_type": "llama3"}


@dataclass(frozen=True)
class ModelConfig:
    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_layers: int
    num_q_heads: int
    num_kv_heads: int
    head_dim: int = 128
    rope_theta: float = 1_000_000.0
    rms_eps: float = 1e-6
    qkv_bias: bool = True
    qk_norm: bool = False    # Qwen3: per-head RMSNorm of q and k (gains q_norm / k_norm, [head_dim]) before RoPE
    fp32_head: bool = False  # keep a bf16 residual of the head (W = hi + lo): fp32-equivalent lm_head
    lm_head_rows: int | None = None  # vocabulary rows of THIS shard's lm_head (vocab-parallel head under TP)
    family: str = "qwen"     # "qwen" (Qwen2 / Qwen3, told apart by qk_norm) or "llama": the config.json a checkpoint gets
    rope_scaling: Llama3RopeScaling | None = None   # None: plain RoPE, inv_freq = 1 / theta^(2i / d)
    tie_word_embeddings: bool = False  # one [V, H] table is both the input embedding and the head (no lm_head tensor)

    def __post_init__(self):
        if self.tie_word_embeddings and self.fp32_head:
            raise ValueError("fp32_head=True with tie_word_embeddings=True: a tied head is the bf16 embedding table, and "
                             "its logits are already computed as the reference computes a tied head, fp32 accumulation "
                             "over the bf16 table (the head kernels with W_lo = NULL); drop fp32_head")

    @property
    def q_size(self) -> int:
        return self.num_q_heads * self.head_dim

    @property
    def kv_size(self) -> int:
        return self.num_kv_heads * self.head_dim

    @property
    def qkv_size(self) -> int:
        return self.q_size + 2 * self.kv_size

    @property
    def head_name(self) -> str:
        """Arena name of the tensor the head reads: the embedding table when the word embeddings are tied."""
        return "embed_tokens.weight" if self.tie_word_embeddings else "lm_head.weight"

    @property
    def head_rows(self) -> int:
        return self.lm_head_rows if self.lm_head_rows is not None else self.vocab_size

    def shard(self, tp: int) -> "ModelConfig":
        """Per-rank configuration under tensor parallelism: heads, MLP width and lm_head rows divided by tp
        (column-parallel qkv / gate_up / head, row-parallel o_proj / down_proj); embeddings and norms replicated."""
        from dataclasses import replace
        if tp == 1:
            return self
        for what, v in (("q heads", self.num_q_heads), ("kv heads", self.num_kv_heads),
                        ("intermediate", self.intermediate_size), ("vocab", self.vocab_size)):
            if v % tp:
                raise ValueError(f"{what} ({v}) not divisible by tp={tp}")
        return replace(self, num_q_heads=self.num_q_heads // tp, num_kv_heads=self.num_kv_heads // tp,
                       intermediate_size=self.intermediate_size // tp, lm_head_rows=self.vocab_size // tp)

    @staticmethod
    def qwen2_5_7b(**kw) -> "ModelConfig":
        return ModelConfig(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_layers=28,
                           num_q_heads=28, num_kv_heads=4, **kw)

    @staticmethod
    def qwen2_5_1_5b(**kw) -> "ModelConfig":
        """Qwen2.5-1.5B's shapes (its checkpoint ties the word embeddings; pass tie_word_embeddings=True to train them
        tied, the default stores an untied copy of the head)."""
        return ModelConfig(vocab_size=151936, hidden_size=1536, intermediate_size=8960, num_layers=28,
                           num_q_heads=12, num_kv_heads=2, **kw)

    @staticmethod
    def qwen2_5_32b(**kw) -> "ModelConfig":
        return ModelConfig(vocab_size=152064, hidden_size=5120, intermediate_size=27648, num_layers=64,
                           num_q_heads=40, num_kv_heads=8, **kw)

    @staticmethod
    def qwen3_8b(**kw) -> "ModelConfig":
        """Qwen3-8B's shapes (keyword arguments override, e.g. num_layers for a bounded sample of layers)."""
        base = dict(vocab_size=151936, hidden_size=4096, intermediate_size=12288, num_layers=36, num_q_heads=32,
                    num_kv_heads=8, qkv_bias=False, qk_norm=True)
        return ModelConfig(**{**base, **kw})

    @staticmethod
    def qwen3_1_7b(**kw) -> "ModelConfig":
        """Qwen3-1.7B's shapes, word embeddings tied as in its published config.json."""
        base = dict(vocab_size=151936, hidden_size=2048, intermediate_size=6144, num_layers=28, num_q_heads=16,
                    num_kv_heads=8, qkv_bias=False, qk_norm=True, tie_word_embeddings=True)
        return ModelConfig(**{**base, **kw})

    @staticmethod
    def qwen3_14b(**kw) -> "ModelConfig":
        base = dict(vocab_size=151936, hidden_size=5120, intermediate_size=17408, num_layers=40, num_q_heads=40,
                    num_kv_heads=8, qkv_bias=False, qk_norm=True)
        return ModelConfig(**{**base, **kw})

    @staticmethod
    def llama3_1_8b(**kw) -> "ModelConfig":
        """Llama-3.1-8B(-Instruct)'s shapes and RoPE scaling."""
        base = dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_layers=32, num_q_heads=32,
                    num_kv_heads=8, rope_theta=500_000.0, rms_eps=1e-5, qkv_bias=False, family="llama",
                    rope_scaling=Llama3RopeScaling(8.0, 1.0, 4.0, 8192))
        return ModelConfig(**{**base, **kw})

    @staticmethod
    def llama3_2_3b(**kw) -> "ModelConfig":
        """Llama-3.2-3B(-Instruct)'s shapes and RoPE scaling (its checkpoint ties the word embeddings; the default stores an
        untied copy of the head, tie_word_embeddings=True trains them tied)."""
        base = dict(vocab_size=128256, hidden_size=3072, intermediate_size=8192, num_layers=28, num_q_heads=24,
                    num_kv_heads=8, rope_theta=500_000.0, rms_eps=1e-5, qkv_bias=False, family="llama",
                    rope_scaling=Llama3RopeScaling(32.0, 1.0, 4.0, 8192))
        return ModelConfig(**{**base, **kw})

    @staticmethod
    def from_hf_config(d: dict, keep_tied: bool = False) -> "ModelConfig":
        """ModelConfig of an HF `config.json` dict of model_type "qwen2", "qwen3" (dense) or "llama" (Llama 3).  Tied
        word embeddings are accepted: by default the arena keeps an untied copy of the head
        (ParamArena.load_hf_state_dict); with keep_tied, `tie_word_embeddings` follows `d` and one table serves both."""
        mt = d.get("model_type")
        if mt not in ("qwen2", "qwen3", "llama"):
            raise ValueError(f"unsupported model_type {mt!r}: only 'qwen2', 'qwen3' (dense) and 'llama' are implemented")
        arch = {"qwen2": "Qwen2ForCausalLM", "qwen3": "Qwen3ForCausalLM", "llama": "LlamaForCausalLM"}[mt]
        if d.get("architectures") and arch not in d["architectures"]:
            raise ValueError(f"model_type {mt!r} does not match architectures {d['architectures']}")
        heads = int(d["num_attention_heads"])
        head_dim = int(d.get("head_dim") or d["hidden_size"] // heads)
        if head_dim != 128:
            raise ValueError(f"head_dim {head_dim} is not supported: the attention and RoPE kernels are built for 128")
        rope = d.get("rope_parameters") or {}
        common = dict(vocab_size=int(d["vocab_size"]), hidden_size=int(d["hidden_size"]),
                      intermediate_size=int(d["intermediate_size"]), num_layers=int(d["num_hidden_layers"]),
                      num_q_heads=heads, num_kv_heads=int(d.get("num_key_value_heads", heads)), head_dim=head_dim,
                      rms_eps=float(d.get("rms_norm_eps", 1e-6)))
        if keep_tied:
            common["tie_word_embeddings"] = bool(d.get("tie_word_embeddings", False))
        if mt == "llama":
            return ModelConfig(**common, **_llama_fields(d))
        theta = d.get("rope_theta", rope.get("rope_theta", 1_000_000.0))
        return ModelConfig(**common, rope_theta=float(theta), qkv_bias=bool(d.get("attention_bias", mt == "qwen2")),
                           qk_norm=mt == "qwen3")

    @staticmethod
    def tiny(**kw) -> "ModelConfig":
        """Plumbing / parity-test model (config 1 of BASELINE.json is not defined by the reference)."""
        base = dict(vocab_size=512, hidden_size=256, intermediate_size=640, num_layers=2, num_q_heads=4,
                    num_kv_heads=2)
        base.update(kw)
        return ModelConfig(**base)

    def num_params(self) -> int:
        return sum(n for _, n in ((name, _numel(shape)) for name, shape in fused_shapes(self)))


def _llama_fields(d: dict) -> dict:
    """The Llama-specific ModelConfig fields of a `config.json` dict: RoPE from `rope_scaling` (transformers 4.x, what
    Hub checkpoints ship) or `rope_parameters` (5.x); no biases anywhere."""
    for name in ("attention_bias", "mlp_bias"):
        if d.get(name):
            raise ValueError(f"{name}=true is not supported: the arena has no slot for Llama's o_proj / MLP biases")
    rope = d.get("rope_scaling") or d.get("rope_parameters") or {}
    kind = rope.get("rope_type", rope.get("type", "default"))
    if kind == "default":
        scaling = None
    elif kind == "llama3":
        scaling = Llama3RopeScaling(float(rope["factor"]), float(rope["low_freq_factor"]), float(rope["high_freq_factor"]),
                                    int(rope["original_max_position_embeddings"]))
    else:
        raise ValueError(f"rope_type {kind!r} is not supported: only 'default' and 'llama3' are implemented")
    theta = d.get("rope_theta", rope.get("rope_theta", 10_000.0))
    return dict(rope_theta=float(theta), qkv_bias=False, family="llama", rope_scaling=scaling)


def rope_inv_freq(cfg: ModelConfig) -> torch.Tensor:
    """fp32 [head_dim / 2] RoPE inverse frequencies, the table every RoPE kernel reads.  Without scaling it is HF's
    1 / theta^(2i / d); with Llama 3 scaling it restates transformers' `_compute_llama3_parameters` operation for
    operation, so both tables match transformers bit for bit."""
    d = cfg.head_dim
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.int64).float() / d))
    s = cfg.rope_scaling
    if s is None:
        return inv
    low_wavelen = s.original_max_position_embeddings / s.low_freq_factor
    high_wavelen = s.original_max_position_embeddings / s.high_freq_factor
    wavelen = 2 * math.pi / inv
    scaled = torch.where(wavelen > low_wavelen, inv / s.factor, inv)
    smooth = (s.original_max_position_embeddings / wavelen - s.low_freq_factor) / (s.high_freq_factor - s.low_freq_factor)
    smoothed = (1 - smooth) * scaled / s.factor + smooth * scaled
    medium = ~(wavelen < high_wavelen) * ~(wavelen > low_wavelen)
    return torch.where(medium, smoothed, scaled)


def _numel(shape) -> int:
    n = 1
    for s in shape:
        n *= s
    return n


def is_norm_gain(name: str) -> bool:
    """RMSNorm gains (initialised to 1): the layer norms, the final norm and Qwen3's per-head q_norm / k_norm."""
    return name.endswith("layernorm.weight") or name == "norm.weight" or name.endswith((".q_norm.weight", ".k_norm.weight"))


def fused_shapes(cfg: ModelConfig) -> list[tuple[str, tuple[int, ...]]]:
    """Arena order.  Names are the fused (kernel-side) tensor names."""
    H, I = cfg.hidden_size, cfg.intermediate_size
    out: list[tuple[str, tuple[int, ...]]] = []
    for l in range(cfg.num_layers):
        p = f"layers.{l}."
        out.append((p + "input_layernorm.weight", (H,)))
        out.append((p + "qkv_proj.weight", (cfg.qkv_size, H)))
        if cfg.qkv_bias:
            out.append((p + "qkv_proj.bias", (cfg.qkv_size,)))
        if cfg.qk_norm:
            out.append((p + "q_norm.weight", (cfg.head_dim,)))
            out.append((p + "k_norm.weight", (cfg.head_dim,)))
        out.append((p + "o_proj.weight", (H, cfg.q_size)))
        out.append((p + "post_attention_layernorm.weight", (H,)))
        out.append((p + "gate_up_proj.weight", (2 * I, H)))
        out.append((p + "down_proj.weight", (H, I)))
    out.append(("embed_tokens.weight", (cfg.vocab_size, H)))
    out.append(("norm.weight", (H,)))
    if cfg.tie_word_embeddings:
        return out
    out.append(("lm_head.weight", (cfg.head_rows, H)))
    if cfg.fp32_head:
        out.append(("lm_head.weight_lo", (cfg.head_rows, H)))
    return out


@dataclass
class ArenaLayout:
    cfg: ModelConfig
    offsets: dict[str, int] = field(default_factory=dict)
    shapes: dict[str, tuple[int, ...]] = field(default_factory=dict)
    total: int = 0

    @staticmethod
    def build(cfg: ModelConfig, align: int = 64) -> "ArenaLayout":
        lay = ArenaLayout(cfg)
        at = 0
        for name, shape in fused_shapes(cfg):
            lay.offsets[name] = at
            lay.shapes[name] = shape
            at = (at + _numel(shape) + align - 1) // align * align  # 128-byte aligned tensors (TMA needs 16)
        lay.total = at
        return lay

    # HF name -> (fused name, row start, row count)
    def hf_slices(self) -> dict[str, tuple[str, int, int]]:
        c = self.cfg
        m: dict[str, tuple[str, int, int]] = {}
        for l in range(c.num_layers):
            hp, fp = f"model.layers.{l}.", f"layers.{l}."
            m[hp + "input_layernorm.weight"] = (fp + "input_layernorm.weight", 0, c.hidden_size)
            m[hp + "post_attention_layernorm.weight"] = (fp + "post_attention_layernorm.weight", 0, c.hidden_size)
            for kind in ("weight", "bias") if c.qkv_bias else ("weight",):
                m[hp + f"self_attn.q_proj.{kind}"] = (fp + f"qkv_proj.{kind}", 0, c.q_size)
                m[hp + f"self_attn.k_proj.{kind}"] = (fp + f"qkv_proj.{kind}", c.q_size, c.kv_size)
                m[hp + f"self_attn.v_proj.{kind}"] = (fp + f"qkv_proj.{kind}", c.q_size + c.kv_size, c.kv_size)
            if c.qk_norm:
                m[hp + "self_attn.q_norm.weight"] = (fp + "q_norm.weight", 0, c.head_dim)
                m[hp + "self_attn.k_norm.weight"] = (fp + "k_norm.weight", 0, c.head_dim)
            m[hp + "self_attn.o_proj.weight"] = (fp + "o_proj.weight", 0, c.hidden_size)
            m[hp + "mlp.gate_proj.weight"] = (fp + "gate_up_proj.weight", 0, c.intermediate_size)
            m[hp + "mlp.up_proj.weight"] = (fp + "gate_up_proj.weight", c.intermediate_size, c.intermediate_size)
            m[hp + "mlp.down_proj.weight"] = (fp + "down_proj.weight", 0, c.hidden_size)
        m["model.embed_tokens.weight"] = ("embed_tokens.weight", 0, c.vocab_size)
        m["model.norm.weight"] = ("norm.weight", 0, c.hidden_size)
        if not c.tie_word_embeddings:
            m["lm_head.weight"] = ("lm_head.weight", 0, c.vocab_size)
        return m


class ParamArena:
    """Flat bf16 parameter buffer + named views."""

    def __init__(self, cfg: ModelConfig, device, dtype=torch.bfloat16, data: torch.Tensor | None = None):
        self.cfg = cfg
        self.layout = ArenaLayout.build(cfg)
        if data is None:
            data = torch.zeros(self.layout.total, dtype=dtype, device=device)
        assert data.numel() == self.layout.total and data.dtype == dtype
        self.data = data
        self.version = 0

    def view(self, name: str) -> torch.Tensor:
        off, shape = self.layout.offsets[name], self.layout.shapes[name]
        return self.data[off:off + _numel(shape)].view(shape)

    def ptr(self, name: str) -> int:
        return self.data.data_ptr() + self.layout.offsets[name] * self.data.element_size()

    def names(self) -> list[str]:
        return list(self.layout.offsets)

    def nbytes(self) -> int:
        return self.data.numel() * self.data.element_size()

    def init_random(self, seed: int = 42, std: float = 0.02) -> "ParamArena":
        """normal(0, 0.02) weights, unit norm gains (q_norm / k_norm included), zero biases — HF's Qwen2 / Qwen3 / Llama
        initialisation; seed = conf/base.yaml:7."""
        g = torch.Generator(device=self.data.device).manual_seed(seed)
        for name in self.names():
            v = self.view(name)
            if is_norm_gain(name):
                v.fill_(1.0)
            elif name.endswith(".bias") or name.endswith("_lo"):
                v.zero_()
            else:
                # chunked to bound the fp32 temporary for [152064, 3584] tensors
                flat = v.view(-1)
                step = 1 << 26
                for s in range(0, flat.numel(), step):
                    n = min(step, flat.numel() - s)
                    flat[s:s + n] = (torch.randn(n, generator=g, device=self.data.device, dtype=torch.float32)
                                     * std).to(self.data.dtype)
        return self

    def load_hf_state_dict(self, sd: dict[str, torch.Tensor]) -> None:
        """HF-named tensors -> the arena.  A tied config takes a state dict with or without `lm_head.weight`; one that
        has it must hold the embedding table there, or the checkpoint is not tied."""
        slices = self.layout.hf_slices()
        if self.cfg.tie_word_embeddings and "lm_head.weight" in sd:
            sd = dict(sd)
            head = sd.pop("lm_head.weight")
            emb = sd.get("model.embed_tokens.weight")
            if emb is None or not torch.equal(head, emb):
                raise ValueError("tie_word_embeddings=True but the state dict's lm_head.weight differs from "
                                 "model.embed_tokens.weight: the checkpoint is not tied")
        seen = set()
        for hf_name, t in sd.items():
            if hf_name not in slices:
                raise KeyError(f"unexpected parameter {hf_name}")
            fused, r0, rn = slices[hf_name]
            dst = self.view(fused)[r0:r0 + rn]
            if self.cfg.fp32_head and hf_name == "lm_head.weight":
                hi = t.to(torch.bfloat16)
                dst.copy_(hi)
                self.view("lm_head.weight_lo").copy_((t.float() - hi.float()).to(torch.bfloat16))
            else:
                dst.copy_(t.to(self.data.dtype))
            seen.add(hf_name)
        missing = set(slices) - seen
        if missing == {"lm_head.weight"}:  # tied embeddings
            self.view("lm_head.weight").copy_(self.view("embed_tokens.weight"))
        elif missing:
            raise KeyError(f"missing parameters: {sorted(missing)[:4]} ...")

    def hf_state_dict(self) -> dict[str, torch.Tensor]:
        return {hf: self.view(fused)[r0:r0 + rn] for hf, (fused, r0, rn) in self.layout.hf_slices().items()}


def shard_fused_weights(cfg: ModelConfig, full: dict[str, torch.Tensor], rank: int, tp: int) -> dict[str, torch.Tensor]:
    """Slice full fused tensors (names of fused_shapes(cfg)) into rank `rank`'s tensor-parallel shard."""
    loc = cfg.shard(tp)
    d, out = cfg.head_dim, {}
    ql, kl, I, Il = loc.q_size, loc.kv_size, cfg.intermediate_size, loc.intermediate_size
    for name, t in full.items():
        if name.endswith("qkv_proj.weight") or name.endswith("qkv_proj.bias"):
            q, k, v = t[:cfg.q_size], t[cfg.q_size:cfg.q_size + cfg.kv_size], t[cfg.q_size + cfg.kv_size:]
            out[name] = torch.cat([q[rank * ql:(rank + 1) * ql], k[rank * kl:(rank + 1) * kl], v[rank * kl:(rank + 1) * kl]])
        elif name.endswith("o_proj.weight"):
            out[name] = t[:, rank * ql:(rank + 1) * ql].contiguous()
        elif name.endswith("gate_up_proj.weight"):
            out[name] = torch.cat([t[rank * Il:(rank + 1) * Il], t[I + rank * Il:I + (rank + 1) * Il]])
        elif name.endswith("down_proj.weight"):
            out[name] = t[:, rank * Il:(rank + 1) * Il].contiguous()
        elif name.startswith("lm_head.weight"):
            out[name] = t[rank * loc.head_rows:(rank + 1) * loc.head_rows]
        else:
            out[name] = t
    return out

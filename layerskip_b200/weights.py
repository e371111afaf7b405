"""Weight sources for the engine: HF state dicts and on-device synthetic Llamas.

The engine ingests HF-named tensors (`model.layers.3.self_attn.q_proj.weight`, ...) one at a
time (`lsk_load_weights`), slices its tensor-parallel shard and repacks — so a source only ever
has to materialise ONE full tensor on the GPU at a time.
"""
from __future__ import annotations

import re
from dataclasses import dataclass
from typing import Dict, Iterator, Optional, Tuple

import torch

from . import _lib

_LAYER_RE = re.compile(r"^model\.layers\.(\d+)\.(.+)\.weight$")
_LAYER_ROLES = {
    "input_layernorm": _lib.LSK_W_LN1, "self_attn.q_proj": _lib.LSK_W_Q,
    "self_attn.k_proj": _lib.LSK_W_K, "self_attn.v_proj": _lib.LSK_W_V,
    "self_attn.o_proj": _lib.LSK_W_O, "post_attention_layernorm": _lib.LSK_W_LN2,
    "mlp.gate_proj": _lib.LSK_W_GATE, "mlp.up_proj": _lib.LSK_W_UP,
    "mlp.down_proj": _lib.LSK_W_DOWN,
}
_GLOBAL_ROLES = {"model.embed_tokens.weight": _lib.LSK_W_EMBED,
                 "model.norm.weight": _lib.LSK_W_FINAL_NORM,
                 "lm_head.weight": _lib.LSK_W_LM_HEAD}


ROPE_KINDS = {"default": _lib.LSK_ROPE_DEFAULT, "linear": _lib.LSK_ROPE_LINEAR,
              "llama3": _lib.LSK_ROPE_LLAMA3}


def parse_rope(cfg_get) -> Dict[str, float]:
    """RoPE settings from an HF config, whichever spelling it uses: transformers 4.x keeps
    `rope_theta` + `rope_scaling` (keys `rope_type` or the older `type`), transformers 5.x one
    `rope_parameters` dict.  `cfg_get(name)` returns the attribute / key or None.  Unsupported
    rule -> NotImplementedError (an unscaled table would give silently wrong logits)."""
    theta = cfg_get("rope_theta")
    out = dict(rope_scaling="default", rope_factor=1.0, rope_low_freq_factor=1.0,
               rope_high_freq_factor=4.0, rope_original_max_pos=8192)
    for key in ("rope_parameters", "rope_scaling"):
        rp = cfg_get(key)
        if not isinstance(rp, dict):
            continue
        if rp.get("rope_theta") is not None:
            theta = rp["rope_theta"]
        kind = rp.get("rope_type", rp.get("type", "default")) or "default"
        if kind == "default":
            continue
        if kind not in ROPE_KINDS:
            raise NotImplementedError(f"rope scaling {kind!r} is not supported (default, linear, llama3)")
        out["rope_scaling"] = kind
        out["rope_factor"] = float(rp["factor"])
        if kind == "llama3":
            out["rope_low_freq_factor"] = float(rp["low_freq_factor"])
            out["rope_high_freq_factor"] = float(rp["high_freq_factor"])
            out["rope_original_max_pos"] = int(rp["original_max_position_embeddings"])
    out["rope_theta"] = float(theta if theta is not None else 10000.0)
    return out


@dataclass(frozen=True)
class LlamaArch:
    """Architecture numbers the engine needs (what the reference reads from `model.config`)."""
    vocab: int
    hidden: int
    inter: int
    layers: int
    heads: int
    kv_heads: int
    head_dim: int = 128
    rms_eps: float = 1e-5
    rope_theta: float = 10000.0
    rope_scaling: str = "default"          # default | linear | llama3 (HF modeling_rope_utils.py)
    rope_factor: float = 1.0
    rope_low_freq_factor: float = 1.0
    rope_high_freq_factor: float = 4.0
    rope_original_max_pos: int = 8192

    @staticmethod
    def from_hf_config(cfg) -> "LlamaArch":
        head_dim = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
        rope = parse_rope(lambda name: getattr(cfg, name, None))
        return LlamaArch(vocab=cfg.vocab_size, hidden=cfg.hidden_size,
                         inter=cfg.intermediate_size, layers=cfg.num_hidden_layers,
                         heads=cfg.num_attention_heads, kv_heads=cfg.num_key_value_heads,
                         head_dim=head_dim, rms_eps=float(cfg.rms_norm_eps), **rope)

    def rope_config(self) -> Dict:
        """HF-style `rope_scaling` dict (None for the default rule)."""
        if self.rope_scaling == "default":
            return None
        d = {"rope_type": self.rope_scaling, "factor": self.rope_factor}
        if self.rope_scaling == "llama3":
            d.update(low_freq_factor=self.rope_low_freq_factor,
                     high_freq_factor=self.rope_high_freq_factor,
                     original_max_position_embeddings=self.rope_original_max_pos)
        return d

    def lsk_config(self, max_ctx: int, tp_rank: int = 0, tp_size: int = 1, attn_splits: int = 0,
                   flags: int = 0) -> "_lib.lsk_config":
        """The engine config (`lsk_config`) of this architecture."""
        return _lib.lsk_config(
            vocab=self.vocab, hidden=self.hidden, inter=self.inter, n_layers=self.layers,
            n_heads=self.heads, n_kv_heads=self.kv_heads, head_dim=self.head_dim,
            rms_eps=self.rms_eps, rope_theta=self.rope_theta, max_ctx=max_ctx, tp_rank=tp_rank,
            tp_size=tp_size, attn_splits=attn_splits, flags=flags,
            rope_scaling=ROPE_KINDS[self.rope_scaling], rope_factor=self.rope_factor,
            rope_low_freq_factor=self.rope_low_freq_factor,
            rope_high_freq_factor=self.rope_high_freq_factor,
            rope_original_max_pos=self.rope_original_max_pos)

    @property
    def q_dim(self) -> int:
        return self.heads * self.head_dim

    @property
    def kv_dim(self) -> int:
        return self.kv_heads * self.head_dim

    def param_bytes(self) -> int:
        per_layer = 2 * self.hidden * self.q_dim + 2 * self.hidden * self.kv_dim + \
            3 * self.hidden * self.inter
        return 2 * (self.layers * per_layer + 2 * self.vocab * self.hidden)


# Named architectures of BASELINE.json's configs (public HF configs; SURVEY.md Appendix C)
ARCHS: Dict[str, LlamaArch] = {
    "llama2-7b": LlamaArch(32000, 4096, 11008, 32, 32, 32, 128, 1e-5, 10000.0),
    "llama3-8b": LlamaArch(128256, 4096, 14336, 32, 32, 8, 128, 1e-5, 500000.0),
    "llama2-13b": LlamaArch(32000, 5120, 13824, 40, 40, 40, 128, 1e-5, 10000.0),
    "llama2-70b": LlamaArch(32000, 8192, 28672, 80, 64, 8, 128, 1e-5, 10000.0),
    # small shapes for tests / smoke (head_dim 128 as the kernels require)
    "tiny-mha": LlamaArch(512, 256, 704, 4, 2, 2, 128, 1e-5, 10000.0),
    "tiny-gqa": LlamaArch(640, 512, 1408, 6, 4, 2, 128, 1e-5, 10000.0),
    "small-1b": LlamaArch(32000, 2048, 5632, 8, 16, 16, 128, 1e-5, 10000.0),
    # two layers of Llama-2-7B width: numerics probes without 32 layers of perturbation growth
    "llama2-7b-l2": LlamaArch(32000, 4096, 11008, 2, 32, 32, 128, 1e-5, 10000.0),
    # per-rank shapes of Llama-2-70B at TP=8 when run at TP=4 (8 layers): hidden 8192, 8 q heads and
    # 1 kv head per rank, 3584 FFN columns per rank — multi-GPU smoke test of config 5 on 4 GPUs
    "mini70b-tp4": LlamaArch(32000, 8192, 14336, 8, 32, 4, 128, 1e-5, 10000.0),
    # facebook/layerskip-llama3.2-1B shape (the reference's own test model, tests/tests_constants.py:9):
    # head_dim 64, grouped KV, llama3 RoPE scaling, tied embeddings
    "llama3.2-1b": LlamaArch(128256, 2048, 8192, 16, 32, 8, 64, 1e-5, 500000.0, "llama3", 32.0, 1.0, 4.0, 8192),
    # correctness.py's CPU-runnable config (BASELINE.json configs[0]; SURVEY.md Appendix C)
    "survey-tiny": LlamaArch(512, 256, 688, 4, 8, 8, 32, 1e-5, 10000.0),
}


def classify(name: str) -> Optional[Tuple[int, int]]:
    """HF parameter name -> (role, layer) or None for tensors the engine does not need."""
    if name in _GLOBAL_ROLES:
        return _GLOBAL_ROLES[name], 0
    m = _LAYER_RE.match(name)
    if m and m.group(2) in _LAYER_ROLES:
        return _LAYER_ROLES[m.group(2)], int(m.group(1))
    return None


def iter_state_dict(sd: Dict[str, torch.Tensor], device: torch.device
                    ) -> Iterator[Tuple[int, int, torch.Tensor]]:
    """Yield (role, layer, bf16 tensor on `device`) for every tensor the engine consumes.
    A missing `lm_head.weight` means tied embeddings (HF omits it)."""
    seen_head = False
    for name, t in sd.items():
        rl = classify(name)
        if rl is None:
            continue
        seen_head |= rl[0] == _lib.LSK_W_LM_HEAD
        yield rl[0], rl[1], t.detach().to(device=device, dtype=torch.bfloat16).contiguous()
    if not seen_head:
        t = sd["model.embed_tokens.weight"]
        yield _lib.LSK_W_LM_HEAD, 0, t.detach().to(device=device, dtype=torch.bfloat16).contiguous()


class SyntheticLlama:
    """Random-init Llama whose tensors are generated on demand on the GPU.

    HF default init (N(0, 0.02^2) linears / embeddings, unit RMSNorm weights, SURVEY.md §8(d)),
    one `torch.Generator` per tensor seeded from (seed, tensor name) so every rank of a
    tensor-parallel job — and the CPU baseline — sees the same logical tensor.  `alpha` scales
    `o_proj` / `down_proj` of layers >= `damp_from` (SURVEY.md Appendix C) to control the greedy
    acceptance rate; values are rounded to bf16.
    """

    def __init__(self, arch: LlamaArch, seed: int = 0, alpha: float = 1.0,
                 damp_from: Optional[int] = None, device: str = "cuda", std: float = 0.02):
        self.arch = arch
        self.seed = seed
        self.alpha = alpha
        self.damp_from = damp_from
        self.device = torch.device(device)
        self.std = std

    # duck-typed like an HF model where the strategy needs it
    @property
    def config(self):
        a = self.arch
        return type("Cfg", (), dict(
            vocab_size=a.vocab, hidden_size=a.hidden, intermediate_size=a.inter,
            num_hidden_layers=a.layers, num_attention_heads=a.heads,
            num_key_value_heads=a.kv_heads, head_dim=a.head_dim, rms_norm_eps=a.rms_eps,
            rope_theta=a.rope_theta, rope_scaling=a.rope_config()))()

    def names(self):
        a = self.arch
        yield "model.embed_tokens.weight", (a.vocab, a.hidden)
        for i in range(a.layers):
            p = f"model.layers.{i}."
            yield p + "input_layernorm.weight", (a.hidden,)
            yield p + "self_attn.q_proj.weight", (a.q_dim, a.hidden)
            yield p + "self_attn.k_proj.weight", (a.kv_dim, a.hidden)
            yield p + "self_attn.v_proj.weight", (a.kv_dim, a.hidden)
            yield p + "self_attn.o_proj.weight", (a.hidden, a.q_dim)
            yield p + "post_attention_layernorm.weight", (a.hidden,)
            yield p + "mlp.gate_proj.weight", (a.inter, a.hidden)
            yield p + "mlp.up_proj.weight", (a.inter, a.hidden)
            yield p + "mlp.down_proj.weight", (a.hidden, a.inter)
        yield "model.norm.weight", (a.hidden,)
        yield "lm_head.weight", (a.vocab, a.hidden)

    def tensor(self, name: str, shape) -> torch.Tensor:
        if name.endswith("layernorm.weight") or name == "model.norm.weight":
            return torch.ones(shape, dtype=torch.bfloat16, device=self.device)
        # stable per-tensor seed (python's hash() is salted per process)
        h = 1469598103934665603
        for ch in f"{self.seed}:{name}".encode():
            h = ((h ^ ch) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
        g = torch.Generator(device=self.device).manual_seed(h & 0x7FFFFFFFFFFFFFFF)
        t = torch.randn(shape, generator=g, device=self.device, dtype=torch.float32) * self.std
        m = _LAYER_RE.match(name)
        if (m and self.damp_from is not None and int(m.group(1)) >= self.damp_from
                and m.group(2) in ("self_attn.o_proj", "mlp.down_proj")):
            t = t * self.alpha
        return t.to(torch.bfloat16)

    def iter_weights(self, device: torch.device) -> Iterator[Tuple[int, int, torch.Tensor]]:
        for name, shape in self.names():
            role, layer = classify(name)
            yield role, layer, self.tensor(name, shape).to(device)

    def state_dict(self, dtype: torch.dtype = torch.bfloat16, device: str = "cpu"
                   ) -> Dict[str, torch.Tensor]:
        """Materialise everything (used to hand the CPU baseline the same weights)."""
        return {name: self.tensor(name, shape).to(device=device, dtype=dtype)
                for name, shape in self.names()}

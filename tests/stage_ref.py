"""Float64 restatement of the engine's decoder layer that rounds to bf16 exactly where the kernels do.

The kernels' comments are the specification (gemm_skinny.cuh, prefill_tc.cuh, attention.cuh):

- residual stream: fp32, starting from the bf16 embedding row;
- RMSNorm (`rms_rows_group`, `rms_canon_kernel`): rstd = rsqrt(mean(x^2) + eps), then ONE rounding
  to bf16 of w * (x * rstd) — not HF's two roundings (the oracle tests cover HF parity).  rstd and
  both products are fp32 as in the kernels: a row whose fp32 rstd has a short mantissa puts many
  products exactly on bf16 ties, and only the fp32 products break those ties the kernels' way;
- q / k / v: dot products of the bf16 operands, RoPE on the unrounded q / k, then bf16;
- RoPE table: the engine's own (engine.cu, `lsk_create`): float32 inv_freq through C `powf` and the
  float32 scaling rules in the same operation order, the angle as a float32 product, cos / sin in
  double of the float angle, rounded to float;
- attention: scores times the float32 1/sqrtf(head_dim), causal mask by absolute position,
  probabilities rounded to bf16 before P.V, output rounded to bf16 (the kernel rounds
  exp(s - running max) per 16-key slice instead: the tolerances cover that);
- O / down projections added to the fp32 residual; SiLU.up = bf16(silu(g) * u) from unrounded g, u;
- final RMSNorm + LM head: fp32 logits, arg-max with the lowest index winning.

Everything runs in float64 on the GPU; weights stay bf16 and are widened per product.  A layer can
start from K/V rows read back from the engine, so one stage is checked without the rounding flips
of the stages before it.  The `check_*` functions compare an engine tensor with the reference and
return a `Report` naming the stage and the (layer, head, position) of the worst element.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import numpy as np
import torch

F64 = torch.float64


def bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(x.dtype)


def f32(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(x.dtype)


_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.powf.restype = ctypes.c_float
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]


def rope_table(arch, n_pos: int):
    """(cos, sin) float32 [n_pos, head_dim / 2], bit for bit the engine's table."""
    f = np.float32
    hd, half = arch.head_dim, arch.head_dim // 2
    cos = np.empty((n_pos, half), np.float32)
    sin = np.empty((n_pos, half), np.float32)
    for d in range(half):
        inv = f(1.0) / f(_libm.powf(f(arch.rope_theta), f(2 * d) / f(hd)))
        if arch.rope_scaling == "linear":
            inv = inv / f(arch.rope_factor)
        elif arch.rope_scaling == "llama3":
            old = f(arch.rope_original_max_pos)
            lo_f, hi_f, fac = f(arch.rope_low_freq_factor), f(arch.rope_high_freq_factor), f(arch.rope_factor)
            low_wl, high_wl = old / lo_f, old / hi_f
            wl = f(2.0) * f(math.pi) / inv
            scaled = inv / fac if wl > low_wl else inv
            if not (wl < high_wl) and not (wl > low_wl):
                smooth = (old / wl - lo_f) / (hi_f - lo_f)
                scaled = (f(1.0) - smooth) * scaled / fac + smooth * scaled
            inv = scaled
        for p in range(n_pos):
            ang = float(f(p) * inv)
            cos[p, d] = math.cos(ang)
            sin[p, d] = math.sin(ang)
    return torch.from_numpy(cos), torch.from_numpy(sin)


class RefModel:
    """The engine's arithmetic on bf16 weights (HF-named state dict), float64 on `device`."""

    def __init__(self, arch, sd: Dict[str, torch.Tensor], n_pos: int, device="cuda"):
        self.arch, self.dev = arch, device
        b = lambda name: sd[name].to(device=device, dtype=torch.bfloat16)
        self.embed_w = b("model.embed_tokens.weight")
        self.final_norm = b("model.norm.weight")
        self.lm_head = b("lm_head.weight") if "lm_head.weight" in sd else self.embed_w
        self.layers = []
        for i in range(arch.layers):
            p = f"model.layers.{i}."
            self.layers.append(dict(
                ln1=b(p + "input_layernorm.weight"), wq=b(p + "self_attn.q_proj.weight"),
                wk=b(p + "self_attn.k_proj.weight"), wv=b(p + "self_attn.v_proj.weight"),
                wo=b(p + "self_attn.o_proj.weight"), ln2=b(p + "post_attention_layernorm.weight"),
                wg=b(p + "mlp.gate_proj.weight"), wu=b(p + "mlp.up_proj.weight"),
                wd=b(p + "mlp.down_proj.weight")))
        cos, sin = rope_table(arch, n_pos)
        self.cos, self.sin = cos.to(device, F64), sin.to(device, F64)
        self.scale = float(np.float32(1.0) / np.sqrt(np.float32(arch.head_dim)))

    # ---------------------------------------------------------------- stages
    def embed(self, ids: Sequence[int]) -> torch.Tensor:
        return self.embed_w[torch.tensor(list(ids), device=self.dev)].to(F64)

    def rstd(self, x: torch.Tensor) -> torch.Tensor:
        """fp32 rsqrtf(sum(x^2) / K + eps) (rounded correctly here; rsqrtf is within 2 ulp)."""
        eps = float(np.float32(self.arch.rms_eps))
        return f32(torch.rsqrt(f32(f32(x.pow(2).mean(-1, keepdim=True)) + eps)))

    def norm(self, x: torch.Tensor, w: torch.Tensor, rstd: Optional[torch.Tensor] = None) -> torch.Tensor:
        return bf16(f32(w.to(F64) * f32(x * (self.rstd(x) if rstd is None else rstd))))

    @staticmethod
    def mm(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
        return x @ w.to(F64).t()

    def rope(self, x: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        """x [n, heads, hd] unrounded, pos [n] absolute positions."""
        half = x.shape[-1] // 2
        c, s = self.cos[pos][:, None, :], self.sin[pos][:, None, :]
        lo, hi = x[..., :half], x[..., half:]
        return torch.cat([lo * c - hi * s, hi * c + lo * s], -1)

    def qkv(self, li: int, x: torch.Tensor, pos: torch.Tensor, rstd: Optional[torch.Tensor] = None):
        """fp32 residual rows [n, hidden] at positions pos [n] -> bf16 q [n, H, hd], k / v [n, KV, hd]."""
        a, L = self.arch, self.layers[li]
        xn = self.norm(x, L["ln1"], rstd)
        q = self.mm(xn, L["wq"]).view(-1, a.heads, a.head_dim)
        k = self.mm(xn, L["wk"]).view(-1, a.kv_heads, a.head_dim)
        v = self.mm(xn, L["wv"]).view(-1, a.kv_heads, a.head_dim)
        return bf16(self.rope(q, pos)), bf16(self.rope(k, pos)), bf16(v)

    def attend(self, q: torch.Tensor, pos: torch.Tensor, K: torch.Tensor, V: torch.Tensor,
               n_keys: Optional[torch.Tensor] = None) -> torch.Tensor:
        """q [n, H, hd] at positions pos [n]; K / V [ctx, KV, hd] for positions 0 .. ctx-1.
        Row i sees keys 0 .. pos[i] (or the first n_keys[i] keys) -> bf16 [n, H * hd].  Long
        contexts run in row chunks that keep the float64 scores near 1 GiB (rows are independent)."""
        a = self.arch
        step = max(1, 2 ** 27 // (a.heads * K.shape[0]))
        if q.shape[0] > step:
            return torch.cat([self.attend(q[i:i + step], pos[i:i + step], K, V,
                                          None if n_keys is None else n_keys[i:i + step])
                              for i in range(0, q.shape[0], step)])
        group = a.heads // a.kv_heads
        Kh = K.permute(1, 0, 2).repeat_interleave(group, 0)           # [H, ctx, hd]
        Vh = V.permute(1, 0, 2).repeat_interleave(group, 0)
        s = torch.einsum("nhd,hcd->hnc", q, Kh) * self.scale
        lim = (pos + 1) if n_keys is None else n_keys
        visible = torch.arange(K.shape[0], device=self.dev)[None, :] < lim[:, None]
        s = s.masked_fill(~visible[None], float("-inf"))
        p = bf16(torch.softmax(s, -1))
        return bf16(torch.einsum("hnc,hcd->nhd", p, Vh)).reshape(q.shape[0], -1)

    def layer_rest(self, li: int, x: torch.Tensor, attn: torch.Tensor) -> torch.Tensor:
        """O projection, residual, RMSNorm, gate / up, SiLU.up, down, residual (fp32 rows)."""
        L = self.layers[li]
        x = f32(x + self.mm(attn, L["wo"]))
        xn = self.norm(x, L["ln2"])
        act = bf16(torch.nn.functional.silu(self.mm(xn, L["wg"])) * self.mm(xn, L["wu"]))
        return f32(x + self.mm(act, L["wd"]))

    def logits(self, x: torch.Tensor, rstd: Optional[torch.Tensor] = None) -> torch.Tensor:
        return f32(self.mm(self.norm(x, self.final_norm, rstd), self.lm_head))


# -------------------------------------------------------------------- comparisons
@dataclass
class Report:
    stage: str
    ok: bool
    worst: float                  # the statistic the bound applies to, at its worst
    where: str                    # (layer, head, position) of the worst element
    detail: str = ""

    def __str__(self):
        return f"{self.stage}: {'ok' if self.ok else 'VIOLATION'} worst={self.worst:.4g} at {self.where} {self.detail}"


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |x| (8 significant bits)."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))      # |x| = f * 2^e, f in [0.5, 1): exact
    return torch.ldexp(torch.ones_like(x), e - 8)


def _where(layer, idx, heads_axis: bool, pos0: int):
    if heads_axis:                # [pos, head, dim]
        p, h, d = idx
        return f"(layer {layer}, head {h}, position {pos0 + p}, dim {d})"
    p, d = idx
    return f"(layer {layer}, position {pos0 + p}, column {d})"


def check_direct(stage: str, got: torch.Tensor, want: torch.Tensor, layer: int, pos0: int = 0,
                 units: float = 1.0, floor: float = 2.0 ** -12, min_identical: float = 0.99,
                 min_identical_pos: float = 0.0) -> Report:
    """bf16 outputs of one fp32-accumulated GEMM, [pos, head, dim]: every element within `units`
    bf16 ulps of the reference (an absolute floor of `floor` x the (position, head) row's RMS per
    unit covers near-zero values after the RoPE subtraction), at least `min_identical` of all
    elements bit-identical, and at least `min_identical_pos` of each position's elements."""
    got, want = got.to(F64), want.to(F64).to(got.device)
    rms = want.pow(2).mean(-1, keepdim=True).sqrt()
    tol = torch.maximum(bf16_ulp(torch.maximum(got.abs(), want.abs())), floor * rms)
    ratio = (got - want).abs() / tol
    i = int(ratio.argmax())
    idx = np.unravel_index(i, tuple(ratio.shape))
    worst = float(ratio.reshape(-1)[i])
    per_pos = (got == want).double().flatten(1).mean(1)
    same, low = float(per_pos.mean()), int(per_pos.argmin())
    ok = (worst <= units and same >= min_identical and float(per_pos[low]) >= min_identical_pos
          and bool(torch.isfinite(got).all()))
    return Report(stage, ok, worst, _where(layer, idx, True, pos0),
                  f"(|d| / (1 ulp or floor), bound {units:g}; got {float(got[idx]):.6g} want {float(want[idx]):.6g}; "
                  f"identical {same:.5f}, least at position {pos0 + low}: {float(per_pos[low]):.4f})")


def check_rows(stage: str, got: torch.Tensor, want: torch.Tensor, bound: float, layer: int, pos0: int = 0
               ) -> Report:
    """Downstream stages: per row (last axis), max|got - want| <= bound x that row's RMS."""
    got, want = got.to(F64), want.to(F64).to(got.device)
    rms = want.pow(2).mean(-1, keepdim=True).sqrt().clamp_min(1e-30)
    rel = ((got - want).abs() / rms).amax(-1)
    i = int(rel.argmax())
    idx = np.unravel_index(i, tuple(rel.shape))
    worst = float(rel.reshape(-1)[i])
    heads_axis = rel.dim() == 2
    where = (f"(layer {layer}, head {idx[1]}, position {pos0 + idx[0]})" if heads_axis
             else f"(layer {layer}, position {pos0 + idx[0]})")
    ok = worst <= bound and bool(torch.isfinite(got).all())
    return Report(stage, ok, worst, where, f"(max|d| / row RMS, bound {bound:.3g})")

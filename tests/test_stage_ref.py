"""CPU: the float64 stage reference (tests/stage_ref.py) itself — its RoPE table agrees with the
oracle's fp32 HF restatement for all three scaling rules, and its comparisons accept a one-ulp bf16
rounding flip but report a two-ulp error or a shifted row, naming where."""
import pytest
import torch

from layerskip_b200.weights import LlamaArch
from oracle import llama_oracle as orc
from tests import stage_ref as sr

ROPES = {
    "default": {},
    "linear": dict(rope_scaling="linear", rope_factor=4.0),
    "llama3": dict(rope_scaling="llama3", rope_factor=32.0, rope_low_freq_factor=1.0,
                   rope_high_freq_factor=4.0, rope_original_max_pos=8192),
}


@pytest.mark.parametrize("kind", list(ROPES))
def test_rope_table_matches_the_hf_float32_table(kind):
    arch = LlamaArch(512, 256, 688, 2, 8, 4, 64, 1e-5, 500000.0, **ROPES[kind])
    dims = orc.LlamaDims(512, 256, 688, 2, 8, 4, 64, 1e-5, 500000.0, arch.rope_config())
    cos, sin = sr.rope_table(arch, 2100)
    c2, s2 = orc.rope_tables(dims, torch.arange(2100), torch.float32)
    # the same float32 angles; cos / sin through double here, float32 in torch: <= 1 float ulp apart
    assert float((cos - c2[:, :32]).abs().max()) <= 2 ** -23
    assert float((sin - s2[:, :32]).abs().max()) <= 2 ** -23


def test_comparisons_name_the_worst_element():
    g = torch.Generator().manual_seed(0)
    want = torch.randn(40, 4, 64, generator=g, dtype=torch.float64).to(torch.bfloat16).double()
    assert sr.check_direct("k", want.clone(), want, 0).ok
    got = want.clone()
    got[7, 2, 5] = want[7, 2, 5] + sr.bf16_ulp(want[7, 2, 5])          # one ulp: a rounding flip
    assert sr.check_direct("k", got, want, 0).ok
    got[7, 2, 5] = want[7, 2, 5] + 2 * sr.bf16_ulp(want[7, 2, 5])      # two ulps: an error
    rep = sr.check_direct("k", got, want, 3, pos0=100)
    assert not rep.ok and "head 2, position 107, dim 5" in rep.where, rep
    rows = torch.randn(16, 4096, generator=g, dtype=torch.float64)
    assert sr.check_rows("h", rows, rows, 1e-3, 0).ok
    bad = rows.clone()
    bad[9] = rows[10]
    rep = sr.check_rows("h", bad, rows, 1e-3, 1, pos0=60)
    assert not rep.ok and rep.where == "(layer 1, position 69)", rep

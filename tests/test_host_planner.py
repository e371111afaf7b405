"""CPU: the host-side GEMM launch planner (engine.cu: plan_sched, through lsk_plan_gemm) for the
architectures BASELINE.json names — shared-memory fit, K-chunking, ring depth, even-wave grids."""
import ctypes as C

import pytest

from layerskip_b200 import _lib
from layerskip_b200.weights import ARCHS

PRO_RMS, PRO_BF16 = 0, 1
EPI_QKV, EPI_RESID, EPI_STORE, EPI_SILU, EPI_LMHEAD = range(5)
SMS = 132                      # H100 SXM


def plan(n_rows, k, m, pro, epi, sms=SMS):
    lib = _lib.load()
    out = _lib.lsk_gemm_plan()
    _lib.check(lib.lsk_plan_gemm(n_rows, k, m, pro, epi, sms, C.byref(out)))
    return out


def gemms_of(arch, tp=1):
    h, q, kv, i, v = arch.hidden, arch.q_dim // tp, arch.kv_dim // tp, arch.inter // tp, arch.vocab // tp
    v = (v + 15) // 16 * 16
    return {"qkv": (q + 2 * kv, h, PRO_RMS, EPI_QKV), "o": (h, q, PRO_BF16, EPI_RESID),
            "gate_up": (2 * i, h, PRO_RMS, EPI_SILU), "down": (h, i, PRO_BF16, EPI_RESID),
            "lm_head": (v, h, PRO_RMS, EPI_LMHEAD)}


@pytest.mark.parametrize("name,tp", [("llama2-7b", 1), ("llama3-8b", 1), ("llama2-13b", 2),
                                     ("llama2-13b", 8), ("llama2-70b", 8), ("tiny-gqa", 1)])
@pytest.mark.parametrize("m", [1, 7, 8])
def test_every_decode_gemm_fits_and_keeps_a_deep_ring(name, tp, m):
    for gname, (n, k, pro, epi) in gemms_of(ARCHS[name], tp).items():
        p = plan(n, k, m, pro, epi)
        assert p.ok, (name, gname)
        assert p.smem_bytes <= p.smem_limit == 227 * 1024
        assert p.block == 640 and 1 <= p.grid <= SMS
        assert p.ring_stages * p.stage_bytes >= 64 * 1024 or p.n_tiles * k < 2 ** 18, (name, gname, p.ring_stages)
        assert p.n_chunks == 1 or (p.tiles_per_pass == 2 and pro == PRO_BF16)
        assert p.n_chunks * p.chunk_cols >= k


def test_7b_schedules_match_design_md():
    a = ARCHS["llama2-7b"]
    g = gemms_of(a)
    p = plan(*g["qkv"][:2], 1, *g["qkv"][2:])
    assert (p.n_tiles, p.grid, p.n_chunks, p.ring_stages) == (768, 128, 1, 8)      # 768 = 6 x 128
    p = plan(*g["gate_up"][:2], 1, *g["gate_up"][2:])
    assert (p.n_tiles, p.grid) == (1376, 126)                                      # 11 waves of 126
    p = plan(*g["lm_head"][:2], 1, *g["lm_head"][2:])
    assert (p.n_tiles, p.grid) == (2000, 125)                                      # 16 waves of 125
    p1 = plan(*g["down"][:2], 1, *g["down"][2:])
    p7 = plan(*g["down"][:2], 7, *g["down"][2:])
    assert p1.n_chunks == 1 and p1.ring_stages == 8          # one resident row: no chunking
    assert p7.n_chunks == 2 and p7.tiles_per_pass == 2       # 7 rows x 22 KB do not fit next to the ring
    assert p7.grid == 128


def test_sixteen_row_blocks_and_their_limits():
    a = ARCHS["llama2-7b"]
    n, k, pro, epi = gemms_of(a)["qkv"]
    p = plan(n, k, 16, pro, epi)
    assert p.ok and p.nt == 2
    assert p.n_chunks == 1                                        # hidden 4096: 16 whole rows fit
    # hidden 8192 / 5120: 16 whole rows do not fit next to the ring -> K-chunked RMSNorm mode
    # (statistics up front, rows normalised chunk by chunk); up to 8 rows stay resident as before
    for name, tp in (("llama2-70b", 8), ("llama2-13b", 1)):
        for key in ("qkv", "gate_up", "lm_head"):
            n, k, pro, epi = gemms_of(ARCHS[name], tp)[key]
            p16, p8 = plan(n, k, 16, pro, epi), plan(n, k, 8, pro, epi)
            assert p16.ok and p16.nt == 2 and p16.n_chunks > 1 and p16.tiles_per_pass == 2, (name, key)
            assert p16.ring_stages >= 2 and p16.smem_bytes <= p16.smem_limit
            assert p8.ok and p8.n_chunks == 1, (name, key)


def test_bad_queries_are_rejected():
    lib = _lib.load()
    out = _lib.lsk_gemm_plan()
    assert lib.lsk_plan_gemm(100, 4096, 1, 0, 0, SMS, C.byref(out)) != 0      # rows % 16
    assert lib.lsk_plan_gemm(128, 100, 1, 0, 0, SMS, C.byref(out)) != 0       # k % 32
    assert lib.lsk_plan_gemm(128, 4096, 17, 0, 0, SMS, C.byref(out)) != 0     # rows > 16
    assert b"bad plan query" in lib.lsk_last_error()


def attn_plan(arch, m, tp=1, sms=SMS):
    lib = _lib.load()
    out = _lib.lsk_attn_plan()
    _lib.check(lib.lsk_plan_attention(arch.head_dim, arch.heads // tp, arch.kv_heads // tp, m, sms, C.byref(out)))
    return out


def test_attention_launch_plan_for_the_baseline_architectures():
    """engine.cu: attn_default_splits / plan_attention_launch (through lsk_plan_attention): the split
    count is min(4, SMs / local kv heads), the K/V ring is as deep as shared memory allows, and a grid
    that fits one wave gets more than half an SM's shared memory per CTA (one CTA per SM)."""
    p = attn_plan(ARCHS["llama2-7b"], 7)                       # 32 kv heads: 32 x 4 CTAs on 132 SMs
    assert (p.ok, p.n_splits, p.grid, p.ring_stages, p.row_blocks) == (1, 4, 128, 4, 1)
    assert p.smem_bytes > 114 * 1024 and p.kv_refetched_per_row_block == 1   # merge buffer aliases the ring
    p = attn_plan(ARCHS["llama3-8b"], 7)                       # GQA 4: 28 query rows -> 2 row blocks, K/V resident
    assert (p.n_splits, p.grid, p.row_blocks, p.kv_refetched_per_row_block) == (4, 32, 2, 0)
    p = attn_plan(ARCHS["llama2-13b"], 7)                      # 40 kv heads -> 3 splits (120 CTAs)
    assert (p.n_splits, p.grid) == (3, 120)
    p = attn_plan(ARCHS["llama2-70b"], 7, tp=8)                # one kv head per rank, 8 q heads share it
    assert (p.ok, p.n_splits, p.grid, p.row_blocks) == (1, 4, 4, 4)
    p = attn_plan(ARCHS["llama2-7b"], 128)                     # prompt pass: 128 query rows per launch
    assert p.ok == 1 and p.row_blocks == 8 and p.smem_bytes <= p.smem_limit
    p = attn_plan(ARCHS["llama3-8b"], 128)                     # 512 rows do not fit: the engine launches 48 at a time
    assert p.ok == 0
    assert attn_plan(ARCHS["llama3-8b"], 48).ok == 1
    p = attn_plan(ARCHS["llama3.2-1b"], 16)                    # head_dim 64: 8 KiB K/V blocks
    assert p.ok == 1 and p.ring_stages == 4
    for bad in ((96, 32, 32, 7), (128, 32, 5, 7), (128, 32, 32, 0)):
        out = _lib.lsk_attn_plan()
        assert _lib.load().lsk_plan_attention(bad[0], bad[1], bad[2], bad[3], SMS, C.byref(out)) == -1

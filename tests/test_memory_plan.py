"""CPU: the HBM budget (layerskip_b200/memory.py) for the architectures BASELINE.json names."""
import pytest

from layerskip_b200.memory import HBM_PER_GPU, check_fits, plan_memory
from layerskip_b200.weights import ARCHS


def test_weight_bytes_match_the_architecture():
    for name in ("llama2-7b", "llama3-8b", "llama2-13b", "llama2-70b"):
        a = ARCHS[name]
        p = plan_memory(a, max_ctx=704, prefill_tc=False)
        assert abs(p["weights"] + p["embed"] + p["lm_head"] - a.param_bytes()) < 2e-3 * a.param_bytes(), name
        # default: + the canonical-layout copy of the LAYER weights for the tensor-core prompt pass
        both = plan_memory(a, max_ctx=704)
        layer_bytes = a.param_bytes() - 2 * 2 * a.vocab * a.hidden
        assert abs(both["weights"] - p["weights"] - layer_bytes) < 2e-2 * layer_bytes, name
    p7 = plan_memory(ARCHS["llama2-7b"], max_ctx=704, prefill_tc=False)
    assert 13.3e9 < p7["weights"] + p7["embed"] + p7["lm_head"] < 13.6e9
    assert abs(p7["kv_pool"] - 11 * 64 * 32 * 4096 * 2 * 2) == 0          # 512 KiB per token


def test_tensor_parallel_shards_divide_weights_and_kv():
    a = ARCHS["llama2-70b"]
    one, eight = plan_memory(a, 4096, 1, prefill_tc=False), plan_memory(a, 4096, 8, prefill_tc=False)
    assert abs(eight["weights"] * 8 - one["weights"]) < 1e-3 * one["weights"]   # norms are replicated
    assert eight["kv_pool"] * 8 == one["kv_pool"]
    assert eight["embed"] == one["embed"]                                   # replicated


def test_baseline_configs_fit_an_h100_and_70b_needs_tp():
    free = int(HBM_PER_GPU * 0.97)
    check_fits(ARCHS["llama2-7b"], free, max_ctx=4096)
    check_fits(ARCHS["llama3-8b"], free, max_ctx=8192, sampling=True)
    check_fits(ARCHS["llama2-13b"], free, max_ctx=4096, tp_size=2)
    check_fits(ARCHS["llama2-13b"], free, max_ctx=4096, tp_size=1)                      # 55 GB with both copies
    check_fits(ARCHS["llama2-70b"], free, max_ctx=4096, tp_size=8)
    check_fits(ARCHS["llama2-70b"], free, max_ctx=4096, tp_size=2, prefill_tc=False)   # 69 GB of weights per rank: fits alone
    with pytest.raises(MemoryError):
        check_fits(ARCHS["llama2-70b"], free, max_ctx=4096, tp_size=2)      # ... but not with the second copy
    with pytest.raises(MemoryError):
        check_fits(ARCHS["llama2-70b"], free, max_ctx=4096, tp_size=1, prefill_tc=False)   # 140 GB: needs TP
    with pytest.raises(MemoryError, match="larger tp_size or a smaller max_ctx"):
        check_fits(ARCHS["llama2-70b"], free, max_ctx=131072, tp_size=2, prefill_tc=False)    # + 21 GB of KV does not
    with pytest.raises(MemoryError):
        check_fits(ARCHS["llama2-7b"], 8 * 10 ** 9, max_ctx=704)


def test_engine_refuses_a_configuration_that_cannot_fit_before_creating_an_engine(monkeypatch):
    """Engine.__init__ runs the budget check first: with 8 GB 'free' a 7B engine must raise
    MemoryError and lsk_create must never be called."""
    import torch
    from layerskip_b200 import _lib, engine

    calls = []
    real = _lib.load()

    class FakeLib:
        def lsk_create(self, *a):
            calls.append("create")
            return -2

        def lsk_plan_memory(self, *a):
            return real.lsk_plan_memory(*a)

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "get_device_properties",
                        lambda dev=None: type("Props", (), dict(multi_processor_count=132))())
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (8 * 10 ** 9, 80 * 10 ** 9))
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    with pytest.raises(MemoryError, match="only 8.0 GB are free"):
        engine.Engine(ARCHS["llama2-7b"], max_ctx=704)
    assert calls == []


def _lib_plan(arch, sm_count=132, max_ctx=4096, tp_size=1, flags=0, **uses):
    import ctypes as C
    from layerskip_b200 import _lib
    cfg = arch.lsk_config(max_ctx, tp_size=tp_size, flags=flags)
    plan = _lib.lsk_memory_plan()
    code = _lib.load().lsk_plan_memory(C.byref(cfg), sm_count, C.byref(_lib.lsk_memory_uses(**uses)),
                                       C.byref(plan))
    return code, plan


def test_plan_refuses_the_configs_lsk_create_refuses_with_its_code_and_message():
    import ctypes as C
    from layerskip_b200 import _lib
    lib = _lib.load()
    base = dict(vocab=512, hidden=256, inter=704, n_layers=2, n_heads=2, n_kv_heads=2, head_dim=128, rms_eps=1e-5,
                rope_theta=1e4, max_ctx=128, tp_rank=0, tp_size=1, attn_splits=0, flags=0, rope_scaling=0,
                rope_factor=1.0)
    uses, plan = _lib.lsk_memory_uses(), _lib.lsk_memory_plan()
    for bad in (dict(head_dim=96), dict(tp_rank=2, tp_size=2), dict(n_heads=3), dict(hidden=8200), dict(inter=700),
                dict(rope_scaling=2, rope_factor=0.0), dict(max_ctx=1), dict(vocab=511, tp_size=2),
                dict(n_heads=32, n_kv_heads=1)):
        c = _lib.lsk_config(**{**base, **bad})
        h = C.c_void_p()
        want = lib.lsk_create(C.byref(c), C.byref(h)), lib.lsk_last_error()
        assert want[0] == -1 and not h.value, bad
        assert (lib.lsk_plan_memory(C.byref(c), 132, C.byref(uses), C.byref(plan)), lib.lsk_last_error()) == want, bad
    c = _lib.lsk_config(**base)
    assert lib.lsk_plan_memory(C.byref(c), 132, C.byref(uses), C.byref(plan)) == 0
    assert lib.lsk_plan_memory(C.byref(c), 0, C.byref(uses), C.byref(plan)) == -1
    assert lib.lsk_plan_memory(None, 132, C.byref(uses), C.byref(plan)) == -1


def test_plan_counts_the_peer_region_of_the_one_shot_collectives():
    """tp_size > 1: the peer region lsk_comm_init allocates, at tp_peer.cuh's peer_region_layout size
    (256-byte aligned blocks: fp32 rows, LL lines, all-reduce flags, arg-max slots and flags, GEMM
    flags, the owner's counters)."""
    def align(b):
        return (b + 255) // 256 * 256

    for name, tp in (("llama2-13b", 2), ("llama2-70b", 8)):
        a = ARCHS[name]
        rows = 16 * a.hidden
        region = (align(2 * tp * rows * 4) + align(2 * tp * rows * 8) + align(tp * 64 * 4) + align(2 * tp * 32 * 4)
                  + align(tp * 4) + align(tp * 160 * 4) + align(16))
        code, without = _lib_plan(a, tp_size=tp)
        assert code == 0
        p = plan_memory(a, tp_size=tp)
        assert p["scratch"] - without.scratch == region, name
        assert p["total"] - without.total == region, name


def test_plan_scales_the_scratch_with_the_sm_count():
    """One arg-max candidate slot per SM and row; the default attention split count is
    floor(SMs / kv heads) up to 4, so fewer SMs can also mean fewer split partials."""
    a = ARCHS["tiny-mha"]                         # 2 kv heads: 4 splits at 132 and at 96 SMs
    big, small = plan_memory(a, sm_count=132), plan_memory(a, sm_count=96)
    assert big["scratch"] - small["scratch"] == (132 - 96) * 16 * 8
    assert {k: v for k, v in big.items() if k not in ("scratch", "total")} == \
        {k: v for k, v in small.items() if k not in ("scratch", "total")}
    a = ARCHS["llama2-7b"]                        # 32 kv heads: 4 splits at 132 SMs, 3 at 96
    big, small = plan_memory(a, sm_count=132), plan_memory(a, sm_count=96)
    assert big["scratch"] - small["scratch"] == (132 - 96) * 16 * 8 + 32 * 128 * (128 + 2) * 4

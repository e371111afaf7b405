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


def test_engine_refuses_a_configuration_that_cannot_fit_before_touching_the_library(monkeypatch):
    """Engine.__init__ runs the budget check first: with 8 GB 'free' a 7B engine must raise
    MemoryError and lsk_create must never be called."""
    import torch
    from layerskip_b200 import _lib, engine

    calls = []

    class FakeLib:
        def lsk_create(self, *a):
            calls.append("create")
            return -2

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (8 * 10 ** 9, 80 * 10 ** 9))
    monkeypatch.setattr(_lib, "load", lambda: FakeLib())
    with pytest.raises(MemoryError, match="only 8.0 GB are free"):
        engine.Engine(ARCHS["llama2-7b"], max_ctx=704)
    assert calls == []

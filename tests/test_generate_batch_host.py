"""CPU: batched generation's host side — the memory plan of its buffers, the slot sizes of a batch and
the refusals of `generate_batch` that need no device."""
import ctypes as C
import json
import os

import pytest

from layerskip_b200 import _lib
from layerskip_b200.engine import batch_slot_positions
from layerskip_b200.memory import plan_memory
from layerskip_b200.plugin import GenerationConfig
from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy
from layerskip_b200.weights import ARCHS

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "memory_plan_parent.json")
DEVSTATE_BYTES = 56 * 4          # common.cuh: DevState, 56 four-byte fields


def _plan(arch, max_ctx, tp_size, flags, sm_count, **uses):
    cfg = arch.lsk_config(max_ctx, tp_size=tp_size, flags=flags)
    plan = _lib.lsk_memory_plan()
    code = _lib.load().lsk_plan_memory(C.byref(cfg), sm_count, C.byref(_lib.lsk_memory_uses(**uses)),
                                       C.byref(plan))
    assert code == 0, _lib.load().lsk_last_error()
    return [getattr(plan, f) for f, _ in _lib.lsk_memory_plan._fields_]


def test_plans_without_a_batch_are_the_recorded_plans():
    """Every recorded (architecture, tp, flags, uses) plan of the library before batched generation
    existed is unchanged with batch_seqs = 0."""
    g = json.load(open(GOLDEN))
    assert g["fields"] == [f for f, _ in _lib.lsk_memory_plan._fields_]
    for r in g["rows"]:
        got = _plan(ARCHS[r["arch"]], r["max_ctx"], r["tp_size"], r["flags"], g["sm_count"],
                    tp_peer=int(r["tp_size"] > 1), batch_seqs=0, **g["uses"][r["uses"]])
        assert got == r["plan"], r


@pytest.mark.parametrize("name", ["tiny-mha", "tiny-gqa", "llama2-7b", "llama2-13b"])
def test_a_batch_adds_exactly_its_buffers(name):
    """batch_seqs > 0 adds the per-sequence states, the round's d_seq / active flags and the attention
    arrival counters, all sized for 16 sequences whatever the count; nothing else changes."""
    a = ARCHS[name]
    base = plan_memory(a, max_ctx=1000)
    extra = 16 * DEVSTATE_BYTES + 2 * 16 * 4 + 16 * a.kv_heads * 4
    for n in (1, 3, 16):
        p = plan_memory(a, max_ctx=1000, batch_seqs=n)
        assert p["scratch"] - base["scratch"] == extra, n
        assert p["total"] - base["total"] == extra, n
        assert {k: v for k, v in p.items() if k not in ("scratch", "total")} == \
            {k: v for k, v in base.items() if k not in ("scratch", "total")}


def test_plan_refuses_a_batch_beyond_the_row_limit():
    a = ARCHS["tiny-mha"]
    cfg = a.lsk_config(1000)
    plan = _lib.lsk_memory_plan()
    lib = _lib.load()
    for bad in (-1, 17):
        assert lib.lsk_plan_memory(C.byref(cfg), 132, C.byref(_lib.lsk_memory_uses(batch_seqs=bad)),
                                   C.byref(plan)) == -1
        assert b"batch_seqs" in lib.lsk_last_error()


def test_slot_sizes():
    """ceil(max_ctx / 64) pages split into n_seqs slots of whole pages; the remainder goes unused."""
    assert batch_slot_positions(4096, 1) == 4096
    assert batch_slot_positions(4096, 3) == 21 * 64          # 64 pages: 3 slots of 21, one page spare
    assert batch_slot_positions(4096, 16) == 256
    assert batch_slot_positions(1000, 1) == 1024             # 16 pages: the pool rounds max_ctx up
    assert batch_slot_positions(1000, 2) == 512
    assert batch_slot_positions(1000, 3) == 5 * 64
    assert batch_slot_positions(1000, 7) == 2 * 64
    assert batch_slot_positions(1000, 16) == 64
    assert batch_slot_positions(1000, 17) == 0               # more sequences than pages: nothing fits
    assert batch_slot_positions(65, 5) == 0
    with pytest.raises(ValueError):
        batch_slot_positions(1000, 0)


class _FakeEngine:
    max_rows, max_ctx = 16, 1000

    def begin(self, *a, **k):
        raise AssertionError("refused too late: begin ran")

    prefill_batch = begin


def _strategy():
    s = B200SelfSpeculativeGenerationStrategy(max_ctx=1000)
    s.engines.get = lambda model: _FakeEngine()
    return s


def _cfg(**over):
    kw = dict(max_steps=32, exit_layer=1, num_speculations=3, sample=False)
    kw.update(over)
    return GenerationConfig(**kw)


PROMPTS = [[5, 6, 7], [8, 9]]


@pytest.mark.parametrize("kw,exc,needle", [
    (dict(cfg=_cfg(sample=True)), NotImplementedError, "greedy"),
    (dict(logits_processors=[object()]), NotImplementedError, "logits processors"),
    (dict(cfg=_cfg(no_repeat_ngram_size=2)), NotImplementedError, "n-gram"),
    (dict(stopping_criteria=[object()]), NotImplementedError, "stopping criteria"),
    (dict(cfg=_cfg(stop_words=["x"])), NotImplementedError, "stopping criteria"),
    (dict(streamer=object()), NotImplementedError, "stream"),
    (dict(cfg=_cfg(draft_confidence_threshold=0.5)), NotImplementedError, "draft_confidence_threshold"),
    (dict(cfg=_cfg(num_speculations=16)), ValueError, "num_speculations"),
    (dict(prompts=[[1]] * 5, cfg=_cfg(num_speculations=3)), ValueError, "token rows"),        # 5 x 4 > 16
    (dict(prompts=[[1], []]), ValueError, "at least one token"),
    # 2 slots of 512: 400 + 100 + 3 + 1 = 504 fits, 410 + 100 + 3 + 1 = 514 does not
    (dict(prompts=[[1] * 410, [2]], cfg=_cfg(max_steps=100)), ValueError, "KV positions"),
])
def test_refusals_before_prefill(kw, exc, needle):
    s = _strategy()
    cfg = kw.pop("cfg", _cfg())
    prompts = kw.pop("prompts", PROMPTS)
    with pytest.raises(exc, match=needle):
        s.generate_batch(object(), prompts, [0], cfg, **kw)


def test_a_fitting_batch_reaches_the_engine():
    s = _strategy()
    with pytest.raises(AssertionError, match="begin ran"):
        s.generate_batch(object(), [[1] * 400, [2]], [0], _cfg(max_steps=100))
    with pytest.raises(AssertionError, match="begin ran"):
        s.generate_batch(object(), [[1]] * 4, [0], _cfg(num_speculations=3))     # 4 x 4 = 16 rows
    assert s.generate_batch(object(), [], [0], _cfg()) == []

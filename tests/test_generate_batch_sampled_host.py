"""CPU: the host side of sampled batched generation — the seeded prefill's C ABI symbol, the memory
plan of its seed buffer, and `generate_batch`'s seed checks, which refuse before the engine runs."""
import os
import re

import pytest

from layerskip_b200 import _lib
from layerskip_b200.memory import plan_memory
from layerskip_b200.weights import ARCHS
from tests.test_generate_batch_host import PROMPTS, _cfg, _strategy

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "lsk.h")
SEED_BYTES = 16 * 8              # engine.cu: batch_seeds, one uint64 per possible sequence


def test_seeded_prefill_is_declared_and_bound():
    header = open(HEADER).read()
    assert re.search(r"int lsk_prefill_batch_seeded\(lsk_engine\* e, const int32_t\* ids, const int32_t\* offsets,"
                     r"\s+int32_t n_seqs,\s+const uint64_t\* seeds, int32_t\* slot_positions_out\);", header)
    restype, args = _lib.SIGNATURES["lsk_prefill_batch_seeded"]
    assert restype is _lib.C.c_int and len(args) == 6
    assert args[4] is _lib.C.POINTER(_lib.C.c_uint64)
    assert hasattr(_lib.load(), "lsk_prefill_batch_seeded")


@pytest.mark.parametrize("name", ["tiny-mha", "tiny-gqa", "llama2-7b", "llama2-13b"])
def test_a_sampled_batch_adds_exactly_the_seeds(name):
    """sampling + batch_seqs > 0 adds the 16 seeds to what sampling and the batch each add alone;
    without sampling, or without a batch, the plan is what it was."""
    a = ARCHS[name]
    for max_ctx in (1000, 4096):
        base = plan_memory(a, max_ctx=max_ctx)
        samp = plan_memory(a, max_ctx=max_ctx, sampling=True)
        for n in (1, 3, 16):
            batch = plan_memory(a, max_ctx=max_ctx, batch_seqs=n)
            both = plan_memory(a, max_ctx=max_ctx, sampling=True, batch_seqs=n)
            for key in ("scratch", "total"):
                assert both[key] - samp[key] - (batch[key] - base[key]) == SEED_BYTES, (n, key)
            assert {k: v for k, v in both.items() if k not in ("scratch", "total")} == \
                {k: v for k, v in samp.items() if k not in ("scratch", "total")}


@pytest.mark.parametrize("seeds,needle", [
    ([1], "one seed"),                       # two prompts
    ([1, 2, 3], "one seed"),
    ([1, -1], "2\\*\\*64"),
    ([1, 2 ** 64], "2\\*\\*64"),
])
def test_bad_seeds_are_refused_before_begin(seeds, needle):
    with pytest.raises(ValueError, match=needle):
        _strategy().generate_batch(object(), PROMPTS, [0], _cfg(sample=True), seeds=seeds)


def test_sampling_without_seeds_is_refused_before_begin():
    with pytest.raises(NotImplementedError, match="greedy"):
        _strategy().generate_batch(object(), PROMPTS, [0], _cfg(sample=True))


def test_seeded_batches_reach_the_engine():
    s = _strategy()
    for seeds in ([0, 2 ** 64 - 1], [7, 7]):
        with pytest.raises(AssertionError, match="begin ran"):
            s.generate_batch(object(), PROMPTS, [0], _cfg(sample=True), seeds=seeds)
    with pytest.raises(AssertionError, match="begin ran"):          # greedy ignores the seeds
        s.generate_batch(object(), PROMPTS, [0], _cfg(), seeds=[1])

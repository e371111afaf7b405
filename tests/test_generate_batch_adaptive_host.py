"""CPU: the host side of confidence-threshold drafting in batches — the C ABI symbol, the memory plan
of its confidence scratch, and `Engine.round_batch_adaptive`'s argument checks and result unpacking
against a stand-in for the library."""
import contextlib
import ctypes as C
import os
import re

import pytest
import torch

from layerskip_b200 import _lib
from layerskip_b200.engine import Engine
from layerskip_b200.memory import plan_memory
from layerskip_b200.weights import ARCHS

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "lsk.h")
# sampling.cuh: ConfSeqsScratch, (max, sum) partials of 64 column slices for 16 sequences, 16 arrival
# counters, the decided counter, 16 d_stop values and the threshold
CONF_SEQS_BYTES = 2 * 16 * 64 * 4 + 16 * 4 + 4 + 16 * 4 + 4


def test_round_batch_adaptive_is_declared_and_bound():
    header = open(HEADER).read()
    assert re.search(r"int lsk_round_batch_adaptive\(lsk_engine\* e, int32_t d_max, const int32_t\* d_seq, "
                     r"const int32_t\* active,\s+float min_confidence, lsk_round_out\* outs, "
                     r"float\* draft_conf_out\);", header)
    restype, args = _lib.SIGNATURES["lsk_round_batch_adaptive"]
    assert restype is C.c_int and len(args) == 7
    assert args[4] is C.c_float and args[6] is C.POINTER(C.c_float)
    assert hasattr(_lib.load(), "lsk_round_batch_adaptive")


@pytest.mark.parametrize("name", ["tiny-mha", "tiny-gqa", "llama2-7b", "llama2-13b"])
def test_an_adaptive_batch_adds_exactly_the_confidence_scratch(name):
    """adaptive + batch_seqs > 0 adds the batched confidence scratch to what `adaptive` and the batch
    each add alone, for every batch size, with or without sampling; the other categories are
    those of `adaptive` alone."""
    a = ARCHS[name]
    for max_ctx in (1000, 4096):
        for sampling in (False, True):
            base = plan_memory(a, max_ctx=max_ctx, sampling=sampling)
            adaptive = plan_memory(a, max_ctx=max_ctx, sampling=sampling, adaptive=True)
            for n in range(1, 17):
                batch = plan_memory(a, max_ctx=max_ctx, sampling=sampling, batch_seqs=n)
                both = plan_memory(a, max_ctx=max_ctx, sampling=sampling, adaptive=True, batch_seqs=n)
                for key in ("scratch", "total"):
                    assert both[key] - adaptive[key] - (batch[key] - base[key]) == CONF_SEQS_BYTES, \
                        (n, sampling, key)
                assert {k: v for k, v in both.items() if k not in ("scratch", "total")} == \
                    {k: v for k, v in adaptive.items() if k not in ("scratch", "total")}


class _FakeLib:
    """lsk_round_batch_adaptive for a batch of n: sequence s drafts s + 1 tokens 10 s + i with
    confidences (s + 1) / 100 + i / 1000 (stored at [s][LSK_MAX_SPEC])."""

    def __init__(self):
        self.calls = []

    def lsk_round_batch_adaptive(self, h, d_max, ds, act, t, outs, conf):
        n = 3
        self.calls.append((d_max, None if ds is None else list(ds[:n]), None if act is None else list(act[:n]), t))
        for s in range(n):
            o = outs[s]
            o.n_drafted = o.n_matches = s + 1
            o.n_emitted = s + 2
            for i in range(s + 1):
                o.draft_ids[i] = o.emitted_ids[i] = o.verified_ids[i] = 10 * s + i
                conf[s * _lib.LSK_MAX_SPEC + i] = (s + 1) / 100 + i / 1000
            o.emitted_ids[s + 1] = o.verified_ids[s + 1] = 99
            o.kv_len = 50 + s
        return 0


def _fake_engine():
    eng = Engine.__new__(Engine)
    eng._lib, eng._h, eng.device, eng._batch_n = _FakeLib(), None, None, 3
    return eng


def test_outputs_carry_each_sequences_confidences(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())   # no device here
    eng = _fake_engine()
    outs = eng.round_batch_adaptive(4, 0.25, d_seq=[4, 2, 3], active=[1, 0, True])
    assert eng._lib.calls == [(4, [4, 2, 3], [1, 0, 1], 0.25)]
    for s, o in enumerate(outs):
        assert (o.n_drafted, o.draft, o.emitted, o.kv_len) == \
            (s + 1, [10 * s + i for i in range(s + 1)], [10 * s + i for i in range(s + 1)] + [99], 50 + s)
        assert o.draft_confidence == pytest.approx([(s + 1) / 100 + i / 1000 for i in range(s + 1)], abs=1e-7)
    eng.round_batch_adaptive(2, 1.0)
    assert eng._lib.calls[-1] == (2, None, None, 1.0)


@pytest.mark.parametrize("kw", [dict(d_seq=[1, 2]), dict(d_seq=[1, 2, 3, 4]), dict(active=[True]),
                                dict(active=[1, 1, 1, 1])])
def test_length_mismatches_are_refused_before_the_library(kw):
    eng = _fake_engine()
    with pytest.raises(ValueError, match="entries for a batch of 3"):
        eng.round_batch_adaptive(3, 0.5, **kw)
    assert eng._lib.calls == []

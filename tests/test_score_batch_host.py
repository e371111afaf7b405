"""CPU: the host side of batched scoring — `Engine.loglikelihood_batch` against a stand-in for
`Engine.score_batch` (truncation, slicing, float64 sums, the greedy flag, validation, order and the
fallback to `loglikelihood`), and the memory plan of the batch buffers."""
import pytest
import torch

from layerskip_b200.engine import Engine
from layerskip_b200.memory import plan_memory
from layerskip_b200.weights import ARCHS, LlamaArch


def _lp(ids):
    """logprob[i] = -(i + 1) / 8 * ids[i+1]: every entry distinct and exact in float32."""
    return torch.tensor([-(i + 1) / 8 * ids[i + 1] for i in range(len(ids) - 1)], dtype=torch.float32)


def _fake_engine(max_ctx, prefill_tc=True, greedy_fn=None, hidden=256):
    eng = Engine.__new__(Engine)
    eng.max_ctx = max_ctx
    eng.prefill_tc = prefill_tc
    eng.arch = LlamaArch(512, hidden, 688, 2, 8, 8, 32)
    eng.batch_calls, eng.calls = [], []
    g = greedy_fn or (lambda s, i: s[i + 1])

    def score(ids, exit_layer=-1):
        eng.calls.append((list(ids), exit_layer))
        assert 2 <= len(ids) <= max_ctx
        return _lp(ids), torch.tensor([g(ids, i) for i in range(len(ids) - 1)], dtype=torch.int64)

    def score_batch(seqs, exit_layer=-1):
        eng.batch_calls.append(([list(s) for s in seqs], exit_layer))
        return [(_lp(s), torch.tensor([g(s, i) for i in range(len(s) - 1)], dtype=torch.int64)) for s in seqs]

    eng.score, eng.score_batch = score, score_batch
    return eng


def test_loglikelihood_batch_equals_loglikelihood_in_order_with_one_call():
    reqs = [([5, 6, 7], [8, 9]), ([1], [2]), ([3, 4, 5, 6, 7, 8], [9, 10, 11]), ([2, 2], [2, 2, 2])]
    eng = _fake_engine(64)
    got = eng.loglikelihood_batch(reqs, exit_layer=3)
    assert len(eng.batch_calls) == 1 and not eng.calls
    assert eng.batch_calls[0] == ([c + k for c, k in reqs], 3)
    ref = _fake_engine(64)
    want = [ref.loglikelihood(c, k, exit_layer=3) for c, k in reqs]
    assert got == want
    for (ctx, cont), (ll, greedy) in zip(reqs, got):
        ids = ctx + cont
        rows = range(len(ctx) - 1, len(ids) - 1)                  # the rows predicting the continuation
        assert ll == pytest.approx(sum(-(i + 1) / 8 * ids[i + 1] for i in rows), abs=0)
        assert greedy is True


def test_loglikelihood_batch_truncates_from_the_left():
    eng = _fake_engine(4)
    got = eng.loglikelihood_batch([([1, 2, 3, 4, 5], [6, 7]), ([1], [2, 3, 4])])
    assert eng.batch_calls[0][0] == [[4, 5, 6, 7], [1, 2, 3, 4]]
    assert got[0][0] == pytest.approx(-(2 / 8) * 6 - (3 / 8) * 7, abs=0)


def test_loglikelihood_batch_validates_every_request_before_scoring():
    eng = _fake_engine(4)
    for bad in ([([1], [2]), ([1], [2, 3, 4, 5])], [([1], [2]), ([], [2])], [([1], [2]), ([1], [])]):
        with pytest.raises(ValueError):
            eng.loglikelihood_batch(bad)
    assert not eng.batch_calls and not eng.calls
    assert eng.loglikelihood_batch([]) == []


def test_loglikelihood_batch_greedy_flag_looks_at_each_continuation_only():
    # greedy disagrees at row 0 of every sequence: inside the context of the first request, inside
    # the continuation of the second (its context is one token)
    eng = _fake_engine(64, greedy_fn=lambda s, i: 0 if i == 0 else s[i + 1])
    got = eng.loglikelihood_batch([([5, 6, 7], [8, 9]), ([5], [6, 7])])
    assert [g for _, g in got] == [True, False]


def test_loglikelihood_batch_sums_in_float64():
    eng = _fake_engine(8192)
    eng.score_batch = lambda seqs, e=-1: [(torch.full((len(s) - 1,), -0.1, dtype=torch.float32),
                                           torch.tensor(s[1:], dtype=torch.int64)) for s in seqs]
    got = eng.loglikelihood_batch([([1], [2] * 4000), ([1], [2] * 3)])
    f = float(torch.tensor(-0.1, dtype=torch.float32))
    assert got[0][0] == pytest.approx(4000 * f, rel=1e-12)
    assert got[1][0] == pytest.approx(3 * f, rel=1e-12)


@pytest.mark.parametrize("prefill_tc,hidden", [(False, 256), (True, 96)])
def test_loglikelihood_batch_falls_back_without_the_prompt_pass(prefill_tc, hidden):
    reqs = [([5, 6, 7], [8, 9]), ([1], [2])]
    eng = _fake_engine(64, prefill_tc=prefill_tc, hidden=hidden)
    got = eng.loglikelihood_batch(reqs, exit_layer=2)
    assert not eng.batch_calls
    assert eng.calls == [([5, 6, 7, 8, 9], 2), ([1, 2], 2)]
    assert got == [_fake_engine(64).loglikelihood(c, k, 2) for c, k in reqs]


@pytest.mark.parametrize("name", ["llama2-7b", "llama3-8b", "tiny-gqa"])
def test_plan_memory_batch_scoring_adds_exactly_the_packed_scoring_buffers(name):
    """The buffers the first lsk_score_batch or lsk_score_prefixed call allocates: the group upload,
    the view table and the piece arrival counters, on top of lsk_score's."""
    arch = ARCHS[name]
    max_ctx = 2048
    kvh = arch.kv_heads
    vpad = (arch.vocab + 15) // 16 * 16
    for keep in (False, True):
        base = plan_memory(arch, max_ctx=max_ctx, keep_logits=keep)
        assert plan_memory(arch, max_ctx=max_ctx, keep_logits=keep, batch_scoring=False) == base
        sc = plan_memory(arch, max_ctx=max_ctx, keep_logits=keep, scoring=True)
        batch_only = 9 * max_ctx * 4 + 128 * kvh * 4          # group arrays, view table, arrival counters
        for scoring in (False, True):
            b = plan_memory(arch, max_ctx=max_ctx, keep_logits=keep, scoring=scoring, batch_scoring=True)
            assert b["scratch"] - sc["scratch"] == batch_only
            assert b["total"] - base["total"] == batch_only + 2 * max_ctx * 4 + (0 if keep else 16 * vpad * 4)
            assert {k: v for k, v in b.items() if k not in ("scratch", "total")} == \
                {k: v for k, v in base.items() if k not in ("scratch", "total")}
    # without the prompt pass the call is refused before it allocates anything
    assert plan_memory(arch, max_ctx=max_ctx, prefill_tc=False, batch_scoring=True) == \
        plan_memory(arch, max_ctx=max_ctx, prefill_tc=False)

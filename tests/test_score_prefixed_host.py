"""CPU: the host side of prefix-shared scoring — how `Engine.loglikelihood_batch` groups requests by
their cut context, what it passes to `score_prefixed`, how it maps results back, when it routes to
`score_prefixed` rather than `score_batch`, and validation before scoring.  (The memory plan of
its buffers is `batch_scoring`'s, checked in test_score_batch_host.py.)"""
import pytest
import torch

from layerskip_b200.engine import Engine
from layerskip_b200.weights import LlamaArch


def _lp(ids):
    """logprob[i] = -(i + 1) / 8 * ids[i+1]: every entry distinct and exact in float32."""
    return torch.tensor([-(i + 1) / 8 * ids[i + 1] for i in range(len(ids) - 1)], dtype=torch.float32)


def _fake_engine(max_ctx, greedy_fn=None):
    """score_batch / score_prefixed stand-ins that agree entry for entry, as the engine's do."""
    eng = Engine.__new__(Engine)
    eng.max_ctx = max_ctx
    eng.prefill_tc = True
    eng.arch = LlamaArch(512, 256, 688, 2, 8, 8, 32)
    eng.batch_calls, eng.prefixed_calls, eng.calls = [], [], []
    g = greedy_fn or (lambda s, i: s[i + 1])

    def score(ids, exit_layer=-1):
        eng.calls.append((list(ids), exit_layer))
        return _lp(ids), torch.tensor([g(ids, i) for i in range(len(ids) - 1)], dtype=torch.int64)

    def score_batch(seqs, exit_layer=-1):
        eng.batch_calls.append(([list(s) for s in seqs], exit_layer))
        return [(_lp(s), torch.tensor([g(s, i) for i in range(len(s) - 1)], dtype=torch.int64)) for s in seqs]

    def score_prefixed(prefixes, branches, exit_layer=-1):
        eng.prefixed_calls.append(([list(p) for p in prefixes], [(i, list(b)) for i, b in branches], exit_layer))
        out = []
        for i, b in branches:
            s = list(prefixes[i]) + list(b)
            rows = range(len(prefixes[i]) - 1, len(s) - 1)
            out.append((_lp(s)[len(prefixes[i]) - 1:],
                        torch.tensor([g(s, r) for r in rows], dtype=torch.int64)))
        return out

    eng.score, eng.score_batch, eng.score_prefixed = score, score_batch, score_prefixed
    return eng


def _mc(ctx_len, n_choices, choice_len, base):
    ctx = [(base + 3 * i) % 500 + 1 for i in range(ctx_len)]
    return [(ctx, [(base + 7 * j + 11 * i) % 500 + 1 for i in range(choice_len)]) for j in range(n_choices)]


def test_shared_contexts_go_to_score_prefixed_and_match_score_batch():
    # two 4-choice questions with 200-id contexts, and one lone request
    reqs = _mc(200, 4, 3, 5) + [([9, 8, 7], [6, 5])] + _mc(200, 4, 2, 77)
    eng = _fake_engine(1024)
    got = eng.loglikelihood_batch(reqs, exit_layer=2)
    assert not eng.batch_calls and not eng.calls and len(eng.prefixed_calls) == 1
    prefixes, branches, e = eng.prefixed_calls[0]
    assert e == 2
    assert prefixes == [reqs[0][0], [9], reqs[5][0]]
    assert branches == [(0, c) for _, c in reqs[:4]] + [(1, [8, 7, 6, 5])] + [(2, c) for _, c in reqs[5:]]
    ref = _fake_engine(1024)
    assert got == [ref.loglikelihood(c, k, exit_layer=2) for c, k in reqs]
    for (ctx, cont), (ll, greedy) in zip(reqs, got):
        ids = ctx + cont
        assert ll == pytest.approx(sum(-(i + 1) / 8 * ids[i + 1] for i in range(len(ctx) - 1, len(ids) - 1)), abs=0)
        assert greedy is True


def test_distinct_contexts_go_to_score_batch():
    reqs = [([5, 6, 7], [8, 9]), ([1], [2]), ([3, 4, 5, 6, 7, 8], [9, 10, 11]), ([2, 2], [2, 2, 2])]
    eng = _fake_engine(64)
    eng.loglikelihood_batch(reqs)
    assert not eng.prefixed_calls and len(eng.batch_calls) == 1
    assert eng.batch_calls[0][0] == [c + k for c, k in reqs]


@pytest.mark.parametrize("ctx_len,choices,choice_len,prefixed", [
    (200, 2, 1, True),     # 400 rows as sequences: 4 chunks; shared 199 + 2 rows: 2 + 1
    (30, 8, 4, True),      # 264 rows: 3 chunks; shared 29 + 32 rows: 1 + 1
    (60, 2, 8, False),     # 134 rows: 2 chunks; shared 59 + 16 rows: 1 + 1
    (70, 2, 1, False),     # 140 rows: 2 chunks; shared 69 + 2 rows: 1 + 1
])
def test_routing_rule_counts_chunks(ctx_len, choices, choice_len, prefixed):
    reqs = _mc(ctx_len, choices, choice_len, 3)
    seq_chunks = (sum(len(c) + len(k) - 1 for c, k in reqs) + 127) // 128
    shared_chunks = (ctx_len - 1 + 127) // 128 + (choices * choice_len + 127) // 128
    assert (shared_chunks < seq_chunks) == prefixed
    eng = _fake_engine(1024)
    got = eng.loglikelihood_batch(reqs)
    assert len(eng.prefixed_calls) == int(prefixed) and len(eng.batch_calls) == int(not prefixed)
    assert got == [_fake_engine(1024).loglikelihood(c, k) for c, k in reqs]


def test_left_cut_can_split_a_shared_context():
    # three requests with the same context; the long continuation's cut drops context ids, so its cut
    # context differs and it becomes a branch of its own first id
    ctx = list(range(1, 101))
    reqs = [(ctx, [200]), (ctx, [201]), (ctx, [202]), (ctx, list(range(300, 330)))]
    eng = _fake_engine(120)
    # 419 rows as sequences (4 chunks) against 99 prefix rows and 122 branch rows (1 + 1)
    got = eng.loglikelihood_batch(reqs)
    assert len(eng.prefixed_calls) == 1
    prefixes, branches, _ = eng.prefixed_calls[0]
    cut = (ctx + list(range(300, 330)))[-120:]
    assert prefixes == [ctx, cut[:1]]
    assert branches == [(0, [200]), (0, [201]), (0, [202]), (1, cut[1:])]
    ref = _fake_engine(120)
    assert got == [ref.loglikelihood(c, k) for c, k in reqs]


def test_results_map_back_with_float64_sums_and_greedy_flags():
    # greedy disagrees wherever the predicted id is 202: inside the third request's continuation only
    reqs = _mc(300, 4, 5, 1)
    reqs[2] = (reqs[2][0], [202, 3, 4, 5, 6])
    g = lambda s, i: 0 if s[i + 1] == 202 else s[i + 1]   # noqa: E731
    eng = _fake_engine(1024, greedy_fn=g)
    got = eng.loglikelihood_batch(reqs)
    assert len(eng.prefixed_calls) == 1
    assert [f for _, f in got] == [True, True, False, True]
    eng2 = _fake_engine(8192)
    eng2.score_prefixed = lambda p, b, e=-1: [(torch.full((len(x),), -0.1, dtype=torch.float32),
                                              torch.tensor(x, dtype=torch.int64)) for _, x in b]
    got = eng2.loglikelihood_batch([([1] * 300, [2] * 4000), ([1] * 300, [2] * 3)])
    f = float(torch.tensor(-0.1, dtype=torch.float32))
    assert got[0][0] == pytest.approx(4000 * f, rel=1e-12)
    assert got[1][0] == pytest.approx(3 * f, rel=1e-12)


def test_validation_comes_before_any_scoring():
    eng = _fake_engine(4)
    ctx = [1, 2]
    for bad in ([(ctx, [3]), (ctx, [3]), (ctx, [2, 3, 4, 5])], [(ctx, [3]), (ctx, [4]), ([], [2])],
                [(ctx, [3]), (ctx, [4]), (ctx, [])]):
        with pytest.raises(ValueError):
            eng.loglikelihood_batch(bad)
    assert not eng.batch_calls and not eng.prefixed_calls and not eng.calls


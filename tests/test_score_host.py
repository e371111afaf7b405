"""CPU: the host side of scoring — `Engine.loglikelihood` slicing, left truncation and the greedy
flag against a stand-in for `Engine.score`, the memory plan of the scoring buffers, and the
`score` command line's flags."""
import sys

import pytest
import torch

from layerskip_b200 import cli
from layerskip_b200.engine import Engine
from layerskip_b200.memory import plan_memory
from layerskip_b200.weights import ARCHS


def _fake_engine(max_ctx, greedy_fn=None):
    """An Engine whose score() returns logprob[i] = -(i + 1) / 8 * ids[i+1] (every entry distinct,
    exact in float32) and greedy[i] = greedy_fn(ids, i) (default: the true next id)."""
    eng = Engine.__new__(Engine)
    eng.max_ctx = max_ctx
    eng.calls = []

    def score(ids, exit_layer=-1):
        eng.calls.append((list(ids), exit_layer))
        n = len(ids)
        assert 2 <= n <= max_ctx
        lp = torch.tensor([-(i + 1) / 8 * ids[i + 1] for i in range(n - 1)], dtype=torch.float32)
        g = greedy_fn or (lambda s, i: s[i + 1])
        return lp, torch.tensor([g(ids, i) for i in range(n - 1)], dtype=torch.int64)

    eng.score = score
    return eng


def test_loglikelihood_sums_the_continuation_entries():
    eng = _fake_engine(64)
    ctx, cont = [5, 6, 7], [8, 9]
    ll, greedy = eng.loglikelihood(ctx, cont, exit_layer=3)
    ids = ctx + cont
    want = sum(-(i + 1) / 8 * ids[i + 1] for i in (2, 3))         # rows predicting 8 and 9
    assert ll == pytest.approx(want, abs=0) and greedy is True
    assert eng.calls == [(ids, 3)]


def test_loglikelihood_truncates_from_the_left():
    eng = _fake_engine(4)
    ll, _ = eng.loglikelihood([1, 2, 3, 4, 5], [6, 7])
    assert eng.calls[-1][0] == [4, 5, 6, 7]                      # the last max_ctx tokens
    assert ll == pytest.approx(-(2 / 8) * 6 - (3 / 8) * 7, abs=0)
    eng.loglikelihood([1], [2, 3, 4])                             # continuation of max_ctx - 1 fits
    assert eng.calls[-1][0] == [1, 2, 3, 4]
    with pytest.raises(ValueError):
        eng.loglikelihood([1], [2, 3, 4, 5])                      # nothing left to condition on
    with pytest.raises(ValueError):
        eng.loglikelihood([], [2])
    with pytest.raises(ValueError):
        eng.loglikelihood([1], [])


def test_loglikelihood_greedy_flag_looks_at_the_continuation_only():
    # greedy disagrees inside the context only: still greedy
    eng = _fake_engine(64, lambda s, i: 0 if i == 0 else s[i + 1])
    assert eng.loglikelihood([5, 6, 7], [8, 9])[1] is True
    # one continuation position disagrees: not greedy
    eng = _fake_engine(64, lambda s, i: 0 if i == len(s) - 2 else s[i + 1])
    assert eng.loglikelihood([5, 6, 7], [8, 9])[1] is False
    eng = _fake_engine(64, lambda s, i: 0 if i == len(s) - 3 else s[i + 1])
    assert eng.loglikelihood([5, 6, 7], [8, 9])[1] is False


def test_loglikelihood_sums_in_float64():
    eng = Engine.__new__(Engine)
    eng.max_ctx = 8192
    eng.score = lambda ids, e=-1: (torch.full((len(ids) - 1,), -0.1, dtype=torch.float32),
                                   torch.tensor(ids[1:], dtype=torch.int64))
    ll, _ = eng.loglikelihood([1], [2] * 4000)
    assert ll == pytest.approx(4000 * float(torch.tensor(-0.1, dtype=torch.float32)), rel=1e-12)


@pytest.mark.parametrize("name", ["llama2-7b", "llama3-8b", "tiny-gqa"])
def test_plan_memory_scoring_adds_exactly_the_scoring_buffers(name):
    arch = ARCHS[name]
    for keep in (False, True):
        base = plan_memory(arch, max_ctx=2048, keep_logits=keep)
        assert plan_memory(arch, max_ctx=2048, keep_logits=keep, scoring=False) == base
        sc = plan_memory(arch, max_ctx=2048, keep_logits=keep, scoring=True)
        vpad = (arch.vocab + 15) // 16 * 16
        extra = 2 * 2048 * 4 + (0 if keep else 16 * vpad * 4)
        assert sc["scratch"] - base["scratch"] == extra
        assert sc["total"] - base["total"] == extra
        assert {k: v for k, v in sc.items() if k not in ("scratch", "total")} == \
            {k: v for k, v in base.items() if k not in ("scratch", "total")}


def test_score_flags_parse(monkeypatch):
    monkeypatch.setattr(sys, "argv", ["score.py", "--model", "synthetic:llama2-7b", "--num_samples", "3",
                                      "--prompt_len", "256", "--exit_layers", "4,8,-1",
                                      "--continuation_len", "32", "--output_dir", "./out",
                                      "--model_args", "alpha=0.1,seed=2"])
    args, bargs, sargs = cli.parse(cli.Arguments, cli.BenchmarkArguments, cli.ScoreArguments)
    assert (bargs.num_samples, bargs.prompt_len, sargs.continuation_len) == (3, 256, 32)
    assert cli.parse_exit_layers(sargs.exit_layers) == [4, 8, -1]
    assert cli.parse_model_args(args.model_args) == {"alpha": 0.1, "seed": 2}
    assert args.output_dir == "./out"
    monkeypatch.setattr(sys, "argv", ["score.py"])
    _a, _b, sargs = cli.parse(cli.Arguments, cli.BenchmarkArguments, cli.ScoreArguments)
    assert cli.parse_exit_layers(sargs.exit_layers) == [4, 8, 16, -1]

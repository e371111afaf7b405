"""CPU: the host side of multi-exit scoring and the acceptance prediction — `predict.greedy_rounds`
against a direct port of the reference's greedy self-speculation loop, the sampled estimate, the
memory plan of the `lsk_score_exits` buffers, and the `predict` command line."""
import hashlib
import sys

import pytest
import torch

from layerskip_b200 import cli, predict
from layerskip_b200.memory import plan_memory
from layerskip_b200.plugin import GenerationConfig
from layerskip_b200.weights import ARCHS

VOCAB = 50


def _h(prefix, salt):
    return int(hashlib.md5((salt + ",".join(map(str, prefix[-4:]))).encode()).hexdigest(), 16)


def _verify_fn(prefix):
    return _h(prefix, "v") % VOCAB


def _draft_fn(kind):
    def f(prefix):
        v = _verify_fn(prefix)
        if kind == "all":
            return v
        if kind == "never":
            return (v + 1) % VOCAB
        return v if _h(prefix, "d" + kind) % 100 < int(kind) else (v + 7) % VOCAB
    return f


def _reference_greedy(prompt, draft_fn, verify_fn, D, max_steps):
    """self_speculation_generator.py:51-99 and 186-205, greedy, with the draft and verify models
    replaced by deterministic functions of the prefix; returns (rounds, output, acceptance)."""
    out, rounds, matches, generations = [], [], 0, 0
    while len(out) < max_steps:
        d = min(D, max_steps - len(out) - 1)
        prefix = prompt + out
        drafts = []
        for _ in range(d):
            drafts.append(draft_fn(prefix + drafts))
        verified = [verify_fn(prefix + drafts[:i]) for i in range(d + 1)]
        n = 0
        while n < d and drafts[n] == verified[n]:
            n += 1
        out += drafts[:n] + [verified[n]]
        rounds.append((d, n))
        matches += n
        generations += d
    return rounds, out, (matches / generations if generations else None)


@pytest.mark.parametrize("kind", ["all", "never", "30", "70", "90"])
def test_greedy_rounds_equal_the_reference_loop(kind):
    draft_fn = _draft_fn(kind)
    for prompt in ([3, 4, 5], [11, 2, 9, 40, 1]):
        steps_max = 60
        cont = []
        for _ in range(steps_max):                                 # full-depth greedy continuation
            cont.append(_verify_fn(prompt + cont))
        agree = [draft_fn(prompt + cont[:q]) == cont[q] for q in range(steps_max)]
        for max_steps in (1, 2, 3, 7, 16, 17, 31, 60):
            for D in range(1, 16):
                want_rounds, out, want_acc = _reference_greedy(prompt, draft_fn, _verify_fn, D, max_steps)
                assert out == cont[:max_steps]
                got = predict.greedy_rounds(agree[:max_steps], D, max_steps)
                assert got == want_rounds, (kind, max_steps, D)
                assert predict.acceptance_rate(got) == want_acc
                assert predict.tokens_per_round(got) == max_steps / len(got)


def test_greedy_rounds_clamp_and_tail():
    # max_steps 5, D 3, all agree: 3 drafts -> 4 tokens, then a tail round drafting 0
    assert predict.greedy_rounds([True] * 5, 3, 5) == [(3, 3), (0, 0)]
    assert predict.greedy_rounds([False] * 5, 3, 5) == [(3, 0), (3, 0), (2, 0), (1, 0), (0, 0)]
    assert predict.acceptance_rate([(0, 0)]) is None
    with pytest.raises(ValueError):
        predict.greedy_rounds([True] * 3, 2, 8)


def test_sampled_estimate():
    for d in (1, 3, 6, 15):
        assert predict.sampled_estimate(0.0, d) == (0.0, 1.0)
        assert predict.sampled_estimate(1.0, d) == (1.0, d + 1.0)
        a = 0.7
        acc, tpr = predict.sampled_estimate(a, d)
        want_n = sum(a ** i for i in range(1, d + 1))              # expected leading acceptances
        assert tpr == pytest.approx(1 + want_n, rel=1e-12)
        assert acc == pytest.approx(want_n / d, rel=1e-12)
    assert predict.mean([None, 1.0, 2.0]) == 1.5 and predict.mean([None]) is None


@pytest.mark.parametrize("name", ["llama2-7b", "llama3-8b", "tiny-gqa"])
def test_plan_memory_score_exits_adds_exactly_the_buffers_it_allocates(name):
    arch = ARCHS[name]
    vpad = (arch.vocab + 15) // 16 * 16
    for prefill_tc in (True, False):
        for keep in (False, True):
            base = plan_memory(arch, max_ctx=2048, keep_logits=keep, prefill_tc=prefill_tc)
            assert plan_memory(arch, max_ctx=2048, keep_logits=keep, prefill_tc=prefill_tc, score_exits=0,
                               score_exits_sampled=True) == base
            for k in (1, 5, 32):
                plain = plan_memory(arch, max_ctx=2048, keep_logits=keep, prefill_tc=prefill_tc, score_exits=k)
                extra = 2 * k * 2048 * 4 + (0 if keep else 16 * vpad * 4)
                assert plain["scratch"] - base["scratch"] == extra
                # lsk_score's result arrays are row 0 of these: scoring as well costs nothing more
                assert plan_memory(arch, max_ctx=2048, keep_logits=keep, prefill_tc=prefill_tc, score_exits=k,
                                   scoring=True) == plain
                assert plain["total"] - base["total"] == extra
                assert {x: v for x, v in plain.items() if x not in ("scratch", "total")} == \
                    {x: v for x, v in base.items() if x not in ("scratch", "total")}
                smp = plan_memory(arch, max_ctx=2048, keep_logits=keep, prefill_tc=prefill_tc, score_exits=k,
                                  score_exits_sampled=True)
                rows = 128 if (prefill_tc and arch.hidden % 64 == 0) else 16
                # one exit has no draft exit: lsk_score_exits allocates no acceptance buffers
                assert smp["total"] - plain["total"] == \
                    ((k - 1) * (2048 + rows * arch.vocab) * 4 + 16 * arch.vocab * 4 if k > 1 else 0)


class _FakeEngine:
    """begin / prefill / ar_step / score_exits with a deterministic full model (_verify_fn) and
    draft exits that agree with it at a per-exit rate; accept rows are a function of the position."""

    def __init__(self):
        self.calls = []

    def begin(self, exit_layer, max_steps, eos, **kw):
        assert exit_layer == -1 and eos == []
        self.kw = kw

    def prefill(self, ids):
        self.text = list(ids)

    def ar_step(self):
        t = _verify_fn(self.text)
        self.text.append(t)
        return t

    def score_exits(self, ids, exits, sampling=None):
        self.calls.append((list(ids), list(exits), sampling))
        n = len(ids)
        greedy = torch.tensor([[_draft_fn(str(10 * e))(ids[:i + 1]) for i in range(n - 1)] for e in exits])
        acc = None
        if sampling is not None:
            acc = torch.tensor([[(e * 7 + i) % 10 / 10 for i in range(n - 1)] for e in exits[:-1]])
        return torch.zeros(len(exits), n - 1), greedy, acc


def test_predict_grid_greedy_uses_one_pass_per_prompt():
    eng = _FakeEngine()
    prompts = [[3, 4, 5, 6], [7, 8]]
    cfg = GenerationConfig(max_steps=24, sample=False)
    rows = cli.predict_grid(eng, prompts, [2, 4], [1, 3, 6], cfg, n_layers=8)
    assert len(eng.calls) == 2 and all(c[1] == [2, 4, 8] and c[2] is None for c in eng.calls)
    assert [(r["exit_layer"], r["num_speculations"]) for r in rows] == [(2, 1), (2, 3), (2, 6), (4, 1), (4, 3), (4, 6)]
    for r in rows:
        accs, tprs = [], []
        for p in prompts:
            cont = []
            for _ in range(24):
                cont.append(_verify_fn(p + cont))
            draft_fn = _draft_fn(str(10 * r["exit_layer"]))
            want_rounds, _, acc = _reference_greedy(p, draft_fn, _verify_fn, r["num_speculations"], 24)
            accs.append(acc)
            tprs.append(24 / len(want_rounds))
        assert r["exact"] is True
        assert r["acceptance_rate"] == pytest.approx(sum(accs) / 2, abs=1e-15)
        assert r["tokens_per_round"] == pytest.approx(sum(tprs) / 2, abs=1e-15)


def test_predict_grid_sampled_uses_the_mean_acceptance_probability():
    eng = _FakeEngine()
    cfg = GenerationConfig(max_steps=10, sample=True, temperature=0.7, top_k=5, top_p=0.8)
    rows = cli.predict_grid(eng, [[3, 4, 5]], [8], [2, 4], cfg, n_layers=8)
    assert eng.calls[0][1] == [8] and eng.calls[0][2] == {"temperature": 0.7, "top_k": 5, "top_p": 0.8}
    assert eng.kw["sample"] is True and eng.kw["temperature"] == 0.7
    # an exit at full depth drafts from the verifier's distribution: every draft is accepted
    assert [(r["mean_alpha"], r["tokens_per_round"]) for r in rows] == [(1.0, 3.0), (1.0, 5.0)]


def test_predict_grid_sampled_alpha():
    eng = _FakeEngine()
    cfg = GenerationConfig(max_steps=10, sample=True)
    rows = cli.predict_grid(eng, [[3, 4, 5]], [2], [3], cfg, n_layers=8)
    # rows 2 .. 11 of exit 2: (14 + i) % 10 / 10
    alpha = sum((14 + i) % 10 / 10 for i in range(2, 12)) / 10
    assert rows[0]["mean_alpha"] == pytest.approx(alpha, rel=1e-7)     # float32 entries
    assert rows[0]["exact"] is False
    assert (rows[0]["acceptance_rate"], rows[0]["tokens_per_round"]) == predict.sampled_estimate(rows[0]["mean_alpha"], 3)


def test_predict_flags_parse(monkeypatch):
    monkeypatch.setattr(sys, "argv", ["predict.py", "--model", "synthetic:llama2-7b", "--num_samples", "3",
                                      "--exit_layer_first", "4", "--exit_layer_last", "16", "--exit_layer_step", "4",
                                      "--num_speculations_first", "2", "--num_speculations_last", "6",
                                      "--num_speculations_step", "2", "--max_steps", "128", "--sample", "false",
                                      "--model_args", "alpha=0.1"])
    args, bargs, sargs, gcfg = cli.parse(cli.Arguments, cli.BenchmarkArguments, cli.SweepArguments, GenerationConfig)
    assert (sargs.exit_layer_first, sargs.exit_layer_last, sargs.exit_layer_step) == (4, 16, 4)
    assert (sargs.num_speculations_first, sargs.num_speculations_last, sargs.num_speculations_step) == (2, 6, 2)
    assert gcfg.max_steps == 128 and gcfg.sample is False and bargs.num_samples == 3
    assert cli.parse_model_args(args.model_args) == {"alpha": 0.1}


def test_predict_refuses_the_ngram_ban(monkeypatch):
    with pytest.raises(NotImplementedError, match="n-gram"):
        cli.main_predict(["--no_repeat_ngram_size", "3"])

"""CPU: the host side of confidence-threshold drafting.  A scripted engine stands in for the GPU:
the strategy calls `round` exactly as before when the threshold is absent or 0 and `round_adaptive`
otherwise, counts the drafts a round actually made, and still takes the reference's own
GenerationConfig (which has no threshold field); the flag parses on the command lines."""
import sys
from dataclasses import dataclass, field
from typing import List, Optional

import pytest

from layerskip_b200 import cli
from layerskip_b200.engine import RoundOutput
from layerskip_b200.plugin import GenerationConfig
from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy


class ScriptedEngine:
    """Every round emits one matched draft and one bonus token; an adaptive round drafts
    min(d_max, 2) tokens, a fixed one d_req."""

    def __init__(self):
        self.calls = []

    def begin(self, **kw):
        pass

    def prefill(self, ids):
        pass

    def _out(self, n):
        m = min(n, 1)
        return RoundOutput(n_drafted=n, n_matches=m, emitted=[7] * (m + 1), draft=[7] * n,
                           verified=[7] * (n + 1), kv_len=0)

    def round(self, d_req):
        self.calls.append(("round", d_req))
        return self._out(d_req)

    def round_adaptive(self, d_max, min_confidence):
        self.calls.append(("adaptive", d_max, min_confidence))
        r = self._out(min(d_max, 2))
        r.draft_confidence = [0.5] * r.n_drafted
        return r


def _run(cfg):
    eng = ScriptedEngine()
    s = B200SelfSpeculativeGenerationStrategy.__new__(B200SelfSpeculativeGenerationStrategy)
    s.engines = type("Cache", (), {"get": lambda self, model: eng})()
    s.last_rounds = []
    res = s.generate_token_ids(object(), [1, 2, 3], [99], cfg)
    return eng, res


def test_zero_or_absent_threshold_keeps_fixed_rounds():
    for cfg in (GenerationConfig(max_steps=9, exit_layer=2, num_speculations=4, sample=False),
                GenerationConfig(max_steps=9, exit_layer=2, num_speculations=4, sample=False,
                                 draft_confidence_threshold=0.0)):
        eng, res = _run(cfg)
        # two tokens a round; the max_steps clamp shortens the last two rounds
        assert eng.calls == [("round", 4)] * 3 + [("round", 2), ("round", 0)]
        assert res.predicted_tokens == [7] * 9
        assert res.acceptance_rate == pytest.approx(4 / 14)


def test_positive_threshold_calls_round_adaptive_and_counts_actual_drafts():
    cfg = GenerationConfig(max_steps=9, exit_layer=2, num_speculations=4, sample=False,
                           draft_confidence_threshold=0.3)
    eng, res = _run(cfg)
    assert eng.calls == [("adaptive", 4, 0.3)] * 3 + [("adaptive", 2, 0.3), ("adaptive", 0, 0.3)]
    assert res.predicted_tokens == [7] * 9
    assert res.acceptance_rate == pytest.approx(4 / 8)       # 2 drafts per round, not d_max = 4


@dataclass
class ReferenceGenerationConfig:
    """The reference's GenerationConfig (generator_base.py:33-49): no threshold field."""
    max_steps: int = 512
    exit_layer: int = -1
    num_speculations: int = -1
    generation_strategy: str = "autoregressive"
    sample: bool = True
    temperature: float = 0.6
    top_k: int = 0
    top_p: float = 0.9
    no_repeat_ngram_size: Optional[int] = None
    stop_words: Optional[List[str]] = None
    stop_token_ids: Optional[List[int]] = field(default=None)


def test_reference_generation_config_still_works():
    eng, res = _run(ReferenceGenerationConfig(max_steps=5, exit_layer=2, num_speculations=3, sample=False))
    assert not hasattr(ReferenceGenerationConfig(), "draft_confidence_threshold")
    assert [c[0] for c in eng.calls] == ["round"] * len(eng.calls)
    assert res.predicted_tokens == [7] * 5


def test_round_output_confidence_field_is_optional():
    r = RoundOutput(n_drafted=0, n_matches=0, emitted=[1], draft=[], verified=[1], kv_len=3)
    assert r.draft_confidence is None
    assert GenerationConfig().draft_confidence_threshold == 0.0


@pytest.mark.parametrize("script", ["generate.py", "benchmark.py", "sweep.py"])
def test_threshold_flag_parses(monkeypatch, script):
    argv = [script, "--model", "synthetic:tiny-gqa", "--draft_confidence_threshold", "0.4"]
    monkeypatch.setattr(sys, "argv", argv)
    if script == "generate.py":
        parsed = cli.parse(cli.Arguments, cli.GenerateArguments, GenerationConfig)
    elif script == "sweep.py":
        parsed = cli.parse(cli.Arguments, cli.BenchmarkArguments, cli.SweepArguments, GenerationConfig)
    else:
        parsed = cli.parse(cli.Arguments, cli.BenchmarkArguments, GenerationConfig)
    assert parsed[-1].draft_confidence_threshold == pytest.approx(0.4)

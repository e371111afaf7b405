"""Self-speculation acceptance predicted from one teacher-forced pass (`Engine.score_exits`).

Pure host code.  The sweep (sweep.py:47-57, `cli.main_sweep`) runs a full benchmark of
generations for every (exit layer E, drafts D) pair; the quantities it reports follow from one
scoring pass over a text the full model generated:

* Greedy.  Let the text be prompt + the full-depth greedy continuation.  A draft at continuation
  position q is accepted exactly when the arg-max at E after the prefix equals the continuation's
  token q, and the verifier's bonus token is the continuation's next token.  So the rounds of
  greedy self-speculation, (n_drafted, n_matches) each, follow exactly from the agreement vector:
  `greedy_rounds`.
* Sampling.  The accept test u < min(1, p_L(t) / p_E(t)) with t ~ p_E accepts with probability
  alpha = sum_v min(p_E(v), p_L(v)) (p the warped distributions), which `score_exits` returns per
  position.  The mean alpha is exact as an expectation per evaluated draft; tokens per round and
  acceptance rate for D drafts then come from the i.i.d. formula, an estimate
  (`sampled_estimate`).

Neither models EOS inside a draft, stop words or the n-gram ban: the continuation is assumed to
draft no EOS id.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple


def greedy_rounds(agree: Sequence[bool], num_speculations: int, max_steps: int) -> List[Tuple[int, int]]:
    """(n_drafted, n_matches) of every round of greedy self-speculation
    (self_speculation_generator.py:51-99, 186-205) over a scored full-depth greedy continuation:
    agree[q] says whether the draft exit's arg-max at continuation position q equals the
    continuation's token q.  Each round drafts d = min(D, max_steps - len(out) - 1) tokens (the
    reference's clamp, so the last round may draft 0), accepts the leading agreeing drafts and
    appends them plus the verifier's token.  Assumes no EOS id is drafted."""
    if max_steps > 0 and len(agree) < max_steps - 1:
        raise ValueError(f"agreement vector of {len(agree)} positions is shorter than max_steps - 1 = {max_steps - 1}")
    rounds, out = [], 0
    while out < max_steps:
        d = min(num_speculations, max_steps - out - 1)
        n = 0
        while n < d and agree[out + n]:
            n += 1
        rounds.append((d, n))
        out += n + 1
    return rounds


def acceptance_rate(rounds: Sequence[Tuple[int, int]]) -> Optional[float]:
    """matches per drafted token over one generation (self_speculation_generator.py:96-99); None
    when nothing was drafted (the reference divides by zero there)."""
    drafted = sum(d for d, _ in rounds)
    return sum(n for _, n in rounds) / drafted if drafted else None


def tokens_per_round(rounds: Sequence[Tuple[int, int]]) -> Optional[float]:
    """tokens emitted per round (matches + the verifier's token)."""
    return sum(n + 1 for _, n in rounds) / len(rounds) if rounds else None


def mean(values) -> Optional[float]:
    """Mean over prompts, skipping None, as `cli.benchmark` averages per-prompt metrics."""
    vals = [float(v) for v in values if v is not None]
    return sum(vals) / len(vals) if vals else None


def sampled_estimate(alpha: float, num_speculations: int) -> Tuple[Optional[float], float]:
    """(acceptance rate, tokens per round) of sampled self-speculation with D drafts per round if
    every draft were accepted independently with probability `alpha`: an estimate, not exact
    (acceptance varies along the text).  Tokens per round = (1 - a^(D+1)) / (1 - a); acceptance
    rate = expected matches per drafted token.  The max_steps clamp is not modelled."""
    d = num_speculations
    tpr = float(d + 1) if alpha >= 1.0 else (1.0 - alpha ** (d + 1)) / (1.0 - alpha)
    return ((tpr - 1.0) / d if d > 0 else None), tpr

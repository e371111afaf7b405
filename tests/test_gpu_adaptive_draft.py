"""GPU: confidence-threshold drafting (`lsk_round_adaptive` / `Engine.round_adaptive`).

On tiny-mha, tiny-gqa and a two-layer Llama-2-7B-width model, greedy and sampled:
1. threshold 0 gives `round(d_max)`, round by round, every field;
2. replay: an adaptive generation and `round(n_drafted_j)` per round from a fresh begin / prefill
   with the same seed give the same rounds bit for bit (also with the n-gram ban, and as the first
   round of a fresh engine, whose skipped hidden rows were never written); greedy adaptive
   generation through the strategy equals autoregressive generation token for token;
3. the stop rule holds on the returned confidences;
4. confidences: sampled ones are the warped draft rows' probabilities bit for bit; greedy ones agree
   with the float64 early-exit oracle within DESIGN.md §7's log-probability bound;
5. in graph mode the skipped draft steps do not run (their layer-0 K rows stay untouched), and the
   eager engine returns the same rounds;
6. refusals."""
import math

import pytest
import torch

from oracle import llama_oracle as orc
from tests import parity_util as pu
from tests.test_gpu_engine import _Model
from tests.test_gpu_score import _dims, _engine, _ids

pytestmark = pytest.mark.gpu

D_MAX = 6
THRESHOLDS = (0.05, 0.3, 0.9, 1.0)
ROUNDS = 10
B_LOGPROB = 0.012          # DESIGN.md §7: engine vs oracle |d logprob| on the tiny models
# name: dims, exit layer, damping alpha of layers >= E
ARCHS = {
    "tiny-mha": (_dims(512, 256, 704, 4, 2, 2, 128), 2, 0.1),
    "tiny-gqa": (_dims(640, 512, 1408, 6, 4, 2, 128), 3, 0.1),
    "llama2-7b-l2": (_dims(32000, 4096, 11008, 2, 32, 32, 128), 1, 0.3),
}
SAMPLING = dict(sample=True, temperature=0.8, top_k=0, top_p=0.95)

_cache = {}


def _setup(name):
    if name not in _cache:
        dims, E, alpha = ARCHS[name]
        sd = orc.random_state_dict(dims, seed=5, damp_from_layer=E, alpha=alpha)
        _cache[name] = (dims, E, sd, _engine(dims, sd, 512))
    return _cache[name]


@pytest.fixture(scope="module", autouse=True)
def _close():
    yield
    for _d, _e, _s, eng in _cache.values():
        eng.close()
    _cache.clear()


def _start(eng, dims, E, sample, seed=11, ngram=0, prompt_seed=3):
    kw = SAMPLING if sample else dict(sample=False)
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=[dims.vocab - 1], seed=seed,
              no_repeat_ngram_size=ngram, **kw)
    prompt = _ids(dims.vocab, 24, prompt_seed)
    eng.prefill(prompt)
    return prompt


def _fields(r):
    return (r.n_drafted, r.n_matches, r.emitted, r.draft, r.verified, r.kv_len)


def _adaptive_rounds(eng, t, n=ROUNDS):
    return [eng.round_adaptive(D_MAX, t) for _ in range(n)]


def _check_stop_rule(rounds, t, eos):
    for r in rounds:
        c = r.draft_confidence
        assert len(c) == r.n_drafted >= 1 and all(0.0 <= x <= 1.0 for x in c)
        for i in range(r.n_drafted - 1):
            assert c[i] >= t and r.draft[i] != eos
        assert c[-1] < t or r.draft[-1] == eos or r.n_drafted == D_MAX


CASES = [(a, s) for a in ARCHS for s in (False, True)]
IDS = [f"{a}-{'sampled' if s else 'greedy'}" for a, s in CASES]


@pytest.mark.parametrize("name,sample", CASES, ids=IDS)
def test_threshold_zero_is_round_d_max(name, sample):
    dims, E, _sd, eng = _setup(name)
    _start(eng, dims, E, sample)
    got = _adaptive_rounds(eng, 0.0)
    _start(eng, dims, E, sample)
    want = [eng.round(D_MAX) for _ in range(ROUNDS)]
    assert [_fields(r) for r in got] == [_fields(r) for r in want]
    assert all(r.n_drafted == D_MAX or r.draft[-1] == dims.vocab - 1 for r in got)


def _quantile_thresholds(eng, dims, E, sample):
    """Random-init models are unsure of nearly every token (confidences near 1 / vocab), so the
    fixed thresholds all stop after one draft; thresholds at low quantiles of the model's own
    confidences make rounds stop at every length."""
    _start(eng, dims, E, sample)
    conf = sorted(c for r in _adaptive_rounds(eng, 0.0) for c in r.draft_confidence)
    return [conf[len(conf) // 10], conf[len(conf) // 4]]


@pytest.mark.parametrize("name,sample", CASES, ids=IDS)
def test_replay_with_fixed_rounds_and_stop_rule(name, sample):
    dims, E, _sd, eng = _setup(name)
    seen = set()
    for t in list(THRESHOLDS) + _quantile_thresholds(eng, dims, E, sample):
        _start(eng, dims, E, sample)
        got = _adaptive_rounds(eng, t)
        _check_stop_rule(got, t, dims.vocab - 1)
        _start(eng, dims, E, sample)
        want = [eng.round(r.n_drafted) for r in got]
        assert [_fields(r) for r in got] == [_fields(r) for r in want], f"t={t}"
        seen |= {r.n_drafted for r in got}
    assert len(seen) >= 3, f"rounds drafted only {sorted(seen)} tokens: the stop rule is not exercised"


def test_replay_with_ngram_ban():
    dims, E, _sd, eng = _setup("tiny-gqa")
    for sample in (False, True):
        t = _quantile_thresholds(eng, dims, E, sample)[0]
        _start(eng, dims, E, sample, ngram=2)
        got = _adaptive_rounds(eng, t, 16)
        _check_stop_rule(got, t, dims.vocab - 1)
        _start(eng, dims, E, sample, ngram=2)
        want = [eng.round(r.n_drafted) for r in got]
        assert [_fields(r) for r in got] == [_fields(r) for r in want]


@pytest.mark.parametrize("sample", (False, True), ids=("greedy", "sampled"))
def test_first_round_on_a_fresh_engine(sample):
    dims, E, sd, _ = _setup("tiny-gqa")
    outs = []
    for adaptive in (True, False):
        eng = _engine(dims, sd, 512)
        try:
            _start(eng, dims, E, sample)
            outs.append(eng.round_adaptive(D_MAX, 1.0) if adaptive else eng.round(outs[0].n_drafted))
        finally:
            eng.close()
    assert outs[0].n_drafted < D_MAX
    assert _fields(outs[0]) == _fields(outs[1])


@pytest.mark.parametrize("name", list(ARCHS))
def test_greedy_adaptive_generation_equals_autoregressive(name):
    from layerskip_b200 import GenerationConfig
    from layerskip_b200.strategy import (B200AutoRegressiveGenerationStrategy,
                                         B200SelfSpeculativeGenerationStrategy)
    dims, E, sd, _ = _setup(name)
    model = _Model(dims, sd)
    prompt = _ids(dims.vocab, 24, 3)
    spec = B200SelfSpeculativeGenerationStrategy(max_ctx=256)
    try:
        ar = B200AutoRegressiveGenerationStrategy(engine_cache=spec.engines).generate_token_ids(
            model, prompt, [dims.vocab - 1], GenerationConfig(max_steps=48, sample=False))
        for t in list(THRESHOLDS) + _quantile_thresholds(spec.engine_for(model), dims, E, False):
            cfg = GenerationConfig(max_steps=48, exit_layer=E, num_speculations=D_MAX, sample=False,
                                   draft_confidence_threshold=t)
            got = spec.generate_token_ids(model, prompt, [dims.vocab - 1], cfg)
            assert got.predicted_tokens == ar.predicted_tokens, f"t={t}"
            assert all(r.draft_confidence is not None for r in spec.last_rounds)
    finally:
        spec.engines.close()


@pytest.mark.parametrize("name", list(ARCHS))
def test_sampled_confidence_is_the_warped_draft_probability(name):
    dims, E, _sd, eng = _setup(name)
    t = _quantile_thresholds(eng, dims, E, True)[0]
    _start(eng, dims, E, True)
    for _ in range(ROUNDS):
        r = eng.round_adaptive(D_MAX, t)
        probs = eng.debug_probs("draft", r.n_drafted)
        assert r.draft_confidence == [float(probs[i, t]) for i, t in enumerate(r.draft)]


@pytest.mark.parametrize("name", ["tiny-mha", "tiny-gqa"])
def test_greedy_confidence_against_the_early_exit_oracle(name):
    dims, E, sd, eng = _setup(name)
    w = orc.weights_from_state_dict(dims, sd)
    pu.set_oracle_threads()
    worst = 0.0
    for prompt_seed in range(4):
        prompt = _start(eng, dims, E, False, prompt_seed=prompt_seed)
        r = eng.round_adaptive(D_MAX, 0.0)
        with torch.inference_mode():
            logits = orc.early_exit_logits(w, prompt, r.draft, E).double()
        want = torch.log_softmax(logits, dim=-1)[torch.arange(r.n_drafted), torch.tensor(r.draft)]
        got = torch.tensor(r.draft_confidence, dtype=torch.float64).log()
        worst = max(worst, float((got - want).abs().max()))
    print(f"MEASURED greedy_confidence_dlogprob {worst:.4g}", flush=True)
    assert worst <= B_LOGPROB


@pytest.mark.parametrize("sample", (False, True), ids=("greedy", "sampled"))
def test_skipped_steps_do_not_run_and_eager_agrees(sample):
    dims, E, sd, eng = _setup("tiny-gqa")
    prompt_seed = 20 + int(sample)                   # a prompt no other test writes rows for
    _start(eng, dims, E, sample, prompt_seed=prompt_seed)
    p = eng.kv_len
    before = eng.debug_kv_rows("k", 0, 0, p + 2, D_MAX - 1)
    r = eng.round_adaptive(D_MAX, 1.0)
    assert r.n_drafted == 1 and r.draft_confidence[0] < 1.0
    assert torch.equal(eng.debug_kv_rows("k", 0, 0, p + 2, D_MAX - 1), before)
    _start(eng, dims, E, sample, prompt_seed=prompt_seed)
    eng.round(D_MAX)                                  # a fixed round writes those rows: the check can fail
    assert not torch.equal(eng.debug_kv_rows("k", 0, 0, p + 2, D_MAX - 1), before)

    eager = _engine(dims, sd, 512, use_graph=False)
    try:
        for t in [0.3] + _quantile_thresholds(eng, dims, E, sample):
            runs = []
            for e in (eng, eager):
                _start(e, dims, E, sample)
                runs.append([_fields(x) + (x.draft_confidence,) for x in _adaptive_rounds(e, t)])
            assert runs[0] == runs[1], f"t={t}"
    finally:
        eager.close()


def test_refusals_leave_the_engine_usable():
    from layerskip_b200._lib import LskError
    dims, E, _sd, eng = _setup("tiny-mha")
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
    with pytest.raises(LskError) as ex:
        eng.round_adaptive(D_MAX, 0.5)                    # before prefill
    assert ex.value.code == -3
    _start(eng, dims, E, False)
    for t in (-0.1, 1.5, math.nan):
        with pytest.raises(LskError) as ex:
            eng.round_adaptive(D_MAX, t)
        assert ex.value.code == -1
    for d in (-1, eng.max_rows):
        with pytest.raises(LskError) as ex:
            eng.round_adaptive(d, 0.5)
        assert ex.value.code == -1
    r = eng.round_adaptive(D_MAX, 0.5)
    assert r.kv_len > 24 - 1 and len(r.draft_confidence) == r.n_drafted
    assert eng.round_adaptive(0, 0.5).n_drafted == 0

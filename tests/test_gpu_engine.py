"""GPU parity tests proper: the CUDA engine, driven through the reference-shaped strategies and
the C ABI, against (a) the committed golden traces of the unmodified reference and (b) the CPU
oracle on the same seeded weights."""
import pytest
import torch

from oracle import llama_oracle as orc
from tests import golden_util as gu
from tests import parity_util as pu

pytestmark = pytest.mark.gpu

ENGINE_MODELS = ("tiny_mha128", "tiny_gqa128", "survey_mha32")   # survey_mha32 = correctness.py's config (head_dim 32)


def _engine_cases(greedy=True):
    return [c for c in gu.spec_cases(greedy=greedy) if c["model"] in ENGINE_MODELS]


class _Model:
    """Minimal model handle: `.config` + `.state_dict()` like an HF LlamaForCausalLM."""

    def __init__(self, dims, sd):
        self._sd = sd
        self.config = type("Cfg", (), dict(
            vocab_size=dims.vocab, hidden_size=dims.hidden, intermediate_size=dims.inter,
            num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
            num_key_value_heads=dims.kv_heads, head_dim=dims.head_dim,
            rms_norm_eps=dims.rms_eps, rope_theta=dims.rope_theta))()

    def state_dict(self):
        return self._sd


def _gen_cfg(case, **over):
    from layerskip_b200 import GenerationConfig
    cfg = dict(case["cfg"])
    cfg.update(over)
    return GenerationConfig(**cfg)


@pytest.fixture(scope="module")
def strategies():
    from layerskip_b200.strategy import (B200AutoRegressiveGenerationStrategy,
                                         B200SelfSpeculativeGenerationStrategy)
    spec = B200SelfSpeculativeGenerationStrategy(max_ctx=512, keep_logits=True)
    ar = B200AutoRegressiveGenerationStrategy(engine_cache=spec.engines)
    yield spec, ar
    spec.engines.close()


_models = {}


def _model_for(case):
    key = (case["model"], case["weight_seed"], case["damp_from"], case["alpha"])
    if key not in _models:
        dims, sd = gu.state_dict_for(case)
        _models[key] = (dims, _Model(dims, sd), orc.weights_from_state_dict(dims, sd))
    return _models[key]


@pytest.mark.parametrize("case", _engine_cases(), ids=lambda c: c["name"])
def test_speculative_tokens_match_reference_golden(case, strategies):
    """Greedy self-speculative output == the reference's (margin-gated, teacher-forced)."""
    spec, _ = strategies
    dims, model, w = _model_for(case)
    ref = case["reference"]

    def generate(prompt, n):
        cfg = _gen_cfg(case, max_steps=n)
        return spec.generate_token_ids(model, prompt, case["eos"], cfg).predicted_tokens

    flips, gaps = pu.check_stream(w, case["prompt"], ref["spec_tokens"], generate)
    assert flips <= max(2, len(ref["spec_tokens"]) // 8), gaps   # each flip already gated by TAU


@pytest.mark.parametrize("case", _engine_cases(), ids=lambda c: c["name"])
def test_round_trace_matches_reference_golden(case, strategies):
    """Per-round (drafted, matched, emitted, kv length) equal the reference's when the token
    streams agree (they do unless a benign flip occurred; then only invariants are checked)."""
    spec, _ = strategies
    dims, model, w = _model_for(case)
    ref = case["reference"]
    res = spec.generate_token_ids(model, case["prompt"], case["eos"], _gen_cfg(case))
    rounds = spec.last_rounds
    for r in rounds:
        assert r.n_matches <= r.n_drafted                 # reference test: matches <= specs
        assert len(r.emitted) == r.n_matches + 1
    n_prompt = len(case["prompt"])
    total = 0
    for r in rounds:
        total += len(r.emitted)
        assert r.kv_len == n_prompt + total - 1           # rollback invariant (:219-221)
    if res.predicted_tokens != ref["spec_tokens"]:
        return                       # a benign flip in the full model: covered by check_stream
    # Same tokens: the round structure must match the reference's too, except after a benign
    # near-tie flip inside the DRAFT sub-model (layers < E), which changes how many drafts are
    # accepted but never the emitted tokens.  Such a flip must be within TAU under the
    # oracle's early-exit logits.
    oracle = orc.self_speculative_generate(w, case["prompt"], case["eos"], **case["cfg"])
    assert [len(r.draft) for r in oracle.rounds] == [t["d_actual"] for t in ref["rounds"]]
    history = list(case["prompt"])
    for mine, theirs in zip(rounds, oracle.rounds):
        if mine.draft == theirs.draft:
            assert mine.n_matches == theirs.n_matches
            assert mine.emitted == theirs.emitted
            assert mine.kv_len == theirs.kv_len_after
            history += theirs.emitted
            continue
        i = next(k for k in range(min(len(mine.draft), len(theirs.draft)))
                 if mine.draft[k] != theirs.draft[k])
        # the draft model is fed its own previous drafts: history + [input] + draft[:i]
        fed = theirs.draft[:i]
        logits = orc.early_exit_logits(w, history, fed + [0], case["cfg"]["exit_layer"])
        row = logits[len(fed)]
        gap = float(row[theirs.draft[i]] - row[mine.draft[i]])
        assert 0 <= gap < pu.TAU, f"draft flip with logit gap {gap}"
        break
    else:
        assert len(rounds) == len(oracle.rounds)
        assert res.acceptance_rate == pytest.approx(ref["acceptance_rate"], abs=1e-12)


@pytest.mark.parametrize("case", _engine_cases(), ids=lambda c: c["name"])
def test_speculative_equals_autoregressive_on_engine(case, strategies):
    """correctness.py:82-88 on the engine itself — exact, because the kernels are
    batch-invariant (no margin gate needed)."""
    spec, ar = strategies
    dims, model, w = _model_for(case)
    s = spec.generate_token_ids(model, case["prompt"], case["eos"], _gen_cfg(case))
    a = ar.generate_token_ids(model, case["prompt"], case["eos"],
                              _gen_cfg(case, exit_layer=-1, num_speculations=-1))
    assert s.predicted_tokens == a.predicted_tokens


@pytest.mark.parametrize("case", _engine_cases()[:4], ids=lambda c: c["name"])
def test_autoregressive_and_early_exit_match_reference_golden(case, strategies):
    _, ar = strategies
    dims, model, w = _model_for(case)
    ref = case["reference"]

    def gen_full(prompt, n):
        return ar.generate_token_ids(model, prompt, case["eos"],
                                     _gen_cfg(case, max_steps=n, exit_layer=-1,
                                              num_speculations=-1)).predicted_tokens

    pu.check_stream(w, case["prompt"], ref["ar_tokens"], gen_full)

    def gen_early(prompt, n):
        return ar.generate_token_ids(model, prompt, case["eos"],
                                     _gen_cfg(case, max_steps=n, num_speculations=-1)
                                     ).predicted_tokens

    pu.check_stream(w, case["prompt"], ref["early_exit_tokens"], gen_early,
                    exit_layer=case["cfg"]["exit_layer"])


@pytest.mark.parametrize("mname,seed", [("tiny_mha128", 1), ("tiny_gqa128", 4), ("survey_mha32", 0)])
def test_logits_close_to_oracle(mname, seed, strategies):
    """Engine logits vs the oracle's (and hence the reference's forward, see
    tests/golden/layer_arith.json) on a prompt: max |delta| must stay well under TAU/2."""
    spec, ar = strategies
    case = next(c for c in gu.load("layer_arith.json")["cases"] if c["model"] == mname)
    dims, sd = gu.state_dict_for(case, alpha_key=False)
    model = _Model(dims, sd)
    w = orc.weights_from_state_dict(dims, sd)
    eng = spec.engine_for(model)
    prompt = case["prompt"]
    eng.begin(exit_layer=-1, max_steps=4, eos_token_ids=[dims.vocab - 1])
    eng.prefill(prompt)
    tok = eng.ar_step()
    got = eng.debug_logits(1)[0]
    want = torch.tensor(case["full_logits_last"])
    err = float((got - want).abs().max())
    assert err < pu.TAU / 2, err
    assert tok == int(want.argmax()) or float(want.max() - want[tok]) < pu.TAU
    # K/V rows written by the prefill (keys are stored post-RoPE)
    kv = orc.KVStore(dims.layers)
    orc.step_all_layers(w, prompt, kv)
    for pos in (0, 5, len(prompt) - 1):
        k = eng.debug_kv_row("k", 0, 0, pos)
        v = eng.debug_kv_row("v", 0, 0, pos)
        torch.testing.assert_close(k, kv.k[0][0, pos], rtol=2e-2, atol=2e-2)
        torch.testing.assert_close(v, kv.v[0][0, pos], rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(eng.debug_kv_row("k", 0, 0, len(prompt) - 1),
                               torch.tensor(case["k_cache_l0_h0_last"]), rtol=2e-2, atol=2e-2)


def test_page_table_indirection(strategies):
    """Same tokens with a permuted logical->physical KV page map."""
    spec, _ = strategies
    case = next(c for c in _engine_cases() if c["name"] == "gqa128_a0.05_long")
    dims, model, w = _model_for(case)
    base = spec.generate_token_ids(model, case["prompt"], case["eos"], _gen_cfg(case))
    eng = spec.engine_for(model)
    n_pages = (eng.max_ctx + 63) // 64
    perm = list(reversed(range(n_pages)))
    eng.debug_set_page_table(perm)
    try:
        again = spec.generate_token_ids(model, case["prompt"], case["eos"], _gen_cfg(case))
    finally:
        eng.debug_set_page_table(list(range(n_pages)))
    assert again.predicted_tokens == base.predicted_tokens


@pytest.mark.parametrize("n", [1, 2, 3])
def test_no_repeat_ngram_ban_on_the_device_matches_the_oracle(n, strategies):
    """`--no_repeat_ngram_size` (generator_base.py:77-85): the device ban list gives the oracle's
    (= HF processor's) tokens, the continuation never completes an n-gram that is already in the
    sequence, and speculative == autoregressive still holds exactly."""
    from transformers.generation.logits_process import LogitsProcessorList, NoRepeatNGramLogitsProcessor
    spec, ar = strategies
    case = next(c for c in _engine_cases() if c["name"] == "gqa128_a0.1")
    dims, model, w = _model_for(case)
    prompt = [11, 500, 23, 11, 500, 23, 8, 8, 8, 639 - 1, 100]            # repeats inside the prompt
    procs = LogitsProcessorList([NoRepeatNGramLogitsProcessor(n)])
    cfg = _gen_cfg(case, max_steps=40)
    s = spec.generate_token_ids(model, prompt, case["eos"], cfg, logits_processors=procs)
    a = ar.generate_token_ids(model, prompt, case["eos"], _gen_cfg(case, max_steps=40, exit_layer=-1,
                                                                  num_speculations=-1), logits_processors=procs)
    assert s.predicted_tokens == a.predicted_tokens
    seq = prompt + s.predicted_tokens
    for pos in range(len(prompt), len(seq)):                  # the token at `pos` never completes a seen n-gram
        gram = tuple(seq[pos - n + 1: pos + 1])
        assert all(tuple(seq[i:i + n]) != gram for i in range(0, pos - n + 1)), (n, pos, gram)
    want = orc.self_speculative_generate(w, prompt, case["eos"], **{**case["cfg"], "max_steps": 40},
                                         no_repeat_ngram_size=n).predicted_tokens
    j = next((k for k in range(min(len(want), len(s.predicted_tokens))) if want[k] != s.predicted_tokens[k]),
             None)
    if j is not None:                                         # only a near-tie may differ (margin gate)
        logits = orc.teacher_forced_logits(w, prompt, want[:j + 1])[j:j + 1]
        row = orc.ban_repeated_ngrams(logits, [prompt + want[:j]], n)[0]
        assert float(row[want[j]] - row[s.predicted_tokens[j]]) < pu.TAU
    else:
        assert len(want) == len(s.predicted_tokens)
    # sampling with the ban runs and respects it too
    torch.manual_seed(1)
    smp = spec.generate_token_ids(model, prompt, case["eos"], _gen_cfg(case, max_steps=40, sample=True),
                                  logits_processors=procs)
    seq = prompt + smp.predicted_tokens
    for pos in range(len(prompt), len(seq)):
        gram = tuple(seq[pos - n + 1: pos + 1])
        assert all(tuple(seq[i:i + n]) != gram for i in range(0, pos - n + 1)), ("sample", n, pos)


def test_unsupported_inputs_fail_loudly(strategies):
    spec, _ = strategies
    case = _engine_cases()[0]
    dims, model, w = _model_for(case)
    with pytest.raises(NotImplementedError):
        spec.generate_token_ids(model, case["prompt"], case["eos"], _gen_cfg(case),
                                logits_processors=[lambda i, s: s])


def test_wgmma_prefill_matches_the_decode_kernel_prefill(monkeypatch):
    """lsk_prefill through the 128-token wgmma GEMMs (csrc/prefill_tc.cuh) vs the same prompt
    16 rows at a time through the decode kernels: same K/V rows up to bf16 rounding of different
    accumulation orders, next-step logits within the usual engine-vs-oracle tolerance, same token."""
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    case = next(c for c in gu.spec_cases() if c["name"] == "gqa128_a0.05_long")   # 70-token prompt
    dims, model, w = _model_for(case)
    arch = LlamaArch.from_hf_config(model.config)
    g = torch.Generator().manual_seed(7)
    prompt = torch.randint(3, dims.vocab - 1, (300,), generator=g).tolist()      # 3 chunks: 128 + 128 + 43
    out = {}
    for tc in (True, False):
        eng = Engine(arch, max_ctx=512, keep_logits=True, prefill_tc=tc)
        eng.load_model(model)
        eng.begin(exit_layer=-1, max_steps=4, eos_token_ids=[dims.vocab - 1])
        eng.prefill(prompt)
        rows = [eng.debug_kv_row(which, layer, 0, pos) for which in "kv" for layer in (0, dims.layers - 1)
                for pos in (0, 127, 128, 298)]
        tok = eng.ar_step()
        out[tc] = (torch.stack(rows), eng.debug_logits(1)[0], tok)
        eng.close()
    torch.testing.assert_close(out[True][0], out[False][0], rtol=2e-2, atol=2e-2)
    assert float((out[True][1] - out[False][1]).abs().max()) < pu.TAU / 2
    want = orc.teacher_forced_logits(w, prompt, [0])[0]
    assert float((out[True][1] - want).abs().max()) < pu.TAU / 2
    assert out[True][2] == out[False][2] or float(want.max() - want[out[True][2]]) < pu.TAU

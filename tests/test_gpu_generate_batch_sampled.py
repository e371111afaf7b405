"""GPU: sampled batched generation (`lsk_prefill_batch_seeded` / `lsk_round_batch` with sample = 1,
`Engine.prefill_batch(prompts, seeds)`, `generate_batch(..., seeds=...)`).

On tiny-mha, tiny-gqa (group 2), a head_dim-64 model, a two-layer Llama-2-7B-width model and a
two-layer model with Llama 3's 128256-token vocabulary, with damped late layers so drafts are
accepted:
1. every active sequence's rounds equal `lsk_round(d_seq)` of that sequence alone, begun with its own
   seed and the same warp settings, every field, for (B, D) in (2, 6), (3, 4), (4, 3), (8, 1),
   (16, 0), with per-sequence draft limits and a sequence that stops early on EOS (then inactive);
   its committed K/V rows in the first and last layer equal the solo run's;
2. the same prompt with two seeds diverges, and with one seed repeats, whatever its neighbours are;
3. a permuted page table, eager mode and no PDL give the same rounds;
4. greedy, sampled and greedy batches of one (E, d, B) each match their own reference (graph key);
5. `generate_batch(seeds=...)` equals per-prompt `generate_token_ids` with those engine seeds;
6. the memory the engine holds after a sampled batch is the plan with sampling + batch_seqs."""
import ctypes as C

import pytest
import torch

from layerskip_b200 import _lib
from layerskip_b200.engine import batch_slot_positions
from oracle import llama_oracle as orc
from tests.test_gpu_engine import _Model
from tests.test_gpu_score import _dims, _engine, _ids

pytestmark = pytest.mark.gpu

MAX_CTX = 2048
ROUNDS = 8
LENGTHS = (200, 1, 65, 2, 64, 17, 63, 5)
# name: dims, exit, damping alpha of layers >= the exit
ARCHS = {
    "tiny-mha": (_dims(512, 256, 704, 4, 2, 2, 128), 2, 0.1),
    "tiny-gqa": (_dims(640, 512, 1408, 6, 4, 2, 128), 3, 0.1),
    "hd64": (_dims(512, 256, 704, 3, 4, 2, 64), 1, 0.1),
    "llama2-7b-l2": (_dims(32000, 4096, 11008, 2, 32, 32, 128), 1, 0.3),
    "vocab128k-l2": (_dims(128256, 3072, 8192, 2, 24, 8, 128, 500000.0), 1, 0.3),
}
BATCHES = ((2, 6), (3, 4), (4, 3), (8, 1), (16, 0))     # (B, D): B * (D + 1) <= 16
# (temperature, top_k, top_p)
WARPS = ((0.6, 0, 0.9), (1.0, 50, 1.0), (0.3, 5, 0.5))

_cache = {}


def _setup(name):
    if name not in _cache:
        for _d, _s, eng in list(_cache.values()):
            eng.close()
        _cache.clear()
        dims, exit_layer, alpha = ARCHS[name]
        sd = orc.random_state_dict(dims, seed=5, damp_from_layer=exit_layer, alpha=alpha)
        _cache[name] = (dims, sd, _engine(dims, sd, MAX_CTX))
    return _cache[name]


@pytest.fixture(scope="module", autouse=True)
def _close():
    yield
    for _d, _s, eng in _cache.values():
        eng.close()
    _cache.clear()


def _fields(r):
    return (r.n_drafted, r.n_matches, r.emitted, r.draft, r.verified, r.kv_len)


def _warp(w):
    return dict(sample=True, temperature=w[0], top_k=w[1], top_p=w[2])


def _seeds(B, base):
    return [base + 7919 * s for s in range(B)]


def _lengths(B):
    return LENGTHS[:B] if B <= 8 else [1 + (7 * j) % 60 for j in range(B)]


def _first_token(eng, E, prompt, D, eos, warp, seed):
    """The first token a sampled solo round of D drafts emits: as an EOS id it ends that sequence in
    that round (the same draws pick it again, and it then truncates the output)."""
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, seed=seed, **_warp(warp))
    eng.prefill(prompt)
    return eng.round(D).emitted[0]


def _run_batch(eng, E, prompts, seeds, D, eos, warp, rounds=ROUNDS, vary=True):
    """Sampled batched rounds with per-sequence draft limits (all D unless `vary`); a sequence whose
    output reaches an EOS id turns inactive.  Returns [(d_seq, active, outs)] and the committed lengths."""
    B = len(prompts)
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, seed=12345, **_warp(warp))
    assert eng.prefill_batch(prompts, seeds) == batch_slot_positions(MAX_CTX, B)
    done = [False] * B
    trace = []
    for r in range(rounds):
        d_seq = [D - (s + r) % (D + 1) if vary else D for s in range(B)]
        active = [not x for x in done]
        outs = eng.round_batch(D, d_seq, active)
        trace.append((d_seq, active, outs))
        for s, o in enumerate(outs):
            if active[s] and any(t in eos for t in o.emitted):
                done[s] = True
    lens = [len(p) - 1 + sum(len(outs[s].emitted) for _d, _a, outs in trace) for s, p in enumerate(prompts)]
    return trace, lens


def _kv(eng, dims, pos0, count):
    if count == 0:
        return []
    return [eng.debug_kv_rows(w, l, 0, pos0, count) for w in "kv" for l in (0, dims.layers - 1)]


def _check_against_solo(eng, dims, E, prompts, seeds, eos, warp, trace, lens):
    slot = batch_slot_positions(MAX_CTX, len(prompts))
    batch_kv = [_kv(eng, dims, s * slot, lens[s]) for s in range(len(prompts))]
    for s, p in enumerate(prompts):
        eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, seed=seeds[s], **_warp(warp))
        eng.prefill(p)
        kv_len = len(p) - 1
        for r, (d_seq, active, outs) in enumerate(trace):
            o = outs[s]
            if not active[s]:
                assert (o.n_drafted, o.n_matches, o.emitted, o.kv_len) == (0, 0, [], kv_len), (s, r)
                continue
            want = eng.round(d_seq[s])
            assert _fields(o) == _fields(want), (s, r, d_seq[s])
            kv_len = want.kv_len
        assert kv_len == lens[s]
        solo_kv = _kv(eng, dims, 0, lens[s])
        assert all(torch.equal(a, b) for a, b in zip(batch_kv[s], solo_kv)), f"slot {s}: K/V rows differ"


CASES = [(name, B, D, w) for name in ARCHS for i, (B, D) in enumerate(BATCHES)
         for w in (range(3) if name == "tiny-gqa" else (i % 3,))
         if not (name in ("llama2-7b-l2", "vocab128k-l2") and B < 4)]


@pytest.mark.parametrize("name,B,D,w", CASES, ids=[f"{n}-B{b}-D{d}-W{w}" for n, b, d, w in CASES])
def test_rounds_equal_solo_rounds(name, B, D, w):
    dims, _sd, eng = _setup(name)
    E, warp = ARCHS[name][1], WARPS[w]
    prompts = [_ids(dims.vocab, n, 100 * B + j) for j, n in enumerate(_lengths(B))]
    seeds = _seeds(B, 1000 * B + w)
    eos = [dims.vocab - 1]
    eos.append(_first_token(eng, E, prompts[0], D, eos, warp, seeds[0]))
    trace, lens = _run_batch(eng, E, prompts, seeds, D, eos, warp)
    assert not trace[1][1][0], "the first sequence was meant to stop on EOS in its first round"
    assert sum(o.n_matches for _d, _a, outs in trace for o in outs) > 0 or D == 0, "no draft was accepted"
    _check_against_solo(eng, dims, E, prompts, seeds, eos, warp, trace, lens)


def _tokens(trace, s):
    return [t for _d, _a, outs in trace for t in outs[s].emitted]


def test_seeds_make_independent_and_repeatable_samples():
    name = "tiny-gqa"
    dims, _sd, eng = _setup(name)
    E, D, warp = ARCHS[name][1], 3, WARPS[1]
    p, q, r = (_ids(dims.vocab, n, 40 + n) for n in (30, 70, 5))
    eos = [dims.vocab - 1]
    # p with seeds 1 and 2 next to q; then p with seed 1 twice next to r, in another order
    a, _ = _run_batch(eng, E, [p, q, p, r], [1, 9, 2, 4], D, eos, warp, vary=False)
    b, _ = _run_batch(eng, E, [r, p, p], [4, 1, 1], D, eos, warp, vary=False)
    assert len(_tokens(a, 0)) >= ROUNDS
    assert _tokens(a, 0) != _tokens(a, 2), "two seeds gave the same sample"
    assert _tokens(a, 0) == _tokens(b, 1) == _tokens(b, 2)
    assert [_fields(o[0]) for _d, _a, o in a] == [_fields(o[1]) for _d, _a, o in b]
    assert _tokens(a, 3) == _tokens(b, 0)


def test_page_table_eager_and_no_pdl_agree():
    name = "tiny-gqa"
    dims, sd, eng = _setup(name)
    E, D, warp = ARCHS[name][1], 3, WARPS[0]
    prompts = [_ids(dims.vocab, n, 300 + n) for n in (200, 1, 65, 17)]
    seeds = _seeds(4, 77)
    eos = [dims.vocab - 1]
    ref, ref_lens = _run_batch(eng, E, prompts, seeds, D, eos, warp)
    slot = batch_slot_positions(MAX_CTX, 4)
    ref_kv = [_kv(eng, dims, s * slot, ref_lens[s]) for s in range(4)]
    perm = torch.randperm(MAX_CTX // 64, generator=torch.Generator().manual_seed(1)).tolist()
    for kw in (dict(use_graph=False), dict(use_pdl=False), dict(page_perm=perm)):
        perm_kw = kw.pop("page_perm", None)
        other = _engine(dims, sd, MAX_CTX, **kw)
        try:
            if perm_kw is not None:
                other.debug_set_page_table(perm_kw)
            got, lens = _run_batch(other, E, prompts, seeds, D, eos, warp)
            assert [[_fields(o) for o in outs] for _d, _a, outs in got] == \
                [[_fields(o) for o in outs] for _d, _a, outs in ref], kw
            kv = [_kv(other, dims, s * slot, lens[s]) for s in range(4)]
            assert all(torch.equal(a, b) for x, y in zip(kv, ref_kv) for a, b in zip(x, y)), kw
        finally:
            other.close()


def _greedy_batch(eng, E, prompts, D, eos):
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, sample=False)
    eng.prefill_batch(prompts)
    return [[_fields(o) for o in eng.round_batch(D)] for _ in range(4)]


def _sampled_batch(eng, E, prompts, seeds, D, eos):
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, seed=3, **_warp(WARPS[0]))
    eng.prefill_batch(prompts, seeds)
    return [[_fields(o) for o in eng.round_batch(D)] for _ in range(4)]


def test_greedy_and_sampled_batches_of_one_shape_keep_their_graphs():
    name = "tiny-mha"
    dims, sd, eng = _setup(name)
    E, D = ARCHS[name][1], 3
    prompts = [_ids(dims.vocab, n, 500 + n) for n in (20, 40, 9)]
    seeds = _seeds(3, 5)
    eos = [dims.vocab - 1]
    g1 = _greedy_batch(eng, E, prompts, D, eos)
    s1 = _sampled_batch(eng, E, prompts, seeds, D, eos)
    g2 = _greedy_batch(eng, E, prompts, D, eos)
    fresh = _engine(dims, sd, MAX_CTX)
    try:
        s_ref = _sampled_batch(fresh, E, prompts, seeds, D, eos)
        g_ref = _greedy_batch(fresh, E, prompts, D, eos)
    finally:
        fresh.close()
    assert g1 == g2 == g_ref
    assert s1 == s_ref
    assert s1 != g1
    # greedy generation ignores the seeds
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, sample=False)
    eng.prefill_batch(prompts, [11, 12, 13])
    assert [[_fields(o) for o in eng.round_batch(D)] for _ in range(4)] == g1


def test_refusals():
    name = "tiny-mha"
    dims, _sd, eng = _setup(name)
    E = ARCHS[name][1]
    prompts = [_ids(dims.vocab, n, 600 + n) for n in (10, 20)]
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], seed=1, **_warp(WARPS[0]))
    with pytest.raises(_lib.LskError) as ex:
        eng.prefill_batch(prompts)                                  # sampling needs seeds
    assert ex.value.code == -1
    ids = (C.c_int32 * 30)(*(prompts[0] + prompts[1]))
    off = (C.c_int32 * 3)(0, 10, 30)
    assert eng._lib.lsk_prefill_batch_seeded(eng._h, ids, off, 2, None, None) == -1
    for bad in ([1], [1, 2, 3], [-1, 2], [2 ** 64, 2]):
        with pytest.raises(ValueError):
            eng.prefill_batch(prompts, bad)
    eng.prefill_batch(prompts, [2 ** 64 - 1, 0])
    assert len(eng.round_batch(2)) == 2
    # the n-gram ban stays refused with seeds
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], seed=1, no_repeat_ngram_size=2,
              **_warp(WARPS[0]))
    with pytest.raises(_lib.LskError):
        eng.prefill_batch(prompts, [1, 2])


@pytest.mark.parametrize("name", ["tiny-mha", "hd64", "llama2-7b-l2"])
def test_generate_batch_equals_generate_token_ids(name, monkeypatch):
    from layerskip_b200 import GenerationConfig
    from layerskip_b200 import strategy as strategy_mod
    from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy
    dims, sd, _eng = _setup(name)
    E = ARCHS[name][1]
    prompts = [_ids(dims.vocab, n, 700 + n) for n in (65, 3, 200, 17)]
    seeds = [31, 2 ** 63 + 5, 31, 8]
    model = _Model(dims, sd)
    spec = B200SelfSpeculativeGenerationStrategy(max_ctx=MAX_CTX)
    try:
        for w, max_steps in ((WARPS[0], 37), (WARPS[2], 64)):
            cfg = GenerationConfig(max_steps=max_steps, exit_layer=E, num_speculations=3, sample=True,
                                   temperature=w[0], top_k=w[1], top_p=w[2])
            got = spec.generate_batch(model, prompts, [dims.vocab - 1], cfg, seeds=seeds)
            for p, sd_j, g in zip(prompts, seeds, got):
                monkeypatch.setattr(strategy_mod, "_generation_seed", lambda cache, eng, sample, s=sd_j: s)
                want = spec.generate_token_ids(model, p, [dims.vocab - 1], cfg)
                assert g.predicted_tokens == want.predicted_tokens
                assert g.acceptance_rate == want.acceptance_rate
    finally:
        spec.engines.close()


def test_memory_in_use_is_the_plan_with_sampling_and_batch_seqs():
    name = "tiny-gqa"
    dims, sd, _ = _setup(name)
    eng = _engine(dims, sd, MAX_CTX)
    try:
        eng.begin(exit_layer=3, max_steps=64, eos_token_ids=[dims.vocab - 1], seed=1, **_warp(WARPS[0]))
        eng.prefill_batch([_ids(dims.vocab, n, n) for n in (9, 70, 3)], [1, 2, 3])
        eng.round_batch(3)
        flags = 0 if eng.prefill_tc else _lib.LSK_FLAG_NO_PREFILL_TC
        cfg = eng.arch.lsk_config(MAX_CTX, flags=flags)
        sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
        want, got = _lib.lsk_memory_plan(), _lib.lsk_memory_plan()
        uses = _lib.lsk_memory_uses(sampling=1, batch_seqs=3)
        _lib.check(eng._lib.lsk_plan_memory(C.byref(cfg), sms, C.byref(uses), C.byref(want)))
        _lib.check(eng._lib.lsk_memory_in_use(eng._h, C.byref(got)))
        fields = [f for f, _ in _lib.lsk_memory_plan._fields_]
        assert [getattr(got, f) for f in fields] == [getattr(want, f) for f in fields]
    finally:
        eng.close()

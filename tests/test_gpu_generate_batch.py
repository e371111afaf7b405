"""GPU: batched greedy generation (`lsk_prefill_batch` / `lsk_round_batch`, `Engine.round_batch`,
`B200SelfSpeculativeGenerationStrategy.generate_batch`).

On tiny-mha, tiny-gqa (group 2), a head_dim-64 model and a two-layer Llama-2-7B-width model, with
damped late layers so drafts are accepted:
1. every active sequence's rounds equal `lsk_round(d_seq)` of that sequence alone from a fresh
   begin / prefill, every field, for B in {2, 3, 4, 8} at several exits, with per-sequence draft
   limits, prompts of 1, 2, max_rows + 1, 63, 64, 65 and 200 tokens and a sequence that stops early
   on EOS (then inactive: no tokens, kv_len unchanged);
2. after the batch, every slot's committed K/V rows equal the solo run's rows at the same
   positions (no cross-slot writes, inactive sequences untouched);
3. B = 16 at d = 0 equals `lsk_round(0)` per sequence;
4. `generate_batch` equals per-prompt `generate_token_ids`: tokens and acceptance rate, with the
   max_steps clamp;
5. a permuted page table, eager mode and no PDL give the same rounds;
6. refusals and state rules;
7. the memory the engine holds after a batch is the plan with batch_seqs."""
import ctypes as C

import pytest
import torch

from layerskip_b200 import _lib
from layerskip_b200._lib import LskError
from layerskip_b200.engine import batch_slot_positions
from oracle import llama_oracle as orc
from tests.test_gpu_engine import _Model
from tests.test_gpu_score import _dims, _engine, _ids

pytestmark = pytest.mark.gpu

MAX_CTX = 2048
ROUNDS = 8
LENGTHS = (200, 1, 65, 2, 64, 17, 63, 5)     # 17 = max_rows + 1: the longest decode-route prompt
# name: dims, exits to test, damping alpha of layers >= the first exit
ARCHS = {
    "tiny-mha": (_dims(512, 256, 704, 4, 2, 2, 128), (2, 1), 0.1),
    "tiny-gqa": (_dims(640, 512, 1408, 6, 4, 2, 128), (3, 5), 0.1),
    "hd64": (_dims(512, 256, 704, 3, 4, 2, 64), (1, 2), 0.1),
    "llama2-7b-l2": (_dims(32000, 4096, 11008, 2, 32, 32, 128), (1,), 0.3),
}
BATCHES = ((2, 6), (3, 4), (4, 3), (8, 1))     # (B, D): B * (D + 1) <= 16

_cache = {}


def _setup(name):
    if name not in _cache:
        for _k, (_d, _s, eng) in list(_cache.items()):
            eng.close()
        _cache.clear()
        dims, exits, alpha = ARCHS[name]
        sd = orc.random_state_dict(dims, seed=5, damp_from_layer=exits[0], alpha=alpha)
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


def _prompts(dims, lengths, seed=0):
    return [_ids(dims.vocab, n, 100 * seed + j) for j, n in enumerate(lengths)]


def _early_token(eng, dims, E, prompt, D):
    """A token among the first D + 1 that greedy generation of `prompt` emits: as an EOS id it stops
    that sequence within its first D + 1 tokens."""
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=[dims.vocab - 1], sample=False)
    eng.prefill(prompt)
    return eng.round(D).emitted[-1]


def _run_batch(eng, dims, E, prompts, D, eos, rounds=ROUNDS, vary=True):
    """Batched rounds with per-sequence draft limits; a sequence whose output reaches an EOS id
    turns inactive.  Returns the rounds as [(d_seq, active, outs)] and the committed lengths."""
    B = len(prompts)
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, sample=False)
    slot = eng.prefill_batch(prompts)
    assert slot == batch_slot_positions(MAX_CTX, B)
    done = [False] * B
    trace = []
    for r in range(rounds):
        d_seq = [(D - (s + r) % (D + 1)) if vary else D for s in range(B)]
        active = [not x for x in done]
        outs = eng.round_batch(D, d_seq, active)
        trace.append((d_seq, active, outs))
        for s, o in enumerate(outs):
            if active[s] and any(t in eos for t in o.emitted):
                done[s] = True
    lens = [len(p) - 1 + sum(len(outs[s].emitted) for _d, _a, outs in trace) for s, p in enumerate(prompts)]
    return trace, lens, slot


def _kv(eng, dims, pos0, count):
    """K and V rows at positions pos0 .. pos0 + count - 1 of kv head 0 in the first and last layer."""
    if count == 0:
        return []
    return [eng.debug_kv_rows(w, l, 0, pos0, count) for w in "kv" for l in (0, dims.layers - 1)]


def _check_against_solo(eng, dims, E, prompts, eos, trace, lens, slot):
    batch_kv = [_kv(eng, dims, s * slot, lens[s]) for s in range(len(prompts))]
    for s, p in enumerate(prompts):
        eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, sample=False)
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


CASES = [(name, B, D, E) for name, (_d, exits, _a) in ARCHS.items() for (B, D) in BATCHES for E in exits
         if not (name == "llama2-7b-l2" and B < 4)]


@pytest.mark.parametrize("name,B,D,E", CASES, ids=[f"{n}-B{b}-D{d}-E{e}" for n, b, d, e in CASES])
def test_rounds_equal_solo_rounds(name, B, D, E):
    dims, _sd, eng = _setup(name)
    lengths = LENGTHS[:B] if B < 8 else LENGTHS
    prompts = _prompts(dims, lengths, seed=B)
    eos = [dims.vocab - 1, _early_token(eng, dims, E, prompts[0], D)]
    trace, lens, slot = _run_batch(eng, dims, E, prompts, D, eos)
    assert any(not a[0] for _d, a, _o in trace), "the first sequence was meant to stop early on EOS"
    _check_against_solo(eng, dims, E, prompts, eos, trace, lens, slot)


@pytest.mark.parametrize("name", ["tiny-gqa", "llama2-7b-l2"])
def test_sixteen_sequences_at_d0(name):
    dims, _sd, eng = _setup(name)
    E = ARCHS[name][1][0]
    prompts = _prompts(dims, [1 + (7 * j) % 60 for j in range(16)], seed=16)
    trace, lens, slot = _run_batch(eng, dims, E, prompts, 0, [dims.vocab - 1], rounds=6, vary=False)
    _check_against_solo(eng, dims, E, prompts, [dims.vocab - 1], trace, lens, slot)


@pytest.mark.parametrize("name", ["tiny-mha", "hd64", "llama2-7b-l2"])
def test_generate_batch_equals_generate_token_ids(name):
    from layerskip_b200 import GenerationConfig
    from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy
    dims, sd, eng = _setup(name)
    E = ARCHS[name][1][0]
    prompts = _prompts(dims, (65, 3, 200, 17), seed=7)
    early = _early_token(eng, dims, E, prompts[1], 3)
    model = _Model(dims, sd)
    spec = B200SelfSpeculativeGenerationStrategy(max_ctx=MAX_CTX)
    try:
        for max_steps, eos in ((37, [dims.vocab - 1]), (64, [dims.vocab - 1]), (37, [dims.vocab - 1, early])):
            cfg = GenerationConfig(max_steps=max_steps, exit_layer=E, num_speculations=3, sample=False)
            got = spec.generate_batch(model, prompts, eos, cfg)
            for p, g in zip(prompts, got):
                want = spec.generate_token_ids(model, p, eos, cfg)
                assert g.predicted_tokens == want.predicted_tokens
                assert g.acceptance_rate == want.acceptance_rate
            if early in eos:
                assert len(got[1].predicted_tokens) < 4                # stopped on EOS in its first round
            else:
                assert any(len(g.predicted_tokens) == max_steps for g in got)   # ran into the clamp
    finally:
        spec.engines.close()


def test_page_table_eager_and_no_pdl_agree():
    name = "tiny-gqa"
    dims, sd, eng = _setup(name)
    E, D = ARCHS[name][1][0], 3
    prompts = _prompts(dims, (200, 1, 65, 17), seed=3)
    eos = [dims.vocab - 1]
    ref, ref_lens, slot = _run_batch(eng, dims, E, prompts, D, eos)
    ref_kv = [_kv(eng, dims, s * slot, ref_lens[s]) for s in range(len(prompts))]
    n_pages = MAX_CTX // 64
    perm = torch.randperm(n_pages, generator=torch.Generator().manual_seed(1)).tolist()
    for kw in (dict(use_graph=False), dict(use_pdl=False), dict(page_perm=perm)):
        perm_kw = kw.pop("page_perm", None)
        other = _engine(dims, sd, MAX_CTX, **kw)
        try:
            if perm_kw is not None:
                other.debug_set_page_table(perm_kw)
            got, lens, _ = _run_batch(other, dims, E, prompts, D, eos)
            assert [[_fields(o) for o in outs] for _d, _a, outs in got] == \
                [[_fields(o) for o in outs] for _d, _a, outs in ref], kw
            kv = [_kv(other, dims, s * slot, lens[s]) for s in range(len(prompts))]
            assert all(torch.equal(a, b) for x, y in zip(kv, ref_kv) for a, b in zip(x, y)), kw
        finally:
            other.close()


def _code(fn, *a):
    with pytest.raises(LskError) as ex:
        fn(*a)
    return ex.value.code


def test_refusals_and_state_rules():
    dims, _sd, eng = _setup("tiny-mha")
    E = 2
    prompts = _prompts(dims, (10, 20, 30), seed=9)
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
    assert _code(eng.round_batch, 0) == -3                           # no batch yet
    lib, h = eng._lib, eng._h
    outs = (_lib.lsk_round_out * 16)()
    # the generation must be greedy, without the n-gram ban, with a self-speculation exit
    for kw in (dict(sample=True), dict(no_repeat_ngram_size=2), dict(exit_layer=0)):
        args = dict(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
        args.update(kw)
        eng.begin(**args)
        assert _code(eng.prefill_batch, prompts) == -1, kw
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
    assert _code(eng.prefill_batch, []) == -1
    assert _code(eng.prefill_batch, [[5]] * 17) == -1
    assert _code(eng.prefill_batch, [[5], []]) == -1
    assert _code(eng.prefill_batch, [[5], [dims.vocab]]) == -1
    slot = batch_slot_positions(MAX_CTX, 3)
    assert _code(eng.prefill_batch, [[5], [6] * slot, [7]]) == -6        # prompt + 1 > slot
    eng.prefill_batch([[5], [6] * (slot - 1), [7]])                       # prompt + 1 == slot fits
    eng.round_batch(0)                                                    # kv_len + 2 == slot
    assert _code(eng.round_batch, 0) == -6
    eng.prefill_batch(prompts)
    for d_req, d_seq in ((5, None), (-1, None), (3, [0, 4, 0]), (3, [0, -1, 0])):
        assert _code(eng.round_batch, d_req, d_seq) == -1, (d_req, d_seq)
    # kv_len + d_req + 2 > slot of an INACTIVE sequence is refused too
    eng.prefill_batch([[5], [6] * (slot - 3), [7]])
    assert eng.round_batch(0, None, [True, False, True])[1].emitted == []
    assert _code(eng.round_batch, 3, None, [True, False, True]) == -6    # slot - 4 + 3 + 2 > slot
    eng.prefill_batch(prompts)
    first = eng.round_batch(3)
    # a batch ends the single-sequence generation, and a prefill or scoring call ends the batch
    assert _code(eng.round, 1) == -3
    assert _code(eng.round_adaptive, 1, 0.5) == -3
    assert _code(eng.ar_step) == -3
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
    eng.prefill(prompts[0])
    assert lib.lsk_round_batch(h, 0, None, None, outs) == -3
    after = [eng.round(2) for _ in range(3)]
    eng.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
    eng.prefill_batch(prompts)
    assert [_fields(r) for r in eng.round_batch(3)] == [_fields(r) for r in first]
    eng.score(prompts[1])
    assert lib.lsk_round_batch(h, 0, None, None, outs) == -3
    # a begin + prefill after a batch behaves as on a fresh engine
    fresh = _engine(dims, _sd, MAX_CTX)
    try:
        fresh.begin(exit_layer=E, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
        fresh.prefill(prompts[0])
        assert [_fields(fresh.round(2)) for _ in range(3)] == [_fields(r) for r in after]
    finally:
        fresh.close()


def test_memory_in_use_is_the_plan_with_batch_seqs():
    name = "tiny-gqa"
    dims, sd, _ = _setup(name)
    eng = _engine(dims, sd, MAX_CTX)
    try:
        eng.begin(exit_layer=3, max_steps=64, eos_token_ids=[dims.vocab - 1], sample=False)
        eng.prefill_batch(_prompts(dims, (9, 70, 3), seed=4))
        eng.round_batch(3)
        flags = 0 if eng.prefill_tc else _lib.LSK_FLAG_NO_PREFILL_TC
        cfg = eng.arch.lsk_config(MAX_CTX, flags=flags)
        sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
        want, got = _lib.lsk_memory_plan(), _lib.lsk_memory_plan()
        _lib.check(eng._lib.lsk_plan_memory(C.byref(cfg), sms, C.byref(_lib.lsk_memory_uses(batch_seqs=3)),
                                            C.byref(want)))
        _lib.check(eng._lib.lsk_memory_in_use(eng._h, C.byref(got)))
        fields = [f for f, _ in _lib.lsk_memory_plan._fields_]
        assert [getattr(got, f) for f in fields] == [getattr(want, f) for f in fields]
    finally:
        eng.close()

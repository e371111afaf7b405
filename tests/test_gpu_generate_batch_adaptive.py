"""GPU: confidence-threshold drafting in batches (`lsk_round_batch_adaptive` /
`Engine.round_batch_adaptive`).

On tiny-mha, tiny-gqa, a head_dim-64 model, a two-layer Llama-2-7B-width model and a two-layer model
with Llama 3's 128256-token vocabulary, greedy and sampled:
1. every active sequence's rounds equal `round_adaptive(d_seq[s], t)` of that sequence alone, every
   field and the confidences, for (B, D) in (2, 7), (3, 4), (4, 3), (8, 1), at thresholds 0, 1 and two
   quantiles of the model's own confidences, with per-sequence draft limits and a sequence that stops
   early on EOS (then inactive); its committed K/V rows in the first and last layer equal the solo
   run's; at threshold 0 the rounds equal `round_batch(D, d_seq, active)`; the stop rule is exercised
   (sequences of one round stop at different drafts, and rounds skip draft steps);
2. in graph mode the skipped draft steps do not run (layer-0 K rows of every slot stay untouched),
   rows of a stopped sequence are written while another drafts on, and eager and no-PDL engines give
   the same rounds;
3. fixed batched, adaptive batched and solo adaptive rounds of one (E, d, B) shape alternate on one
   engine, greedy and sampled, and each matches a fresh engine (graph keys);
4. refusals leave the engine usable;
5. the memory the engine holds after an adaptive batch is the plan with adaptive + batch_seqs."""
import ctypes as C
import math

import pytest
import torch

from layerskip_b200 import _lib
from layerskip_b200.engine import batch_slot_positions
from oracle import llama_oracle as orc
from tests.test_gpu_score import _dims, _engine, _ids

pytestmark = pytest.mark.gpu

MAX_CTX = 2048
ROUNDS = 6
LENGTHS = (200, 1, 65, 2, 64, 17, 63, 5)
# name: dims, exit, damping alpha of layers >= the exit
ARCHS = {
    "tiny-mha": (_dims(512, 256, 704, 4, 2, 2, 128), 2, 0.1),
    "tiny-gqa": (_dims(640, 512, 1408, 6, 4, 2, 128), 3, 0.1),
    "hd64": (_dims(512, 256, 704, 3, 4, 2, 64), 1, 0.1),
    "llama2-7b-l2": (_dims(32000, 4096, 11008, 2, 32, 32, 128), 1, 0.3),
    "vocab128k-l2": (_dims(128256, 3072, 8192, 2, 24, 8, 128, 500000.0), 1, 0.3),
}
BATCHES = ((2, 7), (3, 4), (4, 3), (8, 1))     # (B, D): B * (D + 1) <= 16
SAMPLING = dict(sample=True, temperature=0.8, top_k=0, top_p=0.95)

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


def _begin(eng, E, eos, sample, seed):
    eng.begin(exit_layer=E, max_steps=256, eos_token_ids=eos, seed=seed,
              **(SAMPLING if sample else dict(sample=False)))


def _seeds(B, base):
    return [base + 7919 * s for s in range(B)]


def _d_seq(B, D, r):
    """Most sequences may draft D tokens; every third one, in turn, D // 2."""
    return [D // 2 if (s + r) % 3 == 2 else D for s in range(B)]


def _run_batch(eng, E, prompts, seeds, D, eos, sample, t, rounds=ROUNDS, schedule=None):
    """Batched rounds, adaptive at threshold t (None: fixed `round_batch`); a sequence whose output
    reaches an EOS id turns inactive.  `schedule` replays the (d_seq, active) of an earlier trace.
    Returns [(d_seq, active, outs)] and the committed lengths."""
    B = len(prompts)
    _begin(eng, E, eos, sample, 12345)
    assert eng.prefill_batch(prompts, seeds if sample else None) == batch_slot_positions(MAX_CTX, B)
    done = [False] * B
    trace = []
    for r in range(rounds):
        d_seq, active = schedule[r] if schedule else (_d_seq(B, D, r), [not x for x in done])
        outs = eng.round_batch(D, d_seq, active) if t is None else eng.round_batch_adaptive(D, t, d_seq, active)
        trace.append((d_seq, active, outs))
        for s, o in enumerate(outs):
            if active[s] and any(x in eos for x in o.emitted):
                done[s] = True
    lens = [len(p) - 1 + sum(len(outs[s].emitted) for _d, _a, outs in trace) for s, p in enumerate(prompts)]
    return trace, lens


def _kv(eng, dims, pos0, count):
    if count == 0:
        return []
    return [eng.debug_kv_rows(w, l, 0, pos0, count) for w in "kv" for l in (0, dims.layers - 1)]


def _check_against_solo(eng, dims, E, prompts, seeds, eos, sample, t, trace, lens):
    slot = batch_slot_positions(MAX_CTX, len(prompts))
    batch_kv = [_kv(eng, dims, s * slot, lens[s]) for s in range(len(prompts))]
    for s, p in enumerate(prompts):
        _begin(eng, E, eos, sample, seeds[s])
        eng.prefill(p)
        kv_len = len(p) - 1
        for r, (d_seq, active, outs) in enumerate(trace):
            o = outs[s]
            if not active[s]:
                assert (o.n_drafted, o.n_matches, o.emitted, o.kv_len) == (0, 0, [], kv_len), (s, r)
                continue
            want = eng.round_adaptive(d_seq[s], t)
            assert _fields(o) + (o.draft_confidence,) == _fields(want) + (want.draft_confidence,), \
                (t, s, r, d_seq[s])
            kv_len = want.kv_len
        assert kv_len == lens[s]
        solo_kv = _kv(eng, dims, 0, lens[s])
        assert all(torch.equal(a, b) for a, b in zip(batch_kv[s], solo_kv)), f"t={t}: slot {s}: K/V rows differ"


def _check_stop_rule(trace, t, eos):
    for d_seq, active, outs in trace:
        for s, r in enumerate(outs):
            if not active[s]:
                continue
            c = r.draft_confidence
            assert len(c) == r.n_drafted <= d_seq[s] and all(0.0 <= x <= 1.0 for x in c)
            for i in range(r.n_drafted - 1):
                assert c[i] >= t and r.draft[i] not in eos
            if r.n_drafted:
                assert c[-1] < t or r.draft[-1] in eos or r.n_drafted == d_seq[s]


def _first_token(eng, E, prompt, D, eos, sample, seed):
    """The first token a solo round of D drafts emits: as an EOS id it ends that sequence in its first
    batched round (the same draws pick it again)."""
    _begin(eng, E, eos, sample, seed)
    eng.prefill(prompt)
    return eng.round(D).emitted[0]


def _quantiles(trace):
    conf = sorted(c for _d, a, outs in trace for s, o in enumerate(outs) if a[s] for c in o.draft_confidence)
    return [conf[len(conf) // 10], conf[len(conf) // 4]]


CASES = [(name, B, D, sample) for name in ARCHS for (B, D) in BATCHES for sample in (False, True)]


@pytest.mark.parametrize("name,B,D,sample", CASES,
                         ids=[f"{n}-B{b}-D{d}-{'sampled' if s else 'greedy'}" for n, b, d, s in CASES])
def test_rounds_equal_solo_adaptive_rounds(name, B, D, sample):
    dims, _sd, eng = _setup(name)
    E = ARCHS[name][1]
    prompts = [_ids(dims.vocab, n, 100 * B + j) for j, n in enumerate(LENGTHS[:B])]
    seeds = _seeds(B, 1000 * B + int(sample))
    eos = [dims.vocab - 1]
    eos.append(_first_token(eng, E, prompts[0], D, eos, sample, seeds[0]))
    zero, lens = _run_batch(eng, E, prompts, seeds, D, eos, sample, 0.0)
    assert not zero[1][1][0], "the first sequence was meant to stop on EOS in its first round"
    fixed, _ = _run_batch(eng, E, prompts, seeds, D, eos, sample, None, schedule=[x[:2] for x in zero])
    assert [[_fields(o) for o in outs] for _d, _a, outs in zero] == \
        [[_fields(o) for o in outs] for _d, _a, outs in fixed], "threshold 0 is not round_batch"
    _check_against_solo(eng, dims, E, prompts, seeds, eos, sample, 0.0, zero, lens)
    split = skipped = False
    for t in [1.0] + _quantiles(zero):
        trace, lens = _run_batch(eng, E, prompts, seeds, D, eos, sample, t)
        _check_stop_rule(trace, t, eos)
        _check_against_solo(eng, dims, E, prompts, seeds, eos, sample, t, trace, lens)
        for d_seq, active, outs in trace:
            live = [(d_seq[s], o.n_drafted) for s, o in enumerate(outs) if active[s]]
            # a sequence stopped by its confidence while another in the round drafted more
            split |= any(n < d and any(m > n for _, m in live) for d, n in live)
            # no active sequence reached the full D although one was allowed to: steps were skipped
            skipped |= any(d == D for d, _ in live) and max(n for _, n in live) < D
    # (sequence 0 ends in round 0, so a batch of two has one round with two active sequences)
    if D >= 3:
        assert skipped and (split or B == 2), f"stop rule not exercised (split {split}, skipped {skipped})"


@pytest.mark.parametrize("sample", (False, True), ids=("greedy", "sampled"))
def test_skipped_steps_do_not_run_and_eager_and_no_pdl_agree(sample):
    name = "tiny-gqa"
    dims, sd, eng = _setup(name)
    E, B, D = ARCHS[name][1], 3, 4
    slot = batch_slot_positions(MAX_CTX, B)
    eos = [dims.vocab - 1]
    seeds = _seeds(B, 31 + int(sample))

    def fresh_prefill(base):           # prompts no other test writes rows for
        prompts = [_ids(dims.vocab, n, base + n) for n in (30, 7, 90)]
        _begin(eng, E, eos, sample, 1)
        eng.prefill_batch(prompts, seeds if sample else None)
        lens = [len(p) - 1 for p in prompts]
        return lens, [eng.debug_kv_rows("k", 0, 0, s * slot + lens[s] + 2, D - 1) for s in range(B)]

    lens, before = fresh_prefill(900 + 10 * int(sample))
    outs = eng.round_batch_adaptive(D, 1.0)
    assert all(o.n_drafted == 1 and o.draft_confidence[0] < 1.0 for o in outs)
    for s in range(B):
        assert torch.equal(eng.debug_kv_rows("k", 0, 0, s * slot + lens[s] + 2, D - 1), before[s]), s
    # sequence 1 drafts on: every sequence's later rows are written, the stopped ones' included
    lens, before = fresh_prefill(950 + 10 * int(sample))
    outs = eng.round_batch_adaptive(D, 0.0, d_seq=[1, D, 1])
    assert [o.n_drafted for o in outs][::2] == [1, 1] and outs[1].n_drafted >= 2
    for s in range(B):
        assert not torch.equal(eng.debug_kv_rows("k", 0, 0, s * slot + lens[s] + 2, D - 1), before[s]), s

    prompts = [_ids(dims.vocab, n, 300 + n) for n in (200, 1, 65)]
    eos2 = eos + [_first_token(eng, E, prompts[0], D, eos, sample, seeds[0])]
    zero, _ = _run_batch(eng, E, prompts, seeds, D, eos2, sample, 0.0)
    thresholds = [0.3] + _quantiles(zero)
    ref = []
    for t in thresholds:
        trace, lens = _run_batch(eng, E, prompts, seeds, D, eos2, sample, t)
        ref.append(([[_fields(o) + (o.draft_confidence,) for o in outs] for _d, _a, outs in trace],
                    [_kv(eng, dims, s * slot, lens[s]) for s in range(B)]))
    for kw in (dict(use_graph=False), dict(use_pdl=False)):
        other = _engine(dims, sd, MAX_CTX, **kw)
        try:
            for t, (want, want_kv) in zip(thresholds, ref):
                trace, lens = _run_batch(other, E, prompts, seeds, D, eos2, sample, t)
                assert [[_fields(o) + (o.draft_confidence,) for o in outs] for _d, _a, outs in trace] == want, (kw, t)
                kv = [_kv(other, dims, s * slot, lens[s]) for s in range(B)]
                assert all(torch.equal(a, b) for x, y in zip(kv, want_kv) for a, b in zip(x, y)), (kw, t)
        finally:
            other.close()


def _kinds(eng, dims, E, prompts, seeds, D, t, sample):
    """Four rounds each of a fixed batch, an adaptive batch and a solo adaptive generation of one shape."""
    eos = [dims.vocab - 1]
    out = []
    for kind in ("fixed", "adaptive", "solo"):
        _begin(eng, E, eos, sample, seeds[0])
        if kind == "solo":
            eng.prefill(prompts[0])
            out.append([_fields(r) + (r.draft_confidence,) for r in (eng.round_adaptive(D, t) for _ in range(4))])
            continue
        eng.prefill_batch(prompts, seeds if sample else None)
        rounds = (eng.round_batch(D) if kind == "fixed" else eng.round_batch_adaptive(D, t) for _ in range(4))
        out.append([[_fields(o) + (o.draft_confidence,) for o in outs] for outs in rounds])
    return out


def test_fixed_adaptive_and_solo_rounds_of_one_shape_keep_their_graphs():
    name = "tiny-mha"
    dims, sd, eng = _setup(name)
    E, D = ARCHS[name][1], 3
    prompts = [_ids(dims.vocab, n, 500 + n) for n in (20, 40, 9)]
    seeds = _seeds(3, 5)
    # one engine: greedy, sampled, greedy again, each at two thresholds (one graph serves both)
    got = [((s, t), _kinds(eng, dims, E, prompts, seeds, D, t, s)) for s in (False, True, False) for t in (0.3, 0.05)]
    fresh = {}
    for s in (True, False):
        for t in (0.05, 0.3):
            other = _engine(dims, sd, MAX_CTX)
            try:
                fresh[(s, t)] = _kinds(other, dims, E, prompts, seeds, D, t, s)
            finally:
                other.close()
    for key, runs in got:
        assert runs == fresh[key], key
    assert fresh[(False, 0.3)] != fresh[(True, 0.3)]


def test_refusals_leave_the_engine_usable():
    name = "tiny-mha"
    dims, _sd, eng = _setup(name)
    E = ARCHS[name][1]
    prompts = [_ids(dims.vocab, n, 600 + n) for n in (10, 20)]
    _begin(eng, E, [dims.vocab - 1], False, 1)
    with pytest.raises(_lib.LskError) as ex:
        eng.round_batch_adaptive(3, 0.5)                       # before prefill_batch
    assert ex.value.code == -3
    eng.prefill_batch(prompts)
    for t in (-0.1, 1.5, math.nan):
        with pytest.raises(_lib.LskError) as ex:
            eng.round_batch_adaptive(3, t)
        assert ex.value.code == -1
    for d, d_seq in ((-1, None), (8, None), (3, [4, 1]), (3, [-1, 1])):
        with pytest.raises(_lib.LskError) as ex:
            eng.round_batch_adaptive(d, 0.5, d_seq)
        assert ex.value.code == -1, (d, d_seq)
    outs = eng.round_batch_adaptive(3, 0.5)
    assert all(o.kv_len > len(p) - 1 and len(o.draft_confidence) == o.n_drafted for o, p in zip(outs, prompts))
    assert [o.n_drafted for o in eng.round_batch_adaptive(0, 0.5)] == [0, 0]
    # a single-sequence prefill ends the batch
    eng.prefill(prompts[0])
    with pytest.raises(_lib.LskError) as ex:
        eng.round_batch_adaptive(3, 0.5)
    assert ex.value.code == -3
    assert eng.round_adaptive(3, 0.5).n_drafted >= 1


@pytest.mark.parametrize("sample", (False, True), ids=("greedy", "sampled"))
def test_memory_in_use_is_the_plan_with_adaptive_and_batch_seqs(sample):
    name = "tiny-gqa"
    dims, sd, _ = _setup(name)
    eng = _engine(dims, sd, MAX_CTX)
    try:
        _begin(eng, 3, [dims.vocab - 1], sample, 1)
        eng.prefill_batch([_ids(dims.vocab, n, n) for n in (9, 70, 3)], [1, 2, 3] if sample else None)
        eng.round_batch_adaptive(3, 0.2)
        flags = 0 if eng.prefill_tc else _lib.LSK_FLAG_NO_PREFILL_TC
        cfg = eng.arch.lsk_config(MAX_CTX, flags=flags)
        sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
        want, got = _lib.lsk_memory_plan(), _lib.lsk_memory_plan()
        uses = _lib.lsk_memory_uses(sampling=int(sample), adaptive=1, batch_seqs=3)
        _lib.check(eng._lib.lsk_plan_memory(C.byref(cfg), sms, C.byref(uses), C.byref(want)))
        _lib.check(eng._lib.lsk_memory_in_use(eng._h, C.byref(got)))
        fields = [f for f, _ in _lib.lsk_memory_plan._fields_]
        assert [getattr(got, f) for f in fields] == [getattr(want, f) for f in fields]
    finally:
        eng.close()

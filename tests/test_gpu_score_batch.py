"""GPU: batched scoring (`lsk_score_batch` / `Engine.score_batch` / `Engine.loglikelihood_batch`).

1. equal to solo scoring bit for bit: a shuffled batch of 2 .. 1101-id sequences on a golden model
   and on 2-layer models at the 7B, 8B (GQA: pieces cut below 128 rows), llama3.2-1B (head_dim 64)
   and head_dim-32 widths, at full depth and E = 1, and E = 2 on a 4-layer model.  A sequence of more
   than max_rows + 1 ids equals `score(seq)`; a shorter one (which `score` runs on the decode route)
   equals the first n - 1 entries of `score(seq + filler)` at 40 ids, which by causality depend on
   `seq` only and take the wgmma route;
2. packing does not matter: reversed order, each sequence alone, three or more KV groups, a permuted
   page table and a repeat run give the same bits;
3. no leak between sequences, and the check can fail: changing A's first id leaves its neighbour B
   unchanged, while B scored as the tail of the single sequence A + B differs in most rows;
4. one attention launch per layer per chunk: 1024 rows of one sequence and of 64 sequences launch
   the same number of kernels;
5. `loglikelihood_batch` against `loglikelihood` (bit for bit above max_rows + 1 joined ids, within
   the oracle bounds below, exactly without the prompt pass);
6. state after a batch;
7. argument errors."""
import ctypes as C
import random

import pytest
import torch

from oracle import llama_oracle as orc
from tests import golden_util as gu
from tests.test_gpu_score import B_GOLDEN, REL_WIDTH, WIDTHS, _dims, _engine, _golden_models, _ids

pytestmark = pytest.mark.gpu

LENGTHS = (2, 3, 9, 17, 18, 19, 64, 65, 127, 128, 129, 130, 300, 1101)
FILLED = 40                      # a short sequence is compared inside a 40-id sequence (wgmma route)


def _batch(vocab, seed, lengths=LENGTHS):
    order = list(lengths)
    random.Random(seed).shuffle(order)
    return [_ids(vocab, n, seed * 1000 + i) for i, n in enumerate(order)]


def _solo(eng, seq, E):
    """What score_batch must return for `seq`: score(seq), or for a sequence short enough to take
    the decode route in score(), the first n - 1 entries of a 40-id sequence that starts with it."""
    if len(seq) > eng.max_rows + 1:
        return eng.score(seq, E)
    filler = _ids(eng.arch.vocab, FILLED - len(seq), 7 + len(seq))
    lp, gr = eng.score(seq + filler, E)
    return lp[:len(seq) - 1], gr[:len(seq) - 1]


def _assert_same(got, want, tag):
    assert len(got) == len(want), tag
    for j, ((lp, gr), (wl, wg)) in enumerate(zip(got, want)):
        assert torch.equal(lp, wl), f"{tag}: sequence {j} ({lp.numel() + 1} ids) log-probabilities differ"
        assert torch.equal(gr, wg), f"{tag}: sequence {j} ({lp.numel() + 1} ids) greedy ids differ"


def _model(name):
    if name == "golden":
        return gu.state_dict_for(_golden_models()[0])
    (v, h, i, nl, nh, nkv, hd), theta, scaling, tied, seed, _ = WIDTHS[name]
    dims = _dims(v, h, i, nl, nh, nkv, hd, theta, scaling)
    sd = orc.random_state_dict(dims, seed)
    if tied:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    return dims, sd


def _four_layer():
    dims = _dims(1000, 512, 1408, 4, 8, 4, 64)
    return dims, orc.random_state_dict(dims, 51)


# ------------------------------------------------------------------------------------------------
# 1. equal to solo scoring
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["golden", "w7b", "w8b", "l32_1b", "mha32"])
def test_score_batch_equals_solo_scoring(name):
    dims, sd = _model(name)
    eng = _engine(dims, sd, max(LENGTHS) + 8)
    try:
        seqs = _batch(dims.vocab, 3)
        for E in (-1, 1):
            got = eng.score_batch(seqs, E)
            _assert_same(got, [_solo(eng, s, E) for s in seqs], f"{name} E={E}")
    finally:
        eng.close()


def test_score_batch_early_exit_on_four_layers():
    dims, sd = _four_layer()
    eng = _engine(dims, sd, max(LENGTHS) + 8)
    try:
        seqs = _batch(dims.vocab, 4)
        _assert_same(eng.score_batch(seqs, 2), [_solo(eng, s, 2) for s in seqs], "E=2")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 2. packing does not matter
# ------------------------------------------------------------------------------------------------
def test_score_batch_is_blind_to_packing():
    dims, sd = _four_layer()
    lengths = [n for n in LENGTHS if n <= 300]
    seqs = _batch(dims.vocab, 5, lengths)
    eng = _engine(dims, sd, 1109)
    small = _engine(dims, sd, 320)            # 5 pages: the 300 + 130 + 129 + 128 ... ids need >= 3 groups
    perm = _engine(dims, sd, 1109)
    try:
        assert sum((len(s) - 1 + 63) // 64 for s in seqs) > 2 * 5
        perm.debug_set_page_table(torch.randperm((1109 + 63) // 64, generator=torch.Generator().manual_seed(8)).tolist())
        for E in (2, -1):
            base = eng.score_batch(seqs, E)
            _assert_same(eng.score_batch(seqs, E), base, f"repeat E={E}")
            _assert_same(eng.score_batch(seqs[::-1], E)[::-1], base, f"reversed E={E}")
            _assert_same([eng.score_batch([s], E)[0] for s in seqs], base, f"alone E={E}")
            _assert_same(small.score_batch(seqs, E), base, f"groups E={E}")
            _assert_same(perm.score_batch(seqs, E), base, f"page table E={E}")
    finally:
        eng.close()
        small.close()
        perm.close()


# ------------------------------------------------------------------------------------------------
# 3. no leak between sequences
# ------------------------------------------------------------------------------------------------
def test_score_batch_keeps_sequences_apart():
    dims, sd = _four_layer()
    eng = _engine(dims, sd, 1109)
    try:
        for la, lb in ((50, 60), (100, 200), (7, 300)):       # B inside A's chunk, straddling, after a short A
            a = _ids(dims.vocab, la, la)
            b = _ids(dims.vocab, lb, lb + 1)
            a2 = [(a[0] + 1) % dims.vocab or 3] + a[1:]
            base = eng.score_batch([a, b])
            changed = eng.score_batch([a2, b])
            assert torch.equal(base[1][0], changed[1][0]) and torch.equal(base[1][1], changed[1][1]), (la, lb)
            assert not torch.equal(base[0][0], changed[0][0]), "A's own rows must see its first id"
            # the check can fail: B's rows as the tail of the one sequence A + B attend to A
            joined, _ = eng.score(a + b)
            tail = joined[la:]                                 # rows predicting b[1:]
            differ = float((tail != base[1][0]).float().mean())
            print(f"MEASURED joined_rows_differ_{la}_{lb} {differ:.3f}")
            assert differ > 0.5, (la, lb, differ)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 4. one attention launch per layer per chunk
# ------------------------------------------------------------------------------------------------
def test_score_batch_launches_do_not_depend_on_the_sequence_count():
    dims, sd = _model("mha32")
    eng = _engine(dims, sd, 4096)
    try:
        one = [_ids(dims.vocab, 1025, 1)]
        many = [_ids(dims.vocab, 17, 100 + i) for i in range(64)]
        eng.score_batch(one)                                     # first-call allocations
        counts = []
        for seqs in (one, many):
            n0 = eng.launch_count
            eng.score_batch(seqs)
            counts.append(eng.launch_count - n0)
        assert counts[0] == counts[1], counts
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 5. loglikelihood_batch
# ------------------------------------------------------------------------------------------------
def _requests(vocab):
    out = []
    for i, (lc, lk) in enumerate(((1, 1), (3, 2), (10, 5), (12, 6), (30, 4), (100, 20), (5, 200), (400, 1))):
        ids = _ids(vocab, lc + lk, 900 + i)
        out.append((ids[:lc], ids[lc:]))
    return out


def test_loglikelihood_batch_matches_loglikelihood():
    dims, sd = gu.state_dict_for(_golden_models()[0])
    reqs = _requests(dims.vocab)
    eng = _engine(dims, sd, 512)
    try:
        for E in (-1, 1):
            got = eng.loglikelihood_batch(reqs, E)
            worst = 0.0
            for (ctx, cont), (ll, greedy) in zip(reqs, got):
                want = eng.loglikelihood(ctx, cont, E)
                if len(ctx) + len(cont) > eng.max_rows + 1:
                    assert (ll, greedy) == want, (len(ctx), len(cont), E)
                else:   # wgmma route here, decode route in loglikelihood: both within B_GOLDEN per token of the oracle
                    d = abs(ll - want[0])
                    worst = max(worst, d / len(cont))
                    assert d <= 2 * B_GOLDEN * len(cont), (len(ctx), len(cont), E, d)
            print(f"MEASURED short_request_per_token_delta_E{E} {worst:.4g}")
    finally:
        eng.close()


def test_loglikelihood_batch_at_width_within_oracle_bounds():
    dims, sd = _model("w8b")
    reqs = [r for r in _requests(dims.vocab) if len(r[0]) + len(r[1]) <= 17]
    w = orc.weights_from_state_dict(dims, sd)
    eng = _engine(dims, sd, 512)
    try:
        got = eng.loglikelihood_batch(reqs)
        for (ctx, cont), (ll, _) in zip(reqs, got):
            ids = ctx + cont
            with torch.inference_mode():
                logits = orc.teacher_forced_logits(w, ids[:1], ids[1:]).double()
            lp = logits.gather(1, torch.tensor(ids[1:]).view(-1, 1)).squeeze(1) - torch.logsumexp(logits, -1)
            k = len(cont)
            bound = float((REL_WIDTH * logits.abs().amax(-1))[-k:].sum())
            assert abs(ll - float(lp[-k:].sum())) <= bound, (len(ctx), k)
    finally:
        eng.close()


def test_loglikelihood_batch_without_the_prompt_pass_is_loglikelihood():
    dims, sd = gu.state_dict_for(_golden_models()[0])
    reqs = _requests(dims.vocab)
    eng = _engine(dims, sd, 512, prefill_tc=False)
    try:
        assert eng.loglikelihood_batch(reqs, 1) == [eng.loglikelihood(c, k, 1) for c, k in reqs]
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 6. state
# ------------------------------------------------------------------------------------------------
def test_score_batch_ends_the_generation_and_leaves_rounds_unchanged():
    from layerskip_b200 import _lib as L
    dims, sd = _four_layer()
    prompt = _ids(dims.vocab, 40, 12)

    def rounds(eng):
        eng.begin(2, 40, [])
        eng.prefill(prompt)
        return [eng.round(4) for _ in range(6)]

    fresh = _engine(dims, sd, 384)
    eng = _engine(dims, sd, 384)
    try:
        want = rounds(fresh)
        assert rounds(eng) == want
        eng.score_batch(_batch(dims.vocab, 6, (2, 20, 200, 300)), 2)
        for fn in (lambda: eng.round(4), eng.ar_step):
            with pytest.raises(L.LskError) as ex:
                fn()
            assert ex.value.code == -3
        assert rounds(eng) == want
    finally:
        fresh.close()
        eng.close()


# ------------------------------------------------------------------------------------------------
# 7. argument errors
# ------------------------------------------------------------------------------------------------
def test_score_batch_argument_errors():
    from layerskip_b200 import _lib as L
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    dims = _dims(512, 256, 688, 2, 8, 8, 32)
    sd = orc.random_state_dict(dims, 0)
    eng = _engine(dims, sd, 64)
    arch = LlamaArch(512, 256, 688, 2, 8, 8, 32)
    good = [[5, 6, 7], [8, 9]]

    def expect(code, needles, fn):
        with pytest.raises(L.LskError) as ex:
            fn()
        assert ex.value.code == code, (ex.value.code, str(ex.value))
        for n in needles:
            assert n in str(ex.value), str(ex.value)
        assert eng.score_batch(good)[1][0].numel() == 1          # still usable

    try:
        want = eng.score_batch(good)
        expect(-1, ["n_seqs"], lambda: eng.score_batch([]))
        expect(-1, ["sequence 1", "at least 2"], lambda: eng.score_batch([[5, 6], [7], [8, 9]]))
        expect(-6, ["sequence 2", "max_ctx"], lambda: eng.score_batch([[5, 6], [7, 8], list(range(3, 3 + 65))]))
        expect(-1, ["sequence 1", "out of range"], lambda: eng.score_batch([[5, 6], [7, 512]]))
        expect(-1, ["sequence 0", "out of range"], lambda: eng.score_batch([[-1, 6]]))
        expect(-1, ["exit_layer"], lambda: eng.score_batch(good, 3))
        lib = L.load()
        ids = (C.c_int32 * 5)(5, 6, 7, 8, 9)
        out = (C.c_float * 3)()
        for offs in ((0, 3, 3, 5), (0, 4, 3, 5)):
            off = (C.c_int32 * 4)(*offs)
            expect(-1, ["not increasing"], lambda: L.check(lib.lsk_score_batch(eng._h, ids, off, 3, -1, out, None)))
        off = (C.c_int32 * 3)(0, 3, 5)
        assert lib.lsk_score_batch(None, ids, off, 2, -1, out, None) == -1
        assert lib.lsk_score_batch(eng._h, None, off, 2, -1, out, None) == -1
        assert lib.lsk_score_batch(eng._h, ids, None, 2, -1, out, None) == -1
        assert lib.lsk_score_batch(eng._h, ids, off, 2, -1, None, None) == -1
        assert lib.lsk_score_batch(eng._h, ids, off, 2, -1, out, None) == 0    # greedy_out may be NULL
        assert torch.equal(torch.tensor(list(out)), torch.cat([w[0] for w in want]))
        _assert_same(eng.score_batch(good), want, "after the refusals")
        nopf = Engine(arch, max_ctx=64, prefill_tc=False)
        try:
            with pytest.raises(L.LskError) as ex:
                nopf.score_batch(good)
            assert ex.value.code == -1 and "prompt pass" in str(ex.value)
        finally:
            nopf.close()
        tp = Engine(arch, max_ctx=64, tp_rank=0, tp_size=2)
        try:
            with pytest.raises(L.LskError) as ex:
                tp.score_batch(good)
            assert ex.value.code == -1 and "tensor-parallel" in str(ex.value)
        finally:
            tp.close()
    finally:
        eng.close()

"""GPU: prefix-shared scoring (`lsk_score_prefixed` / `Engine.score_prefixed` and the shared-context
route of `Engine.loglikelihood_batch`).  Every check is exact (`torch.equal`) unless stated.

1. every branch equals the matching slice of `score_batch([P + B])`, and of `score(P + B)` above
   max_rows + 1 ids: prefixes of 1 .. 1000 ids (s = len(P) - 1 covers s mod 64 = 0, 1, 63 and chunk
   edges), branches of 1 .. 130 ids, three or more branches per prefix, shuffled parents and one
   branch that fills max_ctx, on a golden model and on 2-layer models at the 7B, 8B (GQA),
   llama3.2-1B and head_dim-32 widths, at full depth and E = 1, and E = 2 on a 4-layer model;
2. packing does not matter: reversed branches, each branch alone, three or more KV groups with one
   prefix split across groups, a permuted page table and a repeat run give the same bits;
3. no leak, and the check can fail: changing sibling A leaves sibling B unchanged, changing the
   prefix's first id changes every branch, and B as the tail of the one sequence P + A + B differs;
4. the launch count follows the per-group formula;
5. `loglikelihood_batch` on multiple-choice requests equals the requests one at a time, with fewer
   launches than `score_batch` of the joined sequences;
6. state after a call, and argument errors that leave the engine usable."""
import ctypes as C
import random

import pytest
import torch

from tests.test_gpu_score import _ids
from tests.test_gpu_score_batch import _engine, _four_layer, _model

pytestmark = pytest.mark.gpu

PREFIXES = (1, 2, 17, 64, 65, 66, 127, 128, 129, 300, 1000)
BRANCHES = (1, 2, 16, 17, 63, 64, 65, 130)
MAX_CTX = 1160                   # the last branch of the 1000-id prefix fills it exactly


def _workload(vocab, seed, prefixes=PREFIXES, branches=BRANCHES, per_prefix=3, fill=MAX_CTX):
    """Prefixes and shuffled (parent, ids) branches: per_prefix branches per prefix with lengths
    cycling through `branches`, plus (fill) one branch that makes the longest prefix fill max_ctx."""
    ps = [_ids(vocab, n, seed * 100 + i) for i, n in enumerate(prefixes)]
    bs, k = [], 0
    for p in range(len(ps)):
        for _ in range(per_prefix):
            bs.append((p, _ids(vocab, branches[k % len(branches)], seed * 1000 + k)))
            k += 1
    if fill:
        longest = max(range(len(ps)), key=lambda p: len(ps[p]))
        bs.append((longest, _ids(vocab, fill - len(ps[longest]), seed * 1000 + k)))
    random.Random(seed).shuffle(bs)
    return ps, bs


def _want(eng, ps, bs, E):
    """The slices of score_batch([P + B]) that score_prefixed must return."""
    full = eng.score_batch([ps[p] + b for p, b in bs], E)
    return [(lp[len(ps[p]) - 1:], gr[len(ps[p]) - 1:]) for (p, _), (lp, gr) in zip(bs, full)]


def _assert_same(got, want, tag):
    assert len(got) == len(want), tag
    for j, ((lp, gr), (wl, wg)) in enumerate(zip(got, want)):
        assert lp.numel() == wl.numel(), f"{tag}: branch {j} has {lp.numel()} entries, want {wl.numel()}"
        assert torch.equal(lp, wl), f"{tag}: branch {j} ({lp.numel()} ids) log-probabilities differ"
        assert torch.equal(gr, wg), f"{tag}: branch {j} ({lp.numel()} ids) greedy ids differ"


# ------------------------------------------------------------------------------------------------
# 1. equal to score_batch of the joined sequence
# ------------------------------------------------------------------------------------------------
def _check_against_joined(eng, ps, bs, E, tag):
    got = eng.score_prefixed(ps, bs, E)
    _assert_same(got, _want(eng, ps, bs, E), f"{tag} score_batch")
    assert max(len(ps[p]) + len(b) for p, b in bs) == eng.max_ctx
    for j, (p, b) in enumerate(bs):
        seq = ps[p] + b
        if len(seq) > eng.max_rows + 1:
            lp, gr = eng.score(seq, E)
            _assert_same([got[j]], [(lp[len(ps[p]) - 1:], gr[len(ps[p]) - 1:])], f"{tag} score branch {j}")


@pytest.mark.parametrize("name", ["golden", "w7b", "w8b", "l32_1b", "mha32"])
def test_score_prefixed_equals_the_joined_sequences(name):
    dims, sd = _model(name)
    eng = _engine(dims, sd, MAX_CTX)
    try:
        ps, bs = _workload(dims.vocab, 3)
        for E in (-1, 1):
            _check_against_joined(eng, ps, bs, E, f"{name} E={E}")
    finally:
        eng.close()


def test_score_prefixed_early_exit_on_four_layers():
    dims, sd = _four_layer()
    eng = _engine(dims, sd, MAX_CTX)
    try:
        ps, bs = _workload(dims.vocab, 4)
        _check_against_joined(eng, ps, bs, 2, "E=2")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 2. packing does not matter
# ------------------------------------------------------------------------------------------------
def test_score_prefixed_is_blind_to_packing():
    dims, sd = _four_layer()
    small_ctx = 320                                          # 5 pages
    ps, bs = _workload(dims.vocab, 5, prefixes=(1, 2, 65, 66, 128, 129, 200), per_prefix=4, fill=small_ctx)
    eng = _engine(dims, sd, 1160)
    small = _engine(dims, sd, small_ctx)
    perm = _engine(dims, sd, 1160)
    try:
        # the 200-id prefix (4 pages, partial page of 7 slots) and its 5 branches need more than 5 pages
        big = max(range(len(ps)), key=lambda p: len(ps[p]))
        assert sum(1 for p, _ in bs if p == big) == 5
        perm.debug_set_page_table(torch.randperm((1160 + 63) // 64, generator=torch.Generator().manual_seed(8)).tolist())
        for E in (2, -1):
            base = eng.score_prefixed(ps, bs, E)
            _assert_same(base, _want(eng, ps, bs, E), f"joined E={E}")
            _assert_same(eng.score_prefixed(ps, bs, E), base, f"repeat E={E}")
            _assert_same(eng.score_prefixed(ps, bs[::-1], E)[::-1], base, f"reversed E={E}")
            _assert_same([eng.score_prefixed([ps[p]], [(0, b)], E)[0] for p, b in bs], base, f"alone E={E}")
            _assert_same(small.score_prefixed(ps, bs, E), base, f"groups E={E}")
            _assert_same(perm.score_prefixed(ps, bs, E), base, f"page table E={E}")
    finally:
        eng.close()
        small.close()
        perm.close()


# ------------------------------------------------------------------------------------------------
# 3. no leak between siblings, and the prefix is seen
# ------------------------------------------------------------------------------------------------
def test_score_prefixed_keeps_siblings_apart():
    dims, sd = _four_layer()
    eng = _engine(dims, sd, 1160)
    try:
        for lp_, la, lb in ((66, 20, 30), (300, 100, 70), (129, 5, 200)):   # t = 1, 43, 0
            P = _ids(dims.vocab, lp_, lp_)
            a = _ids(dims.vocab, la, la + 1)
            b = _ids(dims.vocab, lb, lb + 2)
            c = _ids(dims.vocab, 40, 3)
            a2 = [(a[0] + 1) % dims.vocab or 3] + a[1:]
            base = eng.score_prefixed([P], [(0, a), (0, b), (0, c)])
            changed = eng.score_prefixed([P], [(0, a2), (0, b), (0, c)])
            for j in (1, 2):
                assert torch.equal(base[j][0], changed[j][0]) and torch.equal(base[j][1], changed[j][1]), (lp_, j)
            assert not torch.equal(base[0][0], changed[0][0]), "A's own rows must see its first id"
            P2 = [(P[0] + 1) % dims.vocab or 3] + P[1:]
            moved = eng.score_prefixed([P2], [(0, a), (0, b), (0, c)])
            for j in range(3):
                assert not torch.equal(base[j][0], moved[j][0]), f"branch {j} must see the prefix's first id"
            # the check can fail: B's rows as the tail of the one sequence P + A + B attend to A
            joined, _ = eng.score(P + a + b)
            tail = joined[lp_ + la - 1:]
            differ = float((tail != base[1][0]).float().mean())
            print(f"MEASURED joined_rows_differ_{lp_}_{la}_{lb} {differ:.3f}")
            assert differ > 0.5, (lp_, la, lb, differ)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 4. launch count
# ------------------------------------------------------------------------------------------------
def _chunks_launches(rows, E, complete, max_rows):
    """enqueue_prefill_chunk: embed, 7 launches per layer (norm, QKV, attention, O, norm, gate/up,
    down) and the final norm when complete; the prompt pass (not complete) stops the last layer after
    its QKV GEMM.  Scoring adds the LM head and the log-softmax kernel per max_rows slice."""
    n = 0
    for c0 in range(0, rows, 128):
        m = min(rows - c0, 128)
        n += 1 + 7 * E + 1 + 2 * ((m + max_rows - 1) // max_rows) if complete else 1 + 7 * (E - 1) + 2
    return n


def test_score_prefixed_launch_count_follows_the_formula():
    dims, sd = _model("mha32")
    eng = _engine(dims, sd, 2048)
    try:
        ps = [_ids(dims.vocab, n, 60 + n) for n in (300, 1, 65, 129)]     # t = 43, -, 0, 0
        bs = [(0, _ids(dims.vocab, 10, 1)), (1, _ids(dims.vocab, 5, 2)), (0, _ids(dims.vocab, 130, 3)),
              (2, _ids(dims.vocab, 64, 4)), (3, _ids(dims.vocab, 7, 5)), (2, _ids(dims.vocab, 3, 6)),
              (0, _ids(dims.vocab, 1, 7))]
        eng.score_prefixed(ps, bs)                                     # first-call allocations
        for E, layers in ((-1, dims.layers), (1, 1)):
            # the constants agree with score_batch's launches
            n0 = eng.launch_count
            eng.score_batch([_ids(dims.vocab, 301, 9)], E)
            assert eng.launch_count - n0 == _chunks_launches(300, layers, True, eng.max_rows)
            n0 = eng.launch_count
            eng.score_prefixed(ps, bs, E)
            prefix_rows = sum(len(p) - 1 for p in ps)
            branch_rows = sum(len(b) for _, b in bs)
            want = (_chunks_launches(prefix_rows, layers, False, eng.max_rows) + 1
                    + _chunks_launches(branch_rows, layers, True, eng.max_rows))
            assert eng.launch_count - n0 == want, (E, eng.launch_count - n0, want)
            # no copy launch when no prefix with a partial page has a second branch
            n0 = eng.launch_count
            eng.score_prefixed(ps[1:], [(p - 1, b) for p, b in bs if p != 0], E)
            want = (_chunks_launches(prefix_rows - 299, layers, False, eng.max_rows)
                    + _chunks_launches(branch_rows - 141, layers, True, eng.max_rows))
            assert eng.launch_count - n0 == want, (E, eng.launch_count - n0, want)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 5. loglikelihood_batch shares contexts
# ------------------------------------------------------------------------------------------------
def _mc_requests(vocab):
    reqs = []
    for q, (lc, n, lk) in enumerate(((650, 4, 1), (120, 4, 28), (60, 5, 8), (300, 2, 1))):
        ctx = _ids(vocab, lc, 500 + q)
        reqs += [(ctx, _ids(vocab, lk, 600 + 10 * q + j)) for j in range(n)]
    reqs.append((_ids(vocab, 40, 700), _ids(vocab, 6, 701)))            # a context of its own
    return reqs


def test_loglikelihood_batch_shares_contexts_bit_for_bit():
    dims, sd = _four_layer()
    reqs = _mc_requests(dims.vocab)
    eng = _engine(dims, sd, 1024)
    try:
        for E in (-1, 2):
            n0 = eng.launch_count
            got = eng.loglikelihood_batch(reqs, E)
            shared = eng.launch_count - n0
            assert got == [eng.loglikelihood_batch([r], E)[0] for r in reqs], E
            n0 = eng.launch_count
            eng.score_batch([c + k for c, k in reqs], E)
            joined = eng.launch_count - n0
            print(f"MEASURED loglikelihood_batch_launches_E{E} shared {shared} joined {joined}")
            assert shared < joined, (shared, joined)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 6. state and argument errors
# ------------------------------------------------------------------------------------------------
def test_score_prefixed_ends_the_generation_and_leaves_rounds_unchanged():
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
        ps, bs = _workload(dims.vocab, 6, prefixes=(2, 66, 200), branches=(3, 40, 100), fill=384)
        eng.score_prefixed(ps, bs, 2)
        assert eng.last_device_ms > 0
        for fn in (lambda: eng.round(4), eng.ar_step):
            with pytest.raises(L.LskError) as ex:
                fn()
            assert ex.value.code == -3
        assert rounds(eng) == want
    finally:
        fresh.close()
        eng.close()


def test_score_prefixed_argument_errors():
    from layerskip_b200 import _lib as L
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    from tests.test_gpu_score import _dims
    from oracle import llama_oracle as orc
    dims = _dims(512, 256, 688, 2, 8, 8, 32)
    sd = orc.random_state_dict(dims, 0)
    eng = _engine(dims, sd, 64)
    arch = LlamaArch(512, 256, 688, 2, 8, 8, 32)
    ps, bs = [[5, 6, 7], [8]], [(1, [9, 10]), (0, [11])]

    def expect(code, needles, fn):
        with pytest.raises(L.LskError) as ex:
            fn()
        assert ex.value.code == code, (ex.value.code, str(ex.value))
        for n in needles:
            assert n in str(ex.value), str(ex.value)
        _assert_same(eng.score_prefixed(ps, bs), want, "still usable")

    try:
        want = eng.score_prefixed(ps, bs)
        _assert_same(want, _want(eng, ps, bs, -1), "joined")
        expect(-1, ["n_prefixes"], lambda: eng.score_prefixed([], [(0, [1])]))
        expect(-1, ["n_branches"], lambda: eng.score_prefixed(ps, []))
        expect(-1, ["prefix", "at least 1 id"], lambda: eng.score_prefixed([[5], []], [(0, [1]), (1, [2])]))
        expect(-1, ["branch", "at least 1 id"], lambda: eng.score_prefixed(ps, [(0, [1]), (1, [])]))
        expect(-1, ["branch 1", "prefix index 2"], lambda: eng.score_prefixed(ps, [(0, [1]), (2, [2])]))
        expect(-1, ["branch 0", "prefix index -1"], lambda: eng.score_prefixed(ps, [(-1, [1]), (1, [2])]))
        expect(-1, ["prefix 1 has no branch"], lambda: eng.score_prefixed(ps, [(0, [1])]))
        expect(-6, ["branch 1", "max_ctx"], lambda: eng.score_prefixed(ps, [(0, [1]), (1, list(range(3, 3 + 64)))]))
        expect(-1, ["prefix 0", "out of range"], lambda: eng.score_prefixed([[5, 512]], [(0, [1])]))
        expect(-1, ["branch 0", "out of range"], lambda: eng.score_prefixed([[5]], [(0, [-1])]))
        expect(-1, ["exit_layer"], lambda: eng.score_prefixed(ps, bs, 3))
        lib = L.load()
        i32 = lambda v: (C.c_int32 * len(v))(*v)   # noqa: E731
        pid, poff, bid, boff, bpar = i32([5, 6, 7, 8]), i32([0, 3, 4]), i32([9, 10, 11]), i32([0, 2, 3]), i32([1, 0])
        out = (C.c_float * 3)()
        expect(-1, ["offsets[0]"], lambda: L.check(lib.lsk_score_prefixed(eng._h, pid, i32([1, 3, 4]), 2, bid, boff, bpar, 2, -1, out, None)))
        expect(-1, ["not increasing"], lambda: L.check(lib.lsk_score_prefixed(eng._h, pid, poff, 2, bid, i32([0, 2, 1]), bpar, 2, -1, out, None)))
        args = [eng._h, pid, poff, 2, bid, boff, bpar, 2, -1, out, None]
        for k in (0, 1, 2, 4, 5, 6, 9):
            bad = list(args)
            bad[k] = None
            assert lib.lsk_score_prefixed(*bad) == -1, k
        assert lib.lsk_score_prefixed(*args) == 0                     # greedy_out may be NULL
        assert torch.equal(torch.tensor(list(out)), torch.cat([w[0] for w in want]))
        _assert_same(eng.score_prefixed(ps, bs), want, "after the refusals")
        nopf = Engine(arch, max_ctx=64, prefill_tc=False)
        try:
            with pytest.raises(L.LskError) as ex:
                nopf.score_prefixed(ps, bs)
            assert ex.value.code == -1 and "prompt pass" in str(ex.value)
        finally:
            nopf.close()
        tp = Engine(arch, max_ctx=64, tp_rank=0, tp_size=2)
        try:
            with pytest.raises(L.LskError) as ex:
                tp.score_prefixed(ps, bs)
            assert ex.value.code == -1 and "tensor-parallel" in str(ex.value)
        finally:
            tp.close()
    finally:
        eng.close()

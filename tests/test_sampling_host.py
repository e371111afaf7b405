"""CPU: the host side of tests/test_gpu_sampling_kernels.py against itself, and the reason the
inverse-CDF draw claims tokens the way it does.

* Philox4x32-10 on the Random123 known answers;
* the float64 warp against the oracle's restatement of the HF warpers on rows without ties;
* the inverse-CDF check accepts an exact draw and rejects a CDF one token off;
* `scan_draw`, a numpy float32 restatement of `block_sample_index`'s block scan.  With the rule
  "thread t owns [before_t, before_t + local_t)" the fp32 intervals do not tile [0, total): a target
  in a gap is claimed by nobody and falls to the last positive token of the row, a target in an
  overlap is claimed twice.  With the rule the kernel uses, "the last thread with tokens whose
  before_t <= target", every target has exactly one owner and the pick is the inverse-CDF token."""
import numpy as np
import pytest
import torch

from oracle import llama_oracle as orc
from tests import test_gpu_sampling_kernels as sk

f32 = np.float32


def test_philox_known_answers():
    for counter, key, want in (
            ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
            ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
            ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
             "d16cfe09 94fdcceb 5001e420 24126ea1")):
        assert " ".join(f"{int(x):08x}" for x in sk.philox4x32_10(counter, key)) == want


def test_uniforms_lie_on_the_24_bit_grid_and_streams_differ():
    steps = np.arange(4096)
    u = [sk.rng_uniform(77, steps, 0, p) for p in (1, 2, 3, 4)] + [sk.rng_uniform(77, steps, 1, 1)]
    for a in u:
        assert a.min() >= 0 and a.max() < 1 and np.array_equal(a * 2 ** 24, np.rint(a * 2 ** 24))
        assert abs(a.mean() - 0.5) < 0.03
    for i in range(len(u)):
        for j in range(i):
            assert (u[i] == u[j]).mean() < 0.01 and abs(np.corrcoef(u[i], u[j])[0, 1]) < 0.08
    assert float(sk.rng_uniform(77, 5, 0, 1)) == u[0][5]
    assert float(sk.rng_uniform(77 << 32, 5, 0, 1)) != u[0][5]              # the seed's high word is keyed


@pytest.mark.parametrize("warp", [w for w in sk.WARPS if not isinstance(w[1], str)])
def test_float64_warp_equals_the_oracle_warpers_without_ties(warp):
    temperature, top_k, top_p = warp
    g = np.random.default_rng(12)
    for vocab, sigma in ((512, 1.0), (4000, 3.0)):
        row = (g.standard_normal(vocab) * sigma).astype(np.float32)
        row[g.random(vocab) < 0.05] = -np.inf
        p, keep, either = sk.warp_ref(row, temperature, top_k, top_p)
        want = torch.softmax(orc.warp_top_k_top_p(torch.from_numpy(row).double()[None] / temperature, top_k, top_p), -1)[0]
        assert np.array_equal(keep | either, (want.numpy() > 0) | either)
        if not either.any():
            assert np.abs(p - want.numpy()).max() < 1e-12


def test_tie_groups_stay_or_go_whole_in_the_float64_warp():
    row = np.random.default_rng(2).standard_normal(32000).astype(np.float32)
    tied, inside, outside = sk.plant_nucleus_ties(row, 0.6, 0.9)
    p, keep, either = sk.warp_ref(tied, 0.6, 0, 0.9)
    assert keep[inside].all() and not keep[outside].any() and not either[inside].any() and not either[outside].any()
    q = sk.softmax64(tied.astype(np.float64) / 0.6)
    ml = sk.mass_of_larger(q)
    assert ml[inside[0]] < 0.9 - 2 * sk.GATE_P and ml[inside[0]] + q[inside].sum() > 0.9 + 2 * sk.GATE_P
    assert len(set(tied[inside].tolist())) == 1 and len(set(tied[outside].tolist())) == 1
    tied, group = sk.plant_kth_tie(row, 0.7, 5)
    assert int(sk.warp_ref(tied, 0.7, 5, 1.0)[1].sum()) == 8 and sk.warp_ref(tied, 0.7, 5, 1.0)[1][group].all()


def test_draw_check_accepts_the_exact_draw_and_rejects_a_shifted_cdf():
    w = sk.draw_rows()["softmax32000"]
    u, n_edge = sk.draw_points(w, 1)
    c = np.cumsum(w.astype(np.float64))
    exact = np.minimum(np.searchsorted(c, u * c[-1], side="right"), len(w) - 1)
    excess, positive = sk.draw_excess(w, u, exact)
    assert positive.all() and excess.max() <= 0
    assert (sk.draw_excess(w, u, exact, shift=1)[0] > sk.B_DRAW).mean() > 0.5
    assert (sk.draw_excess(w, u, np.minimum(exact + 1, len(w) - 1))[0] > sk.B_DRAW).mean() > 0.5
    assert n_edge > 5 * 900


def test_chi_square_p_value():
    p = np.full(10, 0.1)
    assert sk.chi_square_p(np.full(10, 100), 1000 * p)[0] == pytest.approx(1.0)
    pval, stat, df = sk.chi_square_p(np.array([120, 80] + [100] * 8), 1000 * p)
    assert df == 9 and stat == pytest.approx(8.0) and pval == pytest.approx(0.5341, abs=1e-3)
    assert sk.chi_square_p(np.array([5, 5, 10, 980]), np.array([5.0, 5.0, 10.0, 980.0]))[2] == 1   # 5 + 5 + 10 merge


def scan_draw(w, u, claim_by_interval):
    """`block_sample_index` in numpy float32, operation for operation: per-thread serial sums of
    contiguous chunks, shuffle-up (Hillis-Steele) scan inside each warp, the same scan over the 32 warp
    totals, before_t = warp prefix + (inclusive - local).  Returns (picks, number of claiming threads
    per target).  claim_by_interval: thread t claims before_t <= target < before_t + local_t and an
    unclaimed target takes the last positive token of the row (several claims: the last thread shown);
    otherwise the last thread with tokens and before_t <= target claims."""
    vocab, n_thr = len(w), sk.THREADS
    chunk = sk.chunk_of(vocab)
    padded = np.zeros(n_thr * chunk, dtype=f32)
    padded[:vocab] = w
    padded = padded.reshape(n_thr, chunk)
    local = np.zeros(n_thr, dtype=f32)
    for j in range(chunk):
        local = local + padded[:, j]

    def warp_scan(v):                                           # v: [n_warps, 32]
        v = v.copy()
        for o in (1, 2, 4, 8, 16):
            v[:, o:] = v[:, o:] + v[:, :-o].copy()
        return v

    incl = warp_scan(local.reshape(32, 32))
    totals = incl[:, 31].copy()
    ti = warp_scan(totals[None, :])[0]
    warp_before = ti - totals
    total = ti[31]
    before = (warp_before[:, None] + (incl - local.reshape(32, 32))).reshape(-1)
    target = np.asarray(u, dtype=f32) * total
    has = local > 0
    ge = has[None, :] & (target[:, None] >= before[None, :])
    claims = ge & (target[:, None] < (before + local)[None, :]) if claim_by_interval else ge
    n_claims = claims.sum(1) if claim_by_interval else np.minimum(ge.sum(1), 1)
    owner = np.where(claims.any(1), n_thr - 1 - np.argmax(claims[:, ::-1], axis=1), -1)
    last_positive = int(np.nonzero(w > 0)[0][-1])
    picks = np.empty(len(target), dtype=np.int64)
    for i, t in enumerate(owner):
        if t < 0:
            picks[i] = last_positive
            continue
        run = np.cumsum(np.concatenate([[before[t]], padded[t]]).astype(f32), dtype=f32)[1:]
        hit = np.nonzero(target[i] < run)[0]
        in_chunk = np.nonzero(padded[t] > 0)[0]
        picks[i] = t * chunk + (hit[0] if len(hit) else (in_chunk[-1] if not claim_by_interval else chunk - 1))
    return np.minimum(picks, vocab - 1), n_claims


@pytest.mark.parametrize("vocab", [32000, 128256])
def test_interval_claims_leave_gaps_and_the_last_owner_rule_does_not(vocab):
    w = sk.draw_rows()[f"softmax{vocab}"]
    u = sk.boundary_grid(w, np.arange(sk.chunk_of(vocab), vocab, sk.chunk_of(vocab)))
    old, n_claims = scan_draw(w, u, claim_by_interval=True)
    gaps, overlaps = int((n_claims == 0).sum()), int((n_claims > 1).sum())
    excess, _ = sk.draw_excess(w, u, old)
    print(f"vocab {vocab}: {len(u)} boundary targets, {gaps} unclaimed, {overlaps} claimed twice; "
          f"worst excess {excess.max():.3g} x 2^-24 total")
    assert gaps >= 1 and overlaps >= 1
    assert (excess[n_claims == 0] > sk.B_DRAW).all()
    assert np.median(excess[n_claims == 0]) > 1e4 * sk.B_DRAW               # the far end of the vocabulary
    new, one = scan_draw(w, u, claim_by_interval=False)
    assert (one == 1).all()
    excess, positive = sk.draw_excess(w, u, new)
    assert positive.all() and excess.max() <= sk.B_DRAW

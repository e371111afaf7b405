"""GPU: the sampling kernels alone (`csrc/sampling.cuh`) against float64 references.

a. `lsk_test_draw`: `block_sample_index` returns the token the inverse CDF names, at every thread-chunk
   boundary of the block scan, on normalised, filtered, one-hot and unnormalised rows;
b. `lsk_test_sample`: the warped rows (temperature, top-k, top-p) token by token at real vocabularies,
   with -inf entries and planted exact ties; rows near the nucleus edge repeat bit for bit;
c. `lsk_test_sample`: the drawn token is the inverse CDF of the returned row at the Philox uniform of
   (step, row_base + row, purpose); chi-square goodness of fit of 200 000 draws;
d. `lsk_test_accept_sample`: every field of a round from the Philox uniforms, EOS truncation, the
   residual draw, and the speculative-sampling identity (the emitted token follows the verifier).

The host side (Philox4x32-10, inverse-CDF check, the warp in float64, the accept rule) is plain numpy
and is tested without a GPU in tests/test_sampling_host.py.  Every case is a fixed seeded input run
once.  Bounds: DESIGN.md §7; measured values are printed as `MEASURED <name> <value>`."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

M24 = 2.0 ** -24
THREADS = 1024                                   # kSampleThreads
RNG_DRAFT, RNG_VERIFY, RNG_ACCEPT, RNG_RESID = 1, 2, 3, 4
# inverse CDF: u * total may lie outside the picked token's float64 interval by this many 2^-24 * total
# (the fp32 scan's rounding; doubled where a thread sums more than 64 tokens serially)
B_DRAW = 8.0


def draw_bound(vocab):
    return B_DRAW * (2 if -(-vocab // THREADS) > 64 else 1)

# warped probabilities on the common support: |p - p_ref| <= B_WARP_REL * p_ref + B_WARP_ABS
B_WARP_REL, B_WARP_ABS = 2e-5, 1e-8
GATE_P = 1e-5                                    # |mass of strictly larger tokens - top_p| below this: either way
TINY = 1e-37                                     # a softmax value fp32 cannot hold: either way
WARPS = [(0.6, 0, 0.9), (1.0, 0, 0.5), (0.9, 12, 0.95), (0.7, 5, 1.0), (1.3, 0, 0.0), (0.6, 50, 0.9),
         (1.0, 1, 1.0), (1.0, "V", 1.0), (0.8, "V+7", 0.9), (1.0, 0, 1.0)]


def _measured(name, value):
    print(f"MEASURED {name} {value:.4g}", flush=True)


# ------------------------------------------------------------------------------------------------
# host references (numpy, float64 unless the kernel's own fp32 step is being restated)
# ------------------------------------------------------------------------------------------------
def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., Random123): four uint32 counter words and two key words, scalars
    or arrays that broadcast; returns the four output words as uint64 arrays."""
    c = [np.asarray(x, dtype=np.uint64) for x in counter]
    k = [np.asarray(x, dtype=np.uint64) for x in key]
    m32 = np.uint64(0xFFFFFFFF)
    s32 = np.uint64(32)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> s32) ^ c[1] ^ k[0], p1 & m32, (p0 >> s32) ^ c[3] ^ k[1], p0 & m32]
        k = [(k[0] + np.uint64(0x9E3779B9)) & m32, (k[1] + np.uint64(0xBB67AE85)) & m32]
    return c


def rng_uniform(seed, step, row, purpose):
    """The kernels' `rng_uniform`: counter (step, row, purpose, 0x4c534b), key (seed low, seed high),
    u = (first word >> 8) * 2^-24, as float64 (exact)."""
    x = philox4x32_10((step, row, purpose, 0x4C534B), (seed & 0xFFFFFFFF, seed >> 32))[0]
    return (x >> np.uint64(8)).astype(np.float64) * M24


def draw_excess(w, u, picks, shift=0):
    """How far u * total lies outside the picked token's interval of the float64 CDF of w, in units of
    2^-24 * total (<= 0: inside), and whether the picked weight is positive.  `shift` plants an error:
    the CDF of the row moved by that many tokens."""
    w = np.roll(np.asarray(w, dtype=np.float64), shift)
    picks = np.asarray(picks, dtype=np.int64)
    c = np.cumsum(w)
    total = c[-1]
    lo = np.where(picks > 0, c[np.maximum(picks - 1, 0)], 0.0)
    x = np.asarray(u, dtype=np.float64) * total
    return np.maximum(lo - x, x - c[picks]) / (M24 * total), w[picks] > 0


def chunk_of(vocab):
    return -(-vocab // THREADS)


def boundary_grid(w, positions):
    """The five grid points k * 2^-24 nearest the float64 CDF of w in front of each token position."""
    c = np.cumsum(np.asarray(w, dtype=np.float64))
    k0 = np.rint(c[np.asarray(positions) - 1] / c[-1] * 2.0 ** 24).astype(np.int64)
    k = (k0[:, None] + np.arange(-2, 3)[None, :]).ravel()
    return np.unique(np.clip(k, 0, 2 ** 24 - 1)).astype(np.float64) * M24


def draw_points(w, seed):
    """The u values of one row: both ends, every thread-chunk boundary (every token boundary up to
    vocab 1025), 65 536 seeded random grid points."""
    vocab = len(w)
    chunk = chunk_of(vocab)
    pos = np.arange(1, vocab) if vocab <= 1025 else np.arange(chunk, vocab, chunk)
    rnd = np.random.default_rng(seed).integers(0, 2 ** 24, 65536).astype(np.float64) * M24
    edge = np.concatenate([[0.0, 1.0 - M24], boundary_grid(w, pos)])
    return np.concatenate([edge, rnd]), len(edge)


def softmax64(x):
    x = np.asarray(x, dtype=np.float64)
    e = np.exp(x - np.max(x))
    return e / e.sum()


def mass_of_larger(q):
    """Per token the total of the strictly larger entries of q (tied tokens share one value)."""
    order = np.argsort(-q, kind="stable")
    qs = q[order]
    cs = np.cumsum(qs)
    first = np.searchsorted(-qs, -qs, side="left")            # start of each tie group
    ml = np.where(first > 0, cs[np.maximum(first - 1, 0)], 0.0)
    out = np.empty_like(q)
    out[order] = ml
    return out


def warp_ref(logits, temperature, top_k, top_p, kernel_keep=None):
    """The HF warpers the reference calls (temperature, TopK, TopP, softmax) in float64 on one row.
    Top-k keeps every score >= the k-th largest.  The nucleus keeps a token iff the mass of the
    STRICTLY larger tokens is below top_p (HF's rule wherever scores differ; tied scores stay or go
    together, where HF's cut inside a tie depends on its sort order), and always the maximum.
    Returns (probabilities, keep, either): `either` marks tokens whose membership fp32 cannot decide
    (within GATE_P of top_p or tied in fp32 with such a token, within one fp32 ulp of the k-th score, or
    a softmax value below TINY);
    they follow `kernel_keep` when it is given, and the probabilities are renormalised accordingly."""
    s = np.asarray(logits, dtype=np.float64) / temperature
    vocab = len(s)
    keep = np.isfinite(s)
    either = np.zeros(vocab, dtype=bool)
    if 0 < top_k < vocab:
        kth = np.partition(s, vocab - top_k)[vocab - top_k]
        if np.isfinite(kth):
            keep &= s >= kth
            either |= np.isfinite(s) & (np.abs(s - kth) <= np.spacing(np.float32(abs(kth)))) & (s != kth)
    q = np.where(keep, np.exp(s - np.max(s[keep])), 0.0)
    q /= q.sum()
    either |= keep & (q < TINY)
    if 0.0 <= top_p < 1.0:
        ml = mass_of_larger(q)
        top = q == q.max()
        either |= keep & ~top & (np.abs(ml - top_p) <= GATE_P)
        # scores that differ in float64 but round to one fp32 value of (score / T - max) are a tie to
        # the kernel and cross the edge together
        s32 = np.asarray(logits, dtype=np.float32) * (np.float32(1) / np.float32(temperature))
        q32 = np.where(keep, np.exp((s32 - np.max(s32[keep])).astype(np.float64)), 0.0)
        either |= keep & ~top & ((ml < top_p) != (mass_of_larger(q32 / q32.sum()) < top_p))
        keep &= (ml < top_p) | top
    if kernel_keep is not None:
        keep = np.where(either, kernel_keep, keep)
    p = np.where(keep, q, 0.0)
    return p / p.sum(), keep, either


def host_round(p_draft, p_verify, draft, verified, eos, seed, step, kv_len0):
    """accept_sample_kernel on the host from the Philox uniforms: the fields of the round, with the
    bonus token left open on a rejection (`residual_u` then says where the residual must be drawn)."""
    d = len(draft)
    d_act = next((i + 1 for i, t in enumerate(draft) if t in eos), d)
    n, reject = 0, -1
    for i in range(d_act):
        t = draft[i]
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.minimum(np.float32(1.0), np.float32(p_verify[i, t]) / np.float32(p_draft[i, t]))
        if float(rng_uniform(seed, step, i, RNG_ACCEPT)) < float(ratio):
            n += 1
        else:
            reject = i
            break
    out = dict(n_drafted=d_act, n_matches=n, n_emitted=n + 1, kv_len=kv_len0 + n + 1, draft=list(draft[:d_act]),
               verified=list(verified[:d_act + 1]), reject=reject, residual_u=None)
    if reject >= 0:
        out["residual_u"] = float(rng_uniform(seed, step, reject, RNG_RESID))
    return out


def chi_square_p(counts, expected, min_expected=20.0):
    """p-value of Pearson's chi-square of counts against expected, bins merged in index order until
    each holds at least min_expected."""
    obs, exp, o_acc, e_acc = [], [], 0.0, 0.0
    for o, e in zip(counts, expected):
        o_acc += o
        e_acc += e
        if e_acc >= min_expected:
            obs.append(o_acc)
            exp.append(e_acc)
            o_acc = e_acc = 0.0
    obs[-1] += o_acc
    exp[-1] += e_acc
    obs, exp = np.array(obs), np.array(exp)
    stat = float(((obs - exp) ** 2 / exp).sum())
    df = len(obs) - 1
    return float(torch.special.gammaincc(torch.tensor(df / 2.0, dtype=torch.float64),
                                         torch.tensor(stat / 2.0, dtype=torch.float64))), stat, df


# ------------------------------------------------------------------------------------------------
# device calls
# ------------------------------------------------------------------------------------------------
def _dev(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def _draw(w, u):
    from layerskip_b200 import _lib as L
    wd, ud = _dev(w, torch.float32), _dev(u, torch.float32)
    picks = torch.full((len(u),), -7, dtype=torch.int32, device="cuda")
    L.check(L.load().lsk_test_draw(wd.data_ptr(), len(w), ud.data_ptr(), len(u), picks.data_ptr()))
    return picks.cpu().numpy()


def _gen(temperature=1.0, top_k=0, top_p=1.0, seed=0, eos=()):
    from layerskip_b200 import _lib as L
    g = L.lsk_generation(sample=1, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed, n_eos=len(eos))
    for i, t in enumerate(eos):
        g.eos_ids[i] = t
    return g


def _sample(logits, vocab, gen, step0=0, n_steps=1, purpose=RNG_VERIFY, row_base=0):
    """logits: float32 tensor [rows][ld] (host).  Returns (warped rows [rows][vocab], tokens [n_steps][rows])."""
    from layerskip_b200 import _lib as L
    rows, ld = logits.shape
    ld_dev = logits.cuda()
    probs = torch.full((rows, vocab), float("nan"), dtype=torch.float32, device="cuda")
    toks = torch.full((n_steps, rows), -7, dtype=torch.int32, device="cuda")
    L.check(L.load().lsk_test_sample(ld_dev.data_ptr(), rows, vocab, ld, C.byref(gen), step0, n_steps, purpose,
                                     row_base, probs.data_ptr(), toks.data_ptr()))
    return probs.cpu().numpy(), toks.cpu().numpy()


def _accept_sample(p_draft, p_verify, draft, verified, gen, kv_len0=0, step0=0):
    """p_draft [d][V], p_verify [d+1][V] float32; draft [n_steps][d], verified [n_steps][d+1] ints.
    Returns (int32 array [n_steps][52] of lsk_round_out fields, residual scratch [V])."""
    from layerskip_b200 import _lib as L
    draft = np.ascontiguousarray(draft, dtype=np.int32)
    verified = np.ascontiguousarray(verified, dtype=np.int32)
    n_steps, d = draft.shape
    vocab = p_draft.shape[1]
    pd, pv = _dev(p_draft, torch.float32), _dev(p_verify, torch.float32)
    resid = torch.full((vocab,), float("nan"), dtype=torch.float32, device="cuda")
    out = (L.lsk_round_out * n_steps)()
    i32p = C.POINTER(C.c_int32)
    L.check(L.load().lsk_test_accept_sample(pd.data_ptr(), pv.data_ptr(), vocab, d, draft.ctypes.data_as(i32p),
                                            verified.ctypes.data_as(i32p), C.byref(gen), kv_len0, step0, n_steps,
                                            out, resid.data_ptr()))
    return np.frombuffer(out, dtype=np.int32).reshape(n_steps, 52).copy(), resid.cpu().numpy()


def _fields(row):
    """One lsk_round_out as a dict of its scalar fields and its three id lists."""
    return dict(n_drafted=int(row[0]), n_matches=int(row[1]), n_emitted=int(row[2]), kv_len=int(row[3]),
                draft=row[4:20].tolist(), emitted=row[20:36].tolist(), verified=row[36:52].tolist())


# ------------------------------------------------------------------------------------------------
# a. the draw
# ------------------------------------------------------------------------------------------------
def _softmax_row(vocab, seed, sigma=2.0):
    x = np.random.default_rng(seed).standard_normal(vocab) * sigma
    return softmax64(x).astype(np.float32)


def draw_rows():
    """name -> fp32 weight row."""
    rows = {f"softmax{v}": _softmax_row(v, v) for v in (1000, 1024, 1025, 32000, 32001, 128256)}
    base = _softmax_row(32000, 5)
    nucleus = np.where(base >= np.sort(base)[-200], base, 0).astype(np.float32)
    nucleus[:50] = 0
    nucleus[-50:] = 0
    rows["nucleus"] = nucleus                                   # > 99 % zeros, zeros at both ends
    for name, idx in (("onehot_first", 0), ("onehot_last", 31999), ("onehot_mid", 32 * 500 + 13)):
        rows[name] = np.zeros(32000, dtype=np.float32)
        rows[name][idx] = 1.0
    other = softmax64(np.log(base.astype(np.float64)) + 0.3 * np.random.default_rng(6).standard_normal(32000))
    resid = np.maximum(other - base, 0)
    rows["residual"] = (resid * (0.03 / resid.sum())).astype(np.float32)      # total 0.03, half of it zeros
    rows["total40"] = (_softmax_row(32000, 7).astype(np.float64) * 40).astype(np.float32)
    rows["partial_chunk"] = _softmax_row(33 * 1000 + 5, 8)      # chunk 33: thread 1000 holds the last 5
    return rows


@pytest.mark.parametrize("name", list(draw_rows()))
def test_draw_returns_the_inverse_cdf_token(name):
    w = draw_rows()[name]
    u, n_edge = draw_points(w, len(w))
    picks = _draw(w, u)
    assert picks.min() >= 0 and picks.max() < len(w)
    excess, positive = draw_excess(w, u, picks)
    bad = (~positive) | (excess > draw_bound(len(w)))
    _measured(f"draw_excess[{name}]", excess.max())
    print(f"{name}: {len(u)} u values ({n_edge} at boundaries), {int(bad.sum())} outside the bound "
          f"({int(bad[:n_edge].sum())} at boundaries), worst {excess.max():.3g} x 2^-24 total", flush=True)
    assert not bad.any(), (name, int(bad.sum()), float(excess.max()), u[bad][:5], picks[bad][:5])
    assert np.array_equal(_draw(w, u), picks), "the same draws differ on a repeat"
    if name.startswith("softmax"):                              # the check can fail: CDF one token off
        shifted, _ = draw_excess(w, u[n_edge:], picks[n_edge:], shift=1)
        assert (shifted > draw_bound(len(w))).mean() > 0.5


def test_draw_from_an_all_zero_row_is_token_zero():
    picks = _draw(np.zeros(32000, dtype=np.float32), np.array([0.0, 0.5, 1.0 - M24]))
    assert picks.tolist() == [0, 0, 0]


# ------------------------------------------------------------------------------------------------
# b. the warp
# ------------------------------------------------------------------------------------------------
def _resolve_k(top_k, vocab):
    return {"V": vocab, "V+7": vocab + 7}.get(top_k, top_k)


def plant_kth_tie(row, temperature, top_k):
    """Three lower-ranked tokens (first, middle and last index among them) raised to the k-th score."""
    row = row.copy()
    order = np.argsort(-row, kind="stable")
    lower = np.sort(order[top_k + 10:])
    group = [lower[0], lower[len(lower) // 2], lower[-1]]
    row[group] = row[order[top_k - 1]]
    return row, [order[top_k - 1]] + group


def plant_nucleus_ties(row, temperature, top_p):
    """Two tie groups at the nucleus edge: the first starts at least 3 * GATE_P inside top_p and its
    mass carries it at least that far beyond (HF would cut it in two; it must stay whole), the second
    follows it (every member has at least top_p above it: none stays)."""
    row = row.copy()
    q = softmax64(row.astype(np.float64) / temperature)
    order = np.argsort(-q, kind="stable")
    ml = mass_of_larger(q)[order]
    r = int(np.searchsorted(ml, top_p - 3 * GATE_P, side="left")) - 1        # last rank that far inside
    n = int(math.ceil((top_p - ml[r] + 3 * GATE_P) / q[order[r]])) + 1
    inside = order[r:r + n]
    outside = order[r + n:r + n + 4]
    row[inside] = row[order[r]]
    row[outside] = row[order[r + n]]
    return row, list(inside), list(outside)


def warp_rows(vocab, temperature, top_k, top_p, seed):
    """name -> (fp32 logits row, tie groups that must stay whole, tie groups that must go)."""
    g = np.random.default_rng(seed)
    n1 = g.standard_normal(vocab).astype(np.float32)
    rows = {"sigma1": (n1, [], []), "sigma8": ((g.standard_normal(vocab) * 8).astype(np.float32), [], [])}
    peaked = g.standard_normal(vocab).astype(np.float32)
    peaked[vocab // 3] = 20.0
    rows["peaked"] = (peaked, [], [])
    banned = n1.copy()
    banned[g.random(vocab) < 0.1] = -np.inf
    banned[[0, vocab - 1]] = -np.inf
    rows["banned"] = (banned, [], [])
    if 0 < top_k < vocab:
        kth_banned = n1.copy()
        kth_banned[np.argsort(-n1, kind="stable")[top_k - 1]] = -np.inf
        rows["kth_banned"] = (kth_banned, [], [])
        if top_k >= 3:
            few = np.full(vocab, -np.inf, dtype=np.float32)                 # fewer finite scores than k
            few[[1, vocab - 2]] = [0.5, 1.5]
            rows["few_finite"] = (few, [], [])
        tied, group = plant_kth_tie(n1, temperature, top_k)
        rows["kth_tie"] = (tied, [group] if top_p >= 1.0 else [], [])
    if top_k == 0 and 0.0 < top_p < 1.0:
        tied, inside, outside = plant_nucleus_ties(n1, temperature, top_p)
        rows["nucleus_tie"] = (tied, [inside], [outside])
    return rows


def compare_warp(got, logits, temperature, top_k, top_p):
    """Worst |p - p_ref| / (B_WARP_REL * p_ref + B_WARP_ABS) of one warped row against the float64
    reference, and the number of tokens whose membership differs outside the either-way margins."""
    got = got.astype(np.float64)
    ref, keep, either = warp_ref(logits, temperature, top_k, top_p, kernel_keep=got > 0)
    wrong = int((((got > 0) != keep) & ~either).sum())
    return float((np.abs(got - ref) / (B_WARP_REL * ref + B_WARP_ABS)).max()), wrong, int(either.sum())


@pytest.mark.parametrize("vocab", [512, 32000, 32001, 128256])
def test_warped_rows_match_float64_token_by_token(vocab):
    ld = (vocab + 15) // 16 * 16 + 16
    worst = 0.0
    for si, (temperature, top_k, top_p) in enumerate(WARPS):
        top_k = _resolve_k(top_k, vocab)
        rows = warp_rows(vocab, temperature, top_k, top_p, 1000 * vocab + si)
        logits = torch.full((len(rows), ld), 1e30)                          # pad columns must never count
        for r, (row, _, _) in enumerate(rows.values()):
            logits[r, :vocab] = torch.from_numpy(row)
        probs, toks = _sample(logits, vocab, _gen(temperature, top_k, top_p, seed=si))
        assert np.isfinite(probs).all() and (probs >= 0).all()
        assert np.abs(probs.astype(np.float64).sum(-1) - 1).max() <= 1e-5
        for r, (name, (row, whole, none)) in enumerate(rows.items()):
            tag = (vocab, temperature, top_k, top_p, name)
            ratio, wrong, either = compare_warp(probs[r], row, temperature, top_k, top_p)
            assert wrong == 0, (tag, wrong)
            assert ratio <= 1.0, (tag, ratio)
            worst = max(worst, ratio)
            assert either <= max(64, vocab // 20), (tag, either)           # the margins must not swallow the check
            assert probs[r, toks[0, r]] > 0, tag                            # drawn from the support
            for group in whole:
                assert (probs[r, group] > 0).all(), (tag, "a tie group was cut")
                assert len(set(probs[r, group].tolist())) == 1
            for group in none:
                assert (probs[r, group] == 0).all(), (tag, "a tie group beyond the nucleus stayed")
            if name == "kth_tie" and top_p >= 1.0:
                assert int((probs[r] > 0).sum()) == top_k + 3, tag        # every score >= the k-th stays
            if (top_k == 1 or top_p == 0.0) and name != "kth_tie":
                assert int((probs[r] > 0).sum()) == 1 and probs[r].max() == 1.0, tag
    _measured(f"warp_ratio[{vocab}]", worst)


def test_warp_check_can_fail():
    """Planted errors: the reference at k - 1, at a top_p 1e-3 lower, and at a temperature 0.1 % off."""
    vocab = 32000
    row = np.random.default_rng(3).standard_normal(vocab).astype(np.float32)
    logits = torch.from_numpy(row)[None, :].contiguous()
    probs, _ = _sample(logits, vocab, _gen(0.9, 12, 1.0))
    assert compare_warp(probs[0], row, 0.9, 12, 1.0)[1] == 0
    assert compare_warp(probs[0], row, 0.9, 11, 1.0)[1] == 1
    probs, _ = _sample(logits, vocab, _gen(0.6, 0, 0.9))
    ratio, wrong, _ = compare_warp(probs[0], row, 0.6, 0, 0.9)
    assert wrong == 0 and ratio <= 1.0
    assert compare_warp(probs[0], row, 0.6, 0, 0.899)[1] >= 1
    ratio_t = compare_warp(probs[0], row, 0.6006, 0, 0.9)[0]
    _measured("warp_planted_temperature_ratio", ratio_t)
    assert ratio_t > 3.0


@pytest.mark.parametrize("vocab", [32000, 128256])
def test_rows_at_the_nucleus_edge_repeat_bit_for_bit(vocab):
    """top_p set to the fp32 value of the mass above a token, so that the nucleus search compares sums
    that agree to the last bits: eight copies of the row in one launch, and the launch again, must give
    the same support and the same bits whatever order the CTAs accumulated in."""
    row = np.random.default_rng(vocab + 1).standard_normal(vocab).astype(np.float32)
    logits = torch.from_numpy(row)[None, :].repeat(8, 1).contiguous()
    q = softmax64(row.astype(np.float64) / 0.8)
    ml = np.sort(mass_of_larger(q))
    differing = 0
    for frac in (0.3, 0.5, 0.7, 0.8, 0.9, 0.95, 0.99, 0.999):
        top_p = float(np.float32(ml[int(np.searchsorted(ml, frac))]))
        gen = _gen(0.8, 0, top_p, seed=1)
        a, ta = _sample(logits, vocab, gen)
        b, tb = _sample(logits, vocab, gen)
        same = all(np.array_equal(a[0].view(np.int32), x.view(np.int32)) for x in list(a[1:]) + list(b))
        differing += not same
        assert same, (vocab, top_p, [int((x > 0).sum()) for x in list(a) + list(b)])
        assert np.array_equal(ta, tb) and len(set(ta[0].tolist())) > 1      # rows draw at their own counters
        ratio, wrong, _ = compare_warp(a[0], row, 0.8, 0, top_p)
        assert wrong == 0 and ratio <= 1.0
    assert differing == 0


# ------------------------------------------------------------------------------------------------
# c. the drawn token
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("purpose,row_base", [(RNG_DRAFT, 3), (RNG_VERIFY, 0)])
@pytest.mark.parametrize("warp", [(0.6, 0, 0.9), (1.0, 0, 1.0)])
def test_sampled_token_is_the_inverse_cdf_at_the_philox_uniform(warp, purpose, row_base):
    vocab, rows, n_steps, step0, seed = 32000, 4, 4096, 17, 0x1234567890ABCDEF
    g = torch.Generator().manual_seed(11)
    logits = torch.randn(rows, vocab, generator=g) * 2
    probs, toks = _sample(logits, vocab, _gen(*warp, seed=seed), step0, n_steps, purpose, row_base)
    steps = step0 + np.arange(n_steps)
    worst = -np.inf
    for r in range(rows):
        u = rng_uniform(seed, steps, row_base + r, purpose)
        excess, positive = draw_excess(probs[r], u, toks[:, r])
        assert positive.all() and excess.max() <= B_DRAW, (r, float(excess.max()))
        worst = max(worst, float(excess.max()))
        # the check can fail: another row's counter, the other purpose, another row base, the seed's halves swapped, the next step
        for wrong_u in (rng_uniform(seed, steps, row_base + (r + 1) % rows, purpose),
                        rng_uniform(seed, steps, row_base + r, 3 - purpose),
                        rng_uniform(seed, steps, r + 4, purpose),
                        rng_uniform((seed >> 32) | ((seed & 0xFFFFFFFF) << 32), steps, row_base + r, purpose),
                        rng_uniform(seed, steps + 1, row_base + r, purpose)):
            assert (draw_excess(probs[r], wrong_u, toks[:, r])[0] > B_DRAW).mean() > 0.5
    _measured("sample_draw_excess", worst)


def test_sampled_tokens_follow_their_row_chi_square():
    vocab, rows, n_steps, seed = 64, 16, 12500, 99
    x = (np.random.default_rng(4).standard_normal(vocab) * 1.5).astype(np.float32)
    logits = torch.from_numpy(x)[None, :].repeat(rows, 1).contiguous()
    probs, toks = _sample(logits, vocab, _gen(seed=seed), 0, n_steps, RNG_DRAFT, 0)
    p = softmax64(x)
    assert np.abs(probs.astype(np.float64) - p).max() <= 1e-6
    counts = np.bincount(toks.ravel(), minlength=vocab)
    n = rows * n_steps
    pval, stat, df = chi_square_p(counts, n * p)
    print(f"chi-square of {n} draws: {stat:.1f} on {df} degrees of freedom, p = {pval:.3g}", flush=True)
    assert pval >= 1e-4, (stat, df)
    assert chi_square_p(counts, n * np.roll(p, 1))[0] < 1e-12             # planted: the row one token off


# ------------------------------------------------------------------------------------------------
# d. accept / resample
# ------------------------------------------------------------------------------------------------
def _pair(vocab, d, seed, noise=1.0):
    g = np.random.default_rng(seed)
    base = g.standard_normal((d + 1, vocab)) * 1.5
    p_d = np.stack([softmax64(r) for r in base[:d]]).astype(np.float32)
    p_v = np.stack([softmax64(r) for r in base + noise * g.standard_normal((d + 1, vocab))]).astype(np.float32)
    return p_d, p_v


def _check_rounds(p_d, p_v, draft, verified, eos, seed, step0, kv_len0):
    out, resid = _accept_sample(p_d, p_v, draft, verified, _gen(seed=seed, eos=eos), kv_len0, step0)
    worst, rejections, last_reject = -np.inf, 0, None
    for s in range(len(draft)):
        got = _fields(out[s])
        want = host_round(p_d, p_v, draft[s].tolist(), verified[s].tolist(), eos, seed, step0 + s, kv_len0)
        n, d_act = want["n_matches"], want["n_drafted"]
        for key in ("n_drafted", "n_matches", "n_emitted", "kv_len"):
            assert got[key] == want[key], (s, key, got, want)
        bonus = got["emitted"][n]
        if want["reject"] >= 0:
            i = want["reject"]
            w = np.maximum(p_v[i] - p_d[i], np.float32(0))
            excess, positive = draw_excess(w, [want["residual_u"]], [bonus])
            assert positive[0] and excess[0] <= B_DRAW, (s, i, bonus, float(excess[0]))
            worst = max(worst, float(excess[0]))
            rejections += 1
            last_reject = w
        else:
            assert bonus == verified[s][n], (s, got)
        assert got["draft"][:d_act] == want["draft"]
        assert got["emitted"][:n + 1] == want["draft"][:n] + [bonus]
        assert got["verified"][:d_act + 1] == want["verified"][:n] + [bonus] + want["verified"][n + 1:]
    if last_reject is not None:
        assert np.array_equal(resid, last_reject)                           # max(p_v - p_d, 0), unnormalised
    return out, worst, rejections


@pytest.mark.parametrize("vocab", [64, 1000])
@pytest.mark.parametrize("d", [1, 6, 15])
def test_accept_sample_round_equals_the_host_rule(vocab, d):
    n_steps, seed, step0, kv_len0 = 512, 0xFEDCBA9876543210 + d, 5, 40
    p_d, p_v = _pair(vocab, d, 10 * vocab + d, noise=0.5)
    g = np.random.default_rng(vocab + d)
    draft = np.stack([g.choice(vocab, size=n_steps, p=softmax64(np.log(p_d[i].astype(np.float64)))) for i in range(d)], 1)
    verified = g.integers(0, vocab, (n_steps, d + 1))
    out, worst, rejections = _check_rounds(p_d, p_v, draft, verified, [], seed, step0, kv_len0)
    matches = out[:, 1]
    assert rejections > n_steps // 10
    assert matches.min() == 0 and (d == 15 or matches.max() == d)
    _measured(f"residual_draw_excess[{vocab},{d}]", worst)
    # the check can fail: the uniforms of another seed
    swapped = sum(host_round(p_d, p_v, draft[s].tolist(), verified[s].tolist(), [], seed ^ 1, step0 + s,
                             kv_len0)["n_matches"] != matches[s] for s in range(n_steps))
    assert swapped > n_steps // 10


@pytest.mark.parametrize("n_eos", [1, 8])
def test_accept_sample_truncates_the_draft_at_eos(n_eos):
    vocab, d, n_steps = 64, 6, 256
    p_d, p_v = _pair(vocab, d, 77, noise=0.3)
    eos = [60] if n_eos == 1 else [50, 51, 52, 53, 54, 55, 56, 60]
    g = np.random.default_rng(5)
    for where in (0, 3, d - 1):
        draft = g.integers(0, 50, (n_steps, d))
        draft[:, where] = eos[-1] if where else eos[0]
        draft[: n_steps // 2, d - 1] = eos[n_eos // 2]                     # a later EOS does not matter
        verified = g.integers(0, vocab, (n_steps, d + 1))
        out, _, _ = _check_rounds(p_d, p_v, draft, verified, eos, 31 + where, 0, 9)
        assert (out[:, 0] == where + 1).all() and (out[:, 1] <= where + 1).all()
        assert (out[:, 1] == where + 1).any()                               # rounds that accept the EOS itself


def test_accept_sample_equal_rows_never_reject_and_zero_mass_always_rejects():
    vocab, d, n_steps = 1000, 6, 512
    p_d, p_v = _pair(vocab, d, 3)
    g = np.random.default_rng(9)
    draft = g.integers(0, vocab, (n_steps, d))
    verified = g.integers(0, vocab, (n_steps, d + 1))
    same = np.concatenate([p_d, p_v[d:]])
    out, _, rejections = _check_rounds(p_d, same, draft, verified, [], 8, 0, 0)
    assert rejections == 0 and (out[:, 1] == d).all()
    assert (out[:, 20 + d] == verified[:, d]).all()                         # the verifier's own draw follows
    t = 123
    p_v0 = p_v.copy()
    p_v0[2, t] = 0.0
    draft[:, 2] = t
    out, _, _ = _check_rounds(p_d, p_v0, draft, verified, [], 8, 0, 0)
    assert (out[:, 1] <= 2).all() and (out[:, 1] == 2).any()
    at2 = out[:, 1] == 2
    assert (out[at2, 20 + 2] != t).all()                                    # the bonus is never the rejected token


@pytest.mark.parametrize("shift", [0.7, 4.0])
def test_speculative_sampling_emits_the_verifier_distribution(shift):
    """Draft drawn from p_d by the generation kernel, accept test and residual by the accept kernel, at
    the same seed and step: the first emitted token follows p_v and drafts are accepted with
    probability sum min(p_d, p_v)."""
    vocab, n_steps, seed = 64, 200000, 4242
    g = np.random.default_rng(21)
    x = g.standard_normal(vocab) * 1.2
    y = x + shift * g.standard_normal(vocab)
    logits = torch.tensor(np.stack([x, y]), dtype=torch.float32)
    gen = _gen(seed=seed)
    p_d, draft = _sample(logits[:1].contiguous(), vocab, gen, 0, n_steps, RNG_DRAFT, 0)
    p_v, _ = _sample(logits[[1, 1]].contiguous(), vocab, gen)
    pd64, pv64 = softmax64(logits[0].numpy()), softmax64(logits[1].numpy())
    tv = 0.5 * np.abs(pd64 - pv64).sum()
    verified = np.tile(np.array([[5, 7]]), (n_steps, 1))
    out, _ = _accept_sample(p_d, p_v, draft, verified, gen)
    assert np.array_equal(out[:, 4], draft[:, 0])
    first = out[:, 20]
    accepted = out[:, 1] == 1
    alpha = np.minimum(pd64, pv64).sum()
    z = (accepted.mean() - alpha) / math.sqrt(alpha * (1 - alpha) / n_steps)
    pval, stat, df = chi_square_p(np.bincount(first, minlength=vocab), n_steps * pv64)
    print(f"TV {tv:.3f}: acceptance {accepted.mean():.4f} vs {alpha:.4f} (z = {z:.2f}); emitted vs p_v chi-square "
          f"{stat:.1f} on {df}, p = {pval:.3g}", flush=True)
    assert abs(tv - (0.2 if shift < 1 else 0.7)) < 0.08
    assert abs(z) <= 4.0
    assert pval >= 1e-4
    assert (first[accepted] == draft[accepted, 0]).all() and (out[accepted, 21] == 7).all()
    # planted: the accept test with p_d / p_v (residual drawn on the host from the same uniforms)
    steps = np.arange(n_steps)
    t = draft[:, 0]
    u_acc = rng_uniform(seed, steps, 0, RNG_ACCEPT)
    resid_cdf = np.cumsum(np.maximum(pv64 - pd64, 0))
    host_bonus = np.minimum(np.searchsorted(resid_cdf, rng_uniform(seed, steps, 0, RNG_RESID) * resid_cdf[-1],
                                            side="right"), vocab - 1)
    right = np.where(u_acc < np.minimum(1, pv64[t] / pd64[t]), t, host_bonus)
    wrong = np.where(u_acc < np.minimum(1, pd64[t] / pv64[t]), t, host_bonus)
    assert (right == first).mean() > 0.9999                                 # the host restatement is the kernel's rule
    assert chi_square_p(np.bincount(wrong, minlength=vocab), n_steps * pv64)[0] < 1e-12

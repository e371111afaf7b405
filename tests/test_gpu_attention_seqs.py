"""GPU: the attention kernel's sequence grid alone (`lsk_test_attn_seqs`: attn_piece_kernel launched as
a batched round launches it, one piece per sequence over its own slot of the page pool, committed
lengths DevState-strided) against

1. `lsk_test_attn` of each sequence alone: bit-identical rows (DESIGN.md §3.7: a batched round
   computes every row as a round of that sequence alone);
2. test_gpu_attention.py's float64 reference, within its ROW_REL_TOL.

Layouts: groups 1, 2, 3, 4, 5, 7, 8 and 16 at head_dim 128, 64 and 32, 1 .. 16 rows per sequence,
1, 3, 4 and 8 splits.  With group 3 and 4-row sequences each sequence's 12 query rows per kv head sit
at rows 0, 12, 24, .. of the shared partials: not 16-aligned.  One launch mixes a 1-key sequence with
ones of 1100, 8192 and 32768 keys on permuted pages: some sequences' splits hold no key group while
others hold far more groups than the K/V ring (the per-row-block reload path).  Needles: every row's
own diagonal key dominates, and keys in the neighbouring slots' edge pages that would dominate it
if they were read never win."""
import ctypes as C

import pytest
import torch

from tests.test_gpu_attention import ROW_REL_TOL, _assert_rows_close, _launch, _reference

pytestmark = pytest.mark.gpu


def _launch_seqs(q, k, v, n_heads, n_kv, hd, ctx, rows, slot, splits, perm_seed=None):
    from layerskip_b200 import _lib
    lib = _lib.load()
    n = len(ctx)
    out = torch.full((n * rows, n_heads * hd), float("nan"), device="cuda", dtype=torch.bfloat16)
    pp = None
    if perm_seed is not None:
        n_pages = n * slot // 64
        order = torch.randperm(n_pages, generator=torch.Generator().manual_seed(perm_seed)).tolist()
        pp = (C.c_int32 * n_pages)(*order)
    torch.cuda.synchronize()
    _lib.check(lib.lsk_test_attn_seqs(q.data_ptr(), k.data_ptr(), v.data_ptr(), n_heads, n_kv, hd, n, rows,
                                      (C.c_int32 * n)(*ctx), slot, splits, pp, out.data_ptr()))
    torch.cuda.synchronize()
    return out


def _check(q, k, v, n_heads, n_kv, hd, ctx, rows, slot, splits, perm_seed=None):
    """The batched launch against each sequence alone (bit for bit) and the float64 reference;
    returns the launch's output [n * rows, n_heads, hd] (float64)."""
    got = _launch_seqs(q, k, v, n_heads, n_kv, hd, ctx, rows, slot, splits, perm_seed)
    worst = 0.0
    for s, c in enumerate(ctx):
        qs = q[s * rows:(s + 1) * rows].contiguous()
        ks, vs = k[s, :, :c].contiguous(), v[s, :, :c].contiguous()
        solo, _ = _launch(qs, ks, vs, n_heads, n_kv, hd, c, rows, splits, perm=perm_seed is not None, seed=s)
        mine = got[s * rows:(s + 1) * rows].double()
        assert torch.equal(mine, solo), f"sequence {s} (ctx {c}): batched rows differ from the solo launch"
        want = _reference(qs, ks, vs, n_heads, n_kv, hd, c, rows)
        g, w = mine.view(rows, n_heads, hd), want.view(rows, n_heads, hd)
        rel = float(((g - w).abs().amax(-1) / w.pow(2).mean(-1).sqrt()).max())
        worst = max(worst, rel)
        assert torch.isfinite(mine).all() and rel <= ROW_REL_TOL, (s, c, rel)
    print(f"  worst max|d| / row RMS over {len(ctx)} sequences = {worst:.4g} (bound {ROW_REL_TOL})")
    return got.double().view(len(ctx) * rows, n_heads, hd)


def _inputs(n, n_heads, n_kv, hd, rows, slot, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(n * rows, n_heads * hd, generator=g, device="cuda").to(torch.bfloat16)
    k = torch.randn(n, n_kv, slot, hd, generator=g, device="cuda").to(torch.bfloat16)
    v = torch.randn(n, n_kv, slot, hd, generator=g, device="cuda").to(torch.bfloat16)
    return q, k, v


GROUPS = (1, 2, 3, 4, 5, 7, 8, 16)
ROWS = (1, 2, 4, 5, 8, 16)
# (group, head_dim, rows per sequence, splits): every group at every row count, head_dim and split count
# cycling so that each group meets each head_dim and each split count
LAYOUTS = [(g, (128, 64, 32)[(i + j) % 3], r, (1, 3, 4, 8)[(i + 2 * j) % 4])
           for i, g in enumerate(GROUPS) for j, r in enumerate(ROWS)]
SLOT = 1280                                    # 20 pages: up to 5 key groups per split at 4 splits


@pytest.mark.parametrize("group,hd,rows,splits", LAYOUTS,
                         ids=[f"g{g}-hd{h}-r{r}-s{s}" for g, h, r, s in LAYOUTS])
def test_sequences_equal_solo_launches_and_the_reference(group, hd, rows, splits):
    n_kv = 8 if group <= 4 else 2
    n_heads = group * n_kv
    n = 16 // rows
    # lengths from the sequence's own rows to the whole slot, across page edges
    lens = (rows, 64, 65, SLOT, 700, 129, 1000, 63 + rows, 1215, 300, 2 * rows, 1279, 511, 640, 900, 77)
    ctx = [max(rows, c) for c in lens[:n]]
    q, k, v = _inputs(n, n_heads, n_kv, hd, rows, SLOT, seed=group * 100 + rows)
    _check(q, k, v, n_heads, n_kv, hd, ctx, rows, SLOT, splits, perm_seed=(group + rows) if splits != 4 else None)


@pytest.mark.parametrize("n_heads,n_kv,hd,rows,splits", [
    (32, 8, 64, 1, 4), (32, 8, 64, 1, 8), (24, 8, 128, 1, 1), (32, 8, 128, 1, 3),
])
def test_mixed_lengths_in_one_launch(n_heads, n_kv, hd, rows, splits):
    """A 1-key sequence next to ones of 1100, 8192 and 32768 keys on permuted pages: the short
    sequence's splits past the first hold no key group, the long ones' hold up to 512 (the ring
    holds 4 and is re-streamed per row block)."""
    slot = 32768
    ctx = [1, 1100, 8192, slot]
    q, k, v = _inputs(len(ctx), n_heads, n_kv, hd, rows, slot, seed=n_heads + splits)
    _check(q, k, v, n_heads, n_kv, hd, ctx, rows, slot, splits, perm_seed=splits)


@pytest.mark.parametrize("n_heads,n_kv,hd,rows", [(24, 8, 128, 4), (32, 8, 64, 2), (16, 8, 32, 4)])
def test_mixed_lengths_with_several_rows(n_heads, n_kv, hd, rows):
    slot = 32768
    ctx = [rows, 8192, 1100, slot]
    q, k, v = _inputs(len(ctx), n_heads, n_kv, hd, rows, slot, seed=7 * rows)
    _check(q, k, v, n_heads, n_kv, hd, ctx, rows, slot, 4, perm_seed=rows)


def _needles(n_heads, n_kv, hd, ctx, rows, slot):
    """Query row r (sequence s = r // rows, token t) of every head is sqrt(hd) e_r, so only component r
    of a key scores for it.  Component r is 20 at the row's own position (its last visible key), 25
    at the next token's position (a row that sees one key too many picks it), and 40 in every key of
    the last page of slot s - 1 and the first page of slot s + 1 (a wrong page view picks those).
    Random keys score ~N(0, 1)."""
    n = len(ctx)
    gen = torch.Generator(device="cuda").manual_seed(sum(ctx) + rows)
    k = torch.randn(n, n_kv, slot, hd, generator=gen, device="cuda", dtype=torch.float64)
    v = torch.randn(n, n_kv, slot, hd, generator=gen, device="cuda", dtype=torch.float64)
    q = torch.zeros(n * rows, n_heads, hd, device="cuda", dtype=torch.float64)
    for s in range(n):
        for t in range(rows):
            r, p = s * rows + t, ctx[s] - rows + t
            q[r, :, r] = hd ** 0.5
            k[s, :, p, r] = 20.0
            if t + 1 < rows:
                k[s, :, p + 1, r] = 25.0
            if s > 0:
                k[s - 1, :, slot - 64:, r] = 40.0
            if s + 1 < n:
                k[s + 1, :, :64, r] = 40.0
    bf = lambda x: x.to(torch.bfloat16)
    return bf(q.reshape(n * rows, n_heads * hd)), bf(k), bf(v)


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,rows,splits", [
    (24, 8, 128, (4, 2048, 1100, 2047), 4, 8),
    (32, 2, 128, (2048, 700), 8, 4),
    (20, 4, 64, tuple(64 * j + 1 for j in range(16)), 1, 3),
    (8, 8, 32, (5, 1984, 1985), 5, 1),
    (28, 4, 128, (1023, 8), 8, 8),
])
def test_needles_win_and_neighbouring_slots_never_do(n_heads, n_kv, hd, ctx, rows, splits):
    slot = 2048
    q, k, v = _needles(n_heads, n_kv, hd, ctx, rows, slot)
    got = _check(q, k, v, n_heads, n_kv, hd, list(ctx), rows, slot, splits, perm_seed=splits)
    group = n_heads // n_kv
    for s, c in enumerate(ctx):
        for t in range(rows):
            r, p = s * rows + t, c - rows + t
            for h in range(n_heads):
                vn = v[s, h // group, p].double()
                err = float((got[r, h] - vn).abs().max() / vn.pow(2).mean().sqrt())
                assert err <= 2 ** -6, (s, t, h, p, err)

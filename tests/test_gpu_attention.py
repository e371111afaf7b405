"""GPU: the paged split-KV attention kernel alone (through the C ABI: `lsk_test_attn`) against a
plain float64 torch restatement of HF's eager attention (transformers modeling_llama.py:187-221:
scores * head_dim^-0.5 + causal mask, softmax, probabilities rounded to bf16, P.V) on
BASELINE head layouts: 32 heads x 32 kv (Llama-2-7B), 32 x 8 (Llama-3-8B), 40 x 40 (13B), 64 x 8
(70B), head_dim 64 (llama3.2-1B) and 32 (correctness.py's tiny model); contexts that give a split
1, 2, 3 and more key groups; 1 / 7 / 9 / 16 query rows (decode blocks) and 17 .. 128 rows (the
prompt pass's launches for one chunk); permuted page tables.

Tolerance: max|d| of each (token, head) output row over that row's RMS.  An output element is
~1/sqrt(ctx), so an absolute bound would hide a row that sees one key too many or too few at long
contexts; the needle test plants keys whose score dominates by ~20, so a wrong key or a mask off
by one moves a whole row."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _reference(q, k, v, n_heads, n_kv, hd, ctx, m):
    group = n_heads // n_kv
    qf = q.double().view(m, n_heads, hd).transpose(0, 1)                # [H, m, hd]
    kf = k.double().repeat_interleave(group, 0)                         # [H, ctx, hd]
    vf = v.double().repeat_interleave(group, 0)
    scores = (qf @ kf.transpose(1, 2)) * hd ** -0.5
    pos = torch.arange(ctx - m, ctx, device=q.device)[:, None]
    scores = scores.masked_fill(torch.arange(ctx, device=q.device)[None, :] > pos, float("-inf"))
    probs = torch.softmax(scores, -1).to(torch.bfloat16).double()
    return (probs @ vf).transpose(0, 1).reshape(m, n_heads * hd)


def _launch(q, k, v, n_heads, n_kv, hd, ctx, m, splits=8, perm=False, iters=0, seed=0):
    from layerskip_b200 import _lib
    lib = _lib.load()
    out = torch.full((m, n_heads * hd), float("nan"), device="cuda", dtype=torch.bfloat16)
    n_pages = (ctx + 63) // 64
    pp = None
    if perm:
        order = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed)).tolist()
        pp = (C.c_int32 * n_pages)(*order)
    ms = C.c_float(0)
    torch.cuda.synchronize()
    _lib.check(lib.lsk_test_attn(q.data_ptr(), k.data_ptr(), v.data_ptr(), n_heads, n_kv, hd, ctx, m,
                                 splits, pp, out.data_ptr(), iters, C.byref(ms)))
    torch.cuda.synchronize()
    return out.double(), ms.value


def _run(n_heads, n_kv, hd, ctx, m, splits=8, perm=False, iters=0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed + ctx * 31 + m)
    q = torch.randn(m, n_heads * hd, generator=g, device="cuda").to(torch.bfloat16)
    k = torch.randn(n_kv, ctx, hd, generator=g, device="cuda").to(torch.bfloat16)
    v = torch.randn(n_kv, ctx, hd, generator=g, device="cuda").to(torch.bfloat16)
    got, ms = _launch(q, k, v, n_heads, n_kv, hd, ctx, m, splits, perm, iters, seed)
    return got, _reference(q, k, v, n_heads, n_kv, hd, ctx, m), ms


# max|got - want| per (token, head) row over that row's RMS; measured worst 0.0199 over every case
# here on an H100 80GB HBM3 at a 400 W power limit (DESIGN.md §7)
ROW_REL_TOL = 0.035


def _assert_rows_close(got, want, n_heads, hd):
    assert torch.isfinite(got).all()
    m = got.shape[0]
    g, w = got.view(m, n_heads, hd), want.view(m, n_heads, hd)
    rel = (g - w).abs().amax(-1) / w.pow(2).mean(-1).sqrt()
    worst = float(rel.max())
    tok, head = divmod(int(rel.argmax()), n_heads)
    print(f"  worst max|d| / row RMS = {worst:.4g} (token row {tok}, head {head})")
    assert worst <= ROW_REL_TOL, (worst, tok, head)


CASES = [
    # heads, kv, hd, ctx, m
    (32, 32, 128, 70, 1), (32, 32, 128, 70, 7), (32, 32, 128, 520, 1), (32, 32, 128, 520, 9),
    (32, 32, 128, 640, 7), (32, 32, 128, 1100, 7), (32, 32, 128, 1100, 16),
    (32, 8, 128, 520, 7), (32, 8, 128, 1100, 9), (32, 8, 128, 70, 1),
    (40, 40, 128, 1100, 7), (64, 8, 128, 520, 7), (64, 8, 128, 1100, 1),
    (32, 8, 64, 700, 9), (32, 8, 64, 70, 1), (8, 8, 32, 70, 5), (8, 8, 32, 200, 16),
    (2, 2, 128, 63, 1), (2, 2, 128, 64, 1), (2, 2, 128, 65, 2), (4, 2, 128, 9, 9),
    # 16 < m <= 128: the prompt pass's launches for one chunk at c0 = ctx - m (base length 0,
    # positions through pos_off, several row blocks, canonical output)
    (32, 32, 128, 17, 17), (32, 32, 128, 145, 17), (32, 32, 128, 320, 64), (32, 32, 128, 1152, 128),
    (32, 8, 128, 273, 17), (32, 8, 128, 192, 64), (32, 8, 128, 640, 128),
    (64, 8, 128, 145, 17), (64, 8, 128, 320, 64), (64, 8, 128, 1152, 128),
    (32, 8, 64, 300, 44), (8, 8, 32, 228, 100),
]


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,m", CASES)
def test_attention_matches_fp32_reference(n_heads, n_kv, hd, ctx, m):
    """Against `_reference`, the float64 restatement above (the test id keeps its original name)."""
    got, want, _ = _run(n_heads, n_kv, hd, ctx, m)
    _assert_rows_close(got, want, n_heads, hd)


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,m,splits", [
    (32, 32, 128, 2100, 7, 8),     # 33 key groups: 4-5 per split, the K/V ring wraps
    (32, 8, 128, 2100, 9, 8),      # ... with two row blocks re-streaming the ring
    (32, 32, 128, 1100, 7, 4), (32, 32, 128, 520, 7, 1), (32, 8, 64, 1500, 16, 2),
    (32, 32, 128, 2100, 128, 8),   # prompt chunk at c0 = 1972: one 128-row launch, 8 row blocks reload
    (64, 8, 128, 2100, 64, 3),     # prompt chunk: 4 launches of 16 tokens x 8 heads
])
def test_long_contexts_fewer_splits_and_permuted_pages(n_heads, n_kv, hd, ctx, m, splits):
    got, want, _ = _run(n_heads, n_kv, hd, ctx, m, splits=splits, perm=True, seed=5)
    _assert_rows_close(got, want, n_heads, hd)


def _needles(n_heads, n_kv, hd, ctx, m, splits):
    """q / k / v where every query row (token t, head h) has ONE planted key whose score beats every
    other key by ~20, so its output is ~ that key's v row.  Query rows sharing a kv head are basis
    vectors e_b (b = their row index in the head), so planted keys for other rows score 0.  Planted
    positions cycle through key 0, the page edge 63 / 64, the last group of every split, the
    boundary group (the rows' own) and each row's diagonal.  The key at each row's position also
    carries 25 e_b of the PREVIOUS token's rows: a row that sees one key too many outputs that v."""
    group = n_heads // n_kv
    R = group * m
    assert R <= hd
    n_groups = (ctx + 63) // 64
    last = [max(g for g in range(n_groups) if g % splits == s) * 64 + 17 for s in range(min(splits, n_groups))]
    cands = [0, 63, 64] + last + [(n_groups - 1) * 64 + 5, None]           # None: the row's diagonal
    gen = torch.Generator(device="cuda").manual_seed(ctx + m)
    sq = hd ** 0.5
    k = torch.randn(n_kv, ctx, hd, generator=gen, device="cuda", dtype=torch.float64)
    v = torch.randn(n_kv, ctx, hd, generator=gen, device="cuda", dtype=torch.float64)
    q = torch.zeros(m, n_heads, hd, device="cuda", dtype=torch.float64)
    needle = torch.zeros(m, n_heads, dtype=torch.long)
    k[:, ctx - m:] = 0.0                              # the rows' own keys: planted components only
    for t in range(m):
        p_t = ctx - m + t
        for h in range(n_heads):
            kvh, b = h // group, t * group + h % group
            q[t, h, b] = sq
            c = cands[(t * n_heads + h) % len(cands)]
            p = p_t if c is None or c > p_t else c
            needle[t, h] = p
            k[kvh, p, b] = 20.0
            if t > 0:
                k[kvh, p_t, (t - 1) * group + h % group] = 25.0
    # q_b = sqrt(hd): a planted key scores 20 after the 1/sqrt(hd) scale, random keys ~N(0, 1)
    bf = lambda x: x.to(torch.bfloat16)
    return bf(q.reshape(m, n_heads * hd)), bf(k), bf(v), needle


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,m,splits", [
    (32, 32, 128, 2100, 7, 8), (32, 8, 128, 2100, 16, 8), (64, 8, 128, 2100, 16, 3),
    (32, 32, 128, 2100, 64, 8), (32, 32, 128, 2100, 128, 8), (32, 8, 128, 2100, 32, 8),
    (8, 8, 32, 2100, 4, 8), (32, 8, 64, 2100, 16, 4),
])
def test_needles_pick_their_planted_key(n_heads, n_kv, hd, ctx, m, splits):
    """Each row's output is the v row of its planted key (a wrong key, group or page, or a mask
    off by one, replaces a whole row); ctx 2100 with permuted pages: the K/V ring wraps and, above
    16 query rows per kv head, the row blocks reload it."""
    q, k, v, needle = _needles(n_heads, n_kv, hd, ctx, m, splits)
    got, _ = _launch(q, k, v, n_heads, n_kv, hd, ctx, m, splits, perm=True, seed=9)
    _assert_rows_close(got, _reference(q, k, v, n_heads, n_kv, hd, ctx, m), n_heads, hd)
    group = n_heads // n_kv
    got = got.view(m, n_heads, hd)
    for t in range(m):
        for h in range(n_heads):
            vn = v[h // group, int(needle[t, h])].double()
            err = float((got[t, h] - vn).abs().max() / vn.pow(2).mean().sqrt())
            assert err <= 2 ** -6, (t, h, int(needle[t, h]), err)
            if t + 1 < m:                              # the next token's diagonal key stays invisible
                vx = v[h // group, ctx - m + t + 1].double()
                assert float((got[t, h] - vx).abs().max()) > 0.5, (t, h)


def test_rows_are_batch_invariant():
    """A query row computed alone is bit-identical to the same row inside a 7-row block (the
    property `speculative == autoregressive` rests on): same keys, same partition, same order."""
    from layerskip_b200 import _lib
    lib = _lib.load()
    n_heads, n_kv, hd, ctx, m = 32, 8, 128, 700, 7
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(m, n_heads * hd, generator=g, device="cuda").to(torch.bfloat16)
    k = torch.randn(n_kv, ctx, hd, generator=g, device="cuda").to(torch.bfloat16)
    v = torch.randn(n_kv, ctx, hd, generator=g, device="cuda").to(torch.bfloat16)
    out = torch.zeros(m, n_heads * hd, device="cuda", dtype=torch.bfloat16)
    _lib.check(lib.lsk_test_attn(q.data_ptr(), k.data_ptr(), v.data_ptr(), n_heads, n_kv, hd, ctx, m, 8,
                                 None, out.data_ptr(), 0, None))
    for row in (0, 3, 6):
        c1 = ctx - m + row + 1                       # keys visible to that row
        one = torch.zeros(1, n_heads * hd, device="cuda", dtype=torch.bfloat16)
        q1 = q[row:row + 1].contiguous()
        k1, v1 = k[:, :c1].contiguous(), v[:, :c1].contiguous()
        _lib.check(lib.lsk_test_attn(q1.data_ptr(), k1.data_ptr(), v1.data_ptr(), n_heads, n_kv, hd, c1, 1, 8,
                                     None, one.data_ptr(), 0, None))
        torch.cuda.synchronize()
        assert torch.equal(one[0], out[row]), row


def test_attention_latency_at_the_bench_shape():
    """Llama-2-7B, ctx 640, 7 rows (the verify block of the headline config): report the latency
    (informative; the roofline for 4.3 MB of K/V is ~0.7 us, the kernel is latency-bound)."""
    for m in (1, 7):
        _, _, ms = _run(32, 32, 128, 640, m, iters=200)
        print(f"attention 7B ctx 640 m={m}: {ms * 1e3:.2f} us per launch (back-to-back launches)")
        assert ms < 0.05

"""GPU: the attention kernel alone (`lsk_test_attn`) outside the head layouts and contexts of
test_gpu_attention.py, against the same float64 reference and row bound:

- GQA groups 3, 5, 6, 7 and 16 at head_dim 128 and 64.  The kernel stacks group x M query rows of a
  kv head in 16-row blocks, row r = (token r / group, head r % group): with a group that does not
  divide 16 one token's heads straddle two row blocks and the causal limit changes inside a block.
  Decode blocks of 1, 5, 7, 9 and 16 rows; prompt launches of 17, 80, 81 and 128 rows, which the
  engine cuts at prompt_attn_rows (80 tokens at group 3, 48 at group 5, 16 at group 16);
- 4096, 8192 and 32768 keys with 1, 3, 4 and 8 splits on permuted pages: each split walks up to 512
  key groups through its K/V ring, and the ring's mbarrier parities flip hundreds of times;
- needles (test_gpu_attention.py: one dominant planted key per row, including the last page and
  every split's last key group) at 8192 and 32768 keys;
- batch invariance at group 3 and at 8192 keys: a row alone equals that row inside a block."""
import pytest
import torch

from tests import test_gpu_attention as ta
from tests.test_gpu_attention import _assert_rows_close, _run

pytestmark = pytest.mark.gpu

GROUPS = (3, 5, 6, 7, 16)


def _layout(group, hd):
    n_kv = 2 if hd == 128 else 4
    return group * n_kv, n_kv


@pytest.mark.parametrize("hd", [128, 64])
@pytest.mark.parametrize("group", GROUPS)
def test_decode_blocks_whose_row_blocks_split_a_token(group, hd):
    n_heads, n_kv = _layout(group, hd)
    for ctx, m in ((70, 1), (700, 5), (129, 7), (700, 9), (1100, 16)):
        print(f"group {group} hd {hd} ctx {ctx} m {m}")
        got, want, _ = _run(n_heads, n_kv, hd, ctx, m)
        _assert_rows_close(got, want, n_heads, hd)


@pytest.mark.parametrize("hd", [128, 64])
@pytest.mark.parametrize("group", GROUPS)
def test_prompt_launches_across_the_row_cut(group, hd):
    """17 .. 128 token rows through launch_prompt_attention: at group 3, 81 and 128 rows cross the
    80-token cut, at group 16 every 16 tokens start a new launch."""
    n_heads, n_kv = _layout(group, hd)
    for ctx, m in ((17, 17), (145, 17), (80, 80), (400, 81), (81, 81), (1152, 128)):
        print(f"group {group} hd {hd} ctx {ctx} m {m}")
        got, want, _ = _run(n_heads, n_kv, hd, ctx, m, perm=True, seed=2)
        _assert_rows_close(got, want, n_heads, hd)


# heads, kv, hd, m at each context; every context runs at 1, 3, 4 and 8 splits
LONG_LAYOUTS = [(24, 8, 128, 7), (32, 8, 64, 16), (32, 32, 128, 1), (28, 4, 128, 9)]


@pytest.mark.parametrize("ctx", [4096, 8192, 32768])
@pytest.mark.parametrize("splits", [1, 3, 4, 8])
def test_long_contexts_on_permuted_pages(ctx, splits):
    n_heads, n_kv, hd, m = LONG_LAYOUTS[(splits + ctx // 4096) % len(LONG_LAYOUTS)]
    print(f"{n_heads}/{n_kv} hd {hd} m {m}")
    got, want, _ = _run(n_heads, n_kv, hd, ctx, m, splits=splits, perm=True, seed=6)
    _assert_rows_close(got, want, n_heads, hd)


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,m,splits", [
    (24, 8, 128, 8192, 128, 4),    # prompt chunk at c0 = 8064, group 3: launches of 80 + 48 tokens
    (32, 8, 128, 8192, 128, 8),    # group 4: launches of 48 + 48 + 32 tokens
    (40, 8, 64, 32768, 48, 4),     # group 5, head_dim 64
])
def test_prompt_chunks_at_long_contexts(n_heads, n_kv, hd, ctx, m, splits):
    got, want, _ = _run(n_heads, n_kv, hd, ctx, m, splits=splits, perm=True, seed=8)
    _assert_rows_close(got, want, n_heads, hd)


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,m,splits", [
    (24, 8, 128, 8192, 16, 8), (32, 8, 64, 8192, 16, 3), (28, 4, 128, 8192, 9, 4),
    (28, 4, 128, 32768, 16, 4), (32, 2, 128, 32768, 8, 8), (24, 8, 128, 32768, 7, 1),
])
def test_needles_at_long_contexts(n_heads, n_kv, hd, ctx, m, splits):
    """test_gpu_attention.py's needle test: planted keys at key 0, the page edge 63 / 64, the last
    key group of every split, the last page and each row's diagonal; the next token's diagonal key
    stays invisible."""
    ta.test_needles_pick_their_planted_key(n_heads, n_kv, hd, ctx, m, splits)


def _alone_equals_block(n_heads, n_kv, hd, ctx, m, rows, splits=8):
    from layerskip_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(ctx + m)
    q = torch.randn(m, n_heads * hd, generator=g, device="cuda").to(torch.bfloat16)
    k = torch.randn(n_kv, ctx, hd, generator=g, device="cuda").to(torch.bfloat16)
    v = torch.randn(n_kv, ctx, hd, generator=g, device="cuda").to(torch.bfloat16)
    out = torch.zeros(m, n_heads * hd, device="cuda", dtype=torch.bfloat16)
    _lib.check(lib.lsk_test_attn(q.data_ptr(), k.data_ptr(), v.data_ptr(), n_heads, n_kv, hd, ctx, m, splits,
                                 None, out.data_ptr(), 0, None))
    for row in rows:
        c1 = ctx - m + row + 1
        one = torch.zeros(1, n_heads * hd, device="cuda", dtype=torch.bfloat16)
        q1 = q[row:row + 1].contiguous()
        k1, v1 = k[:, :c1].contiguous(), v[:, :c1].contiguous()
        _lib.check(lib.lsk_test_attn(q1.data_ptr(), k1.data_ptr(), v1.data_ptr(), n_heads, n_kv, hd, c1, 1, splits,
                                     None, one.data_ptr(), 0, None))
        torch.cuda.synchronize()
        assert torch.equal(one[0], out[row]), (n_heads, n_kv, ctx, m, row)


@pytest.mark.parametrize("n_heads,n_kv,hd,ctx,m,rows", [
    (24, 8, 128, 700, 7, (0, 5, 6)),       # group 3: token 5's heads sit in rows 15 | 16, 17
    (24, 8, 128, 8192, 16, (0, 5, 10, 15)),
    (32, 8, 128, 8192, 7, (0, 3, 6)),
    (28, 4, 64, 8192, 9, (2, 8)),          # group 7
])
def test_rows_are_batch_invariant_at_new_groups_and_long_contexts(n_heads, n_kv, hd, ctx, m, rows):
    _alone_equals_block(n_heads, n_kv, hd, ctx, m, rows)

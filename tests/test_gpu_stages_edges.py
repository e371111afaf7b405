"""GPU: test_gpu_stages.py's stage-by-stage float64 checks, with its bounds, at layouts and contexts
outside its widths:

B. layouts (2 layers each; prompts of 2 .. 300 tokens, decode blocks of 1 / 7 / 9 / 16 rows):
   - `l32_3b`: Llama-3.2-3B (24 heads over 8 kv heads: group 3, llama3 RoPE, tied embeddings).  The
     prompt pass's attention runs 80 tokens per launch, and a 16-row block of the attention kernel
     splits one token's heads (token 5: heads 0 | 1, 2);
   - `g5_hd64` (group 5 at head_dim 64), `g7` (28 heads over 4 kv heads, hidden 3584);
   - `g16`: 32 heads over 2 kv heads at head_dim 128, the largest group that fits (232 064 of
     232 448 bytes of shared memory for a 16-token launch; 16 tokens per prompt launch);
   - `odd_k`: hidden 4128 (no wgmma prompt pass: hidden % 64 != 0; K-chunked RMSNorm with a partial
     K block), inter 11000 (zero-padded down-projection columns), vocab 32003;
   - `tiny`: hidden 96, 3 heads over 1 kv head at head_dim 32, inter 264, vocab 37 (smaller than one
     LM-head tile).
   Each width runs the sensitivity checks of test_gpu_stages.py; at `l32_3b`, `g5_hd64` and `g7` the
   attention outputs of the two heads of one token on either side of the first 16-row block boundary
   are swapped in the reference, and the next layer's K must report it.
C. long prompts: 7B width at 4096 tokens, 8B at 8192, llama3.2-1B at 32768, on permuted page tables.
   Layer-0 K/V at every position; layer-1 K/V on sampled rows (every row of the first and last
   128-token chunk, rows 63 / 64 / 127 / 128 of each 1024-token stretch and 64 random rows) from the
   engine's layer-0 K/V; decode blocks of 1, 7 and 16 rows across a page boundary near max_ctx.
   Planted: a K row rotated for position p + 1 at p = 8000."""
import random
from unittest import mock

import pytest
import torch

from tests import stage_ref as sr
from tests import test_gpu_stages as ts
from tests.test_gpu_stages import B_DECODE_L1, B_PROMPT_L1, DIRECT, _build, _decode, _kv, _prompt

pytestmark = pytest.mark.gpu

SHORT = ts.SHORT
# Layer-0 K/V of prompts of 4096 .. 32768 tokens: DIRECT with 6 ulp-or-floor units instead of 4
# (measured worst 4.59, llama3.2-1B width at 32768 tokens, position 26725; 4.13 at 4096 tokens).
# The rows past 4 units are single rows whose normalised products sit on many bf16 ties that the
# kernels' rsqrtf breaks differently: with its rstd moved by one fp32 ulp, the least identical row
# of each long prompt goes from 84-87 % to >= 99.7 % bit-identical (printed below).  More rows reach
# further into that tail.
DIRECT_LONG = dict(DIRECT, units=6.0)
# name: (vocab, hidden, inter, layers, heads, kv heads, head_dim), options (test_gpu_stages.WIDTHS)
WIDTHS = {
    "l32_3b": ((128256, 3072, 8192, 2, 24, 8, 128), dict(theta=500000.0, seed=31, prompts=SHORT, tied=True,
                                                         rope=ts.LLAMA3)),
    "g5_hd64": ((32000, 1280, 3456, 2, 20, 4, 64), dict(theta=10000.0, seed=32, prompts=SHORT, perm=True)),
    "g7": ((32000, 3584, 18944, 2, 28, 4, 128), dict(theta=1000000.0, seed=33, prompts=SHORT)),
    "g16": ((32000, 4096, 11008, 2, 32, 2, 128), dict(theta=10000.0, seed=34, prompts=SHORT)),
    "odd_k": ((32003, 4128, 11000, 2, 32, 8, 128), dict(theta=10000.0, seed=35, prompts=SHORT)),
    "tiny": ((37, 96, 264, 2, 3, 1, 32), dict(theta=10000.0, seed=36, prompts=SHORT)),
}
LONG = {
    "w7b_4k": ((32000, 4096, 11008, 2, 32, 32, 128), dict(theta=10000.0, seed=41, prompts=(4096,), perm=True)),
    "w8b_8k": ((128256, 4096, 14336, 2, 32, 8, 128), dict(theta=500000.0, seed=42, prompts=(8192,), perm=True)),
    "l32_1b_32k": ((128256, 2048, 8192, 2, 32, 8, 64), dict(theta=500000.0, seed=43, prompts=(32768,), tied=True,
                                                            rope=ts.LLAMA3, perm=True)),
}


def _built(name, table):
    with mock.patch.dict(ts.WIDTHS, {name: table[name]}):
        return _build(name)


def _report(name, worst):
    bad = worst.pop("_violations", [])
    agg = {}
    for stage, w in worst.items():
        key = " ".join(t for t in stage.split() if "=" not in t)
        agg[key] = max(agg.get(key, 0.0), w)
    for k, w in sorted(agg.items()):
        print(f"  WORST {name} {k}: {w:.4g}")
    assert not bad, "\n".join(bad)


def _split_token(group):
    """(token, head a, head b) of the first token whose heads straddle the kernel's first 16-row
    block boundary (row r = token r // group, head r % group), or None when group divides 16."""
    if 16 % group == 0:
        return None
    t = 16 // group
    return t, 16 - group * t - 1, 16 - group * t


def _swapped_heads_show(arch, eng, ref, ids, L, m):
    """After `_decode(L, m)`: the reference with the attention outputs of two heads of one token
    swapped across the row-block boundary, in every kv head, must violate the layer-1 K bound."""
    group = arch.heads // arch.kv_heads
    t, ha, hb = _split_token(group)
    pos = torch.arange(L, L + m, device="cuda")
    k_ctx, v_ctx = _kv(eng, 0, 0, L + m)
    x = ref.embed(ids[L:L + m])
    q = ref.qkv(0, x, pos)[0]
    attn = ref.attend(q, pos, k_ctx, v_ctx).view(m, arch.heads, arch.head_dim).clone()
    for kvh in range(arch.kv_heads):
        a, b = kvh * group + ha, kvh * group + hb
        attn[t, [a, b]] = attn[t, [b, a]]
    kb = ref.qkv(1, ref.layer_rest(0, x, attn.view(m, -1)), pos)[1]
    k1 = _kv(eng, 1, 0, L + m)[0][L:]
    ts._expect_violation(sr.check_rows(f"decode L={L} m={m} layer-1 K, token {t} heads {ha} / {hb} swapped",
                                       k1, kb, B_DECODE_L1, 1, L))


@pytest.mark.parametrize("name", list(WIDTHS))
def test_stages_at_new_layouts(name):
    arch, eng, ref, ids = _built(name, WIDTHS)
    worst = {}
    try:
        with torch.inference_mode():
            for n in SHORT:
                # at `tiny` (3 heads of 32 dims) row 127 one key short moves layer-1 K by only 0.044 of
                # the row RMS, under B_PROMPT_L1; its decode plants below still apply
                _prompt(arch, eng, ref, ids, n, worst, sensitivity=(n == 300 and name != "tiny"))
            for L in ts.DECODE_LENS:
                for m in ts.DECODE_ROWS:
                    if m <= eng.max_rows:
                        _decode(arch, eng, ref, ids, L, m, worst, sensitivity=(L == 60 and m == eng.max_rows))
                        # not at `tiny`: its attention moves the next layer so little that even two
                        # whole rows swapped show only 1.4x the bound in the residual
                        if (L == 60 and m == eng.max_rows and _split_token(arch.heads // arch.kv_heads)
                                and name != "tiny"):
                            _swapped_heads_show(arch, eng, ref, ids, L, m)
            if arch.vocab % 16:
                ts._padded_columns_never_win(arch, eng, ref, ids, worst)
    finally:
        eng.close()
        del ref
        torch.cuda.empty_cache()
    _report(name, worst)


def _sampled_rows(rows, seed):
    s = set(range(min(128, rows)))
    s |= set(range((rows - 1) // 128 * 128, rows))
    for base in range(0, rows, 1024):
        s |= {base + r for r in (63, 64, 127, 128) if base + r < rows}
    s |= set(random.Random(seed).sample(range(rows), 64))
    return sorted(s)


def _rstd_ulps_of_the_least_identical_row(ref, x, pos, k_eng, v_eng, k, v):
    """Print how many of the least identical row's K / V elements match the reference with its
    fp32 rstd moved by -2 .. +2 ulp (rsqrtf's error bound): the rows behind DIRECT_LONG."""
    same = ((k_eng == k).flatten(1).double().mean(1) + (v_eng == v).flatten(1).double().mean(1)) / 2
    p = int(same.argmin())
    xr, pr = x[p:p + 1], pos[p:p + 1]
    rs = ref.rstd(xr).float()
    out = []
    for d in (-2, -1, 0, 1, 2):
        r = rs.clone()
        for _ in range(abs(d)):
            r = torch.nextafter(r, torch.full_like(r, float("inf") if d > 0 else 0.0))
        _, kr, vr = ref.qkv(0, xr, pr, r.double())
        out.append(f"{d:+d} ulp: {float(((kr == k_eng[p:p + 1]).double().mean() + (vr == v_eng[p:p + 1]).double().mean()) / 2):.4f}")
    print(f"    position {p} (least identical K/V row), share identical with its rstd moved " + ", ".join(out))


def _long_prompt(arch, eng, ref, ids, n, worst, sensitivity):
    """Layer-0 K/V of every position; layer-1 K/V of the sampled rows, from the engine's layer 0."""
    eng.begin(exit_layer=-1, max_steps=8, eos_token_ids=[arch.vocab - 1])
    eng.prefill(ids[:n])
    rows = n - 1
    pos = torch.arange(rows, device="cuda")
    x = ref.embed(ids[:rows])
    k_eng, v_eng = _kv(eng, 0, 0, rows)
    q, k, v = ref.qkv(0, x, pos)
    ts._expect(sr.check_direct(f"prompt n={n} layer-0 K", k_eng, k, 0, **DIRECT_LONG), worst)
    ts._expect(sr.check_direct(f"prompt n={n} layer-0 V", v_eng, v, 0, **DIRECT_LONG), worst)
    _rstd_ulps_of_the_least_identical_row(ref, x, pos, k_eng, v_eng, k, v)
    if sensitivity:
        p = 8000
        bad = k.clone()
        bad[p] = ref.qkv(0, x[p:p + 1], pos[p:p + 1] + 1)[1][0]
        ts._expect_violation(sr.check_direct(f"layer-0 K, row {p} rotated for position {p + 1}", k_eng, bad, 0,
                                             **DIRECT_LONG))
    del k, v
    sel = torch.tensor(_sampled_rows(rows, n), device="cuda")
    print(f"    layer 1: {sel.numel()} sampled rows of {rows}")
    x1 = ref.layer_rest(0, x[sel], ref.attend(q[sel], pos[sel], k_eng, v_eng))
    _, k1, v1 = ref.qkv(1, x1, pos[sel])
    k_eng1, v_eng1 = _kv(eng, 1, 0, rows)
    ts._expect(sr.check_rows(f"prompt n={n} layer-1 K (sampled rows)", k_eng1[sel], k1, B_PROMPT_L1, 1), worst)
    ts._expect(sr.check_rows(f"prompt n={n} layer-1 V (sampled rows)", v_eng1[sel], v1, B_PROMPT_L1, 1), worst)


@pytest.mark.parametrize("name", list(LONG))
def test_stages_at_long_contexts(name):
    arch, eng, ref, ids = _built(name, LONG)
    n = LONG[name][1]["prompts"][0]
    worst = {}
    try:
        with torch.inference_mode():
            _long_prompt(arch, eng, ref, ids, n, worst, sensitivity=(n == 8192))
            # block rows L .. L + m - 1 straddle the page boundary at L + 4 (for m > 4), near max_ctx
            L = (eng.max_ctx - 80) // 64 * 64 + 60
            for m in (1, 7, 16):
                _decode(arch, eng, ref, ids, L, m, worst, sensitivity=(m == 16))
    finally:
        eng.close()
        del ref
        torch.cuda.empty_cache()
    _report(name, worst)

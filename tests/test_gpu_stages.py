"""GPU: the prompt pass and the decode layer, stage by stage, against tests/stage_ref.py — a float64
restatement of the engine's arithmetic that rounds to bf16 where the kernels do.  Tight enough to
see one wrong element, and each failure names the stage and the (layer, head, position) of its
worst element:

(a) prompt-pass K/V rows, every position of every kv head, for prompts of 2 and 17 tokens (the
    decode kernels' prompt path), 18 (smallest wgmma prompt), 129 (one 128-token chunk), 130,
    300 and 1101 (w7b / w8b).  Layer 0 isolates the RMSNorm (`rms_canon_kernel`), the QKV + RoPE
    epilogue and the page scatter; layer 1 (started from the engine's own layer-0 K/V) adds the
    prompt-pass attention launches, split-K O / down, the partial sums of `rms_canon_kernel` and
    SiLU.up, checked per (position, kv head) row;
(b) decode K/V rows of a teacher-forced block of m = 1, 7, 9, 16 rows whose positions straddle a
    page boundary: the skinny GEMM's RMSNorm prologue (resident, and K-chunked above hidden 4096)
    and QKV epilogue;
(c) the decode block's residual rows after every layer (attention, O, gate/up, down; reference
    started from the engine's own K/V) and the mma.sync LM head's logits (reference started from
    the engine's final residual); the engine's own greedy token (`LSK_DBG_ARGMAX`) is the reference
    arg-max unless the top-2 margin is within the bound; with a vocab that is not a multiple of 16
    the padded columns are never written and never win, even when every real logit is negative;
(d) sensitivity: each comparison reports a violation for a single-row / single-key error planted
    in the reference.

Weights: `oracle.random_state_dict`, with RMSNorm weights drawn around 1 so the norm weights'
rounding order is exercised.  Bounds: see DESIGN.md §7 (measured worst on an H100 80GB HBM3 at a
400 W power limit; every bound is at most 2x its measured worst).  The planted errors of (d) exceed
their bounds by the factors DESIGN.md §7 lists."""
import ctypes as C

import pytest
import torch

from oracle import llama_oracle as orc
from tests import stage_ref as sr

pytestmark = pytest.mark.gpu

# Bounds, each with its worst value measured over every width here on an H100 80GB HBM3 at a 400 W
# power limit (DESIGN.md §7).  Directly computed bf16 GEMM outputs (layer-0 K/V, prompt and decode):
# |d| <= 4 x max(1 bf16 ulp, 2^-12 x the (position, head) row's RMS) (measured worst 2.44, w70b
# prompt layer-0 K); >= 99 % of all elements bit-identical (measured >= 99.2 %) and >= 75 % of every
# position's (measured >= 86.7 %).  Most rows are bit-identical; the worst values sit in single rows
# whose products land on bf16 ties that the kernels' rsqrtf breaks differently.
DIRECT = dict(units=4.0, min_identical=0.99, min_identical_pos=0.75)
# per-row max|d| / row RMS of the downstream stages
B_PROMPT_L1 = 0.06               # layer-1 prompt K/V rows                (measured worst 0.0387)
B_DECODE_L1 = 0.06               # layer-1 decode K/V rows                (measured worst 0.0381)
B_HIDDEN = 0.06                  # decode residual rows after the last layer (measured worst 0.0377)
B_LOGITS = 1e-3                  # LM head logits from the engine's final residual (measured worst 5.4e-4)

LLAMA3 = dict(rope_scaling="llama3", rope_factor=32.0, rope_low_freq_factor=1.0,
              rope_high_freq_factor=4.0, rope_original_max_pos=8192)
SHORT = (2, 17, 18, 129, 130, 300)
LONG = SHORT + (1101,)
# name: (vocab, hidden, inter, layers, heads, kv heads, head_dim), options
WIDTHS = {
    "w7b": ((32000, 4096, 11008, 2, 32, 32, 128), dict(theta=10000.0, seed=11, prompts=LONG, perm=True)),
    "w8b": ((128256, 4096, 14336, 2, 32, 8, 128), dict(theta=500000.0, seed=12, prompts=LONG)),
    "w13b": ((32000, 5120, 13824, 2, 40, 40, 128), dict(theta=10000.0, seed=13, prompts=SHORT)),
    "w70b": ((32000, 8192, 28672, 1, 64, 8, 128), dict(theta=10000.0, seed=15, prompts=SHORT)),
    "l32_1b": ((128256, 2048, 8192, 2, 32, 8, 64), dict(theta=500000.0, seed=14, prompts=SHORT, tied=True,
                                                        rope=LLAMA3)),
    "survey_mha32": ((512, 256, 688, 2, 8, 8, 32), dict(theta=10000.0, seed=0, prompts=SHORT)),
    "survey_mha32_no_tc": ((512, 256, 688, 2, 8, 8, 32), dict(theta=10000.0, seed=0, prompts=SHORT,
                                                              prefill_tc=False)),
    "linear_rope": ((1000, 512, 1408, 2, 8, 4, 64), dict(theta=10000.0, seed=21, prompts=SHORT,
                                                         rope=dict(rope_scaling="linear", rope_factor=4.0))),
    "odd_vocab": ((32001, 1024, 2816, 2, 16, 4, 64), dict(theta=10000.0, seed=22, prompts=(2, 18, 130))),
}
DECODE_LENS = (60, 120)           # block rows kv_len .. kv_len + m - 1 straddle a page boundary
DECODE_ROWS = (1, 7, 9, 16)


def _build(name):
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    (v, h, i, nl, nh, nkv, hd), o = WIDTHS[name]
    arch = LlamaArch(v, h, i, nl, nh, nkv, hd, 1e-5, o["theta"], **o.get("rope", {}))
    dims = orc.LlamaDims(vocab=v, hidden=h, inter=i, layers=nl, heads=nh, kv_heads=nkv, head_dim=hd,
                         rope_theta=o["theta"])
    sd = orc.random_state_dict(dims, o["seed"])
    g = torch.Generator().manual_seed(o["seed"] + 100)
    for k in list(sd):
        if k.endswith("norm.weight"):
            sd[k] = (1 + 0.25 * torch.randn(h, generator=g)).to(torch.bfloat16).float()
    if o.get("tied"):
        del sd["lm_head.weight"]
    max_ctx = max(o["prompts"] + (DECODE_LENS[-1] + 17,)) + 64
    eng = Engine(arch, max_ctx=max_ctx, keep_logits=True, prefill_tc=o.get("prefill_tc"))
    eng.load_state_dict(sd)
    if o.get("perm"):
        n_pages = (max_ctx + 63) // 64
        eng.debug_set_page_table(torch.randperm(n_pages, generator=torch.Generator().manual_seed(7)).tolist())
    ref = sr.RefModel(arch, sd, max_ctx + 64)
    del sd
    ids = torch.randint(3, v - 1, (max_ctx,), generator=torch.Generator().manual_seed(o["seed"] + 200)).tolist()
    return arch, eng, ref, ids


def _kv(eng, layer, pos0, count):
    """Engine K / V rows [count, kv_heads, head_dim] at positions pos0 .. pos0+count-1 (cuda f64)."""
    out = []
    for which in ("k", "v"):
        rows = [eng.debug_kv_rows(which, layer, h, pos0, count) for h in range(eng.arch.kv_heads)]
        out.append(torch.stack(rows, 1).to("cuda", torch.float64))
    return out


def _raw_logits(eng, rows):
    from layerskip_b200 import _lib
    vpad = (eng.arch.vocab + 15) // 16 * 16
    buf = (C.c_float * (rows * vpad))()
    _lib.check(eng._lib.lsk_debug_read(eng._h, _lib.LSK_DBG_LOGITS, 0, 0, buf, rows * vpad))
    return torch.frombuffer(buf, dtype=torch.float32).clone().view(rows, vpad)


def _expect(rep, worst):
    """Record a comparison; violations are collected and reported together at the end."""
    print(f"    {rep}", flush=True)
    worst.setdefault("_violations", [])
    worst[rep.stage] = max(worst.get(rep.stage, 0.0), rep.worst)
    if not rep.ok:
        worst["_violations"].append(str(rep))


def _expect_violation(rep):
    print(f"    sensitivity {rep}", flush=True)
    assert not rep.ok, f"planted error not seen: {rep}"


def _prompt(arch, eng, ref, ids, n, worst, sensitivity):
    """(a): K/V rows of every prompt position (0 .. n-2) of every kv head in every layer."""
    eng.begin(exit_layer=-1, max_steps=8, eos_token_ids=[arch.vocab - 1])
    eng.prefill(ids[:n])
    rows = n - 1
    pos = torch.arange(rows, device="cuda")
    x = ref.embed(ids[:rows])
    k_eng, v_eng = _kv(eng, 0, 0, rows)
    q, k, v = ref.qkv(0, x, pos)
    _expect(sr.check_direct(f"prompt n={n} layer-0 K", k_eng, k, 0, **DIRECT), worst)
    _expect(sr.check_direct(f"prompt n={n} layer-0 V", v_eng, v, 0, **DIRECT), worst)
    if sensitivity and rows > 128:
        # RoPE of one row at the next position
        bad = k.clone()
        bad[127] = ref.qkv(0, x[127:128], pos[127:128] + 1)[1][0]
        _expect_violation(sr.check_direct("layer-0 K, row 127 rotated for position 128", k_eng, bad, 0,
                                          **DIRECT))
        # two positions in different pages swapped
        bad = k.clone()
        bad[[10, 70]] = bad[[70, 10]]
        _expect_violation(sr.check_direct("layer-0 K, positions 10 / 70 swapped", k_eng, bad, 0, **DIRECT))
    for li in range(1, arch.layers):
        attn = ref.attend(q, pos, k_eng, v_eng)
        x = ref.layer_rest(li - 1, x, attn)
        k_eng_n, v_eng_n = _kv(eng, li, 0, rows)
        q, k, v = ref.qkv(li, x, pos)
        _expect(sr.check_rows(f"prompt n={n} layer-{li} K", k_eng_n, k, B_PROMPT_L1, li), worst)
        _expect(sr.check_rows(f"prompt n={n} layer-{li} V", v_eng_n, v, B_PROMPT_L1, li), worst)
        if sensitivity and li == 1 and rows > 128:
            # the last row of the first chunk (and of its attention launch) sees one key fewer
            q0 = ref.qkv(0, ref.embed(ids[:rows]), pos)[0]
            k0, v0 = _kv(eng, 0, 0, rows)
            n_keys = pos + 1
            n_keys[127] -= 1
            x1 = ref.layer_rest(0, ref.embed(ids[:rows]), ref.attend(q0, pos, k0, v0, n_keys))
            _, kb, vb = ref.qkv(1, x1, pos)
            _expect_violation(sr.check_rows("layer-1 K, row 127 one key short", k_eng_n, kb, B_PROMPT_L1, 1))
        k_eng, v_eng = k_eng_n, v_eng_n


def _decode(arch, eng, ref, ids, L, m, worst, sensitivity):
    """(b) + (c): a teacher-forced block of m rows at positions L .. L+m-1 on top of L committed."""
    eng.begin(exit_layer=-1, max_steps=8, eos_token_ids=[arch.vocab - 1])
    eng.prefill(ids[:L + 1])
    block = ids[L:L + m]
    eng.debug_forward_rows(block)
    pos = torch.arange(L, L + m, device="cuda")
    x = ref.embed(block)
    for li in range(arch.layers):
        k_ctx, v_ctx = _kv(eng, li, 0, L + m)              # committed context + the block's own rows
        q, k, v = ref.qkv(li, x, pos)
        tag = f"decode L={L} m={m} layer-{li}"
        if li == 0:
            _expect(sr.check_direct(f"{tag} K", k_ctx[L:], k, li, L, **DIRECT), worst)
            _expect(sr.check_direct(f"{tag} V", v_ctx[L:], v, li, L, **DIRECT), worst)
            if sensitivity and m == 16:
                # one row normalised with its neighbour's rstd
                rs = ref.rstd(x)
                rs_bad = rs.clone()
                rs_bad[3] = rs[4]
                kb = ref.qkv(0, x, pos, rs_bad)[1]
                print(f"    sensitivity: rstd of rows 3 / 4 differ by {float(rs[4] / rs[3] - 1):+.4%}")
                _expect_violation(sr.check_direct(f"{tag} K, row 3 with row 4's rstd", k_ctx[L:], kb, 0, L,
                                                  **DIRECT))
        else:
            _expect(sr.check_rows(f"{tag} K", k_ctx[L:], k, B_DECODE_L1, li, L), worst)
            _expect(sr.check_rows(f"{tag} V", v_ctx[L:], v, B_DECODE_L1, li, L), worst)
        if sensitivity and li == arch.layers - 1:
            # the last two rows' attention outputs swapped on their way into the O projection
            attn = ref.attend(q, pos, k_ctx, v_ctx)
            x_swap = ref.layer_rest(li, x, attn[[*range(m - 2), m - 1, m - 2]])
        x = ref.layer_rest(li, x, ref.attend(q, pos, k_ctx, v_ctx))
    hidden = eng.debug_hidden(m).to("cuda", torch.float64)
    tag = f"decode L={L} m={m}"
    _expect(sr.check_rows(f"{tag} residual after layer {arch.layers - 1}", hidden, x, B_HIDDEN,
                          arch.layers - 1, L), worst)
    if sensitivity:
        _expect_violation(sr.check_rows(f"{tag} residual, attention rows {m - 2} / {m - 1} swapped", hidden, x_swap,
                                        B_HIDDEN, arch.layers - 1, L))
    # LM head from the engine's own final residual rows
    want = ref.logits(hidden)
    _check_lm_head(arch, eng, tag, hidden, want, m, L, worst)
    if sensitivity:
        rs = ref.rstd(hidden)
        rs[3] = rs[4]
        _expect_violation(sr.check_rows(f"{tag} LM head logits, row 3 with row 4's final rstd",
                                        _raw_logits(eng, m)[:, :arch.vocab].to("cuda", torch.float64),
                                        ref.logits(hidden, rs), B_LOGITS, -1, L))


def _check_lm_head(arch, eng, tag, hidden, want, m, L, worst):
    """Logits against the reference from the engine's residual; the engine's own greedy choice (the
    LM-head epilogue's candidates, merged as the accept kernels merge them) is the reference
    arg-max unless the reference's top-2 margin is within the bound; padded vocab columns stay
    unwritten and never win."""
    vocab = arch.vocab
    raw = _raw_logits(eng, m)
    assert torch.equal(raw[:, vocab:], torch.zeros_like(raw[:, vocab:])), "padded vocab columns were written"
    got = raw[:, :vocab].to("cuda", torch.float64)
    _expect(sr.check_rows(f"{tag} LM head logits", got, want, B_LOGITS, -1, L), worst)
    val, tok = eng.debug_argmax(m)
    rms = want.pow(2).mean(-1).sqrt()
    for r in range(m):
        t, b = int(tok[r]), int(want[r].argmax())
        assert 0 <= t < vocab, f"{tag} row {r}: the engine picked token {t} of a {vocab}-token vocab"
        assert float(val[r]) == float(got[r, t]), (tag, r, t, float(val[r]), float(got[r, t]))
        assert t == b or float(want[r, b] - want[r, t]) <= 2 * B_LOGITS * float(rms[r]), \
            f"{tag} row {r}: engine picked {t}, reference arg-max {b} (margin {float(want[r, b] - want[r, t]):.4g})"


def _padded_columns_never_win(arch, eng, ref, ids, worst):
    """Vocab not a multiple of 16: the last LM-head tile has padded (zero) rows, whose logit is 0.
    Shift the head so that every real logit of row 0 is negative: a padded column that took part
    in the arg-max would then win."""
    from layerskip_b200 import _lib
    L, m = 60, 7
    block = ids[L:L + m]
    eng.begin(exit_layer=-1, max_steps=8, eos_token_ids=[arch.vocab - 1])
    eng.prefill(ids[:L + 1])
    eng.debug_forward_rows(block)
    hidden = eng.debug_hidden(m).to("cuda", torch.float64)
    xn0 = ref.norm(hidden[:1], ref.final_norm)[0]
    lg = ref.logits(hidden)[0]
    shift = float(lg.max()) + 4 * float(lg.pow(2).mean().sqrt())
    w = (ref.lm_head.double() - shift * (xn0 / xn0.pow(2).sum())[None, :]).to(torch.bfloat16).contiguous()
    eng.load_weights([(_lib.LSK_W_LM_HEAD, 0, w)])
    ref.lm_head = w
    eng.debug_forward_rows(block)
    hidden = eng.debug_hidden(m).to("cuda", torch.float64)
    want = ref.logits(hidden)
    assert float(want[0].max()) < 0, "row 0 still has a non-negative real logit"
    _check_lm_head(arch, eng, f"padded vocab L={L} m={m}", hidden, want, m, L, worst)


@pytest.mark.parametrize("name", list(WIDTHS))
def test_stages_match_the_float64_reference(name):
    arch, eng, ref, ids = _build(name)
    worst = {}
    try:
        with torch.inference_mode():
            for n in WIDTHS[name][1]["prompts"]:
                _prompt(arch, eng, ref, ids, n, worst, sensitivity=(name == "w7b" and n == 300))
            for L in DECODE_LENS:
                for m in DECODE_ROWS:
                    if m <= eng.max_rows:
                        _decode(arch, eng, ref, ids, L, m, worst, sensitivity=(name == "w7b" and m == 16))
            if arch.vocab % 16:
                _padded_columns_never_win(arch, eng, ref, ids, worst)
    finally:
        eng.close()
        del ref
        torch.cuda.empty_cache()
    bad = worst.pop("_violations", [])
    agg = {}
    for stage, w in worst.items():
        key = " ".join(t for t in stage.split() if "=" not in t)
        agg[key] = max(agg.get(key, 0.0), w)
    for k, w in sorted(agg.items()):
        print(f"  WORST {name} {k}: {w:.4g}")
    assert not bad, "\n".join(bad)

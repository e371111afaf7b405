"""GPU: batched greedy rounds (`lsk_prefill_batch` / `lsk_round_batch`) and single rounds outside the
layouts, widths and slot lengths of test_gpu_generate_batch.py, reading every kv head of every layer.

(a) batch == solo, bit for bit (test_gpu_generate_batch.py's `_run_batch` / `_check_against_solo`), at
    the layouts of test_gpu_stages.py / test_gpu_stages_edges.py: group 3 with llama3 RoPE and a
    128256 vocab (`l32_3b`), head_dim 64 with tied weights (`l32_1b`), group 4 (`w8b`), hidden 5120
    (`w13b`: 9-16-row verifies run the K-chunked RMSNorm under EPI_QKV_SEQS), hidden 8192 with group
    8 (`w70b`), groups 5 / 7 / 16, a partial K block with vocab 32003 (`odd_k`), head_dim 32
    (`survey_mha32`) and hidden 96 (`tiny`); B x (D + 1) in (2, 7), (3, 5), (4, 4), (8, 2), (16, 1).
(b) float64 stage check of a round's own rows (tests/stage_ref.py, test_gpu_stages.py's bounds),
    batched and single (`lsk_round`): K/V of every layer and kv head at the round's positions (layer
    0 DIRECT, deeper layers from the engine's own K/V), the committed rows of earlier rounds, the final
    residual rows, the logits from the engine's residual, the verified ids (margin-gated arg-max) and
    the draft ids (the reference exit head's arg-max, gated by DRAFT_GATE).  Four planted reference
    errors must each be reported.
(c) long slots (max_ctx 32768, permuted pages) at the `l32_1b` and `w8b` widths: B = 2, 4, 8 with
    prompts of up to ~12000 ids, batch == solo, and the committed rows against float64 at sampled
    positions as test_gpu_stages_edges.py checks long prompts.
(d) attn_splits 1, 3 and 8 at `l32_3b`: batch == solo on the same engine, and (b).
(e) slot edges: every slot's committed rows (all layers, all kv heads) and the pages no slot owns are
    bit-identical before and after each round, with a sequence at kv_len + d_req + 2 == slot (active
    and inactive) next to neighbours holding rows from position 0, 16 one-page slots, and 3 slots of 640
    positions with 2 leftover pages that a long single prefill filled first.

Bounds and measured worst values: DESIGN.md §7."""
from unittest import mock

import pytest
import torch

from oracle import llama_oracle as orc
from tests import stage_ref as sr
from tests import test_gpu_generate_batch as tgb
from tests import test_gpu_stages as ts
from tests import test_gpu_stages_edges as te
from tests.test_gpu_stages import B_DECODE_L1, B_HIDDEN, B_LOGITS, B_PROMPT_L1, DIRECT

pytestmark = pytest.mark.gpu

E = 1                      # every layout has two layers: the exit is layer 1
ALPHA = 0.3                # damping of layers >= E so that drafts are accepted
# (b) the engine's draft ids vs the reference exit head's arg-max: a draft may differ from it only
# where the reference's top-2 margin is within DRAFT_GATE x the exit logits row's RMS
DRAFT_GATE = 0.003
LAYOUTS = {**ts.WIDTHS, **te.WIDTHS}
NAMES = ("l32_3b", "l32_1b", "w8b", "w13b", "w70b", "g5_hd64", "g7", "g16", "odd_k", "survey_mha32", "tiny")
BATCHES = ((2, 6), (3, 4), (4, 3), (8, 1), (16, 0))

_cache = {}


def _setup(name, max_ctx=2048, attn_splits=0, perm=None):
    """(arch, dims, engine, reference) of a two-layer model at layout `name`, one cached at a time."""
    key = (name, max_ctx, attn_splits, perm)
    if key not in _cache:
        _drop()
        from layerskip_b200.engine import Engine
        from layerskip_b200.weights import LlamaArch
        (v, h, i, _nl, nh, nkv, hd), o = LAYOUTS[name]
        arch = LlamaArch(v, h, i, 2, nh, nkv, hd, 1e-5, o["theta"], **o.get("rope", {}))
        dims = tgb._dims(v, h, i, 2, nh, nkv, hd, o["theta"])
        sd = orc.random_state_dict(dims, seed=o["seed"], damp_from_layer=E, alpha=ALPHA)
        # RMSNorm weights around 1, as test_gpu_stages.py draws them: with unit weights the normalised
        # bf16 embedding rows sit on many bf16 ties that the kernels' rsqrtf breaks differently (a
        # w13b prompt row measured 6.4 ulp-or-floor units at layer 0 against DIRECT's 4)
        g = torch.Generator().manual_seed(o["seed"] + 100)
        for k in list(sd):
            if k.endswith("norm.weight"):
                sd[k] = (1 + 0.25 * torch.randn(h, generator=g)).to(torch.bfloat16).float()
        if o.get("tied"):
            del sd["lm_head.weight"]
        eng = Engine(arch, max_ctx=max_ctx, keep_logits=True, attn_splits=attn_splits)
        eng.load_state_dict(sd)
        if perm is not None:
            n_pages = (max_ctx + 63) // 64
            eng.debug_set_page_table(torch.randperm(n_pages, generator=torch.Generator().manual_seed(perm)).tolist())
        ref = sr.RefModel(arch, sd, max_ctx + 64)
        del sd
        _cache[key] = (arch, dims, eng, ref)
    return _cache[key]


def _drop():
    for _a, _d, eng, _r in _cache.values():
        eng.close()
    _cache.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _close():
    yield
    _drop()


def _kv_all(eng, dims, pos0, count):
    """K and V rows at positions pos0 .. pos0 + count - 1 of every kv head in every layer."""
    if count == 0:
        return []
    return [eng.debug_kv_rows(w, l, h, pos0, count) for w in "kv" for l in range(eng.arch.layers)
            for h in range(eng.arch.kv_heads)]


def _batch_equals_solo(eng, dims, prompts, D, rounds, eos, vary=True):
    with mock.patch.object(tgb, "MAX_CTX", eng.max_ctx), mock.patch.object(tgb, "_kv", _kv_all):
        trace, lens, slot = tgb._run_batch(eng, dims, E, prompts, D, eos, rounds=rounds, vary=vary)
        tgb._check_against_solo(eng, dims, E, prompts, eos, trace, lens, slot)
    return trace


def _prompts(dims, lengths, seed):
    return tgb._prompts(dims, lengths, seed=seed)


# ------------------------------------------------------------------------------------------------
# (a) batch == solo at new layouts
# ------------------------------------------------------------------------------------------------
CASES = [(n, B, D) for n in NAMES for B, D in BATCHES]


@pytest.mark.parametrize("name,B,D", CASES, ids=[f"{n}-B{b}-D{d}" for n, b, d in CASES])
def test_rounds_equal_solo_rounds_at_new_layouts(name, B, D):
    arch, dims, eng, _ref = _setup(name)
    if B * (D + 1) > eng.max_rows:
        pytest.skip(f"{B} x {D + 1} rows exceed this layout's {eng.max_rows}-row steps")
    if B < 16:
        prompts = _prompts(dims, tgb.LENGTHS[:B] if B < 8 else tgb.LENGTHS, seed=B)
        eos = [dims.vocab - 1, tgb._early_token(eng, dims, E, prompts[0], D)]
        trace = _batch_equals_solo(eng, dims, prompts, D, 4, eos)
        assert any(not a[0] for _d, a, _o in trace), "the first sequence was meant to stop early on EOS"
    else:
        prompts = _prompts(dims, [1 + (7 * j) % 60 for j in range(16)], seed=16)
        _batch_equals_solo(eng, dims, prompts, 0, 4, [dims.vocab - 1], vary=False)


# ------------------------------------------------------------------------------------------------
# (b) float64 stage check of a round's own rows
# ------------------------------------------------------------------------------------------------
def _stage_round(arch, eng, ref, prompts, d, rounds_before, batched, worst, plants=False):
    """Rounds of d drafts for every sequence (no EOS), then one more whose rows are checked against
    the reference fed each sequence's committed tokens + [pending] + its drafts."""
    eng.begin(exit_layer=E, max_steps=4096, eos_token_ids=[], sample=False)
    if batched:
        slot = eng.prefill_batch(prompts)
    else:
        assert len(prompts) == 1
        eng.prefill(prompts[0])
        slot = 0
    B = len(prompts)
    full = [list(p) for p in prompts]
    step = (lambda: eng.round_batch(d)) if batched else (lambda: [eng.round(d)])
    for _ in range(rounds_before):
        for s, o in enumerate(step()):
            full[s] += o.emitted
    lens = [len(f) - 1 for f in full]                      # committed; full[s][-1] is pending
    outs = step()
    m = B * (d + 1)
    hidden = eng.debug_hidden(m).to("cuda", torch.float64)
    raw = ts._raw_logits(eng, m)
    val, tok = eng.debug_argmax(m)
    vocab = arch.vocab
    assert torch.equal(raw[:, vocab:], torch.zeros_like(raw[:, vocab:])), "padded vocab columns were written"
    logits = raw[:, :vocab].to("cuda", torch.float64)
    mode = f"{'batch' if batched else 'single'} B={B} d={d}"
    finals, draft_worst = [], [0.0, float("inf")]          # worst mismatch margin, least margin
    for s, o in enumerate(outs):
        assert o.n_drafted == d, (s, o.n_drafted)
        L, base = lens[s], s * slot
        toks = full[s] + o.draft
        n = L + d + 1
        pos = torch.arange(n, device="cuda")
        x = ref.embed(toks)
        tag = f"{mode} seq={s} kv_len={L}"
        for li in range(arch.layers):
            K, V = ts._kv(eng, li, base, n)
            q, k, v = ref.qkv(li, x, pos)
            for which, got, want in (("K", K, k), ("V", V, v)):
                if li == 0:
                    ts._expect(sr.check_direct(f"{tag} committed layer-0 {which}", got[:L], want[:L], 0, **DIRECT), worst)
                    ts._expect(sr.check_direct(f"{tag} round layer-0 {which}", got[L:], want[L:], 0, L, **DIRECT), worst)
                else:
                    ts._expect(sr.check_rows(f"{tag} committed layer-{li} {which}", got[:L], want[:L], B_PROMPT_L1, li),
                               worst)
                    ts._expect(sr.check_rows(f"{tag} round layer-{li} {which}", got[L:], want[L:], B_DECODE_L1, li, L),
                               worst)
            if plants and li == 0 and s + 1 < B:
                # a draft row given the next sequence's committed length (layer 0: the draft's layers)
                bad_pos = pos[L:].clone() - L + lens[s + 1]
                kb = ref.qkv(0, x[L:], bad_pos)[1]
                ts._expect_violation(sr.check_direct(f"{tag} round layer-0 K at sequence {s + 1}'s length "
                                                     f"{lens[s + 1]}", K[L:], kb, 0, L, **DIRECT))
            if plants and li == E:
                # a verify row rotated for the next position
                kb = k[L:].clone()
                kb[1] = ref.qkv(li, x[L + 1:L + 2], pos[L + 1:L + 2] + 1)[1][0]
                ts._expect_violation(sr.check_rows(f"{tag} round layer-{li} K, row 1 rotated for the next position",
                                                   K[L:], kb, B_DECODE_L1, li, L))
            if plants and li == 1 and s + 1 < B:
                # the layer-0 attention over slot s + 1's K/V instead of slot s's
                K1, V1 = ts._kv(eng, 0, base + slot, n)
                x1 = ref.layer_rest(0, ref.embed(toks), ref.attend(ref.qkv(0, ref.embed(toks), pos)[0], pos, K1, V1))
                kb = ref.qkv(1, x1, pos)[1]
                ts._expect_violation(sr.check_rows(f"{tag} layer-1 K over slot {s + 1}'s K/V", K[:n], kb,
                                                   B_PROMPT_L1, 1))
            x = ref.layer_rest(li, x, ref.attend(q, pos, K, V))
            if li == E - 1:
                exit_logits = ref.logits(x[L:L + d])
        own = slice(s * (d + 1), (s + 1) * (d + 1))
        finals.append(x[L:])
        ts._expect(sr.check_rows(f"{tag} residual after layer {arch.layers - 1}", hidden[own], x[L:], B_HIDDEN,
                                 arch.layers - 1, L), worst)
        # logits from the engine's own residual; the verified ids are the engine's arg-max, which is
        # the reference's unless its top-2 margin is within the logits bound
        want = ref.logits(hidden[own])
        ts._expect(sr.check_rows(f"{tag} LM head logits", logits[own], want, B_LOGITS, -1, L), worst)
        rms = want.pow(2).mean(-1).sqrt()
        for i in range(d + 1):
            r = s * (d + 1) + i
            t, b = int(tok[r]), int(want[i].argmax())
            assert float(val[r]) == float(logits[r, t]), (tag, i)
            assert o.verified[i] == t, f"{tag} row {i}: verified id {o.verified[i]}, LM-head arg-max {t}"
            assert t == b or float(want[i, b] - want[i, t]) <= 2 * B_LOGITS * float(rms[i]), (tag, i, t, b)
        # draft ids against the reference exit head (layers < E from the engine's own K/V)
        erms = exit_logits.pow(2).mean(-1).sqrt()
        for i in range(d):
            b, t = int(exit_logits[i].argmax()), o.draft[i]
            top2 = exit_logits[i].topk(2).values
            draft_worst[1] = min(draft_worst[1], float((top2[0] - top2[1]) / erms[i]))
            if t != b:
                margin = float((exit_logits[i, b] - exit_logits[i, t]) / erms[i])
                draft_worst[0] = max(draft_worst[0], margin)
                assert margin <= DRAFT_GATE, f"{tag} draft {i}: engine {t}, reference exit arg-max {b} (margin {margin:.4g})"
    worst[f"{mode} draft mismatch margin"] = max(worst.get(f"{mode} draft mismatch margin", 0.0), draft_worst[0])
    print(f"    {mode}: draft ids: worst mismatch margin / row RMS {draft_worst[0]:.4g} (gate {DRAFT_GATE}), "
          f"least top-2 margin / row RMS {draft_worst[1]:.4g}")
    if plants and B > 1:
        # two sequences' final residual rows swapped
        h01 = torch.cat([hidden[:d + 1], hidden[d + 1:2 * (d + 1)]])
        x01 = torch.cat([finals[1], finals[0]])
        ts._expect_violation(sr.check_rows(f"{mode} residual, sequences 0 / 1 swapped", h01, x01, B_HIDDEN,
                                           arch.layers - 1))


STAGE_CASES = [  # name, attn_splits, B, d, batched
    ("l32_3b", 0, 4, 3, True), ("l32_3b", 0, 1, 6, False), ("w13b", 0, 2, 6, True), ("w13b", 0, 1, 15, False),
    ("g5_hd64", 0, 3, 4, True), ("tiny", 0, 8, 1, True), ("odd_k", 0, 2, 7, True),
]


@pytest.mark.parametrize("name,splits,B,d,batched", STAGE_CASES,
                         ids=[f"{n}-B{b}-d{d}-{'batch' if x else 'single'}" for n, _s, b, d, x in STAGE_CASES])
def test_round_rows_match_the_float64_reference(name, splits, B, d, batched):
    arch, dims, eng, ref = _setup(name, attn_splits=splits)
    if B * (d + 1) > eng.max_rows:
        pytest.skip(f"{B} x {d + 1} rows exceed this layout's {eng.max_rows}-row steps")
    worst = {}
    with torch.inference_mode():
        prompts = _prompts(dims, (130, 17, 64, 2, 65, 9, 33, 100)[:B], seed=B + d)
        _stage_round(arch, eng, ref, prompts, d, 3, batched, worst, plants=(name == "l32_3b" and batched))
    te._report(f"{name}", worst)


# ------------------------------------------------------------------------------------------------
# (c) long slots
# ------------------------------------------------------------------------------------------------
LONG_CASES = [("l32_1b", 2, 3, (12000, 3)), ("l32_1b", 4, 3, (7000, 1, 4097, 129)), ("l32_1b", 8, 1, (4000,) * 8),
              ("w8b", 2, 3, (12000, 3)), ("w8b", 4, 3, (7000, 1, 4097, 129)), ("w8b", 8, 1, (4000,) * 8)]


def _committed_rows_sampled(arch, eng, ref, toks, base, worst, tag):
    """Committed rows 0 .. len(toks) - 2 of one slot: layer-0 K/V of every kv head at sampled positions
    (DIRECT_LONG), layer-1 rows there from the engine's layer-0 K/V."""
    n = len(toks) - 1
    sel = torch.tensor(te._sampled_rows(n, n), device="cuda")
    pos = torch.arange(n, device="cuda")[sel]
    x = ref.embed([toks[i] for i in sel.tolist()])
    K0, V0 = ts._kv(eng, 0, base, n)
    q, k, v = ref.qkv(0, x, pos)
    ts._expect(sr.check_direct(f"{tag} layer-0 K (sampled rows)", K0[sel], k, 0, **te.DIRECT_LONG), worst)
    ts._expect(sr.check_direct(f"{tag} layer-0 V (sampled rows)", V0[sel], v, 0, **te.DIRECT_LONG), worst)
    x1 = ref.layer_rest(0, x, ref.attend(q, pos, K0, V0))
    _, k1, v1 = ref.qkv(1, x1, pos)
    K1, V1 = ts._kv(eng, 1, base, n)
    ts._expect(sr.check_rows(f"{tag} layer-1 K (sampled rows)", K1[sel], k1, B_PROMPT_L1, 1), worst)
    ts._expect(sr.check_rows(f"{tag} layer-1 V (sampled rows)", V1[sel], v1, B_PROMPT_L1, 1), worst)


@pytest.mark.parametrize("name,B,D,lengths", LONG_CASES, ids=[f"{n}-B{b}" for n, b, _d, _l in LONG_CASES])
def test_long_slots(name, B, D, lengths):
    arch, dims, eng, ref = _setup(name, max_ctx=32768, perm=3)
    prompts = _prompts(dims, lengths, seed=B)
    eos = [dims.vocab - 1]
    trace = _batch_equals_solo(eng, dims, prompts, D, 4, eos)
    # the batch again (the solo replays above reused the pool), then its committed rows against float64
    with mock.patch.object(tgb, "MAX_CTX", eng.max_ctx):
        again, _lens, slot = tgb._run_batch(eng, dims, E, prompts, D, eos, rounds=4)
    assert [[tgb._fields(o) for o in outs] for _d, _a, outs in again] == \
        [[tgb._fields(o) for o in outs] for _d, _a, outs in trace]
    worst = {}
    with torch.inference_mode():
        for s, p in enumerate(prompts):
            if len(p) > 1000:
                toks = list(p) + [t for _d, _a, outs in trace for t in outs[s].emitted]
                _committed_rows_sampled(arch, eng, ref, toks, s * slot, worst, f"B={B} seq {s} ({len(p)} ids)")
    te._report(name, worst)


# ------------------------------------------------------------------------------------------------
# (d) split overrides
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("splits", [1, 3, 8])
def test_split_overrides(splits):
    arch, dims, eng, ref = _setup("l32_3b", attn_splits=splits)
    for B, D in ((4, 3), (8, 1), (2, 6)):
        prompts = _prompts(dims, tgb.LENGTHS[:B], seed=B + splits)
        _batch_equals_solo(eng, dims, prompts, D, 4, [dims.vocab - 1])
    worst = {}
    with torch.inference_mode():
        _stage_round(arch, eng, ref, _prompts(dims, (130, 17, 64, 2), seed=splits), 3, 3, True, worst)
    te._report(f"l32_3b splits={splits}", worst)


# ------------------------------------------------------------------------------------------------
# (e) slot edges
# ------------------------------------------------------------------------------------------------
def _snapshot(eng, slot, lens, spare):
    """Every slot's committed rows (all layers, all kv heads) and the rows `spare` of the pages no
    slot owns."""
    snap = [_kv_all(eng, None, s * slot, n) for s, n in enumerate(lens)]
    if spare:
        snap.append(_kv_all(eng, None, spare[0], spare[1] - spare[0]))
    return snap


def _round_keeps_committed(eng, slot, lens, d_req, d_seq=None, active=None, spare=None):
    before = _snapshot(eng, slot, lens, spare)
    outs = eng.round_batch(d_req, d_seq, active)
    after = _snapshot(eng, slot, lens, spare)
    for i, (a, b) in enumerate(zip(before, after)):
        assert all(torch.equal(x, y) for x, y in zip(a, b)), f"round changed committed rows of slot {i}"
    return [n if not (active is None or active[s]) else o.kv_len for s, (n, o) in enumerate(zip(lens, outs))]


def test_sequence_at_the_end_of_its_slot():
    """Sequence 1 starts a round at kv_len + d_req + 2 == slot, active and then inactive, between
    neighbours that hold rows from position 0; the two pages past the last slot stay untouched."""
    arch, dims, eng, _ref = _setup("l32_3b")
    B, d = 3, 3
    slot = tgb.batch_slot_positions(eng.max_ctx, B)                # 10 of 32 pages each: 2 spare pages
    spare = (B * slot, eng.max_ctx)
    for active in (None, [True, False, True]):
        eng.begin(exit_layer=E, max_steps=4096, eos_token_ids=[], sample=False)
        prompts = _prompts(dims, (300, slot - d - 1, 5), seed=11)
        eng.prefill_batch(prompts)
        lens = [len(p) - 1 for p in prompts]
        assert lens[1] + d + 2 == slot
        _round_keeps_committed(eng, slot, lens, d, None, active, spare)


def test_sixteen_one_page_slots():
    """16 slots of one page each (max_ctx 1024): rounds of d_req 0 until every sequence sits at
    kv_len + 2 == 64; a sequence that reached it idles, inactive, while the others go on."""
    arch, dims, eng, _ref = _setup("tiny", max_ctx=1024)
    slot = tgb.batch_slot_positions(1024, 16)
    assert slot == 64
    eng.begin(exit_layer=E, max_steps=4096, eos_token_ids=[], sample=False)
    prompts = _prompts(dims, [40 + (7 * j) % 21 for j in range(16)], seed=5)
    eng.prefill_batch(prompts)
    lens = [len(p) - 1 for p in prompts]
    while any(n + 2 < slot for n in lens):
        lens = _round_keeps_committed(eng, slot, lens, 0, None, [n + 2 < slot for n in lens])
    assert lens == [slot - 2] * 16


def test_leftover_pages_and_the_batch_prompt_bound():
    """max_ctx 2000: 32 pages, 3 slots of 640 positions and 2 pages no slot owns.  A long single
    prefill fills those pages first; no batched round touches them.  A batch of one may not take a
    prompt that `lsk_prefill` refuses, even though its 2048-position slot would hold it."""
    from layerskip_b200._lib import LskError
    arch, dims, eng, _ref = _setup("g5_hd64", max_ctx=2000)
    B, d = 3, 4
    slot = tgb.batch_slot_positions(2000, B)
    assert slot == 640
    spare = (B * slot, 1998)                                       # rows lsk_debug_read reaches (< max_ctx)
    eng.begin(exit_layer=E, max_steps=4096, eos_token_ids=[], sample=False)
    eng.prefill(_prompts(dims, (1999,), seed=1)[0])                # rows 0 .. 1997
    filled = _kv_all(eng, None, spare[0], spare[1] - spare[0])
    assert any(float(t.abs().max()) > 0 for t in filled)
    eng.begin(exit_layer=E, max_steps=4096, eos_token_ids=[], sample=False)
    prompts = _prompts(dims, (630 - d, 1, 200), seed=2)
    eng.prefill_batch(prompts)
    lens = [len(p) - 1 for p in prompts]
    for r in range(4):
        d_req = d if max(lens) + d + 2 <= slot else 0
        lens = _round_keeps_committed(eng, slot, lens, d_req, spare=spare)
    after = _kv_all(eng, None, spare[0], spare[1] - spare[0])
    assert all(torch.equal(a, b) for a, b in zip(filled, after))
    # the prompt bound of a batch of one is lsk_prefill's
    with pytest.raises(LskError) as ex:
        eng.prefill_batch([[5] * 2000])
    assert ex.value.code == -6
    with pytest.raises(LskError) as ex:
        eng.prefill([5] * 2000)
    assert ex.value.code == -6
    eng.prefill_batch([[5] * 1999])

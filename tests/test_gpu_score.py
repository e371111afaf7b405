"""GPU: teacher-forced scoring (`lsk_score` / `Engine.score` / `Engine.loglikelihood`).

1. the log-softmax kernel alone against float64 torch (vocab 512 / 32000 / 32001 with +1e30 in the
   pad columns / 128256; peaked, flat, all below -50, exact ties, targets at both ends);
2. exact against the decode path: on an engine without the wgmma prompt pass, the greedy token of
   row p is the arg-max of `debug_forward_rows` after `prefill(ids[:p+1])` bit for bit, and its
   log-probability is the float64 log softmax of those logits within the kernel bound;
3. exact early exit: score(model, E) is bit-identical to score(model cut to its first E layers);
4. against the oracle (`teacher_forced_logits` / `early_exit_logits`): golden spec-case models, and
   7B / 8B / 13B / llama3.2-1B / 32001-vocab / head_dim-32 widths as 2-layer models, within bounds
   tighter than the ones the project's logit bounds imply (`pu.TAU`, 2 x 2.5 % of the row's max
   |logit|); greedy == oracle arg-max wherever the oracle's margin is at least the implied bound;
5. against greedy generation on the same engine, full depth and early exit;
6. state and determinism (repeat, page table, state after a score, keep_logits, LSK_LMHEAD_TC=1,
   the last slice's logits);
7. argument errors;
8. each comparison fails on a planted error (shifted targets, a neighbour's row, E off by one,
   pad columns included).

Bounds: DESIGN.md §7, each at most 2x its worst value measured on an H100 80GB HBM3 at a 400 W
power limit.  Measured values are printed as `MEASURED <name> <value>`."""
import ctypes as C

import pytest
import torch

from oracle import llama_oracle as orc
from tests import golden_util as gu
from tests import parity_util as pu

pytestmark = pytest.mark.gpu

# |logprob - float64 log softmax| / (1 + |logsumexp|) of the kernel on fp32 logits (measured worst
# 6.8e-8 over every row of tests 1, 2 and 6)
B_KERNEL = 1.3e-7
# engine vs oracle logprob.  A logprob error is at most twice the logit error, so the project's
# logit bounds give |d| <= pu.TAU (golden models) and |d| <= 2 x 2.5 % of the row's max |logit|
# (widths); the greedy token is checked wherever the oracle's top-2 margin is at least that.  The
# asserted bounds are tighter, at most 2x the measured worst:
REL_LOGIT = 0.025
B_GOLDEN = 0.012                 # absolute, golden spec-case models      (measured worst 0.0059)
REL_WIDTH = 0.018                # x the row's max |logit|, widths       (measured worst 0.0089)

LLAMA3 = {"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
          "original_max_position_embeddings": 8192}
SHORT = (2, 17, 18, 129, 130, 300)
LONG = SHORT + (1101,)
# name: (vocab, hidden, inter, layers, heads, kv heads, head_dim), theta, rope scaling, tied, seed, lengths
WIDTHS = {
    "w7b": ((32000, 4096, 11008, 2, 32, 32, 128), 10000.0, None, False, 11, LONG),
    "w8b": ((128256, 4096, 14336, 2, 32, 8, 128), 500000.0, None, False, 12, LONG),
    "w13b": ((32000, 5120, 13824, 2, 40, 40, 128), 10000.0, None, False, 13, SHORT),
    "l32_1b": ((128256, 2048, 8192, 2, 32, 8, 64), 500000.0, LLAMA3, True, 14, SHORT),
    "odd_vocab": ((32001, 1024, 2816, 2, 16, 4, 64), 10000.0, None, False, 22, SHORT),
    "mha32": ((512, 256, 688, 2, 8, 8, 32), 10000.0, None, False, 0, SHORT),
}


def _measured(name, value):
    print(f"MEASURED {name} {value:.4g}", flush=True)


def _lib():
    from layerskip_b200 import _lib as L
    return L


def _ref_logprob(logits, targets):
    """float64 log softmax of fp32 logits rows at `targets`, its logsumexp, and the arg-max."""
    x = logits.to(torch.float64)
    lse = torch.logsumexp(x, dim=-1)
    return x.gather(1, targets.view(-1, 1)).squeeze(1) - lse, lse, torch.argmax(x, dim=-1)


def _kernel_rel(lp, ref_lp, lse):
    return float(((lp.to(torch.float64) - ref_lp).abs() / (1 + lse.abs())).max())


def _engine(dims, sd, max_ctx, **kw):
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    cfg = type("Cfg", (), dict(
        vocab_size=dims.vocab, hidden_size=dims.hidden, intermediate_size=dims.inter,
        num_hidden_layers=dims.layers, num_attention_heads=dims.heads, num_key_value_heads=dims.kv_heads,
        head_dim=dims.head_dim, rms_norm_eps=dims.rms_eps, rope_theta=dims.rope_theta,
        rope_scaling=dims.rope_scaling))()
    eng = Engine(LlamaArch.from_hf_config(cfg), max_ctx=max_ctx, **kw)
    eng.load_state_dict(sd)
    return eng


def _dims(v, h, i, nl, nh, nkv, hd, theta=10000.0, scaling=None):
    return orc.LlamaDims(vocab=v, hidden=h, inter=i, layers=nl, heads=nh, kv_heads=nkv, head_dim=hd,
                         rms_eps=1e-5, rope_theta=theta, rope_scaling=scaling)


def _ids(vocab, n, seed):
    return torch.randint(3, vocab - 1, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


# ------------------------------------------------------------------------------------------------
# 1. the kernel alone
# ------------------------------------------------------------------------------------------------
def _kernel_rows(vocab):
    g = torch.Generator().manual_seed(vocab)
    rows, targets = [], []
    r = torch.randn(vocab, generator=g) * 0.5                       # peaked
    r[vocab // 3] = 20.0
    rows.append(r); targets.append(vocab // 3)
    rows.append(torch.zeros(vocab)); targets.append(vocab - 1)      # flat: every id ties, id 0 wins
    rows.append(-60.0 + torch.randn(vocab, generator=g) * 2); targets.append(0)    # all below -50
    r = torch.randn(vocab, generator=g)                              # exact tie at two ids
    lo, hi = vocab // 5, vocab - 2
    r[lo] = r[hi] = float(r.max()) + 1.0
    rows.append(r); targets.append(hi)
    r = torch.randn(vocab, generator=g) * 3                          # tie between the first and last id
    r[0] = r[vocab - 1] = float(r.max()) + 0.5
    rows.append(r); targets.append(vocab - 1)
    rows.append(torch.randn(vocab, generator=g) * 4); targets.append(0)
    return torch.stack(rows).float(), torch.tensor(targets, dtype=torch.int32)


def _run_kernel(logits, vocab, ld, targets):
    L = _lib()
    lib = L.load()
    rows = logits.shape[0]
    lp = torch.empty(rows, dtype=torch.float32, device="cuda")
    gr = torch.empty(rows, dtype=torch.int32, device="cuda")
    L.check(lib.lsk_test_logprob(logits.data_ptr(), rows, vocab, ld, targets.data_ptr(), lp.data_ptr(),
                                 gr.data_ptr()))
    return lp.cpu(), gr.cpu().to(torch.int64)


@pytest.mark.parametrize("vocab", [512, 32000, 32001, 128256])
def test_logprob_kernel_matches_float64(vocab):
    logits, targets = _kernel_rows(vocab)
    ld = (vocab + 15) // 16 * 16
    padded = torch.full((logits.shape[0], ld), 1e30)                 # pad columns must never count
    padded[:, :vocab] = logits
    lp, gr = _run_kernel(padded.cuda(), vocab, ld, targets.cuda())
    ref, lse, am = _ref_logprob(logits, targets.long())
    rel = _kernel_rel(lp, ref, lse)
    _measured(f"kernel_rel_v{vocab}", rel)
    assert rel <= B_KERNEL, rel
    assert torch.equal(gr, am), (gr, am)
    assert int(gr[1]) == 0 and int(gr[3]) == vocab // 5 and int(gr[4]) == 0      # lowest id wins ties
    # 8. planted: pad columns included in the reference
    if ld > vocab:
        ref_bad, lse_bad, _ = _ref_logprob(padded, targets.long())
        bad = float(((lp.double() - ref_bad).abs() / (1 + lse.abs())).max())
        _measured("planted_pad_columns_factor", bad / B_KERNEL)
        assert bad > B_KERNEL


# ------------------------------------------------------------------------------------------------
# 2. exact against the decode path
# ------------------------------------------------------------------------------------------------
def test_score_is_exact_against_the_decode_path():
    dims = _dims(32001, 1024, 2816, 2, 16, 4, 64)
    sd = orc.random_state_dict(dims, 22)
    eng = _engine(dims, sd, 128, keep_logits=True, prefill_tc=False)
    try:
        ids = _ids(dims.vocab, 48, 5)
        lp, greedy = eng.score(ids)
        worst = 0.0
        for p in (1, 15, 16, 17, 40):
            eng.begin(-1, 4, [])
            eng.prefill(ids[:p + 1])
            logits = eng.debug_forward_rows([ids[p]])
            ref, lse, am = _ref_logprob(logits, torch.tensor([ids[p + 1]]))
            assert int(greedy[p]) == int(am[0]), (p, int(greedy[p]), int(am[0]))
            rel = _kernel_rel(lp[p:p + 1], ref, lse)
            worst = max(worst, rel)
            assert rel <= B_KERNEL, (p, rel)
        _measured("decode_path_kernel_rel", worst)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 3. exact early exit
# ------------------------------------------------------------------------------------------------
def _cut(sd, E):
    out = {}
    for k, v in sd.items():
        if k.startswith("model.layers."):
            if int(k.split(".")[2]) >= E:
                continue
        out[k] = v
    return out


@pytest.mark.parametrize("prefill_tc", [True, False], ids=["wgmma", "decode"])
def test_early_exit_is_bit_identical_to_the_cut_model(prefill_tc):
    dims = _dims(1000, 512, 1408, 4, 8, 4, 64)
    sd = orc.random_state_dict(dims, 31)
    seqs = [_ids(dims.vocab, n, 40 + n) for n in (2, 40, 300)]       # 300: three 128-token chunks
    eng = _engine(dims, sd, 320, prefill_tc=prefill_tc)
    try:
        got = {(E, len(s)): eng.score(s, E) for E in (1, 2) for s in seqs}
        full = {len(s): eng.score(s, -1) for s in seqs}
        full4 = {len(s): eng.score(s, 4) for s in seqs}
    finally:
        eng.close()
    for s in seqs:
        assert torch.equal(full[len(s)][0], full4[len(s)][0]), "E = L must equal full depth"
    for E in (1, 2):
        cut_dims = _dims(1000, 512, 1408, E, 8, 4, 64)
        cut = _engine(cut_dims, _cut(sd, E), 320, prefill_tc=prefill_tc)
        try:
            for s in seqs:
                lp, gr = cut.score(s)
                assert torch.equal(lp, got[(E, len(s))][0]), (E, len(s))
                assert torch.equal(gr, got[(E, len(s))][1]), (E, len(s))
                # 8. planted: E off by one is a different sub-model
                other = got.get((3 - E, len(s)))
                if other is not None and len(s) > 2:
                    assert not torch.equal(lp, other[0])
        finally:
            cut.close()


# ------------------------------------------------------------------------------------------------
# 4. against the oracle
# ------------------------------------------------------------------------------------------------
def _oracle_logprob(w, ids, E, keep_logits=False):
    """Oracle log-probabilities of ids[1:], arg-max, top-2 margin and max |logit| per row."""
    with torch.inference_mode():
        if E > 0:
            logits = orc.early_exit_logits(w, ids[:1], ids[1:], E)
        else:
            logits = orc.teacher_forced_logits(w, ids[:1], ids[1:])
    ref, _lse, am = _ref_logprob(logits, torch.tensor(ids[1:]))
    top = torch.topk(logits, 2, dim=-1).values.double()
    out = (ref, am, top[:, 0] - top[:, 1], logits.abs().amax(dim=-1).double())
    return out + (logits,) if keep_logits else out


def _check_rows(lp, greedy, ref, am, margin, bound, gate_bound, tag):
    d = (lp.double() - ref).abs()
    assert bool((d <= bound).all()), f"{tag}: worst |dlogprob| {float((d / bound).max()):.3g} x bound"
    gate = margin >= gate_bound
    bad = (greedy != am) & gate
    assert not bool(bad.any()), f"{tag}: greedy differs from the oracle at rows {bad.nonzero().flatten().tolist()}"
    return float(d.max()), float((d / bound).max())


def _golden_models():
    out, seen = [], set()
    for c in gu.spec_cases(greedy=True):
        key = (c["model"], c["weight_seed"], c["damp_from"], c["alpha"])
        if c["name"] in ("survey_a0.1", "mha128_a1.0", "gqa128_a0.1", "gqa128_a0.05_long") and key not in seen:
            seen.add(key)
            out.append(c)
    return out


@pytest.mark.parametrize("case", _golden_models(), ids=lambda c: c["name"])
def test_score_matches_oracle_on_golden_models(case):
    dims, sd = gu.state_dict_for(case)
    w = orc.weights_from_state_dict(dims, sd)
    ids = list(case["prompt"]) + list(case["reference"]["spec_tokens"])
    E = case["cfg"]["exit_layer"]
    eng = _engine(dims, sd, 512)
    pu.set_oracle_threads()
    try:
        for e in (-1, E):
            lp, greedy = eng.score(ids, e)
            ref, am, margin, _ = _oracle_logprob(w, ids, e)
            worst, _ = _check_rows(lp, greedy, ref, am, margin, torch.full_like(ref, B_GOLDEN),
                                   torch.full_like(ref, pu.TAU), f"{case['name']} E={e}")
            _measured(f"golden_{case['name']}_E{e}_abs", worst)
    finally:
        eng.close()


@pytest.mark.parametrize("name", list(WIDTHS))
def test_score_matches_oracle_at_width(name):
    (v, h, i, nl, nh, nkv, hd), theta, scaling, tied, seed, lengths = WIDTHS[name]
    dims = _dims(v, h, i, nl, nh, nkv, hd, theta, scaling)
    sd = orc.random_state_dict(dims, seed)
    if tied:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    w = orc.weights_from_state_dict(dims, sd)
    ids = _ids(v, max(lengths), 300 + seed)
    pu.set_oracle_threads()
    refs = {E: _oracle_logprob(w, ids, E, keep_logits=(name == "w7b" and E == -1)) for E in (1, -1)}
    paths = (True, False) if name == "mha32" else (None,)
    for prefill_tc in paths:
        eng = _engine(dims, sd, max(lengths) + 8, prefill_tc=prefill_tc)
        try:
            worst = 0.0
            for E in (1, -1):
                ref, am, margin, mx = refs[E][:4]
                for n in lengths:
                    lp, greedy = eng.score(ids[:n], E)
                    k = n - 1
                    bound = REL_WIDTH * mx[:k]
                    _, f = _check_rows(lp, greedy, ref[:k], am[:k], margin[:k], bound, 2 * REL_LOGIT * mx[:k],
                                       f"{name} E={E} n={n}")
                    worst = max(worst, f)
                    if n == max(lengths) and E == -1 and name == "w7b":
                        _planted(lp, ids[:n], ref[:k], bound, eng, refs[E][4])
            _measured(f"width_{name}_{'tc' if prefill_tc is not False else 'decode'}_worst_rel", worst * REL_WIDTH)
        finally:
            eng.close()


def _planted(lp, ids, ref, bound, eng, logits):
    """8. shifted targets, a neighbour's row and E off by one must each exceed the oracle bound."""
    d = lp.double()
    x = logits.double()
    lse = torch.logsumexp(x, -1)
    shifted = x[:-1].gather(1, torch.tensor(ids[2:]).view(-1, 1)).squeeze(1) - lse[:-1]   # target of the next row
    f_shift = float(((d[:-1] - shifted).abs() / bound[:-1]).max())
    f_neigh = float(((d[1:] - ref[:-1]).abs() / bound[:-1]).max())
    lp1, _ = eng.score(ids, 1)                                        # E = 1 against the full-depth oracle
    f_exit = float(((lp1.double() - ref).abs() / bound).max())
    _measured("planted_shifted_targets_factor", f_shift)
    _measured("planted_neighbour_row_factor", f_neigh)
    _measured("planted_exit_off_by_one_factor", f_exit)
    assert f_shift > 1 and f_neigh > 1 and f_exit > 1, (f_shift, f_neigh, f_exit)


# ------------------------------------------------------------------------------------------------
# 5. against greedy generation
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prefill_tc", [True, False], ids=["wgmma", "decode"])
def test_score_greedy_matches_generation(prefill_tc):
    case = next(c for c in gu.spec_cases(greedy=True) if c["name"] == "gqa128_a0.05_long")
    dims, sd = gu.state_dict_for(case)
    w = orc.weights_from_state_dict(dims, sd)
    prompt = list(case["prompt"])
    E = case["cfg"]["exit_layer"]
    eng = _engine(dims, sd, 512, prefill_tc=prefill_tc)
    pu.set_oracle_threads()
    try:
        for e in (-1, E):
            eng.begin(e, 64, [])
            eng.prefill(prompt)
            out = [eng.ar_step() for _ in range(64)]
            ids = prompt + out
            _, greedy = eng.score(ids, e)
            got = greedy[len(prompt) - 1:].tolist()
            flips = [j for j in range(64) if got[j] != out[j]]
            if not prefill_tc:
                assert not flips, f"decode path must equal generation exactly (E={e}): {flips}"
            if flips:
                _, _, margin, _ = _oracle_logprob(w, ids, e)
                for j in flips:
                    assert float(margin[len(prompt) - 1 + j]) < pu.TAU, (e, j)
            _measured(f"generation_flips_{'tc' if prefill_tc else 'decode'}_E{e}", len(flips))
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 6. state and determinism
# ------------------------------------------------------------------------------------------------
def _state_model():
    dims = _dims(1000, 512, 1408, 4, 8, 4, 64)
    return dims, orc.random_state_dict(dims, 51)


def test_score_is_deterministic_and_page_table_blind():
    dims, sd = _state_model()
    ids = _ids(dims.vocab, 300, 9)
    eng = _engine(dims, sd, 384)
    perm = _engine(dims, sd, 384)
    try:
        n_pages = (384 + 63) // 64
        perm.debug_set_page_table(torch.randperm(n_pages, generator=torch.Generator().manual_seed(3)).tolist())
        for E in (2, -1):
            a, b, p = eng.score(ids, E), eng.score(ids, E), perm.score(ids, E)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
            assert torch.equal(a[0], p[0]) and torch.equal(a[1], p[1])
    finally:
        eng.close()
        perm.close()


def test_score_ends_the_generation_and_leaves_rounds_unchanged():
    from layerskip_b200 import _lib as L
    dims, sd = _state_model()
    prompt = _ids(dims.vocab, 40, 12)

    def rounds(eng):
        eng.begin(2, 40, [])
        eng.prefill(prompt)
        return [eng.round(4) for _ in range(6)]

    fresh = _engine(dims, sd, 384)
    eng = _engine(dims, sd, 384)
    try:
        want = rounds(fresh)
        first = rounds(eng)
        assert first == want
        eng.score(_ids(dims.vocab, 200, 13), 2)
        with pytest.raises(L.LskError) as ex:
            eng.round(4)
        assert ex.value.code == -3
        with pytest.raises(L.LskError) as ex:
            eng.ar_step()
        assert ex.value.code == -3
        assert rounds(eng) == want
    finally:
        fresh.close()
        eng.close()


def test_score_independent_of_keep_logits_and_lm_head_choice(monkeypatch):
    dims, sd = _state_model()
    ids = _ids(dims.vocab, 300, 14)
    plain = _engine(dims, sd, 384)
    keep = _engine(dims, sd, 384, keep_logits=True)
    monkeypatch.setenv("LSK_LMHEAD_TC", "1")
    tc = _engine(dims, sd, 384)
    monkeypatch.delenv("LSK_LMHEAD_TC")
    try:
        for E in (1, -1):
            a, b, c = plain.score(ids, E), keep.score(ids, E), tc.score(ids, E)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
            assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
            # the last LM-head slice's logits reproduce its log-probabilities (target offset inside
            # the engine): rows 0 .. n-2 in 128-row chunks, each in max_rows slices
            rows = len(ids) - 1
            c0 = (rows - 1) // 128 * 128
            r0 = c0 + (rows - c0 - 1) // keep.max_rows * keep.max_rows
            M = rows - r0
            logits = keep.debug_logits(M)
            ref, lse, am = _ref_logprob(logits, torch.tensor(ids[r0 + 1:r0 + 1 + M]))
            rel = _kernel_rel(b[0][r0:], ref, lse)
            _measured("last_slice_kernel_rel", rel)
            assert rel <= B_KERNEL
            assert torch.equal(b[1][r0:], am)
            # 8. planted: targets shifted by one inside the slice
            ref_s, _, _ = _ref_logprob(logits[:-1], torch.tensor(ids[r0 + 2:r0 + 1 + M]))
            f = _kernel_rel(b[0][r0:-1], ref_s, lse[:-1]) / B_KERNEL
            _measured("planted_slice_target_shift_factor", f)
            assert f > 1
    finally:
        plain.close()
        keep.close()
        tc.close()


# ------------------------------------------------------------------------------------------------
# 7. errors
# ------------------------------------------------------------------------------------------------
def test_score_argument_errors():
    from layerskip_b200 import _lib as L
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    dims = _dims(512, 256, 688, 2, 8, 8, 32)
    sd = orc.random_state_dict(dims, 0)
    eng = _engine(dims, sd, 64)
    arch = LlamaArch(512, 256, 688, 2, 8, 8, 32)

    def expect(code, needle, fn):
        with pytest.raises(L.LskError) as ex:
            fn()
        assert ex.value.code == code, (ex.value.code, str(ex.value))
        assert needle in str(ex.value), str(ex.value)

    try:
        expect(-1, "at least 2", lambda: eng.score([5]))
        expect(-1, "out of range", lambda: eng.score([5, 512]))
        expect(-1, "out of range", lambda: eng.score([-1, 5]))
        expect(-1, "exit_layer", lambda: eng.score([5, 6], 3))
        expect(-6, "max_ctx", lambda: eng.score(list(range(3, 3 + 65))))
        lib = L.load()
        arr = (C.c_int32 * 2)(5, 6)
        out = (C.c_float * 1)()
        assert lib.lsk_score(None, arr, 2, -1, out, None) == -1
        assert lib.lsk_score(eng._h, None, 2, -1, out, None) == -1
        assert lib.lsk_score(eng._h, arr, 2, -1, None, None) == -1
        assert lib.lsk_score(eng._h, arr, 2, -1, out, None) == 0          # greedy_out may be NULL
        empty = Engine(arch, max_ctx=64)
        try:
            expect(-3, "weights", lambda: empty.score([5, 6]))
        finally:
            empty.close()
        tp = Engine(arch, max_ctx=64, tp_rank=0, tp_size=2)
        try:
            expect(-1, "tensor-parallel", lambda: tp.score([5, 6]))
        finally:
            tp.close()
    finally:
        eng.close()

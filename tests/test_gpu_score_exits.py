"""GPU: multi-exit scoring (`lsk_score_exits` / `Engine.score_exits`) and the acceptance prediction.

1. bit-identity: every exit's log-probability and greedy rows equal `score(ids, E)` bit for bit, on
   both prompt routes, at the golden spec-case models and at 7B / 8B / llama3.2-1B / head_dim-32
   widths (3-layer models), at 2 .. 1101 ids, for one exit, {1, 2, 3} and sets with and without
   full depth; also with the acceptance rows on, a permuted page table and a repeat run;
2. one pass: the launch count is `score(ids, max exit)`'s plus exactly the heads of the other exits
   and the warp / acceptance kernels;
3. the acceptance kernels alone against a float64 sum of min of the oracle's warped softmaxes;
4. greedy prediction: `predict.greedy_rounds` over one scoring pass of prompt + output equals the
   rounds greedy self-speculation ran, exactly on the decode-kernel engine, and on the wgmma engine
   up to the first round that touches an oracle near-tie;
5. sampled prediction: over 128 prompts x 128 tokens of sampled self-speculation, the accepted
   drafts minus their acceptance probabilities form a martingale; its z statistic (and that of the
   alpha-weighted sum) stays within 3, and planted errors (alpha one position off, alpha at E - 1)
   fail it;
6. state and refusals.

Bounds: DESIGN.md §7, at most 2x the worst value measured on an H100 80GB HBM3.  Measured values
are printed as `MEASURED <name> <value>`."""
import ctypes as C
import math

import pytest
import torch

from oracle import llama_oracle as orc
from tests import golden_util as gu
from tests import parity_util as pu
from tests.test_gpu_engine import _Model
from tests.test_gpu_score import LLAMA3, _dims, _engine, _golden_models, _ids, _oracle_logprob

pytestmark = pytest.mark.gpu

# |alpha - float64 sum min| of the acceptance kernels on fp32 logits (measured worst 4.2e-7)
B_ALPHA = 8e-7
LENGTHS = (2, 17, 18, 40, 129, 300, 1101)
WARPS = [(0.6, 0, 0.9), (1.0, 0, 0.5), (0.9, 12, 0.95), (0.7, 5, 1.0), (1.3, 0, 0.0)]
# name: (vocab, hidden, inter, layers, heads, kv heads, head_dim), theta, rope scaling, tied, seed
WIDTHS = {
    "w7b": ((32000, 4096, 11008, 3, 32, 32, 128), 10000.0, None, False, 31),
    "w8b": ((128256, 4096, 14336, 3, 32, 8, 128), 500000.0, None, False, 32),
    "l32_1b": ((128256, 2048, 8192, 3, 32, 8, 64), 500000.0, LLAMA3, True, 34),
    "mha32": ((512, 256, 688, 3, 8, 8, 32), 10000.0, None, False, 35),
}


def _measured(name, value):
    print(f"MEASURED {name} {value:.4g}", flush=True)


def _exit_sets(L):
    return [[L], [1], sorted({1, 2, min(4, L)}), list(range(1, L)) or [1], list(range(1, L + 1))]


def _check_identical(eng, ids, exits, sampling=None, tag=""):
    lp, gr, acc = eng.score_exits(ids, exits, sampling)
    assert lp.shape == (len(exits), len(ids) - 1) and gr.shape == lp.shape
    for j, E in enumerate(exits):
        a, b = eng.score(ids, E)
        assert torch.equal(lp[j], a), f"{tag} exits={exits} E={E}: log-probabilities differ"
        assert torch.equal(gr[j], b), f"{tag} exits={exits} E={E}: greedy ids differ"
    return lp, gr, acc


# ------------------------------------------------------------------------------------------------
# 1. bit-identity with score(ids, E)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", _golden_models(), ids=lambda c: c["name"])
def test_score_exits_equals_score_on_golden_models(case):
    dims, sd = gu.state_dict_for(case)
    ids = list(case["prompt"]) + list(case["reference"]["spec_tokens"])
    for prefill_tc in (True, False):
        eng = _engine(dims, sd, 512, prefill_tc=prefill_tc)
        try:
            for exits in _exit_sets(dims.layers):
                _check_identical(eng, ids, exits, tag=case["name"])
            _check_identical(eng, ids, list(range(1, dims.layers + 1)),
                             {"temperature": 0.6, "top_k": 0, "top_p": 0.9}, tag=case["name"] + " sampled")
        finally:
            eng.close()


@pytest.mark.parametrize("name", list(WIDTHS))
def test_score_exits_equals_score_at_width(name):
    (v, h, i, nl, nh, nkv, hd), theta, scaling, tied, seed = WIDTHS[name]
    dims = _dims(v, h, i, nl, nh, nkv, hd, theta, scaling)
    sd = orc.random_state_dict(dims, seed)
    if tied:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    ids = _ids(v, max(LENGTHS), 400 + seed)
    sampled = {"temperature": 0.8, "top_k": 40, "top_p": 0.95}
    for prefill_tc in (True, False):
        eng = _engine(dims, sd, max(LENGTHS) + 8, prefill_tc=prefill_tc)
        try:
            for n in LENGTHS:
                for exits in _exit_sets(nl):
                    _check_identical(eng, ids[:n], exits, tag=f"{name} n={n} tc={prefill_tc}")
            _, _, acc = _check_identical(eng, ids[:300], [1, 2, nl], sampled, tag=f"{name} sampled")
            assert acc.shape == (2, 299) and bool(((acc >= 0) & (acc <= 1.0001)).all())
        finally:
            eng.close()


def test_score_exits_is_repeatable_and_page_table_blind():
    dims = _dims(1000, 512, 1408, 4, 8, 4, 64)
    sd = orc.random_state_dict(dims, 51)
    ids = _ids(dims.vocab, 300, 9)
    warp = {"temperature": 0.7, "top_k": 0, "top_p": 0.9}
    eng = _engine(dims, sd, 384)
    perm = _engine(dims, sd, 384)
    try:
        perm.debug_set_page_table(torch.randperm(6, generator=torch.Generator().manual_seed(3)).tolist())
        for exits in ([1, 2, 4], [2, 3]):
            a = _check_identical(eng, ids, exits, warp if exits[-1] == 4 else None, "plain")
            b = eng.score_exits(ids, exits, warp if exits[-1] == 4 else None)
            p = _check_identical(perm, ids, exits, warp if exits[-1] == 4 else None, "permuted")
            for x, y, z in zip(a, b, p):
                assert (x is None and y is None and z is None) or (torch.equal(x, y) and torch.equal(x, z))
    finally:
        eng.close()
        perm.close()


# ------------------------------------------------------------------------------------------------
# 2. one pass
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prefill_tc", [True, False], ids=["wgmma", "decode"])
def test_score_exits_launches_one_pass(prefill_tc):
    dims = _dims(1000, 512, 1408, 4, 8, 4, 64)
    sd = orc.random_state_dict(dims, 52)
    eng = _engine(dims, sd, 384, prefill_tc=prefill_tc)
    warp = {"temperature": 0.7, "top_k": 0, "top_p": 0.9}

    def launches(fn):
        before = eng.launch_count
        fn()
        return eng.launch_count - before

    try:
        # launches of one head (LM-head GEMM + log-probability kernel): a 1-row score is the embed
        # gather, E layers and one head
        l1, l2 = launches(lambda: eng.score([5, 6], 1)), launches(lambda: eng.score([5, 6], 2))
        head = l1 - 1 - (l2 - l1)
        assert head >= 2
        for n in (2, 18, 300):
            ids = _ids(dims.vocab, n, n)
            rows = n - 1
            if prefill_tc and rows > eng.max_rows:
                slices = sum(-(-min(128, rows - c0) // eng.max_rows) for c0 in range(0, rows, 128))
            else:
                slices = -(-rows // eng.max_rows)
            for exits, sampled in (([4], False), ([1, 2, 4], False), ([1, 3, 4], True), ([2, 3], False)):
                base = launches(lambda: eng.score(ids, exits[-1]))
                k = len(exits)
                got = launches(lambda: eng.score_exits(ids, exits, warp if sampled else None))
                want = base + slices * (k - 1) * head + (slices * k if sampled and k > 1 else 0)
                assert got == want, (n, exits, sampled, got, want)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# 3. the acceptance kernels alone
# ------------------------------------------------------------------------------------------------
def _run_accept(draft, verify, vocab, ld, t, k, p):
    from layerskip_b200 import _lib as L
    lib = L.load()
    rows = draft.shape[0]
    out = torch.empty(rows, dtype=torch.float32, device="cuda")
    gen = L.lsk_generation(sample=1, temperature=t, top_k=k, top_p=p)
    L.check(lib.lsk_test_accept(draft.data_ptr(), verify.data_ptr(), rows, vocab, ld, C.byref(gen), out.data_ptr()))
    return out.cpu()


def _ref_accept(draft, verify, t, k, p):
    pd = torch.softmax(orc.warp_top_k_top_p(draft.double() / t, k, p), dim=-1)
    pv = torch.softmax(orc.warp_top_k_top_p(verify.double() / t, k, p), dim=-1)
    return torch.minimum(pd, pv).sum(-1)


@pytest.mark.parametrize("vocab", [512, 32000, 32001, 128256])
def test_accept_kernel_matches_float64(vocab):
    g = torch.Generator().manual_seed(vocab)
    base = torch.randn(6, vocab, generator=g) * 3
    draft = base + torch.randn(6, vocab, generator=g) * torch.tensor([0.1, 0.5, 1.0, 2.0, 4.0, 8.0]).view(-1, 1)
    verify = base.clone()
    same = torch.randn(2, vocab, generator=g) * 2                     # identical rows: alpha = 1
    dis_d = torch.randn(2, vocab, generator=g) * 0.1                  # disjoint supports: alpha = 0
    dis_v = dis_d.clone()
    for r in range(2):
        dis_d[r, :5] = torch.tensor([30.0, 29.0, 28.0, 27.0, 26.0])
        dis_v[r, vocab - 5:] = torch.tensor([30.0, 29.0, 28.0, 27.0, 26.0])
    draft = torch.cat([draft, same, dis_d])
    verify = torch.cat([verify, same, dis_v])
    ld = (vocab + 15) // 16 * 16 + 16
    pad_d = torch.full((draft.shape[0], ld), 1e30)                     # pad columns must never count
    pad_v = pad_d.clone()
    pad_d[:, :vocab], pad_v[:, :vocab] = draft, verify
    worst = 0.0
    for t, k, p in WARPS:
        got = _run_accept(pad_d.cuda(), pad_v.cuda(), vocab, ld, t, k, p)
        want = _ref_accept(draft, verify, t, k, p)
        d = (got.double() - want).abs()
        worst = max(worst, float(d.max()))
        assert float(d.max()) <= B_ALPHA, (t, k, p, d.tolist())
        assert bool((got[6:8] - 1).abs().max() <= B_ALPHA), got[6:8]
        assert torch.equal(got[8:], torch.zeros(2)), got[8:]
        assert torch.equal(got, _run_accept(pad_d.cuda(), pad_v.cuda(), vocab, ld, t, k, p))   # reproducible
    _measured(f"accept_kernel_abs_vocab{vocab}", worst)


# ------------------------------------------------------------------------------------------------
# 4. greedy prediction
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prefill_tc", [False, True], ids=["decode", "wgmma"])
def test_greedy_prediction_equals_the_rounds(prefill_tc):
    from layerskip_b200 import GenerationConfig, predict
    from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy
    case = next(c for c in gu.spec_cases(greedy=True) if c["name"] == "gqa128_a0.05_long")
    dims, sd = gu.state_dict_for(case)
    model = _Model(dims, sd)
    E0 = case["cfg"]["exit_layer"]
    others = [e for e in range(1, dims.layers) if e != E0]
    exits = sorted({E0, others[-1]})
    prompt = list(case["prompt"])
    steps = 96
    strat = B200SelfSpeculativeGenerationStrategy(max_ctx=512, prefill_tc=prefill_tc)
    w = orc.weights_from_state_dict(dims, sd) if prefill_tc else None
    checked = differing = 0
    try:
        eng = strat.engine_for(model)
        for E in exits:
            for D in (1, 3, 6, 15):
                cfg = GenerationConfig(max_steps=steps, exit_layer=E, num_speculations=D, sample=False)
                res = strat.generate_token_ids(model, prompt, [], cfg)
                out = res.predicted_tokens
                assert len(out) == steps
                want = [(r.n_drafted, r.n_matches) for r in strat.last_rounds]
                _, greedy, _ = eng.score_exits(prompt + out, [E])
                agree = (greedy[0, len(prompt) - 1:] == torch.tensor(out)).tolist()
                got = predict.greedy_rounds(agree, D, steps)
                checked += 1
                if not prefill_tc:
                    assert got == want, (E, D)
                    assert predict.acceptance_rate(got) == res.acceptance_rate
                    continue
                if got == want:
                    assert predict.acceptance_rate(got) == res.acceptance_rate
                    continue
                # the first differing round must touch a near-tie of the oracle (E or full depth)
                differing += 1
                i = next(j for j, (a, b) in enumerate(zip(got, want)) if a != b)
                o = sum(n + 1 for _, n in want[:i])
                pos = range(len(prompt) - 1 + o, len(prompt) - 1 + o + want[i][0] + 1)
                ids = prompt + out
                pu.set_oracle_threads()
                m = min(float(_oracle_logprob(w, ids, e)[2][q]) for e in (E, -1) for q in pos)
                assert m < pu.TAU, (E, D, i, m)
    finally:
        strat.engines.close()
    _measured(f"greedy_prediction_differing_runs_{'tc' if prefill_tc else 'decode'}", differing)
    assert checked == 2 * 4


# ------------------------------------------------------------------------------------------------
# 5. sampled prediction: alpha is the acceptance probability
# ------------------------------------------------------------------------------------------------
def _z(events):
    """events: (accepted 0/1, alpha).  z of sum(acc - alpha), and of the alpha-weighted sum
    sum((alpha - mean) (acc - alpha)): both are martingales when alpha is each draft's acceptance
    probability given its prefix."""
    a = torch.tensor([x for x, _ in events], dtype=torch.float64)
    p = torch.tensor([y for _, y in events], dtype=torch.float64).clamp(0, 1)
    var = p * (1 - p)
    z1 = float((a - p).sum() / var.sum().sqrt())
    wgt = p - p.mean()
    z2 = float((wgt * (a - p)).sum() / (wgt * wgt * var).sum().sqrt())
    return z1, z2


def test_sampled_alpha_is_the_acceptance_probability():
    from layerskip_b200 import GenerationConfig
    from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy
    case = next(c for c in gu.spec_cases() if c["name"] == "gqa128_sample_s3")
    dims, sd = gu.state_dict_for(case)
    # Random weights give nearly flat next-token distributions, whose overlap alpha is almost the
    # same at every position, so alpha one position off would pass unnoticed.  A sharpened LM head
    # makes the distributions peaked: alpha then varies along the text (near 1 where E and full
    # depth agree, lower where they do not).  The model is damped from layer 3, so E = 2 is where
    # the two differ.
    sd = dict(sd, **{"lm_head.weight": sd["lm_head.weight"] * 8})
    model = _Model(dims, sd)
    E, D, steps = 2, 6, 128
    warp = {"temperature": 0.6, "top_k": 0, "top_p": 0.9}
    cfg = GenerationConfig(max_steps=steps, exit_layer=E, num_speculations=D, sample=True, **warp)
    strat = B200SelfSpeculativeGenerationStrategy(max_ctx=512)
    prompts = torch.randint(3, dims.vocab - 1, (128, 12), generator=torch.Generator().manual_seed(2025)).tolist()
    true_ev, shift_ev, lower_ev = [], [], []
    try:
        eng = strat.engine_for(model)
        for i, p in enumerate(prompts):
            torch.manual_seed(700 + i)
            out = strat.generate_token_ids(model, p, [], cfg).predicted_tokens
            rounds = strat.last_rounds
            _, _, acc = eng.score_exits(p + out, [E - 1, E, dims.layers], warp)
            base = len(p) - 1
            o = 0
            for r in rounds:
                for j in range(min(r.n_matches + 1, r.n_drafted)):          # drafts the accept test evaluated
                    q = base + o + j
                    hit = 1.0 if j < r.n_matches else 0.0
                    true_ev.append((hit, float(acc[1, q])))
                    lower_ev.append((hit, float(acc[0, q])))
                    if q + 1 < acc.shape[1]:
                        shift_ev.append((hit, float(acc[1, q + 1])))
                o += r.n_matches + 1
    finally:
        strat.engines.close()
    z = _z(true_ev)
    al = torch.tensor([b for _, b in true_ev], dtype=torch.float64)
    print(f"sampled acceptance: {len(true_ev)} evaluated drafts, accepted {sum(a for a, _ in true_ev) / len(true_ev):.4f}, "
          f"mean alpha {float(al.mean()):.4f} (std {float(al.std()):.4f}), z = {z[0]:.2f}, weighted z = {z[1]:.2f}")
    _measured("sampled_z", abs(z[0]))
    _measured("sampled_weighted_z", abs(z[1]))
    assert abs(z[0]) <= 3 and abs(z[1]) <= 3, z
    for tag, ev in (("shifted_by_one", shift_ev), ("exit_minus_one", lower_ev)):
        f = max(abs(x) for x in _z(ev)) / 3
        _measured(f"planted_{tag}_factor", f)
        assert f > 1, (tag, _z(ev))


# ------------------------------------------------------------------------------------------------
# 6. state and refusals
# ------------------------------------------------------------------------------------------------
def test_score_exits_refusals_and_state():
    from layerskip_b200 import _lib as L
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import LlamaArch
    dims = _dims(1000, 512, 1408, 4, 8, 4, 64)
    sd = orc.random_state_dict(dims, 53)
    prompt = _ids(dims.vocab, 40, 12)
    warp = {"temperature": 0.7, "top_k": 0, "top_p": 0.9}

    def rounds(eng):
        eng.begin(2, 40, [])
        eng.prefill(prompt)
        return [eng.round(4) for _ in range(6)]

    def expect(code, needle, fn):
        with pytest.raises(L.LskError) as ex:
            fn()
        assert ex.value.code == code, (ex.value.code, str(ex.value))
        assert needle in str(ex.value), str(ex.value)

    fresh = _engine(dims, sd, 128)
    eng = _engine(dims, sd, 128)
    ids = _ids(dims.vocab, 100, 13)
    try:
        want = rounds(fresh)
        assert rounds(eng) == want
        good = eng.score_exits(ids, [1, 2, 4], warp)
        expect(-1, "at least 2", lambda: eng.score_exits([5], [1]))
        expect(-6, "max_ctx", lambda: eng.score_exits(list(range(3, 3 + 129)), [1]))
        expect(-1, "out of range", lambda: eng.score_exits([5, dims.vocab], [1]))
        expect(-1, "out of range", lambda: eng.score_exits([-1, 5], [1]))
        expect(-1, "n_exits", lambda: eng.score_exits(ids, []))
        expect(-1, "n_exits", lambda: eng.score_exits(ids, list(range(1, 34))))
        expect(-1, "strictly increasing", lambda: eng.score_exits(ids, [2, 1]))
        expect(-1, "strictly increasing", lambda: eng.score_exits(ids, [2, 2]))
        expect(-1, "outside", lambda: eng.score_exits(ids, [0, 2]))
        expect(-1, "outside", lambda: eng.score_exits(ids, [1, 5]))
        expect(-1, "full depth", lambda: eng.score_exits(ids, [1, 2], warp))
        expect(-1, "temperature", lambda: eng.score_exits(ids, [1, 4], dict(warp, temperature=0.0)))
        lib = L.load()
        arr = (C.c_int32 * 3)(5, 6, 7)
        ex = (C.c_int32 * 2)(1, 4)
        lp = (C.c_float * 4)()
        acc = (C.c_float * 2)()
        greedy_gen = L.lsk_generation(sample=0, temperature=0.7, top_p=0.9)
        ngram_gen = L.lsk_generation(sample=1, temperature=0.7, top_p=0.9, no_repeat_ngram_size=3)
        assert lib.lsk_score_exits(None, arr, 3, ex, 2, None, lp, None, None) == -1
        assert lib.lsk_score_exits(eng._h, None, 3, ex, 2, None, lp, None, None) == -1
        assert lib.lsk_score_exits(eng._h, arr, 3, None, 2, None, lp, None, None) == -1
        assert lib.lsk_score_exits(eng._h, arr, 3, ex, 2, None, None, None, None) == -1
        assert lib.lsk_score_exits(eng._h, arr, 3, ex, 2, None, lp, None, acc) == -1          # accept without settings
        assert lib.lsk_score_exits(eng._h, arr, 3, ex, 2, C.byref(greedy_gen), lp, None, acc) == -1
        assert lib.lsk_score_exits(eng._h, arr, 3, ex, 2, C.byref(ngram_gen), lp, None, acc) == -1
        assert "n-gram" in lib.lsk_last_error().decode()
        assert lib.lsk_score_exits(eng._h, arr, 3, ex, 2, None, lp, None, None) == 0           # greedy_out may be NULL
        # every refusal left the engine usable: the same call gives the same bits
        again = eng.score_exits(ids, [1, 2, 4], warp)
        assert all(torch.equal(x, y) for x, y in zip(good, again))
        # the call ended the generation: rounds need a new prefill, then equal a fresh engine's
        expect(-3, "", lambda: eng.round(4))
        expect(-3, "", lambda: eng.ar_step())
        assert rounds(eng) == want
        arch = LlamaArch(512, 256, 688, 2, 8, 8, 32)
        empty = Engine(arch, max_ctx=64)
        try:
            expect(-3, "weights", lambda: empty.score_exits([5, 6], [1]))
        finally:
            empty.close()
        tp = Engine(arch, max_ctx=64, tp_rank=0, tp_size=2)
        try:
            expect(-1, "tensor-parallel", lambda: tp.score_exits([5, 6], [1]))
        finally:
            tp.close()
    finally:
        fresh.close()
        eng.close()

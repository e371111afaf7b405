"""GPU: the library's memory plan (`lsk_plan_memory`) is what an engine really holds
(`lsk_memory_in_use`), per category and to the byte: after `lsk_create`, and after each call that
allocates on first use, against the plan of the uses made so far.

On tiny-mha, tiny-gqa and a two-layer Llama-2-7B-width model, each with the default flags, with
LSK_FLAG_KEEP_LOGITS, without the prompt pass and with attn_splits = 3.  The two-layer model has at
most two exits, so its exit counts are capped at two."""
import ctypes as C
import os

import pytest
import torch

from layerskip_b200 import _lib
from oracle import llama_oracle as orc
from tests.test_gpu_score import _dims, _engine, _ids

pytestmark = pytest.mark.gpu

MAX_CTX = 512
ARCHS = {
    "tiny-mha": _dims(512, 256, 704, 4, 2, 2, 128),
    "tiny-gqa": _dims(640, 512, 1408, 6, 4, 2, 128),
    "llama2-7b-l2": _dims(32000, 4096, 11008, 2, 32, 32, 128),
}
VARIANTS = {
    "default": {},
    "keep_logits": dict(keep_logits=True),
    "no_prefill_tc": dict(prefill_tc=False),
    "attn_splits_3": dict(attn_splits=3),
}
SAMPLING = dict(temperature=0.8, top_k=0, top_p=0.95)

_sd = {}


def _state_dict(name):
    if name not in _sd:
        _sd.clear()
        _sd[name] = orc.random_state_dict(ARCHS[name], seed=7)
    return _sd[name]


def _fields(plan):
    return {name: getattr(plan, name) for name, _ in _lib.lsk_memory_plan._fields_}


def _planned(eng, attn_splits, **uses):
    flags = (_lib.LSK_FLAG_KEEP_LOGITS if eng.keep_logits else 0) | \
        (0 if eng.prefill_tc else _lib.LSK_FLAG_NO_PREFILL_TC)
    cfg = eng.arch.lsk_config(MAX_CTX, attn_splits=attn_splits, flags=flags)
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    u = _lib.lsk_memory_uses(lm_head_tc=int(os.environ.get("LSK_LMHEAD_TC", "0") not in ("", "0")), **uses)
    plan = _lib.lsk_memory_plan()
    _lib.check(eng._lib.lsk_plan_memory(C.byref(cfg), sms, C.byref(u), C.byref(plan)))
    return _fields(plan)


def _in_use(eng):
    plan = _lib.lsk_memory_plan()
    _lib.check(eng._lib.lsk_memory_in_use(eng._h, C.byref(plan)))
    return _fields(plan)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", list(ARCHS))
def test_memory_in_use_is_the_plan_after_every_call(name, variant):
    dims, kw = ARCHS[name], VARIANTS[variant]
    eng = _engine(dims, _state_dict(name), MAX_CTX, **kw)
    try:
        L, V = dims.layers, dims.vocab
        uses = {}

        def check(step):
            assert _in_use(eng) == _planned(eng, kw.get("attn_splits", 0), **uses), step

        check("lsk_create")
        eng.begin(exit_layer=1, max_steps=64, eos_token_ids=[V - 1], sample=True, seed=3, **SAMPLING)
        uses["sampling"] = 1
        check("begin(sample=True)")
        eng.begin(exit_layer=1, max_steps=64, eos_token_ids=[V - 1], no_repeat_ngram_size=3)
        uses["ngram_ban"] = 1
        check("begin(no_repeat_ngram_size=3)")
        eng.prefill(_ids(V, 40, 1))
        eng.round_adaptive(4, 0.5)
        uses["adaptive"] = 1
        check("round_adaptive")
        eng.score(_ids(V, 200, 2), 1)
        uses["score_exits"] = 1
        check("score")
        eng.score_exits(_ids(V, 150, 3), [L], sampling=SAMPLING)
        uses["accept_exits"] = 1
        check("score_exits, one exit, sampled: no draft exit")
        for k in (3, 2, 4):                        # grow, no shrink, regrow
            k = min(k, L)
            eng.score_exits(_ids(V, 150, 4 + k), list(range(L - k + 1, L + 1)), sampling=SAMPLING)
            uses["score_exits"] = max(uses["score_exits"], k)
            uses["accept_exits"] = max(uses["accept_exits"], k)
            check(f"score_exits, {k} exits, sampled")
        seqs = [_ids(V, n, 10 + n) for n in (30, 150, 7)]
        uses["packed_scoring"] = 1
        if eng.prefill_tc:
            eng.score_batch(seqs, 1)
        else:                                      # refused before it allocates
            with pytest.raises(_lib.LskError, match="wgmma prompt pass"):
                eng.score_batch(seqs, 1)
        check("score_batch")
        if eng.prefill_tc:
            eng.score_prefixed([_ids(V, 70, 20)], [(0, _ids(V, 9, 21)), (0, _ids(V, 140, 22))], 1)
            check("score_prefixed")
    finally:
        eng.close()


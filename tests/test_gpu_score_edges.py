"""GPU: the exact equalities of packed, prefix-shared and multi-exit scoring at Llama-3.2-3B's layout
(24 heads over 8 kv heads: group 3), where the prompt pass's attention runs 80 tokens per launch and
packed scoring cuts its pieces at 80-token points instead of 128 / 64 / 32, with sequences of more
than 2000 ids (test_gpu_score_batch.py, test_gpu_score_prefixed.py, test_gpu_score_exits.py):

- `score_batch` == `score` of each sequence alone;
- `score_prefixed` == `score_batch` / `score` of the joined sequences;
- `score_exits` == `score` at every exit, on both prompt routes."""
import pytest
import torch

from oracle import llama_oracle as orc
from tests import test_gpu_score_batch as sb
from tests import test_gpu_score_exits as se
from tests import test_gpu_score_prefixed as sp
from tests.test_gpu_score import LLAMA3, _dims, _engine, _ids

pytestmark = pytest.mark.gpu

LONGEST = 2300


@pytest.fixture(scope="module")
def l32_3b():
    dims = _dims(128256, 3072, 8192, 2, 24, 8, 128, 500000.0, LLAMA3)
    sd = orc.random_state_dict(dims, 61)
    sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    return dims, sd


def test_score_batch_equals_solo_scoring_at_group_3(l32_3b):
    dims, sd = l32_3b
    eng = _engine(dims, sd, LONGEST + 8)
    try:
        seqs = sb._batch(dims.vocab, 3, sb.LENGTHS + (79, 80, 81, 161, LONGEST))
        for E in (-1, 1):
            sb._assert_same(eng.score_batch(seqs, E), [sb._solo(eng, s, E) for s in seqs], f"l32_3b E={E}")
    finally:
        eng.close()


def test_score_prefixed_equals_the_joined_sequences_at_group_3(l32_3b):
    dims, sd = l32_3b
    eng = _engine(dims, sd, LONGEST)
    try:
        ps, bs = sp._workload(dims.vocab, 3, prefixes=sp.PREFIXES + (80, 81, 2100), fill=LONGEST)
        for E in (-1, 1):
            sp._check_against_joined(eng, ps, bs, E, f"l32_3b E={E}")
    finally:
        eng.close()


def test_score_exits_equals_score_at_group_3(l32_3b):
    dims, sd = l32_3b
    ids = _ids(dims.vocab, LONGEST, 461)
    for prefill_tc in (True, False):
        eng = _engine(dims, sd, LONGEST + 8, prefill_tc=prefill_tc)
        try:
            for n in (18, 81, 300, LONGEST):
                for exits in se._exit_sets(dims.layers):
                    se._check_identical(eng, ids[:n], exits, tag=f"l32_3b n={n} tc={prefill_tc}")
        finally:
            eng.close()

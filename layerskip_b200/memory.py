"""HBM budget of one engine (per GPU), from the library's own table of the buffers it allocates
(`lsk_plan_memory`, `csrc/engine.cu: mem_table`) — so a configuration that cannot fit is refused with
an explanation BEFORE `cudaMalloc` runs out half-way (H100: 80 GB of HBM3 per GPU).

Dominant terms: packed bf16 weights (the per-rank shard under tensor parallelism; embeddings are
replicated), and the paged KV pool `2 x layers x pages x kv_heads_local x 64 x 128 x 2 B`.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

from . import _lib
from .weights import LlamaArch

HBM_PER_GPU = 80e9                  # H100 SXM


def plan_memory(arch: LlamaArch, max_ctx: int = 4096, tp_size: int = 1, sampling: bool = False,
                keep_logits: bool = False, lm_head_tc: bool = False, prefill_tc: bool = True,
                scoring: bool = False, batch_scoring: bool = False, score_exits: int = 0,
                score_exits_sampled: bool = False, adaptive: bool = False, ngram_ban: bool = False,
                batch_seqs: int = 0, sm_count: int = 132) -> Dict[str, int]:
    """Bytes the engine allocates on ONE rank of a GPU with `sm_count` SMs (132: H100 SXM).  Keys:
    weights, embed, lm_head, kv_pool, scratch, total (+ weights_source_peak: the largest single
    tensor staged on the GPU while loading).
    Beyond what `lsk_create` allocates, each flag adds what its first call allocates: `sampling` and
    `ngram_ban` a `begin` with sampling / the n-gram ban, `adaptive` a `round_adaptive`, `scoring`
    an `lsk_score`, `score_exits` = k an `lsk_score_exits` with k exits (`score_exits_sampled`: with
    acceptance probabilities), `batch_scoring` an `lsk_score_batch` or `lsk_score_prefixed`,
    `batch_seqs` > 0 an `lsk_prefill_batch` of up to that many sequences (the same buffers for any count;
    with `adaptive`, also `round_batch_adaptive`'s confidence scratch).  With
    tp_size > 1 the peer region of the one-shot collectives is counted."""
    cfg = arch.lsk_config(max_ctx, tp_size=tp_size,
                          flags=(_lib.LSK_FLAG_KEEP_LOGITS if keep_logits else 0) |
                          (0 if prefill_tc else _lib.LSK_FLAG_NO_PREFILL_TC))
    uses = _lib.lsk_memory_uses(lm_head_tc=int(lm_head_tc), sampling=int(sampling), ngram_ban=int(ngram_ban),
                                adaptive=int(adaptive), score_exits=max(score_exits, int(scoring)),
                                accept_exits=score_exits if score_exits_sampled else 0,
                                packed_scoring=int(batch_scoring), tp_peer=int(tp_size > 1),
                                batch_seqs=int(batch_seqs))
    plan = _lib.lsk_memory_plan()
    _lib.check(_lib.load().lsk_plan_memory(C.byref(cfg), sm_count, C.byref(uses), C.byref(plan)))
    out = {name: getattr(plan, name) for name, _ in _lib.lsk_memory_plan._fields_}
    out["weights_source_peak"] = 2 * max(arch.vocab * arch.hidden, arch.inter * arch.hidden)   # one full bf16 tensor while repacking
    return out


def check_fits(arch: LlamaArch, free_bytes: int, **kw) -> Dict[str, int]:
    """Raise MemoryError with the breakdown when the engine (plus the transient source tensor of
    the weight upload) cannot fit into `free_bytes`."""
    plan = plan_memory(arch, **kw)
    need = plan["total"] + plan["weights_source_peak"]
    if need > free_bytes:
        gb = lambda b: f"{b / 1e9:.1f} GB"   # noqa: E731
        raise MemoryError(
            f"engine needs {gb(need)} of HBM on this GPU (weights {gb(plan['weights'])}, embedding "
            f"{gb(plan['embed'])}, LM head {gb(plan['lm_head'])}, KV pool {gb(plan['kv_pool'])} at "
            f"max_ctx={kw.get('max_ctx', 4096)}, upload staging {gb(plan['weights_source_peak'])}) but "
            f"only {gb(free_bytes)} are free; use a larger tp_size or a smaller max_ctx")
    return plan

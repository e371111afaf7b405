"""HBM budget of one engine (per GPU), from the same formulas as the allocations in
`csrc/engine.cu: create_into` — so a configuration that cannot fit is refused with an explanation
BEFORE `cudaMalloc` runs out half-way (H100: 80 GB of HBM3 per GPU).

Dominant terms: packed bf16 weights (the per-rank shard under tensor parallelism; embeddings are
replicated), and the paged KV pool `2 x layers x pages x kv_heads_local x 64 x 128 x 2 B`.
"""
from __future__ import annotations

from typing import Dict

from .weights import LlamaArch

PAGE_TOKENS = 64
MAX_ROWS = 16
HBM_PER_GPU = 80e9                  # H100 SXM
SM_COUNT = 132                      # H100 SXM: one arg-max candidate slot per SM


def plan_memory(arch: LlamaArch, max_ctx: int = 4096, tp_size: int = 1, sampling: bool = False,
                keep_logits: bool = False, lm_head_tc: bool = False, prefill_tc: bool = True,
                scoring: bool = False, batch_scoring: bool = False, score_exits: int = 0,
                score_exits_sampled: bool = False) -> Dict[str, int]:
    """Bytes the engine allocates on ONE rank.  Keys: weights, embed, lm_head, kv_pool, scratch,
    total (+ weights_source_peak: the largest single tensor staged on the GPU while loading).
    `scoring` adds what the first `lsk_score` call allocates: the logits rows (unless already
    there) and one float + one int per position.  `score_exits` = k adds what the first
    `lsk_score_exits` call with k exits allocates: the logits rows and k floats + k ints per
    position; the two share these result arrays, which grow to the most exits asked for.
    `score_exits_sampled` adds, for the k - 1 draft exits, one float per position and the warped
    draft rows of a chunk (128 rows with the prompt pass, 16 without), plus 16 warped full-depth
    rows.  `batch_scoring` adds what the first `lsk_score_batch` or `lsk_score_prefixed` call
    allocates: the scoring buffers, eight ints per position (row ids, targets, row maps, attention
    pieces of a group), one int per position for the table of page-table views and one arrival
    counter per (piece, kv head) of a 128-row chunk (nothing without the prompt pass, which
    refuses the call)."""
    h, L = arch.hidden, arch.layers
    batch_scoring = batch_scoring and prefill_tc and h % 64 == 0
    scoring = scoring or batch_scoring
    q_l = arch.heads // tp_size * arch.head_dim
    kv_l = arch.kv_heads // tp_size * arch.head_dim
    inter_l = arch.inter // tp_size
    inter_l_pad = (inter_l + 31) // 32 * 32                 # K of the down projection
    vocab_l = arch.vocab // tp_size
    vocab_l_pad = (vocab_l + 15) // 16 * 16
    per_layer = 2 * ((q_l + 2 * kv_l) * h + h * q_l + 2 * inter_l * h + h * inter_l_pad) + 2 * 2 * h
    weights = L * per_layer
    if prefill_tc and h % 64 == 0:
        # second, canonical-layout copy of the layer weights for the tensor-core prompt pass
        # (128-row tiles x 64-wide k stages of 16 KiB) + its 128-token activation buffers
        up = lambda x, m: (x + m - 1) // m     # noqa: E731
        t_qkv, t_h, t_gu = up(q_l + 2 * kv_l, 128), up(h, 128), up(2 * inter_l, 128)
        k_h, k_q, k_i = h // 64, up(q_l, 64), up(inter_l, 64)
        weights += L * 16384 * (t_qkv * k_h + t_h * k_q + t_gu * k_h + t_h * k_i)
    embed = 2 * arch.vocab * h + 2 * h                       # replicated embedding + final norm
    lm_head = 2 * vocab_l_pad * h
    if lm_head_tc:
        lm_head += 2 * ((vocab_l + 127) // 128 * 128) * h     # canonical-layout copy for the wgmma head
    n_pages = (max_ctx + PAGE_TOKENS - 1) // PAGE_TOKENS
    max_pos = n_pages * PAGE_TOKENS
    kv_pool = 2 * L * n_pages * (arch.kv_heads // tp_size) * PAGE_TOKENS * arch.head_dim * 2
    scratch = (
        (MAX_ROWS + 1) * h * 4                 # residual rows
        + 2 * MAX_ROWS * q_l * 2               # q, attention out
        + MAX_ROWS * inter_l_pad * 2           # SiLU * up
        + MAX_ROWS * h * 4                     # TP partial sums
        + max_pos * (arch.head_dim // 2) * 8 + max_pos * 4 + n_pages * 4   # RoPE table, prompt ids, page table
        + SM_COUNT * MAX_ROWS * 8 + tp_size * MAX_ROWS * 8)      # arg-max candidates
    kvh_l = arch.kv_heads // tp_size                          # attention split partials + counters
    splits = max(1, min(4, SM_COUNT // kvh_l))
    scratch += kvh_l * splits * ((arch.heads // arch.kv_heads * 128 + 15) // 16 * 16) * (arch.head_dim + 2) * 4 + kvh_l * 4
    if prefill_tc and h % 64 == 0:
        scratch += 6 * 128 * h * 4 + 128 * q_l * 2 + 16384 * (h // 64 + (q_l + 63) // 64 + (inter_l + 63) // 64)
    if keep_logits or sampling or scoring or score_exits > 0:
        scratch += MAX_ROWS * vocab_l_pad * 4
    result_exits = max(score_exits, 1 if scoring else 0)
    scratch += 2 * result_exits * max_pos * 4               # per-exit log-probabilities + arg-max ids
    if score_exits > 0 and score_exits_sampled:
        draft_rows = 128 if (prefill_tc and h % 64 == 0) else MAX_ROWS
        scratch += (score_exits - 1) * (max_pos + draft_rows * arch.vocab) * 4 + MAX_ROWS * arch.vocab * 4
    if batch_scoring:
        scratch += 9 * max_pos * 4 + 128 * kvh_l * 4        # group arrays, view table, piece arrival counters
    if sampling:
        scratch += (2 * MAX_ROWS + 1) * arch.vocab * 4
        if tp_size > 1:
            scratch += tp_size * MAX_ROWS * vocab_l_pad * 4 + MAX_ROWS * arch.vocab * 4
    if tp_size > 1:
        scratch += 2 * tp_size * MAX_ROWS * h * 4           # peer region of the one-shot collectives
    source_peak = 2 * max(arch.vocab * h, arch.inter * h)   # one full bf16 tensor while repacking
    total = weights + embed + lm_head + kv_pool + scratch
    return {"weights": weights, "embed": embed, "lm_head": lm_head, "kv_pool": kv_pool,
            "scratch": scratch, "total": total, "weights_source_peak": source_peak}


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

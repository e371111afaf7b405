"""Python handle on one liblsk engine (one per process / GPU).

Host code here is plumbing only: it marshals arguments into the C ABI (include/lsk.h).  All
arithmetic, the draft/verify/accept logic and the KV bookkeeping run in the CUDA library.
"""
from __future__ import annotations

import os

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .weights import LlamaArch, SyntheticLlama, iter_state_dict


def batch_slot_positions(max_ctx: int, n_seqs: int) -> int:
    """Positions each sequence of an `n_seqs` batch owns in an engine built with `max_ctx`: the pool's
    ceil(max_ctx / 64) pages split into n_seqs slots of whole 64-token pages (engine.cu:
    batch_slot_positions)."""
    if n_seqs < 1:
        raise ValueError(f"n_seqs must be >= 1 (got {n_seqs})")
    return ((max_ctx + 63) // 64) // n_seqs * 64


@dataclass
class RoundOutput:
    """One speculation round as seen by the host (lsk_round_out)."""
    n_drafted: int
    n_matches: int
    emitted: List[int]
    draft: List[int]
    verified: List[int]
    kv_len: int
    draft_confidence: Optional[List[float]] = None   # round_adaptive: confidence of each kept draft


class Engine:
    def __init__(self, arch: LlamaArch, max_ctx: int = 4096, tp_rank: int = 0, tp_size: int = 1,
                 keep_logits: bool = False, use_pdl: bool = True, use_graph: bool = True,
                 attn_splits: int = 0, device: Optional[torch.device] = None,
                 tp_nccl: bool = False, prefill_tc: Optional[bool] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("layerskip_b200 needs a CUDA device (H100); there is no CPU path")
        self._lib = _lib.load()
        self.arch = arch
        self.device = torch.device(device) if device is not None else \
            torch.device("cuda", torch.cuda.current_device())
        self.tp_rank, self.tp_size = tp_rank, tp_size
        # the memory plan counts per-SM buffers: asked only when there is free memory to plan against
        sm_count = lambda: torch.cuda.get_device_properties(self.device).multi_processor_count  # noqa: E731
        # the tensor-core prompt pass needs a second (canonical-layout) copy of the layer weights: on by
        # default, dropped automatically when the two copies would not fit this GPU
        try:
            free_now = torch.cuda.mem_get_info(self.device)[0]
        except Exception:  # pragma: no cover
            free_now = None
        if prefill_tc is None:
            prefill_tc = os.environ.get("LSK_PREFILL_TC", "1") not in ("0",)
            if prefill_tc and free_now is not None:
                from .memory import plan_memory
                plan = plan_memory(arch, max_ctx=max_ctx, tp_size=tp_size, keep_logits=keep_logits,
                                   prefill_tc=True, sm_count=sm_count())
                if plan["total"] + plan["weights_source_peak"] > free_now:
                    prefill_tc = False
        self.prefill_tc = bool(prefill_tc)
        flags = (_lib.LSK_FLAG_KEEP_LOGITS if keep_logits else 0) | \
                (0 if prefill_tc else _lib.LSK_FLAG_NO_PREFILL_TC) | \
                (0 if use_pdl else _lib.LSK_FLAG_NO_PDL) | (0 if use_graph else _lib.LSK_FLAG_NO_GRAPH) | \
                (_lib.LSK_FLAG_TP_NCCL if tp_nccl else 0)
        cfg = arch.lsk_config(max_ctx, tp_rank=tp_rank, tp_size=tp_size, attn_splits=attn_splits, flags=flags)
        self.max_ctx = max_ctx
        self.keep_logits = keep_logits
        # refuse a configuration that cannot fit BEFORE cudaMalloc fails half-way (memory.py)
        try:
            free_bytes = torch.cuda.mem_get_info(self.device)[0]
        except Exception:  # pragma: no cover - very old drivers
            free_bytes = None
        if free_bytes is not None:
            from .memory import check_fits
            check_fits(arch, free_bytes, max_ctx=max_ctx, tp_size=tp_size, keep_logits=keep_logits,
                       sampling=False, lm_head_tc=os.environ.get("LSK_LMHEAD_TC", "0") not in ("", "0"),
                       prefill_tc=self.prefill_tc, sm_count=sm_count())
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_create(C.byref(cfg), C.byref(handle)))
        self._h = handle
        self._exit_layer = -1
        self._batch_n = 0                  # sequences of the last prefill_batch
        # token rows one step can carry (engine.cu: max_rows): 16 when the host planner finds a
        # schedule for the 16-row RMSNorm GEMM at K = hidden (whole rows resident up to hidden 4096,
        # K-chunked normalisation above), else 8
        plan = _lib.lsk_gemm_plan()
        qkv_rows = (arch.heads + 2 * arch.kv_heads) // tp_size * arch.head_dim
        ok = self._lib.lsk_plan_gemm((qkv_rows + 15) // 16 * 16, arch.hidden, 16, 0, 0, sm_count(), C.byref(plan))
        self.max_rows = 16 if (ok == 0 and plan.ok) else 8

    # ------------------------------------------------------------------ lifetime
    def close(self) -> None:
        if getattr(self, "_h", None):
            with torch.cuda.device(self.device):
                self._lib.lsk_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ tensor parallel
    def init_comm(self, process_group=None) -> None:
        """Create the engine's NCCL communicator; the unique id travels over torch.distributed
        (plumbing only — the data path uses the engine's own communicator and stream)."""
        if self.tp_size == 1:
            return
        import torch.distributed as dist
        from .parallel_util import broadcast_bytes
        uid = (C.c_uint8 * 128)()
        if dist.get_rank(process_group) == 0:
            _lib.check(self._lib.lsk_comm_unique_id(uid))
        raw = broadcast_bytes(bytes(uid), 128, src=0, group=process_group, device=self.device)
        arr = (C.c_uint8 * 128)(*raw)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_comm_init(self._h, arr))

    # ------------------------------------------------------------------ weights
    def load_weights(self, source: Iterable[Tuple[int, int, torch.Tensor]]) -> None:
        with torch.cuda.device(self.device):
            for role, layer, t in source:
                assert t.is_cuda and t.dtype == torch.bfloat16 and t.is_contiguous()
                # the tensor was produced on torch's stream; the engine packs on its own
                torch.cuda.current_stream(self.device).synchronize()
                rows = t.shape[0]
                cols = t.shape[1] if t.dim() == 2 else 1
                desc = _lib.lsk_weight_desc(role=role, layer=layer, data=t.data_ptr(), rows=rows,
                                            cols=cols)
                _lib.check(self._lib.lsk_load_weights(self._h, C.byref(desc), 1))

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        self.load_weights(iter_state_dict(sd, self.device))

    def load_model(self, model) -> None:
        """HF `LlamaForCausalLM` (any device / float dtype), or a streaming source with
        `iter_weights(device)` (`SyntheticLlama`, `checkpoint.CheckpointLlama`)."""
        if hasattr(model, "iter_weights"):
            self.load_weights(model.iter_weights(self.device))
        else:
            self.load_state_dict(model.state_dict())
        if not self._lib.lsk_weights_complete(self._h):
            raise RuntimeError("model did not provide every tensor the engine needs")

    # ------------------------------------------------------------------ generation
    def begin(self, exit_layer: int, max_steps: int, eos_token_ids: Sequence[int],
              sample: bool = False, temperature: float = 0.6, top_k: int = 0, top_p: float = 0.9,
              seed: int = 0, no_repeat_ngram_size: int = 0) -> None:
        eos = list(eos_token_ids)
        if len(eos) > _lib.LSK_MAX_EOS:
            raise ValueError(f"at most {_lib.LSK_MAX_EOS} eos ids are supported")
        gen = _lib.lsk_generation(exit_layer=exit_layer, max_steps=max_steps, n_eos=len(eos),
                                  sample=int(bool(sample)), temperature=temperature, top_k=top_k,
                                  top_p=top_p, seed=seed,
                                  no_repeat_ngram_size=int(no_repeat_ngram_size or 0))
        for i, t in enumerate(eos):
            gen.eos_ids[i] = int(t)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_begin(self._h, C.byref(gen)))
        self._exit_layer = exit_layer

    def prefill(self, prompt_ids: Sequence[int]) -> None:
        n = len(prompt_ids)
        arr = (C.c_int32 * n)(*[int(t) for t in prompt_ids])
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_prefill(self._h, arr, n))

    def round(self, d_req: int) -> RoundOutput:
        out = _lib.lsk_round_out()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_round(self._h, d_req, C.byref(out)))
        return RoundOutput(
            n_drafted=out.n_drafted, n_matches=out.n_matches,
            emitted=list(out.emitted_ids[:out.n_emitted]),
            draft=list(out.draft_ids[:out.n_drafted]),
            verified=list(out.verified_ids[:out.n_drafted + 1]), kv_len=out.kv_len)

    def round_adaptive(self, d_max: int, min_confidence: float) -> RoundOutput:
        """A round that drafts up to `d_max` tokens and stops after the first draft that is an EOS or
        whose probability under the distribution it was chosen from is below `min_confidence`
        (Hugging Face's `assistant_confidence_threshold`); the draft steps after it do not run.  The
        result is bit-identical to `round(n_drafted)` from the same state; `draft_confidence` holds
        the kept drafts' confidences."""
        out = _lib.lsk_round_out()
        conf = (C.c_float * (_lib.LSK_MAX_SPEC + 1))()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_round_adaptive(self._h, int(d_max), float(min_confidence), C.byref(out), conf))
        return RoundOutput(
            n_drafted=out.n_drafted, n_matches=out.n_matches,
            emitted=list(out.emitted_ids[:out.n_emitted]),
            draft=list(out.draft_ids[:out.n_drafted]),
            verified=list(out.verified_ids[:out.n_drafted + 1]), kv_len=out.kv_len,
            draft_confidence=[float(x) for x in conf[:out.n_drafted]])

    @staticmethod
    def _round_output(out) -> RoundOutput:
        return RoundOutput(
            n_drafted=out.n_drafted, n_matches=out.n_matches,
            emitted=list(out.emitted_ids[:out.n_emitted]),
            draft=list(out.draft_ids[:out.n_drafted]),
            verified=list(out.verified_ids[:out.n_drafted + 1]) if out.n_emitted else [],
            kv_len=out.kv_len)

    # ------------------------------------------------------------------ batched generation
    def prefill_batch(self, prompts: Sequence[Sequence[int]], seeds: Optional[Sequence[int]] = None) -> int:
        """Prefill every prompt into its own slot of the KV pool (after `begin`, no n-gram ban, one
        GPU).  Returns the positions each slot holds: `batch_slot_positions(max_ctx, len(prompts))`.
        Each prompt is prefilled exactly as `prefill` would prefill it alone.  A sampled generation
        needs `seeds`, one Philox seed in [0, 2**64) per prompt: sequence s then samples as a solo
        generation begun with `seed=seeds[s]`.  Greedy generation ignores the seeds."""
        prompts = [[int(t) for t in p] for p in prompts]
        if seeds is not None:
            seeds = [int(x) for x in seeds]
            if len(seeds) != len(prompts):
                raise ValueError(f"{len(seeds)} seeds for {len(prompts)} prompts")
            if any(not 0 <= x < 2 ** 64 for x in seeds):
                raise ValueError("seeds must be in [0, 2**64)")
        offsets = [0]
        for p in prompts:
            offsets.append(offsets[-1] + len(p))
        flat = [t for p in prompts for t in p]
        arr = (C.c_int32 * max(len(flat), 1))(*flat)
        off = (C.c_int32 * len(offsets))(*offsets)
        slot = C.c_int32()
        with torch.cuda.device(self.device):
            if seeds is None:
                _lib.check(self._lib.lsk_prefill_batch(self._h, arr, off, len(prompts), C.byref(slot)))
            else:
                sd = (C.c_uint64 * max(len(seeds), 1))(*seeds)
                _lib.check(self._lib.lsk_prefill_batch_seeded(self._h, arr, off, len(prompts), sd, C.byref(slot)))
        self._batch_n = len(prompts)
        return slot.value

    def round_batch(self, d_req: int, d_seq: Optional[Sequence[int]] = None,
                    active: Optional[Sequence[bool]] = None) -> List[RoundOutput]:
        """One round for every sequence of the batch (len(prompts) * (d_req + 1) <= max_rows): sequence s
        drafts d_seq[s] <= d_req tokens (default d_req) and, when active (default), commits exactly what
        `round(d_seq[s])` of that sequence alone would.  An inactive sequence commits nothing and gets
        an empty RoundOutput (no tokens, kv_len unchanged)."""
        n = self._batch_n
        ds, act = self._batch_ctl(d_seq, active)
        outs = (_lib.lsk_round_out * (_lib.LSK_MAX_SPEC + 1))()    # up to max_rows sequences
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_round_batch(self._h, int(d_req), ds, act, outs))
        return [self._round_output(o) for o in outs[:n]]

    def round_batch_adaptive(self, d_max: int, min_confidence: float, d_seq: Optional[Sequence[int]] = None,
                             active: Optional[Sequence[bool]] = None) -> List[RoundOutput]:
        """`round_batch(d_max, d_seq, active)` with `round_adaptive`'s stop rule for every sequence:
        sequence s stops drafting after its first draft that is an EOS or whose confidence is below
        `min_confidence`, or after d_seq[s] drafts, and a draft step runs only while some active
        sequence is still drafting.  Each active sequence's output is bit-identical to
        `round_adaptive(d_seq[s], min_confidence)` of that sequence alone, `draft_confidence` included;
        an inactive one gets an empty RoundOutput."""
        n = self._batch_n
        ds, act = self._batch_ctl(d_seq, active)
        outs = (_lib.lsk_round_out * (_lib.LSK_MAX_SPEC + 1))()
        conf = (C.c_float * ((_lib.LSK_MAX_SPEC + 1) * _lib.LSK_MAX_SPEC))()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_round_batch_adaptive(self._h, int(d_max), ds, act, float(min_confidence),
                                                          outs, conf))
        res = []
        for s, o in enumerate(outs[:n]):
            r = self._round_output(o)
            base = s * _lib.LSK_MAX_SPEC
            r.draft_confidence = [float(x) for x in conf[base:base + o.n_drafted]]
            res.append(r)
        return res

    def _batch_ctl(self, d_seq, active):
        """round_batch's d_seq and active flags as C arrays (None stays None: the library's default)."""
        n = self._batch_n
        for name, v in (("d_seq", d_seq), ("active", active)):
            if v is not None and len(v) != n:
                raise ValueError(f"{name} has {len(v)} entries for a batch of {n} sequences")
        ds = (C.c_int32 * n)(*[int(x) for x in d_seq]) if d_seq is not None else None
        act = (C.c_int32 * n)(*[int(bool(x)) for x in active]) if active is not None else None
        return ds, act

    KERNEL_CLASSES = ("qkv", "attention", "o_proj", "gate_up", "down", "lm_head", "small", "comm")

    def profile_round(self, d_req: int):
        """Eager round with per-kernel-class device times (ms) and launch counts."""
        out = _lib.lsk_round_out()
        ms = (C.c_float * 8)()
        cnt = (C.c_int64 * 8)()
        total = C.c_float()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_profile_round(self._h, d_req, C.byref(out), ms, cnt,
                                                   C.byref(total)))
        r = RoundOutput(n_drafted=out.n_drafted, n_matches=out.n_matches,
                        emitted=list(out.emitted_ids[:out.n_emitted]),
                        draft=list(out.draft_ids[:out.n_drafted]),
                        verified=list(out.verified_ids[:out.n_drafted + 1]), kv_len=out.kv_len)
        return r, dict(zip(self.KERNEL_CLASSES, [float(x) for x in ms])), \
            dict(zip(self.KERNEL_CLASSES, [int(x) for x in cnt])), float(total.value)

    def ar_step(self) -> int:
        tok = C.c_int32()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_ar_step(self._h, C.byref(tok)))
        return tok.value

    # ------------------------------------------------------------------ scoring
    def score(self, ids: Sequence[int], exit_layer: int = -1) -> Tuple[torch.Tensor, torch.Tensor]:
        """Teacher-forced pass over `ids` (2 <= len(ids) <= max_ctx) through layers < exit_layer
        (all layers when exit_layer <= 0), the final norm and the LM head.  Returns
        (logprobs float32[n-1], greedy int64[n-1]): entry i is the log-probability of ids[i+1] and
        the arg-max token after ids[0..i].  Ends any generation in progress (the next round needs
        a new prefill)."""
        n = len(ids)
        arr = (C.c_int32 * max(n, 1))(*[int(t) for t in ids])
        lp = (C.c_float * max(n - 1, 1))()
        gr = (C.c_int32 * max(n - 1, 1))()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_score(self._h, arr, n, int(exit_layer), lp, gr))
        logprobs = torch.frombuffer(lp, dtype=torch.float32).clone()[:n - 1]
        greedy = torch.frombuffer(gr, dtype=torch.int32).clone()[:n - 1].to(torch.int64)
        return logprobs, greedy

    def score_batch(self, seqs: Sequence[Sequence[int]],
                    exit_layer: int = -1) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """`score` of every sequence in `seqs`, in one call on the wgmma prompt pass: the rows of all
        sequences share 128-token chunks, so short sequences no longer pay a whole weight pass each.
        Returns one (logprobs float32[n-1], greedy int64[n-1]) per sequence, in order.  Each entry
        is bit-identical to `score` of that sequence alone when it has more than max_rows + 1 ids
        (shorter ones take the decode route in `score`).  Needs an engine with the prompt pass."""
        seqs = [[int(t) for t in s] for s in seqs]
        offsets = [0]
        for s in seqs:
            offsets.append(offsets[-1] + len(s))
        flat = [t for s in seqs for t in s]
        rows = offsets[-1] - len(seqs)
        arr = (C.c_int32 * max(len(flat), 1))(*flat)
        off = (C.c_int32 * len(offsets))(*offsets)
        lp = (C.c_float * max(rows, 1))()
        gr = (C.c_int32 * max(rows, 1))()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_score_batch(self._h, arr, off, len(seqs), int(exit_layer), lp, gr))
        logprobs = torch.frombuffer(lp, dtype=torch.float32).clone()
        greedy = torch.frombuffer(gr, dtype=torch.int32).clone().to(torch.int64)
        out = []
        for j, s in enumerate(seqs):
            r0 = offsets[j] - j
            out.append((logprobs[r0:r0 + len(s) - 1], greedy[r0:r0 + len(s) - 1]))
        return out

    def score_prefixed(self, prefixes: Sequence[Sequence[int]], branches: Sequence[Tuple[int, Sequence[int]]],
                       exit_layer: int = -1) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """Score continuations that share contexts: `branches` holds (prefix index, ids B) pairs, each
        scoring prefixes[index] + B.  Each prefix's own rows run once (per KV group) and only write
        keys and values; the branches' rows are packed into shared 128-token chunks on top of them.
        Returns one (logprobs float32[len(B)], greedy int64[len(B)]) per branch, in order: entry i is
        the log-probability of B[i] after P + B[:i] and the arg-max token there, bit-identical to
        entries len(P)-1 .. of `score_batch([P + B])`.  Every prefix and branch needs at least one
        id, every prefix at least one branch.  Needs an engine with the prompt pass."""
        prefixes = [[int(t) for t in p] for p in prefixes]
        branches = [(int(p), [int(t) for t in b]) for p, b in branches]
        p_off, b_off = [0], [0]
        for p in prefixes:
            p_off.append(p_off[-1] + len(p))
        for _, b in branches:
            b_off.append(b_off[-1] + len(b))
        p_ids = [t for p in prefixes for t in p]
        b_ids = [t for _, b in branches for t in b]
        i32 = lambda v: (C.c_int32 * max(len(v), 1))(*v)   # noqa: E731
        rows = max(b_off[-1], 1)
        lp = (C.c_float * rows)()
        gr = (C.c_int32 * rows)()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_score_prefixed(self._h, i32(p_ids), i32(p_off), len(prefixes), i32(b_ids),
                                                    i32(b_off), i32([p for p, _ in branches]), len(branches),
                                                    int(exit_layer), lp, gr))
        logprobs = torch.frombuffer(lp, dtype=torch.float32).clone()
        greedy = torch.frombuffer(gr, dtype=torch.int32).clone().to(torch.int64)
        return [(logprobs[b_off[j]:b_off[j + 1]], greedy[b_off[j]:b_off[j + 1]]) for j in range(len(branches))]

    def score_exits(self, ids: Sequence[int], exits: Sequence[int], sampling: Optional[Dict] = None
                    ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """`score(ids, E)` at every exit E of `exits` (strictly increasing, in [1, layers]) in one
        pass: layers below each exit run once.  Returns (logprobs float32[k, n-1], greedy
        int64[k, n-1], accept): row j is bit-identical to `score(ids, exits[j])`.

        With `sampling` (a dict with `temperature`, `top_k`, `top_p`), `exits[-1]` must be the full
        depth, and accept float32[k-1, n-1] holds, for the row predicting ids[i+1], the probability
        sum_v min(p_E(v), p_full(v)) that sampled self-speculation accepts a draft drawn at exit
        exits[j]: p are the warped distributions generation draws from.  accept is None without
        `sampling`.  Ends any generation in progress, like `score`."""
        n, k = len(ids), len(exits)
        arr = (C.c_int32 * max(n, 1))(*[int(t) for t in ids])
        ex = (C.c_int32 * max(k, 1))(*[int(e) for e in exits])
        rows = max(n - 1, 1)
        lp = (C.c_float * (max(k, 1) * rows))()
        gr = (C.c_int32 * (max(k, 1) * rows))()
        gen, acc = None, None
        if sampling is not None:
            gen = _lib.lsk_generation(sample=1, temperature=float(sampling.get("temperature", 1.0)),
                                      top_k=int(sampling.get("top_k", 0) or 0),
                                      top_p=float(sampling.get("top_p", 1.0)))
            acc = (C.c_float * (max(k - 1, 1) * rows))()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_score_exits(self._h, arr, n, ex, k, C.byref(gen) if gen is not None else None,
                                                 lp, gr, acc))
        logprobs = torch.frombuffer(lp, dtype=torch.float32).clone()[:k * (n - 1)].view(k, n - 1)
        greedy = torch.frombuffer(gr, dtype=torch.int32).clone()[:k * (n - 1)].view(k, n - 1).to(torch.int64)
        accept = None
        if acc is not None:
            accept = torch.frombuffer(acc, dtype=torch.float32).clone()[:(k - 1) * (n - 1)].view(k - 1, n - 1)
        return logprobs, greedy, accept

    def _loglikelihood_ids(self, context: Sequence[int], continuation: Sequence[int]) -> List[int]:
        """The ids `loglikelihood` scores: validated, joined and truncated from the left."""
        if not context or not continuation:
            raise ValueError("context and continuation must both be non-empty")
        if len(continuation) >= self.max_ctx:
            raise ValueError(f"a continuation of {len(continuation)} tokens does not fit max_ctx "
                             f"{self.max_ctx} with at least one context token")
        return (list(context) + list(continuation))[-self.max_ctx:]

    @staticmethod
    def _continuation_score(logprobs: torch.Tensor, greedy: torch.Tensor,
                            continuation: List[int]) -> Tuple[float, bool]:
        k = len(continuation)
        return float(logprobs[-k:].to(torch.float64).sum()), bool(greedy[-k:].tolist() == continuation)

    def loglikelihood(self, context: Sequence[int], continuation: Sequence[int],
                      exit_layer: int = -1) -> Tuple[float, bool]:
        """Log-likelihood of `continuation` following `context`, and whether greedy decoding from
        the context would have produced exactly the continuation.

        The two parts are joined and, when longer than max_ctx, the oldest tokens are dropped so
        the last max_ctx remain.  One teacher-forced pass scores every position; the continuation's
        tokens are the last len(continuation) targets, and their log-probabilities are summed in
        float64.  Both parts must be non-empty, and at least one token must precede the
        continuation after truncation (len(continuation) < max_ctx)."""
        context, continuation = [int(t) for t in context], [int(t) for t in continuation]
        logprobs, greedy = self.score(self._loglikelihood_ids(context, continuation), exit_layer)
        return self._continuation_score(logprobs, greedy, continuation)

    @staticmethod
    def _prefix_plan(seqs: List[List[int]], conts: List[List[int]]):
        """Requests grouped by their (cut) context: a context that two or more requests share becomes
        one prefix with their continuations as branches; every other request becomes a branch of a
        prefix of its own first id.  Returns (prefixes, branches, use), `use` telling whether
        `score_prefixed` needs fewer 128-row chunks than `score_batch` of the joined sequences."""
        ctxs = [tuple(s[:len(s) - len(k)]) for s, k in zip(seqs, conts)]
        count: Dict[tuple, int] = {}
        for c in ctxs:
            count[c] = count.get(c, 0) + 1
        prefixes: List[List[int]] = []
        branches: List[Tuple[int, List[int]]] = []
        index: Dict[tuple, int] = {}
        for s, k, c in zip(seqs, conts, ctxs):
            if count[c] >= 2:
                if c not in index:
                    index[c] = len(prefixes)
                    prefixes.append(list(c))
                branches.append((index[c], k))
            else:
                prefixes.append(s[:1])
                branches.append((len(prefixes) - 1, s[1:]))
        chunks = lambda rows: (rows + 127) // 128    # noqa: E731
        prefix_rows = sum(len(p) - 1 for p in prefixes)
        branch_rows = sum(len(b) for _, b in branches)
        batch_rows = sum(len(s) - 1 for s in seqs)
        return prefixes, branches, chunks(prefix_rows) + chunks(branch_rows) < chunks(batch_rows)

    def loglikelihood_batch(self, requests: Sequence[Tuple[Sequence[int], Sequence[int]]],
                            exit_layer: int = -1) -> List[Tuple[float, bool]]:
        """`loglikelihood` of every (context, continuation) request, in order, with one
        `score_batch` call for all of them (every request is validated before any is scored).  On an
        engine without the wgmma prompt pass it calls `loglikelihood` once per request.

        Requests that share a context (after the left cut), such as the choices of a multiple-choice
        question, are scored with one `score_prefixed` call instead when that packs into fewer
        128-row chunks: the shared context then runs once rather than once per request.  Both calls
        give the same bits, so the choice changes only the time taken.

        Caveat: a request whose joined ids number at most max_rows + 1 is scored here on the wgmma
        route, while `loglikelihood` scores it on the decode route.  The two then agree within the
        oracle bounds, not bit for bit; longer requests agree bit for bit."""
        reqs = [([int(t) for t in ctx], [int(t) for t in cont]) for ctx, cont in requests]
        seqs = [self._loglikelihood_ids(ctx, cont) for ctx, cont in reqs]
        if not reqs:
            return []
        if not (self.prefill_tc and self.arch.hidden % 64 == 0):
            return [self.loglikelihood(ctx, cont, exit_layer) for ctx, cont in reqs]
        prefixes, branches, use_prefixed = self._prefix_plan(seqs, [cont for _, cont in reqs])
        if use_prefixed:
            scored = self.score_prefixed(prefixes, branches, exit_layer)
        else:
            scored = self.score_batch(seqs, exit_layer)
        return [self._continuation_score(lp, gr, cont) for (lp, gr), (_, cont) in zip(scored, reqs)]

    # ------------------------------------------------------------------ introspection
    @property
    def kv_len(self) -> int:
        v = C.c_int32()
        _lib.check(self._lib.lsk_kv_len(self._h, C.byref(v)))
        return v.value

    @property
    def launch_count(self) -> int:
        v = C.c_int64()
        _lib.check(self._lib.lsk_launch_count(self._h, C.byref(v)))
        return v.value

    @property
    def last_device_ms(self) -> float:
        v = C.c_float()
        _lib.check(self._lib.lsk_last_device_ms(self._h, C.byref(v)))
        return v.value

    def round_bytes(self, d: int, ctx: int) -> float:
        v = C.c_double()
        _lib.check(self._lib.lsk_round_bytes(self._h, d, ctx, C.byref(v)))
        return v.value

    def ar_bytes(self, ctx: int) -> float:
        v = C.c_double()
        _lib.check(self._lib.lsk_ar_bytes(self._h, ctx, C.byref(v)))
        return v.value

    def debug_forward_rows(self, ids: Sequence[int]) -> torch.Tensor:
        """Teacher-forced block (parity tests): logits [len(ids), vocab_local] of the given ids
        run as ONE block on top of the committed context; nothing is committed."""
        m = len(ids)
        arr = (C.c_int32 * m)(*[int(t) for t in ids])
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_forward_rows(self._h, arr, m))
        return self.debug_logits(m)

    def debug_argmax(self, rows: int):
        """The engine's greedy choice for each of the first `rows` rows of the last LM head (the
        LM-head epilogue's candidates merged as the accept kernels merge them): (logits, token ids)."""
        buf = (C.c_float * (2 * rows))()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_read(self._h, _lib.LSK_DBG_ARGMAX, 0, 0, buf, 2 * rows))
        t = torch.frombuffer(buf, dtype=torch.float32).clone().view(rows, 2)
        return t[:, 0], t[:, 1].to(torch.int64)

    def debug_hidden(self, rows: int = 16) -> torch.Tensor:
        n = rows * self.arch.hidden
        buf = (C.c_float * n)()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_read(self._h, _lib.LSK_DBG_HIDDEN, 0, 0, buf, n))
        return torch.tensor(list(buf), dtype=torch.float32).view(rows, self.arch.hidden)

    def debug_logits(self, rows: int = 16) -> torch.Tensor:
        vloc = self.arch.vocab // self.tp_size
        vpad = (vloc + 15) // 16 * 16
        n = rows * vpad
        buf = (C.c_float * n)()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_read(self._h, _lib.LSK_DBG_LOGITS, 0, 0, buf, n))
        return torch.frombuffer(buf, dtype=torch.float32).clone().view(rows, vpad)[:, :vloc]

    def debug_probs(self, which: str, rows: int = 16) -> torch.Tensor:
        """Warped sampling distributions of the last round: 'draft' or 'verify' -> [rows, vocab]."""
        n = rows * self.arch.vocab
        buf = (C.c_float * n)()
        what = _lib.LSK_DBG_PROBS_DRAFT if which == "draft" else _lib.LSK_DBG_PROBS_VERIFY
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_read(self._h, what, 0, 0, buf, n))
        return torch.frombuffer(buf, dtype=torch.float32).clone().view(rows, self.arch.vocab)

    def debug_residual(self) -> torch.Tensor:
        """max(p_verify - p_draft, 0) of the last rejected draft position (unnormalised) [vocab]."""
        n = self.arch.vocab
        buf = (C.c_float * n)()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_read(self._h, _lib.LSK_DBG_RESIDUAL, 0, 0, buf, n))
        return torch.frombuffer(buf, dtype=torch.float32).clone()

    def debug_kv_row(self, which: str, layer: int, kv_head: int, pos: int) -> torch.Tensor:
        return self.debug_kv_rows(which, layer, kv_head, pos, 1)[0]

    def debug_kv_rows(self, which: str, layer: int, kv_head: int, pos0: int, count: int) -> torch.Tensor:
        """K ('k') or V ('v') cache rows of one kv head at positions pos0 .. pos0+count-1 as fp32
        [count, head_dim] (bf16 values), in one call."""
        hd = self.arch.head_dim
        buf = (C.c_float * (count * hd))()
        what = _lib.LSK_DBG_KROW if which == "k" else _lib.LSK_DBG_VROW
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_read(self._h, what, layer, kv_head * self.max_ctx + pos0,
                                                buf, count * hd))
        return torch.frombuffer(buf, dtype=torch.float32).clone().view(count, hd)

    def debug_set_page_table(self, pages: Sequence[int]) -> None:
        arr = (C.c_int32 * len(pages))(*[int(p) for p in pages])
        with torch.cuda.device(self.device):
            _lib.check(self._lib.lsk_debug_set_page_table(self._h, arr, len(pages)))

"""Drop-in generation strategies backed by the CUDA engine.

`B200SelfSpeculativeGenerationStrategy` replaces the reference's
`SelfSpeculativeGenerationStrategy` (self_speculation/self_speculation_generator.py:31-229) and
`B200AutoRegressiveGenerationStrategy` its `AutoRegressiveGenerationStrategy`
(self_speculation/autoregressive_generator.py:25-80) behind the same
`generate_token_ids(model, input_ids, eos_token_ids, generation_config, logits_processors,
stopping_criteria, streamer)` call.  The Python below is the reference's OUTER loop only
(max_steps clamp, acceptance accounting, EOS truncation, streamer hand-off); each round — draft
steps, verify, accept test, KV rewind — is one `lsk_round` on the device.
"""
from __future__ import annotations

import weakref
from typing import Any, Dict, List, Optional, Tuple

import torch

from .engine import Engine, batch_slot_positions
from .plugin import GenerationConfig, GenerationStrategy, GenerationStrategyResult
from .weights import LlamaArch, SyntheticLlama


class _EngineCache:
    """One engine per model object (weights are repacked once, then stay resident in HBM)."""

    def __init__(self, **engine_kwargs):
        self.kwargs = engine_kwargs
        self.process_group = engine_kwargs.get("process_group")
        self._by_id: Dict[int, Tuple[Any, Engine]] = {}

    def get(self, model) -> Engine:
        key = id(model)
        hit = self._by_id.get(key)
        if hit is not None and hit[0]() is model:
            return hit[1]
        arch = model.arch if isinstance(getattr(model, "arch", None), LlamaArch) \
            else LlamaArch.from_hf_config(model.config)
        kw = dict(self.kwargs)
        group = kw.pop("process_group", None)
        eng = Engine(arch, **kw)
        eng.init_comm(group)
        eng.load_model(model)
        try:
            ref = weakref.ref(model, lambda _r, k=key: self._evict(k))
        except TypeError:
            ref = (lambda m: (lambda: m))(model)
        self._by_id[key] = (ref, eng)
        return eng

    def _evict(self, key) -> None:
        hit = self._by_id.pop(key, None)
        if hit is not None:
            hit[1].close()

    def close(self) -> None:
        for _ref, eng in self._by_id.values():
            eng.close()
        self._by_id.clear()


def _generation_seed(cache: "_EngineCache", eng: Engine, sample: bool) -> int:
    """The reference draws from torch's global generator, so two sampled calls differ while a run
    under `torch.manual_seed` stays reproducible.  The engine's Philox streams are keyed by a
    per-generation seed: draw it FROM the global generator (which advances it, like the
    reference's own draws would).  Under tensor parallelism every rank must draw the SAME
    tokens, so rank 0's seed is broadcast (only when sampling: greedy needs no collective)."""
    if not sample:
        return 0
    seed = int(torch.randint(0, 2 ** 31 - 1, ()).item())
    if eng.tp_size > 1:
        from .parallel_util import broadcast_bytes
        raw = broadcast_bytes(seed.to_bytes(4, "little"), 4, src=0,
                              group=cache.process_group, device=eng.device)
        seed = int.from_bytes(raw, "little")
    return seed


def _check_num_speculations(cfg: GenerationConfig, eng) -> None:
    """The reference accepts any positive `num_speculations`; a verify block carries at most
    `eng.max_rows` token rows here (16; 8 when hidden > 4096).  Fail before prefill, clearly."""
    limit = getattr(eng, "max_rows", 16) - 1
    if cfg.num_speculations < 0 or cfg.num_speculations > limit:
        raise ValueError(f"num_speculations={cfg.num_speculations} is outside [0, {limit}] for this model "
                         "(the verify block holds num_speculations + 1 token rows)")


def _check_context(eng, n_prompt: int, cfg: GenerationConfig) -> None:
    """The KV pool is sized once (`max_ctx`): fail before the first kernel rather than mid-way.
    The last round / step touches position n_prompt + max_steps (engine.cu: lsk_round, lsk_ar_step)."""
    max_ctx = getattr(eng, "max_ctx", None)
    need = n_prompt + cfg.max_steps + 1
    if max_ctx is not None and need > max_ctx:
        raise ValueError(f"prompt ({n_prompt}) + max_steps ({cfg.max_steps}) needs {need} KV positions but "
                         f"the engine was built with max_ctx={max_ctx}; construct the strategy with a "
                         "larger max_ctx")


def _ngram_size_of(logits_processors) -> int:
    """The reference builds at most ONE logits processor: HF's `NoRepeatNGramLogitsProcessor`
    (`generator_base.py:77-85`, from `--no_repeat_ngram_size`).  The engine applies it on the device
    (csrc/misc_kernels.cuh: ngram_ban_kernel) over the whole sequence so far — prompt, output and the
    round's drafts — which is HF's documented semantics.  (The reference itself hands the processor
    only the current step's `input_ids`, a single token after the first step, so its ban list is
    empty from then on: INTEGRATION.md.)  Any other processor would need the logits on the host:
    refused, there is no CPU fallback."""
    size = 0
    for proc in (logits_processors or []):
        n = getattr(proc, "ngram_size", None)
        if type(proc).__name__ != "NoRepeatNGramLogitsProcessor" or not isinstance(n, int) or n <= 0:
            raise NotImplementedError(
                f"logits processor {type(proc).__name__} is not supported: only NoRepeatNGramLogitsProcessor "
                "runs on the device; the B200 engine keeps the logits on chip and has no CPU fallback")
        if n > 16:
            raise NotImplementedError("no_repeat_ngram_size > 16 is not supported")
        size = n if size == 0 else min(size, n)
    return size


class B200SelfSpeculativeGenerationStrategy(GenerationStrategy):
    def __init__(self, max_ctx: int = 4096, tp_rank: int = 0, tp_size: int = 1,
                 process_group=None, **engine_kwargs):
        self.engines = _EngineCache(max_ctx=max_ctx, tp_rank=tp_rank, tp_size=tp_size,
                                    process_group=process_group, **engine_kwargs)
        self.last_rounds: List[Any] = []      # per-round trace of the last generation

    def engine_for(self, model) -> Engine:
        return self.engines.get(model)

    def generate_token_ids(self, model, input_ids: List[int], eos_token_ids: List[int],
                           generation_config: GenerationConfig, logits_processors=None,
                           stopping_criteria=None, streamer=None) -> GenerationStrategyResult:
        ngram = _ngram_size_of(logits_processors)
        cfg = generation_config
        eng = self.engines.get(model)
        _check_context(eng, len(input_ids), cfg)
        _check_num_speculations(cfg, eng)
        eng.begin(exit_layer=cfg.exit_layer, max_steps=cfg.max_steps, eos_token_ids=eos_token_ids,
                  sample=cfg.sample, temperature=cfg.temperature, top_k=cfg.top_k, top_p=cfg.top_p,
                  seed=_generation_seed(self.engines, eng, cfg.sample), no_repeat_ngram_size=ngram)
        eng.prefill(input_ids)
        output_ids: List[int] = []
        matches = drafted = 0
        self.last_rounds = []
        speculative_streamer = streamer is not None and hasattr(streamer, "delete")
        # the reference's own GenerationConfig has no such field
        threshold = float(getattr(cfg, "draft_confidence_threshold", 0.0) or 0.0)
        while len(output_ids) < cfg.max_steps:                       # :51
            d_req = min(cfg.num_speculations, cfg.max_steps - len(output_ids) - 1)   # :63-66
            r = eng.round_adaptive(d_req, threshold) if threshold > 0 else eng.round(d_req)
            self.last_rounds.append(r)
            output_ids.extend(r.emitted)                             # :204-205
            matches += r.n_matches                                   # :80
            drafted += r.n_drafted                                   # :81
            if streamer is not None:                                 # :158-161, 207-216
                if speculative_streamer:
                    streamer.put(torch.tensor([r.draft], dtype=torch.long), is_draft=True)
                    streamer.delete(len(r.draft))
                    streamer.put(torch.tensor(r.emitted[:-1], dtype=torch.long))
                    streamer.put(torch.tensor(r.emitted[-1:], dtype=torch.long))
                else:
                    streamer.put(torch.tensor(r.emitted, dtype=torch.long))
            hit = False
            for eos in eos_token_ids:                                # :82-91
                if eos in output_ids:
                    output_ids = output_ids[: output_ids.index(eos)]
                    hit = True
                    break
            if hit:
                break
            if stopping_criteria:                                    # :92-95
                nxt = torch.tensor([[r.emitted[-1]]], dtype=torch.long)
                if torch.all(torch.as_tensor(stopping_criteria(nxt, scores=None))):
                    break
        return GenerationStrategyResult(predicted_tokens=output_ids,
                                        acceptance_rate=matches / drafted)   # :96-99

    def generate_batch(self, model, prompts: List[List[int]], eos_token_ids: List[int],
                       generation_config: GenerationConfig, logits_processors=None, stopping_criteria=None,
                       streamer=None, seeds: Optional[List[int]] = None) -> List[GenerationStrategyResult]:
        """Self-speculative generation of several prompts at once: every round runs all the
        sequences still generating through the same weight passes (`Engine.round_batch`).  Result j
        equals `generate_token_ids(model, prompts[j], ...)` with the same config: the outer loop
        below is the reference's, per sequence (max_steps clamp, acceptance accounting, EOS
        truncation), and each sequence's rounds are bit-identical to its rounds alone.  Sampling
        (`cfg.sample`) needs `seeds`, one per prompt in [0, 2**64): prompt j then samples as
        `generate_token_ids` does with the engine seed `seeds[j]`, whatever it is batched with.
        Logits processors, stopping criteria and streamers are not supported here.  The prompts share
        the KV pool: each gets ceil(max_ctx / 64) // len(prompts) whole 64-token pages."""
        cfg = generation_config
        if cfg.sample and seeds is None:
            raise NotImplementedError("generate_batch without seeds is greedy only: set sample=False, or pass "
                                      "one seed per prompt to sample")
        if cfg.sample and (len(seeds) != len(prompts) or any(not 0 <= int(x) < 2 ** 64 for x in seeds)):
            raise ValueError(f"sampling needs one seed in [0, 2**64) per prompt ({len(seeds)} seeds for "
                             f"{len(prompts)} prompts)")
        if logits_processors or cfg.no_repeat_ngram_size:
            raise NotImplementedError("generate_batch supports no logits processors (no n-gram ban)")
        if stopping_criteria or cfg.stop_words:
            raise NotImplementedError("generate_batch supports no stopping criteria (stop_words); use eos ids")
        if streamer is not None:
            raise NotImplementedError("generate_batch does not stream")
        if getattr(cfg, "draft_confidence_threshold", 0.0):
            raise NotImplementedError("generate_batch does not support draft_confidence_threshold")
        prompts = [[int(t) for t in p] for p in prompts]
        if not prompts:
            return []
        if any(len(p) == 0 for p in prompts):
            raise ValueError("every prompt needs at least one token")
        eng = self.engines.get(model)
        _check_num_speculations(cfg, eng)
        n, D = len(prompts), cfg.num_speculations
        if n * (D + 1) > eng.max_rows:
            raise ValueError(f"{n} prompts x (num_speculations {D} + 1) rows exceed the {eng.max_rows} token rows "
                             "of a step; generate fewer prompts at once or draft fewer tokens")
        slot = batch_slot_positions(eng.max_ctx, n)
        need = max(len(p) for p in prompts) + cfg.max_steps + D + 1
        if need > slot:
            raise ValueError(f"the longest prompt + max_steps ({cfg.max_steps}) + num_speculations ({D}) + 1 needs "
                             f"{need} KV positions but each of {n} prompts gets {slot} (max_ctx={eng.max_ctx}); "
                             "construct the strategy with a larger max_ctx or generate fewer prompts at once")
        eng.begin(exit_layer=cfg.exit_layer, max_steps=cfg.max_steps, eos_token_ids=eos_token_ids,
                  sample=cfg.sample, temperature=cfg.temperature, top_k=cfg.top_k, top_p=cfg.top_p)
        eng.prefill_batch(prompts, seeds if cfg.sample else None)
        outs: List[List[int]] = [[] for _ in prompts]
        matches, drafted = [0] * n, [0] * n
        active = [cfg.max_steps > 0] * n
        while any(active):
            d_seq = [min(D, cfg.max_steps - len(o) - 1) if a else 0 for o, a in zip(outs, active)]
            d_req = max(d for d, a in zip(d_seq, active) if a)
            rounds = eng.round_batch(d_req, d_seq, active)
            for s, r in enumerate(rounds):
                if not active[s]:
                    continue
                outs[s].extend(r.emitted)
                matches[s] += r.n_matches
                drafted[s] += r.n_drafted
                for eos in eos_token_ids:
                    if eos in outs[s]:
                        outs[s] = outs[s][: outs[s].index(eos)]
                        active[s] = False
                        break
                if len(outs[s]) >= cfg.max_steps:
                    active[s] = False
        return [GenerationStrategyResult(predicted_tokens=o, acceptance_rate=m / d if d else None)
                for o, m, d in zip(outs, matches, drafted)]


class B200AutoRegressiveGenerationStrategy(GenerationStrategy):
    """Greedy / sampled autoregressive decoding on the same engine (all layers, or layers < E
    when `exit_layer > 0`: the reference's early-exit mode, autoregressive_generator.py:44-51)."""

    def __init__(self, max_ctx: int = 4096, tp_rank: int = 0, tp_size: int = 1,
                 process_group=None, engine_cache: Optional[_EngineCache] = None, **engine_kwargs):
        self.engines = engine_cache or _EngineCache(max_ctx=max_ctx, tp_rank=tp_rank,
                                                    tp_size=tp_size, process_group=process_group,
                                                    **engine_kwargs)

    def generate_token_ids(self, model, input_ids: List[int], eos_token_ids: List[int],
                           generation_config: GenerationConfig, logits_processors=None,
                           stopping_criteria=None, streamer=None) -> GenerationStrategyResult:
        ngram = _ngram_size_of(logits_processors)
        cfg = generation_config
        eng = self.engines.get(model)
        _check_context(eng, len(input_ids), cfg)
        eng.begin(exit_layer=cfg.exit_layer, max_steps=cfg.max_steps, eos_token_ids=eos_token_ids,
                  sample=cfg.sample, temperature=cfg.temperature, top_k=cfg.top_k, top_p=cfg.top_p,
                  seed=_generation_seed(self.engines, eng, cfg.sample), no_repeat_ngram_size=ngram)
        eng.prefill(input_ids)
        output_ids: List[int] = []
        prev = input_ids[-1]
        for _ in range(cfg.max_steps):                               # :34
            tok = eng.ar_step()
            if streamer is not None:
                streamer.put(torch.tensor([tok], dtype=torch.long))
            if tok in eos_token_ids:                                 # :66-67
                break
            if stopping_criteria:                                    # :68-71 (current input)
                cur = torch.tensor([[prev]], dtype=torch.long)
                if torch.all(torch.as_tensor(stopping_criteria(cur, scores=None))):
                    break
            output_ids.append(tok)
            prev = tok
        return GenerationStrategyResult(predicted_tokens=output_ids, acceptance_rate=None)

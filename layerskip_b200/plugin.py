"""The reference's generation plug-in surface, kept field-for-field so callers can switch.

Mirrors `self_speculation/generator_base.py` of facebookresearch/LayerSkip:
  * `GenerationStrategyResult`  (generator_base.py:17-20)
  * `GenerationResult`          (generator_base.py:23-30)
  * `GenerationConfig`          (generator_base.py:33-49) — same fields, same defaults
  * `GenerationStrategy`        (generator_base.py:51-62) — `generate_token_ids(...)` contract
  * `HuggingfaceLlamaGenerator` (generator_base.py:65-130) — tokenise / time / decode façade

Only the façade's internals are new: timing uses `time.perf_counter`, and the logits-processor /
stopping-criteria factories import transformers lazily so the package also works with the
synthetic integer tokenizer (no network, no HF tokenizer files).
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Any, List, Optional


@dataclass
class GenerationStrategyResult:
    predicted_tokens: List[int]
    acceptance_rate: Optional[float] = None


@dataclass
class GenerationResult:
    generation_strategy_result: GenerationStrategyResult
    decoded_prediction: str
    num_tokens_generated: int
    total_time: float
    time_per_token: Optional[float]
    tokens_per_second: float


@dataclass
class GenerationConfig:
    max_steps: int = 512
    exit_layer: int = -1
    num_speculations: int = -1
    generation_strategy: str = "autoregressive"
    sample: bool = True
    temperature: float = 0.6
    top_k: int = 0
    top_p: float = 0.9
    no_repeat_ngram_size: Optional[int] = None
    stop_words: Optional[List[str]] = None
    stop_token_ids: Optional[List[int]] = field(default=None)
    # self-speculation only (not in the reference): stop a round's drafting after the first draft
    # whose probability under the early-exit head is below this; 0 drafts num_speculations tokens
    draft_confidence_threshold: float = 0.0

    def __post_init__(self):
        if self.stop_token_ids is None:
            self.stop_token_ids = []


class GenerationStrategy:
    """A strategy turns prompt ids into generated ids (generator_base.py:51-62)."""

    def generate_token_ids(self, model: Any, input_ids: List[int], eos_token_ids: List[int],
                           generation_config: GenerationConfig, logits_processors: Any = None,
                           stopping_criteria: Any = None, streamer: Any = None
                           ) -> GenerationStrategyResult:
        raise NotImplementedError()


class HuggingfaceLlamaGenerator:
    """tokenizer + model + strategy -> text (generator_base.py:65-130).

    `generate()` measures exactly what the reference measures (generator_base.py:107-129): the
    wall time of `generate_token_ids` only — prompt ingestion included, tokenising / decoding
    excluded — and derives tokens/s from the number of returned ids.
    """

    def __init__(self, tokenizer: Any, model: Any, generation_strategy: GenerationStrategy):
        self.tokenizer = tokenizer
        self.model = model
        self.generation_strategy = generation_strategy

    def create_logits_processors(self, generation_config: GenerationConfig):
        if not generation_config.no_repeat_ngram_size:        # generator_base.py:77-85
            return []
        from transformers.generation.logits_process import (LogitsProcessorList,
                                                            NoRepeatNGramLogitsProcessor)
        return LogitsProcessorList(
            [NoRepeatNGramLogitsProcessor(generation_config.no_repeat_ngram_size)])

    def create_stopping_criteria(self, generation_config: GenerationConfig):
        if not generation_config.stop_words:                  # generator_base.py:87-95
            return []
        import transformers
        return transformers.StoppingCriteriaList(
            [transformers.StopStringCriteria(self.tokenizer, generation_config.stop_words)])

    def generate(self, prompt: str, generation_config: GenerationConfig,
                 streamer: Any = None) -> GenerationResult:
        encoded = self.tokenizer(prompt, return_tensors="pt", add_special_tokens=True)
        prompt_ids = encoded["input_ids"].tolist()[0]
        processors = self.create_logits_processors(generation_config)
        criteria = self.create_stopping_criteria(generation_config)
        eos_ids = list(generation_config.stop_token_ids) + [self.tokenizer.eos_token_id]
        t0 = time.perf_counter()
        result = self.generation_strategy.generate_token_ids(
            model=self.model, input_ids=prompt_ids, eos_token_ids=eos_ids,
            generation_config=generation_config, logits_processors=processors,
            stopping_criteria=criteria, streamer=streamer)
        elapsed = time.perf_counter() - t0
        n = len(result.predicted_tokens)
        return GenerationResult(
            generation_strategy_result=result,
            decoded_prediction=self.tokenizer.decode(result.predicted_tokens),
            num_tokens_generated=n, total_time=elapsed,
            time_per_token=(elapsed / n) if n > 0 else None,
            tokens_per_second=n / elapsed)

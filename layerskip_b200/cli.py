"""Command lines with the reference's flag surface (arguments.py:19-24, generator_base.py:33-49,
benchmark.py:43-50, sweep.py:27-34, generate.py:32-39), parsed like the reference does: one
`HfArgumentParser` over dataclasses.  What differs is only where models and prompts come from —
this image has no network — so `--model` is either a local HF checkpoint directory or
`synthetic:<arch>` (random-init Llama of a named architecture, see weights.ARCHS) and the
dataset is `synthetic` (seeded integer prompts).  `--model_args "alpha=0.1,seed=0,max_ctx=2048"`
uses the reference's own (otherwise unused) key=value channel (arguments.py:28-55).
"""
from __future__ import annotations

import csv
import json
import os
import sys
import time
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import torch

from .plugin import GenerationConfig, GenerationResult, HuggingfaceLlamaGenerator
from .synthetic import IntegerTokenizer, synthetic_prompts
from .weights import ARCHS, SyntheticLlama


@dataclass
class Arguments:                      # arguments.py:19-24
    model: str = "synthetic:tiny-gqa"
    model_args: Optional[str] = None
    seed: Optional[int] = 42
    output_dir: str = "./logs"


@dataclass
class BenchmarkArguments:             # benchmark.py:43-50
    dataset: str = "synthetic"
    data_path: Optional[str] = None
    random_shuffle: bool = True
    num_samples: Optional[int] = 8
    n_shot: Optional[int] = 0
    template: Optional[str] = None
    prompt_len: int = 128             # synthetic dataset only
    # not in the reference: generate the prompts this many at a time (self-speculation only,
    # B200SelfSpeculativeGenerationStrategy.generate_batch); 1 generates them one by one
    batch_size: int = 1


@dataclass
class SweepArguments:                 # sweep.py:27-34
    exit_layer_first: Optional[int] = 1
    exit_layer_last: Optional[int] = 15
    exit_layer_step: Optional[int] = 1
    num_speculations_first: Optional[int] = 1
    num_speculations_last: Optional[int] = 6
    num_speculations_step: Optional[int] = 1


@dataclass
class GenerateArguments:              # generate.py:32-39
    streamer: str = "standard"        # none | standard | speculative


@dataclass
class ScoreArguments:
    exit_layers: str = "4,8,16,-1"    # comma-separated; -1 (or any value <= 0) = full depth
    # synthetic dataset only: extend each prompt by this many tokens of the model's own full-depth
    # greedy output, so the scored text is one the full model finds likely (0 = prompts only)
    continuation_len: int = 64


def parse_model_args(text: Optional[str]) -> Dict[str, Any]:
    """`k=v,k=v` -> dict with bool/int/float coercion (arguments.py:28-55)."""
    out: Dict[str, Any] = {}
    for item in (text or "").strip().split(","):
        if not item:
            continue
        k, v = item.split("=")
        if v.lower() in ("true", "false"):
            out[k] = v.lower() == "true"
        elif v.isnumeric():
            out[k] = int(v)
        else:
            try:
                out[k] = float(v)
            except ValueError:
                out[k] = v
    return out


def parse(*dataclasses_):
    import transformers
    return transformers.HfArgumentParser(dataclasses_).parse_args_into_dataclasses()


def load_model_and_tokenizer(args: Arguments, exit_layer: int):
    """generate.py:54-67 — local HF checkpoint, or a synthetic model + integer tokenizer."""
    margs = parse_model_args(args.model_args)
    if args.model.startswith("synthetic:"):
        arch = ARCHS[args.model.split(":", 1)[1]]
        model = SyntheticLlama(arch, seed=int(margs.get("seed", 0)), alpha=float(margs.get("alpha", 1.0)),
                               damp_from=exit_layer if exit_layer > 0 else None)
        return model, IntegerTokenizer(arch.vocab), margs
    # local HF checkpoint directory: streamed shard by shard into the engine (checkpoint.py);
    # the HF model object is never built, so host memory stays at one tensor
    from .checkpoint import CheckpointLlama
    model = CheckpointLlama(args.model)
    has_tok = any(os.path.exists(os.path.join(args.model, f))
                  for f in ("tokenizer.model", "tokenizer.json", "tokenizer_config.json"))
    if has_tok:
        import transformers
        tok = transformers.AutoTokenizer.from_pretrained(args.model, use_fast=False)
    else:
        tok = IntegerTokenizer(model.arch.vocab)
    return model, tok, margs


def make_strategy(name: str, margs: Dict[str, Any]):
    """The dispatch of generate.py:86-93 / benchmark.py:162-169, B200 strategies only."""
    from .strategy import (B200AutoRegressiveGenerationStrategy,
                           B200SelfSpeculativeGenerationStrategy)
    max_ctx = int(margs.get("max_ctx", 4096))
    if name in ("autoregressive", "b200_autoregressive"):
        return B200AutoRegressiveGenerationStrategy(max_ctx=max_ctx)
    if name in ("self_speculative", "b200_self_speculative"):
        return B200SelfSpeculativeGenerationStrategy(max_ctx=max_ctx)
    raise ValueError(f"unknown generation strategy {name!r}")


def synthetic_examples(vocab: int, n: int, prompt_len: int) -> List[str]:
    tok = IntegerTokenizer(vocab)
    return [tok.decode(p) for p in synthetic_prompts(vocab, n, prompt_len)]


class Mean:
    def __init__(self):
        self.s, self.n = 0.0, 0

    def update(self, v):
        if v is not None:
            self.s += float(v)
            self.n += 1

    def compute(self):
        return self.s / self.n if self.n else None


def benchmark(model, tokenizer, bench_args: BenchmarkArguments, gen_cfg: GenerationConfig,
              margs: Dict[str, Any], seed: int = 0) -> Dict[str, Any]:
    """benchmark.py:155-204 without the text metrics: means of acceptance rate, total time,
    time per token, tokens per second (benchmark.py:149-153)."""
    if bench_args.dataset != "synthetic":
        raise NotImplementedError("only --dataset synthetic is available offline")
    torch.manual_seed(seed)
    generator = HuggingfaceLlamaGenerator(tokenizer, model, make_strategy(gen_cfg.generation_strategy, margs))
    vocab = model.config.vocab_size
    means = {k: Mean() for k in ("acceptance_rate", "total_time", "time_per_token", "tokens_per_second")}
    n = bench_args.num_samples or 8
    examples = synthetic_examples(vocab, n, bench_args.prompt_len)
    # the reference times an already-loaded model: build the engine (weight upload / repack, CUDA
    # graph capture) and run one short generation BEFORE the timed loop
    warm = GenerationConfig(**{**vars(gen_cfg), "max_steps": min(8, gen_cfg.max_steps)})
    if bench_args.batch_size > 1:
        return _benchmark_batched(generator, examples, bench_args.batch_size, gen_cfg, warm, means)
    generator.generate(examples[0], warm)
    for prompt in examples:
        res: GenerationResult = generator.generate(prompt, gen_cfg)
        means["acceptance_rate"].update(res.generation_strategy_result.acceptance_rate)
        means["total_time"].update(res.total_time)
        means["time_per_token"].update(res.time_per_token)
        means["tokens_per_second"].update(res.tokens_per_second)
    generator.generation_strategy.engines.close()
    return {k: {"mean": v.compute()} for k, v in means.items()}


def _benchmark_batched(generator, examples: List[str], batch_size: int, gen_cfg: GenerationConfig,
                       warm: GenerationConfig, means: Dict[str, Mean]) -> Dict[str, Any]:
    """`benchmark` with the prompts generated batch_size at a time (generate_batch).  Each prompt's
    acceptance rate is its own; total time is the wall time of its group's generate_batch call, and
    time per token / tokens per second count every token of the group over that time.  When
    sampling, each prompt gets its own seed, drawn in prompt order from torch's global generator as
    a one-by-one generation draws its seed (a run under torch.manual_seed repeats)."""
    strategy = generator.generation_strategy
    if not hasattr(strategy, "generate_batch"):
        raise ValueError("--batch_size > 1 needs --generation_strategy self_speculative")
    tok = generator.tokenizer
    eos_ids = list(gen_cfg.stop_token_ids) + [tok.eos_token_id]
    ids = [tok(p, return_tensors="pt", add_special_tokens=True)["input_ids"].tolist()[0] for p in examples]

    def seeds(n):
        return [int(torch.randint(0, 2 ** 31 - 1, ()).item()) for _ in range(n)] if gen_cfg.sample else None

    strategy.generate_batch(generator.model, ids[:batch_size], eos_ids, warm, seeds=seeds(len(ids[:batch_size])))
    for g in range(0, len(ids), batch_size):
        group = ids[g:g + batch_size]
        group_seeds = seeds(len(group))
        t0 = time.perf_counter()
        results = strategy.generate_batch(generator.model, group, eos_ids, gen_cfg, seeds=group_seeds)
        elapsed = time.perf_counter() - t0
        n = sum(len(r.predicted_tokens) for r in results)
        for r in results:
            means["acceptance_rate"].update(r.acceptance_rate)
            means["total_time"].update(elapsed)
        means["time_per_token"].update(elapsed / n if n else None)
        means["tokens_per_second"].update(n / elapsed)
    strategy.engines.close()
    return {k: {"mean": v.compute()} for k, v in means.items()}


def main_benchmark(argv=None):
    if argv is not None:
        sys.argv = [sys.argv[0]] + list(argv)
    args, bargs, gcfg = parse(Arguments, BenchmarkArguments, GenerationConfig)
    model, tok, margs = load_model_and_tokenizer(args, gcfg.exit_layer)
    gcfg.stop_token_ids = gcfg.stop_token_ids or []
    metrics = benchmark(model, tok, bargs, gcfg, margs, args.seed or 0)
    os.makedirs(args.output_dir, exist_ok=True)
    path = os.path.join(args.output_dir, f"benchmark_{time.strftime('%Y%m%d_%H%M%S')}.json")
    with open(path, "w") as f:
        json.dump({"args": vars(args), "benchmark_arguments": vars(bargs),
                   "generation_config": vars(gcfg), "metrics": metrics}, f, indent=1)
    print(json.dumps(metrics))
    return metrics


def main_sweep(argv=None):
    """sweep.py:36-74: exit_layer x num_speculations grid, CSV rewritten after every point."""
    if argv is not None:
        sys.argv = [sys.argv[0]] + list(argv)
    args, bargs, sargs, gcfg = parse(Arguments, BenchmarkArguments, SweepArguments, GenerationConfig)
    os.makedirs(args.output_dir, exist_ok=True)
    path = os.path.join(args.output_dir, f"sweep_{time.strftime('%Y%m%d_%H%M%S')}.csv")
    rows: List[Dict[str, Any]] = []
    model_cache: Dict[int, Any] = {}
    for e in range(sargs.exit_layer_first, sargs.exit_layer_last + 1, sargs.exit_layer_step):
        for d in range(sargs.num_speculations_first, sargs.num_speculations_last + 1,
                       sargs.num_speculations_step):
            gcfg.exit_layer, gcfg.num_speculations = e, d
            gcfg.generation_strategy = "self_speculative"
            if e not in model_cache:
                model_cache.clear()
                model_cache[e] = load_model_and_tokenizer(args, e)
            model, tok, margs = model_cache[e]
            m = benchmark(model, tok, bargs, gcfg, margs, args.seed or 0)
            rows.append({"exit_layer": e, "num_speculations": d,
                         "acceptance_rate": m["acceptance_rate"]["mean"],
                         "total_time": m["total_time"]["mean"],
                         "time_per_token": m["time_per_token"]["mean"],
                         "tokens_per_second": m["tokens_per_second"]["mean"]})
            with open(path, "w", newline="") as f:
                wr = csv.DictWriter(f, fieldnames=list(rows[0]))
                wr.writeheader()
                wr.writerows(rows)
            print(rows[-1], flush=True)
    return rows


def main_correctness(argv=None):
    """correctness.py:38-92: self-speculative vs autoregressive decoded text, error count."""
    if argv is not None:
        sys.argv = [sys.argv[0]] + list(argv)
    args, bargs, gcfg = parse(Arguments, BenchmarkArguments, GenerationConfig)
    model, tok, margs = load_model_and_tokenizer(args, gcfg.exit_layer)
    from copy import copy
    spec_cfg = copy(gcfg)
    spec_cfg.generation_strategy = "self_speculative"
    ar_cfg = copy(gcfg)
    ar_cfg.exit_layer, ar_cfg.num_speculations, ar_cfg.generation_strategy = -1, -1, "autoregressive"
    spec_strategy = make_strategy("self_speculative", margs)
    from .strategy import B200AutoRegressiveGenerationStrategy
    spec = HuggingfaceLlamaGenerator(tok, model, spec_strategy)
    ar = HuggingfaceLlamaGenerator(tok, model, B200AutoRegressiveGenerationStrategy(
        engine_cache=spec_strategy.engines))
    prompts = synthetic_examples(model.config.vocab_size, bargs.num_samples or 8, bargs.prompt_len)
    errors = sum(spec.generate(p, spec_cfg).decoded_prediction != ar.generate(p, ar_cfg).decoded_prediction
                 for p in prompts)
    result = {"errors": errors, "error_pct": errors / len(prompts)}
    os.makedirs(args.output_dir, exist_ok=True)
    with open(os.path.join(args.output_dir, f"correctness_{time.strftime('%Y%m%d_%H%M%S')}.json"), "w") as f:
        json.dump(result, f)
    print(result)
    spec_strategy.engines.close()
    return result


def parse_exit_layers(text: str) -> List[int]:
    """`"4,8,16,-1"` -> [4, 8, 16, -1]; values <= 0 mean full depth."""
    return [int(t) for t in text.split(",") if t.strip()]


def main_score(argv=None):
    """Per-exit-layer quality of the early-exit sub-model (layers < E + shared norm and head) in one
    teacher-forced pass per sequence: mean NLL per token and perplexity, greedy accuracy (arg-max
    == next token), agreement with full depth (arg-max at E == arg-max at full depth: what greedy
    self-speculation accepts), and scored tokens per second of device time."""
    if argv is not None:
        sys.argv = [sys.argv[0]] + list(argv)
    args, bargs, sargs = parse(Arguments, BenchmarkArguments, ScoreArguments)
    if bargs.dataset != "synthetic":
        raise NotImplementedError("only --dataset synthetic is available offline")
    exits = parse_exit_layers(sargs.exit_layers)
    positive = [e for e in exits if e > 0]
    # alpha damping (--model_args alpha=...) starts at the shallowest exit layer
    model, _tok, margs = load_model_and_tokenizer(args, min(positive) if positive else -1)
    arch = model.arch
    if any(e > arch.layers for e in exits):
        raise ValueError(f"--exit_layers {sargs.exit_layers}: the model has {arch.layers} layers")
    from .engine import Engine
    cont = max(0, sargs.continuation_len)
    max_ctx = max(int(margs.get("max_ctx", 0)), bargs.prompt_len + cont + 2)
    eng = Engine(arch, max_ctx=max_ctx)
    eng.load_model(model)
    texts = []
    for p in synthetic_prompts(arch.vocab, bargs.num_samples or 8, bargs.prompt_len):
        if cont:
            eng.begin(-1, cont, [])
            eng.prefill(p)
            p = p + [eng.ar_step() for _ in range(cont)]
        texts.append(p)
    full = {}
    for i, ids in enumerate(texts):
        full[i] = eng.score(ids, -1)[1]
    results = []
    for e in exits:
        lp_all, hit, agree, ms = [], 0, 0, 0.0
        for i, ids in enumerate(texts):
            lp, greedy = eng.score(ids, e)
            ms += eng.last_device_ms
            lp_all.append(lp.to(torch.float64))
            hit += int((greedy == torch.tensor(ids[1:])).sum())
            agree += int((greedy == full[i]).sum())
        lp = torch.cat(lp_all)
        n_tok = lp.numel()
        nll = float(-lp.mean())
        results.append({"exit_layer": e if e > 0 else arch.layers, "mean_nll": nll,
                        "perplexity": float(torch.exp(torch.tensor(nll, dtype=torch.float64))),
                        "greedy_accuracy": hit / n_tok, "agreement_with_full": agree / n_tok,
                        "scored_tokens": n_tok, "device_ms": ms,
                        "tokens_per_second": n_tok / (ms / 1e3) if ms > 0 else None})
    eng.close()
    print(f"{'exit':>5} {'nll/token':>10} {'perplexity':>12} {'greedy acc':>11} {'agree full':>11} {'tokens/s':>11}")
    for r in results:
        print(f"{r['exit_layer']:>5} {r['mean_nll']:>10.4f} {r['perplexity']:>12.2f} {r['greedy_accuracy']:>11.4f} "
              f"{r['agreement_with_full']:>11.4f} {r['tokens_per_second'] or 0:>11.0f}")
    os.makedirs(args.output_dir, exist_ok=True)
    path = os.path.join(args.output_dir, f"score_{time.strftime('%Y%m%d_%H%M%S')}.json")
    with open(path, "w") as f:
        json.dump({"args": vars(args), "benchmark_arguments": vars(bargs), "score_arguments": vars(sargs),
                   "results": results}, f, indent=1)
    return results


def predict_grid(eng, prompts: List[List[int]], exit_layers: List[int], num_speculations: List[int],
                 gcfg: GenerationConfig, n_layers: int, seed: int = 0) -> List[Dict[str, Any]]:
    """The sweep's (exit layer, num_speculations) grid predicted from one `score_exits` pass per
    prompt (predict.py).  Each prompt is extended by max_steps tokens of full-depth generation: AR
    greedy, or AR sampled with the generation config's warp, which has the distribution of sampled
    self-speculation's output.  Greedy rows are exact; sampled rows use each exit's mean
    acceptance probability in the i.i.d. formula and are marked exact = False."""
    from . import predict
    steps = gcfg.max_steps
    exits = sorted(set(exit_layers) | {n_layers})
    warp = {"temperature": gcfg.temperature, "top_k": gcfg.top_k, "top_p": gcfg.top_p} if gcfg.sample else None
    g = torch.Generator().manual_seed(seed)
    per_prompt: List[Dict[int, Any]] = []
    for p in prompts:
        eng.begin(-1, steps, [], sample=gcfg.sample, temperature=gcfg.temperature, top_k=gcfg.top_k,
                  top_p=gcfg.top_p, seed=int(torch.randint(0, 2 ** 31 - 1, (), generator=g)))
        eng.prefill(p)
        cont = [eng.ar_step() for _ in range(steps)]
        _lp, greedy, accept = eng.score_exits(p + cont, exits, warp)
        rows = slice(len(p) - 1, len(p) - 1 + steps)      # row len(p) - 1 + q predicts cont[q]
        want = torch.tensor(cont, dtype=torch.int64)
        per = {}
        for j, e in enumerate(exits):
            if e not in exit_layers:
                continue
            if not warp:
                per[e] = (greedy[j, rows] == want).tolist()
            else:   # a draft at full depth is drawn from the verifier's own distribution: alpha = 1
                per[e] = accept[j, rows] if e < n_layers else torch.ones(steps)
        per_prompt.append(per)
    out = []
    for e in exit_layers:
        if warp:
            alpha = float(torch.cat([pp[e].to(torch.float64) for pp in per_prompt]).mean())
        for d in num_speculations:
            if warp:
                acc, tpr = predict.sampled_estimate(alpha, d)
                out.append({"exit_layer": e, "num_speculations": d, "acceptance_rate": acc,
                            "tokens_per_round": tpr, "exact": False, "mean_alpha": alpha})
            else:
                rounds = [predict.greedy_rounds(pp[e], d, steps) for pp in per_prompt]
                out.append({"exit_layer": e, "num_speculations": d,
                            "acceptance_rate": predict.mean(predict.acceptance_rate(r) for r in rounds),
                            "tokens_per_round": predict.mean(predict.tokens_per_round(r) for r in rounds),
                            "exact": True})
    return out


def main_predict(argv=None):
    """The sweep's grid (sweep.py:36-74 arguments) predicted from ONE teacher-forced pass per prompt
    at every exit at once, instead of one benchmark per (E, D).  Writes predict_*.csv with
    exit_layer, num_speculations, acceptance_rate, tokens_per_round, exact.  With --model_args
    alpha=... the damping starts at exit_layer_first (as in `main_score`): the prediction is for
    generations on that one model, not for `main_sweep`'s per-E models."""
    if argv is not None:
        sys.argv = [sys.argv[0]] + list(argv)
    args, bargs, sargs, gcfg = parse(Arguments, BenchmarkArguments, SweepArguments, GenerationConfig)
    if bargs.dataset != "synthetic":
        raise NotImplementedError("only --dataset synthetic is available offline")
    if gcfg.no_repeat_ngram_size:
        raise NotImplementedError("the prediction does not model the n-gram ban (--no_repeat_ngram_size)")
    exit_layers = list(range(sargs.exit_layer_first, sargs.exit_layer_last + 1, sargs.exit_layer_step))
    specs = list(range(sargs.num_speculations_first, sargs.num_speculations_last + 1, sargs.num_speculations_step))
    model, _tok, margs = load_model_and_tokenizer(args, sargs.exit_layer_first)
    arch = model.arch
    if not exit_layers or min(exit_layers) < 1 or max(exit_layers) > arch.layers:
        raise ValueError(f"exit layers {exit_layers} must lie in [1, {arch.layers}]")
    from .engine import Engine
    max_ctx = max(int(margs.get("max_ctx", 0)), bargs.prompt_len + gcfg.max_steps + 2)
    eng = Engine(arch, max_ctx=max_ctx)
    try:
        eng.load_model(model)
        prompts = synthetic_prompts(arch.vocab, bargs.num_samples or 8, bargs.prompt_len)
        rows = predict_grid(eng, prompts, exit_layers, specs, gcfg, arch.layers, args.seed or 0)
    finally:
        eng.close()
    os.makedirs(args.output_dir, exist_ok=True)
    path = os.path.join(args.output_dir, f"predict_{time.strftime('%Y%m%d_%H%M%S')}.csv")
    fields = ["exit_layer", "num_speculations", "acceptance_rate", "tokens_per_round", "exact"]
    with open(path, "w", newline="") as f:
        wr = csv.DictWriter(f, fieldnames=fields, extrasaction="ignore")
        wr.writeheader()
        wr.writerows(rows)
    for r in rows:
        print({k: r[k] for k in fields + (["mean_alpha"] if "mean_alpha" in r else [])}, flush=True)
    return rows


class _PrintStreamer:
    """Plain-text stand-in for transformers.TextStreamer / SpeculativeTextStreamer."""

    def __init__(self, tokenizer, speculative: bool):
        self.tok = tokenizer
        if speculative:
            self.delete = lambda n: print(f"\n  <rejected the draft: {n} tokens>", flush=True)

    def put(self, ids, is_draft: bool = False):
        text = self.tok.decode(ids.flatten().tolist())
        print(("  draft: " if is_draft else "") + text, end=" ", flush=True)

    def end(self):
        print()


def main_generate(argv=None):
    """generate.py:69-142: read prompts from stdin, stream the continuation."""
    if argv is not None:
        sys.argv = [sys.argv[0]] + list(argv)
    args, gargs, gcfg = parse(Arguments, GenerateArguments, GenerationConfig)
    model, tok, margs = load_model_and_tokenizer(args, gcfg.exit_layer)
    generator = HuggingfaceLlamaGenerator(tok, model, make_strategy(gcfg.generation_strategy, margs))
    streamer = None if gargs.streamer == "none" else _PrintStreamer(tok, gargs.streamer == "speculative")
    for line in sys.stdin:
        line = line.strip()
        if not line:
            continue
        res = generator.generate(line, gcfg, streamer=streamer)
        print(f"\n[{res.num_tokens_generated} tokens, {res.tokens_per_second:.1f} tok/s, acceptance "
              f"{res.generation_strategy_result.acceptance_rate}]", flush=True)
    generator.generation_strategy.engines.close()

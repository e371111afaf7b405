#!/usr/bin/env python
"""Confidence-threshold drafting: `Engine.round_adaptive` against fixed-length `Engine.round`.

Synthetic Llama-2-7B with layers >= E damped by alpha (the bench's model family), E = 8, greedy
512-token generations on the bench's prompts.  Per alpha and per mode — `round(d_max)`, `round(1)`
and `round_adaptive(d_max, t)` for every threshold t — it reports tokens/s (wall time of the whole
generation, prefill included, as the bench measures), the acceptance rate (matches / actual drafts),
the mean drafts per round and the mean device ms per round.  The modes alternate prompt by prompt.
Prints the GPU name and power limit first (read-only nvidia-smi query), then one JSON line per point.

    python tools/adaptive_probe.py [--alphas 1.0,0.3,0.1] [--thresholds 0,0.001,0.003,0.1,0.3,0.6,1.0] [--prompts 8]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from score_probe import gpu_name_and_power_limit  # noqa: E402


def generate(eng, prompt, eos, exit_layer, max_steps, d_max, threshold):
    """The strategy's outer loop (max_steps clamp, EOS truncation) with one round kind."""
    eng.begin(exit_layer=exit_layer, max_steps=max_steps, eos_token_ids=eos, sample=False)
    eng.prefill(prompt)
    out, ms, drafted, matched = [], [], 0, 0
    while len(out) < max_steps:
        d = min(d_max, max_steps - len(out) - 1)
        r = eng.round(d) if threshold is None else eng.round_adaptive(d, threshold)
        ms.append(eng.last_device_ms)
        drafted += r.n_drafted
        matched += r.n_matches
        out += r.emitted
        if any(t in out for t in eos):
            break
    return out, ms, drafted, matched


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="llama2-7b")
    ap.add_argument("--exit_layer", type=int, default=8)
    ap.add_argument("--d_max", type=int, default=6)
    ap.add_argument("--alphas", default="1.0,0.3,0.1")
    ap.add_argument("--thresholds", default="0,0.001,0.003,0.1,0.3,0.6,1.0")
    ap.add_argument("--prompts", type=int, default=8, help="how many of the bench's 8 prompts to run")
    ap.add_argument("--prompt_len", type=int, default=128)
    ap.add_argument("--max_steps", type=int, default=512)
    a = ap.parse_args()
    import torch
    from layerskip_b200.engine import Engine
    from layerskip_b200.synthetic import synthetic_prompts
    from layerskip_b200.weights import ARCHS, SyntheticLlama
    arch = ARCHS[a.arch]
    prompts = synthetic_prompts(arch.vocab, 8, a.prompt_len)[:a.prompts]
    eos = [arch.vocab - 1]
    modes = [(f"round({a.d_max})", a.d_max, None), ("round(1)", 1, None)] + \
            [(f"adaptive(t={t})", a.d_max, float(t)) for t in a.thresholds.split(",")]
    print(json.dumps({"gpu": gpu_name_and_power_limit(), "arch": a.arch, "exit_layer": a.exit_layer,
                      "d_max": a.d_max, "prompts": len(prompts), "max_steps": a.max_steps}), flush=True)
    for alpha in [float(x) for x in a.alphas.split(",")]:
        eng = Engine(arch, max_ctx=a.prompt_len + a.max_steps + 64)
        eng.load_model(SyntheticLlama(arch, seed=0, alpha=alpha, damp_from=a.exit_layer))
        for _, d, t in modes:                                  # warm-up: graph capture of every shape
            generate(eng, prompts[0][:16], eos, a.exit_layer, 2 * a.d_max + 2, d, t)
        stats = {name: {"tokens": 0, "s": 0.0, "ms": [], "drafted": 0, "matched": 0, "rounds": 0}
                 for name, _, _ in modes}
        outputs = {}
        for p in prompts:
            for name, d, t in modes:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out, ms, drafted, matched = generate(eng, p, eos, a.exit_layer, a.max_steps, d, t)
                s = stats[name]
                s["s"] += time.perf_counter() - t0
                s["tokens"] += len(out)
                s["ms"] += ms
                s["drafted"] += drafted
                s["matched"] += matched
                s["rounds"] += len(ms)
                outputs.setdefault(name, []).append(out)
        ref = outputs[modes[0][0]]
        for name, _, _ in modes:
            s = stats[name]
            print(json.dumps({
                "alpha": alpha, "mode": name, "tokens_per_s": round(s["tokens"] / s["s"], 2),
                "acceptance": round(s["matched"] / max(1, s["drafted"]), 4),
                "drafts_per_round": round(s["drafted"] / max(1, s["rounds"]), 3),
                "device_ms_per_round": round(statistics.mean(s["ms"]), 4),
                "device_ms_per_round_median": round(statistics.median(s["ms"]), 4),
                "tokens_per_round": round(s["tokens"] / max(1, s["rounds"]), 3),
                "same_tokens_as_round": outputs[name] == ref}), flush=True)
        eng.close()
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

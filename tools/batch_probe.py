#!/usr/bin/env python
"""Batched self-speculation: aggregate throughput of B prompts generated together.

Synthetic Llama-2-7B with layers >= E damped by alpha (the bench's model family), E = 8, greedy
generations of the bench's prompts.  For B = 1, 2, 4, 8, 16 with D = 16 / B - 1 drafts (so every
verify carries 16 rows), B prompts run together through `Engine.round_batch` (B = 1 runs
`Engine.round`, B = 16 runs d = 0): the strategy's outer loop per sequence (max_steps clamp, EOS
deactivation).  Per B it reports aggregate tokens/s over the whole generation (wall time, prefill
included), rounds/s, mean device ms per round and the acceptance rate (matches / drafts).  Every B
runs once untimed first (graph capture of every round shape).  Prints the GPU name and power limit
first (read-only nvidia-smi query), then one JSON line per B.  With --sample each B runs greedy and
then sampled (temperature 0.6, top-p 0.9, the reference's defaults; sequence s seeded with 1000 + s),
one JSON line per mode.  With --thresholds t1,t2,.. each (B, mode) also runs with
confidence-threshold drafting at each threshold (`Engine.round_batch_adaptive`, B = 1:
`Engine.round_adaptive`) after the fixed rounds, one JSON line per threshold; every line also
reports the drafts per round per active sequence.

    python tools/batch_probe.py [--batches 1,2,4,8,16] [--alpha 0.3] [--max_steps 128] [--sample]
                                [--thresholds 0.003,0.1,1.0]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from score_probe import gpu_name_and_power_limit  # noqa: E402


SAMPLING = dict(temperature=0.6, top_k=0, top_p=0.9)


def generate(eng, prompts, eos, exit_layer, max_steps, D, sample=False, threshold=None):
    """Generation of `prompts` together, with fixed rounds or (`threshold` set) adaptive ones; returns
    (outputs, device ms per round, drafts, matches, sequence-rounds)."""
    seeds = [1000 + s for s in range(len(prompts))]
    eng.begin(exit_layer=exit_layer, max_steps=max_steps, eos_token_ids=eos, sample=sample,
              seed=seeds[0], **SAMPLING)
    if len(prompts) == 1:
        eng.prefill(prompts[0])
    else:
        eng.prefill_batch(prompts, seeds if sample else None)
    outs = [[] for _ in prompts]
    active = [True] * len(prompts)
    ms, drafted, matched, seq_rounds = [], 0, 0, 0
    while any(active):
        d_seq = [min(D, max_steps - len(o) - 1) if a else 0 for o, a in zip(outs, active)]
        d_req = max(d for d, a in zip(d_seq, active) if a)
        if threshold is None:
            rounds = [eng.round(d_req)] if len(prompts) == 1 else eng.round_batch(d_req, d_seq, active)
        elif len(prompts) == 1:
            rounds = [eng.round_adaptive(d_req, threshold)]
        else:
            rounds = eng.round_batch_adaptive(d_req, threshold, d_seq, active)
        ms.append(eng.last_device_ms)
        for s, r in enumerate(rounds):
            if not active[s]:
                continue
            seq_rounds += 1
            outs[s] += r.emitted
            drafted += r.n_drafted
            matched += r.n_matches
            if any(t in outs[s] for t in eos):
                outs[s] = outs[s][:min(outs[s].index(t) for t in eos if t in outs[s])]
                active[s] = False
            if len(outs[s]) >= max_steps:
                active[s] = False
    return outs, ms, drafted, matched, seq_rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="llama2-7b")
    ap.add_argument("--exit_layer", type=int, default=8)
    ap.add_argument("--alpha", type=float, default=0.3)
    ap.add_argument("--batches", default="1,2,4,8,16")
    ap.add_argument("--prompt_len", type=int, default=128)
    ap.add_argument("--max_steps", type=int, default=128)
    ap.add_argument("--sample", action="store_true", help="also run each B sampled (T 0.6, top-p 0.9)")
    ap.add_argument("--thresholds", default="", help="comma-separated confidence thresholds to run adaptively")
    a = ap.parse_args()
    import torch
    from layerskip_b200.engine import Engine
    from layerskip_b200.synthetic import synthetic_prompts
    from layerskip_b200.weights import ARCHS, SyntheticLlama
    arch = ARCHS[a.arch]
    batches = [int(b) for b in a.batches.split(",")]
    thresholds = [None] + [float(t) for t in a.thresholds.split(",") if t]
    n_max = max(batches)
    prompts = synthetic_prompts(arch.vocab, n_max, a.prompt_len)
    eos = [arch.vocab - 1]
    # every slot of the largest batch holds prompt + max_steps + D + 1 positions
    slot = (a.prompt_len + a.max_steps + 16 + 63) // 64 * 64
    eng = Engine(arch, max_ctx=n_max * slot)
    eng.load_model(SyntheticLlama(arch, seed=0, alpha=a.alpha, damp_from=a.exit_layer))
    print(json.dumps({"gpu": gpu_name_and_power_limit(), "arch": a.arch, "exit_layer": a.exit_layer,
                      "alpha": a.alpha, "prompt_len": a.prompt_len, "max_steps": a.max_steps,
                      "max_rows": eng.max_rows}), flush=True)
    for B in batches:
        for sample in ((False, True) if a.sample else (False,)):
            for t in thresholds:
                D = eng.max_rows // B - 1
                group = prompts[:B]
                args = (eng, group, eos, a.exit_layer, a.max_steps, D, sample, t)
                generate(*args)                                 # warm-up: capture every shape
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs, ms, drafted, matched, seq_rounds = generate(*args)
                s = time.perf_counter() - t0
                tokens = sum(len(o) for o in outs)
                print(json.dumps({"B": B, "D": D, "mode": "sampled" if sample else "greedy", "threshold": t,
                                  "tokens": tokens, "seconds": round(s, 4),
                                  "tokens_per_s": round(tokens / s, 1), "rounds": len(ms),
                                  "rounds_per_s": round(len(ms) / s, 1),
                                  "device_ms_per_round": round(sum(ms) / len(ms), 4),
                                  "drafts_per_round_per_seq": round(drafted / seq_rounds, 3),
                                  "acceptance": round(matched / drafted, 4) if drafted else None}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()

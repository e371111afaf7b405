#!/usr/bin/env python
"""Prefix-shared scoring: `Engine.loglikelihood_batch` (which scores requests that share a context
with one `score_prefixed` call) against `Engine.score_batch` of the same joined sequences.

Llama-2-7B shape with synthetic weights and seeded multiple-choice workloads:
  mmlu:      64 contexts of 400-900 ids x 4 one-id choices,
  hellaswag: 128 contexts of 80-160 ids x 4 endings of 15-40 ids,
  arc:       256 contexts of 40-80 ids x 4 choices of 3-12 ids,
  control:   no sharing, workload A of tools/score_batch_probe.py (256 requests of 8-64 ids, each
             cut into a one-id context and its continuation), which must keep taking score_batch.
Each runs at every exit layer, `--reps` times alternating the two calls.  Per point: the route
`loglikelihood_batch` took, the median device ms of each call, requests/s, and the max |d| between
the two over the continuations' summed log-probabilities (must be 0) and whether every greedy flag
agrees.  Prints one JSON line per point and the GPU name and power limit (read-only nvidia-smi query).

    python tools/score_prefixed_probe.py [--arch llama2-7b] [--exits 8,32] [--max_ctx 8192] [--reps 3]
"""
import argparse
import json
import os
import random
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from score_batch_probe import requests as batch_requests  # noqa: E402
from score_probe import gpu_name_and_power_limit  # noqa: E402

# contexts, (context ids lo, hi), choices per context, (choice ids lo, hi)
WORKLOADS = {"mmlu": (64, (400, 900), 4, (1, 1)), "hellaswag": (128, (80, 160), 4, (15, 40)),
             "arc": (256, (40, 80), 4, (3, 12))}


def mc_requests(vocab, name, seed=7):
    n, (clo, chi), k, (blo, bhi) = WORKLOADS[name]
    rng = random.Random(f"{name}{seed}")
    tok = lambda m: [rng.randrange(3, vocab - 1) for _ in range(m)]   # noqa: E731
    out = []
    for _ in range(n):
        ctx = tok(rng.randint(clo, chi))
        out += [(ctx, tok(rng.randint(blo, bhi))) for _ in range(k)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="llama2-7b")
    ap.add_argument("--exits", default="8,32")
    ap.add_argument("--max_ctx", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="mmlu,hellaswag,arc,control")
    a = ap.parse_args()
    import torch
    from layerskip_b200.engine import Engine
    from layerskip_b200.weights import ARCHS, SyntheticLlama
    arch = ARCHS[a.arch]
    exits = [int(x) for x in a.exits.split(",")]
    print(json.dumps({"gpu": gpu_name_and_power_limit(), "arch": a.arch, "max_ctx": a.max_ctx}), flush=True)
    eng = Engine(arch, max_ctx=a.max_ctx, prefill_tc=True)
    eng.load_model(SyntheticLlama(arch, seed=0))
    for name in a.workloads.split(","):
        if name == "control":
            reqs = [(r[:1], r[1:]) for r in batch_requests(arch.vocab, "A")]
        else:
            reqs = mc_requests(arch.vocab, name)
        seqs = [c + k for c, k in reqs]
        _, _, prefixed = Engine._prefix_plan(seqs, [k for _, k in reqs])
        for e in exits:
            eng.loglikelihood_batch(reqs[:8], e)               # warm-up: lazy buffers, first launches
            eng.score_batch(seqs[:8], e)
            shared_ms, joined_ms = [], []
            for _ in range(a.reps):
                got = eng.loglikelihood_batch(reqs, e)
                shared_ms.append(eng.last_device_ms)
                joined = eng.score_batch(seqs, e)
                joined_ms.append(eng.last_device_ms)
            want = [Engine._continuation_score(lp, gr, k) for (lp, gr), (_, k) in zip(joined, reqs)]
            point = {"workload": name, "requests": len(reqs), "exit_layer": e,
                     "route": "score_prefixed" if prefixed else "score_batch"}
            for mode, ms in (("loglikelihood_batch", shared_ms), ("score_batch", joined_ms)):
                med = statistics.median(ms)
                point[f"{mode}_ms"] = round(med, 3)
                point[f"{mode}_ms_range"] = [round(min(ms), 3), round(max(ms), 3)]
                point[f"{mode}_requests_per_s"] = round(len(reqs) / (med / 1e3), 1)
            point["speedup"] = round(statistics.median(joined_ms) / statistics.median(shared_ms), 3)
            point["max_abs_dloglikelihood"] = max(abs(g[0] - w[0]) for g, w in zip(got, want))
            point["greedy_flags_equal"] = all(g[1] == w[1] for g, w in zip(got, want))
            print(json.dumps(point), flush=True)
    eng.close()
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

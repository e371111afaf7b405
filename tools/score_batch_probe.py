#!/usr/bin/env python
"""Batched scoring against a per-request scoring loop on the same requests.

Llama-2-7B shape with synthetic weights and seeded requests, three workloads:
  A: 256 requests of 8-64 ids (lm-eval `loglikelihood`-sized),
  B: 64 requests of 96-400 ids,
  C: 64 requests of 1024 ids.
Each runs at every exit layer, once as a loop of `Engine.score` calls and once as one
`Engine.score_batch` call.  Per point: device ms (the sum of the loop's calls), requests/s and scored
tokens/s, and the max |d logprob| between the two over requests of more than max_rows + 1 ids (the
loop takes the same wgmma route there: must be 0) and over all requests (shorter ones take the
decode route in the loop).  Prints one JSON line per point and the GPU name and power limit
(read-only nvidia-smi query).

    python tools/score_batch_probe.py [--arch llama2-7b] [--exits 8,32] [--max_ctx 8192] [--workloads A,B,C]
"""
import argparse
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from score_probe import gpu_name_and_power_limit  # noqa: E402

WORKLOADS = {"A": (256, 8, 64), "B": (64, 96, 400), "C": (64, 1024, 1024)}


def requests(vocab, name, seed=7):
    n, lo, hi = WORKLOADS[name]
    rng = random.Random(f"{name}{seed}")
    return [[rng.randrange(3, vocab - 1) for _ in range(rng.randint(lo, hi))] for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="llama2-7b")
    ap.add_argument("--exits", default="8,32")
    ap.add_argument("--max_ctx", type=int, default=8192)
    ap.add_argument("--workloads", default="A,B,C")
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
        reqs = requests(arch.vocab, name)
        tokens = sum(len(r) - 1 for r in reqs)
        for e in exits:
            eng.score(reqs[0], e)                              # warm-up: lazy buffers, first launches
            eng.score_batch(reqs[:4], e)
            loop, loop_ms = [], 0.0
            for r in reqs:
                loop.append(eng.score(r, e))
                loop_ms += eng.last_device_ms
            batch = eng.score_batch(reqs, e)
            batch_ms = eng.last_device_ms
            d_long, d_all = 0.0, 0.0
            for r, (lp, _), (bl, _) in zip(reqs, loop, batch):
                d = float((lp - bl).abs().max())
                d_all = max(d_all, d)
                if len(r) > eng.max_rows + 1:
                    d_long = max(d_long, d)
            point = {"workload": name, "requests": len(reqs), "scored_tokens": tokens, "exit_layer": e}
            for mode, ms in (("loop", loop_ms), ("batch", batch_ms)):
                point[f"{mode}_ms"] = round(ms, 3)
                point[f"{mode}_requests_per_s"] = round(len(reqs) / (ms / 1e3), 1)
                point[f"{mode}_tokens_per_s"] = round(tokens / (ms / 1e3))
            point["speedup"] = round(loop_ms / batch_ms, 3)
            point["max_abs_dlogprob_long"] = d_long
            point["max_abs_dlogprob_all"] = d_all
            print(json.dumps(point), flush=True)
    eng.close()
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

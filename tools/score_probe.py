#!/usr/bin/env python
"""Cost of teacher-forced scoring against the prompt pass on the same ids.

Llama-2-7B shape with synthetic weights, wgmma prompt path, 8 sequences each of 1024 and of 128
tokens, exit layers 8 and 32.  Per (length, E): `lsk_score` device ms per sequence, scored tokens
per second, and `lsk_prefill` device ms for the same ids, so the extra cost of scoring (the last
layer run to the end, the LM head on every row and the log softmax) shows separately.  Prints one
JSON line per point and the GPU name and power limit (read-only nvidia-smi query).

    python tools/score_probe.py [--arch llama2-7b] [--seqs 8] [--lens 1024,128] [--exits 8,32]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_name_and_power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:  # pragma: no cover
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="llama2-7b")
    ap.add_argument("--seqs", type=int, default=8)
    ap.add_argument("--lens", default="1024,128")
    ap.add_argument("--exits", default="8,32")
    a = ap.parse_args()
    import torch
    from layerskip_b200.engine import Engine
    from layerskip_b200.synthetic import synthetic_prompts
    from layerskip_b200.weights import ARCHS, SyntheticLlama
    arch = ARCHS[a.arch]
    lens = [int(x) for x in a.lens.split(",")]
    exits = [int(x) for x in a.exits.split(",")]
    print(json.dumps({"gpu": gpu_name_and_power_limit(), "arch": a.arch}), flush=True)
    eng = Engine(arch, max_ctx=max(lens) + 64, prefill_tc=True)
    eng.load_model(SyntheticLlama(arch, seed=0))
    for n in lens:
        seqs = synthetic_prompts(arch.vocab, a.seqs, n, seed=99)
        eng.score(seqs[0], exits[0])                          # warm-up (lazy buffers, first launches)
        pre = []
        for ids in seqs:
            eng.begin(-1, 1, [])
            eng.prefill(ids)
            pre.append(eng.last_device_ms)
        for e in exits:
            ms = []
            for ids in seqs:
                eng.score(ids, e)
                ms.append(eng.last_device_ms)
            score_ms = statistics.median(ms)
            print(json.dumps({"tokens": n, "exit_layer": e, "score_ms": round(score_ms, 3),
                              "scored_tokens_per_s": round((n - 1) / (score_ms / 1e3)),
                              "prefill_ms_same_ids": round(statistics.median(pre), 3),
                              "score_ms_all": [round(x, 3) for x in ms]}), flush=True)
    eng.close()
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Multi-exit scoring: its speed against one `lsk_score` per exit, and how well it predicts the
acceptance of self-speculative generation.

Llama-2-7B shape with synthetic weights damped from layer 4 (`alpha`), wgmma prompt path.
* speed: device ms of one `score_exits` pass against the sum of `score` calls at every exit, for
  exit sets {4, 8, 16, 24, 32} and {1 .. 15, 32}, at 128 and 1024 ids (median over sequences);
* greedy prediction: for E x D, acceptance rate and tokens per round predicted from one pass per
  prompt against the generated rounds, and how many runs differ (prompt-pass scoring and decode
  kernels round differently);
* sampled prediction: mean alpha per exit against the measured acceptance per evaluated draft.
Prints one JSON line per point and the GPU name and power limit (read-only nvidia-smi query).

    python tools/score_exits_probe.py [--seqs 4] [--prompts 4] [--steps 128] [--alpha 0.2]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from score_probe import gpu_name_and_power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="llama2-7b")
    ap.add_argument("--seqs", type=int, default=4)
    ap.add_argument("--prompts", type=int, default=4)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--alpha", type=float, default=0.2)
    ap.add_argument("--exits", default="4,8,16")
    ap.add_argument("--specs", default="2,4,6")
    a = ap.parse_args()
    import torch
    from layerskip_b200 import GenerationConfig, predict
    from layerskip_b200.engine import Engine
    from layerskip_b200.strategy import B200SelfSpeculativeGenerationStrategy
    from layerskip_b200.synthetic import synthetic_prompts
    from layerskip_b200.weights import ARCHS, SyntheticLlama
    arch = ARCHS[a.arch]
    L = arch.layers
    print(json.dumps({"gpu": gpu_name_and_power_limit(), "arch": a.arch, "alpha": a.alpha}), flush=True)
    model = SyntheticLlama(arch, seed=0, alpha=a.alpha, damp_from=4)

    # ---- speed
    eng = Engine(arch, max_ctx=1024 + 64, prefill_tc=True)
    eng.load_model(model)
    for n in (128, 1024):
        seqs = synthetic_prompts(arch.vocab, a.seqs, n, seed=99)
        for exits in ([4, 8, 16, 24, L], list(range(1, 16)) + [L]):
            eng.score_exits(seqs[0], exits)                      # warm-up (lazy buffers)
            one, each = [], []
            for ids in seqs:
                eng.score_exits(ids, exits)
                one.append(eng.last_device_ms)
                tot = 0.0
                for e in exits:
                    eng.score(ids, e)
                    tot += eng.last_device_ms
                each.append(tot)
            print(json.dumps({"tokens": n, "exits": exits, "score_exits_ms": round(statistics.median(one), 3),
                              "sum_of_score_ms": round(statistics.median(each), 3),
                              "speedup": round(statistics.median(each) / statistics.median(one), 3)}), flush=True)
    eng.close()

    # ---- prediction against generation (one model: damping from layer 4)
    exits = [int(x) for x in a.exits.split(",")]
    specs = [int(x) for x in a.specs.split(",")]
    prompts = synthetic_prompts(arch.vocab, a.prompts, 64, seed=7)
    strat = B200SelfSpeculativeGenerationStrategy(max_ctx=64 + a.steps + 8)
    eng = strat.engine_for(model)
    for sample in (False, True):
        warp = {"temperature": 0.6, "top_k": 0, "top_p": 0.9} if sample else None
        for E in exits:
            ev_acc, ev_alpha = [], []
            for D in specs:
                cfg = GenerationConfig(max_steps=a.steps, exit_layer=E, num_speculations=D, sample=sample,
                                       **(warp or {}))
                got_acc, got_tpr, pred_acc, pred_tpr, differ = [], [], [], [], 0
                for i, p in enumerate(prompts):
                    torch.manual_seed(1000 + i)
                    res = strat.generate_token_ids(model, p, [], cfg)
                    out, rounds = res.predicted_tokens, strat.last_rounds
                    got = [(r.n_drafted, r.n_matches) for r in rounds]
                    got_acc.append(res.acceptance_rate)
                    got_tpr.append(predict.tokens_per_round(got))
                    _, greedy, acc = eng.score_exits(p + out, [E, L] if sample else [E], warp)
                    base = len(p) - 1
                    if not sample:
                        agree = (greedy[0, base:] == torch.tensor(out)).tolist()
                        pr = predict.greedy_rounds(agree, D, a.steps)
                        differ += int(pr != got)
                        pred_acc.append(predict.acceptance_rate(pr))
                        pred_tpr.append(predict.tokens_per_round(pr))
                        continue
                    o = 0
                    for r in rounds:
                        for j in range(min(r.n_matches + 1, r.n_drafted)):
                            ev_acc.append(1.0 if j < r.n_matches else 0.0)
                            ev_alpha.append(float(acc[0, base + o + j]))
                        o += r.n_matches + 1
                    alpha = float(acc[0, base:base + a.steps].double().mean())
                    pa, pt = predict.sampled_estimate(alpha, D)
                    pred_acc.append(pa)
                    pred_tpr.append(pt)
                row = {"sample": sample, "exit_layer": E, "num_speculations": D,
                       "generated_acceptance_rate": predict.mean(got_acc),
                       "predicted_acceptance_rate": predict.mean(pred_acc),
                       "generated_tokens_per_round": predict.mean(got_tpr),
                       "predicted_tokens_per_round": predict.mean(pred_tpr)}
                if not sample:
                    row["runs_with_differing_rounds"] = differ
                print(json.dumps(row), flush=True)
            if sample:
                print(json.dumps({"sample": True, "exit_layer": E, "evaluated_drafts": len(ev_acc),
                                  "measured_acceptance_per_draft": sum(ev_acc) / len(ev_acc),
                                  "mean_alpha_of_evaluated_drafts": sum(ev_alpha) / len(ev_alpha)}), flush=True)
    strat.engines.close()
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

"""Prefill timing probe: python tools/prefill_probe.py [arch] [n_tokens ...]
Device time of lsk_prefill (CUDA events on the engine's stream) for the given prompt lengths, with
the wgmma path and (LSK_PREFILL_TC=0) the decode-kernel path."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from layerskip_b200.engine import Engine
from layerskip_b200.weights import ARCHS, SyntheticLlama

arch = ARCHS[sys.argv[1] if len(sys.argv) > 1 else "llama2-7b"]
lens = [int(x) for x in sys.argv[2:]] or [128, 1024]
eng = Engine(arch, max_ctx=max(lens) + 128)
eng.load_model(SyntheticLlama(arch, seed=0))
g = torch.Generator().manual_seed(1)
for n in lens:
    ids = torch.randint(3, arch.vocab - 1, (n,), generator=g).tolist()
    best = 1e9
    for rep in range(3):
        eng.begin(exit_layer=min(8, arch.layers), max_steps=8, eos_token_ids=[arch.vocab - 1])
        eng.prefill(ids)
        best = min(best, eng.last_device_ms)
    print(f"prefill {n} tokens: {best:.3f} ms (wgmma path: {eng.prefill_tc})", flush=True)
eng.close()

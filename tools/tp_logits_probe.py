"""torchrun --nproc-per-node N tools/tp_logits_probe.py arch [arch ...]
max |logit(TP=N engine) - logit(single-GPU engine)| at the first decode step after a 128-id prompt,
and after a 12-id prompt (decode-kernel prefill instead of the wgmma prefill)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

import bench
from layerskip_b200.synthetic import synthetic_prompts
from layerskip_b200.weights import ARCHS, SyntheticLlama

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
for name in sys.argv[1:]:
    arch = ARCHS[name]
    model = SyntheticLlama(arch, seed=0, device="cuda")
    for n in (128, 12):
        prompt = synthetic_prompts(arch.vocab, 1, n)[0]
        diff, scale = bench.tp_logits_check(model, arch, prompt, [arch.vocab - 1], 768, rank, world)
        if rank == 0:
            print(f"{name} tp={world} prompt={n}: max|dlogit| = {diff:.6f} of max|logit| {scale:.3f}", flush=True)
    del model
    torch.cuda.empty_cache()
dist.destroy_process_group()

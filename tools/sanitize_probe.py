"""Small end-to-end run for compute-sanitizer (memcheck / racecheck): tiny GQA model, a 40-token
prompt (wgmma prefill path) and a 13-token prompt (decode-kernel prefill), greedy and sampled
speculative rounds, autoregressive steps."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from layerskip_b200 import GenerationConfig
from layerskip_b200.strategy import (B200AutoRegressiveGenerationStrategy,
                                     B200SelfSpeculativeGenerationStrategy)
from layerskip_b200.weights import ARCHS, SyntheticLlama

arch = ARCHS[sys.argv[1] if len(sys.argv) > 1 else "tiny-gqa"]
model = SyntheticLlama(arch, seed=0, alpha=0.1, damp_from=3)
spec = B200SelfSpeculativeGenerationStrategy(max_ctx=256)
ar = B200AutoRegressiveGenerationStrategy(engine_cache=spec.engines)
g = torch.Generator().manual_seed(3)
eos = [arch.vocab - 1]
for n_prompt in (40, 13):
    prompt = torch.randint(3, arch.vocab - 1, (n_prompt,), generator=g).tolist()
    a = spec.generate_token_ids(model, prompt, eos, GenerationConfig(max_steps=20, exit_layer=3, num_speculations=6,
                                                                     sample=False)).predicted_tokens
    b = ar.generate_token_ids(model, prompt, eos, GenerationConfig(max_steps=20, exit_layer=-1, num_speculations=-1,
                                                                   sample=False)).predicted_tokens
    assert a == b, (a, b)
    torch.manual_seed(5)
    s = spec.generate_token_ids(model, prompt, eos, GenerationConfig(max_steps=20, exit_layer=3, num_speculations=6,
                                                                     sample=True)).predicted_tokens
    print(f"prompt {n_prompt}: greedy spec == ar ({len(a)} tokens), sampled {len(s)} tokens", flush=True)
spec.engines.close()
print("sanitize probe ok")

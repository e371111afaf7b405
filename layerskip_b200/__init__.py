"""layerskip_b200 — H100-native self-speculative (LayerSkip) decoding engine.

Public surface = the reference's plug-in surface (`plugin`), two drop-in strategies
(`strategy`) and the engine handle (`engine`).  The compute lives in `liblsk.so`
(hand-written sm_90a CUDA behind the C ABI of include/lsk.h); importing the engine without it
fails loudly.
"""
from .plugin import (GenerationConfig, GenerationResult, GenerationStrategy,  # noqa: F401
                     GenerationStrategyResult, HuggingfaceLlamaGenerator)

__all__ = ["GenerationConfig", "GenerationResult", "GenerationStrategy",
           "GenerationStrategyResult", "HuggingfaceLlamaGenerator"]

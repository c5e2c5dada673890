"""starvector_b200 — H100-native image→SVG generation engine behind StarVector's own API.

Importing this package never touches CUDA; the first `Engine(...)` loads
`libstarvector_b200.so` (built by `python -m starvector_b200.build`) and fails loudly if it is
missing or no sm_90 (H100) GPU is visible.  There is no CPU / PyTorch fallback path.
"""
from .config import ModelDims, StarVectorConfig, dims_1b, dims_tiny  # noqa: F401

__all__ = ["ModelDims", "StarVectorConfig", "dims_1b", "dims_tiny", "StarVectorForCausalLM", "Engine", "GenerationParams"]


def __getattr__(name):
    if name in ("StarVectorForCausalLM",):
        from .modeling import StarVectorForCausalLM
        return StarVectorForCausalLM
    if name in ("Engine", "GenerationParams"):
        from . import engine
        return getattr(engine, name)
    raise AttributeError(name)

"""Import the reference's own in-tree modules from a checkout of joanrod/star-vector named by $STARVECTOR_REF.

Only `oracle/make_golden.py` needs it; callers must check `available()` first.
Only the fairscale import (used for grad-checkpointing, clip_model.py:10) needs a shim
(SURVEY.md §8c).  Nothing here copies reference code: it imports it in place.
"""
from __future__ import annotations

import os
import sys
import types

REF_ROOT = os.environ.get("STARVECTOR_REF", "")


def available() -> bool:
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "starvector"))


def load():
    """Returns (VisionTransformer, LayerNorm, Adapter) classes of the reference."""
    if not available():
        raise RuntimeError("set STARVECTOR_REF to a checkout of joanrod/star-vector")
    for n in ("fairscale", "fairscale.nn", "fairscale.nn.checkpoint",
              "fairscale.nn.checkpoint.checkpoint_activations"):
        sys.modules.setdefault(n, types.ModuleType(n))
    sys.modules["fairscale.nn.checkpoint.checkpoint_activations"].checkpoint_wrapper = lambda m, **k: m
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    from starvector.model.image_encoder.clip_model import VisionTransformer, LayerNorm
    from starvector.model.adapters.adapter import Adapter
    return VisionTransformer, LayerNorm, Adapter

"""lungmask_b200 — H100-native drop-in for the hot path of JoHof/lungmask (`LMInferer.apply`)."""
from .mask import LMInferer  # noqa: F401  (lungmask/__init__.py:1 exports exactly this)

__all__ = ["LMInferer"]

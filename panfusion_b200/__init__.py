"""panfusion_b200 — H100-native (sm_90a) denoise hot path of PanFusion behind the reference's interfaces."""
from . import _lib  # noqa: F401

__all__ = ["_lib"]

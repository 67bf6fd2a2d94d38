"""openhevc_b200 — H100 (sm_90a) back end for openHEVC's per-CTU pixel-reconstruction path.

The product is the C-ABI library `libb200hevc.so` (include/b200hevc.h) plus the table shim that
re-populates the reference's HEVCDSPContext / HEVCPredContext (include/b200hevc_tables.h).  This
Python package is a thin host-side mirror used by tests and bench.py: it never computes pixels
itself and has no CPU fallback.
"""
from .engine import FrameEngine, B200Error  # noqa: F401
from .device_output import yuv_to_rgb  # noqa: F401
from . import worklist  # noqa: F401

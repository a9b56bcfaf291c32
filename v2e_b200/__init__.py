"""v2e_b200 -- H100-native (sm_90a) implementation of the two data-parallel hot paths of
SensorsINI/v2e: the DVS pixel model (EventEmulator) and the SuperSloMo frame interpolator.

Import is cheap and GPU-free; the CUDA library (v2e_b200/lib/libv2e_b200.so, C ABI in
include/v2e_b200.h) is loaded on first use and there is no CPU fallback.
"""
from .emulator import EventEmulator  # noqa: F401
from .slomo import SuperSloMo  # noqa: F401
from .pipeline import V2EPipeline  # noqa: F401
from .video import MjpegWriter  # noqa: F401

__all__ = ["EventEmulator", "SuperSloMo", "V2EPipeline", "MjpegWriter"]

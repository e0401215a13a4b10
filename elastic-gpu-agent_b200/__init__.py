"""elastic-gpu-agent_b200 — H100-native best-fit allocation path for elastic-gpu-agent.

Only what the hot path needs: csrc/ (sm_90a kernels + the C ABI of
include/egpu_alloc.h), the ctypes binding, a thin host wrapper and the
synthetic-workload generator.  Import as `elastic_gpu_agent_b200` (the
directory name carries a hyphen; the sibling shim package maps it).
"""
from . import synth  # noqa: F401
from ._lib import (EgpuError, LIB_PATH, VARIANT_AUTO, VARIANT_GRID, VARIANT_SORTED, VARIANT_LUT,  # noqa: F401
                   EV_ALLOC, EV_FREE, EV_RELEASE, load, strerror)
from .alloc import BestFitAllocator  # noqa: F401

__all__ = ["BestFitAllocator", "EgpuError", "synth", "load", "strerror", "LIB_PATH",
           "VARIANT_AUTO", "VARIANT_GRID", "VARIANT_SORTED", "VARIANT_LUT", "EV_ALLOC", "EV_FREE",
           "EV_RELEASE"]

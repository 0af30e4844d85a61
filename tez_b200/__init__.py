"""tez_b200 -- H100-native (sm_90a) implementation of Apache Tez's shuffle sort/merge hot path.

The compute path lives in libtezgpu.so (hand-written CUDA behind the C ABI of include/tezgpu.h).
This package is the host-side mirror used where no JVM exists; it never falls back to CPU code.
"""
from . import _lib  # noqa: F401
from .constants import *  # noqa: F401,F403
from .native import GpuSorter, GpuMerger, PeerBuffer, PeerMapping, debug_total_order, fetch_ranges, fetch_segments_verified  # noqa: F401

__all__ = ["GpuSorter", "GpuMerger", "PeerBuffer", "PeerMapping", "debug_total_order", "fetch_ranges", "fetch_segments_verified"]

"""CPU: host-layer behaviour that needs no device -- configuration validation of OrderedPartitionedKVOutput
(mirrors the argument checks of TestOnFileSortedOutput / ExternalSorter.getInitialMemoryRequirement), the C ABI
exports, and the loud failure without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import tez_b200 as T
from tez_b200 import _lib
from tez_b200.runtime_library import (BYTES_WRITABLE, TEXT, InputContext, OrderedGroupedKVInput,
                                      OrderedPartitionedKVOutput, OutputContext)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(tez(?:gpu|rt)_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = C.CDLL(_lib.LIB_PATH)
    names = _declared("tezgpu.h") + _declared("tez_runtime.h")
    assert len(names) > 40
    for n in names:
        assert hasattr(L, n), "libtezgpu.so does not export %s" % n
    bound = {n for n, _, _ in _lib.SYMBOLS + _lib.RT_SYMBOLS}
    assert set(names) <= bound, "ctypes table misses %s" % (set(names) - bound)
    assert _lib.load().tezgpu_abi_version() == T.ABI_VERSION


def test_io_sort_mb_must_fit_task_memory(tmp_path):
    ctx = OutputContext({"tez.runtime.io.sort.mb": 2048, "tez.runtime.key.class": TEXT}, str(tmp_path),
                        total_memory_available_to_task=1 << 30)
    out = OrderedPartitionedKVOutput(ctx, 4)
    with pytest.raises(IOError, match="should be larger than 0 and should be less than the available task memory"):
        out.initialize()


def test_invalid_sorter_class_and_unsupported_key_class(tmp_path):
    ctx = OutputContext({"tez.runtime.sorter.class": "bogus", "tez.runtime.key.class": TEXT}, str(tmp_path))
    out = OrderedPartitionedKVOutput(ctx, 2)
    assert out.initialize() == []
    assert out.requested_memory == 100 << 20          # tez.runtime.io.sort.mb default
    with pytest.raises(IOError, match="Invalid sorter class specified in config"):
        out.start()
    ctx = OutputContext({"tez.runtime.key.class": "org.example.MyKey"}, str(tmp_path))
    out = OrderedPartitionedKVOutput(ctx, 2)
    out.initialize()
    with pytest.raises(IOError, match="no device comparator"):
        out.start()
    ctx = OutputContext({"tez.runtime.key.class": TEXT, "tez.runtime.compress": True}, str(tmp_path))
    out = OrderedPartitionedKVOutput(ctx, 2)
    out.initialize()
    with pytest.raises(IOError, match="codecs are not supported"):
        out.start()


def test_lifecycle_order_is_enforced(tmp_path):
    out = OrderedPartitionedKVOutput(OutputContext({"tez.runtime.key.class": TEXT}, str(tmp_path)), 2)
    with pytest.raises(IOError, match="before initialize"):
        out.start()
    inp = OrderedGroupedKVInput(InputContext({"tez.runtime.key.class": BYTES_WRITABLE}, str(tmp_path)), 3)
    with pytest.raises(IOError):
        inp.start()
    inp.initialize()
    inp.start()
    with pytest.raises(IOError, match="have not been delivered"):
        inp.waitForInputReady()


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_without_a_device(tmp_path):
    with pytest.raises(IOError, match="no CUDA device"):
        T.GpuSorter(4)
    out = OrderedPartitionedKVOutput(OutputContext({"tez.runtime.key.class": TEXT}, str(tmp_path)), 2)
    out.initialize()
    with pytest.raises(IOError, match="no CUDA device"):
        out.start()
    assert _lib.load().tezgpu_device_count() == 0


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
def test_device_argument_calls_without_a_device():
    """the calls that take a device argument report a missing device as the handle calls do"""
    from tez_b200 import native
    import numpy as np
    calls = [lambda: T.PeerBuffer(16), lambda: T.fetch_ranges([(16, 32, 16)]), lambda: T.fetch_segments_verified([(16, 32, 16)]),
             lambda: native.shuffle_serve(16, np.zeros((1, 3), dtype=np.int64), "m", 0, 1)]
    for call in calls:
        with pytest.raises(_lib.TezGpuError, match="no CUDA device available") as e:
            call()
        assert e.value.code == T.E_CUDA

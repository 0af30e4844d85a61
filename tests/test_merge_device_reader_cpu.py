"""CPU: tezgpu_merge_next_batch_device without a device -- the symbol, the argument check that needs no handle, the
route seeds of the GPU file, and tools/device_reader_bench.py's --help and byte accounting."""
import ctypes as C
import os
import subprocess
import sys

import merge_scenarios as MS
import tez_b200 as T
from tez_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = os.path.join(ROOT, "tools", "device_reader_bench.py")
sys.path.insert(0, os.path.join(ROOT, "tools"))


def test_symbol_resolves_and_a_null_handle_is_refused():
    L = _lib.load()
    assert L.tezgpu_merge_next_batch_device.restype is C.c_int32
    n, b = C.c_uint32(5), C.c_uint64(5)
    assert L.tezgpu_merge_next_batch_device(None, None, 0, None, None, None, None, 16, C.byref(n), C.byref(b)) == T.E_INVALID
    assert (n.value, b.value) == (0, 0)
    assert "null argument" in L.tezgpu_last_error().decode()


def test_route_seeds_cover_every_axis():
    from test_merge_device_reader_gpu import ROUTE_SEEDS
    shapes = [MS.shape(s) for s in ROUTE_SEEDS]
    assert {s["cmp"] for s in shapes} == set(MS.CMP_NAMES)
    assert {s["fixed"] for s in shapes} == {True, False} and {s["check"] for s in shapes} == {True, False}
    assert {s["has_header"] for s in shapes} == {True, False} and {s["P"] for s in shapes} == set(MS.PS)
    assert any(MS.scenario(s)["encoded"] for s in ROUTE_SEEDS if not MS.shape(s)["large"])


def test_bench_help_runs_without_a_device():
    r = subprocess.run([sys.executable, BENCH, "--help"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "--reps" in r.stdout


def test_bench_byte_accounting():
    import device_reader_bench as B
    # a batch moves its key + value bytes twice (read from the segments, written to the batch) plus its table
    assert B.moved_bytes(kv_bytes=1000, records=10, same_key=True) == 2 * 1000 + 10 * (8 + 8 + 4 + 1) + 10 * B.META_READ
    assert B.moved_bytes(kv_bytes=0, records=0, same_key=False) == 0
    assert B.moved_bytes(kv_bytes=64, records=1, same_key=False) == 2 * 64 + 20 + B.META_READ
    assert abs(B.share_of_peak(3.35e12, 1.0) - 1.0) < 1e-12 and abs(B.share_of_peak(3.35e12, 2.0) - 0.5) < 1e-12

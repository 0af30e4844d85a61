"""One process sorts on two devices: kernels that need more than 48 KB of dynamic shared memory (the onesweep radix
passes, k_emit_fast4) get their limit raised on each device they run on, not only on the first."""
import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T

pytestmark = pytest.mark.gpu


def _sort_c2(device, kv, P):
    with T.GpuSorter(P, fixed=(16, 64), device=device) as s:
        s.collect_fixed(kv)
        out, index_bytes, index, st = s.flush_to_memory()
    return bytes(out), index_bytes, index, st


def test_config2_sort_on_device_0_then_device_1():
    if T._lib.load().tezgpu_device_count() < 2:
        pytest.skip("needs two visible CUDA devices")
    n, P = 200000, 64   # config-2 records: 16-byte keys, 64-byte values, 64 partitions (the k_emit_fast4 path)
    kv = O.gen_c2(0, n, seed=7)
    out0, index_bytes0, index0, st0 = _sort_c2(0, kv, P)
    out1, index_bytes1, index1, st1 = _sort_c2(1, kv, P)
    assert out1 == out0, "file.out differs between device 0 and device 1"
    assert index_bytes1 == index_bytes0
    assert np.array_equal(index1, index0)
    assert st1["kernel_launches"] == st0["kernel_launches"]

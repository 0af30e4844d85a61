"""GPU parity for fixed-width records wider than eight 16-byte pieces (strides above 128 bytes).  The software-pipelined
emit kernel for packed, 16-byte aligned records (emit_pipe.cuh) packs a piece's offset in its record into 7 bits and
serves at most eight pieces per record; wider records must take the other source-oriented kernel and still come out
bit-exact, with several tiles per partition.  On the reduce side the records sit at arbitrary offsets of the merged
segments: up to 31 pieces take the pipelined kernel for them (emit_pipe_u.cuh) with its round-filled tiles, wider
records the other source-oriented kernel."""
import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kl,vl,n", [(16, 112, 20011), (16, 128, 20011), (16, 240, 12007), (32, 480, 6001), (16, 4096, 1501)])
def test_wide_aligned_strides_bit_exact(kl, vl, n):
    rng = np.random.default_rng(kl * 10000 + vl)
    P = 3
    kv = rng.integers(0, 256, size=n * (kl + vl), dtype=np.uint8)     # random keys: unique; RLE off (policy 0)
    ko = np.arange(n, dtype=np.uint64) * (kl + vl)
    exp = O.pipelined_sort(O.sorter_conf(P, rle_policy=0), kv, ko, np.full(n, kl, np.uint32), np.full(n, vl, np.uint32))
    with T.GpuSorter(P, fixed=(kl, vl), rle_policy=0) as s:
        s.collect_fixed(kv)
        out, index_bytes, _, _ = s.flush_to_memory()
    assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]


@pytest.mark.parametrize("kl,vl,n", [(16, 480, 6001), (32, 480, 6001), (16, 4096, 1501)])
def test_wide_strides_merge_bit_exact(kl, vl, n):
    """Strides 496 (31 pieces: the pipelined kernel, 40-record tiles), 512 and 4112 (the other kernel)."""
    rng = np.random.default_rng(kl * 10000 + vl + 1)
    segs = []
    for _ in range(2):
        kv = rng.integers(0, 256, size=n * (kl + vl), dtype=np.uint8)  # random keys: unique, so no record is a repeat
        segs.append(O.pipelined_sort_fixed(O.sorter_conf(1, rle_policy=0), kv, kl, vl)["file_out"])
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, fixed=(kl, vl)) as m:
        seg, _, _, _ = m.write_ifile(rle=False)
    assert seg == exp["ifile"]

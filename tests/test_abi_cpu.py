"""CPU: checks of libtezgpu that need no device -- the GF(2) algebra of the tiled, parallel CRC32 (host emulation on
the same tables the kernels use) against zlib."""
import random
import zlib

from tez_b200 import _lib


def test_tiled_crc_algebra_matches_zlib():
    L = _lib.load()
    rng = random.Random(1)
    for n in [0, 1, 3, 4, 5, 15, 16, 17, 63, 64, 1000, 1027, 4096 * 3 + 5, 24 * 1024 - 7, 24 * 1024 + 9, 100000, 1 << 20]:
        d = bytes(rng.getrandbits(8) for _ in range(n))
        for piece in (64, 1040, 24 * 1024):
            for lead in (0, 1, 7, 12, 15):
                assert L.tezgpu_debug_crc_emulate(d, n, piece, lead) == zlib.crc32(d), (n, piece, lead)


def test_chunk_fold_two_deep_form_matches_zlib():
    """crc32.cuh CrcChunkFold: the two-maps-deep chunk update (and the x^(-128*(T-1)) correction it needs, which rests
    on x having order 2^32-1 modulo the CRC-32 polynomial) gives the same remainder as the textbook chain and as zlib."""
    L = _lib.load()
    rng = random.Random(7)
    for nchunks in [1, 2, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1000, 1290, 2048, 5000]:
        d = bytes(rng.getrandbits(8) for _ in range(16 * nchunks))
        raw = zlib.crc32(d) ^ zlib.crc32(bytes(16 * nchunks))       # linear part: init 0, no final xor
        assert L.tezgpu_debug_chunk_fold_emulate(d, nchunks, 0) == raw, nchunks
        assert L.tezgpu_debug_chunk_fold_emulate(d, nchunks, 1) == raw, nchunks


def test_segment_table_fast_path_matches_ctypes_layout():
    """GpuMerger builds the tezgpu_segment table through numpy when there are many device-resident runs; the bytes must
    equal what the ctypes structure assignment produces (include/tezgpu.h: data, len, flags, partition)."""
    import ctypes as C
    import numpy as np
    from tez_b200 import native
    from tez_b200._lib import Segment
    rng = np.random.default_rng(1)
    n = 200
    segs = [(int(a), int(b)) for a, b in zip(rng.integers(1 << 33, 1 << 47, n), rng.integers(10, 1 << 30, n))]
    parts = [int(p) for p in rng.integers(0, 128, n)]
    m = object.__new__(native.GpuMerger)          # no device needed: only the table builder is exercised
    m._has_header, m._device_ptrs, m.h = True, True, None
    fast = m._segments(segs, parts)
    fast_bytes = C.string_at(fast, n * C.sizeof(Segment))
    slow = (Segment * n)()
    for i, (p, ln) in enumerate(segs):
        slow[i].data, slow[i].len = p, ln
        slow[i].flags = native.SEG_HAS_HEADER | native.SEG_DEVICE
        slow[i].partition = parts[i]
    assert C.sizeof(Segment) == 24
    assert fast_bytes == bytes(slow)
    few = m._segments(segs[:3], parts[:3])        # the ctypes path (<= 64 runs)
    assert bytes(few)[:3 * 24] == bytes(slow)[:3 * 24]


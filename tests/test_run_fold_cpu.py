"""CPU: the run-organised CRC32 of the packed fixed-width emit kernel (emit_pipe.cuh k_emit_fast4), emulated on the
host with the kernel's tables and constants, against zlib."""
import random
import zlib

from tez_b200 import _lib


def test_run_fold_matches_zlib():
    """Per-thread runs of five 16-byte chunks anchored at the tile end, W on lane-private digit tables, second level by
    Horner with x^(8*80*32) and the per-lane x^(8*80*(31-l)): zlib's remainder for every chunk count a tile image can
    hold (1..1280), whole rounds and ragged ones."""
    L = _lib.load()
    rng = random.Random(11)
    buf = bytes(rng.getrandbits(8) for _ in range(16 * 1280))
    for nchunks in range(1, 1281):
        d = buf[:16 * nchunks]
        raw = zlib.crc32(d) ^ zlib.crc32(bytes(16 * nchunks))       # linear part: init 0, no final xor
        assert L.tezgpu_debug_run_fold_emulate(d, nchunks) == raw, nchunks

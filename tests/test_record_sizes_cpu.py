"""CPU: the fixed-width emit plan (sorter.cuh plan_fixed_emit, through tezgpu_debug_fixed_emit_plan) over every 16-byte
stride up to 2 MiB and every record layout.  The source-oriented emit kernels build a whole tile in one shared-memory
image and never cut it, so the plan must give each of them only tiles that fit that image with the worst-case lead (15
bytes), the segment header (4) and the EOF marker (2); records too large for that take k_emit<true>, which writes a tile
in pieces.  Every stride whose tiles already fitted keeps the kernel and tile size it had before records too large for
the image were sent to k_emit<true> (restated below as `plan_before`), so config 2 (16 + 64 bytes, packed) and every
other existing path keep their kernel."""
import ctypes as C

import pytest

from tez_b200 import _lib

PIPE, FAST, PIPE_U, FAST_U, GENERAL = range(5)
PACKED, OFFSETS, RUNS = range(3)
FE_IMG_BYTES = 22016    # emit_fast.cuh: the image of k_emit_fast and k_emit_fast4u
FE4_IMG_BYTES = 20480   # emit_pipe.cuh: the image of k_emit_fast4
IMAGE = {PIPE: FE4_IMG_BYTES, FAST: FE_IMG_BYTES, PIPE_U: FE_IMG_BYTES, FAST_U: FE_IMG_BYTES}
TILE_EXTRA = 15 + 4 + 2  # worst-case lead, segment header, EOF marker
MAX_STRIDE = 2 << 20


def vint_size(v):
    """WritableUtils.getVIntSize of a non-negative length"""
    return 1 if v <= 127 else 2 if v < 1 << 8 else 3 if v < 1 << 16 else 4 if v < 1 << 24 else 5


def rec_size(klen, vlen):
    return vint_size(klen) + vint_size(vlen) + klen + vlen


def plan_before(klen, vlen, layout):
    """(kernel, records per tile) the plan chose before oversized records were sent to k_emit<true>"""
    stride, rs = klen + vlen, rec_size(klen, vlen)
    cpr = stride // 16
    cap = max(1, min(256, (FE_IMG_BYTES - 32) // rs))
    if stride < 16 or stride % 16:
        return GENERAL, cap
    if layout == PACKED:
        m = min(256, (FE4_IMG_BYTES - TILE_EXTRA) // rs)
        if cpr <= 8 and m * cpr <= 5 * 256:
            return PIPE, min(cap, m)
        return FAST, cap
    w = cpr + 1
    m = 0 if w > 32 else 5 * 8 * (32 // w)
    if m == 0:
        return FAST_U, cap
    top = min(cap, m)
    best, best_eff = top, 0.0
    for r in range(top, top - top // 10 - 1, -1):
        chunks = (r * rs + TILE_EXTRA + 15) // 16
        rounds = (chunks + 255) // 256
        if r / rounds > best_eff:
            best, best_eff = r, r / rounds
    return PIPE_U, best


def plan(klen, vlen, layout):
    L = _lib.load()
    k, r = C.c_int32(), C.c_uint32()
    _lib.check(L.tezgpu_debug_fixed_emit_plan(klen, vlen, layout, C.byref(k), C.byref(r)))
    return k.value, r.value


def fits(kernel, recs, rs):
    return kernel == GENERAL or recs * rs + TILE_EXTRA <= IMAGE[kernel]


def _check(klen, vlen, layout):
    rs = rec_size(klen, vlen)
    kernel, recs = plan(klen, vlen, layout)
    assert 1 <= recs <= 256, (klen, vlen, layout, recs)
    assert fits(kernel, recs, rs), "stride %d + %d, layout %d: %d records of %d bytes overflow kernel %d's image" % (
        klen, vlen, layout, recs, rs, kernel)
    before = plan_before(klen, vlen, layout)
    if fits(before[0], before[1], rs):
        assert (kernel, recs) == before, (klen, vlen, layout)
    else:
        assert kernel == GENERAL, (klen, vlen, layout)
    return kernel, recs


@pytest.mark.parametrize("layout", [PACKED, OFFSETS, RUNS])
def test_every_stride_fits_its_kernel_image(layout):
    """16-byte keys and every 16-byte stride up to 2 MiB: 1- to 4-byte value vints, framings of 2 to 5 bytes"""
    kernels = set()
    for stride in range(16, MAX_STRIDE + 1, 16):
        kernels.add(_check(16, stride - 16, layout)[0])
    assert GENERAL in kernels and len(kernels) >= 2


@pytest.mark.parametrize("layout", [PACKED, OFFSETS, RUNS])
def test_large_keys_and_five_byte_framings(layout):
    """keys of every vint width, values past 2^24 (framings up to 10 bytes), strides that are not a multiple of 16"""
    for klen in (1, 16, 127, 128, 255, 256, 4096, 65535, 65536, (1 << 24) + 16):
        for vlen in (0, 15, 16, 64, 21952, 21968, 65536, (1 << 24) - 1, 1 << 24, (1 << 24) + 16):
            _check(klen, vlen, layout)


def test_strides_around_the_image_edge():
    """The last stride every source-oriented kernel took before its image overflowed, and the first one past it.
    rec_size = stride + 4 (vint(16), vint(vlen) of 3 bytes): 21984 + 4 + 21 <= 22016 < 22000 + 4 + 21."""
    for layout in (PACKED, OFFSETS, RUNS):
        k, r = plan(16, 21984 - 16, layout)
        assert k in (FAST, FAST_U) and r == 1, (layout, k, r)
        assert plan(16, 22000 - 16, layout) == (GENERAL, 1), layout
        for stride in (32768, 65552, (1 << 20) + 16):
            assert plan(16, stride - 16, layout) == (GENERAL, 1), (layout, stride)


def test_config_2_and_reduce_side_paths_keep_their_kernels():
    assert plan(16, 64, PACKED) == (PIPE, 249)
    assert plan(16, 64, RUNS)[0] == PIPE_U and plan(16, 64, OFFSETS)[0] == PIPE_U
    assert plan(16, 4096, PACKED)[0] == FAST
    assert plan(16, 4096, RUNS)[0] == FAST_U
    assert plan(10, 71, PACKED)[0] == GENERAL


def test_plan_argument_checks():
    L = _lib.load()
    k, r = C.c_int32(), C.c_uint32()
    assert L.tezgpu_debug_fixed_emit_plan(16, 64, 3, C.byref(k), C.byref(r)) == -1
    assert L.tezgpu_debug_fixed_emit_plan(0, 0, 0, C.byref(k), C.byref(r)) == -1
    assert L.tezgpu_debug_fixed_emit_plan(16, 64, 0, None, C.byref(r)) == -1

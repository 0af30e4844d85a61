"""Bounded-memory merge (tezgpu_merge_open_bounded) without a device: symbols, argument checks, no CPU fallback."""
import ctypes as C

import pytest

import tez_b200 as T
from tez_b200 import _lib
from tez_b200.native import make_conf
from oracle import tez_oracle as O

E_INVALID, E_CUDA, E_UNSUPPORTED = -1, -2, -6


def _open(segs, budget, codec=0, flags=T.SEG_HAS_HEADER, conf=True):
    L = _lib.load()
    keep = [bytes(s) for s in segs]
    arr = (_lib.Segment * max(1, len(keep)))()
    for i, s in enumerate(keep):
        arr[i].data = C.cast(C.c_char_p(s), C.c_void_p)
        arr[i].len = len(s)
        arr[i].flags = flags
        arr[i].partition = 0
    cf = make_conf(1, comparator=T.CMP_BYTES, partitioner=T.PART_GIVEN)
    h = C.c_void_p()
    rc = L.tezgpu_merge_open_bounded(C.byref(cf) if conf else None, arr, None, len(keep), codec, budget, C.byref(h))
    if rc == 0:
        L.tezgpu_merge_close(h)
    return rc, L.tezgpu_last_error().decode()


def test_bounded_merge_symbols_resolve():
    L = _lib.load()
    for name in ("tezgpu_merge_open_bounded", "tezgpu_merge_bounded_info"):
        assert getattr(L, name) is not None


def test_bounded_merge_argument_checks():
    seg = O.write_ifile([(b"a", b"1"), (b"b", b"2")])[0]
    assert _open([seg], 1 << 30, conf=False)[0] == E_INVALID
    rc, msg = _open([seg], (16 << 20) - 1)
    assert rc == E_INVALID and "below the floor" in msg
    rc, msg = _open([seg], 1 << 30, flags=T.SEG_HAS_HEADER | T.SEG_DEVICE)
    assert rc == E_INVALID and "host segments only" in msg
    rc, msg = _open([seg], 1 << 30, codec=T.CODEC_DEFAULT)
    assert rc == E_UNSUPPORTED and "uncompressed" in msg
    L = _lib.load()
    steps = C.c_int32()
    assert L.tezgpu_merge_bounded_info(None, C.byref(steps), None, None) == E_INVALID


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
def test_bounded_merge_has_no_cpu_fallback():
    seg = O.write_ifile([(b"a", b"1"), (b"b", b"2")])[0]
    for budget in (0, 16 << 20, 1 << 30):
        assert _open([seg, seg], budget)[0] == E_CUDA
    with pytest.raises(IOError):
        T.GpuMerger([seg], comparator=T.CMP_BYTES, device_budget=0)

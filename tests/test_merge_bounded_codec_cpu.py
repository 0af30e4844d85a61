"""Bounded merge with compressed output (tezgpu_merge_open_bounded_write_codec) without a device: the symbols, the
argument checks that come before any device call, no CPU fallback, and the piecewise compression of a partition body
across steps (tezgpu_debug_stitched_compress_emulate) against the codec's stream of the uncut body at every chunk-grid
edge."""
import ctypes as C
import random

import pytest

import tez_b200 as T
from tez_b200 import _lib, native
from tez_b200.native import make_conf
from oracle import tez_oracle as O

E_INVALID, E_CUDA, E_UNSUPPORTED = -1, -2, -6
CODECS = {"default": T.CODEC_DEFAULT, "lz4": T.CODEC_LZ4, "zstd": T.CODEC_ZSTD, "snappy": T.CODEC_SNAPPY}
CHUNK = {T.CODEC_DEFAULT: 32768, T.CODEC_LZ4: T.LZ4_BLOCK_BYTES, T.CODEC_ZSTD: T.ZSTD_BLOCK_BYTES,
         T.CODEC_SNAPPY: T.SNAPPY_BLOCK_BYTES}
UNCUT = {T.CODEC_DEFAULT: "tezgpu_debug_deflate_emulate", T.CODEC_LZ4: "tezgpu_debug_lz4_compress_emulate",
         T.CODEC_ZSTD: "tezgpu_debug_zstd_compress_emulate", T.CODEC_SNAPPY: "tezgpu_debug_snappy_compress_emulate"}


def _open(segs, budget, codec, flags=T.SEG_HAS_HEADER, conf=True):
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
    rc = L.tezgpu_merge_open_bounded_write_codec(C.byref(cf) if conf else None, arr, len(keep), codec, budget, C.byref(h))
    if rc == 0:
        L.tezgpu_merge_close(h)
    return rc, L.tezgpu_last_error().decode()


def _uncut(codec, body):
    L = _lib.load()
    cap = len(body) + len(body) // 255 + 16 * (len(body) // 32768 + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    _lib.check(getattr(L, UNCUT[codec])(bytes(body), len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def test_symbols_resolve():
    L = _lib.load()
    for name in ("tezgpu_merge_open_bounded_write_codec", "tezgpu_debug_stitched_compress_emulate"):
        assert getattr(L, name) is not None


@pytest.mark.parametrize("codec", list(CODECS.values()) + [T.CODEC_NONE])
def test_argument_checks_before_any_device_call(codec):
    seg = O.write_ifile([(b"a", b"1"), (b"b", b"2")])[0]
    assert _open([seg], 1 << 30, codec, conf=False)[0] == E_INVALID
    rc, msg = _open([seg], (16 << 20) - 1, codec)
    assert rc == E_INVALID and "below the floor" in msg
    rc, msg = _open([seg], 1 << 30, codec, flags=T.SEG_HAS_HEADER | T.SEG_DEVICE)
    assert rc == E_INVALID and "host segments only" in msg


@pytest.mark.parametrize("codec", [5, 99, -1])
def test_unknown_codec_is_named(codec):
    seg = O.write_ifile([(b"a", b"1")])[0]
    rc, msg = _open([seg], 1 << 30, codec)
    assert rc == E_UNSUPPORTED and msg.startswith("codec %d is not on the device" % codec)


def test_write_codec_needs_a_budget():
    with pytest.raises(ValueError, match="device_budget"):
        T.GpuMerger([O.write_ifile([(b"a", b"1")])[0]], write_codec=T.CODEC_LZ4)


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
@pytest.mark.parametrize("codec", list(CODECS.values()))
def test_no_cpu_fallback(codec):
    seg = O.write_ifile([(b"a", b"1"), (b"b", b"2")])[0]
    for budget in (0, 16 << 20, 1 << 30):
        assert _open([seg, seg], budget, codec)[0] == E_CUDA
    with pytest.raises(IOError):
        T.GpuMerger([seg], comparator=T.CMP_BYTES, device_budget=0, write_codec=codec)


def _body(n, seed):
    """record-like bytes: repeated words (long matches) and noise, ending in the EOF markers"""
    rng = random.Random(seed)
    words = [bytes(rng.getrandbits(8) for _ in range(rng.randint(3, 12))) for _ in range(300)]
    out = bytearray()
    while len(out) < n - 2:
        out += rng.choice(words) if rng.random() < 0.8 else bytes([rng.getrandbits(8)])
    return bytes(out[:max(0, n - 2)]) + b"\xff\xff"


def _cases(chunk):
    """(name, body, cuts) at the edges of the chunk grid"""
    rng = random.Random(chunk)
    n = 4 * chunk + 777
    b = _body(n, chunk)
    yield "random", b, sorted(rng.randrange(n + 1) for _ in range(9))
    yield "on_chunk_multiples", b, [chunk, 2 * chunk, 4 * chunk]
    yield "byte_before", b, [chunk - 1, 2 * chunk - 1, 3 * chunk - 1]
    yield "byte_after", b, [chunk + 1, 2 * chunk + 1, 3 * chunk + 1]
    yield "before_and_after", b, [chunk - 1, chunk + 1, 3 * chunk - 1, 3 * chunk + 1]
    # pieces shorter than a chunk: the carry grows over several cuts before a chunk fills
    short, at = [], 0
    while at < n - 1000:
        at += rng.randint(1, chunk // 7)
        short.append(min(at, n))
    yield "short_pieces_carry", b, short
    yield "empty_pieces", b, [0, 0, 5, 5, chunk, chunk, n, n]
    for k in (1, 2, 3):
        bk = _body(k * chunk, k)
        yield "exactly_%d_chunks" % k, bk, [chunk // 2, k * chunk - 2]
        yield "exactly_%d_chunks_cut_on_grid" % k, bk, [k * chunk - chunk, k * chunk]
    yield "empty_body", b"\xff\xff", [0, 1, 2]
    yield "empty_body_uncut", b"\xff\xff", []
    yield "one_chunk_and_eof", _body(chunk + 2, 7), [chunk]


@pytest.mark.parametrize("name", list(CODECS))
def test_stitched_emulation_equals_the_uncut_stream(name):
    codec = CODECS[name]
    for case, body, cuts in _cases(CHUNK[codec]):
        assert native.debug_stitched_compress(codec, body, cuts) == _uncut(codec, body), (name, case)


def test_stitched_emulation_random_bodies_and_cuts():
    rng = random.Random(4)
    for i in range(12):
        codec = list(CODECS.values())[i % 4]
        body = _body(rng.randint(2, 3 * CHUNK[codec]), 100 + i)
        cuts = sorted(rng.randrange(len(body) + 1) for _ in range(rng.randint(0, 12)))
        assert native.debug_stitched_compress(codec, body, cuts) == _uncut(codec, body), (codec, len(body), cuts)


def test_stitched_emulation_argument_checks():
    L = _lib.load()
    out = (C.c_uint8 * 64)()
    n = C.c_uint64()
    cuts = (C.c_uint64 * 2)(5, 3)
    assert L.tezgpu_debug_stitched_compress_emulate(T.CODEC_LZ4, b"abcdefgh", 8, cuts, 2, out, 64, C.byref(n)) == E_INVALID
    assert "non-decreasing" in L.tezgpu_last_error().decode()
    assert L.tezgpu_debug_stitched_compress_emulate(7, b"ab", 2, None, 0, out, 64, C.byref(n)) == E_UNSUPPORTED
    assert L.tezgpu_debug_stitched_compress_emulate(T.CODEC_NONE, b"ab", 2, None, 0, out, 64, C.byref(n)) == E_INVALID

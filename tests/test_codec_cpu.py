"""DefaultCodec on the CPU: the device writer and reader run through their host emulations (same __host__ __device__
code) and are checked against the system zlib, an independent implementation of RFC 1950/1951."""
import os
import random
import zlib

import numpy as np
import pytest

import tez_b200 as T
from tez_b200.runtime_library import TEXT, OrderedPartitionedKVOutput, OutputContext
from tez_b200._lib import TezGpuError
import codec_model as M

C = M.CHUNK


def _bound(n):
    return n + 5 * (n // C + 1) + 6


def _roundtrip(body):
    z = M.deflate_emulate(body)
    assert z[:2] == b"\x78\x01"
    assert zlib.decompress(z) == body
    assert M.inflate_emulate(z, len(body)) == body
    assert len(z) <= _bound(len(body))
    return z


# ------------------------------------------------------------------------------------------------ writer
@pytest.mark.parametrize("n", [0, 2, 1, 100, C - 1, C, C + 1, 3 * C + 7, 5 * C])
def test_writer_round_trip_lengths(n):
    rng = random.Random(n)
    body = bytes(rng.choice(b"abcdefgh\xff\x00") for _ in range(n))
    _roundtrip(body)


def test_writer_eof_marker_body():
    z = _roundtrip(b"\xff\xff")
    assert len(z) < 16


@pytest.mark.parametrize("n", [C - 1, C, 4 * C + 3])
def test_writer_random_bytes_take_the_stored_path(n):
    body = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
    z = _roundtrip(body)
    assert len(z) <= _bound(n)
    assert len(z) >= n       # incompressible: stored chunks


@pytest.mark.parametrize("b", [0, 0xFF, 0x41])
def test_writer_long_runs(b):
    body = bytes([b]) * (3 * C + 1000) + b"xyz" + bytes([b]) * 5000
    z = _roundtrip(body)
    assert len(z) < len(body) // 50


def test_writer_is_deterministic_and_chunks_are_byte_aligned_flush_points():
    body = M.wordcount_body(n=50000)
    z1, z2 = M.deflate_emulate(body), M.deflate_emulate(body)
    assert z1 == z2
    # every chunk but the last ends with the empty stored block of a sync flush (or is a stored block itself)
    d = zlib.decompressobj()
    assert d.decompress(z1) == body and d.eof


@pytest.mark.parametrize("name", ["wordcount", "c3", "int_long"])
def test_writer_ratio_against_zlib_level_1(name):
    body = {"wordcount": M.wordcount_body, "c3": M.c3_body, "int_long": M.int_long_body}[name]()
    z = _roundtrip(body)
    ref = len(zlib.compress(body, 1))
    assert len(z) <= 1.25 * ref, (len(z), ref)


# ------------------------------------------------------------------------------------------------ reader vs zlib
STRATEGIES = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FILTERED]


@pytest.mark.parametrize("strategy", STRATEGIES)
@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_reader_zlib_levels_and_strategies(level, strategy):
    body = M.wordcount_body(n=20000) + os.urandom(3000) + M.int_long_body(n=5000)
    seg, raw = M.compressed_segment(body, level, strategy)
    assert M.inflate_emulate(seg[4:-4], raw - 4) == body


@pytest.mark.parametrize("mode", [zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH])
def test_reader_flush_points_and_small_windows(mode):
    body = M.wordcount_body(n=20000)
    for wbits in (9, 12, 15):
        c = zlib.compressobj(6, zlib.DEFLATED, wbits)
        z = b"".join(c.compress(body[a:a + 7000]) + c.flush(mode) for a in range(0, len(body), 7000)) + c.flush()
        assert M.inflate_emulate(z, len(body)) == body


@pytest.mark.parametrize("members", [2, 3, 7])
def test_reader_several_members_in_one_body(members):
    body = M.wordcount_body(n=30000)
    seg, raw = M.compressed_segment(body, 6, members=members)
    assert M.hadoop_inflate(seg[4:-4]) == body
    assert M.inflate_emulate(seg[4:-4], raw - 4) == body


def test_reader_fixture_segments():
    for seg, raw in M.fixture():
        out = M.inflate_emulate(seg[4:-4], raw - 4)
        assert len(out) == raw - 4
        assert out == zlib.decompress(seg[4:-4])


# ------------------------------------------------------------------------------------------------ malformed streams
@pytest.mark.parametrize("case", sorted(M.malformed()[0]))
def test_reader_malformed_streams_fail_with_format_error(case):
    cases, n = M.malformed()
    z = cases[case]
    with pytest.raises(Exception):
        M.hadoop_inflate(z)
    with pytest.raises(TezGpuError) as e:
        M.inflate_emulate(z, n)
    assert e.value.code == T.E_FORMAT
    assert "segment 0" in str(e.value)


@pytest.mark.parametrize("delta", [-1, 1, 100])
def test_reader_wrong_body_length_fails(delta):
    body = b"hello hello hello hello"
    z = zlib.compress(body)
    with pytest.raises(TezGpuError) as e:
        M.inflate_emulate(z, len(body) + delta)
    assert e.value.code == T.E_FORMAT


def test_reader_bit_flip_fuzz_agrees_with_zlib():
    """Seeded single- and multi-bit flips of zlib and device-writer streams: the emulator and hadoop_inflate both fail, or
    both return the same bytes."""
    rng = random.Random(1234)
    bodies = [M.wordcount_body(n=400, vocab=50, seed=s) for s in range(4)] + [bytes(rng.getrandbits(8) for _ in range(300))]
    streams = []
    for b in bodies:
        for level, strat in [(1, zlib.Z_DEFAULT_STRATEGY), (9, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_FIXED), (0, 0)]:
            c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strat)
            streams.append((b, c.compress(b) + c.flush()))
        streams.append((b, M.deflate_emulate(b)))
        streams.append((b + b, zlib.compress(b, 6) + zlib.compress(b, 1)))
    agree = fails = 0
    for i in range(3000):
        body, z = streams[i % len(streams)]
        zz = bytearray(z)
        for _ in range(1 + (i % 3 == 0)):
            bit = rng.randrange(len(zz) * 8)
            zz[bit // 8] ^= 1 << (bit % 8)
        zz = bytes(zz)
        try:
            ref = M.hadoop_inflate(zz)
            if len(ref) != len(body):
                ref = None
        except zlib.error:
            ref = None
        try:
            got = M.inflate_emulate(zz, len(body))
        except TezGpuError as e:
            assert e.code == T.E_FORMAT
            got = None
        assert got == ref, (i, ref is None, got is None)
        agree += 1
        fails += got is None
    assert agree == 3000 and 0 < fails < 3000


# ------------------------------------------------------------------------------------------------ plugin configuration
@pytest.mark.parametrize("codec", ["org.apache.hadoop.io.compress.GzipCodec", "org.apache.hadoop.io.compress.SnappyCodec",
                                   "org.apache.hadoop.io.compress.BZip2Codec"])
def test_plugin_refuses_other_codecs_by_name(tmp_path, codec):
    """Checked before any device call: the class is named in the refusal."""
    ctx = OutputContext({"tez.runtime.key.class": TEXT, "tez.runtime.compress": True, "tez.runtime.compress.codec": codec},
                        str(tmp_path))
    out = OrderedPartitionedKVOutput(ctx, 2)
    out.initialize()
    with pytest.raises(IOError, match=codec.replace(".", r"\.")) as e:
        out.start()
    assert e.value.code == T.E_UNSUPPORTED


def test_plugin_compress_without_a_codec_class_is_still_refused(tmp_path):
    ctx = OutputContext({"tez.runtime.key.class": TEXT, "tez.runtime.compress": True}, str(tmp_path))
    out = OrderedPartitionedKVOutput(ctx, 2)
    out.initialize()
    with pytest.raises(IOError, match="codecs are not supported"):
        out.start()

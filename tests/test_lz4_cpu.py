"""Lz4Codec on the CPU: the device writer and reader run through their host emulations (same __host__ __device__
code) and are checked against a Python restatement of the strict reader (lz4_model) and, where it can be loaded, the
system liblz4."""
import random

import numpy as np
import pytest

import tez_b200 as T
from tez_b200.runtime_library import TEXT, OrderedGroupedKVInput, OrderedPartitionedKVOutput, InputContext, OutputContext
from tez_b200._lib import TezGpuError
import codec_model as CM
import lz4_model as M

B = M.LZ4_BLOCK_BYTES
needs_liblz4 = pytest.mark.skipif(M.liblz4() is None, reason="liblz4 cannot be loaded")


def _check_written(body, z):
    """a device-writer stream: decodes through both readers, blocks within the writer's limits"""
    assert M.decode_stream(z, len(body)) == body
    assert M.decompress_emulate(z, len(body)) == body
    bl = M.blocks(z)
    assert len(bl) == -(-len(body) // B)
    for i, (raw, chunks) in enumerate(bl):
        assert len(chunks) == 1 and raw == (B if i + 1 < len(bl) else len(body) - B * i)
        assert len(chunks[0]) <= M.LZ4_CHUNK_BOUND
        _check_chunk_rules(chunks[0], raw)
        if M.liblz4():
            assert M.lz4_decompress_safe(chunks[0]) == M.decode_chunk(chunks[0])


def _sequences(chunk):
    """(literal start, literal length, match start, offset, match length) of every sequence of a chunk"""
    ip, op, seqs = 0, 0, []
    while True:
        tok = chunk[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                s = chunk[ip]; ip += 1; lit += s
                if s != 255:
                    break
        ip += lit
        if ip == len(chunk):
            seqs.append((op, lit, None, None, None))
            return seqs
        off = chunk[ip] | chunk[ip + 1] << 8
        ip += 2
        m = tok & 15
        if m == 15:
            while True:
                s = chunk[ip]; ip += 1; m += s
                if s != 255:
                    break
        seqs.append((op, lit, op + lit, off, m + 4))
        op += lit + m + 4


def _check_chunk_rules(chunk, raw):
    """offsets < 65536; the last 5 bytes are literals; no match starts within the last 12 bytes"""
    for _, _, ms, off, ml in _sequences(chunk):
        if ms is None:
            continue
        assert 0 < off < 65536
        assert ms + 12 <= raw and ms + ml + 5 <= raw


# ------------------------------------------------------------------------------------------------ writer
@pytest.mark.parametrize("n", [1, 2, 4, 5, 11, 12, 13, 17, 100, B - 13, B - 12, B - 5, B - 1, B, B + 1, B + 5, B + 12,
                               B + 13, 3 * B + 7, 4 * B])
def test_writer_round_trip_sizes_and_tail_rules(n):
    rng = random.Random(n)
    body = bytes(rng.choice(b"abab\xff\x00") for _ in range(n))
    _check_written(body, M.compress_emulate(body))


@pytest.mark.parametrize("n", [B - 1, B, 3 * B + 11])
def test_writer_random_bytes_within_the_bound(n):
    body = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
    z = M.compress_emulate(body)
    _check_written(body, z)
    assert len(z) <= n + n // 255 + 10 * (n // B + 1)


@pytest.mark.parametrize("b", [0, 0xFF, 0x41])
def test_writer_long_runs(b):
    body = bytes([b]) * (3 * B + 1000) + b"xyz" + bytes([b]) * 5000
    z = M.compress_emulate(body)
    _check_written(body, z)
    assert len(z) < len(body) // 50


def test_writer_empty_body_is_an_empty_stream_and_eof_marker_one_block():
    assert M.compress_emulate(b"") == b""
    z = M.compress_emulate(b"\xff\xff")
    assert z == (2).to_bytes(4, "big") + (3).to_bytes(4, "big") + b"\x20\xff\xff"
    _check_written(b"\xff\xff", z)


def test_writer_is_deterministic():
    body = CM.wordcount_body(n=50000)
    assert M.compress_emulate(body) == M.compress_emulate(body)


@needs_liblz4
@pytest.mark.parametrize("name", ["wordcount", "c3", "int_long"])
def test_writer_ratio_against_liblz4_default(name):
    body = {"wordcount": CM.wordcount_body, "c3": CM.c3_body, "int_long": CM.int_long_body}[name]()
    z = M.compress_emulate(body)
    _check_written(body, z)
    ref = sum(len(M.lz4_compress(body[a:a + M.MAX_INPUT])) for a in range(0, len(body), M.MAX_INPUT))
    assert len(z) <= 1.25 * ref, (len(z), ref)


# ------------------------------------------------------------------------------------------------ reader
@needs_liblz4
def test_model_agrees_with_liblz4_on_the_fixture_chunks():
    n = 0
    for name, seg, raw in M.fixture():
        for _, chunks in M.blocks(seg[4:-4]):
            for c in chunks:
                assert M.decode_chunk(c) == M.lz4_decompress_safe(c), name
                n += 1
    assert n >= 8


@needs_liblz4
@pytest.mark.parametrize("mode,accel", [("fast", 1), ("fast", 8), ("fast", 65537), ("hc", 0)])
def test_model_agrees_with_liblz4_made_blocks(mode, accel):
    rng = random.Random(accel)
    bodies = [CM.wordcount_body(n=20000, seed=3), CM.int_long_body(n=20000), bytes(rng.getrandbits(8) for _ in range(5000)),
              b"a", b"abcdefghijkl", bytes(70000), b"xy" * 131072]
    for body in bodies:
        body = body[:M.MAX_INPUT]          # what one Java chunk holds
        c = M.lz4_compress(body, mode=mode, accel=accel)
        assert M.decode_chunk(c) == M.lz4_decompress_safe(c) == body


@needs_liblz4
def test_offset_zero_is_refused_although_liblz4_may_accept_it():
    """liblz4 1.9 takes offset 0 on one code path (copying bytes of its own output buffer that were never written) and
    refuses it on another; the strict reader refuses it always."""
    short = bytes([0x40]) + b"abcd" + b"\x00\x00" + bytes([0x50]) + b"xxxxx"
    longer = bytes([0x80]) + b"abcdefgh" + b"\x00\x00" + bytes([0x50]) + b"x" * 25
    assert M.lz4_decompress_safe(longer) is None
    for c in (short, longer):
        with pytest.raises(M.Lz4FormatError):
            M.decode_chunk(c)


def test_emulated_reader_decodes_the_fixture():
    for name, seg, raw in M.fixture():
        assert seg[:4] == b"TIF\x01"
        body = M.decode_stream(seg[4:-4], raw - 4)
        assert M.decompress_emulate(seg[4:-4], raw - 4) == body, name
    multi = [len(ch) for name, seg, _ in M.fixture() for _, ch in M.blocks(seg[4:-4])]
    assert max(multi) >= 3   # the long value's block


@pytest.mark.parametrize("case", sorted(M.malformed()))
def test_malformed_streams_fail_with_format_error(case):
    z, n = M.malformed()[case]
    with pytest.raises(M.Lz4FormatError):
        M.decode_stream(z, n)
    with pytest.raises(TezGpuError) as e:
        M.decompress_emulate(z, n)
    assert e.value.code == T.E_FORMAT
    assert "segment 0" in str(e.value)


def test_multi_chunk_block_decodes_on_the_exact_path():
    a, b = b"0123456789" * 3, b"abcdefghij" * 2
    z = M.blk(50, M.lit(a), M.lit(b)) + M.blk(3, M.lit(b"end"))
    assert M.decode_stream(z, 53) == a + b + b"end" == M.decompress_emulate(z, 53)


def test_bit_flip_fuzz_emulator_agrees_with_model():
    """3000 seeded single- and multi-bit flips of device-written and Java-framed streams: the emulator and the model
    both fail, or both return the same bytes."""
    rng = random.Random(4321)
    bodies = [CM.wordcount_body(n=300, vocab=40, seed=s) for s in range(3)] + [bytes(rng.getrandbits(8) for _ in range(300))]
    streams = []
    for body in bodies:
        streams.append((body, M.compress_emulate(body)))
        ws = M.ifile_writes(body) if body[-2:] == b"\xff\xff" else [body]
        streams.append((body, M.java_stream(ws, compress=M.device_chunk, max_input=97)))
    fails = 0
    for i in range(3000):
        body, z = streams[i % len(streams)]
        zz = bytearray(z)
        for _ in range(1 + (i % 3 == 0)):
            bit = rng.randrange(len(zz) * 8)
            zz[bit // 8] ^= 1 << (bit % 8)
        try:
            ref = M.decode_stream(bytes(zz), len(body))
        except M.Lz4FormatError:
            ref = None
        try:
            got = M.decompress_emulate(bytes(zz), len(body))
        except TezGpuError as e:
            assert e.code == T.E_FORMAT
            got = None
        assert got == ref, (i, ref is None, got is None)
        fails += got is None
    assert 0 < fails < 3000


# ------------------------------------------------------------------------------------------------ plugin configuration
@pytest.mark.parametrize("size", [1024, M.LZ4_CHUNK_BOUND - 1, 262145, 1 << 20])
@pytest.mark.parametrize("side", ["output", "input"])
def test_plugin_refuses_lz4_buffersize_outside_the_device_range(tmp_path, size, side):
    """Checked before any device call (the output at start, the input at initialize): the key is named in the
    refusal."""
    conf = {"tez.runtime.key.class": TEXT, "tez.runtime.compress": True,
            "tez.runtime.compress.codec": "org.apache.hadoop.io.compress.Lz4Codec", "io.compression.codec.lz4.buffersize": size}
    if side == "output":
        io = OrderedPartitionedKVOutput(OutputContext(conf, str(tmp_path)), 2)
    else:
        io = OrderedGroupedKVInput(InputContext(conf, str(tmp_path)), 1)
    with pytest.raises(IOError, match=r"io\.compression\.codec\.lz4\.buffersize") as e:
        io.initialize()
        io.start()
    assert e.value.code == T.E_UNSUPPORTED

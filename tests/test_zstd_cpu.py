"""ZStandardCodec on the CPU: the device writer and reader run through their host emulations (same __host__ __device__
code) and are checked against the system libzstd, an independent implementation of RFC 8878, where it can be loaded."""
import hashlib
import os
import random

import numpy as np
import pytest

import tez_b200 as T
from tez_b200.runtime_library import TEXT, OrderedGroupedKVInput, OrderedPartitionedKVOutput, InputContext, OutputContext
from tez_b200._lib import TezGpuError
import codec_model as CM
import lz4_model as L4
import zstd_model as M

B = M.ZSTD_BLOCK_BYTES
needs_libzstd = pytest.mark.skipif(M.libzstd() is None, reason="libzstd cannot be loaded")
ZSTD = "org.apache.hadoop.io.compress.ZStandardCodec"


def _bodies():
    rng = np.random.default_rng(9)
    return {
        "wordcount": CM.wordcount_body(n=40000, vocab=3000, seed=31),
        "c3": CM.c3_body(seg_bytes=300000, seed=32),
        "int_long": CM.int_long_body(n=20000, seed=33),
        "random": rng.integers(0, 256, 150000, dtype=np.uint8).tobytes(),
        "long_runs": b"\x00" * 200000 + b"xyz" + b"\xff" * 70000 + b"abc" * 30000,
    }


def _check_written(body, z):
    """a device-writer stream: one Single_Segment frame with Frame_Content_Size and one block per piece, within the
    frame bound, decoded by the emulated reader (and libzstd where it loads).  A frame holds at most B bytes and the
    reader refuses offsets before the frame start, so every offset is below 65,536."""
    fr = M.frames(z)
    assert len(fr) == -(-len(body) // B)
    for i, (f, fhd, fcs, blocks) in enumerate(fr):
        assert fhd & 0x20 and not fhd & 0x07, fhd          # Single_Segment, no checksum, no dictionary
        assert fcs == (B if i + 1 < len(fr) else len(body) - B * i)
        assert len(blocks) == 1 and blocks[0][0] in (0, 2)
        assert len(f) <= M.ZSTD_FRAME_BOUND
    assert M.decompress_emulate(z, len(body)) == body
    if M.libzstd():
        assert M.hadoop_read(z, len(body)) == body


# ------------------------------------------------------------------------------------------------ writer
@pytest.mark.parametrize("n", [1, 2, 3, 4, 31, 32, 63, 64, 65, 100, 255, 256, 257, 4095, 4096, B - 1, B, B + 1, 3 * B + 7])
def test_writer_round_trip_sizes(n):
    rng = random.Random(n)
    body = bytes(rng.choice(b"abab\x7f\x00") for _ in range(n))
    _check_written(body, M.compress_emulate(body))


@pytest.mark.parametrize("name", sorted(_bodies()))
def test_writer_round_trip_bodies(name):
    body = _bodies()[name]
    _check_written(body, M.compress_emulate(body))


def test_writer_empty_body_is_an_empty_stream():
    assert M.compress_emulate(b"") == b""


def test_writer_raw_block_when_compression_does_not_pay():
    body = np.random.default_rng(1).integers(0, 256, B, dtype=np.uint8).tobytes()
    (f, _, _, blocks), = M.frames(M.compress_emulate(body))
    assert blocks == [(0, B)] and len(f) == M.ZSTD_FRAME_BOUND


def test_writer_huffman_literals_only_below_128():
    """Literals are Huffman-coded with direct weights when every literal is below 128, raw otherwise (the literals
    section's type, the low two bits of the block's first byte)"""
    rng = random.Random(2)
    text = bytes(rng.choice(b"etaoin shrdlu") for _ in range(20000))
    lit_type = lambda z: M.frames(z)[0][0][7 + 3] & 3   # frame header 7 bytes (2-byte content size), block header 3
    assert lit_type(M.compress_emulate(text)) == 2
    assert lit_type(M.compress_emulate(text + b"\xc3")) == 0


def test_writer_is_deterministic():
    body = CM.wordcount_body(n=50000)
    assert M.compress_emulate(body) == M.compress_emulate(body)


# ratios measured with libzstd 1.5.5 (DESIGN.md 6): device / LZ4 emulation, device / libzstd level 1
@needs_libzstd
@pytest.mark.parametrize("name", ["wordcount", "c3", "int_long"])
def test_writer_ratio_against_lz4_and_libzstd_level1(name):
    body = {"wordcount": CM.wordcount_body, "c3": CM.c3_body, "int_long": CM.int_long_body}[name]()
    z = M.compress_emulate(body)
    _check_written(body, z)
    lz4 = len(L4.compress_emulate(body))
    ref = len(M.hadoop_stream(body, level=1))
    print("%s: device %d, lz4 emulation %d (%.3f), libzstd level 1 %d (%.3f)" % (name, len(z), lz4, len(z) / lz4, ref, len(z) / ref))
    assert len(z) <= 1.25 * lz4, (len(z), lz4)


# ------------------------------------------------------------------------------------------------ reader
def test_fixture_checksums():
    for line in open(os.path.join(M.GOLDEN, "ZSTD_SHA256SUMS")):
        h, name = line.split()
        assert hashlib.sha256(open(os.path.join(M.GOLDEN, name), "rb").read()).hexdigest() == h, name


def test_emulated_reader_decodes_the_fixture():
    fx = M.fixture()
    assert len(fx) == 8
    for name, seg, raw in fx:
        assert seg[:4] == b"TIF\x01"
        body = M.decompress_emulate(seg[4:-4], raw - 4)
        assert body[-2:] == b"\xff\xff", name     # the EOF marker
        if M.libzstd():
            assert M.hadoop_read(seg[4:-4], raw - 4) == body, name


def _fixture_stream(name):
    seg, raw = [(s, r) for n, s, r in M.fixture() if n == name][0]
    return seg[4:-4], raw - 4


def test_fixture_covers_its_cases():
    z, _ = _fixture_stream("wordcount_oneshot")
    assert M.frames(z)[0][2] is not None                     # Frame_Content_Size
    z, _ = _fixture_stream("wordcount_checksum")
    assert M.frames(z)[0][1] & 4                             # Content_Checksum
    z, _ = _fixture_stream("wordcount_level3")
    assert M.frames(z)[0][2] is None and len(M.frames(z)[0][3]) > 3
    z, _ = _fixture_stream("two_frames_skippable")
    assert z.count(M.MAGIC) >= 2 and (0x184D2A53).to_bytes(4, "little") in z


@needs_libzstd
@pytest.mark.parametrize("level", [-5, 1, 3, 9, 19])
@pytest.mark.parametrize("name", sorted(_bodies()))
def test_reader_agrees_with_libzstd_across_levels(name, level):
    body = _bodies()[name]
    for z in (M.hadoop_stream(body, level=level), M.hadoop_stream(body, level=level, checksum=True),
              M.hadoop_stream(body, level=level, oneshot=True)):
        assert M.hadoop_read(z, len(body)) == body
        assert M.decompress_emulate(z, len(body)) == body


@needs_libzstd
@pytest.mark.parametrize("wlog", [10, 11, 14, 17, 20, 24, 27])
def test_reader_agrees_with_libzstd_across_window_logs(wlog):
    body = CM.wordcount_body(n=40000, vocab=3000, seed=34) * 2
    for ldm in (False, True):
        z = M.hadoop_stream(body, level=3, window_log=wlog, ldm=ldm, buf=1 << 20)
        assert M.hadoop_read(z, len(body)) == body
        assert M.decompress_emulate(z, len(body)) == body


@needs_libzstd
@pytest.mark.parametrize("body", [b"a", b"ab", b"\x00" * 1000, b"\x07" * 200000, bytes(range(256)) * 3,
                                  b"xy" * 70000 + bytes(range(256))])
def test_reader_agrees_with_libzstd_on_tiny_and_rle_bodies(body):
    """small and single-byte bodies give raw and RLE blocks and RLE literals"""
    for lvl in (1, 19):
        for z in (M.hadoop_stream(body, level=lvl), M.hadoop_stream(body, level=lvl, oneshot=True)):
            assert M.hadoop_read(z, len(body)) == body
            assert M.decompress_emulate(z, len(body)) == body
    kinds = {bt for _, _, _, blocks in M.frames(M.hadoop_stream(b"\x07" * 200000)) for bt, _ in blocks}
    assert kinds >= {1}


def test_hand_made_valid_sequences_decode_like_libzstd():
    """the builders of the malformed cases make valid streams with valid parameters: a repeat offset (offset 1); the
    compressed blocks go into frames with a 1 KiB window, as a Single_Segment frame's Block_Maximum_Size would be its
    content size"""
    z = M.make_frame(M.seq_block(b"abcd", 4, 0, 1, b"\x01"))
    assert M.decompress_emulate(z, 8) == b"abcddddd"
    if M.libzstd():
        assert M.hadoop_read(z, 8) == b"abcddddd"


@pytest.mark.parametrize("case", sorted(M.malformed()))
def test_malformed_streams_fail_with_format_error(case):
    z, n, reason = M.malformed()[case]
    with pytest.raises(TezGpuError) as e:
        M.decompress_emulate(z, n)
    assert e.value.code == T.E_FORMAT
    assert str(e.value).endswith("compressed segment 0: " + reason), str(e.value)
    if M.libzstd():
        assert M.hadoop_read(z, n) is None


# ---- bit flips against libzstd
def _modes_reserved(z):
    """a compressed block whose Symbol_Compression_Modes byte has a reserved bit set"""
    z, ip = bytes(z), 0
    try:
        while ip < len(z):
            if z[ip:ip + 4] != M.MAGIC:
                return False
            fhd = z[ip + 4]
            single = (fhd >> 5) & 1
            q = ip + 5 + (0 if single else 1) + [0, 1, 2, 4][fhd & 3] + [single, 2, 4, 8][fhd >> 6]
            while True:
                bh = int.from_bytes(z[q:q + 3], "little")
                bt, bs = (bh >> 1) & 3, bh >> 3
                if bt == 2 and bs:
                    b = z[q + 3:q + 3 + bs]
                    lt, sf = b[0] & 3, (b[0] >> 2) & 3
                    if lt < 2:
                        hs = {0: 1, 1: 2, 2: 1, 3: 3}[sf]
                        size = int.from_bytes(b[:hs], "little") >> (3 if hs == 1 else 4)
                        end = hs + (size if lt == 0 else 1)
                    else:
                        hs, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
                        end = hs + (int.from_bytes(b[:hs], "little") >> (4 + bits) & ((1 << bits) - 1))
                    nb = b[end]
                    e = end + (1 if nb < 128 else 3 if nb == 255 else 2)
                    if nb and b[e] & 3:
                        return True
                q += 3 + (1 if bt == 1 else bs)
                if bh & 1:
                    break
            ip = q + (4 if fhd & 4 else 0)
    except (IndexError, KeyError):
        return False
    return False


# Where the device reader and libzstd 1.5.5 disagree, libzstd accepts and the device reader refuses (DESIGN.md 6):
#   bitstream   -- a Huffman stream or sequence bitstream not consumed exactly (libzstd's fast Huffman decoder checks only
#                  the output length; its sequence decoder takes an over-read);
#   modes       -- a reserved bit of the Symbol_Compression_Modes byte (libzstd 1.5.5 ignores it; RFC 8878 and later
#                  libzstd refuse it).
@needs_libzstd
def test_bit_flip_fuzz_emulator_agrees_with_libzstd():
    """3000 seeded single- and multi-bit flips of device-written and Hadoop-like streams: the emulator and libzstd give
    the same bytes, or both fail, or the case is one of the two named deviations."""
    rng = random.Random(8765)
    bodies = [CM.wordcount_body(n=300, vocab=40, seed=s) for s in range(3)] + [bytes(rng.getrandbits(7) for _ in range(600))]
    streams = []
    for body in bodies:
        streams.append((body, M.compress_emulate(body)))
        streams.append((body, M.hadoop_stream(body, level=3, buf=97)))
        streams.append((body, M.hadoop_stream(body, level=19, checksum=True)))
    fails, deviations = 0, {"bitstream": 0, "modes": 0}
    for i in range(3000):
        body, z = streams[i % len(streams)]
        zz = bytearray(z)
        for _ in range(1 + (i % 3 == 0)):
            bit = rng.randrange(len(zz) * 8)
            zz[bit // 8] ^= 1 << (bit % 8)
        ref = M.hadoop_read(bytes(zz), len(body))
        reason = None
        try:
            got = M.decompress_emulate(bytes(zz), len(body))
        except TezGpuError as e:
            assert e.code == T.E_FORMAT
            got, reason = None, str(e).split(": ")[-1]
        if got != ref:
            assert got is None, (i, "the device reader accepts what libzstd refuses")
            if reason == "bitstream not consumed exactly":
                deviations["bitstream"] += 1
            else:
                assert reason == "reserved bit set" and _modes_reserved(zz), (i, reason, bytes(zz).hex())
                deviations["modes"] += 1
        fails += got is None
    assert 0 < fails < 3000
    print("deviations", deviations)
    assert sum(deviations.values()) < 100


# ------------------------------------------------------------------------------------------------ plugin configuration
@pytest.mark.parametrize("level", [None, -5, 1, 3, 19, 22])
@pytest.mark.parametrize("side", ["output", "input"])
def test_plugin_accepts_zstandard_codec_at_any_level(tmp_path, level, side):
    """The codec check runs before any device call; past it, a machine without a GPU fails on the device, never with
    the codec refusal."""
    conf = {"tez.runtime.key.class": TEXT, "tez.runtime.compress": True, "tez.runtime.compress.codec": ZSTD}
    if level is not None:
        conf["io.compression.codec.zstd.level"] = level
    if side == "output":
        io = OrderedPartitionedKVOutput(OutputContext(conf, str(tmp_path)), 2)
    else:
        io = OrderedGroupedKVInput(InputContext(conf, str(tmp_path)), 1)
    try:
        io.initialize()
        io.start()
    except IOError as e:
        assert e.code != T.E_UNSUPPORTED and "codec" not in str(e), str(e)
    finally:
        try:
            io.close()
        except Exception:
            pass

"""Shared helpers of the DefaultCodec tests: the host runs of the device codec (tezgpu_debug_*_emulate), the reference
reader (Hadoop's DecompressorStream restated over the system zlib) and the segment bodies the ratio checks use."""
import ctypes as C
import os
import random
import struct
import zlib

import numpy as np

from oracle import tez_oracle as O
from tez_b200 import _lib

CHUNK = 32768


def deflate_emulate(body):
    """The zlib stream the device writer produces for one segment body."""
    L = _lib.load()
    body = bytes(body)
    cap = len(body) + 5 * (len(body) // CHUNK + 1) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_deflate_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def inflate_emulate(z, body_len):
    """Decodes with the device reader's decoder; raises TezGpuError (E_FORMAT) on a malformed stream."""
    L = _lib.load()
    z = bytes(z)
    out = (C.c_uint8 * max(1, body_len))()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_inflate_emulate(z, len(z), body_len, out, body_len, C.byref(n)))
    return bytes(out[:n.value])


def hadoop_inflate(z):
    """DecompressorStream over zlib: decode members until the input is used up; a member that does not end, or bytes
    after a member that are not a member, fail (zlib.error)."""
    z = bytes(z)
    out = []
    while True:
        d = zlib.decompressobj()
        out.append(d.decompress(z))
        if not d.eof:
            raise zlib.error("truncated stream")
        z = d.unused_data
        if not z:
            return b"".join(out)


def compressed_segment(body, level=1, strategy=zlib.Z_DEFAULT_STRATEGY, members=1):
    """TIF\\x01 + zlib stream(s) of body + CRC-32 of the compressed bytes (what IFile.Writer writes with DefaultCodec),
    and its rawLength."""
    body = bytes(body)
    parts = []
    cuts = [len(body) * i // members for i in range(members + 1)]
    for a, b in zip(cuts, cuts[1:]):
        c = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
        parts.append(c.compress(body[a:b]) + c.flush())
    z = b"".join(parts)
    return b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big"), len(body) + 4


def body_of(seg):
    """Uncompressed IFile segment -> its body (records, markers, EOF)."""
    return bytes(seg[4:-4])


def wordcount_body(n=200000, vocab=5000, seed=1):
    """Map output of word count: Text words (Zipf-like draw) with IntWritable 1, sorted by key."""
    rng = random.Random(seed)
    words = ["w%x%s" % (i, "abcdefgh"[: i % 7]) for i in range(vocab)]
    weights = [1.0 / (i + 1) for i in range(vocab)]
    keys = rng.choices(words, weights=weights, k=n)
    recs = sorted((bytes([len(w)]) + w.encode(), b"\x00\x00\x00\x01") for w in keys)
    out, _, _ = O.write_ifile(recs, rle=False)
    return body_of(out)


def c3_body(seg_bytes=1 << 20, seed=3):
    segs, _ = O.gen_c3_segments(1, seg_bytes, seed=seed, threads=1)
    return body_of(segs[0].tobytes())


def int_long_body(n=150000, seed=5):
    """IntWritable keys (sorted, with repeats) and LongWritable values."""
    rng = np.random.default_rng(seed)
    keys = np.sort(rng.integers(0, 1 << 20, size=n).astype(np.int64))
    vals = rng.integers(0, 1 << 24, size=n)
    recs = [(struct.pack(">i", int(k)), struct.pack(">q", int(v))) for k, v in zip(keys, vals)]
    out, _, _ = O.write_ifile(recs, rle=False)
    return body_of(out)


# ------------------------------------------------------------------------------------------------ the fixture
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# the fixture's rawLengths and compressed segment lengths (TestIFile.java:395-397)
FIXTURE_RAWS = [2392, 102314, 42576, 31432, 25090]
FIXTURE_COMPRESSED = [723, 25396, 10926, 8203, 6665]


def segment(z):
    """TIF\\x01 + stream + CRC-32 of the stream"""
    return b"TIF\x01" + bytes(z) + zlib.crc32(bytes(z)).to_bytes(4, "big")


def fixture():
    """[(segment bytes, rawLength)] of the reference's five compressed segments (written by the real IFile.Writer)"""
    data = open(os.path.join(GOLDEN, "TestIFile_concatenated_compressed.bin"), "rb").read()
    res, pos = [], 0
    for c, raw in zip(FIXTURE_COMPRESSED, FIXTURE_RAWS):
        res.append((data[pos:pos + c], raw))
        pos += c
    return res


# ------------------------------------------------------------------------------------------------ malformed streams
class Bits:
    """LSB-first bit string builder (Huffman codes are given MSB first, as RFC 1951 writes them)."""

    def __init__(self):
        self.bits = []

    def put(self, v, n):
        self.bits += [(v >> i) & 1 for i in range(n)]
        return self

    def huff(self, code, n):
        self.bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]
        return self

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + k] << k for k in range(8)) for i in range(0, len(b), 8))


def zhdr(cinfo=7, fdict=0):
    cmf = (cinfo << 4) | 8
    flg = fdict << 5
    flg |= (31 - ((cmf << 8) | flg) % 31) % 31
    return bytes([cmf, flg])


def _adler(b):
    return zlib.adler32(b).to_bytes(4, "big")


def malformed():
    good = zlib.compress(b"hello hello hello hello", 6)
    cases = {
        "bad_check": b"\x78\x02" + good[2:],
        "bad_method": bytes([0x77, good[1]]) + good[2:],
        "fdict": zhdr(fdict=1) + b"\0\0\0\0" + good[2:],
        "btype3": zhdr() + Bits().put(1, 1).put(3, 2).bytes() + b"\0" * 8,
        "stored_nlen": zhdr() + b"\x01\x05\x00\x00\x00hello" + _adler(b"hello"),
        # code-length code: all 19 lengths 1 -> over-subscribed
        "cl_oversubscribed": zhdr() + Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(15, 4).put(0x49249249249249, 57).bytes() + b"\0" * 8,
        # code-length code: one code of length 1 -> incomplete (never allowed for this code)
        "cl_incomplete": zhdr() + Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(0, 4).put(1, 3).put(0, 9).bytes() + b"\0" * 8,
        # literal/length symbol 286 in a fixed block (8-bit code 11000110)
        "len_symbol_286": zhdr() + Bits().put(1, 1).put(1, 2).huff(0b11000110, 8).bytes() + b"\0" * 6,
        # 'a', then length 3 (symbol 257, 0000001) with distance symbol 30 (11110)
        "dist_symbol_30": zhdr() + Bits().put(1, 1).put(1, 2).huff(0x30 + ord("a"), 8).huff(1, 7).huff(30, 5).huff(0, 7).bytes() + b"\0" * 4,
        # length 3 at distance 1 before any output
        "dist_too_far": zhdr() + Bits().put(1, 1).put(1, 2).huff(1, 7).huff(0, 5).huff(0, 7).bytes() + b"\0" * 4,
        "truncated": good[:-3],
        "truncated_header": good[:1],
        "adler": good[:-1] + bytes([good[-1] ^ 1]),
        "trailing_garbage": good + b"\x00",
        "trailing_partial_member": good + good[:5],
    }
    return cases, len(b"hello hello hello hello")

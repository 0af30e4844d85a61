"""Shared helpers of the DefaultCodec tests: the host runs of the device codec (tezgpu_debug_*_emulate), the reference
reader (Hadoop's DecompressorStream restated over the system zlib) and the segment bodies the ratio checks use."""
import ctypes as C
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

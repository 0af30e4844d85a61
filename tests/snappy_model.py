"""Shared helpers of the SnappyCodec tests: the host runs of the device codec (tezgpu_debug_snappy_*_emulate), a Python
restatement of the strict reader, libsnappy through pyarrow (where pyarrow imports), Hadoop's BlockCompressorStream
framing at SnappyCodec's buffer size, and hand-made chunks with elements libsnappy never writes."""
import ctypes as C
import json
import os
import random
import zlib

from tez_b200 import _lib
from tez_b200.constants import SNAPPY_BLOCK_BYTES, SNAPPY_CHUNK_BOUND
import codec_model as CM
from lz4_model import ifile_writes, java_stream as _java_stream   # noqa: F401  (the framing is Lz4Codec's)

CHUNK_CAP = 262144                            # io.compression.codec.snappy.buffersize default: SnappyDecompressor's buffer
MAX_INPUT = CHUNK_CAP - (CHUNK_CAP // 6 + 32)   # BlockCompressorStream's MAX_INPUT_SIZE at that buffer: 218,422
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "snappy_segments.bin")
MANIFEST = os.path.join(GOLDEN, "snappy_segments.json")


# ------------------------------------------------------------------------------------------------ device emulations
def compress_emulate(body):
    """The block stream the device writer produces for one segment body."""
    L = _lib.load()
    body = bytes(body)
    cap = len(body) + 14 * (len(body) // SNAPPY_BLOCK_BYTES + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_snappy_compress_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def decompress_emulate(z, body_len):
    """Decodes with the device reader's exact path; raises TezGpuError (E_FORMAT) on a malformed stream."""
    L = _lib.load()
    z = bytes(z)
    out = (C.c_uint8 * max(1, body_len))()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_snappy_decompress_emulate(z, len(z), body_len, out, body_len, C.byref(n)))
    return bytes(out[:n.value])


def device_chunk(data):
    """The device writer's chunk for data of at most one block (the stream without its 8 header bytes)."""
    z = compress_emulate(data)
    assert 0 < len(data) <= SNAPPY_BLOCK_BYTES and int.from_bytes(z[4:8], "big") == len(z) - 8
    return z[8:]


# ------------------------------------------------------------------------------------------------ the strict reader
class SnappyFormatError(Exception):
    pass


def varint(v):
    out = bytearray()
    while v >= 128:
        out.append((v & 127) | 128)
        v >>= 7
    out.append(v)
    return bytes(out)


def preamble(src):
    """(value, bytes) of a chunk's preamble as libsnappy reads it (at most 5 bytes, the fifth below 16), or None"""
    v = 0
    for k in range(min(5, len(src))):
        c = src[k]
        if k == 4 and c > 15:
            return None
        v |= (c & 127) << (7 * k)
        if c < 128:
            return v, k + 1
    return None


def decode_chunk(src):
    """One raw Snappy block, strictly: a preamble of 1 .. 262,144, every element inside the chunk, copy offsets within
    the bytes produced, the output ending exactly at the preamble length with the input consumed."""
    src = bytes(src)
    n = len(src)
    pre = preamble(src)
    if pre is None or pre[0] == 0 or pre[0] > CHUNK_CAP:
        raise SnappyFormatError("invalid chunk preamble")
    raw, ip = pre
    out = bytearray()
    while ip < n:
        tag = src[ip]
        ip += 1
        t = tag & 3
        if t == 0:
            L = tag >> 2
            if L >= 60:
                b = L - 59
                if b > n - ip:
                    raise SnappyFormatError("literal past the end of the chunk")
                L = int.from_bytes(src[ip:ip + b], "little")
                ip += b
            L += 1
            if L > n - ip:
                raise SnappyFormatError("literal past the end of the chunk")
            if L > raw - len(out):
                raise SnappyFormatError("chunk decodes past its preamble length")
            out += src[ip:ip + L]
            ip += L
            continue
        eb = {1: 1, 2: 2, 3: 4}[t]
        if eb > n - ip:
            raise SnappyFormatError("copy past the end of the chunk")
        if t == 1:
            ln, off = ((tag >> 2) & 7) + 4, ((tag >> 5) << 8) | src[ip]
        else:
            ln, off = (tag >> 2) + 1, int.from_bytes(src[ip:ip + eb], "little")
        ip += eb
        if off == 0 or off > len(out):
            raise SnappyFormatError("invalid copy offset")
        if ln > raw - len(out):
            raise SnappyFormatError("chunk decodes past its preamble length")
        for _ in range(ln):
            out.append(out[-off])
    if len(out) != raw:
        raise SnappyFormatError("chunk decodes short of its preamble length")
    return bytes(out)


def decode_stream(z, expect, chunk=decode_chunk):
    """A segment's stream (between TIF\\x01 and the CRC): blocks of raw length > 0 whose chunks' preambles add up to
    exactly that length, the blocks adding up to expect = rawLength - 4, nothing after the last block.  chunk decodes
    one chunk (the model, or libsnappy_chunk)."""
    z = bytes(z)
    n, ip, out = len(z), 0, bytearray()
    while len(out) < expect:
        if ip + 4 > n:
            raise SnappyFormatError("decompressed length differs from rawLength - 4" if ip == n else "truncated block header")
        raw = int.from_bytes(z[ip:ip + 4], "big")
        ip += 4
        if raw == 0 or raw > 0x7FFFFFFF or raw > expect - len(out):
            raise SnappyFormatError("block raw length outside the remaining rawLength - 4")
        got = 0
        while got < raw:
            if ip + 4 > n:
                raise SnappyFormatError("truncated block header")
            c = int.from_bytes(z[ip:ip + 4], "big")
            ip += 4
            if c > CHUNK_CAP or c > n - ip:
                raise SnappyFormatError("chunk length over 262144 or past the end of the stream")
            pre = preamble(z[ip:ip + c])
            if pre is None or pre[0] == 0 or pre[0] > CHUNK_CAP:
                raise SnappyFormatError("invalid chunk preamble")
            if pre[0] > raw - got:
                raise SnappyFormatError("chunks decode past their block's raw length")
            out += chunk(z[ip:ip + c])
            got += pre[0]
            ip += c
    if ip != n:
        raise SnappyFormatError("bytes after the last block")
    return bytes(out)


def blocks(z):
    """(raw length, [chunk, ...]) of every block of a well-framed stream"""
    z, ip, res = bytes(z), 0, []
    while ip < len(z):
        raw = int.from_bytes(z[ip:ip + 4], "big")
        ip += 4
        chunks, got = [], 0
        while got < raw:
            c = int.from_bytes(z[ip:ip + 4], "big")
            chunks.append(z[ip + 4:ip + 4 + c])
            got += preamble(chunks[-1])[0]
            ip += 4 + c
        res.append((raw, chunks))
    return res


# ------------------------------------------------------------------------------------------------ libsnappy
def pyarrow():
    """pyarrow (which bundles libsnappy) or None"""
    try:
        import pyarrow as pa
        return pa
    except ImportError:
        return None


NO_PYARROW = "pyarrow (libsnappy) is not installed: the comparison with libsnappy is skipped"


def snappy_compress(data):
    """libsnappy's raw block of data (snappy::RawCompress)"""
    return pyarrow().compress(bytes(data), codec="snappy", asbytes=True)


def libsnappy_chunk(chunk):
    """libsnappy's decode of one chunk (snappy::RawUncompress into a buffer of its preamble length); raises
    SnappyFormatError where libsnappy refuses it"""
    chunk = bytes(chunk)
    pre = preamble(chunk)
    if pre is None or pre[0] > 16 << 20:
        raise SnappyFormatError("libsnappy: bad preamble")
    try:
        return pyarrow().decompress(chunk, decompressed_size=pre[0], codec="snappy", asbytes=True)
    except (OSError, ValueError) as e:
        raise SnappyFormatError("libsnappy: " + str(e))


def java_stream(writes, compress=None):
    """BlockCompressorStream over SnappyCompressor at the default buffer size (lz4_model.java_stream, MAX_INPUT)"""
    return _java_stream(writes, compress=compress or snappy_compress, max_input=MAX_INPUT)


def java_chunk(d):
    """libsnappy's chunk where pyarrow imports, else an all-literal chunk (the block framing is Java's either way)"""
    if pyarrow() is not None:
        return snappy_compress(d)
    return varint(len(d)) + lit(bytes(d))


def segment(z):
    """TIF\\x01 + stream + CRC-32 of the stream"""
    return b"TIF\x01" + bytes(z) + zlib.crc32(bytes(z)).to_bytes(4, "big")


def one_block(chunks):
    """a stream of one block holding the given chunks"""
    raw = sum(preamble(c)[0] for c in chunks)
    return raw.to_bytes(4, "big") + b"".join(len(c).to_bytes(4, "big") + c for c in chunks)


# ------------------------------------------------------------------------------------------------ hand-made chunks
def lit(data, tag_bytes=None):
    """a literal element; tag_bytes (1-4) forces tags 60-63 even where a shorter form fits"""
    n = len(data) - 1
    if tag_bytes is None:
        if n < 60:
            return bytes([n << 2]) + data
        tag_bytes = 1 if n < 256 else 2 if n < 65536 else 3 if n < 1 << 24 else 4
    return bytes([(59 + tag_bytes) << 2]) + n.to_bytes(tag_bytes, "little") + data


def copy(off, ln, kind):
    """a copy element: kind 1 (4-11 bytes, offset < 2048), 2 or 4 (1-64 bytes)"""
    if kind == 1:
        return bytes([1 | ((ln - 4) << 2) | ((off >> 8) << 5), off & 255])
    if kind == 2:
        return bytes([2 | ((ln - 1) << 2)]) + off.to_bytes(2, "little")
    return bytes([3 | ((ln - 1) << 2)]) + off.to_bytes(4, "little")


def crafted_chunks(seed=21):
    """[(name, chunk)]: copy-4 elements, literal tags 62 and 63, overlapping copies at offsets 1-32 of every kind and
    length shape (1, 4-11, 31-33, 64), each decoding to the model's bytes"""
    rng = random.Random(seed)
    rb = lambda n: bytes(rng.getrandbits(8) for _ in range(n))   # noqa: E731
    res = []

    def add(name, elems):
        body = b"".join(elems)
        chunk = varint(len(decode_chunk_elements(body))) + body
        decode_chunk(chunk)
        res.append((name, chunk))

    e = [lit(rb(70))]
    for off, ln in ((70, 64), (1, 5), (3, 64), (100, 1), (17, 33), (134, 40)):
        e.append(copy(off, ln, 4))
    add("copy4", e)
    add("literal_tags_62_63", [lit(rb(300), 3), lit(rb(5), 4), lit(rb(61), 3), copy(300, 12, 4), lit(rb(70000), 3)])
    e = [lit(rb(32))]
    for off in range(1, 33):
        for ln, kind in ((1, 2), (4, 1), (11, 1), (31, 2), (32, 2), (33, 4), (64, 2), (7, 4)):
            e.append(copy(off, ln, kind))
        e.append(lit(rb(off % 5 + 1)))
    add("overlap_1_32", e)
    e = [lit(b"ab")]
    for _ in range(200):
        e.append(copy(rng.choice((1, 2)), 64, 2))
    add("runs_of_one_and_two", e)
    return res


def decode_chunk_elements(body):
    """the bytes a chunk's elements (no preamble) decode to, where every copy lies within the bytes produced"""
    out, ip = bytearray(), 0
    while ip < len(body):
        tag = body[ip]
        ip += 1
        t = tag & 3
        if t == 0:
            L = tag >> 2
            if L >= 60:
                L, ip = int.from_bytes(body[ip:ip + L - 59], "little"), ip + L - 59
            out += body[ip:ip + L + 1]
            ip += L + 1
            continue
        eb = {1: 1, 2: 2, 3: 4}[t]
        if t == 1:
            ln, off = ((tag >> 2) & 7) + 4, ((tag >> 5) << 8) | body[ip]
        else:
            ln, off = (tag >> 2) + 1, int.from_bytes(body[ip:ip + eb], "little")
        ip += eb
        assert 0 < off <= len(out)
        for _ in range(ln):
            out.append(out[-off])
    return bytes(out)


def fixture():
    """[(name, segment bytes, rawLength)] of tests/golden/snappy_segments.bin"""
    data = open(FIXTURE, "rb").read()
    man = json.load(open(MANIFEST))
    res, pos = [], 0
    for e in man["segments"]:
        res.append((e["name"], data[pos:pos + e["part_length"]], e["raw_length"]))
        pos += e["part_length"]
    assert pos == len(data)
    return res


# ------------------------------------------------------------------------------------------------ mutants
def mutants(streams, count, seed):
    """count seeded corruptions (bit flips, header flips, truncations, rawLength +- 1) of (body, stream) pairs:
    [(stream, expect)]"""
    rng = random.Random(seed)
    res = []
    for i in range(count):
        body, z = streams[i % len(streams)]
        zz = bytearray(z)
        expect = len(body)
        kind = rng.randrange(5)
        if kind == 0 and zz:
            bit = rng.randrange(len(zz) * 8)
            zz[bit >> 3] ^= 1 << (bit & 7)
        elif kind == 1 and zz:
            bit = rng.randrange(min(len(zz), 16) * 8)
            zz[bit >> 3] ^= 1 << (bit & 7)
        elif kind == 2 and zz:
            for _ in range(rng.randint(2, 6)):
                bit = rng.randrange(len(zz) * 8)
                zz[bit >> 3] ^= 1 << (bit & 7)
        elif kind == 3 and zz:
            del zz[rng.randrange(len(zz)):]
        else:
            expect += rng.choice((-1, 1))
        res.append((bytes(zz), max(expect, 0)))
    return res


# ------------------------------------------------------------------------------------------------ malformed and mutated streams
def blk(raw, *chunks):
    return raw.to_bytes(4, "big") + b"".join(len(c).to_bytes(4, "big") + c for c in chunks)


def malformed():
    """{name: (stream, expect, reason)}"""
    body = CM.wordcount_body(n=300, vocab=40, seed=1)
    z = compress_emulate(body)
    (raw, (c,)), = blocks(z)
    abcd = lit(b"abcd")
    return {
        "preamble_runs_past_5_bytes": (blk(8, b"\xff\xff\xff\xff\xff\x01" + abcd), 8, "invalid chunk preamble"),
        "preamble_fifth_byte_over_15": (blk(8, b"\x80\x80\x80\x80\x10" + abcd), 8, "invalid chunk preamble"),
        "preamble_zero": (blk(8, b"\x00", varint(8) + abcd + copy(4, 4, 1)), 8, "invalid chunk preamble"),
        "preamble_over_262144": (blk(300000, varint(262145) + abcd), 300000, "invalid chunk preamble"),
        "preamble_truncated": (blk(200, b"\xc8"), 200, "invalid chunk preamble"),
        "offset_zero": (blk(8, varint(8) + abcd + copy(0, 4, 1)), 8, "invalid copy offset"),
        "offset_zero_copy4": (blk(8, varint(8) + abcd + copy(0, 4, 4)), 8, "invalid copy offset"),
        "offset_past_the_output": (blk(8, varint(8) + abcd + copy(5, 4, 2)), 8, "invalid copy offset"),
        "literal_past_the_chunk": (blk(10, varint(10) + bytes([9 << 2]) + b"abc"), 10, "literal past the end of the chunk"),
        "literal_length_bytes_past_the_chunk": (blk(100, varint(100) + bytes([61 << 2, 99])), 100, "literal past the end of the chunk"),
        "copy_past_the_chunk": (blk(8, varint(8) + abcd + bytes([2 | (3 << 2), 4])), 8, "copy past the end of the chunk"),
        "copy4_past_the_chunk": (blk(8, varint(8) + abcd + bytes([3 | (3 << 2), 4, 0, 0])), 8, "copy past the end of the chunk"),
        "short_output": (blk(9, varint(9) + abcd + copy(4, 4, 1)), 9, "chunk decodes short of its preamble length"),
        "long_output_copy": (blk(7, varint(7) + abcd + copy(4, 4, 1)), 7, "chunk decodes past its preamble length"),
        "long_output_literal": (blk(3, varint(3) + abcd), 3, "chunk decodes past its preamble length"),
        "trailing_element": (blk(4, varint(4) + abcd + copy(4, 4, 1)), 4, "chunk decodes past its preamble length"),
        "trailing_bytes": (z + b"\0\0\0\0", len(body), "bytes after the last block"),
        "chunks_short_of_the_block": (blk(raw + 1, c), len(body) + 1, "truncated block header"),
        "chunks_past_the_block": (blk(raw - 1, c), len(body) - 1, "chunks decode past their block's raw length"),
        "blocks_short_of_rawlength": (z, len(body) + 1, "decompressed length differs from rawLength - 4"),
        "blocks_past_rawlength": (z, len(body) - 1, "block raw length outside the remaining rawLength - 4"),
        "block_raw_zero": (blk(0, c), len(body), "block raw length outside the remaining rawLength - 4"),
        "chunk_over_262144": (blk(8, b"") [:4] + (262145).to_bytes(4, "big") + b"\0" * 262145, 8,
                              "chunk length over 262144 or past the end of the stream"),
        "chunk_past_the_stream": (z[:-1], len(body), "chunk length over 262144 or past the end of the stream"),
        "truncated_header": (z[:6], len(body), "truncated block header"),
        "second_of_two_chunks_bad": (blk(16, varint(8) + abcd + copy(4, 4, 1), varint(8) + abcd + copy(9, 4, 1)), 16,
                                     "invalid copy offset"),
    }


def corpus_streams():
    """(body, stream) pairs the mutant corpus corrupts: device-written, Java-framed libsnappy-like and crafted"""
    bodies = [CM.wordcount_body(n=300, vocab=40, seed=s) for s in range(3)] + [random.Random(9).randbytes(600)]
    res = [(b, compress_emulate(b)) for b in bodies]
    res += [(decode_chunk(c), one_block([c])) for _, c in crafted_chunks() if len(c) < 4096]
    return res

"""Shared helpers of the Lz4Codec tests: the host runs of the device codec (tezgpu_debug_lz4_*_emulate), a Python
restatement of the strict reader, liblz4 through ctypes (where it can be loaded) and Hadoop's BlockCompressorStream
framing as Java's IFile.Writer drives it."""
import ctypes as C
import ctypes.util
import json
import os
import zlib

from tez_b200 import _lib
from tez_b200.constants import LZ4_BLOCK_BYTES, LZ4_CHUNK_BOUND

CHUNK_CAP = 262144                            # io.compression.codec.lz4.buffersize default: Lz4Decompressor's buffer
MAX_INPUT = CHUNK_CAP - (CHUNK_CAP // 255 + 16)   # BlockCompressorStream's MAX_INPUT_SIZE at that buffer: 261,100
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "lz4_segments.bin")
MANIFEST = os.path.join(GOLDEN, "lz4_segments.json")


# ------------------------------------------------------------------------------------------------ device emulations
def compress_emulate(body):
    """The block stream the device writer produces for one segment body."""
    L = _lib.load()
    body = bytes(body)
    cap = len(body) + len(body) // 255 + 10 * (len(body) // LZ4_BLOCK_BYTES + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_lz4_compress_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def decompress_emulate(z, body_len):
    """Decodes with the device reader's exact path; raises TezGpuError (E_FORMAT) on a malformed stream."""
    L = _lib.load()
    z = bytes(z)
    out = (C.c_uint8 * max(1, body_len))()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_lz4_decompress_emulate(z, len(z), body_len, out, body_len, C.byref(n)))
    return bytes(out[:n.value])


def device_chunk(data):
    """The device writer's chunk for data of at most one block (the stream without its 8 header bytes)."""
    z = compress_emulate(data)
    assert 0 < len(data) <= LZ4_BLOCK_BYTES and int.from_bytes(z[4:8], "big") == len(z) - 8
    return z[8:]


# ------------------------------------------------------------------------------------------------ the strict reader
class Lz4FormatError(Exception):
    pass


def decode_chunk(src, cap=CHUNK_CAP):
    """One raw LZ4 block as LZ4_decompress_safe(src, dst, len(src), cap) decodes it, end-of-chunk conditions included
    (a non-final literal run leaves at least 8 input bytes and ends 12 bytes before cap; a match length byte leaves 5
    input bytes; a match ends 5 bytes before cap), except that offset 0 is an error."""
    src = bytes(src)
    n = len(src)
    out = bytearray()
    ip = 0
    while True:
        if ip >= n:
            raise Lz4FormatError("literal run past the end of the chunk")
        tok = src[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                if ip >= n:
                    raise Lz4FormatError("literal run past the end of the chunk")
                s = src[ip]
                ip += 1
                lit += s
                if s != 255:
                    break
        if len(out) + lit + 12 > cap or ip + lit + 8 > n:      # the last literals
            if ip + lit != n or len(out) + lit > cap:
                raise Lz4FormatError("literal run past the end of the chunk")
            out += src[ip:ip + lit]
            return bytes(out)
        out += src[ip:ip + lit]
        ip += lit
        off = src[ip] | (src[ip + 1] << 8)
        ip += 2
        if off == 0 or off > len(out):
            raise Lz4FormatError("invalid match offset")
        m = tok & 15
        if m == 15:
            while True:
                s = src[ip]
                ip += 1
                if ip + 5 > n:
                    raise Lz4FormatError("invalid match length")
                m += s
                if s != 255:
                    break
        m += 4
        if len(out) + m + 5 > cap:
            raise Lz4FormatError("invalid match length")
        for _ in range(m):
            out.append(out[-off])


def decode_stream(z, expect):
    """A segment's stream (between TIF\\x01 and the CRC): blocks of raw length > 0 whose chunks decode to exactly that
    length, adding up to expect = rawLength - 4, nothing after the last block."""
    z = bytes(z)
    n, ip, out = len(z), 0, bytearray()
    while len(out) < expect:
        if ip + 4 > n:
            raise Lz4FormatError("truncated block header")
        raw = int.from_bytes(z[ip:ip + 4], "big")
        ip += 4
        if raw == 0 or raw > 0x7FFFFFFF or raw > expect - len(out):
            raise Lz4FormatError("block raw length outside the remaining rawLength - 4")
        got = bytearray()
        while len(got) < raw:
            if ip + 4 > n:
                raise Lz4FormatError("truncated block header")
            c = int.from_bytes(z[ip:ip + 4], "big")
            ip += 4
            if c > CHUNK_CAP or c > n - ip:
                raise Lz4FormatError("chunk length over 262144 or past the end of the stream")
            got += decode_chunk(z[ip:ip + c])
            ip += c
            if len(got) > raw:
                raise Lz4FormatError("chunks decode past their block's raw length")
        out += got
    if ip != n:
        raise Lz4FormatError("bytes after the last block")
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
            got += len(decode_chunk(chunks[-1]))
            ip += 4 + c
        res.append((raw, chunks))
    return res


# ------------------------------------------------------------------------------------------------ liblz4
_LIB = []


def liblz4():
    """The system liblz4 or None."""
    if not _LIB:
        name = ctypes.util.find_library("lz4") or "liblz4.so.1"
        try:
            _LIB.append(C.CDLL(name))
        except OSError:
            _LIB.append(None)
    return _LIB[0]


def lz4_compress(data, mode="fast", accel=1):
    """One raw LZ4 block of data: LZ4_compress_fast(acceleration) or LZ4_compress_HC (mode "hc")."""
    L = liblz4()
    data = bytes(data)
    cap = len(data) + len(data) // 255 + 16
    out = (C.c_uint8 * cap)()
    if mode == "hc":
        n = L.LZ4_compress_HC(data, out, len(data), cap, 9)
    else:
        n = L.LZ4_compress_fast(data, out, len(data), cap, accel)
    assert n > 0
    return bytes(out[:n])


def lz4_decompress_safe(chunk, cap=CHUNK_CAP):
    """liblz4's LZ4_decompress_safe(chunk, dst, len, cap): the bytes, or None where it fails."""
    L = liblz4()
    chunk = bytes(chunk)
    out = (C.c_uint8 * cap)()
    n = L.LZ4_decompress_safe(chunk, out, len(chunk), cap)
    return bytes(out[:n]) if n >= 0 else None


# ------------------------------------------------------------------------------------------------ Java's writer
def ifile_writes(body):
    """The write() calls IFile.Writer issues for an uncompressed body without RLE markers: every vint byte alone, then
    the key, then the value; the EOF marker is two vint bytes."""
    body = bytes(body)
    writes, p = [], 0

    def vint(p):
        b = body[p] - 256 if body[p] > 127 else body[p]
        n = 1 if b >= -112 else (-119 - b if b < -120 else -111 - b)
        if n == 1:
            return b, 1
        v = int.from_bytes(body[p + 1:p + n], "big")
        return (~v if b < -120 else v), n

    while True:
        kl, a = vint(p)
        writes += [body[p + i:p + i + 1] for i in range(a)]
        p += a
        vl, b = vint(p)
        writes += [body[p + i:p + i + 1] for i in range(b)]
        p += b
        if kl == -1 and vl == -1:
            break
        writes += [body[p:p + kl], body[p + kl:p + kl + vl]]
        p += kl + vl
    assert p == len(body) and b"".join(writes) == body
    return writes


def java_stream(writes, compress=lambda d: lz4_compress(d), max_input=MAX_INPUT):
    """BlockCompressorStream over Lz4Compressor: a write that would take the pending input past max_input first closes
    the pending block; a write longer than max_input becomes one block of chunks of at most max_input raw bytes."""
    out, pending = bytearray(), bytearray()

    def close():
        if pending:
            out.extend(len(pending).to_bytes(4, "big"))
            c = compress(bytes(pending))
            out.extend(len(c).to_bytes(4, "big") + c)
            pending.clear()

    for w in writes:
        if len(w) + len(pending) > max_input and pending:
            close()
        if len(w) > max_input:
            out.extend(len(w).to_bytes(4, "big"))
            for a in range(0, len(w), max_input):
                c = compress(w[a:a + max_input])
                out.extend(len(c).to_bytes(4, "big") + c)
            continue
        pending.extend(w)
    close()
    return bytes(out)


def java_chunk(d, hc=False):
    """liblz4's chunk (LZ4_compress_HC where hc) where liblz4 can be loaded, else an all-literal chunk (the block framing
    is Java's either way)"""
    if liblz4() is not None:
        return lz4_compress(d, mode="hc" if hc else "fast")
    return lit(d)


def segment(z):
    """TIF\\x01 + stream + CRC-32 of the stream"""
    return b"TIF\x01" + bytes(z) + zlib.crc32(bytes(z)).to_bytes(4, "big")


def fixture():
    """[(name, segment bytes, rawLength)] of tests/golden/lz4_segments.bin"""
    data = open(FIXTURE, "rb").read()
    man = json.load(open(MANIFEST))
    res, pos = [], 0
    for e in man["segments"]:
        res.append((e["name"], data[pos:pos + e["part_length"]], e["raw_length"]))
        pos += e["part_length"]
    assert pos == len(data)
    return res


# ------------------------------------------------------------------------------------------------ hand-made streams
def blk(raw, *chunks):
    return raw.to_bytes(4, "big") + b"".join(len(c).to_bytes(4, "big") + c for c in chunks)


def lit(data):
    n = len(data)
    if n < 15:
        return bytes([n << 4]) + data
    r, ext = n - 15, b""
    while r >= 255:
        ext += b"\xff"; r -= 255
    return b"\xf0" + ext + bytes([r]) + data


def malformed():
    good = lit(b"hello world, hello")                      # 18 literal bytes
    cases = {
        "truncated_block_header": (blk(18, good)[:2], 18),
        "truncated_chunk_header": (blk(18, good)[:6], 18),
        "chunk_past_the_end": (blk(18, good)[:-1], 18),
        # 'a', then a match of 262,144 bytes at offset 1, then 5 literals: 262,150 bytes from a 1,038-byte chunk
        "chunk_decodes_past_262144": (blk(262150, b"\x1fa\x01\x00" + b"\xff" * 1027 + bytes([240]) + lit(b"xxxxx")), 262150),
        "block_raw_zero": (blk(0, good) + blk(18, good), 18),
        "block_sum_too_large": (blk(18, good) + blk(18, good), 30),
        "block_sum_too_small": (blk(18, good), 20),
        "trailing_bytes": (blk(18, good) + b"\x00", 18),
        "trailing_zero_block": (blk(18, good) + b"\x00\x00\x00\x00", 18),
        "over_decode": (blk(10, good), 10),
        "offset_zero": (blk(13, bytes([0x40]) + b"abcd\x00\x00" + lit(b"xxxxx")), 13),
        "offset_too_far": (blk(13, bytes([0x40]) + b"abcd\x05\x00" + lit(b"xxxxx")), 13),
        "literal_run_past_the_end": (blk(19, bytes([0xF0, 4]) + b"hello world, hello"), 19),
        "match_at_the_end": (blk(8, bytes([0x40]) + b"abcd\x04\x00"), 8),
        "short_last_literals": (blk(9, bytes([0x40]) + b"abcd\x04\x00" + lit(b"x")), 9),
        "empty_chunk": (blk(18, b""), 18),
        "chunk_over_262144": (blk(18, good)[:4] + (262145).to_bytes(4, "big") + good + bytes(262145 - len(good)), 18),
    }
    return cases

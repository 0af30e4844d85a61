"""Shared helpers of the ZStandardCodec tests: the host runs of the device codec (tezgpu_debug_zstd_*_emulate), the
system libzstd through ctypes (None where it cannot be loaded) as Hadoop's ZStandardCompressor / ZStandardDecompressor
drive it, and the committed fixture."""
import ctypes as C
import ctypes.util
import json
import os
import zlib

from tez_b200 import _lib
from tez_b200.constants import ZSTD_BLOCK_BYTES, ZSTD_FRAME_BOUND

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "zstd_segments.bin")
MANIFEST = os.path.join(GOLDEN, "zstd_segments.json")
IN_SIZE = 131072          # ZSTD_CStreamInSize(): CompressorStream's buffer with io.compression.codec.zstd.buffersize unset
MAGIC = b"\x28\xb5\x2f\xfd"

# ZSTD_cParameter values (zstd.h, stable API)
C_LEVEL, C_WINDOWLOG, C_LDM, C_CONTENTSIZE, C_CHECKSUM = 100, 101, 160, 200, 201
E_CONTINUE, E_FLUSH, E_END = 0, 1, 2


# ------------------------------------------------------------------------------------------------ device emulations
def compress_emulate(body):
    """The frames the device writer produces for one segment body."""
    L = _lib.load()
    body = bytes(body)
    cap = len(body) + 10 * (len(body) // ZSTD_BLOCK_BYTES + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_zstd_compress_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def decompress_emulate(z, body_len):
    """Decodes with the device reader's exact (serial) path; raises TezGpuError (E_FORMAT) on a malformed stream."""
    L = _lib.load()
    z = bytes(z)
    out = (C.c_uint8 * max(1, body_len))()
    n = C.c_uint64()
    _lib.check(L.tezgpu_debug_zstd_decompress_emulate(z, len(z), body_len, out, body_len, C.byref(n)))
    return bytes(out[:n.value])


def frames(z):
    """[(frame bytes, header descriptor, Frame_Content_Size or None, [(block type, block size)])] of a well-formed stream
    of Zstandard frames (no skippable ones)"""
    z, ip, res = bytes(z), 0, []
    while ip < len(z):
        assert z[ip:ip + 4] == MAGIC
        fhd = z[ip + 4]
        single, fcs_flag, did = (fhd >> 5) & 1, fhd >> 6, fhd & 3
        q = ip + 5 + (0 if single else 1) + [0, 1, 2, 4][did]
        fcs_size = [single, 2, 4, 8][fcs_flag]
        fcs = int.from_bytes(z[q:q + fcs_size], "little") + (256 if fcs_size == 2 else 0) if fcs_size else None
        q += fcs_size
        blocks = []
        while True:
            bh = int.from_bytes(z[q:q + 3], "little")
            bt, bs = (bh >> 1) & 3, bh >> 3
            blocks.append((bt, bs))
            q += 3 + (1 if bt == 1 else bs)
            if bh & 1:
                break
        q += 4 if fhd & 4 else 0
        res.append((z[ip:q], fhd, fcs, blocks))
        ip = q
    return res


# ------------------------------------------------------------------------------------------------ libzstd
_LIB = []


class _In(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _Out(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


def libzstd():
    """The system libzstd or None."""
    if not _LIB:
        name = ctypes.util.find_library("zstd") or "libzstd.so.1"
        try:
            L = C.CDLL(name)
            for f in ("ZSTD_createCCtx", "ZSTD_createDCtx"):
                getattr(L, f).restype = C.c_void_p
            for f in ("ZSTD_compressStream2", "ZSTD_decompressStream", "ZSTD_compress", "ZSTD_CCtx_setParameter",
                      "ZSTD_DStreamOutSize", "ZSTD_compressBound", "ZSTD_isError"):
                getattr(L, f).restype = C.c_size_t
            L.ZSTD_compressStream2.argtypes = [C.c_void_p, C.POINTER(_Out), C.POINTER(_In), C.c_int]
            L.ZSTD_decompressStream.argtypes = [C.c_void_p, C.POINTER(_Out), C.POINTER(_In)]
            L.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
            L.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
            L.ZSTD_compressBound.argtypes = [C.c_size_t]
            L.ZSTD_isError.argtypes = [C.c_size_t]
            L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
            L.ZSTD_freeDCtx.argtypes = [C.c_void_p]
            _LIB.append(L)
        except (OSError, AttributeError):
            _LIB.append(None)
    return _LIB[0]


def hadoop_stream(body, level=3, checksum=False, window_log=0, ldm=False, buf=IN_SIZE, oneshot=False):
    """The bytes ZStandardCodec writes for body: CompressorStream over ZStandardCompressor, one ZSTD_compressStream per
    buffer of `buf` bytes followed by a flush, ZSTD_endStream at close (no Frame_Content_Size).  oneshot: one
    ZSTD_compress frame instead (Single_Segment where it fits, with Frame_Content_Size)."""
    L = libzstd()
    body = bytes(body)
    if oneshot:
        cap = L.ZSTD_compressBound(len(body))
        out = C.create_string_buffer(cap)
        n = L.ZSTD_compress(out, cap, body, len(body), level)
        assert not L.ZSTD_isError(n)
        return out.raw[:n]
    cctx = L.ZSTD_createCCtx()
    try:
        for p, v in ((C_LEVEL, level), (C_CHECKSUM, int(checksum)), (C_WINDOWLOG, window_log), (C_LDM, int(ldm))):
            assert not L.ZSTD_isError(L.ZSTD_CCtx_setParameter(cctx, p, v))
        res = bytearray()
        obuf = C.create_string_buffer(1 << 17)

        def run(data, op):
            src = C.create_string_buffer(data, len(data)) if data else None
            inb = _In(C.cast(src, C.c_void_p) if src else None, len(data), 0)
            while True:
                outb = _Out(C.cast(obuf, C.c_void_p), len(obuf), 0)
                r = L.ZSTD_compressStream2(cctx, C.byref(outb), C.byref(inb), op)
                assert not L.ZSTD_isError(r)
                res.extend(obuf.raw[:outb.pos])
                if (op == E_CONTINUE and inb.pos == inb.size) or (op != E_CONTINUE and r == 0):
                    break

        for a in range(0, len(body), buf):
            run(body[a:a + buf], E_CONTINUE)
            run(b"", E_FLUSH)
        run(b"", E_END)
        return bytes(res)
    finally:
        L.ZSTD_freeCCtx(cctx)


def hadoop_read(z, expect):
    """DecompressorStream over ZStandardDecompressor (libzstd's streaming decoder, default parameters, frame after
    frame): the body, or None where libzstd fails, a frame is left unfinished or the output is not exactly `expect`
    bytes."""
    L = libzstd()
    z = bytes(z)
    dctx = L.ZSTD_createDCtx()
    try:
        src = C.create_string_buffer(z, len(z))
        inb = _In(C.cast(src, C.c_void_p), len(z), 0)
        obuf = C.create_string_buffer(L.ZSTD_DStreamOutSize())
        res, r = bytearray(), 0
        while True:
            outb = _Out(C.cast(obuf, C.c_void_p), len(obuf), 0)
            r = L.ZSTD_decompressStream(dctx, C.byref(outb), C.byref(inb))
            if L.ZSTD_isError(r):
                return None
            res.extend(obuf.raw[:outb.pos])
            if len(res) > expect:
                return None
            if inb.pos == inb.size and outb.pos < outb.size:
                break
        if r != 0 or len(res) != expect:
            return None
        return bytes(res)
    finally:
        L.ZSTD_freeDCtx(dctx)


def one_frame(z):
    """The blocks of device-written frames (each Single_Segment, one block) re-framed as one frame without
    Frame_Content_Size and with a 128 KiB window: the shape of a Java-written stream.  The device's blocks use no repeat
    offsets or repeated tables, so they decode the same in one frame."""
    res = bytearray(MAGIC + b"\x00" + bytes([7 << 3]))
    fr = frames(z)
    for i, (f, fhd, fcs, blocks) in enumerate(fr):
        blk = bytearray(f[(7 if fhd >> 6 else 6):])
        if i + 1 < len(fr):
            blk[0] &= 0xFE
        res += blk
    return bytes(res)


def skippable(payload):
    return (0x184D2A50 + 3).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + payload


def segment(z):
    """TIF\\x01 + stream + CRC-32 of the stream"""
    return b"TIF\x01" + bytes(z) + zlib.crc32(bytes(z)).to_bytes(4, "big")


def fixture():
    """[(name, segment bytes, rawLength)] of tests/golden/zstd_segments.bin"""
    data = open(FIXTURE, "rb").read()
    man = json.load(open(MANIFEST))
    res, pos = [], 0
    for e in man["segments"]:
        res.append((e["name"], data[pos:pos + e["part_length"]], e["raw_length"]))
        pos += e["part_length"]
    assert pos == len(data)
    return res


# ---- hand-made streams: one for every error reason
def block_header(last, bt, size):
    return (int(last) | bt << 1 | size << 3).to_bytes(3, "little")


def make_frame(content, fcs=None, checksum=None, fhd_extra=0, window=None, did=None):
    """a frame of the given block bytes; Single_Segment with a 1-byte Frame_Content_Size when fcs is given, else a
    Window_Descriptor byte (default 0: 1 KiB)"""
    fhd = fhd_extra | (4 if checksum is not None else 0) | (1 if did is not None else 0)
    h = b""
    if fcs is not None:
        fhd |= 0x20
    else:
        h += bytes([window or 0])
    if did is not None:
        h += bytes([did])
    if fcs is not None:
        h += bytes([fcs])
    return MAGIC + bytes([fhd]) + h + content + (checksum if checksum is not None else b"")


def raw_block(data, last=True):
    return block_header(last, 0, len(data)) + data


def seq_block(lit, ll_sym, of_sym, ml_sym, bits):
    """a compressed block: raw literals, one sequence with RLE tables for LL / OF / ML, and its bitstream"""
    content = bytes([len(lit) << 3]) + lit + bytes([1, 0x54, ll_sym, of_sym, ml_sym]) + bits
    return block_header(True, 2, len(content)) + content


def malformed():
    good = make_frame(raw_block(b"abcd"), fcs=4)
    return {
        # name: (stream, expected body length, reason)
        "bad_magic": (b"\x00" * 4 + good, 4, "bad frame magic"),
        "reserved_bit": (make_frame(raw_block(b"abcd"), fcs=4, fhd_extra=0x08), 4, "reserved bit set"),
        "reserved_sequence_modes": (make_frame(block_header(True, 2, 7) + bytes([0x20]) + b"abcd" + bytes([1, 0x01])), 4, "reserved bit set"),
        "dictionary_id": (make_frame(raw_block(b"abcd"), fcs=4, did=5), 4, "dictionary id set"),
        "window_too_large": (make_frame(raw_block(b"abcd"), window=18 << 3), 4, "window size over 2^27"),
        "block_type_3": (make_frame(block_header(True, 3, 4) + b"abcd", fcs=4), 4, "reserved block type"),
        "block_over_maximum": (make_frame(raw_block(b"abcdefgh"), fcs=4), 4, "block over Block_Maximum_Size"),
        "treeless_without_table": (make_frame(block_header(True, 2, 6) + bytes([0x43, 0x40, 0x00, 0x00, 0x00, 0x00])), 4,
                                   "malformed literals section"),
        "bytes_after_zero_sequences": (make_frame(block_header(True, 2, 7) + bytes([0x20]) + b"abcd" + b"\x00\x00"), 4,
                                       "malformed sequences section"),
        "sequence_bitstream_zero_last_byte": (make_frame(seq_block(b"abcd", 4, 0, 1, b"\x00")), 8, "bitstream not consumed exactly"),
        "sequence_bitstream_left_over": (make_frame(seq_block(b"abcd", 4, 0, 1, b"\x07")), 8, "bitstream not consumed exactly"),
        "offset_beyond_output": (make_frame(seq_block(b"abcd", 4, 5, 1, b"\x20")), 8, "invalid match offset"),
        "offset_zero": (make_frame(seq_block(b"abcd", 0, 1, 1, b"\x03")), 8, "invalid match offset"),
        "content_size_mismatch": (make_frame(raw_block(b"abcd"), fcs=5), 5, "decoded size differs from Frame_Content_Size"),
        "checksum_mismatch": (make_frame(raw_block(b"abcd"), fcs=4, checksum=b"\x00\x01\x02\x03"), 4, "content checksum mismatch"),
        "frames_short_of_raw_length": (good, 6, "decompressed length differs from rawLength - 4"),
        "frames_past_raw_length": (good + good, 6, "decompressed length differs from rawLength - 4"),
        "trailing_bytes": (good + b"xy", 4, "bytes after the last frame"),
        "truncated": (good[:-1], 4, "truncated frame"),
    }

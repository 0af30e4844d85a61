"""The IFile codecs the device writes and reads, one record each, and the checks and inputs their GPU tests share.

Every compressed segment a test gets from the device is checked by check_segment against its uncompressed body: the
TIF\\x01 header, the CRC-32 of the stream, the codec's decode of the stream, and byte equality with the host run of the
device writer."""
import random
import zlib
from dataclasses import dataclass
from typing import Callable, Optional

import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
import codec_model as CM
import combine_model as CBM
import lz4_model as L4
import snappy_model as SN
import zstd_model as ZS


@dataclass(frozen=True)
class Codec:
    name: str
    id: int                            # TEZGPU_CODEC_*
    hadoop: str                        # the Hadoop class name
    plugin_extra: Optional[dict]       # settings the plugin takes with it besides the class; None: refused by name
    chunk: int                         # raw bytes per chunk, block or frame of the device writer
    emulate: Callable                  # body -> the device writer's stream, run on the host
    emulated_read: Callable            # (stream, body length) -> body through the device reader, run on the host
    decode: Callable                   # (stream, body length) -> body: the decode check_segment applies
    independent: Callable              # (stream, body length) -> body through a reader that is not the device's
    segment: Callable                  # stream -> TIF\x01 + stream + CRC-32 of the stream
    zcap: Callable                     # (raw, P) -> room for a compressed file.out of at most raw uncompressed bytes
    ratio: tuple                       # test_sorter_fixed_width's bounds of compressed / uncompressed: (c2, longs)
    units: Optional[Callable] = None   # stream -> the number of blocks or frames the reader decodes one warp each

    @property
    def plugin(self):
        """the plugin configuration that selects the codec, or None"""
        if self.plugin_extra is None:
            return None
        return dict({"tez.runtime.compress": True, "tez.runtime.compress.codec": self.hadoop}, **self.plugin_extra)


def _zlib_whole(z, n):
    d = zlib.decompressobj()
    out = d.decompress(z)
    assert d.eof and not d.unused_data
    return out


def _lz4_chunks(z):
    """(block raw length, chunk) of every block of a device-written stream, walked by the headers (one chunk each)"""
    ip = 0
    while ip < len(z):
        c = int.from_bytes(z[ip + 4:ip + 8], "big")
        yield int.from_bytes(z[ip:ip + 4], "big"), z[ip + 8:ip + 8 + c]
        ip += 8 + c


def _lz4_independent(z, n):
    """the strict model, and liblz4 on every chunk where it loads"""
    out = L4.decode_stream(z, n)
    if L4.liblz4() is not None:
        got = []
        for raw, chunk in _lz4_chunks(z):
            got.append(L4.lz4_decompress_safe(chunk))
            assert got[-1] is not None and len(got[-1]) == raw
        assert b"".join(got) == out, "liblz4 and the model differ"
    return out


def _snappy_model(z, n):
    """the strict model, and libsnappy on every chunk where pyarrow imports"""
    out = SN.decode_stream(z, n)
    if SN.pyarrow() is not None:
        assert SN.decode_stream(z, n, SN.libsnappy_chunk) == out, "libsnappy and the model differ"
    return out


def _zstd_independent(z, n):
    if ZS.libzstd() is None:
        pytest.skip("libzstd is not loadable here")
    out = ZS.hadoop_read(z, n)
    assert out is not None
    return out


# The Python models decode bodies up to 4 MiB; the emulated readers (checked against the models on the CPU) decode
# larger ones.  zstd: libzstd wherever it loads.
CODECS = {c.name: c for c in [
    Codec("default", T.CODEC_DEFAULT, "org.apache.hadoop.io.compress.DefaultCodec", {}, CM.CHUNK,
          CM.deflate_emulate, CM.inflate_emulate, lambda z, n: zlib.decompress(z), _zlib_whole, CM.segment,
          lambda raw, P: raw + 5 * (raw // CM.CHUNK + P + 1) + 11 * P + 64, (1.001, 0.5)),
    Codec("lz4", T.CODEC_LZ4, "org.apache.hadoop.io.compress.Lz4Codec", {}, T.LZ4_BLOCK_BYTES,
          L4.compress_emulate, L4.decompress_emulate,
          lambda z, n: (L4.decode_stream if n <= 4 << 20 else L4.decompress_emulate)(z, n), _lz4_independent, L4.segment,
          lambda raw, P: raw + raw // 255 + 10 * (raw // L4.LZ4_BLOCK_BYTES + P + 1) + 64, (1.01, 0.75),
          lambda z: sum(1 for _ in _lz4_chunks(z))),
    Codec("zstd", T.CODEC_ZSTD, "org.apache.hadoop.io.compress.ZStandardCodec", {"io.compression.codec.zstd.level": 9},
          T.ZSTD_BLOCK_BYTES, ZS.compress_emulate, ZS.decompress_emulate,
          lambda z, n: (ZS.hadoop_read if ZS.libzstd() is not None else ZS.decompress_emulate)(z, n), _zstd_independent,
          ZS.segment, lambda raw, P: raw + 10 * (raw // ZS.ZSTD_BLOCK_BYTES + P + 1) + 64, (1.01, 0.75),
          lambda z: len(ZS.frames(z))),
    Codec("snappy", T.CODEC_SNAPPY, "org.apache.hadoop.io.compress.SnappyCodec", None, T.SNAPPY_BLOCK_BYTES,
          SN.compress_emulate, SN.decompress_emulate,
          lambda z, n: (_snappy_model if n <= 4 << 20 else SN.decompress_emulate)(z, n), _snappy_model, SN.segment,
          lambda raw, P: raw + 14 * (raw // T.SNAPPY_BLOCK_BYTES + P + 1) + 64, (1.01, 0.8), lambda z: len(SN.blocks(z))),
]}


# ------------------------------------------------------------------------------------------------ checks
def check_segment(codec, seg, body):
    """one device-written segment against its uncompressed body"""
    assert seg[:4] == b"TIF\x01"
    assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])
    assert codec.decode(seg[4:-4], len(body)) == body
    assert seg[4:-4] == codec.emulate(body), "device bytes differ from the host emulation"


def check_file(codec, out, index, exp_file, exp_index):
    """Device file.out / index with the codec against the oracle's uncompressed file.out / index."""
    out = bytes(out)
    pos = 0
    for p in range(len(exp_index)):
        s, raw, part = (int(x) for x in index[p])
        es, eraw, epart = (int(x) for x in exp_index[p])
        assert raw == eraw, p
        if epart == 0:
            assert part == 0 and s in (0, pos), p
            continue
        assert s == pos, p
        seg = out[s:s + part]
        assert len(seg) == part
        check_segment(codec, seg, exp_file[es + 4:es + epart - 4])
        pos += part
    assert pos == len(out)


def check_merged(codec, seg, raw, part, exp_ifile):
    assert part == len(seg) and raw == len(exp_ifile) - 4
    check_segment(codec, seg, exp_ifile[4:-4])


def independent_body(codec, seg, n):
    """a compressed segment's body of n bytes through a reader that is not the device's"""
    assert seg[:4] == b"TIF\x01"
    assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])
    return codec.independent(seg[4:-4], n)


# ------------------------------------------------------------------------------------------------ inputs
def key(cmp_kind, x):
    if cmp_kind == O.CMP_TEXT:
        return O.text("w%d" % x)
    if cmp_kind == O.CMP_BYTESWRITABLE:
        b = x.to_bytes(4, "big").lstrip(b"\0") * (1 + x % 3)
        return len(b).to_bytes(4, "big") + b
    if cmp_kind == O.CMP_INT:
        return O.int_writable(x - 1000)
    if cmp_kind == O.CMP_LONG:
        return O.long_writable(-x * 999983)
    return x.to_bytes(5, "big").lstrip(b"\0") or b"\0"


def records(cmp_kind, n, seed, vocab=3000):
    rng = random.Random(seed)
    return [(key(cmp_kind, min(int(rng.paretovariate(1.1)), vocab)), O.int_writable(1)) for _ in range(n)]


def fixed_kv(kind, n, seed):
    if kind == "c2":
        return O.gen_c2(0, n, seed=seed, threads=8)
    rng = np.random.default_rng(seed)
    k = np.minimum(rng.zipf(1.3, n), 1 << 20).astype(">i8").view(np.uint8).reshape(n, 8)
    v = np.ones(n, dtype=">i8").view(np.uint8).reshape(n, 8)
    return np.ascontiguousarray(np.concatenate([k, v], axis=1)).reshape(-1)


def c3(nseg, seed=3):
    segs, _ = O.gen_c3_segments(nseg, 1 << 17, seed=seed, threads=8)
    return [s.tobytes() for s in segs]


def plain(body):
    return b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")


def input_segment(codec, body, level=6):
    """(segment, rawLength) of body for a merger's input: for DefaultCodec a zlib stream of Python's zlib at level, else
    the host run of the device writer"""
    if codec.id == T.CODEC_DEFAULT:
        return CM.compressed_segment(body, level)
    return codec.segment(codec.emulate(body)), len(body) + 4


def sort_case(codec, recs, P, cmp_kind, rle=-1, send_empty=True, partition=None, combiner=0, unordered=False):
    """one collect batch through a sorter with the codec, against the oracle's uncompressed file.out"""
    kv, ko, kl, vl, vo = CBM.pack(recs)
    part_mode = T.PART_GIVEN if partition is not None else T.PART_HASH
    if combiner:
        exp = CBM.sort_combine(P, cmp_kind, combiner, kv, ko, kl, vl, partition, send_empty=send_empty)
    else:
        conf = O.sorter_conf(P, cmp_kind=cmp_kind, partitioner=part_mode, send_empty=send_empty, rle_policy=rle)
        exp = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl, partition)
    with T.GpuSorter(P, comparator=cmp_kind, partitioner=part_mode, rle_policy=rle, send_empty=send_empty,
                     combiner=combiner, codec=codec.id, unordered=unordered) as s:
        if len(recs):
            s.collect(kv, ko.astype(np.uint32), vo, vl, None if partition is None else np.asarray(partition, np.int32))
        out, index_bytes, index, st = s.flush_to_memory()
    check_file(codec, out, index, exp["file_out"], exp["index"])
    assert st["output_bytes_physical"] == st["file_out_bytes"] == len(out)
    assert st["output_bytes_with_overhead"] == int(exp["index"][:, 1].sum())
    return out, index, st


# ------------------------------------------------------------------------------------------------ malformed inputs
def malformed_inputs(codec):
    """three config-3 bodies and their input segments and rawLengths"""
    bodies = [CM.body_of(s) for s in c3(3, seed=5)]
    zs = [input_segment(codec, b) for b in bodies]
    return bodies, [z for z, _ in zs], [r for _, r in zs]


def opened(codec_id, segs, raws):
    """open a merger over segs with the codec: its counts"""
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=codec_id, raw_lens=raws) as m:
        return m.counts()

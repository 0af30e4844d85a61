"""SnappyCodec on the CPU: the device writer and reader run through their host emulations (same __host__ __device__
code) and are checked against a Python restatement of the strict reader (snappy_model) and, where pyarrow imports,
libsnappy -- the library Java's SnappyCodec reads with."""
import ctypes as C
import random

import pytest
import torch

import tez_b200 as T
from tez_b200 import _lib, native
from tez_b200._lib import TezGpuError
from oracle import tez_oracle as O
import codec_model as CM
import combine_model as CBM
import snappy_model as M

B = T.SNAPPY_BLOCK_BYTES
needs_pyarrow = pytest.mark.skipif(M.pyarrow() is None, reason=M.NO_PYARROW)


def _check_written(body, z):
    """a device-writer stream: decodes through both readers (and libsnappy), blocks of one chunk within the bound"""
    assert M.decode_stream(z, len(body)) == body
    assert M.decompress_emulate(z, len(body)) == body
    bl = M.blocks(z)
    assert len(bl) == -(-len(body) // B)
    for i, (raw, chunks) in enumerate(bl):
        assert len(chunks) == 1 and raw == (B if i + 1 < len(bl) else len(body) - B * i)
        assert len(chunks[0]) <= T.SNAPPY_CHUNK_BOUND
        if M.pyarrow():
            assert M.libsnappy_chunk(chunks[0]) == body[i * B:i * B + raw]


def test_constants_match_the_header():
    assert T.CODEC_SNAPPY == 4 and B == 65024 and T.SNAPPY_CHUNK_BOUND == 65030
    assert M.MAX_INPUT == 218422


# ------------------------------------------------------------------------------------------------ writer
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 12, 60, 61, 100, 2032, 2033, B - 1, B, B + 1, 3 * B + 7])
def test_writer_round_trip_sizes(n):
    body = (CM.wordcount_body(n=n // 8 + 10, vocab=50, seed=n) * 2)[:n]
    _check_written(body, M.compress_emulate(body))


@pytest.mark.parametrize("n", [B - 1, B, 3 * B + 11])
def test_writer_random_bytes_take_the_all_literal_form_within_the_bound(n):
    body = random.Random(n).randbytes(n)
    z = M.compress_emulate(body)
    _check_written(body, z)
    for raw, (c,) in M.blocks(z):
        assert c == M.varint(raw) + M.lit(b"\0" * raw)[:len(c) - raw - len(M.varint(raw))] + c[-raw:]
    assert max(len(c) for _, (c,) in M.blocks(z)) == (T.SNAPPY_CHUNK_BOUND if n >= B else n + 6)


def test_writer_falls_back_to_all_literal_where_the_parse_is_longer():
    """random bytes with one 4-byte repeat per slice at an offset of 2,500: each copy-2 saves 4 literal bytes but costs
    3 copy bytes and a literal tag of 3, so the parsed chunk is longer than the all-literal one, which is written"""
    body = bytearray(random.Random(3).randbytes(B))
    for s0 in range(2032, B, 2032):
        p = s0 + 1000
        body[p:p + 4] = body[p - 2500:p - 2496]
    body = bytes(body)
    z = M.compress_emulate(body)
    _check_written(body, z)
    (raw, (c,)), = M.blocks(z)
    assert c == M.varint(B) + M.lit(body) and len(c) == T.SNAPPY_CHUNK_BOUND


@pytest.mark.parametrize("b", [0, 0xFF, 0x41])
def test_writer_long_runs_split_copies_as_libsnappy(b):
    body = bytes([b]) * (2 * B + 333)
    z = M.compress_emulate(body)
    _check_written(body, z)
    assert len(z) < len(body) // 20


def test_writer_empty_body_and_determinism():
    assert M.compress_emulate(b"") == b""
    body = CM.wordcount_body(n=20000, vocab=800, seed=4)
    assert M.compress_emulate(body) == M.compress_emulate(body)


@needs_pyarrow
@pytest.mark.parametrize("name", ["wordcount", "c3", "int_long"])
def test_writer_ratio_against_libsnappy(name):
    """The device stream is at most 1.25 x libsnappy's chunks of Java's blocks on the LZ4 tests' ratio bodies."""
    body = {"wordcount": CM.wordcount_body, "c3": CM.c3_body, "int_long": CM.int_long_body}[name]()
    z = M.compress_emulate(body)
    _check_written(body, z)
    ref = sum(8 + len(M.snappy_compress(body[a:a + M.MAX_INPUT])) for a in range(0, len(body), M.MAX_INPUT))
    print("%s: device %d, libsnappy %d, ratio %.3f" % (name, len(z), ref, len(z) / ref))
    assert len(z) <= 1.25 * ref, (len(z), ref)


# ------------------------------------------------------------------------------------------------ reader
def test_fixture_checksums_and_emulated_reader():
    fx = M.fixture()
    assert [n for n, _, _ in fx][:4] == ["wordcount", "c3", "incompressible", "long_value"]
    for name, seg, raw in fx:
        assert seg[:4] == b"TIF\x01"
        body = M.decode_stream(seg[4:-4], raw - 4)
        assert M.decompress_emulate(seg[4:-4], raw - 4) == body, name
    multi = [len(ch) for _, ch in M.blocks(dict((n, s) for n, s, _ in fx)["long_value"][4:-4])]
    assert max(multi) >= 3


@needs_pyarrow
def test_model_agrees_with_libsnappy_on_the_fixture_and_libsnappy_chunks():
    n = 0
    for name, seg, raw in M.fixture():
        for _, chunks in M.blocks(seg[4:-4]):
            for c in chunks:
                assert M.decode_chunk(c) == M.libsnappy_chunk(c), name
                n += 1
    assert n >= 12
    rng = random.Random(5)
    for data in (CM.wordcount_body(n=5000, seed=2), CM.c3_body(seg_bytes=100000, seed=3), rng.randbytes(5000), b"a" * 200000):
        c = M.snappy_compress(data)
        assert M.decode_chunk(c) == data == M.libsnappy_chunk(c)


def test_crafted_chunks_have_the_elements_their_names_claim():
    tags = {name: c for name, c in M.crafted_chunks()}
    copy4 = tags["copy4"]
    assert sum(1 for i in range(len(copy4)) if copy4[i] & 3 == 3) >= 6
    assert bytes([62 << 2]) in tags["literal_tags_62_63"] and bytes([63 << 2]) in tags["literal_tags_62_63"]
    for name, c in tags.items():
        assert M.decompress_emulate(M.one_block([c]), M.preamble(c)[0]) == M.decode_chunk(c), name


MALFORMED = M.malformed()


@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_malformed_streams_fail_with_format_error(case):
    z, expect, reason = MALFORMED[case]
    with pytest.raises(M.SnappyFormatError, match=reason):
        M.decode_stream(z, expect)
    with pytest.raises(TezGpuError, match="compressed segment 0: " + reason) as e:
        M.decompress_emulate(z, expect)
    assert e.value.code == T.E_FORMAT


def test_first_error_in_stream_order_wins():
    """a walk error after a bad chunk: the chunk's reason, as the serial emulation meets it"""
    abcd = M.lit(b"abcd")
    z = M.blk(8, M.varint(8) + abcd + M.copy(0, 4, 1)) + b"\0\0"
    with pytest.raises(TezGpuError, match="invalid copy offset"):
        M.decompress_emulate(z, 16)
    z = M.blk(8, M.varint(8) + abcd + M.copy(4, 4, 1)) + b"\0\0"
    with pytest.raises(TezGpuError, match="truncated block header"):
        M.decompress_emulate(z, 16)


def _verdict(fn):
    try:
        return fn()
    except (M.SnappyFormatError, TezGpuError) as e:
        return str(e).split("compressed segment 0: ")[-1]


def test_mutants_emulation_model_and_libsnappy_agree():
    """3000 seeded mutants: the emulation and the model give the same bytes or the same reason; libsnappy (framing
    as ours) decodes the same ones to the same bytes."""
    fails = 0
    for i, (z, e) in enumerate(M.mutants(M.corpus_streams(), 3000, seed=4321)):
        emu = _verdict(lambda: M.decompress_emulate(z, e))
        mod = _verdict(lambda: M.decode_stream(z, e))
        assert emu == mod, (i, z.hex(), e)
        if M.pyarrow():
            lib = _verdict(lambda: M.decode_stream(z, e, M.libsnappy_chunk))
            assert (isinstance(lib, bytes) and lib == mod) or (isinstance(lib, str) and isinstance(mod, str)), (i, lib, mod)
        fails += isinstance(mod, str)
    assert 300 < fails < 3000


# ------------------------------------------------------------------------------------------------ entry points
@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_device_every_snappy_entry_point_fails_with_cuda_error():
    body = CM.wordcount_body(n=300, vocab=40, seed=1)
    seg, raw = M.segment(M.compress_emulate(body)), len(body) + 4
    with pytest.raises(TezGpuError, match="no CUDA device") as e:
        T.GpuSorter(4, comparator=T.CMP_TEXT, codec=T.CODEC_SNAPPY)
    assert e.value.code == T.E_CUDA
    for concat in (False, True):
        with pytest.raises(TezGpuError, match="no CUDA device") as e:
            T.GpuMerger([seg], comparator=T.CMP_TEXT, codec=T.CODEC_SNAPPY, raw_lens=[raw], concat=concat)
        assert e.value.code == T.E_CUDA
    with pytest.raises(TezGpuError, match="no CUDA device"):
        native.decode_segments([seg], [raw], T.CODEC_SNAPPY, 64 << 20)


def test_codec_argument_checks_and_bounds():
    L = _lib.load()
    assert L.tezgpu_debug_device_output_bound(4, T.CODEC_SNAPPY, 100, 10 ** 6) > 10 ** 6
    assert L.tezgpu_debug_device_output_bound(4, 5, 100, 10 ** 6) == 0
    rc = L.tezgpu_decode_segments(C.byref(native.make_conf(1)), None, None, 0, 5, 64 << 20, None, None)
    assert rc == T.E_UNSUPPORTED and "codec 5 is not decoded on the device" in L.tezgpu_last_error().decode()
    assert L.tezgpu_decode_segments(C.byref(native.make_conf(1)), None, None, 0, T.CODEC_SNAPPY, 64 << 20, None, None) in (0, T.E_CUDA)
    out = C.c_uint64()
    assert L.tezgpu_debug_snappy_compress_emulate(None, 0, None, 0, C.byref(out)) == T.E_INVALID
    assert L.tezgpu_debug_snappy_compress_emulate(b"abc", 3, (C.c_uint8 * 4)(), 4, C.byref(out)) == T.E_NOMEM
    assert L.tezgpu_debug_snappy_decompress_emulate(b"", 0, 10, (C.c_uint8 * 4)(), 4, C.byref(out)) == T.E_INVALID


@pytest.mark.parametrize("seed", range(4))
def test_bound_covers_what_the_writer_writes(seed):
    """tezgpu_debug_device_output_bound with SnappyCodec against the oracle's file.out compressed segment by segment
    with the host run of the device writer, incompressible values included"""
    rng = random.Random(seed)
    n, P = rng.choice((1, 300, 5000)), rng.choice((1, 13))
    recs = [(O.text("k%d" % rng.randrange(50)), rng.randbytes(rng.choice((0, 4, 300, 70000)) if rng.random() < 0.05 else 8))
            for _ in range(n)]
    kv, ko, kl, vl, _ = CBM.pack(recs)
    kv_bytes = int(sum(len(k) + len(v) for k, v in recs))
    res = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT, rle_policy=0), kv, ko, kl, vl)
    written = sum(8 + len(M.compress_emulate(res["file_out"][a + 4:a + part - 4])) for a, _, part in res["index"].tolist() if part)
    assert written <= _lib.load().tezgpu_debug_device_output_bound(P, T.CODEC_SNAPPY, n, kv_bytes)

"""Bounded merge with compressed output (tezgpu_merge_open_bounded_write_codec): at the floor budget and at a mid
budget, with several steps, the written file and index equal those of the one-step merge with the same codec
(tezgpu_merge_open_codec) byte for byte, the segments decode with readers independent of the device to the bounded
merge's uncompressed write, and the handle never holds more device memory than its budget."""
import ctypes as C
import os
import random
import zlib

import pytest

from oracle import tez_oracle as O
import tez_b200 as T
import lz4_model as L4
from partitioned_segments import partitioned
import snappy_model as SN
import zstd_model as ZS

pytestmark = pytest.mark.gpu

FLOOR = 16 << 20
CODECS = {"default": T.CODEC_DEFAULT, "lz4": T.CODEC_LZ4, "zstd": T.CODEC_ZSTD, "snappy": T.CODEC_SNAPPY}


def _run(segs, tmp=None, P=1, parts=None, rle=False, check_same=True, combiner=0, iterate=False, **kw):
    """written bytes (P = 1: segment, rawLength, partLength; else file.out, file.out.index, index), records, counts,
    output_bound, bounded_info (None unbounded)"""
    with T.GpuMerger(segs, partitions=parts, num_partitions=P, **kw) as m:
        if not check_same:
            m.set_check_for_same_keys(False)
        if combiner:
            m.set_combiner(combiner)
        recs = list(m.records(batch_records=997, batch_bytes=1 << 16)) if iterate else None
        if P == 1:
            seg, raw, part, _ = m.write_ifile(rle=rle)
            assert part == len(seg)
            out = (seg, raw, part)
        else:
            f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
            index, _ = m.write_partitions(f, fi, rle=rle)
            out = (open(f, "rb").read(), open(fi, "rb").read(), index.tolist())
        info = m.bounded_info() if "device_budget" in kw else None
        return out, recs, m.counts(), m.output_bound(), info


def _check(segs, codec, tmp=None, mid=4, **kw):
    """the one-step codec merge; the bounded handle at the default budget (one step) and at the floor and need // mid
    (several steps, at most the budget): the same outputs.  Returns {budget: (outputs, steps)} of the bounded runs."""
    exp = _run(segs, tmp=tmp, codec=codec, **kw)
    one = _run(segs, tmp=tmp, device_budget=0, write_codec=codec, **kw)
    assert one[4][0] == 1
    assert one[:4] == exp[:4]
    need = one[4][1]
    got = {}
    for b in sorted({FLOOR, max(FLOOR, need // mid)}, reverse=True):
        r = _run(segs, tmp=tmp, device_budget=b, write_codec=codec, **kw)
        steps, peak, _ = r[4]
        assert peak <= b, (b, peak)
        assert steps > 1, (b, need)
        assert r[0] == exp[0], b
        assert r[1] == exp[1] and r[2] == exp[2], b
        assert r[3] >= len(r[0][0])           # output_bound bounds the compressed bytes once the counts are known
        got[b] = (r[0], steps)
    return got


def _decode(codec, z, expect):
    """a compressed segment's body through a reader that is not the device's: Python zlib, or the Lz4Codec, Snappy and
    libzstd models"""
    assert z[:4] == b"TIF\x01"
    assert int.from_bytes(z[-4:], "big") == zlib.crc32(z[4:-4])
    s = z[4:-4]
    if codec == T.CODEC_DEFAULT:
        d = zlib.decompressobj()
        body = d.decompress(s)
        assert d.eof and not d.unused_data
        return body
    if codec == T.CODEC_LZ4:
        return L4.decode_stream(s, expect)
    if codec == T.CODEC_SNAPPY:
        return SN.decode_stream(s, expect)
    if ZS.libzstd() is None:
        pytest.skip("libzstd is not loadable here")
    body = ZS.hadoop_read(s, expect)
    assert body is not None
    return body


def _c3():
    segs, _ = O.gen_c3_segments(24, 160 << 10, seed=5, threads=8, id_bits=12)
    return [s.tobytes() for s in segs]


@pytest.mark.parametrize("rle", [False, True])
@pytest.mark.parametrize("name", list(CODECS))
def test_config3_text_segments_write_ifile(name, rle):
    """config-3 shape, P = 1: 24 Text-key segments of 160 KiB (REPEAT_KEY groups); the records stream as before"""
    codec = CODECS[name]
    segs = _c3()
    got = _check(segs, codec, comparator=T.CMP_TEXT, rle=rle, iterate=True)
    plain = _run(segs, comparator=T.CMP_TEXT, device_budget=FLOOR, rle=rle)[0]
    for (seg, raw, part), steps in got.values():
        assert raw == plain[1]
        assert _decode(codec, seg, raw - 4) == plain[0][4:-4]
    assert max(steps for _, steps in got.values()) >= 4


@pytest.mark.parametrize("name", list(CODECS))
def test_check_for_same_keys_off(name):
    _check(_c3(), CODECS[name], comparator=T.CMP_TEXT, rle=True, check_same=False)


@pytest.mark.parametrize("send_empty", [False, True])
@pytest.mark.parametrize("name", list(CODECS))
def test_partitions_spanning_steps_and_empty_partitions(name, send_empty, tmp_path):
    codec = CODECS[name]
    segs, parts, large = partitioned()
    kw = dict(tmp=str(tmp_path), P=16, parts=parts, send_empty=send_empty, comparator=T.CMP_BYTES)
    got = _check(segs, codec, **kw)
    (out, _, index), steps = got[FLOOR]
    assert steps >= 3 * len(large)
    plain = _run(segs, device_budget=FLOOR, **kw)[0]
    for p in range(16):
        start, raw, part = index[p]
        pstart, praw, ppart = plain[2][p]
        assert raw == praw
        if not part:
            assert not ppart and raw == 0 and send_empty
            continue
        assert _decode(codec, out[start:start + part], raw - 4) == plain[0][pstart + 4:pstart + ppart - 4]


@pytest.mark.parametrize("combiner,width", [(T.COMBINE_SUM_INT, 4), (T.COMBINE_SUM_LONG, 8)])
@pytest.mark.parametrize("name", list(CODECS))
def test_sum_combiners(name, combiner, width):
    rng = random.Random(width)
    segs = []
    for s in range(12):
        keys = sorted(rng.getrandbits(20).to_bytes(3, "big") for _ in range(rng.randint(2000, 8000)))
        segs.append(O.write_ifile([(k, rng.randint(-1000, 1000).to_bytes(width, "big", signed=True)) for k in keys])[0])
    _check(segs, CODECS[name], comparator=T.CMP_BYTES, combiner=combiner)


@pytest.mark.parametrize("name", list(CODECS))
def test_a_handle_that_fits_is_the_one_step_codec_merge(name):
    codec = CODECS[name]
    rng = random.Random(12)
    segs = []
    for s in range(10):
        keys = sorted(rng.getrandbits(64).to_bytes(8, "big") for _ in range(1000))
        segs.append(O.write_ifile([(k, bytes([s]) * 90) for k in keys])[0])
    exp = _run(segs, comparator=T.CMP_BYTES, codec=codec, iterate=True)
    for budget in (0, 256 << 20):
        got = _run(segs, comparator=T.CMP_BYTES, device_budget=budget, write_codec=codec, iterate=True)
        assert got[4][0] == 1 and got[4][1] <= (budget or 1 << 62)
        assert got[:4] == exp[:4]


@pytest.mark.parametrize("name", list(CODECS))
def test_several_steps_written_into_the_callers_buffer(name):
    codec = CODECS[name]
    segs, _ = O.gen_c3_segments(8, 256 << 10, seed=2, threads=8, id_bits=12)
    segs = [s.tobytes() for s in segs]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, device_budget=FLOOR, write_codec=codec) as m:
        exp, raw_exp, part_exp, _ = m.write_ifile()
        assert m.bounded_info()[0] > 1
        assert exp[:4] == b"TIF\x01" and part_exp == len(exp)

        def write(cap):
            buf, raw, part = (C.c_uint8 * cap)(), C.c_int64(), C.c_int64()
            rc = m.L.tezgpu_merge_write_ifile(m.h, None, C.addressof(buf), cap, 0, C.byref(raw), C.byref(part), None)
            return rc, bytes(buf), raw.value, part.value

        assert write(len(exp)) == (0, exp, raw_exp, part_exp)      # writing twice gives the same bytes
        assert write(len(exp) - 1)[0] == T.E_NOMEM
        assert m.L.tezgpu_last_error().decode() == "output buffer too small for the merged segment"
        d = __import__("torch").empty(1 << 20, dtype=__import__("torch").uint8, device="cuda")
        with pytest.raises(IOError, match="no device-resident output"):
            m.write_ifile_device(d.data_ptr(), d.numel())


def test_key_group_larger_than_the_budget_fails_with_nomem():
    segs = []
    for s in range(4):
        keys = [b"a%05d" % i for i in range(200)] + [b"hot"] * 200000 + [b"z%05d" % i for i in range(200)]
        segs.append(O.write_ifile([(k, b"0123456789") for k in keys])[0])
    for codec in CODECS.values():
        with pytest.raises(IOError, match="key group of more than"):
            with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR, write_codec=codec) as m:
                m.write_ifile()


def test_checksum_mismatch_in_the_last_window_names_the_segment():
    rng = random.Random(5)
    segs = []
    for s in range(6):
        keys = sorted(rng.getrandbits(40).to_bytes(5, "big") for _ in range(20000))
        segs.append(bytearray(O.write_ifile([(k, b"value-%d" % s) for k in keys])[0]))
    segs[4][-7] ^= 0x01                                  # a value byte of the last record: the parse still succeeds
    segs = [bytes(s) for s in segs]
    for codec in CODECS.values():
        with pytest.raises(IOError, match="checksum mismatch in segment 4"):
            with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR, write_codec=codec) as m:
                m.write_ifile()

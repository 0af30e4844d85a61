"""Bounded merge with compressed output (tezgpu_merge_open_bounded_write_codec): at the floor budget and at a mid
budget, with several steps, the written file and index equal those of the one-step merge with the same codec
(tezgpu_merge_open_codec) byte for byte, the segments decode with readers independent of the device to the bounded
merge's uncompressed write, and the handle never holds more device memory than its budget."""
import ctypes as C
import random

import pytest

from oracle import tez_oracle as O
import tez_b200 as T
from bounded_runs import FLOOR, check, run
import codec_table as CT
from partitioned_segments import partitioned

pytestmark = pytest.mark.gpu


def _c3():
    segs, _ = O.gen_c3_segments(24, 160 << 10, seed=5, threads=8, id_bits=12)
    return [s.tobytes() for s in segs]


@pytest.mark.parametrize("rle", [False, True])
@pytest.mark.parametrize("name", list(CT.CODECS))
def test_config3_text_segments_write_ifile(name, rle):
    """config-3 shape, P = 1: 24 Text-key segments of 160 KiB (REPEAT_KEY groups); the records stream as before"""
    codec = CT.CODECS[name]
    segs = _c3()
    got = check(segs, codec.id, comparator=T.CMP_TEXT, rle=rle, iterate=True)
    plain = run(segs, comparator=T.CMP_TEXT, device_budget=FLOOR, rle=rle)[0]
    for (seg, raw, part), steps in got.values():
        assert raw == plain[1]
        assert CT.independent_body(codec, seg, raw - 4) == plain[0][4:-4]
    assert max(steps for _, steps in got.values()) >= 4


@pytest.mark.parametrize("name", list(CT.CODECS))
def test_check_for_same_keys_off(name):
    check(_c3(), CT.CODECS[name].id, comparator=T.CMP_TEXT, rle=True, check_same=False)


@pytest.mark.parametrize("send_empty", [False, True])
@pytest.mark.parametrize("name", list(CT.CODECS))
def test_partitions_spanning_steps_and_empty_partitions(name, send_empty, tmp_path):
    codec = CT.CODECS[name]
    segs, parts, large = partitioned()
    kw = dict(tmp=str(tmp_path), P=16, parts=parts, send_empty=send_empty, comparator=T.CMP_BYTES)
    got = check(segs, codec.id, **kw)
    (out, _, index), steps = got[FLOOR]
    assert steps >= 3 * len(large)
    plain = run(segs, device_budget=FLOOR, **kw)[0]
    for p in range(16):
        start, raw, part = index[p]
        pstart, praw, ppart = plain[2][p]
        assert raw == praw
        if not part:
            assert not ppart and raw == 0 and send_empty
            continue
        assert CT.independent_body(codec, out[start:start + part], raw - 4) == plain[0][pstart + 4:pstart + ppart - 4]


@pytest.mark.parametrize("combiner,width", [(T.COMBINE_SUM_INT, 4), (T.COMBINE_SUM_LONG, 8)])
@pytest.mark.parametrize("name", list(CT.CODECS))
def test_sum_combiners(name, combiner, width):
    rng = random.Random(width)
    segs = []
    for s in range(12):
        keys = sorted(rng.getrandbits(20).to_bytes(3, "big") for _ in range(rng.randint(2000, 8000)))
        segs.append(O.write_ifile([(k, rng.randint(-1000, 1000).to_bytes(width, "big", signed=True)) for k in keys])[0])
    check(segs, CT.CODECS[name].id, comparator=T.CMP_BYTES, combiner=combiner)


@pytest.mark.parametrize("name", list(CT.CODECS))
def test_a_handle_that_fits_is_the_one_step_codec_merge(name):
    codec = CT.CODECS[name].id
    rng = random.Random(12)
    segs = []
    for s in range(10):
        keys = sorted(rng.getrandbits(64).to_bytes(8, "big") for _ in range(1000))
        segs.append(O.write_ifile([(k, bytes([s]) * 90) for k in keys])[0])
    exp = run(segs, comparator=T.CMP_BYTES, codec=codec, iterate=True)
    for budget in (0, 256 << 20):
        got = run(segs, comparator=T.CMP_BYTES, device_budget=budget, write_codec=codec, iterate=True)
        assert got[4][0] == 1 and got[4][1] <= (budget or 1 << 62)
        assert got[:4] == exp[:4]


@pytest.mark.parametrize("name", list(CT.CODECS))
def test_several_steps_written_into_the_callers_buffer(name):
    codec = CT.CODECS[name].id
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
    for codec in (c.id for c in CT.CODECS.values()):
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
    for codec in (c.id for c in CT.CODECS.values()):
        with pytest.raises(IOError, match="checksum mismatch in segment 4"):
            with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR, write_codec=codec) as m:
                m.write_ifile()

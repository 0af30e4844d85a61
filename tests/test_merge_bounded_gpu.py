"""Bounded-memory merge (tezgpu_merge_open_bounded): at every budget the merged stream, the written segments and the
counts equal those of the unbounded merge of the same host segments, and the handle never holds more device memory
than its budget."""
import hashlib
import os
import random
import zlib

import pytest

from oracle import tez_oracle as O
from partitioned_segments import partitioned
import tez_b200 as T

pytestmark = pytest.mark.gpu

FLOOR = 16 << 20


def _run(segs, budget=None, rle=False, check_same=True, P=1, parts=None, combiner=0, iterate=True, tmp=None, **kw):
    """records (None with a combiner), written bytes (+ index), counts, bounded_info of one merger"""
    with T.GpuMerger(segs, partitions=parts, num_partitions=P, device_budget=budget, **kw) as m:
        if not check_same:
            m.set_check_for_same_keys(False)
        if combiner:
            m.set_combiner(combiner)
        recs = list(m.records(batch_records=997, batch_bytes=1 << 16)) if iterate and not combiner else None
        if P == 1:
            seg, raw, part, _ = m.write_ifile(rle=rle)
            assert part == len(seg) == raw + 4
            out = (seg, None)
        else:
            f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
            index, _ = m.write_partitions(f, fi, rle=rle)
            out = (open(f, "rb").read(), open(fi, "rb").read(), index.tolist())
        counts = m.counts()
        info = m.bounded_info() if budget is not None else None
    return recs, out, counts, info


def _check_budgets(segs, tmp=None, fracs=(3, 20), max_upload=None, **kw):
    """default budget: one step; ~1/3 and ~1/20 of the one-step need and the floor: several steps, same output.
    max_upload: bound on the bytes uploaded per input byte in each of the two passes _run makes (iterate, write)"""
    base = _run(segs, tmp=tmp, **kw)
    one = _run(segs, budget=0, tmp=tmp, **kw)
    assert one[3][0] == 1
    assert one[:3] == base[:3]
    need = one[3][1]
    seen = []
    for b in sorted({max(FLOOR, need // f) for f in fracs} | {FLOOR}, reverse=True):
        got = _run(segs, budget=b, tmp=tmp, **kw)
        steps, peak, h2d = got[3]
        assert peak <= b, (b, peak)
        assert steps > 1, (b, need)
        assert h2d >= sum(len(s) for s in segs) * 0.9
        if max_upload is not None:
            assert h2d <= 2 * max_upload * sum(len(s) for s in segs), (b, h2d)
        assert got[0] == base[0], b
        assert got[1] == base[1], b
        assert got[2] == base[2], b
        seen.append(steps)
    return seen


@pytest.mark.parametrize("check_same", [True, False])
@pytest.mark.parametrize("rle", [False, True])
def test_config3_text_segments_at_every_budget(check_same, rle):
    """config-3 shape: 24 Text-key segments of 160 KiB, words shared by many segments (REPEAT_KEY groups)"""
    segs, _ = O.gen_c3_segments(24, 160 << 10, seed=5, threads=8, id_bits=12)
    steps = _check_budgets([s.tobytes() for s in segs], comparator=T.CMP_TEXT, rle=rle, check_same=check_same)
    assert max(steps) >= 4


def test_fixed_width_run_table_segments_with_interleaved_partitions(tmp_path):
    """fixed-width records (the run-table path) of P = 64 partitions from 3 producers: file.out and index"""
    P, G = 64, 3
    segs, parts = [], []
    for g in range(G):
        r = O.pipelined_sort_fixed(O.sorter_conf(P), O.gen_c2(g * 40000, 20000, seed=9), 16, 64)
        for p in range(P):
            start, raw, part = (int(x) for x in r["index"][p])
            if part:
                segs.append(bytes(r["file_out"][start:start + part]))
                parts.append(p)
    for fixed in ((16, 64), None):
        # only the lowest unfinished partition gets windows: the uploads stay near the input size, not P times it
        _check_budgets(segs, tmp=str(tmp_path), P=P, parts=parts, fixed=fixed, comparator=T.CMP_BYTES, max_upload=2)


@pytest.mark.parametrize("send_empty", [False, True])
def test_partitions_spanning_steps_and_empty_partitions(send_empty, tmp_path):
    """P = 16: three partitions that each span many steps at the floor, empty partitions first, inside and last; with
    send_empty_partition_details off they get the empty segment, on they get no bytes"""
    segs, parts, large = partitioned()
    steps = _check_budgets(segs, tmp=str(tmp_path), P=16, parts=parts, send_empty=send_empty, comparator=T.CMP_BYTES)
    assert steps[-1] >= 3 * len(large)               # the floor


def _rle_segments(rng, nseg, per, keyspace, header=True):
    """int keys from a small space: long REPEAT_KEY runs (steps cut next to V_END_MARKERs and inside runs)"""
    segs = []
    for s in range(nseg):
        n = rng.randint(1, per) if s % 5 else 1          # one-record segments, segments that end early
        keys = sorted(rng.randint(-keyspace, keyspace) for _ in range(n))
        seg = O.write_ifile([(O.int_writable(k), zlib.crc32(bytes([s, k & 0xFF])).to_bytes(4, "big") * (1 + k % 3))
                             for k in keys], rle=True)[0]
        segs.append(seg if header else seg[4:])
    return segs


@pytest.mark.parametrize("header", [True, False])
def test_rle_inputs_one_record_and_short_segments(header):
    rng = random.Random(11 + header)
    segs = _rle_segments(rng, 30, 6000, 400, header)
    for check_same in (True, False):
        for rle in (False, True):
            _check_budgets(segs, comparator=T.CMP_INT, has_header=header, check_same=check_same, rle=rle)


@pytest.mark.parametrize("combiner,width", [(T.COMBINE_SUM_INT, 4), (T.COMBINE_SUM_LONG, 8)])
def test_sum_combiners(combiner, width):
    rng = random.Random(width)
    segs = []
    for s in range(12):
        keys = sorted(rng.getrandbits(20).to_bytes(3, "big") for _ in range(rng.randint(2000, 8000)))
        segs.append(O.write_ifile([(k, rng.randint(-1000, 1000).to_bytes(width, "big", signed=True)) for k in keys])[0])
    _check_budgets(segs, comparator=T.CMP_BYTES, combiner=combiner)


def test_zipf_hot_key_spanning_many_segments():
    """one key makes up a sixth of every segment (9600 records in all, within what the floor budget holds): its group
    spans many windows and must not be cut"""
    rng = random.Random(3)
    segs = []
    for s in range(16):
        keys = [b"hot"] * 600 + [b"k%07d" % rng.randrange(10 ** 6) for _ in range(3000)]
        keys.sort()
        segs.append(O.write_ifile([(k, bytes([s]) * rng.randint(1, 40)) for k in keys], rle=s % 2 == 0)[0])
    for rle in (False, True):
        _check_budgets(segs, comparator=T.CMP_BYTES, rle=rle)


def test_segment_longer_than_its_window_and_long_records():
    rng = random.Random(8)
    big = sorted(rng.getrandbits(64).to_bytes(8, "big") for _ in range(60000))
    segs = [O.write_ifile([(k, k * rng.randint(1, 60)) for k in big])[0]]
    segs += [O.write_ifile([(k, b"v" * 5000) for k in sorted(rng.getrandbits(64).to_bytes(8, "big") for _ in range(300))])[0]]
    _check_budgets(segs, comparator=T.CMP_BYTES)


def test_key_group_larger_than_the_budget_fails_with_nomem():
    segs = []
    for s in range(4):
        keys = [b"a%05d" % i for i in range(200)] + [b"hot"] * 200000 + [b"z%05d" % i for i in range(200)]
        segs.append(O.write_ifile([(k, b"0123456789") for k in keys])[0])
    with pytest.raises(IOError, match="key group of more than"):
        m = T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR)
        try:
            for _ in m.records():
                pass
        finally:
            m.close()


def test_checksum_mismatch_in_the_last_window_names_the_segment():
    rng = random.Random(5)
    segs = []
    for s in range(6):
        keys = sorted(rng.getrandbits(40).to_bytes(5, "big") for _ in range(20000))
        segs.append(bytearray(O.write_ifile([(k, b"value-%d" % s) for k in keys])[0]))
    segs[4][-7] ^= 0x01                                  # a value byte of the last record: the parse still succeeds
    segs = [bytes(s) for s in segs]
    with pytest.raises(IOError, match="checksum mismatch in segment 4"):
        with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR) as m:
            assert m.bounded_info()[0] >= 1
            for _ in m.records():
                pass
    with pytest.raises(IOError, match="checksum mismatch in segment 4"):
        with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR) as m:
            m.write_ifile()


def test_device_output_and_counts_before_the_stream_on_several_steps():
    import torch
    segs, _ = O.gen_c3_segments(8, 256 << 10, seed=2, threads=8, id_bits=12)
    segs = [s.tobytes() for s in segs]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, device_budget=FLOOR) as m:
        assert m.bounded_info()[0] >= 1
        with pytest.raises(IOError, match="counts its records once"):
            m.counts()
        d = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
        with pytest.raises(IOError, match="no device-resident output"):
            m.write_ifile_device(d.data_ptr(), d.numel())
        seg, _, _, _ = m.write_ifile()
        assert m.bounded_info()[0] > 1
        n = m.counts()[0]
        assert sum(1 for _ in m.records()) == n          # the iterator starts again after a write


def test_several_steps_written_into_the_callers_buffer():
    """tezgpu_merge_write_ifile into a buffer of the caller (the wrapper writes a merge of several steps through a file):
    a buffer that fits receives the file's bytes, one a byte short fails with TEZGPU_E_NOMEM"""
    import ctypes as C
    segs, _ = O.gen_c3_segments(8, 256 << 10, seed=2, threads=8, id_bits=12)
    segs = [s.tobytes() for s in segs]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, device_budget=FLOOR) as m:
        exp, raw_exp, part_exp, _ = m.write_ifile()
        assert m.bounded_info()[0] > 1

        def write(cap):
            buf, raw, part = (C.c_uint8 * cap)(), C.c_int64(), C.c_int64()
            rc = m.L.tezgpu_merge_write_ifile(m.h, None, C.addressof(buf), cap, 0, C.byref(raw), C.byref(part), None)
            return rc, bytes(buf), raw.value, part.value

        assert write(len(exp)) == (0, exp, raw_exp, part_exp)
        assert write(len(exp) - 1)[0] == T.E_NOMEM
        assert m.L.tezgpu_last_error().decode() == "output buffer too small for the merged segment"


def test_scale_digest_equals_the_unbounded_merge():
    """about 1 GiB of config-3 segments at a 256 MiB budget"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip(f"the unbounded run needs ~24 GiB of device memory, {free >> 20} MiB free")
    segs, _ = O.gen_c3_segments(64, 16 << 20, seed=7, threads=16, id_bits=22)
    segs = [s.tobytes() for s in segs]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT) as m:
        exp = hashlib.sha256(m.write_ifile()[0]).hexdigest()
        n = m.counts()
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, device_budget=256 << 20) as m:
        got = hashlib.sha256(m.write_ifile()[0]).hexdigest()
        steps, peak, _ = m.bounded_info()
        assert m.counts() == n
    assert got == exp
    assert steps > 1 and peak <= 256 << 20


def test_one_step_decided_from_the_scanned_records():
    """1 MiB of ~100-byte records at a 64 MiB budget: too much for the one-record-per-byte shortcut, but the first
    step's windows hold every segment and the bound on their scanned records fits, so the handle is a one-step one:
    counts and device output right after open, the host segments no longer read"""
    import torch
    rng = random.Random(12)
    segs = []
    for s in range(10):
        keys = sorted(rng.getrandbits(64).to_bytes(8, "big") for _ in range(1000))
        segs.append(O.write_ifile([(k, bytes([s]) * 90) for k in keys])[0])
    base = _run(segs, comparator=T.CMP_BYTES, iterate=False)
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=64 << 20) as m:
        assert m.bounded_info()[0] == 1
        assert m.counts() == base[2]
        cap = m.output_bound()
        d = torch.empty(cap, dtype=torch.uint8, device="cuda")
        raw, part, _ = m.write_ifile_device(d.data_ptr(), cap)
        assert d[:part].cpu().numpy().tobytes() == base[1][0]
        assert m.bounded_info()[1] <= 64 << 20

"""GPU: the fixed-width emit kernels at every edge of their tile schedule (tests/emit_schedule_model.py builds the
cases): tiles per persistent group at every residue of a wave and so every position of k_emit_fast4's 4-tile and
k_emit_fast4u's 8-tile parked checksum batches; partitions of 0, 1, 2, R-1 .. 2R+1 records and runs of empty ones; a
segment of 33 R records across warps of k_crc_combine's tile array and 2^16 one-record segments; every tile lead on
first and continuation tiles, and a first-and-last tile of R records at the worst lead.

Kernels: k_emit_fast4, k_emit_fast<5, true> and k_emit<true> through sort_device_fixed (collect_fixed and unordered
handles for a few cases); k_emit_fast4u and k_emit_fast<5, false> through GpuMerger(..., fixed=...) over device
segments placed at every residue mod 16, by the run table and (after the record iterator) by explicit offsets.  Every
case asserts the planned kernel and R first, compares file.out and the index byte for byte with the stable reference
(radix_model.spill_file) or, for merges, with O.merge of every partition, and checks that a device output's bytes past
out_len keep their 0xA5 fill."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import tez_b200 as T
from tez_b200 import _lib

import emit_schedule_model as M

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
FILL = 0xA5


def _grid(kid):
    L = _lib.load()

    def groups(ntiles):
        ctas, g = C.c_uint32(), C.c_uint32()
        _lib.check(L.tezgpu_debug_emit_grid(0, kid, ntiles, C.byref(ctas), C.byref(g)))
        return ctas.value * g.value
    return groups


def _same(out, index, exp_out, exp_index, what):
    assert np.array_equal(np.asarray(index), exp_index), "%s: index differs" % what
    out = np.asarray(out)
    if out.size != exp_out.size or not np.array_equal(out, exp_out):
        m = min(out.size, exp_out.size)
        diff = np.nonzero(out[:m] != exp_out[:m])[0]
        pytest.fail("%s: file.out differs (%d vs %d bytes, %d bytes differ, first at %s)" %
                    (what, out.size, exp_out.size, diff.size, diff[0] if diff.size else "end"))


def _tail_untouched(d_out, out_len, what):
    tail = d_out[out_len:]
    assert bool((tail == FILL).all()), "%s: the emit wrote past out_len" % what


def _sort(case, rec, parts, P):
    klen, vlen = case["framing"]
    n = rec.shape[0]
    kw = dict(comparator=T.CMP_BYTES, fixed=(klen, vlen), partitioner=T.PART_GIVEN, rle_policy=T.RLE_OFF,
              send_empty=case["send_empty"], unordered=case["entry"] == "unordered")
    if case["entry"] in ("collect", "unordered"):
        with T.GpuSorter(P, **kw) as s:
            s.collect_fixed(rec.reshape(-1), parts)
            out, _, index, st = s.flush_to_memory()
        assert st["output_records"] == n
        return np.asarray(out), index
    d_kv = torch.from_numpy(rec.reshape(-1)).to(DEV) if n else torch.empty(16, dtype=torch.uint8, device=DEV)
    d_part = torch.from_numpy(parts).to(DEV) if n else torch.empty(1, dtype=torch.int32, device=DEV)
    with T.GpuSorter(P, **kw) as s:
        cap = s.device_output_bound(n, n * (klen + vlen))
        d_out = torch.full((cap + 64,), FILL, dtype=torch.uint8, device=DEV)
        out_len, index, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap, d_part.data_ptr())
    torch.cuda.synchronize()
    assert st["output_records"] == n
    _tail_untouched(d_out, out_len, case["id"])
    return d_out[:out_len].cpu().numpy(), index


def _place(segs):
    """the segments in one device buffer, segment i starting at residue i mod 16, 0xFF between them"""
    offs, at = [], 0
    for i, s in enumerate(segs):
        at = (at + 15) // 16 * 16 + i % 16
        offs.append(at)
        at += len(s)
    img = np.full(at + 64, 0xFF, dtype=np.uint8)
    for o, s in zip(offs, segs):
        img[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    buf = torch.from_numpy(img).to(DEV)
    return [(buf.data_ptr() + o, len(s)) for o, s in zip(offs, segs)], buf


def _merge(case, fr, key, parts, P):
    klen, vlen = case["framing"]
    segs, seg_part = M.merge_inputs(fr, key, parts, P)
    ptrs, keep = _place(segs)
    with T.GpuMerger(ptrs, comparator=T.CMP_BYTES, device_ptrs=True, fixed=(klen, vlen), partitions=seg_part,
                     num_partitions=P, send_empty=case["send_empty"]) as m:
        if segs:
            assert m.parse_info()[0] == 0, "records not addressed in place"
        if case["entry"] == "merge-offsets":
            # the iterator fills the per-record offsets; the write then reads the records through them (layout 1)
            assert sum(1 for _ in m.records()) == fr.shape[0]
        cap = m.output_bound()
        d_out = torch.full((cap + 64,), FILL, dtype=torch.uint8, device=DEV)
        out_len, index, st = m.write_partitions_device(d_out.data_ptr(), cap)
        torch.cuda.synchronize()
    del keep
    _tail_untouched(d_out, out_len, case["id"])
    return d_out[:out_len].cpu().numpy(), index, (segs, seg_part)


@pytest.mark.parametrize("case", M.cases(), ids=lambda c: c["id"])
def test_emit_schedule(case):
    kid, layout_, _ = M.KERNELS[case["kernel"]]
    klen, vlen = case["framing"]
    kernel, R = M.plan(klen, vlen, layout_)
    assert kernel == kid, "%s: planned kernel %d" % (case["id"], kernel)
    if case["entry"] == "merge-offsets":
        assert M.plan(klen, vlen, M.OFFSETS) == (kid, R)
    grid = _grid(kid)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cnt = M.build(case, R, grid, sms)
    rs = M.rec_size(klen, vlen)
    got = M.reached(cnt, R, rs, case["send_empty"], grid, M.BATCH.get(kid, 0))
    for k, v in M.claims(case, R, rs, grid, sms).items():
        assert (v <= got[k]) if isinstance(v, set) else got[k] == v, (case["id"], k)
    P, n = len(cnt), sum(cnt)
    seed = zlib.crc32(case["id"].encode())
    rec, key = M.records(n, klen, vlen, seed)
    parts = M.partition_ids(cnt, seed)
    fr = M.framed(rec, klen, vlen)
    if layout_ == M.PACKED:
        out, index = _sort(case, rec, parts, P)
        unordered = case["entry"] == "unordered"
        exp_out, exp_index = M.expected(fr, M.sorted_order(key, parts, unordered), parts, P, case["send_empty"], unordered)
    else:
        out, index, (segs, seg_part) = _merge(case, fr, key, parts, P)
        exp_out, exp_index = M.expected_merge(segs, seg_part, P, case["send_empty"])
    _same(out, index, exp_out, exp_index, "%s (P=%d, n=%d, R=%d, %d tiles, G=%d)" % (case["id"], P, n, R, got["T"], got["G"]))

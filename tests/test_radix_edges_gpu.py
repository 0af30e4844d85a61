"""GPU: the map-side radix sort (radix_sort.cuh, the sort phase of sorter.cuh) at the shapes where a look-back, rank,
padding or pass-selection change goes wrong, through the public entry points, against the stable host reference of
tests/radix_model.py (itself checked against the oracle by test_radix_edges_cpu.py):

- digit shapes: P = 1 and 4-byte keys, where the sort word is the key -- a constant byte at every subset of the four
  passes, all 0x00, all 0xFF, two alternating values, ascending and descending input, a lone outlier at the first or
  last slot of every tile, one all-0xFF record at the end, Zipf and uniform keys -- at n = 1, one tile -1 / 0 / +1, one
  wave of tiles +-1 and three waves + 1; the same shapes in the high word of 8-byte keys, whose ties go through the tie
  fix and the 64-bit refinement passes;
- partition widths: P = 2^k and 2^k + 1 for pbits 1..25 on ordered and unordered handles, hash and given partitions,
  fixed 4 / 8-byte and Text / BytesWritable keys, with and without empty-partition segments, also against the oracle;
- the size limit: 2^30 - 1 records sorted with every key equal and with uniform keys (checked on the device), and
  2^30 records refused by sort_device_fixed, collect_fixed and collect_batch without touching the output."""
import time

import numpy as np
import pytest
import torch

import tez_b200 as T
from oracle import tez_oracle as O
from tez_b200 import synth

import radix_model as RM

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
N_NAMES = ["1", "6143", "6144", "6145", "wave-1", "wave+1", "3wave+1"]
N_WIDTH = 50_000


def _n(name):
    if name.isdigit():
        return int(name)
    wave = RM.wave_records(torch.cuda.get_device_properties(0))
    return {"wave-1": wave - 1, "wave+1": wave + 1, "3wave+1": 3 * wave + 1}[name]


def _sort_device(rec, cmp, P=1, d_part=None, **kw):
    """sort_device_fixed of host records uint8 [n, w]; returns (file.out uint8, index, device output, out_len)"""
    n, w = rec.shape
    d_kv = torch.from_numpy(np.ascontiguousarray(rec).reshape(-1)).to(DEV)
    with T.GpuSorter(P, comparator=cmp, fixed=(w - 4, 4), rle_policy=T.RLE_OFF,
                     partitioner=T.PART_HASH if d_part is None else T.PART_GIVEN, **kw) as s:
        cap = s.device_output_bound(n, n * w)
        d_out = torch.empty(cap, dtype=torch.uint8, device=DEV)
        out_len, index, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap,
                                                 None if d_part is None else d_part.data_ptr())
    assert st["output_records"] == n
    return d_out[:out_len].cpu().numpy(), index, d_out, out_len


def _same(out, index, exp_out, exp_index, what):
    assert np.array_equal(index, exp_index), "%s: index differs" % what
    if out.size != exp_out.size or not np.array_equal(out, exp_out):
        diff = np.nonzero(out[:min(out.size, exp_out.size)] != exp_out[:min(out.size, exp_out.size)])[0]
        pytest.fail("%s: file.out differs (%d vs %d bytes, first difference at byte %s)" %
                    (what, out.size, exp_out.size, diff[0] if diff.size else "end"))


# ------------------------------------------------------------------------------------------------ digit shapes
@pytest.mark.parametrize("cmp", [O.CMP_BYTES, O.CMP_INT], ids=["bytes", "int"])
@pytest.mark.parametrize("nname", N_NAMES)
@pytest.mark.parametrize("shape", RM.SHAPES)
def test_digit_shape_4byte(shape, nname, cmp):
    n = _n(nname)
    norm = RM.shape_keys(shape, n, seed=11)
    rec = RM.fixed_records(norm, 4, cmp)
    out, index, d_out, out_len = _sort_device(rec, cmp)
    exp_out, exp_index = RM.reference_fixed(rec, cmp, 1, np.zeros(n, dtype=np.int64))
    _same(out, index, exp_out, exp_index, "%s n=%d" % (shape, n))
    if nname == "3wave+1" and cmp == O.CMP_BYTES:
        # the device checker reaches the same verdict as the reference (it alone judges the 2^30 - 1 sorts)
        assert RM.check_device(d_out, out_len, index, n, 4, cmp) == n


@pytest.mark.parametrize("nname", ["6145", "wave+1"])
@pytest.mark.parametrize("low", RM.LOW_SHAPES)
@pytest.mark.parametrize("shape", RM.SHAPES)
def test_digit_shape_8byte(shape, low, nname):
    """the high word carries the shape (the sort word at P = 1), the low word decides the ties: the tie fix for small
    groups, the 64-bit refinement passes (with trivial-pass skipping) for large ones"""
    n = _n(nname)
    cmp = O.CMP_LONG if RM.SHAPES.index(shape) % 2 else O.CMP_BYTES
    rec = RM.fixed_records(RM.shape_keys64(shape, low, n, seed=12), 8, cmp)
    out, index, _, _ = _sort_device(rec, cmp)
    exp_out, exp_index = RM.reference_fixed(rec, cmp, 1, np.zeros(n, dtype=np.int64))
    _same(out, index, exp_out, exp_index, "%s/%s n=%d" % (shape, low, n))


@pytest.mark.parametrize("shape", ["descending", "outlier_last", "alternating"])
def test_digit_shape_unordered(shape):
    """P = 1 on an unordered handle: the first pass still runs, only to reverse the collection order"""
    n = _n("wave+1")
    rec = RM.fixed_records(RM.shape_keys(shape, n, seed=13), 4, O.CMP_BYTES)
    out, index, _, _ = _sort_device(rec, O.CMP_BYTES, unordered=True)
    exp_out, exp_index = RM.reference_fixed(rec, O.CMP_BYTES, 1, np.zeros(n, dtype=np.int64), unordered=True)
    _same(out, index, exp_out, exp_index, shape)


# ------------------------------------------------------------------------------------------------ partition widths
def _sort_width_case(c, data, given):
    P, cmp = c["P"], c["cmp"]
    kw = dict(comparator=cmp, partitioner=T.PART_HASH if c["hashed"] else T.PART_GIVEN, rle_policy=T.RLE_OFF,
              send_empty=c["send_empty"], unordered=c["unordered"])
    part = None if given is None else np.ascontiguousarray(given, dtype=np.int32)
    if c["kind"] == "fixed8":
        d_part = None if part is None else torch.from_numpy(part).to(DEV)
        out, index, _, _ = _sort_device(data, cmp, P, d_part, send_empty=c["send_empty"], unordered=c["unordered"])
        return out, index
    if c["kind"] == "fixed4":
        with T.GpuSorter(P, fixed=(4, 4), **kw) as s:
            s.collect_fixed(data.reshape(-1), part)
            out, _, index, st = s.flush_to_memory()
    else:
        kv, key_off, val_off, val_len = RM.var_batch(data)
        with T.GpuSorter(P, **kw) as s:
            s.collect(kv, key_off, val_off, val_len, part)
            out, _, index, st = s.flush_to_memory()
    assert st["output_records"] == len(data)
    return np.asarray(out), index


@pytest.mark.parametrize("case", RM.width_cases(), ids=RM.case_id)
def test_partition_width(case, record_property):
    data, parts, given = RM.width_case_data(case, N_WIDTH, seed=case["P"] + 1)
    P, cmp = case["P"], case["cmp"]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out, index = _sort_width_case(case, data, given)
    record_property("sort_seconds", round(time.perf_counter() - t0, 3))
    if isinstance(data, np.ndarray):
        exp_out, exp_index = RM.reference_fixed(data, cmp, P, parts, case["send_empty"], case["unordered"])
    else:
        exp_out, exp_index = RM.reference_var(data, cmp, P, parts, None, case["send_empty"], case["unordered"])
    _same(out, index, exp_out, exp_index, RM.case_id(case))
    o_out, o_index = RM.oracle_run(data, cmp, P, given, case["send_empty"], case["unordered"])
    assert np.array_equal(index, o_index) and out.tobytes() == o_out, "%s: differs from the oracle" % RM.case_id(case)


# ------------------------------------------------------------------------------------------------ the size limit
LIMIT = RM.RADIX_MAX_N
GiB = 1 << 30
# 8 GiB of records, 10 GiB of output, 16 GiB for the two radix blocks, 1 GiB of tie flags, 0.7 GiB of look-back state;
# with every key equal, one tie group of n records adds 24 GiB of refinement arrays.  Measured on an H100 80GB HBM3
# (700 W power limit), device memory in use when the sort returned, buffers included: 69.8 GiB with equal keys, 45.7 GiB
# with uniform keys.  The test prints it.
NEED = {"equal": 72 * GiB, "uniform": 48 * GiB}


def _free_or_skip(need):
    free, _ = torch.cuda.mem_get_info(0)
    if free < need:
        pytest.skip("needs %.0f GiB free on cuda:0 for 2^30 records; %.1f GiB free" % (need / GiB, free / GiB))
    return free


def _limit_records(buf, n, kind, chunk=1 << 26):
    """fills buf (uint8 [n * 8]) with n records: 4-byte key (all 0xFFFFFFFF, or uniform), 4-byte index"""
    rows = buf.view(-1, 8)
    shifts = torch.arange(56, -8, -8, device=DEV, dtype=torch.int64)
    for a in range(0, n, chunk):
        m = min(chunk, n - a)
        i = torch.arange(a, a + m, device=DEV, dtype=torch.int64)
        key = torch.full_like(i, 0xFFFFFFFF) if kind == "equal" else synth.splitmix64(i ^ 0x5EED) & 0xFFFFFFFF
        word = (key << 32) | i
        rows[a:a + m] = ((word.unsqueeze(1) >> shifts) & 0xFF).to(torch.uint8)
        del i, key, word


def _out_cap(n):
    return n * 10 + 10 + 64   # RLE off, one partition: framing 2 + key 4 + value 4 per record, one segment


@pytest.mark.parametrize("kind", ["equal", "uniform"])
def test_limit_sort(kind):
    """2^30 - 1 records, the most one sort takes: with every key equal the last tile's inclusive look-back count is
    exactly the 30-bit state mask"""
    free0 = _free_or_skip(NEED[kind])
    d_in = torch.empty(LIMIT * 8, dtype=torch.uint8, device=DEV)
    _limit_records(d_in, LIMIT, kind)
    d_out = torch.empty(_out_cap(LIMIT), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = T.GpuSorter(1, comparator=O.CMP_BYTES, fixed=(4, 4), rle_policy=T.RLE_OFF)
    try:
        out_len, index, st = s.sort_device_fixed(d_in.data_ptr(), LIMIT, d_out.data_ptr(), d_out.numel())
        secs = time.perf_counter() - t0
        held = free0 - torch.cuda.mem_get_info(0)[0]
    finally:
        s.close()
    del d_in
    torch.cuda.empty_cache()
    assert st["output_records"] == LIMIT and out_len == LIMIT * 10 + 10
    t1 = time.perf_counter()
    assert RM.check_device(d_out, out_len, index, LIMIT, 4, O.CMP_BYTES) == LIMIT
    print("\n2^30-1 records (%s keys): sort %.2f s, device check %.1f s, %.1f GiB of device memory held by the "
          "buffers and the sorter when the sort returned" % (kind, secs, time.perf_counter() - t1, held / GiB))
    del d_out
    torch.cuda.empty_cache()


def test_limit_refusals():
    """2^30 records are refused with TEZGPU_E_INVALID before anything is read or written, with buffers of the full
    declared size: a check that regressed gives a wrong result here, not an out-of-bounds access"""
    _free_or_skip(30 * GiB)
    n = LIMIT + 1
    d_in = torch.empty(n * 8, dtype=torch.uint8, device=DEV)
    _limit_records(d_in, n, "uniform")
    d_out = torch.full((_out_cap(n),), 0xA5, dtype=torch.uint8, device=DEV)
    with T.GpuSorter(1, comparator=O.CMP_BYTES, fixed=(4, 4), rle_policy=T.RLE_OFF) as s:
        with pytest.raises(T._lib.TezGpuError, match="2\\^30-1") as e:
            s.sort_device_fixed(d_in.data_ptr(), n, d_out.data_ptr(), d_out.numel())
        assert e.value.code == T.E_INVALID
    torch.cuda.synchronize()
    assert bool((d_out == 0xA5).all()), "the refused sort wrote to the output"
    del d_in, d_out
    torch.cuda.empty_cache()

    # collect_fixed: 2^30 records at once, then one record followed by 2^30 - 1.  The host buffer is never touched when
    # the check holds (its pages stay unmapped).
    host = np.empty(n * 8, dtype=np.uint8)
    one = RM.fixed_records(np.array([0x01020304], dtype=np.uint32), 4, O.CMP_BYTES)
    with T.GpuSorter(1, comparator=O.CMP_BYTES, fixed=(4, 4), rle_policy=T.RLE_OFF) as s:
        for first, m in ((0, n), (1, LIMIT)):
            if first:
                s.collect_fixed(one.reshape(-1))
            with pytest.raises(T._lib.TezGpuError, match="2\\^30-1") as e:
                s.collect_fixed(host.ctypes.data, n=m)
            assert e.value.code == T.E_INVALID
        out, _, index, st = s.flush_to_memory()   # the refusals left the one record collected
        exp_out, exp_index = RM.reference_fixed(one, O.CMP_BYTES, 1, np.zeros(1, dtype=np.int64))
        _same(np.asarray(out), index, exp_out, exp_index, "collect_fixed after refusals")
    del host

    # collect_batch: 2^29 empty records, then 2^29 more (the handle's total would be 2^30)
    half = 1 << 29
    zeros = np.zeros(half, dtype=np.uint32)      # calloc'd: read as zero pages
    kv = np.zeros(16, dtype=np.uint8)
    with T.GpuSorter(1, comparator=O.CMP_BYTES, rle_policy=T.RLE_OFF) as s:
        s.collect(kv, zeros, zeros, zeros)
        with pytest.raises(T._lib.TezGpuError, match="2\\^30-1") as e:
            s.collect(kv, zeros, zeros, zeros)
        assert e.value.code == T.E_INVALID
    del zeros
    torch.cuda.empty_cache()

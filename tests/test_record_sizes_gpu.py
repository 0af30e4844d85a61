"""GPU: records at every vint width of their lengths, and records larger than every fixed-size piece of the path: the
emit kernels' shared-memory tile images, the window parser's 32 KiB windows, the record iterator's batch buffer and a
bounded merge's step windows.

Lengths come from L_SET, the edges of the 1- to 5-byte vints.  Every case compares the device's bytes with the oracle
(oracle/tez_oracle.py): file.out and its index with pipelined_sort / unordered_write, merged records and written segments
with merge, and every segment trailer with zlib.crc32.  Values are a function of their key, so the order inside a group
of equal keys, which the contract does not pin, cannot change a byte.

Run as a script (`python tests/test_record_sizes_gpu.py serial-walker`, with TEZGPU_PARSE_SERIAL=1) it prints the
digests of the sequential walker's merges of the window-parser inputs; the switch is latched per process, so
test_window_parser_equals_the_sequential_walker runs it in a subprocess."""
import ctypes as C
import hashlib
import json
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200._lib import KvIndex, TezGpuError  # noqa: E402
from tez_b200.runtime_library import (BYTES_WRITABLE, TEZ_BYTES_COMPARATOR, InputContext, LocalOutput,  # noqa: E402
                                      OrderedGroupedKVInput, OrderedPartitionedKVOutput, OutputContext, UnorderedKVInput)

import codec_model as CM  # noqa: E402
import lz4_model as L4  # noqa: E402
import zstd_model as ZS  # noqa: E402

pytestmark = pytest.mark.gpu

M24 = 1 << 24
L_SET = [0, 1, 127, 128, 255, 256, 65535, 65536, M24 - 1, M24, M24 + 1]
WINDOW = 32768        # the window parser's window (parse_windows.cuh PW_WINDOW)
FLOOR = 16 << 20      # TEZGPU_MERGE_BUDGET_MIN


def fill(key, n):
    """n bytes that depend on key only"""
    return np.resize(np.frombuffer(hashlib.sha256(bytes(key[:64]) + len(key).to_bytes(4, "big")).digest(), np.uint8), n).tobytes()


def serialize(cmp, content):
    if cmp == O.CMP_TEXT:
        return O.text(content)
    if cmp == O.CMP_BYTESWRITABLE:
        return len(content).to_bytes(4, "big") + content
    return content


def pack(recs):
    """[(key, value)] -> kv, key_off, key_len, val_len"""
    kl = np.array([len(k) for k, _ in recs], dtype=np.uint64)
    vl = np.array([len(v) for _, v in recs], dtype=np.uint64)
    ko = np.zeros(len(recs), dtype=np.uint64)
    ko[1:] = np.cumsum(kl + vl)[:-1]
    kv = np.frombuffer(b"".join(k + v for k, v in recs), dtype=np.uint8)
    return kv, ko, kl, vl


def check_trailers(file_out, index):
    for start, _, part in np.asarray(index).tolist():
        if part:
            seg = bytes(file_out[start:start + part])
            assert seg[:3] == b"TIF"
            assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4]), "segment at %d: trailer" % start


def size_mix(cmp, seed, n_small=3000):
    """values at every L; keys at every L up to 65536 plus one of 2^24 + 1 bytes; thousands of small records around
    them, shuffled so that tiles hold both and large headers land anywhere in an emit piece"""
    rng = random.Random(seed)
    recs = []
    for i, L in enumerate(L_SET):
        k = serialize(cmp, b"value-%02d" % i)
        recs.append((k, fill(k, L)))
    for i, L in enumerate([x for x in L_SET if x <= 65536] + [M24 + 1]):
        k = serialize(cmp, bytes([i]) + rng.randbytes(L)[1:] if L else b"")
        recs.append((k, fill(k, 1 + i % 3 * 100)))
    for _ in range(n_small):
        k = serialize(cmp, rng.randbytes(rng.randint(2, 24)))   # never the 1-byte key above
        recs.append((k, fill(k, (0, 1, 7, 80, 127, 128, 300)[zlib.crc32(k) % 7])))
    rng.shuffle(recs)
    return recs


# ------------------------------------------------------------------------------------------------ 1. variable-width sort
def _sort_case(recs, P, cmp, given, rle=T.RLE_AUTO, unordered=False):
    kv, ko, kl, vl = pack(recs)
    part = np.array([zlib.crc32(k) % P for k, _ in recs], dtype=np.int32) if given else None
    conf = O.sorter_conf(P, cmp_kind=cmp, partitioner=O.PART_GIVEN if given else O.PART_HASH, rle_policy=rle)
    exp = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl, part)
    with T.GpuSorter(P, comparator=cmp, partitioner=T.PART_GIVEN if given else T.PART_HASH, rle_policy=rle,
                     unordered=unordered) as s:
        s.collect(kv, ko, ko + kl, vl, part)
        out, index_bytes, index, st = s.flush_to_memory()
    assert bytes(out) == exp["file_out"]
    assert index_bytes == exp["index_out"]
    check_trailers(out, index)
    return exp, st


@pytest.mark.parametrize("cmp", [O.CMP_TEXT, O.CMP_BYTESWRITABLE, O.CMP_BYTES])
@pytest.mark.parametrize("P,given", [(1, False), (7, False), (7, True)])
def test_variable_width_sort_at_every_length(cmp, P, given):
    _sort_case(size_mix(cmp, seed=cmp * 10 + P + given), P, cmp, given)


@pytest.mark.parametrize("rle", [T.RLE_ON, T.RLE_OFF])
def test_repeated_large_keys_with_and_without_rle(rle):
    """three copies each of keys of 70000 bytes with values past 2^24 (REPEAT_KEY records whose value vint takes 5
    bytes, and the V_END_MARKER after them), among small repeated keys"""
    rng = random.Random(5)
    recs = []
    for i in range(2):
        k = bytes([i]) + rng.randbytes(69999)
        recs += [(k, fill(k, M24 + 1 + i))] * 3
    for _ in range(2000):
        k = rng.randbytes(3)
        recs += [(k, fill(k, 20))] * rng.randint(1, 4)
    rng.shuffle(recs)
    exp, st = _sort_case(recs, 3, O.CMP_BYTES, False, rle=rle)
    assert exp["rle_used"] == (rle == T.RLE_ON)


def test_unordered_handle_at_every_length():
    _sort_case(size_mix(O.CMP_BYTES, seed=77), 7, O.CMP_BYTES, True, unordered=True)


# ------------------------------------------------------------------------------------------------ 2. fixed-width sort
# Strides that are multiples of 16 around the source-oriented kernels' 22016-byte tile image, then 2 to 48 times it.
# With 16-byte keys the framing is vint(16) plus a 3-byte vint, or a 4-byte one from a 65536-byte value on.
STRIDES = [21968, 21984, 22000, 22016, 22032, 32768, 65552, (1 << 20) + 16]


def _fixed_records(stride, seed):
    n = max(12, min(400, (24 << 20) // stride))
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    kv = np.concatenate([np.concatenate([k, np.frombuffer(fill(k.tobytes(), stride - 16), np.uint8)]) for k in keys])
    return kv, n


def _small_partitions(n, seed):
    """partition ids in which every partition holds 1 to 3 records: P about n / 2, so tile leads take every residue"""
    rng = random.Random(seed)
    part, p = [], 0
    while len(part) < n:
        part += [p] * rng.randint(1, 3)
        p += 1
    part = part[:n]
    rng.shuffle(part)
    return np.array(part, dtype=np.int32), p


@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("many", [False, True], ids=["P1", "P_small"])
def test_fixed_width_sort_of_wide_records(stride, many):
    kv, n = _fixed_records(stride, stride)
    part, P = _small_partitions(n, stride) if many else (None, 1)
    ko = np.arange(n, dtype=np.uint64) * stride
    exp = O.pipelined_sort(O.sorter_conf(P, partitioner=O.PART_GIVEN if many else O.PART_HASH, rle_policy=0), kv, ko,
                           np.full(n, 16, np.uint32), np.full(n, stride - 16, np.uint32), part)
    pt = T.PART_GIVEN if many else T.PART_HASH
    with T.GpuSorter(P, fixed=(16, stride - 16), partitioner=pt, rle_policy=T.RLE_OFF) as s:
        s.collect_fixed(kv, partition=part)
        out, index_bytes, index, _ = s.flush_to_memory()
    assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]
    check_trailers(out, index)
    # the same records from device memory
    d_kv = torch.from_numpy(kv.copy()).to("cuda:0")
    d_part = torch.from_numpy(part).to("cuda:0") if many else None
    cap = kv.size + 12 * n + 10 * P + 64
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda:0")
    with T.GpuSorter(P, fixed=(16, stride - 16), partitioner=pt, rle_policy=T.RLE_OFF) as s:
        ln, index, _ = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap,
                                           d_part.data_ptr() if many else None)
    assert d_out[:ln].cpu().numpy().tobytes() == exp["file_out"]
    assert index.tolist() == exp["index"].tolist()


# ------------------------------------------------------------------------------------------------ 3. fixed-width merge
# (klen, vlen) with framings of 2 to 10 bytes, then the strides of the fixed-width sort
FRAMINGS = [(16, 64), (16, 128), (16, 256), (16, 65536), (128, 65536), (256, 65536), (65536, 65536), (65536, M24),
            (M24, M24)] + [(16, s - 16) for s in STRIDES]


def _fixed_segments(kl, vl, nseg, seed):
    stride = kl + vl
    n = 2 if stride >= M24 else max(3, min(300, (12 << 20) // stride))
    rng = np.random.default_rng(seed)
    segs = []
    for _ in range(nseg):
        keys = [rng.bytes(kl) for _ in range(n)]
        kv = np.frombuffer(b"".join(k + fill(k, vl) for k in keys), dtype=np.uint8)
        segs.append(O.pipelined_sort_fixed(O.sorter_conf(1, rle_policy=0), kv, kl, vl)["file_out"])
    return segs


def _place_odd(segs):
    """the segments back to back in one device buffer from offset 3, with odd gaps of 0xFF bytes"""
    offs, at = [], 3
    for s in segs:
        offs.append(at)
        at += len(s) + 5
    img = np.full(at + 64, 0xFF, dtype=np.uint8)
    for o, s in zip(offs, segs):
        img[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    buf = torch.from_numpy(img).to("cuda:0")
    return [(buf.data_ptr() + o, len(s)) for o, s in zip(offs, segs)], buf


def _merge_all(segs, **kw):
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, **kw) as m:
        mode = m.parse_info()[0]
        seg = m.write_ifile(rle=False)[0]
        cap = m.output_bound()
        d = torch.empty(cap + 16, dtype=torch.uint8, device="cuda:0")
        n, index, _ = m.write_partitions_device(d.data_ptr(), cap)
        dev = d[:n].cpu().numpy().tobytes()
        recs = list(m.records())
    return mode, seg, dev, index, recs


@pytest.mark.parametrize("kl,vl", FRAMINGS)
def test_fixed_width_merge_at_every_framing_length(kl, vl):
    segs = _fixed_segments(kl, vl, 2, kl * 7 + vl)
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    host = _merge_all(segs, fixed=(kl, vl))
    ptrs, keep = _place_odd(segs)
    dev = _merge_all(ptrs, fixed=(kl, vl), device_ptrs=True)
    del keep
    for got in (host, dev):
        mode, seg, written, index, recs = got
        assert mode == 0, "records not addressed in place"
        assert seg == exp["ifile"] and written == seg
        check_trailers(written, index)
        assert recs == exp["records"]


# ------------------------------------------------------------------------------------------------ 4. window parser
SPANS = [1, 31, 32, 33, 600]          # windows a record's value covers
KINDS = ["random", "zeros", "ones", "ifile"]


def _value_bytes(kind, n, seed):
    if kind == "random":
        return np.random.default_rng(seed).bytes(n)
    if kind == "zeros":
        return bytes(n)
    if kind == "ones":
        return b"\xff" * n
    # a well-formed IFile body: every window inside the value guesses a plausible exit
    body = O.write_ifile([(b"w%05d" % i, b"v" * (i % 40)) for i in range(800)])[0][4:-6]
    return (body * (n // len(body) + 1))[:n]


def walker_inputs(kind):
    """Two segments of one merge.  Segment 0 holds records whose values span SPANS windows, and for every header width
    2..6 (a 1-byte key vint and a 1- to 5-byte value vint) records whose header starts 0..width bytes before a window
    edge (windows start at the body, after the 4-byte segment header); segment 1 interleaves small records."""
    recs, pos, key_no = [], 0, 0

    def add(vlen):
        nonlocal pos, key_no
        k = b"%07d" % key_no
        key_no += 1
        v = _value_bytes(kind, vlen, key_no)
        recs.append((k, v))
        pos += len(O.vint(len(k))) + len(O.vint(vlen)) + len(k) + vlen

    def pad_to(target):
        """one filler record that ends at body offset target (at least 20 bytes away)"""
        gap = target - pos
        while gap < 20:
            gap += WINDOW
        for hv in (1, 2, 3):
            vlen = gap - 1 - hv - 7
            if len(O.vint(vlen)) == hv and vlen >= 0:
                add(vlen)
                return
        raise AssertionError(gap)

    for s in SPANS:
        add(s * WINDOW - 100 + s)
    for vw, vlen in ((1, 100), (2, 200), (3, 40000), (4, 70000), (5, M24 + 1)):
        hw = 1 + vw
        for back in (range(hw + 1) if vw < 5 else (0, 1, 3, 6)):
            edge = (pos // WINDOW + 2) * WINDOW
            pad_to(edge - back)
            assert pos == edge - back
            add(vlen)
    seg0 = O.write_ifile(recs)[0]
    rng = random.Random(len(kind))
    small = sorted(b"%07d" % rng.randrange(key_no) + b"x" for _ in range(3000))
    seg1 = O.write_ifile([(k, fill(k, rng.randint(0, 300))) for k in small])[0]
    return [seg0, seg1]


def _digest(recs):
    h = hashlib.sha256()
    for k, v, same in recs:
        h.update(len(k).to_bytes(4, "big") + k + len(v).to_bytes(4, "big") + v + bytes([same]))
    return h.hexdigest()


def walker_digests(expect_mode):
    out = {}
    for kind in KINDS:
        segs = walker_inputs(kind)
        with T.GpuMerger(segs, comparator=T.CMP_BYTES) as m:
            assert m.parse_info()[0] == expect_mode, kind
            seg = m.write_ifile()[0]
            out[kind] = [_digest(m.records()), hashlib.sha256(seg).hexdigest()]
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_window_parser_on_records_spanning_many_windows(kind):
    segs = walker_inputs(kind)
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    mode, seg, written, index, recs = _merge_all(segs)
    assert mode == 1
    assert seg == exp["ifile"] == written
    check_trailers(written, index)
    assert recs == exp["records"]


def test_window_parser_equals_the_sequential_walker():
    env = dict(os.environ, TEZGPU_PARSE_SERIAL="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "serial-walker"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    serial = json.loads(r.stdout.strip().splitlines()[-1])
    assert serial == walker_digests(1)


# ------------------------------------------------------------------------------------------------ 5. iterator contract
def _big_record_segments(big):
    """three segments of small records; the first record of the stream is (key, value) of `big` value bytes"""
    rng = random.Random(big)
    segs = []
    for s in range(3):
        keys = sorted(b"k%06d" % rng.randrange(10 ** 6) + bytes([s]) for _ in range(2000))
        recs = [(k, fill(k, rng.randint(0, 200))) for k in keys]
        if s == 1:
            recs.insert(0, (b"a-big", fill(b"a-big", big)))
        segs.append(O.write_ifile(recs)[0])
    return segs


def _next_batch(m, buf_bytes, cap, idx_cap):
    buf = np.empty(max(1, buf_bytes), dtype=np.uint8)
    idx = (KvIndex * max(1, idx_cap))()
    n = C.c_uint32(77)
    rc = m.L.tezgpu_merge_next_batch(m.h, buf.ctypes.data, cap, idx, idx_cap, C.byref(n))
    recs = [(buf[e.key_off:e.key_off + e.key_len].tobytes(), buf[e.val_off:e.val_off + e.val_len].tobytes(),
             bool(e.same_key)) for e in idx[:n.value]] if rc == 0 else None
    return rc, n.value, idx, recs


@pytest.mark.parametrize("handle", ["merge", "concat", "bounded"])
def test_next_batch_reports_a_record_larger_than_the_batch(handle):
    big = 20 << 20
    segs = _big_record_segments(big)
    kw = {"concat": True} if handle == "concat" else {"device_budget": 256 << 20} if handle == "bounded" else {}
    if handle == "concat":
        segs = [segs[1], segs[0], segs[2]]        # the big record first in (segment, position) order
        exp = [(k, v, False) for s in segs for _, k, v in O.read_ifile(s)]
    else:
        exp = O.merge(segs, O.CMP_BYTES, factor=100)["records"]
    need = len(exp[0][0]) + len(exp[0][1])
    assert need == 5 + big
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, **kw) as m:
        for _ in range(2):           # the stream does not move
            rc, n, idx, _ = _next_batch(m, 1 << 20, need - 1, 1 << 10)
            assert (rc, n) == (T.E_NOMEM, 0)
            assert (idx[0].key_len, idx[0].val_len) == (5, big)
        rc, n, idx, _ = _next_batch(m, 1 << 20, need - 1, 1)
        assert (rc, n, idx[0].key_len, idx[0].val_len) == (T.E_NOMEM, 0, 5, big)
        rc, n, _, recs = _next_batch(m, need, need, 1)             # exactly its bytes, one index entry
        assert (rc, n) == (0, 1) and recs == exp[:1]
        rest = sum(len(k) + len(v) for k, v, _ in exp[1:])
        rc, n, _, recs = _next_batch(m, rest, 1 << 40, len(exp))   # a cap past 2^32 counts as 2^32 - 1
        assert rc == 0 and recs == exp[1:]
        assert _next_batch(m, 16, 16, 4)[:2] == (0, 0)
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, **kw) as m:
        assert list(m.records()) == exp                             # default batch of 16 MiB grows to fit


# ------------------------------------------------------------------------------------------------ 6. bounded merge
def _bounded_inputs():
    """four segments of 24 MiB of 2 KiB records; the third holds a 40 MiB record in the middle of its key range"""
    rng = random.Random(40)
    segs = []
    for s in range(4):
        keys = sorted(rng.randbytes(8) for _ in range(12000))
        recs = [(k, fill(k, 1024 + zlib.crc32(k) % 2048)) for k in keys]
        if s == 2:
            k = b"\x80" + bytes(7)
            recs.append((k, fill(k, 40 << 20)))
            recs.sort(key=lambda r: r[0])
        segs.append(O.write_ifile(recs)[0])
    return segs


def test_bounded_merge_with_a_40_mib_record():
    segs = _bounded_inputs()
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    with T.GpuMerger(segs, comparator=T.CMP_BYTES) as m:
        base = (list(m.records()), m.write_ifile()[0])
    assert base[1] == exp["ifile"] and base[0] == exp["records"]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=0) as m:
        assert (list(m.records()), m.write_ifile()[0]) == base
        assert m.bounded_info()[0] == 1
    # Windows of about 35 MiB a segment: the 64 MiB segment is not held whole, and the window that starts at the 40 MiB
    # record holds no complete record until it has doubled.  The step that merges it needs about 5 bytes per byte of
    # it (DESIGN section 3), within the budget.
    budget = 576 << 20
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=budget) as m:
        got = (list(m.records(batch_records=997, batch_bytes=1 << 16)), m.write_ifile()[0])
        steps, peak, _ = m.bounded_info()
    assert steps > 1 and peak <= budget, (steps, peak, budget)
    assert got == base
    with pytest.raises(TezGpuError, match=r"does not fit the device budget of \d+ bytes") as e:
        with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=FLOOR) as m:
            for _ in m.records():
                pass
    assert e.value.code == T.E_NOMEM


# ------------------------------------------------------------------------------------------------ 7. codecs
def _decode(codec, z, body_len):
    if codec == T.CODEC_DEFAULT:
        return CM.hadoop_inflate(z)
    if codec == T.CODEC_LZ4:
        return L4.decompress_emulate(z, body_len)
    return ZS.decompress_emulate(z, body_len)


@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_compressed_partitions_with_a_value_past_2_24(codec):
    rng = random.Random(codec)
    recs = []
    for i, big in enumerate((bytes(M24 + 1), rng.randbytes(M24 + 1))):   # stored / raw blocks for the random one
        k = b"big-%d" % i
        recs.append((k, big))
    for _ in range(3000):
        k = rng.randbytes(rng.randint(1, 12))
        recs.append((k, fill(k, zlib.crc32(k) % 100)))
    kv, ko, kl, vl = pack(recs)
    P = 3
    exp = O.pipelined_sort(O.sorter_conf(P), kv, ko, kl, vl)
    with T.GpuSorter(P, codec=codec) as s:
        s.collect(kv, ko, ko + kl, vl)
        out, _, index, _ = s.flush_to_memory()
    out = bytes(out)
    check_trailers(out, index)
    segs, raws, plain = [], [], []
    for p in range(P):
        start, raw, part = (int(x) for x in index[p])
        e_start, e_raw, e_part = (int(x) for x in exp["index"][p])
        assert raw == e_raw
        seg, eseg = out[start:start + part], exp["file_out"][e_start:e_start + e_part]
        assert seg[:4] == b"TIF\x01"
        assert _decode(codec, seg[4:-4], raw - 4) == eseg[4:-4]
        segs.append(seg)
        raws.append(raw)
        plain.append(eseg)
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        exp_recs = list(m.records())
    assert exp_recs == O.merge(plain, O.CMP_BYTES, factor=100)["records"]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=codec, raw_lens=raws) as m:
        assert list(m.records()) == exp_recs


# ------------------------------------------------------------------------------------------------ 8. plugin mirror
MIB = 1 << 20


def _mirror_records():
    rng = random.Random(8)
    recs = []
    for size in (9 * MIB, 20 * MIB, 9 * MIB + 1):
        k = rng.randbytes(16)
        recs.append((k, fill(k, size)))
    for _ in range(300):
        k = rng.randbytes(16)
        recs.append((k, fill(k, rng.randint(0, 500))))
    rng.shuffle(recs)
    return recs


@pytest.mark.parametrize("sort_mb", [256, 4], ids=["one_spill", "final_merge"])
def test_plugin_mirror_end_to_end_with_records_of_9_and_20_mib(tmp_path, sort_mb):
    P = 2
    recs = _mirror_records()
    conf = {"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
            "tez.runtime.io.sort.mb": sort_mb}
    ctx = OutputContext(conf, str(tmp_path / "m"), total_memory_available_to_task=1 << 30)
    out = OrderedPartitionedKVOutput(ctx, P)
    out.initialize()
    out.start()
    w = out.getWriter()
    for k, v in recs:
        w.write(k, v)
    out.close()
    assert (out.num_spills == 1) == (sort_mb == 256)
    kv, ko, kl, vl = pack(recs)
    exp = O.pipelined_sort(O.sorter_conf(P), kv, ko, kl, vl)
    assert open(out.final_output_file, "rb").read() == exp["file_out"]
    assert open(out.final_index_file, "rb").read() == exp["index_out"]
    for p in range(P):
        mine = sorted((k, v) for k, v in recs if O.partition_of(O.CMP_BYTES, k, P) == p)
        inp = OrderedGroupedKVInput(InputContext(conf, str(tmp_path / ("r%d" % p))), 1)
        inp.initialize()
        inp.start()
        inp.handleEvents([LocalOutput(0, out.final_output_file, out.final_index_file, p)])
        r = inp.getReader()
        groups = []
        while r.next():
            groups.append((r.getCurrentKey(), list(r.getCurrentValues())))
        assert groups == [(k, [v]) for k, v in mine]
        u = UnorderedKVInput(InputContext(conf, str(tmp_path / ("u%d" % p))), 1)
        u.initialize()
        u.start()
        u.handleEvents([LocalOutput(0, out.final_output_file, out.final_index_file, p)])
        r = u.getReader()
        got = []
        while r.next():
            got.append((r.getCurrentKey(), r.getCurrentValue()))
        assert got == mine


if __name__ == "__main__":
    if sys.argv[1:] == ["serial-walker"]:
        print(json.dumps(walker_digests(2)))
    else:
        sys.exit("usage: test_record_sizes_gpu.py serial-walker")

"""The device codec writers on the crafted partition bodies of codec_writer_cases: one-step sorts and merges of one
record per partition (every third partition empty, in orders that put one-chunk and many-chunk segments side by side),
4,096 partitions of which most have no segment, and the output bound.  Every segment is checked against the same write
without a codec (index triple), for its header and CRC-32, byte for byte against the host run of the writer, through a
reader that is not the device's and through the device reader."""
import os
import zlib

import numpy as np
import pytest
import torch

import tez_b200 as T
from tez_b200 import native
from tez_b200._lib import TezGpuError
from oracle import tez_oracle as O
import codec_table as CT
import codec_writer_cases as W
import combine_model as CM

pytestmark = pytest.mark.gpu
BUDGET = 16 << 30
SENTINEL = 0xA5
_STREAM = {}


def _stream(codec, body):
    """the host run of the writer on body, decoded once by an independent reader"""
    key = (codec.name, body)
    if key not in _STREAM:
        z = codec.emulate(body)
        assert codec.independent(z, len(body)) == body
        _STREAM[key] = z
    return _STREAM[key]


def _layout(cases, order):
    """partition bodies in order, every third partition empty: (P, records [(key, value)], partition ids, bodies)"""
    seq = [cases[i] for i in order]
    bodies, recs, parts = [], [], []
    p = 0
    while seq:
        if p % 3 == 2:
            bodies.append(None)
        else:
            c = seq.pop(0)
            bodies.append(c.body)
            if c.rec is not None:
                recs.append(c.rec)
                parts.append(p)
        p += 1
    return p, recs, parts, bodies


def _orders(cases, chunk):
    n = len(cases)
    small = [i for i in range(n) if cases[i].length <= chunk]
    big = [i for i in range(n) if cases[i].length > chunk]
    alt = []
    for k in range(max(len(small), len(big))):
        alt += ([small[k]] if k < len(small) else []) + ([big[k]] if k < len(big) else [])
    return {"forward": list(range(n)), "reversed": list(range(n))[::-1], "alternating": alt}


def check_file(codec, out, index, plain, pindex, bodies=None):
    """file.out / index with the codec against the same write without it; bodies[p]: the body partition p must hold"""
    out, plain = bytes(out), bytes(plain)
    pos, segs, raws, want = 0, [], [], []
    for p in range(len(pindex)):
        s, raw, part = (int(x) for x in index[p])
        ps, praw, ppart = (int(x) for x in pindex[p])
        assert raw == praw, p
        if ppart == 0:
            assert part == 0 and s in (0, pos), p
            continue
        assert s == pos, p
        pos += part
        seg = out[s:s + part]
        body = plain[ps + 4:ps + ppart - 4]
        assert raw == len(body) + 4
        if bodies is not None:
            assert body == (bodies[p] or W.EOF_MARKER), p
        assert seg[:4] == b"TIF\x01", p
        assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4]), p
        assert seg[4:-4] == _stream(codec, body), "partition %d: device bytes differ from the host emulation" % p
        segs.append(seg)
        raws.append(raw)
        want.append(body)
    assert pos == len(out)
    imgs, _ = native.decode_segments(segs, raws, codec.id, BUDGET)
    for i, (img, body) in enumerate(zip(imgs, want)):
        assert img[4:-4] == body, "the device reader's body of segment %d" % i
    return len(segs)


def _sort(P, recs, parts, codec, send_empty):
    kv, ko, kl, vl, vo = CM.pack(recs)
    with T.GpuSorter(P, comparator=T.CMP_BYTES, partitioner=T.PART_GIVEN, rle_policy=T.RLE_OFF, send_empty=send_empty,
                     codec=codec) as s:
        if recs:
            s.collect(kv, ko.astype(np.uint32), vo, vl, np.asarray(parts, np.int32))
        out, _, index, st = s.flush_to_memory()
        assert len(out) <= s.output_bound()
    return bytes(out), index.copy(), st


@pytest.mark.parametrize("send_empty", [False, True])
@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_sorter_crafted_partitions(name, send_empty):
    g = W.GEOMETRY[name]
    cases = W.cases(g)
    for oname, order in _orders(cases, g.chunk).items():
        P, recs, parts, bodies = _layout(cases, order)
        plain, pindex, _ = _sort(P, recs, parts, T.CODEC_NONE, send_empty)
        out, index, st = _sort(P, recs, parts, g.codec, send_empty)
        assert st["file_out_bytes"] == len(out)
        nseg = check_file(CT.CODECS[name], out, index, plain, pindex, None if send_empty else bodies)
        assert nseg == len(recs) + (0 if send_empty else P - len(recs)), oname


def _merge(segs, parts, P, codec, send_empty, tmp):
    with T.GpuMerger(segs, partitions=parts, num_partitions=P, comparator=T.CMP_BYTES, send_empty=send_empty,
                     codec=codec) as m:
        f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
        index, _ = m.write_partitions(f, fi, rle=False)
        return open(f, "rb").read(), np.asarray(index).copy()


@pytest.mark.parametrize("send_empty", [False, True])
@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_merger_crafted_partitions(name, send_empty, tmp_path):
    """one input segment per partition (the empty bodies as segments without records), one-step merge with the codec"""
    g = W.GEOMETRY[name]
    cases = W.cases(g)
    P, _, _, bodies = _layout(cases, _orders(cases, g.chunk)["alternating"])
    segs, parts = [], []
    for p, b in enumerate(bodies):
        if b is not None:
            c = [O.read_ifile(b"TIF\x00" + b + zlib.crc32(b).to_bytes(4, "big"))]
            segs.append(O.write_ifile([(k, v) for _, k, v in c[0]], rle=False)[0])
            assert segs[-1][4:-4] == b
            parts.append(p)
    plain, pindex = _merge(segs, parts, P, T.CODEC_NONE, send_empty, str(tmp_path))
    out, index = _merge(segs, parts, P, g.codec, send_empty, str(tmp_path))
    check_file(CT.CODECS[name], out, index, plain, pindex, None if send_empty else bodies)


@pytest.mark.parametrize("which", ["all", "first", "last"])
@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_many_partitions(name, which):
    """P = 4,096: one tiny record in every partition, or only in the first or the last: the chunk -> partition search
    at depth 12, and segment ranks far from partition numbers"""
    g = W.GEOMETRY[name]
    P = 4096
    live = {"all": range(P), "first": [0], "last": [P - 1]}[which]
    recs = [(b"k%d" % (p % 7), b"v" * (p % 5)) for p in live]
    parts = list(live)
    for send_empty in (False, True):
        plain, pindex, _ = _sort(P, recs, parts, T.CODEC_NONE, send_empty)
        out, index, _ = _sort(P, recs, parts, g.codec, send_empty)
        check_file(CT.CODECS[name], out, index, plain, pindex)


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=dtype))).cuda()


@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_output_bound_and_exact_capacity(name):
    """incompressible bodies of a chunk and one byte, and many one-byte-value partitions: the bytes written are within
    both bounds; sort_device into exactly that many bytes succeeds, into one byte less fails with E_NOMEM and writes
    nothing"""
    g = W.GEOMETRY[name]
    recs, parts = [], []
    for i in range(6):
        recs.append(W.make_case(g, "random", g.chunk + 1, seed=i).rec)
        parts.append(2 * i)
    for i in range(200):
        recs.append(W.make_case(g, "one_value", 100 + 7 * i).rec)
        parts.append(12 + i)
    P = 12 + 200 + 3
    plain, pindex, _ = _sort(P, recs, parts, T.CODEC_NONE, False)
    out, index, _ = _sort(P, recs, parts, g.codec, False)
    check_file(CT.CODECS[name], out, index, plain, pindex)
    kv, ko, kl, vl, vo = CM.pack(recs)
    kv = np.concatenate([kv, np.zeros(64, np.uint8)])
    kv_bytes = int(ko[-1]) + int(kl[-1]) + int(vl[-1])
    d_kv, d_ko, d_vo = _dev(kv, np.uint8), _dev(ko, np.int64), _dev(ko + kl, np.int64)
    d_vl, d_part = _dev(vl, np.int32), _dev(parts, np.int32)
    n = len(recs)

    def run(cap):
        with T.GpuSorter(P, comparator=T.CMP_BYTES, partitioner=T.PART_GIVEN, rle_policy=T.RLE_OFF, send_empty=False,
                         codec=g.codec) as s:
            bound = s.device_output_bound(n, kv_bytes)
            cap = bound if cap is None else cap
            d_out = torch.full((cap + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
            try:
                ln, idx, _ = s.sort_device(d_kv.data_ptr(), kv_bytes, d_ko.data_ptr(), d_vo.data_ptr(), d_vl.data_ptr(), n,
                                           d_out.data_ptr(), cap, d_part.data_ptr())
            except TezGpuError as e:
                assert bool((d_out[cap:] == SENTINEL).all()), "bytes written past the capacity"
                return e, bound, None
            assert bool((d_out[ln:] == SENTINEL).all()), "bytes written past out_len"
            return (d_out[:ln].cpu().numpy().tobytes(), idx), bound, None

    (got, idx), bound, _ = run(None)
    assert got == out and np.array_equal(idx, index)
    assert len(out) <= bound
    (got, idx), _, _ = run(len(out))
    assert got == out and np.array_equal(idx, index)
    e, _, _ = run(len(out) - 1)
    assert isinstance(e, TezGpuError) and e.code == T.E_NOMEM

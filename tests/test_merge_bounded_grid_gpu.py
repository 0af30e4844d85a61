"""Bounded merges whose step cuts all fall on a codec's chunk grid.  A step cuts between records, so when every record's
framed size vint(kl) vint(vl) key value is exactly one chunk, every piece of a partition body ends on the grid: an open
piece keeps exactly one chunk as its carry, and that whole chunk is copied in front of the partition's next piece.
Framed sizes of a chunk less or more one byte move the carry by one byte per record, half a chunk puts every other cut
on the grid.  Each write is checked against the one-step codec merge byte for byte, decoded by readers independent of
the device, and without a codec against the unbounded merge."""
import random
import zlib

import pytest

from oracle import tez_oracle as O
import tez_b200 as T
from bounded_runs import FLOOR, check, run
import codec_table as CT

pytestmark = pytest.mark.gpu
INPUT_BYTES = 12 << 20


def _value_len(size, kl=8):
    """the value length whose record vint(kl) vint(vl) key value frames to exactly size bytes"""
    for w in range(1, 6):
        vl = size - 1 - kl - w
        if vl >= 0 and len(O.vint(vl)) == w:
            return vl
    raise AssertionError(size)


def _segments(size, nseg, parts, seed):
    """nseg sorted segments of records framing to `size` bytes each (unique 8-byte keys; values half compressible,
    half random), about INPUT_BYTES in all; segment s belongs to partition parts[s % len(parts)]"""
    rng = random.Random(seed)
    vl = _value_len(size)
    n = INPUT_BYTES // size
    keys = sorted(rng.sample(range(1 << 62), n))
    segs = [[] for _ in range(nseg)]
    for i, k in enumerate(keys):
        if i % 2:
            v = rng.randbytes(vl)
        else:
            v = (b"value-%d-" % i * (vl // 8 + 1))[:vl]
        rec = (k.to_bytes(8, "big"), v)
        assert len(O.vint(8) + O.vint(vl)) + 8 + vl == size
        segs[rng.randrange(nseg)].append(rec)
    return [O.write_ifile(s, rle=False)[0] for s in segs], [parts[s % len(parts)] for s in range(nseg)], [len(s) for s in segs]


def _grid_case(name, factor, P, send_empty, tmp):
    """name: a codec of codec_table, or "none" for the write without a codec"""
    c = CT.CODECS.get(name)
    codec = c.id if c else T.CODEC_NONE
    chunk = c.chunk if c else 65024
    size = {"chunk": chunk, "chunk-1": chunk - 1, "chunk+1": chunk + 1, "half": chunk // 2}[factor]
    parts = [0] if P == 1 else [0, 2, 3]
    segs, seg_parts, counts = _segments(size, 5, parts, seed=zlib.crc32(b"%d/%s/%d" % (codec, factor.encode(), P)))
    kw = dict(comparator=T.CMP_BYTES)
    if P > 1:
        kw.update(tmp=tmp, P=P, parts=seg_parts, send_empty=send_empty)
    nrec = {p: sum(c for c, q in zip(counts, seg_parts) if q == p) for p in range(P)}
    bounded = run(segs, device_budget=FLOOR, **kw)
    plain = bounded[0]
    assert bounded[4][0] > 1 and bounded[4][1] <= FLOOR
    assert plain == run(segs, **kw)[0], "the uncompressed bounded write is the unbounded merge"
    if P == 1:
        assert plain[1] - 4 == nrec[0] * size + 2, "the body is n records of `size` bytes and FF FF"
    else:
        for p in range(P):
            start, raw, part = plain[2][p]
            if nrec[p]:
                assert raw - 4 == nrec[p] * size + 2, p
            elif send_empty:
                assert raw == 0 and part == 0, p          # no segment
            else:
                assert raw == 6 and part == 10, p         # a segment of FF FF alone
    if c is None:
        return
    got = check(segs, codec, **kw)
    for (out, raw_or_idx, third), steps in got.values():
        assert steps > 1
        if P == 1:
            assert CT.independent_body(c, out, raw_or_idx - 4) == plain[0][4:-4]
            continue
        for p in range(P):
            start, raw, part = third[p]
            pstart, praw, ppart = plain[2][p]
            if part:
                assert CT.independent_body(c, out[start:start + part], raw - 4) == plain[0][pstart + 4:pstart + ppart - 4], p


@pytest.mark.parametrize("factor", ["chunk", "chunk-1", "chunk+1", "half"])
@pytest.mark.parametrize("name", list(CT.CODECS) + ["none"])
def test_one_partition_on_the_grid(name, factor):
    _grid_case(name, factor, 1, True, None)


@pytest.mark.parametrize("send_empty", [False, True])
@pytest.mark.parametrize("name", list(CT.CODECS) + ["none"])
def test_four_partitions_on_the_grid(name, send_empty, tmp_path):
    """P = 4, partition 1 without records: its neighbours close and open at cuts on the grid"""
    _grid_case(name, "chunk", 4, send_empty, str(tmp_path))


@pytest.mark.parametrize("name", list(CT.CODECS))
def test_short_partition_before_a_long_one(name, tmp_path):
    """P = 2: partition 0 (39 records of one chunk each, one segment) closes in an early step while partition 1 (about
    12 MiB) runs on over several, every cut on the grid.

    No public input makes close_open close a partition with its carry and FF FF in a step of their own.  The splitter S
    is the smallest last complete key of the windows that do not reach their segment's EOF markers, so a window's last
    complete record is merged only when that window reaches EOF.  The step that merges a partition's last record
    therefore finishes every segment of the partition, and its piece closes the partition itself."""
    c = CT.CODECS[name]
    size = c.chunk
    rng = random.Random(9)
    vl = _value_len(size)
    small = [((i).to_bytes(8, "big"), rng.randbytes(vl)) for i in range(1, 40)]
    big, _, _ = _segments(size, 4, [1], seed=4)
    segs = [O.write_ifile(small, rle=False)[0]] + big
    kw = dict(comparator=T.CMP_BYTES, tmp=str(tmp_path), P=2, parts=[0, 1, 1, 1, 1], send_empty=True)
    got = check(segs, c.id, **kw)
    plain = run(segs, device_budget=FLOOR, **kw)[0]
    assert plain[2][0][1] - 4 == len(small) * size + 2
    for (out, _, index), steps in got.values():
        for p in range(2):
            start, raw, part = index[p]
            pstart, praw, ppart = plain[2][p]
            assert CT.independent_body(c, out[start:start + part], raw - 4) == plain[0][pstart + 4:pstart + ppart - 4]

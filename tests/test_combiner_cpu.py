"""CPU: the reference combine (tests/combine_model.py: oracle sort / merge + grouping + re-framing) against an
independent model -- a dict of (partition, key) -> wrapped sum, keys in comparator order -- for every comparator and
both sum reducers, on duplicate-heavy data."""
import random

import numpy as np
import pytest

from oracle import tez_oracle as O
import combine_model as CM

CMPS = [O.CMP_BYTES, O.CMP_TEXT, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG]


def make_key(cmp_kind, x):
    if cmp_kind == O.CMP_TEXT:
        return O.text("w%d" % x if x % 7 else "")              # includes the empty string
    if cmp_kind == O.CMP_BYTESWRITABLE:
        b = bytes([x % 251]) * (x % 5)
        return len(b).to_bytes(4, "big") + b
    if cmp_kind == O.CMP_INT:
        return O.int_writable(x - 20)
    if cmp_kind == O.CMP_LONG:
        return O.long_writable(-x * 1000003)
    return b"" if x == 0 else x.to_bytes(3, "big")             # raw bytes, one empty key


def make_value(combiner, rng):
    w = CM.WIDTH[combiner]
    # values near the top of the range: sums wrap
    return rng.choice([(1 << (8 * w - 1)) - 1, 1, (1 << (8 * w)) - 1, rng.getrandbits(8 * w)]).to_bytes(w, "big")


def _serialize(per_partition):
    out = bytearray()
    idx = []
    for recs in per_partition:
        if not recs:                       # empty partition: no segment, reported through the event
            idx.append((len(out), 0, 0))
            continue
        seg, raw, part = O.write_ifile(recs)
        idx.append((len(out), raw, part))
        out += seg
    return bytes(out), np.array(idx, dtype=np.int64).reshape(-1, 3)


@pytest.mark.parametrize("combiner", [CM.SUM_INT, CM.SUM_LONG])
@pytest.mark.parametrize("cmp_kind", CMPS)
@pytest.mark.parametrize("P,given", [(1, False), (7, False), (5, True)])
def test_oracle_combine_matches_model(cmp_kind, combiner, P, given):
    rng = random.Random(cmp_kind * 10 + combiner + P)
    n = 3000
    records = [(make_key(cmp_kind, min(int(rng.paretovariate(1.2)), 60)), make_value(combiner, rng)) for _ in range(n)]
    records += [(make_key(cmp_kind, 1000 + i), make_value(combiner, rng)) for i in range(5)]   # one-record groups
    # GIVEN partitions put the same key into several partitions
    partition = [rng.randrange(P) for _ in records] if given else [O.partition_of(cmp_kind, k, P) for k, _ in records]
    kv, ko, kl, vl, _ = CM.pack(records)
    got = CM.sort_combine(P, cmp_kind, combiner, kv, ko, kl, vl, np.array(partition, np.int32) if given else None)
    model = CM.model(records, partition, cmp_kind, combiner, P)
    exp_file, exp_idx = _serialize(model)
    assert got["file_out"] == exp_file
    assert np.array_equal(got["index"], exp_idx)
    assert got["combine_input"] == len(records)
    assert got["combine_output"] == sum(len(r) for r in model)


def test_int_sum_wraps_like_java_int():
    recs = [(O.text("a"), O.int_writable(0x7FFFFFFF)), (O.text("a"), O.int_writable(1)), (O.text("b"), O.int_writable(-1))]
    out = CM.combine_records(recs, O.CMP_TEXT, CM.SUM_INT)
    assert out == [(O.text("a"), (0x80000000).to_bytes(4, "big")), (O.text("b"), b"\xff\xff\xff\xff")]
    long_recs = [(O.text("a"), O.long_writable(-1)), (O.text("a"), O.long_writable(2))]
    assert CM.combine_records(long_recs, O.CMP_TEXT, CM.SUM_LONG) == [(O.text("a"), O.long_writable(1))]


def test_single_record_groups_reencode_to_their_input():
    """A group of one record re-encodes to exactly its bytes: the combined segment of all-unique keys is the input."""
    recs = sorted({O.text("k%05d" % i): O.int_writable(i * 7919) for i in range(500)}.items(),
                  key=lambda kv: kv[0][1:])
    seg, _, _ = O.write_ifile(recs)
    comb = CM.combine_records([(k, v) for _, k, v in O.read_ifile(seg)], O.CMP_TEXT, CM.SUM_INT)
    assert O.write_ifile(comb)[0] == seg


def test_bad_value_width_is_an_error():
    recs = [(O.text("a"), O.int_writable(1)), (O.text("a"), b"\0\0\0\0\0")]
    with pytest.raises(CM.BadWidth):
        CM.combine_records(recs, O.CMP_TEXT, CM.SUM_INT)
    kv, ko, kl, vl, _ = CM.pack(recs)
    with pytest.raises(CM.BadWidth):
        CM.sort_combine(1, O.CMP_TEXT, CM.SUM_INT, kv, ko, kl, vl)


def test_merge_combine_matches_model():
    rng = random.Random(5)
    segs, all_recs = [], []
    for s in range(4):
        keys = sorted((O.text("w%d" % rng.randrange(40)) for _ in range(300)), key=lambda k: k[1:])
        recs = [(k, O.long_writable(rng.getrandbits(64))) for k in keys]
        all_recs += recs
        segs.append(O.write_ifile(recs, rle=True)[0])
    got = CM.merge_combine(segs, O.CMP_TEXT, CM.SUM_LONG)
    exp = O.write_ifile(CM.model(all_recs, [0] * len(all_recs), O.CMP_TEXT, CM.SUM_LONG, 1)[0])
    assert got == exp

"""CPU: TotalOrderPartitioner's split checks and partition search, run on the host with the device's code
(tezgpu_debug_total_order_emulate), against the model's bisect_right over comparison keys; and the refusals of the
runtime-library mirror, which all happen before any device call."""
import random

import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import runtime_library as RL
import sort_order_model as M
import total_order_model as TO

# (sort comparator, search order): every comparator in its own order, and the natural-order search of Text and
# BytesWritable keys under TezBytesComparator
CASES = [(O.CMP_BYTES, O.CMP_BYTES), (O.CMP_TEXT, O.CMP_TEXT), (O.CMP_BYTESWRITABLE, O.CMP_BYTESWRITABLE),
         (O.CMP_INT, O.CMP_INT), (O.CMP_LONG, O.CMP_LONG), (O.CMP_BYTES, O.CMP_TEXT), (O.CMP_BYTES, O.CMP_BYTESWRITABLE)]
ALPHABET = b"\x00\x01ab\x7f\x80\xfe\xff"


def _key(order, content):
    return M.make_key(order, content)


def _contents(rng, order, n):
    if order in M.FIXED_LEN:
        ln = M.FIXED_LEN[order]
        return [bytes(rng.randrange(256) for _ in range(ln)) for _ in range(n)]
    return [TO.random_content(rng, 14, ALPHABET) for _ in range(n)]


def _splits(rng, sort_cmp, order, P):
    """P - 1 split keys, increasing under the sort comparator and the search order (equal content lengths where the two
    differ: the length prefix leads the raw bytes)."""
    if order in M.FIXED_LEN:
        pool = {bytes(rng.randrange(256) for _ in range(M.FIXED_LEN[order])) for _ in range(4 * P)}
    elif sort_cmp != order:
        pool = {TO.random_content(rng, 0, None) + bytes(rng.choice(ALPHABET) for _ in range(10)) for _ in range(4 * P)}
    else:
        pool = {TO.random_content(rng, 14, ALPHABET) for _ in range(4 * P)}
    keys = [_key(order, c) for c in pool]
    return TO.quantile_splits(keys, P, order)


def _check(keys, splits, sort_cmp, order):
    got = T.debug_total_order(keys, splits, sort_cmp, order)
    exp = TO.partitions(keys, splits, order)
    assert np.array_equal(got, np.array(exp, dtype=np.int32))
    return got


@pytest.mark.parametrize("sort_cmp,order", CASES)
def test_partitions_agree_with_model_on_random_keys(sort_cmp, order):
    rng = random.Random(17 * sort_cmp + order)
    for P in (2, 64, 1000):
        splits = _splits(rng, sort_cmp, order, P)
        keys = [_key(order, c) for c in _contents(rng, order, 100_000 if P == 64 else 20_000)]
        # keys that share 8 or more content bytes with a split, and the splits themselves
        for s in splits[::max(1, P // 16)]:
            c = search_key(order, s)
            keys += [s, _key(order, c[:8] + b"\x00" * (len(c) - 8)) if len(c) > 8 else s]
            if order not in M.FIXED_LEN:
                keys += [_key(order, c + b"\x00"), _key(order, c + b"\xff"), _key(order, c[:-1])]
        got = _check(keys, splits, sort_cmp, order)
        assert got.min() == 0 and got.max() == P - 1


def search_key(order, key):
    return TO.search_key(order, key)


@pytest.mark.parametrize("sort_cmp,order", CASES)
def test_keys_equal_to_splits_below_first_and_above_last(sort_cmp, order):
    rng = random.Random(order)
    splits = _splits(rng, sort_cmp, order, 9)
    got = _check(splits, splits, sort_cmp, order)
    assert list(got) == list(range(1, 9)), "a key equal to split i goes to partition i + 1"
    if order in M.FIXED_LEN:
        lo, hi = b"\x00" * M.FIXED_LEN[order], b"\xff" * M.FIXED_LEN[order]
    else:
        lo, hi = b"", b"\xff" * 40
    assert list(_check([_key(order, lo), _key(order, hi)], splits, sort_cmp, order)) == [0, 8]


def test_long_shared_prefixes_empty_keys_and_ff_bytes():
    """Keys that agree with a split on 8 or more bytes are told apart by the bytes after the prefix word and by length:
    "ab" and "ab\\0" stay distinct even though their zero-padded prefix words are equal."""
    splits = [b"ab", b"ab\x00", b"abcdefgh", b"abcdefgh\x00", b"abcdefghij", b"abcdefghij\xff", b"\xff" * 9]
    keys = [b"", b"a", b"ab", b"ab\x00", b"ab\x00\x00", b"ab\x01", b"abcdefg", b"abcdefgh", b"abcdefgh\x00",
            b"abcdefgh\x00\x00", b"abcdefghi", b"abcdefghij", b"abcdefghij\x00", b"abcdefghij\xff", b"abcdefghij\xff\x00",
            b"\xff" * 8, b"\xff" * 9, b"\xff" * 10]
    got = _check(keys, splits, O.CMP_BYTES, O.CMP_BYTES)
    assert list(got) == [0, 0, 1, 2, 2, 2, 2, 3, 4, 4, 4, 5, 5, 6, 6, 6, 7, 7]


def test_negative_ints_and_longs():
    isplits = [O.int_writable(v) for v in (-2 ** 31 + 1, -1000, -1, 0, 1, 2 ** 31 - 1)]
    ikeys = [O.int_writable(v) for v in (-2 ** 31, -2 ** 31 + 1, -1001, -1000, -2, -1, 0, 1, 5, 2 ** 31 - 1)]
    assert list(_check(ikeys, isplits, O.CMP_INT, O.CMP_INT)) == [0, 1, 1, 2, 2, 3, 4, 5, 5, 6]
    lsplits = [O.long_writable(v) for v in (-2 ** 40, -1, 0, 2 ** 40)]
    lkeys = [O.long_writable(v) for v in (-2 ** 63, -2 ** 40, -5, -1, 0, 7, 2 ** 40, 2 ** 63 - 1)]
    assert list(_check(lkeys, lsplits, O.CMP_LONG, O.CMP_LONG)) == [0, 1, 1, 2, 3, 3, 4, 4]


def test_bytes_sort_with_natural_order_byteswritable_search():
    """TezBytesComparator sorts BytesWritable keys by their raw bytes (length first); the natural-order search compares
    the content alone, so a short key with a large first byte lands after a long key with a small one."""
    bw = lambda c: len(c).to_bytes(4, "big") + c
    splits = [bw(b"b"), bw(b"d")]
    keys = [bw(b"a" * 20), bw(b"c"), bw(b"b"), bw(b"bb" * 30), bw(b"z"), bw(b"")]
    assert list(_check(keys, splits, O.CMP_BYTES, O.CMP_BYTESWRITABLE)) == [0, 1, 1, 1, 2, 0]
    assert list(_check(keys, splits, O.CMP_BYTES, O.CMP_BYTES)) == [2, 1, 1, 2, 2, 0]


def test_hadoop_validation_errors_and_one_partition():
    with pytest.raises(IOError, match="Split points are out of order") as e:
        T.debug_total_order([b"x"], [b"b", b"a"], O.CMP_BYTES)
    assert e.value.code == T.E_INVALID
    with pytest.raises(IOError, match="Split points are out of order"):
        T.debug_total_order([b"x"], [b"a", b"a"], O.CMP_BYTES)
    # strictly increasing under the sort comparator (raw bytes: the length first), even when the content order of the
    # search accepts them
    bw = lambda c: len(c).to_bytes(4, "big") + c
    with pytest.raises(IOError, match="Split points are out of order"):
        T.debug_total_order([], [bw(b"aa"), bw(b"b")], O.CMP_BYTES, O.CMP_BYTESWRITABLE)
    assert list(T.debug_total_order([b"", b"a", b"\xff"], [], O.CMP_BYTES)) == [0, 0, 0]


@pytest.mark.parametrize("sort_cmp,order", [(O.CMP_INT, O.CMP_TEXT), (O.CMP_TEXT, O.CMP_BYTES), (O.CMP_BYTESWRITABLE, O.CMP_TEXT),
                                            (O.CMP_LONG, O.CMP_INT), (O.CMP_BYTES, O.CMP_LONG), (O.CMP_BYTES, 7)])
def test_search_order_must_fit_the_comparator(sort_cmp, order):
    """The search runs in the comparator's own order, or in the natural content order of Text / BytesWritable keys
    that TezBytesComparator sorts; any other pairing is refused."""
    with pytest.raises(IOError, match="does not fit comparator") as e:
        T.debug_total_order([], [], sort_cmp, order)
    assert e.value.code == T.E_INVALID


# ------------------------------------------------------------------------------------------------ the mirror's refusals
def _out_conf(path, key_class=TO.BYTES_WRITABLE, **kw):
    c = {"tez.runtime.key.class": key_class, "tez.runtime.value.class": TO.BYTES_WRITABLE,
         "tez.runtime.partitioner.class": TO.NEW_API, "mapreduce.totalorderpartitioner.path": path}
    c.update(kw)
    return c


def _start(tmp_path, conf, P=4):
    out = RL.OrderedPartitionedKVOutput(RL.OutputContext(conf=conf, work_dir=str(tmp_path)), P)
    out.initialize()
    out.start()
    return out


def _bw(c):
    return len(c).to_bytes(4, "big") + c


def test_mirror_refuses_missing_file(tmp_path):
    with pytest.raises(IOError, match="Can't read partitions file") as e:
        _start(tmp_path, _out_conf("nope.lst"))
    assert e.value.code == T.E_INVALID and "nope.lst" in str(e.value)


def test_mirror_refuses_wrong_key_class(tmp_path):
    (tmp_path / "_partition.lst").write_bytes(TO.sequence_file([O.text("a"), O.text("b"), O.text("c")], TO.TEXT))
    conf = _out_conf("_partition.lst")
    with pytest.raises(IOError, match="wrong key class: %s is not %s" % (TO.BYTES_WRITABLE, TO.TEXT)) as e:
        _start(tmp_path, conf)
    assert e.value.code == T.E_INVALID and "_partition.lst" in str(e.value)


@pytest.mark.parametrize("cut", [3, 10, 40, -3])
def test_mirror_refuses_truncated_file(tmp_path, cut):
    data = TO.sequence_file([_bw(b"a"), _bw(b"b"), _bw(b"c")], TO.BYTES_WRITABLE)
    (tmp_path / "p.lst").write_bytes(data[:cut])
    with pytest.raises(IOError) as e:
        _start(tmp_path, _out_conf("p.lst"))
    assert e.value.code == T.E_INVALID and "p.lst" in str(e.value)


@pytest.mark.parametrize("compression", ["none", "record"])
def test_mirror_reads_sync_escapes_and_record_compressed_values(tmp_path, compression):
    """A partition file of 63 split keys with a sync escape after every other record and (record compression) a zlib
    value per record is parsed to its end: only the count or order check, which needs every key, can then fail."""
    keys = [_bw(b"k%03d" % i) for i in range(63)]
    values = [b"value %d" % i for i in range(63)]
    (tmp_path / "p.lst").write_bytes(TO.sequence_file(keys, TO.BYTES_WRITABLE, compression=compression, sync_every=2,
                                                      values=values))
    with pytest.raises(IOError, match="Wrong number of partitions in keyset"):   # 63 keys are P = 64
        _start(tmp_path, _out_conf("p.lst"), P=63)
    bad = keys[:62] + [_bw(b"k000")]                      # the last key breaks the order
    (tmp_path / "q.lst").write_bytes(TO.sequence_file(bad, TO.BYTES_WRITABLE, compression=compression, sync_every=2,
                                                      values=values))
    with pytest.raises(IOError, match="Split points are out of order"):
        _start(tmp_path, _out_conf("q.lst"), P=64)
    data = bytearray(TO.sequence_file(keys, TO.BYTES_WRITABLE, compression=compression, sync_every=2, values=values))
    sync_at = data.index(b"\xff\xff\xff\xff") + 4        # first sync escape: corrupt its marker
    data[sync_at] ^= 1
    (tmp_path / "r.lst").write_bytes(bytes(data))
    with pytest.raises(IOError, match="sync marker") as e:
        _start(tmp_path, _out_conf("r.lst"), P=64)
    assert e.value.code == T.E_INVALID and "r.lst" in str(e.value)


def test_mirror_refuses_block_compressed_file(tmp_path):
    (tmp_path / "p.lst").write_bytes(TO.sequence_file([_bw(b"a"), _bw(b"b"), _bw(b"c")], TO.BYTES_WRITABLE,
                                                      compression="block"))
    with pytest.raises(IOError, match="block-compressed") as e:
        _start(tmp_path, _out_conf("p.lst"))
    assert e.value.code == T.E_UNSUPPORTED


def test_mirror_refuses_wrong_count_and_disorder(tmp_path):
    (tmp_path / "p.lst").write_bytes(TO.sequence_file([_bw(b"a"), _bw(b"b")], TO.BYTES_WRITABLE))
    with pytest.raises(IOError, match="Wrong number of partitions in keyset"):
        _start(tmp_path, _out_conf("p.lst"))
    (tmp_path / "q.lst").write_bytes(TO.sequence_file([_bw(b"a"), _bw(b"c"), _bw(b"b")], TO.BYTES_WRITABLE))
    with pytest.raises(IOError, match="Split points are out of order"):
        _start(tmp_path, _out_conf("q.lst"))


def test_mirror_refuses_explicit_partition_on_write(tmp_path):
    """On a total-order output the device computes the partition: a given one is refused before anything else, so the
    refusal needs no device and no start()."""
    for cls in (TO.NEW_API, TO.OLD_API):
        conf = _out_conf("p.lst", **{"tez.runtime.partitioner.class": cls})
        out = RL.OrderedPartitionedKVOutput(RL.OutputContext(conf=conf, work_dir=str(tmp_path)), 4)
        out.initialize()
        with pytest.raises(IOError, match="TotalOrderPartitioner") as e:
            out.getWriter().write(_bw(b"a"), b"v", partition=1)
        assert e.value.code == T.E_INVALID

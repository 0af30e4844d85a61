"""GPU: TotalOrderPartitioner on the device.  file.out and file.out.index must equal, byte for byte, the oracle's
PipelinedSorter / UnorderedPartitionedKVWriter fed the model's partitions (bisect_right over comparison keys), across
the five comparators, P = 1 .. 65,536 (beyond the shared-memory split table), the 16-byte fast stage, fixed-width,
variable-width and alphabet-packed (SymTable) sort words, and unordered handles.  With a combiner or a codec the
output must equal the same handle run with the model's partitions given (PART_GIVEN, checked against the oracle by
the suites of those features).  Then the C ABI's errors."""
import random
import zlib

import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
import sort_order_model as M
import total_order_model as TO

pytestmark = pytest.mark.gpu

CMPS = [O.CMP_BYTES, O.CMP_TEXT, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG]
PARTS = [1, 2, 64, 1024, 65536]


def _pack(records):
    kv = bytearray()
    ko, vo, vl = [], [], []
    for k, v in records:
        ko.append(len(kv))
        kv += k
        vo.append(len(kv))
        kv += v
        vl.append(len(v))
    return (np.frombuffer(bytes(kv), dtype=np.uint8) if kv else np.zeros(0, np.uint8), np.array(ko, np.uint32),
            np.array(vo, np.uint32), np.array(vl, np.uint32))


def _content(rng, cmp, alphabet=None):
    if cmp in M.FIXED_LEN:
        return bytes(rng.randrange(256) for _ in range(M.FIXED_LEN[cmp]))
    ln = rng.randrange(0, 13)
    return bytes(rng.choice(alphabet) if alphabet else rng.randrange(256) for _ in range(ln))


def _keys_and_splits(rng, cmp, P, n, alphabet=None):
    keys = [M.make_key(cmp, _content(rng, cmp, alphabet)) for _ in range(n)]
    splits = []
    if P > 1:
        sample = set(keys[: 4 * P])
        while len(sample) < 2 * P:
            sample.add(M.make_key(cmp, _content(rng, cmp, alphabet) + (b"" if cmp in M.FIXED_LEN else bytes([rng.randrange(256)] * 3))))
        splits = TO.quantile_splits(list(sample), P, cmp)
    return keys, splits


def _compare_variable(records, P, cmp, splits, order=None, unordered=False, rle=-1, batches=1):
    kv, ko, vo, vl = _pack(records)
    order = cmp if order is None else order
    part = np.array(TO.partitions([k for k, _ in records], splits, order), dtype=np.int32)
    conf = O.sorter_conf(P, cmp_kind=cmp, partitioner=O.PART_GIVEN, rle_policy=rle)
    run = O.unordered_write if unordered else O.pipelined_sort
    exp = run(conf, kv, ko.astype(np.uint64), vo - ko, vl, part)
    with T.GpuSorter(P, comparator=cmp, partitioner=T.PART_TOTAL_ORDER, rle_policy=rle, unordered=unordered,
                     split_points=splits, split_order=order) as s:
        n = len(records)
        step = max(1, (n + batches - 1) // batches)
        for a in range(0, n, step):
            b = min(n, a + step)
            lo, hi = int(ko[a]), int(vo[b - 1] + vl[b - 1])
            s.collect(kv[lo:hi], ko[a:b] - lo, vo[a:b] - lo, vl[a:b])
        out, index_bytes, index, st = s.flush_to_memory()
    assert bytes(out) == exp["file_out"], "file.out differs from the oracle"
    assert index_bytes == exp["index_out"]
    assert np.array_equal(index, exp["index"])
    return st


@pytest.mark.parametrize("P", PARTS)
@pytest.mark.parametrize("cmp", CMPS)
def test_variable_width_parity(cmp, P):
    rng = random.Random(31 * cmp + P)
    n = 150_000 if P == 65536 else 30_000
    keys, splits = _keys_and_splits(rng, cmp, P, n)
    # value = f(key): the reference leaves the order of equal keys open, so equal keys carry equal records
    recs = [(k, zlib.crc32(k).to_bytes(4, "big") * (len(k) % 5)) for k in keys]
    _compare_variable(recs, P, cmp, splits, rle=0, batches=2)


@pytest.mark.parametrize("P", [2, 64, 1024, 65536])
def test_alphabet_packed_sort_word_and_rle(P):
    """Text words over a small alphabet: the sort word is packed ranks (SymTable), many duplicates switch RLE on."""
    rng = random.Random(P)
    keys, splits = _keys_and_splits(rng, O.CMP_TEXT, P, 120_000, alphabet=b"abcdefghijklmnop")
    recs = [(k, O.int_writable(1)) for k in keys]
    _compare_variable(recs, P, O.CMP_TEXT, splits, rle=-1, batches=3)


@pytest.mark.parametrize("order", [O.CMP_TEXT, O.CMP_BYTESWRITABLE])
def test_bytes_sort_with_natural_order_search(order):
    """TezBytesComparator sort of Text / BytesWritable keys, split search in the content order."""
    rng = random.Random(order)
    keys = [M.make_key(order, bytes(rng.randrange(256) for _ in range(rng.randrange(0, 12)))) for _ in range(40_000)]
    # equal content lengths: increasing in both the raw bytes and the content order
    pool = {M.make_key(order, bytes(rng.randrange(256) for _ in range(6))) for _ in range(400)}
    splits = TO.quantile_splits(list(pool), 64, O.CMP_BYTES)
    recs = [(k, b"v" * (len(k) % 7)) for k in keys]
    _compare_variable(recs, 64, O.CMP_BYTES, splits, order=order, rle=0)


@pytest.mark.parametrize("P", PARTS)
@pytest.mark.parametrize("cmp", CMPS)
def test_unordered_parity(cmp, P):
    rng = random.Random(7 * cmp + P)
    keys, splits = _keys_and_splits(rng, cmp, P, 100_000 if P == 65536 else 20_000)
    recs = [(k, rng.randbytes(rng.randrange(0, 12))) for k in keys]
    _compare_variable(recs, P, cmp, splits, unordered=True, rle=0)


@pytest.mark.parametrize("P", PARTS)
@pytest.mark.parametrize("order", [O.CMP_BYTES, O.CMP_BYTESWRITABLE])
def test_fast16_parity(order, P):
    """16-byte keys, 64-byte values, TezBytesComparator: the 16-byte stage (k_stage<true, true>), searched in raw byte
    order or as BytesWritable content (4-byte length 12, then 12 bytes), on the host path and device-resident."""
    import torch
    n = 400_000
    kv = O.gen_c2(0, n, seed=P + order)
    if order == O.CMP_BYTESWRITABLE:
        kv.reshape(n, 80)[:, :4] = np.frombuffer((12).to_bytes(4, "big"), dtype=np.uint8)
    keys = [bytes(kv[i * 80:i * 80 + 16]) for i in range(n)]
    rng = random.Random(P)
    splits = TO.quantile_splits(rng.sample(keys, 2 * P), P, O.CMP_BYTES) if P > 1 else []
    part = np.array(TO.partitions(keys, splits, order), dtype=np.int32)
    conf = O.sorter_conf(P, partitioner=O.PART_GIVEN)
    exp = O.pipelined_sort(conf, kv, np.arange(n, dtype=np.uint64) * 80, np.full(n, 16, np.uint32), np.full(n, 64, np.uint32), part)
    with T.GpuSorter(P, fixed=(16, 64), partitioner=T.PART_TOTAL_ORDER, split_points=splits, split_order=order) as s:
        s.collect_fixed(kv)
        out, index_bytes, _, _ = s.flush_to_memory()
        assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]
        d_kv = torch.from_numpy(kv).cuda()
        cap = n * 82 + 10 * P + 4096
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        out_len, index, _ = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
        assert np.array_equal(d_out[:out_len].cpu().numpy(), np.frombuffer(exp["file_out"], dtype=np.uint8))
        assert np.array_equal(index, exp["index"])


@pytest.mark.parametrize("P", [2, 1024, 65536])
@pytest.mark.parametrize("cmp,kl,vl", [(O.CMP_INT, 4, 8), (O.CMP_LONG, 8, 8), (O.CMP_BYTES, 10, 7)])
def test_fixed_width_parity(cmp, kl, vl, P):
    rng = np.random.default_rng(P + kl)
    n = 200_000
    kv = rng.integers(0, 256, size=n * (kl + vl), dtype=np.uint8)
    rows = kv.reshape(n, kl + vl)
    rows[:, kl:] = rows[:, [j % kl for j in range(vl)]]      # value = f(key): equal keys carry equal records
    keys = [bytes(kv[i * (kl + vl):i * (kl + vl) + kl]) for i in range(n)]
    splits = TO.quantile_splits(keys[: 3 * P] if 3 * P <= n else keys, P, cmp)
    part = np.array(TO.partitions(keys, splits, cmp), dtype=np.int32)
    conf = O.sorter_conf(P, cmp_kind=cmp, partitioner=O.PART_GIVEN, rle_policy=0)
    exp = O.pipelined_sort(conf, kv, np.arange(n, dtype=np.uint64) * (kl + vl), np.full(n, kl, np.uint32), np.full(n, vl, np.uint32), part)
    with T.GpuSorter(P, comparator=cmp, fixed=(kl, vl), partitioner=T.PART_TOTAL_ORDER, rle_policy=0, split_points=splits) as s:
        s.collect_fixed(kv)
        out, index_bytes, _, _ = s.flush_to_memory()
    assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]


def _given_vs_total(records, P, cmp, splits, **kw):
    kv, ko, vo, vl = _pack(records)
    part = np.array(TO.partitions([k for k, _ in records], splits, cmp), dtype=np.int32)
    outs = []
    for mode in (T.PART_GIVEN, T.PART_TOTAL_ORDER):
        with T.GpuSorter(P, comparator=cmp, partitioner=mode, split_points=splits if mode == T.PART_TOTAL_ORDER else None, **kw) as s:
            s.collect(kv, ko, vo, vl, part if mode == T.PART_GIVEN else None)
            out, index_bytes, _, st = s.flush_to_memory()
            outs.append((bytes(out), index_bytes, st["output_records"], st["spilled_records"]))
    assert outs[0] == outs[1]


@pytest.mark.parametrize("P", [2, 64, 65536])
def test_combiner_equals_given_partitions(P):
    rng = random.Random(P)
    keys, splits = _keys_and_splits(rng, O.CMP_TEXT, P, 120_000, alphabet=b"abcdef")
    _given_vs_total([(k, O.int_writable(rng.randrange(100))) for k in keys], P, O.CMP_TEXT, splits, combiner=T.COMBINE_SUM_INT)


@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_codec_equals_given_partitions(codec):
    rng = random.Random(codec)
    keys, splits = _keys_and_splits(rng, O.CMP_LONG, 64, 50_000)
    _given_vs_total([(k, rng.randbytes(30)) for k in keys], 64, O.CMP_LONG, splits, codec=codec)


def test_split_points_survive_reset():
    rng = random.Random(3)
    keys, splits = _keys_and_splits(rng, O.CMP_BYTES, 16, 5000)
    recs = [(k, b"x") for k in keys]
    kv, ko, vo, vl = _pack(recs)
    exp = O.pipelined_sort(O.sorter_conf(16, partitioner=O.PART_GIVEN, rle_policy=0), kv, ko.astype(np.uint64), vo - ko, vl,
                           np.array(TO.partitions(keys, splits, O.CMP_BYTES), np.int32))
    with T.GpuSorter(16, partitioner=T.PART_TOTAL_ORDER, rle_policy=0, split_points=splits) as s:
        for _ in range(2):
            s.reset()
            s.collect(kv, ko, vo, vl)
            assert bytes(s.flush_to_memory()[0]) == exp["file_out"]


def test_abi_errors():
    kv, ko, vo, vl = _pack([(b"a", b"1"), (b"m", b"2")])
    with T.GpuSorter(4, partitioner=T.PART_HASH) as s:           # not a TOTAL_ORDER handle
        with pytest.raises(IOError) as e:
            s.set_split_points([b"b", b"c", b"d"])
        assert e.value.code == T.E_INVALID
    with T.GpuSorter(4, partitioner=T.PART_TOTAL_ORDER) as s:
        with pytest.raises(IOError, match="Wrong number of partitions in keyset") as e:
            s.set_split_points([b"b", b"c"])
        assert e.value.code == T.E_INVALID
        with pytest.raises(IOError, match="Split points are out of order") as e:
            s.set_split_points([b"b", b"d", b"c"])
        assert e.value.code == T.E_INVALID
        with pytest.raises(IOError) as e:                          # collect before the split points
            s.collect(kv, ko, vo, vl)
        assert e.value.code == T.E_STATE
        with pytest.raises(IOError) as e:                          # flush before the split points
            s.flush_to_memory()
        assert e.value.code == T.E_STATE
        s.set_split_points([b"b", b"c", b"d"])
        with pytest.raises(IOError) as e:                          # a partition array
            s.collect(kv, ko, vo, vl, np.array([0, 1], np.int32))
        assert e.value.code == T.E_INVALID
        s.collect(kv, ko, vo, vl)
        with pytest.raises(IOError) as e:                          # after the first collect
            s.set_split_points([b"b", b"c", b"d"])
        assert e.value.code == T.E_STATE
        out, _, index, _ = s.flush_to_memory()
        assert [int(index[p][1]) > 6 for p in range(4)] == [True, False, False, True]
        with pytest.raises(IOError) as e:                          # after the flush
            s.set_split_points([b"b", b"c", b"d"])
        assert e.value.code == T.E_STATE
    with T.GpuSorter(4, fixed=(16, 64), partitioner=T.PART_TOTAL_ORDER) as s:
        kv2 = O.gen_c2(0, 10, seed=1)
        with pytest.raises(IOError) as e:
            s.collect_fixed(kv2)
        assert e.value.code == T.E_STATE
        s.set_split_points([bytes([0x40]) + bytes(15), bytes([0x80]) + bytes(15), bytes([0xc0]) + bytes(15)])
        with pytest.raises(IOError) as e:
            s.collect_fixed(kv2, np.zeros(10, np.int32))
        assert e.value.code == T.E_INVALID
        import torch
        d_kv = torch.from_numpy(kv2).cuda()
        d_part = torch.zeros(10, dtype=torch.int32, device="cuda")
        d_out = torch.empty(4096, dtype=torch.uint8, device="cuda")
        with pytest.raises(IOError) as e:
            s.sort_device_fixed(d_kv.data_ptr(), 10, d_out.data_ptr(), 4096, d_part.data_ptr())
        assert e.value.code == T.E_INVALID
    with T.GpuSorter(1, partitioner=T.PART_TOTAL_ORDER) as s:      # one partition: no split points needed
        s.collect(kv, ko, vo, vl)
        assert s.flush_to_memory()[3]["output_records"] == 2


def test_sort_example_end_to_end_through_the_mirror(tmp_path):
    """Shaped like Tez's Sort example with -totalOrder: BytesWritable keys, a record-compressed partition file written
    by the model, a sort memory small enough to spill and merge, P reducers through OrderedGroupedKVInput.  Every
    reducer's keys are sorted, every key of reducer p is <= every key of p + 1, and the concatenation is the sorted
    input."""
    from tez_b200 import runtime_library as RL
    rng = random.Random(5)
    P = 16
    keys = [TO.random_content(rng, 20) for _ in range(60_000)]
    bw = [len(k).to_bytes(4, "big") + k for k in keys]
    splits = TO.quantile_splits(rng.sample(bw, 4 * P), P, O.CMP_BYTESWRITABLE)
    (tmp_path / "_partition.lst").write_bytes(TO.sequence_file(splits, TO.BYTES_WRITABLE, compression="record"))
    conf = {"tez.runtime.key.class": TO.BYTES_WRITABLE, "tez.runtime.value.class": TO.BYTES_WRITABLE,
            "tez.runtime.partitioner.class": "org.apache.tez.mapreduce.partition.MRPartitioner",
            "mapred.mapper.new-api": True, "mapreduce.job.partitioner.class": TO.NEW_API, "tez.runtime.io.sort.mb": 1}
    out = RL.OrderedPartitionedKVOutput(RL.OutputContext(conf=conf, work_dir=str(tmp_path)), P)
    out.initialize()
    out.start()
    w = out.getWriter()
    for k in bw:
        w.write(k, b"v" + k[4:8])
    out.close()
    assert out.num_spills > 1, "the sort memory should force spills and a final merge"
    got = []
    for p in range(P):
        inp = RL.OrderedGroupedKVInput(RL.InputContext(conf=conf, work_dir=str(tmp_path)), 1)
        inp.initialize()
        inp.start()
        inp.handleEvents([RL.LocalOutput(0, out.final_output_file, out.final_index_file, p)])
        r = inp.getReader()
        part = []
        while r.next():
            part += [r.getCurrentKey()] * len(list(r.getCurrentValues()))
        cont = [k[4:] for k in part]
        assert cont == sorted(cont), "reducer %d is not sorted" % p
        got.append(cont)
    for a, b in zip(got, got[1:]):
        if a and b:
            assert a[-1] <= b[0]
    assert [k for g in got for k in g] == sorted(keys)

"""GPU: the device combiner (MRCombiner + IntSumReducer / LongSumReducer) against the reference combine of
tests/combine_model.py, byte for byte on file.out and file.out.index, with duplicate-heavy data."""
import collections
import random

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200._lib import TezGpuError
from tez_b200.runtime_library import (INT_WRITABLE, LONG_WRITABLE, TEXT, InputContext, LocalOutput, OrderedGroupedKVInput,
                                      OrderedPartitionedKVOutput, OutputContext, empty_partitions_from_payload)
import combine_model as CM

pytestmark = pytest.mark.gpu

SUM_INT, SUM_LONG = T.COMBINE_SUM_INT, T.COMBINE_SUM_LONG
W = {SUM_INT: 4, SUM_LONG: 8}


# ------------------------------------------------------------------------------------------------ sorter, variable width
def _key(cmp_kind, x):
    if cmp_kind == O.CMP_TEXT:
        return O.text("w%d" % x if x % 11 else "")
    if cmp_kind == O.CMP_BYTESWRITABLE:
        b = x.to_bytes(4, "big").lstrip(b"\0") * (1 + x % 3)
        return len(b).to_bytes(4, "big") + b
    if cmp_kind == O.CMP_INT:
        return O.int_writable(x - 1000)
    if cmp_kind == O.CMP_LONG:
        return O.long_writable(-x * 999983)
    return b"" if x == 0 else x.to_bytes(5, "big").lstrip(b"\0")


def _value(combiner, rng):
    w = W[combiner]
    return rng.choice([(1 << (8 * w - 1)) - 1, (1 << (8 * w)) - 1, rng.getrandbits(8 * w)]).to_bytes(w, "big")


def _keys(kind, n, rng):
    if kind == "zipf":
        return [min(int(rng.paretovariate(1.1)), 100000) for _ in range(n)]
    if kind == "few":
        return [rng.randrange(4) for _ in range(n)]
    return [11 * x + 1 for x in rng.sample(range(50 * n + 1), n)]       # all unique (and no empty Text key)


def _sorter_case(records, P, cmp_kind, combiner, partition=None, rle=-1, batches=1):
    kv, ko, kl, vl, vo = CM.pack(records)
    exp = CM.sort_combine(P, cmp_kind, combiner, kv, ko, kl, vl, partition)
    with T.GpuSorter(P, comparator=cmp_kind, partitioner=T.PART_GIVEN if partition is not None else T.PART_HASH,
                     rle_policy=rle, combiner=combiner) as s:
        n = len(records)
        step = max(1, -(-n // batches))
        for a in range(0, n, step):
            b = min(n, a + step)
            lo, hi = int(ko[a]), int(vo[b - 1] + vl[b - 1])
            s.collect(kv[lo:hi], ko[a:b].astype(np.uint32) - lo, vo[a:b] - lo, vl[a:b],
                      None if partition is None else np.asarray(partition[a:b], np.int32))
        out, index_bytes, index, st = s.flush_to_memory()
    assert bytes(out) == exp["file_out"], "combined file.out differs from the reference combine"
    assert index_bytes == exp["index_out"]
    assert np.array_equal(index, exp["index"])
    assert st["output_records"] == len(records) == exp["combine_input"]
    assert st["spilled_records"] == exp["combine_output"]
    return st


@pytest.mark.parametrize("combiner", [SUM_INT, SUM_LONG])
@pytest.mark.parametrize("cmp_kind", [O.CMP_TEXT, O.CMP_BYTES, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG])
@pytest.mark.parametrize("P,given", [(1, False), (64, False), (1024, False), (64, True)])
def test_sorter_collect_batch_bit_exact(cmp_kind, combiner, P, given):
    rng = random.Random(hash((cmp_kind, combiner, P, given)) & 0xFFFF)
    n = 20000
    recs = [(_key(cmp_kind, x), _value(combiner, rng)) for x in _keys("zipf", n, rng)]
    part = np.array([rng.randrange(P) for _ in recs], np.int32) if given else None
    st = _sorter_case(recs, P, cmp_kind, combiner, part, batches=3)
    assert st["spilled_records"] < n


@pytest.mark.parametrize("kind,n", [("few", 0), ("few", 1), ("few", 5000), ("zipf", 100000), ("unique", 30000)])
def test_sorter_key_spaces_text(kind, n):
    rng = random.Random(n)
    recs = [(_key(O.CMP_TEXT, x), _value(SUM_INT, rng)) for x in _keys(kind, n, rng)]
    st = _sorter_case(recs, 16, O.CMP_TEXT, SUM_INT)
    if kind == "unique":
        assert st["spilled_records"] == n and st["adjacent_equal_keys"] == 0


def test_rle_auto_decision_kept_but_no_repeat_markers():
    """Above the 0.1 threshold the uncombined stream would be run-length encoded: rle_used reports that decision, and
    the combined output has unique keys, so it carries no REPEAT_KEY marker (it equals the reference combine)."""
    rng = random.Random(3)
    recs = [(_key(O.CMP_TEXT, rng.randrange(50)), O.int_writable(1)) for _ in range(10000)]
    st = _sorter_case(recs, 4, O.CMP_TEXT, SUM_INT, rle=T.RLE_AUTO)
    assert st["rle_used"] == 1 and st["adjacent_equal_keys"] > 1000


# ------------------------------------------------------------------------------------------------ sorter, fixed width
def _fixed_records(kind, n, klen, combiner, seed):
    """n packed records: big-endian signed key of klen bytes, value of the combiner's width"""
    rng = np.random.default_rng(seed)
    if kind == "zipf":
        k = np.minimum(rng.zipf(1.2, n), 1 << 40).astype(np.int64) * 7919 - (1 << 30)
    elif kind == "few":
        k = rng.integers(-3, 3, n).astype(np.int64)
    elif kind == "hot":
        k = np.where(rng.random(n) < 0.97, 42, rng.integers(0, 1000, n)).astype(np.int64)
    else:
        k = rng.permutation(n).astype(np.int64) * 3 - n
    w = W[combiner]
    v = rng.integers(0, 1 << 62, n, dtype=np.int64).astype(np.uint64) * np.uint64(3)   # sums wrap
    kb = k.astype(">i8").view(np.uint8).reshape(n, 8)[:, 8 - klen:]
    vb = (v & np.uint64((1 << (8 * w)) - 1)).astype(">u8").view(np.uint8).reshape(n, 8)[:, 8 - w:]
    return np.ascontiguousarray(np.concatenate([kb, vb], axis=1)).reshape(-1), k, v


def _fixed_expected(kv, n, klen, combiner, P, cmp_kind, partition=None):
    """numpy combine of packed fixed records, then the oracle sort of the (unique) combined records"""
    w = W[combiner]
    rows = kv.reshape(n, klen + w)
    keys = np.ascontiguousarray(rows[:, :klen]).view(np.dtype((np.void, klen))).ravel()
    vals = np.zeros(n, np.uint64)
    for b in range(w):
        vals = (vals << np.uint64(8)) | rows[:, klen + b].astype(np.uint64)
    if partition is None:
        uk, first, inv = np.unique(keys, return_index=True, return_inverse=True)
        up = None
    else:
        comb = np.rec.fromarrays([partition.astype(np.int64), keys], names="p,k")
        u, first, inv = np.unique(comb, return_index=True, return_inverse=True)
        up = partition[first]
    sums = np.zeros(len(first), np.uint64)
    np.add.at(sums, inv.ravel(), vals)
    m = len(first)
    sb = (sums & np.uint64((1 << (8 * w)) - 1)).astype(">u8").view(np.uint8).reshape(m, 8)[:, 8 - w:]
    out = np.ascontiguousarray(np.concatenate([rows[first, :klen], sb], axis=1)).reshape(-1)
    stride = klen + w
    ko = np.arange(m, dtype=np.uint64) * stride
    conf = O.sorter_conf(P, cmp_kind=cmp_kind, partitioner=O.PART_GIVEN if up is not None else O.PART_HASH, rle_policy=0)
    exp = O.pipelined_sort(conf, out, ko, np.full(m, klen, np.uint32), np.full(m, w, np.uint32), up)
    return exp, m


@pytest.mark.parametrize("path", ["collect_fixed", "device"])
@pytest.mark.parametrize("kind,n", [("few", 0), ("few", 1), ("few", 100000), ("zipf", 1_000_000), ("unique", 1_000_000),
                                    ("zipf", 10_000_000), ("unique", 10_000_000)])
@pytest.mark.parametrize("P", [64])
def test_fixed_long_long_bit_exact(path, kind, n, P):
    """LongWritable key + LongWritable value (16-byte stride), LongSumReducer; the all-unique inputs take the identity
    shortcut (only the widths are checked)."""
    kv, _, _ = _fixed_records(kind, n, 8, SUM_LONG, seed=n + len(kind))
    exp, m = _fixed_expected(kv, n, 8, SUM_LONG, P, O.CMP_LONG)
    with T.GpuSorter(P, comparator=T.CMP_LONG, fixed=(8, 8), combiner=SUM_LONG) as s:
        if path == "collect_fixed":
            s.collect_fixed(kv)
            out, index_bytes, index, st = s.flush_to_memory()
            out = bytes(out)
        else:
            d_kv = torch.from_numpy(kv).cuda() if n else torch.zeros(16, dtype=torch.uint8, device="cuda")
            cap = n * 28 + 10 * P + 64
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            ln, index, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
            out = d_out[:ln].cpu().numpy().tobytes()
    assert out == exp["file_out"]
    assert np.array_equal(index, exp["index"])
    assert st["output_records"] == n and st["spilled_records"] == m
    if kind == "unique":
        assert m == n


@pytest.mark.parametrize("P,given", [(1, False), (64, True), (1024, False)])
def test_fixed_int_int_given_and_hash(P, given):
    """IntWritable key + IntWritable value (8-byte stride), IntSumReducer; GIVEN partitions split equal keys."""
    n = 300000
    kv, _, _ = _fixed_records("zipf", n, 4, SUM_INT, seed=P)
    part = np.random.default_rng(P).integers(0, P, n).astype(np.int32) if given else None
    exp, m = _fixed_expected(kv, n, 4, SUM_INT, P, O.CMP_INT, part)
    with T.GpuSorter(P, comparator=T.CMP_INT, partitioner=T.PART_GIVEN if given else T.PART_HASH, fixed=(4, 4),
                     combiner=SUM_INT) as s:
        s.collect_fixed(kv, part)
        out, index_bytes, index, st = s.flush_to_memory()
    assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]
    assert st["spilled_records"] == m


def test_one_hot_key_across_many_ctas():
    """One key repeated 3e6 times among 1e5 others: its sum spans thousands of warps and CTAs."""
    n = 3_100_000
    kv, k, _ = _fixed_records("hot", n, 8, SUM_LONG, seed=9)
    assert (k == 42).sum() > 2_000_000
    exp, m = _fixed_expected(kv, n, 8, SUM_LONG, 64, O.CMP_LONG)
    with T.GpuSorter(64, comparator=T.CMP_LONG, fixed=(8, 8), combiner=SUM_LONG) as s:
        s.collect_fixed(kv)
        out, index_bytes, index, st = s.flush_to_memory()
    assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]


def test_int_sums_overflow_and_wrap():
    recs = [(O.text("a"), O.int_writable(0x7FFFFFFF))] * 3 + [(O.text("b"), O.int_writable(-5))] * 4
    _sorter_case(recs, 1, O.CMP_TEXT, SUM_INT)
    with T.GpuSorter(1, comparator=T.CMP_TEXT, combiner=SUM_INT) as s:
        kv, ko, kl, vl, vo = CM.pack(recs)
        s.collect(kv, ko.astype(np.uint32), vo, vl)
        out = bytes(s.flush_to_memory()[0])
    assert [(k, v) for _, k, v in O.read_ifile(out)] == [(O.text("a"), O.int_writable(0x7FFFFFFD)),
                                                        (O.text("b"), O.int_writable(-20))]


@pytest.mark.parametrize("dups", [True, False])
def test_bad_value_width_fails_then_handle_works_after_reset(dups):
    rng = random.Random(1)
    good = [(_key(O.CMP_TEXT, rng.randrange(30 if dups else 10 ** 9)), O.int_writable(1)) for _ in range(2000)]
    bad = good[:700] + [(O.text("x"), b"\0\0\0\0\0\0\0\1")] + good[700:]
    with T.GpuSorter(8, comparator=T.CMP_TEXT, combiner=SUM_INT) as s:
        kv, ko, kl, vl, vo = CM.pack(bad)
        s.collect(kv, ko.astype(np.uint32), vo, vl)
        with pytest.raises(TezGpuError) as e:
            s.flush_to_memory()
        assert e.value.code == T.E_INVALID and "record 700" in str(e.value)
        s.reset()
        kv, ko, kl, vl, vo = CM.pack(good)
        s.collect(kv, ko.astype(np.uint32), vo, vl)
        out, index_bytes, _, _ = s.flush_to_memory()
    exp = CM.sort_combine(8, O.CMP_TEXT, SUM_INT, *CM.pack(good)[:4])
    assert bytes(out) == exp["file_out"] and index_bytes == exp["index_out"]


def test_combiner_rejected_where_it_cannot_run():
    with pytest.raises(TezGpuError) as e:
        T.GpuSorter(4, unordered=True, combiner=SUM_INT)
    assert e.value.code == T.E_INVALID
    with pytest.raises(TezGpuError) as e:
        T.GpuSorter(4, fixed=(8, 4), combiner=SUM_LONG)
    assert e.value.code == T.E_INVALID
    with T.GpuSorter(4, fixed=(8, 8)) as s:
        s.collect_fixed(np.zeros(32, np.uint8))
        with pytest.raises(TezGpuError) as e:
            s.set_combiner(SUM_LONG)
        assert e.value.code == T.E_STATE


# ------------------------------------------------------------------------------------------------ merger
def _text_segments(nseg, rng, rle, vw, nkeys=200, nrec=3000):
    segs, recs_all = [], []
    for _ in range(nseg):
        keys = sorted((O.text("k%d" % rng.randrange(nkeys)) for _ in range(nrec)), key=lambda k: k[1:])
        recs = [(k, rng.getrandbits(8 * vw).to_bytes(vw, "big")) for k in keys]
        recs_all += recs
        segs.append(O.write_ifile(recs, rle=rle)[0])
    return segs, recs_all


@pytest.mark.parametrize("rle_inputs", [False, True])
@pytest.mark.parametrize("check_same", [True, False])
@pytest.mark.parametrize("writer_rle", [False, True])
def test_merger_write_ifile_variable_framing(rle_inputs, check_same, writer_rle):
    rng = random.Random(int(rle_inputs) * 4 + int(check_same) * 2 + int(writer_rle))
    segs, _ = _text_segments(6, rng, rle_inputs, 4)
    exp = CM.merge_combine(segs, O.CMP_TEXT, SUM_INT)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, combiner=SUM_INT) as m:
        m.set_check_for_same_keys(check_same)
        seg, raw, part, st = m.write_ifile(rle=writer_rle)
        with pytest.raises(TezGpuError) as e:
            list(m.records())
        assert e.value.code == T.E_STATE
    assert seg == exp[0] and (raw, part) == (exp[1], exp[2])
    assert st["output_records"] == 6 * 3000 and st["spilled_records"] == len(O.read_ifile(exp[0]))


def test_merger_fixed_framing_run_table():
    """LongWritable keys / values written without repeats: the merge addresses the records through the run table."""
    rng = np.random.default_rng(4)
    segs = []
    for _ in range(8):
        k = np.sort(rng.integers(-500, 500, 20000))
        recs = [(O.long_writable(int(x)), O.long_writable(int(y))) for x, y in zip(k, rng.integers(-(1 << 62), 1 << 62, len(k)))]
        segs.append(O.write_ifile(recs)[0])
    exp = CM.merge_combine(segs, O.CMP_LONG, SUM_LONG)
    with T.GpuMerger(segs, comparator=T.CMP_LONG, fixed=(8, 8), combiner=SUM_LONG) as m:
        assert m.parse_info()[0] == 0
        seg, raw, part, st = m.write_ifile(rle=True)
        seg2 = m.write_ifile(rle=False)[0]      # the merger can write again
    assert seg == exp[0] == seg2
    assert st["spilled_records"] == 1000


def test_merger_bad_width_and_fixed_mismatch():
    rng = random.Random(2)
    segs, _ = _text_segments(3, rng, False, 8)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, combiner=SUM_INT) as m:
        with pytest.raises(TezGpuError) as e:
            m.write_ifile()
        assert e.value.code == T.E_INVALID
    with pytest.raises(TezGpuError) as e:
        T.GpuMerger(segs, comparator=T.CMP_TEXT, fixed=(3, 8), combiner=SUM_INT)
    assert e.value.code == T.E_INVALID


@pytest.mark.parametrize("rle_inputs", [False, True])
def test_merger_write_partitions_device(rle_inputs):
    P = 5
    rng = random.Random(11)
    segs, parts, exp = [], [], []
    for p in range(P):
        s, _ = _text_segments(3, rng, rle_inputs, 8, nkeys=50 + p, nrec=1000)
        segs += s
        parts += [p] * 3
        exp.append(CM.merge_combine(s, O.CMP_TEXT, SUM_LONG))
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P, combiner=SUM_LONG) as m:
        cap = m.output_bound()
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        ln, index, st = m.write_partitions_device(d_out.data_ptr(), cap, rle=True)
        got = d_out[:ln].cpu().numpy().tobytes()
    off = 0
    for p in range(P):
        assert tuple(index[p]) == (off, exp[p][1], exp[p][2])
        assert got[off:off + exp[p][2]] == exp[p][0]
        off += exp[p][2]
    assert ln == off


# ------------------------------------------------------------------------------------------------ plugin level
COMBINE_CONF = {"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE,
                "tez.runtime.combiner.class": "org.apache.tez.mapreduce.combine.MRCombiner",
                "mapred.mapper.new-api": True,
                "mapreduce.job.combine.class": "org.apache.hadoop.mapreduce.lib.reduce.IntSumReducer"}


def _word_records(n, seed):
    rng = random.Random(seed)
    words = ["w%d" % min(int(rng.paretovariate(1.05)), 30000) for _ in range(n)]
    return [(O.text(w), O.int_writable(1)) for w in words], collections.Counter(words)


def _run(tmp, conf, recs, P):
    out = OrderedPartitionedKVOutput(OutputContext(conf, str(tmp)), P)
    out.initialize()
    out.start()
    w = out.getWriter()
    for k, v in recs:
        w.write(k, v)
    return out, out.close()


def _file_sums(out, P):
    data = open(out.final_output_file, "rb").read()
    idx = np.frombuffer(open(out.final_index_file, "rb").read()[:-8], dtype=">i8").reshape(P, 3)
    sums, keys = collections.Counter(), []
    for p in range(P):
        for _, k, v in O.read_ifile(data[idx[p, 0]:idx[p, 0] + idx[p, 2]]):
            sums[k[1:].decode()] += int.from_bytes(v, "big", signed=True)
            keys.append(k)
    return sums, keys


def test_plugin_single_spill_files_and_counters(tmp_path):
    P = 6
    recs, counts = _word_records(50000, 1)
    out, events = _run(tmp_path, COMBINE_CONF, recs, P)
    assert out.num_spills == 1
    exp = CM.sort_combine(P, O.CMP_TEXT, SUM_INT, *CM.pack(recs)[:4])
    assert open(out.final_output_file, "rb").read() == exp["file_out"]
    assert open(out.final_index_file, "rb").read() == exp["index_out"]
    assert out.counter("OUTPUT_RECORDS") == len(recs)
    assert out.counter("COMBINE_INPUT_RECORDS") == len(recs)
    assert out.counter("COMBINE_OUTPUT_RECORDS") == out.counter("SPILLED_RECORDS") == len(counts)


@pytest.mark.parametrize("old_api", [False, True])
def test_plugin_other_reducer_configs(tmp_path, old_api):
    """The old API reads mapred.combiner.class; LongSumReducer over LongWritable; a reducer outside the closed set
    (or a value class it does not sum) is not run, as before."""
    conf = {"tez.runtime.key.class": TEXT, "tez.runtime.value.class": LONG_WRITABLE,
            "tez.runtime.combiner.class": "org.apache.tez.mapreduce.combine.MRCombiner",
            "mapred.mapper.new-api": not old_api}
    red = "org.apache.hadoop.mapred.lib.LongSumReducer" if old_api else "org.apache.hadoop.mapreduce.lib.reduce.LongSumReducer"
    conf["mapred.combiner.class" if old_api else "mapreduce.job.combine.class"] = red
    recs = [(O.text("w%d" % (i % 10)), O.long_writable(i)) for i in range(1000)]
    out, _ = _run(tmp_path / "a", conf, recs, 2)
    assert out.counter("COMBINE_OUTPUT_RECORDS") == 10 and out.counter("SPILLED_RECORDS") == 10
    conf[("mapred.combiner.class" if old_api else "mapreduce.job.combine.class")] = "org.example.TopKReducer"
    out, _ = _run(tmp_path / "b", conf, recs, 2)
    assert out.counter("COMBINE_INPUT_RECORDS") == 0 and out.counter("SPILLED_RECORDS") == 1000


@pytest.mark.parametrize("n,min_spills", [(160000, None), (160000, 2), (420000, None)])
def test_plugin_multi_spill_final_merge(tmp_path, n, min_spills):
    """The final merge combines from tez.runtime.combine.min.spills spills on (default 3, PipelinedSorter.java:815)."""
    P = 4
    recs, counts = _word_records(n, n)
    conf = dict(COMBINE_CONF, **{"tez.runtime.io.sort.mb": 1})
    if min_spills:
        conf["tez.runtime.combine.min.spills"] = min_spills
    out, events = _run(tmp_path, conf, recs, P)
    S = out.num_spills
    assert S >= (3 if n > 400000 else 2)
    combined_final = S >= (min_spills or 3)
    sums, keys = _file_sums(out, P)
    assert sums == counts
    spilled_out = out.counter("SPILLED_RECORDS")
    if combined_final:
        exp = CM.sort_combine(P, O.CMP_TEXT, SUM_INT, *CM.pack(recs)[:4])
        assert open(out.final_output_file, "rb").read() == exp["file_out"]
        assert open(out.final_index_file, "rb").read() == exp["index_out"]
        spill_out = spilled_out - len(counts)
        assert out.counter("COMBINE_INPUT_RECORDS") == n + spill_out
        assert out.counter("COMBINE_OUTPUT_RECORDS") == spilled_out
    else:
        # the final merge is not combined: keys repeat across the two spills, written as the merge writes them
        assert len(keys) > len(counts)
        assert out.counter("COMBINE_INPUT_RECORDS") == n
        assert spilled_out == 2 * out.counter("COMBINE_OUTPUT_RECORDS")
    assert out.counter("OUTPUT_RECORDS") == n
    # the consumer's per-key sums equal a Counter over the input
    got = collections.Counter()
    for p in range(P):
        empty = p in empty_partitions_from_payload(events[-1].payload, P)
        inp2 = OrderedGroupedKVInput(InputContext(COMBINE_CONF, str(tmp_path / ("r%d" % p))), 1)
        inp2.initialize()
        inp2.start()
        inp2.handleEvents([LocalOutput(0, out.final_output_file, out.final_index_file, p, empty=empty)])
        r = inp2.getReader()
        while r.next():
            got[r.getCurrentKey()[1:].decode()] += sum(int.from_bytes(v, "big", signed=True) for v in r.getCurrentValues())
    assert got == counts

"""GPU: the plugin classes end to end (C++ host layer over the CUDA library), in the style of the reference's
TestOnFileSortedOutput / TestOrderedPartitionedKVOutput2 / TestOrderedGroupedKVInput / TestTezJobs.testOrderedWordCount."""
import os
import random
import stat
import zlib

import numpy as np
import pytest

from oracle import tez_oracle as O
import merge_scenarios as MS
import tez_b200 as T
from tez_b200.runtime_library import (BYTES_WRITABLE, INT_WRITABLE, LONG_WRITABLE, TEXT, TEZ_BYTES_COMPARATOR, InputContext,
                                      LocalOutput, OrderedGroupedKVInput, OrderedPartitionedKVOutput, OutputContext,
                                      empty_partitions_from_payload, parse_proto)
from plugin_runs import consume, run_output

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("sorter", ["PIPELINED", "LEGACY"])
@pytest.mark.parametrize("send_empty", [True, False])
def test_output_lifecycle_files_events_counters(tmp_path, sorter, send_empty):
    """TestOnFileSortedOutput.baseTest (RLT/output/TestOnFileSortedOutput.java:156-250) shape."""
    rng = random.Random(1)
    P = 10
    words = ["w%03d" % rng.randint(0, 400) for _ in range(3000)]
    recs = [(O.text(w), O.int_writable(1)) for w in words]
    conf = {"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE, "tez.runtime.sorter.class": sorter,
            "tez.runtime.empty.partitions.info-via-events.enabled": send_empty,
            "tez.runtime.report.partition.stats": "precise"}
    out, events = run_output(tmp_path, conf, recs, P)
    # files: output/<uid>/file.out + .index, mode 0640 (TezTaskOutputFiles, TezSpillRecord.SPILL_FILE_PERMS)
    f, fi = out.final_output_file, out.final_index_file
    assert f == str(tmp_path / "output" / out.context.unique_identifier / "file.out") and fi == f + ".index"
    assert stat.S_IMODE(os.stat(f).st_mode) == 0o640 and stat.S_IMODE(os.stat(fi).st_mode) == 0o640
    assert out.num_spills == 1
    # bytes == oracle (RLE decision: PIPELINED turns RLE on for this duplication level, LEGACY never does)
    kv = b"".join(k + v for k, v in recs)
    ko = np.cumsum([0] + [len(k) + len(v) for k, v in recs[:-1]])
    exp = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT, send_empty=send_empty, legacy=(sorter == "LEGACY")), kv, ko,
                           [len(k) for k, _ in recs], [len(v) for _, v in recs])
    assert open(f, "rb").read() == exp["file_out"]
    assert open(fi, "rb").read() == exp["index_out"]
    assert exp["rle_used"] == (sorter == "PIPELINED")
    # counters (verifyCounters, RLT/common/sort/impl/TestPipelinedSorter.java:593-626)
    c = exp["counters"]
    for name in ("OUTPUT_RECORDS", "OUTPUT_BYTES", "OUTPUT_BYTES_WITH_OVERHEAD", "OUTPUT_BYTES_PHYSICAL", "SPILLED_RECORDS"):
        assert out.counter(name) == c[name], name
    assert out.counter("ADDITIONAL_SPILL_COUNT") == 0 and out.counter("SHUFFLE_CHUNK_COUNT") == 1
    # events: VertexManagerEvent + CompositeDataMovementEvent(0, P) (ShuffleUtils.generateEventOnSpill)
    assert [e.type for e in events] == ["VertexManagerEvent", "CompositeDataMovementEvent"]
    vm = parse_proto(events[0].payload)
    assert vm[1][0] == c["OUTPUT_BYTES"] and vm[4][0] == len(recs)
    sizes_mb = list(parse_proto(vm[3][0])[1][0])
    assert len(sizes_mb) == P and all(s in (0, 1) for s in sizes_mb)
    dm = parse_proto(events[1].payload)
    assert (events[1].source_index_start, events[1].count) == (0, P)
    assert dm[2][0] == b"localhost" and dm[3][0] == 13562 and dm[4][0] == out.context.unique_identifier.encode()
    empties = {p for p in range(P) if not exp["index"][p, 1] > 6}
    if send_empty:
        assert empty_partitions_from_payload(events[1].payload, P) == empties
    else:
        assert 1 not in dm


def test_multiple_spills_and_final_merge_match_single_sort(tmp_path):
    """PipelinedSorter multi-spill + final merge (SORT/PipelinedSorter.java:774-836): unique keys => the final
    file.out is byte-identical to a single sort; ADDITIONAL_SPILL_COUNT / SHUFFLE_CHUNK_COUNT as verifyCounters."""
    n, P = 60000, 8
    kv = O.gen_c2(0, n, seed=7)
    rows = kv.reshape(n, 80)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in rows]
    conf = {"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
            "tez.runtime.io.sort.mb": 1}
    out, events = run_output(tmp_path, conf, recs, P)
    assert out.num_spills >= 4
    exp = O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, 64)
    assert open(out.final_output_file, "rb").read() == exp["file_out"]
    assert open(out.final_index_file, "rb").read() == exp["index_out"]
    assert out.counter("ADDITIONAL_SPILL_COUNT") == out.num_spills - 1
    assert out.counter("SHUFFLE_CHUNK_COUNT") == 1
    assert out.counter("OUTPUT_RECORDS") == n
    assert out.counter("SPILLED_RECORDS") == 2 * n           # every record spilled once and merged once
    assert out.counter("ADDITIONAL_SPILLS_BYTES_READ") > 0 and out.counter("ADDITIONAL_SPILLS_BYTES_WRITTEN") > 0
    assert out.counter("OUTPUT_BYTES_PHYSICAL") == len(exp["file_out"])
    assert not os.path.exists(str(tmp_path / "output" / (out.context.unique_identifier + "_0")))   # spill dirs removed


@pytest.mark.parametrize("key_class,comparator_class,cmp", [
    (TEXT, None, O.CMP_TEXT), (INT_WRITABLE, None, O.CMP_INT), (LONG_WRITABLE, None, O.CMP_LONG),
    (BYTES_WRITABLE, TEZ_BYTES_COMPARATOR, O.CMP_BYTES), (BYTES_WRITABLE, None, O.CMP_BYTESWRITABLE)],
    ids=["text", "int", "long", "byteswritable-tezbytes", "byteswritable"])
def test_final_merge_of_every_key_class_matches_single_sort(tmp_path, key_class, comparator_class, cmp):
    """The final merge of 4+ spills with the device comparator of every key class: the palette keys of
    tests/merge_scenarios.py (raw byte order and comparator order disagree) and random keys, each once, value = f(key),
    so file.out and file.out.index equal the oracle's single sort with that comparator"""
    rng = random.Random(cmp)
    keys = list(MS.PALETTES[cmp])
    seen = set(keys)
    while len(keys) < 70000:
        k = MS._random_key(rng, cmp, False)
        if k not in seen:
            seen.add(k)
            keys.append(k)
    rng.shuffle(keys)
    recs = [(k, zlib.crc32(k).to_bytes(4, "big") * 15) for k in keys]
    P = 8
    conf = {"tez.runtime.key.class": key_class, "tez.runtime.io.sort.mb": 1}
    if comparator_class:
        conf["tez.runtime.key.comparator.class"] = comparator_class
    out, events = run_output(tmp_path, conf, recs, P)
    assert out.num_spills >= 4
    kv = b"".join(k + v for k, v in recs)
    ko = np.cumsum([0] + [len(k) + len(v) for k, v in recs[:-1]])
    exp = O.pipelined_sort(O.sorter_conf(P, cmp_kind=cmp), kv, ko, [len(k) for k, _ in recs], [len(v) for _, v in recs])
    assert not exp["rle_used"]
    assert open(out.final_output_file, "rb").read() == exp["file_out"]
    assert open(out.final_index_file, "rb").read() == exp["index_out"]
    assert out.counter("OUTPUT_RECORDS") == len(recs) and out.counter("SPILLED_RECORDS") == 2 * len(recs)


@pytest.mark.parametrize("dup_pct", [1, 5, 9, 30])
def test_multi_spill_final_merge_with_duplicate_keys(tmp_path, dup_pct):
    """PipelinedSorter.flush final merge with duplicate keys (SORT/PipelinedSorter.java:797-814): checkForSameKeys AND the
    writer's rle are both merger.needsRLE() of the last spill.  <= 10 % duplicates: no spill and no merge output is
    run-length encoded (no FE/FD markers at all); 30 %: every adjacent equal key is.  value = f(key), so the bytes are
    determined; the oracle's single-span sorter gives the same RLE decision at these levels (eq = 1.03 x duplicates)."""
    n, P = 60000, 8
    rng = random.Random(dup_pct)
    nd = n * dup_pct // 100
    base = [bytes(r[:16]) for r in O.gen_c2(0, n - nd, seed=17).reshape(-1, 80)]
    # duplicates stay close to their originals (shuffled inside blocks of 500 records), so every spill sees the same
    # duplicate fraction as the whole input: the RLE decision is per spill (SpanMerger.needsRLE of that spill's sort)
    keys = []
    for blk in range(0, len(base), 500):
        part = base[blk:blk + 500]
        part = part + [part[rng.randrange(len(part))] for _ in range(len(part) * nd // len(base))]
        rng.shuffle(part)
        keys += part
    n = len(keys)
    recs = [(k, zlib.crc32(k).to_bytes(4, "big") * 16) for k in keys]
    conf = {"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
            "tez.runtime.io.sort.mb": 1}
    out, events = run_output(tmp_path, conf, recs, P)
    assert out.num_spills >= 4
    kv = np.frombuffer(b"".join(k + v for k, v in recs), dtype=np.uint8)
    rle = dup_pct > 10
    exp = O.pipelined_sort_fixed(O.sorter_conf(P, rle_policy=1 if rle else 0), kv, 16, 64)
    got = open(out.final_output_file, "rb").read()
    assert got == exp["file_out"]
    assert open(out.final_index_file, "rb").read() == exp["index_out"]
    idx = np.frombuffer(open(out.final_index_file, "rb").read()[:-8], dtype=">i8").reshape(P, 3)
    states = [ks for p in range(P) for ks, _, _ in O.read_ifile(got[idx[p, 0]:idx[p, 0] + idx[p, 2]])]
    assert len(states) == n and (O.SAME_KEY in states) == rle      # <= 10 %: not one RLE / V_END marker in file.out
    assert out.counter("OUTPUT_RECORDS") == n and out.counter("SPILLED_RECORDS") == 2 * n


def test_pipelined_shuffle_spill_events_reach_the_input(tmp_path):
    """tez.runtime.enable.final-merge.in.output=false: one CompositeDataMovementEvent per spill (spill_id, last_event);
    the input must fetch EVERY spill of a producer and only then report ready (OG/ShuffleScheduler.java:540-600)."""
    n, P = 40000, 4
    kv = O.gen_c2(0, n, seed=23)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = {"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
            "tez.runtime.io.sort.mb": 1, "tez.runtime.enable.final-merge.in.output": False,
            "tez.runtime.report.partition.stats": "precise"}
    out, events = run_output(tmp_path, conf, recs, P)
    S = out.num_spills
    assert S >= 3
    dms = [e for e in events if e.type == "CompositeDataMovementEvent"]
    assert len(dms) == S
    spill_ids = [parse_proto(e.payload)[9][0] for e in dms]
    lasts = [parse_proto(e.payload)[8][0] for e in dms]
    assert spill_ids == list(range(S)) and lasts == [0] * (S - 1) + [1]
    # the single VertexManagerEvent reports the sizes accumulated over every spill (partitionStats)
    vms = [e for e in events if e.type == "VertexManagerEvent"]
    assert len(vms) == 1
    sizes_mb = list(parse_proto(parse_proto(vms[0].payload)[3][0])[1][0])
    uid = out.context.unique_identifier
    files = [str(tmp_path / "output" / ("%s_%d" % (uid, s)) / "file.out") for s in range(S)]
    idxs = [np.frombuffer(open(f + ".index", "rb").read()[:-8], dtype=">i8").reshape(P, 3) for f in files]
    total_raw = sum(ix[:, 1] for ix in idxs)
    assert sizes_mb == [int((r + (1 << 20) - 1) >> 20) for r in total_raw]
    p = 2
    inp = OrderedGroupedKVInput(InputContext(conf, str(tmp_path / "r")), 1)
    inp.initialize()
    inp.start()
    order = list(range(S))
    random.Random(5).shuffle(order)          # events may arrive in any order; duplicates are ignored
    for k, s_id in enumerate(order):
        lo = LocalOutput(0, files[s_id], files[s_id] + ".index", p, spill_id=s_id, last_event=(s_id == S - 1))
        if k < S - 1:
            inp.handleEvents([lo, lo])
            with pytest.raises(IOError, match="have not been delivered"):
                inp.waitForInputReady()
        else:
            inp.handleEvents([lo])
    r = inp.getReader()
    got = []
    while r.next():
        got.append((r.getCurrentKey(), list(r.getCurrentValues())))
    mine = sorted((k, v) for k, v in recs if O.partition_of(O.CMP_BYTES, k, P) == p)
    assert [(k, vs[0]) for k, vs in got] == mine and all(len(vs) == 1 for _, vs in got)
    assert inp.counter("NUM_SHUFFLED_INPUTS") == S


def test_custom_partitioner_results_are_passed_through(tmp_path):
    conf = {"tez.runtime.key.class": INT_WRITABLE, "tez.runtime.partitioner.class": "org.example.RangePartitioner"}
    ctx = OutputContext(conf, str(tmp_path))
    out = OrderedPartitionedKVOutput(ctx, 3)
    out.initialize()
    out.start()
    w = out.getWriter()
    with pytest.raises(IOError, match="custom partitioner"):
        w.write(O.int_writable(5), b"x")
    vals = list(range(-50, 50))
    random.Random(2).shuffle(vals)
    for v in vals:
        w.write(O.int_writable(v), b"v%d" % v, partition=0 if v < -10 else (1 if v < 10 else 2))
    with pytest.raises(IOError, match="Illegal partition"):
        w.write(O.int_writable(1), b"x", partition=3)
    out.close()
    data = open(out.final_output_file, "rb").read()
    idx = np.frombuffer(open(out.final_index_file, "rb").read()[:-8], dtype=">i8").reshape(3, 3)
    got = []
    for p in range(3):
        seg = data[idx[p, 0]:idx[p, 0] + idx[p, 2]]
        got.append([int.from_bytes(k, "big", signed=True) for _, k, _ in O.read_ifile(seg)])
    assert got == [list(range(-50, -10)), list(range(-10, 10)), list(range(10, 50))]


def test_ordered_word_count_two_edges(tmp_path):
    """TestTezJobs.testOrderedWordCount (tez-tests/.../TestTezJobs.java:748-854): words a_1..a_10 with counts 20,18,..,2;
    tokenizer -> (word,1) -> summation -> (count, word) -> sorter: final order by count then the known answer."""
    words = []
    for i in range(1, 11):
        words += ["a_%d" % i] * (22 - 2 * i)
    random.Random(3).shuffle(words)
    P = 4
    conf1 = {"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE}
    producers = []
    for t in range(3):                                   # three tokenizer tasks
        mine = words[t::3]
        producers.append(run_output(tmp_path / ("t%d" % t), conf1, [(O.text(w), O.int_writable(1)) for w in mine], P,
                                     uid="attempt_1_0001_1_00_%06d_0_10001" % t))
    counts = {}
    records_seen = 0
    for p in range(P):                                   # P summation tasks
        inp, groups = consume(tmp_path / ("s%d" % p), conf1, producers, p, P)
        for k, vals in groups:
            word = k[1:].decode()
            assert word not in counts
            counts[word] = sum(int.from_bytes(v, "big") for v in vals)
            records_seen += len(vals)
        assert inp.counter("REDUCE_INPUT_GROUPS") == len(groups)
        assert inp.counter("REDUCE_INPUT_RECORDS") == sum(len(v) for _, v in groups)
    assert records_seen == len(words)
    assert counts == {"a_%d" % i: 22 - 2 * i for i in range(1, 11)}
    # second edge: (IntWritable count, Text word), one reducer (OrderedWordCount.java:156-160)
    conf2 = {"tez.runtime.key.class": INT_WRITABLE, "tez.runtime.value.class": TEXT}
    prod2 = [run_output(tmp_path / "sum", conf2, [(O.int_writable(c), O.text(w)) for w, c in counts.items()], 1,
                         uid="attempt_1_0001_1_01_000000_0_10001")]
    _, groups = consume(tmp_path / "sorter", conf2, prod2, 0, 1)
    final = [(int.from_bytes(k, "big", signed=True), v[0][1:].decode()) for k, v in groups]
    assert final == [(22 - 2 * i, "a_%d" % i) for i in range(10, 0, -1)]


def test_input_groups_values_across_producers_and_skips_empty(tmp_path):
    P = 3
    conf = {"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR}
    rng = random.Random(9)
    producers, expect = [], {}
    for t in range(5):
        recs = []
        for _ in range(rng.randint(0, 300) if t != 2 else 0):        # producer 2 writes nothing at all
            k = bytes([rng.randint(0, 40)]) * rng.randint(1, 3)
            v = zlib.crc32(k).to_bytes(4, "big") + bytes([t])
            recs.append((k, v))
        producers.append(run_output(tmp_path / ("m%d" % t), conf, recs, P, uid="attempt_1_0001_1_00_%06d_0_1" % t))
        for k, v in recs:
            if O.partition_of(O.CMP_BYTES, k, P) == 1:
                expect.setdefault(k, []).append(v)
    inp, groups = consume(tmp_path / "r1", conf, producers, 1, P)
    assert [k for k, _ in groups] == sorted(expect)
    for k, vals in groups:
        assert sorted(vals) == sorted(expect[k])
    assert inp.counter("NUM_SKIPPED_INPUTS") >= 1
    assert inp.counter("NUM_SHUFFLED_INPUTS") + inp.counter("NUM_SKIPPED_INPUTS") == 5
    assert inp.counter("REDUCE_INPUT_GROUPS") == len(expect)

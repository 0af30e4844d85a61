"""GPU tests of the unordered edge end to end: tezgpu_concat_open (UnorderedPartitionedKVWriter.mergeAll /
UnorderedKVReader) byte for byte against tests/unordered_model.py, and the plugin mirror's UnorderedPartitionedKVOutput,
UnorderedKVOutput and UnorderedKVInput."""
import random
import zlib

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import _lib
from tez_b200.runtime_library import (InputContext, LocalOutput, OutputContext, UnorderedKVInput, UnorderedKVOutput,
                                      UnorderedPartitionedKVOutput, parse_proto)

import codec_model as CM
import lz4_model as L4
import unordered_model as UM
import zstd_model as ZS

pytestmark = pytest.mark.gpu


def _records(kind, rng, n):
    if kind == "c2":
        return [(rng.randbytes(16), rng.randbytes(64)) for _ in range(n)]
    if kind == "text":
        return [(O.text("w%d" % rng.randrange(10 ** rng.randint(1, 6))), O.int_writable(rng.randrange(1 << 31))) for _ in range(n)]
    return [(O.text("k%d" % rng.randrange(1000)), rng.randbytes(4096)) for _ in range(n)]   # 4 KB values


def _segments(P, runs, kind, seed, max_recs):
    rng = random.Random(seed)
    segs, parts = [], []
    for p in range(P):
        if rng.random() < 0.15:
            continue                                   # a partition without inputs
        for _ in range(runs):
            n = 0 if rng.random() < 0.2 else rng.randint(1, max_recs)   # empty segments too
            segs.append(O.write_ifile(_records(kind, rng, n))[0])
            parts.append(p)
    return segs, parts


def _open(segs, parts, P, mode, **kw):
    """host segments, device segments (packed at arbitrary byte offsets), or device segments marked VERIFIED"""
    if mode == "host":
        return T.GpuMerger(segs, partitions=parts, num_partitions=P, concat=True, **kw), None
    blob = b"".join(segs) or b"\0"
    d = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    offs = np.concatenate([[0], np.cumsum([len(s) for s in segs])[:-1]]).astype(np.int64)
    ptrs = [(d.data_ptr() + int(o), len(s)) for o, s in zip(offs, segs)]
    m = T.GpuMerger(ptrs, device_ptrs=True, partitions=parts, num_partitions=P, concat=True,
                    verified=[mode == "verified"] * len(segs), **kw)
    return m, d


def _write_partitions(m):
    bound = m.output_bound()
    d_out = torch.empty(max(bound, 16), dtype=torch.uint8, device="cuda")
    n, index, st = m.write_partitions_device(d_out.data_ptr(), d_out.numel())
    return d_out[:n].cpu().numpy().tobytes(), [tuple(int(x) for x in r) for r in index], st


@pytest.mark.parametrize("mode", ["host", "device", "verified"])
@pytest.mark.parametrize("kind", ["c2", "text"])
@pytest.mark.parametrize("runs", [1, 2, 9])
@pytest.mark.parametrize("P", [1, 64, 1024])
def test_concat_abi_byte_exact(P, runs, kind, mode):
    max_recs = max(1, 4000 // (P * runs))
    segs, parts = _segments(P, runs, kind, seed=P * 31 + runs, max_recs=max_recs)
    exp_out, exp_index = UM.concat_file(segs, parts, P)
    fixed = (16, 64) if kind == "c2" else None
    m, keep = _open(segs, parts, P, mode, fixed=fixed)
    with m:
        out, index, st = _write_partitions(m)
        assert out == exp_out
        assert index == exp_index
        assert m.parse_info() == (3, 0), "the write must not parse"
        # open: header check, three checksum kernels (not for VERIFIED segments), the input remainders;
        # write: copy (when there are record bytes), combine and finish (when there is a segment).  Nothing else.
        opened = (1 + (0 if mode == "verified" else 3) + 1) if segs else 0
        written = 3 if exp_out else 0
        assert st["kernel_launches"] == opened + written, st
        assert st["output_bytes_with_overhead"] == sum(r for _, r, _ in exp_index)
        order = [r for p in range(P) for r in UM.records([s for s, q in zip(segs, parts) if q == p])]
        got = list(m.records())
        assert [(k, v) for k, v, _ in got] == order
        assert not any(s for _, _, s in got)
        assert m.counts() == (len(order), sum(len(k) + len(v) for k, v in order))
        if segs:   # run table for the declared fixed width, window parser otherwise
            assert m.parse_info()[0] == (0 if kind == "c2" else 1)
    del keep


@pytest.mark.parametrize("runs", [1, 9])
def test_concat_write_ifile_4kb_values(runs):
    segs, _ = _segments(1, runs, "big", seed=runs, max_recs=40)
    exp, raw, part = UM.concat_segment(segs)
    with T.GpuMerger(segs, concat=True) as m:
        seg, r, p, st = m.write_ifile()
        assert (seg, r, p) == (exp, raw, part)
        assert [(k, v) for k, v, _ in m.records(batch_bytes=1 << 16)] == UM.records(segs)


def test_concat_next_batch_one_70mb_segment():
    n = 860000
    kv = O.gen_c2(0, n, seed=9)
    with T.GpuSorter(1, fixed=(16, 64), unordered=True) as s:
        s.collect_fixed(kv)
        out, _, index, _ = s.flush_to_memory()
    seg = bytes(out)
    assert len(seg) > 70_000_000
    small = O.write_ifile([(b"k" * 16, b"v" * 64)])[0]
    with T.GpuMerger([seg, small], fixed=(16, 64), concat=True) as m:
        keys = [k for k, _, _ in m.records()]
    rec = kv.reshape(n, 80)
    assert len(keys) == n + 1 and keys[-1] == b"k" * 16
    got = np.frombuffer(b"".join(keys[:-1]), dtype=np.uint8).reshape(n, 16)
    assert np.array_equal(got, rec[::-1, :16]), "newest first inside the segment, then the next segment"


def _compressed(codec, plain):
    body = CM.body_of(plain)
    raw = len(plain) - 4
    if codec == T.CODEC_DEFAULT:
        z = CM.deflate_emulate(body)
    elif codec == T.CODEC_LZ4:
        z = L4.compress_emulate(body)
    else:
        z = ZS.compress_emulate(body)
    return b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big"), raw


@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_concat_codecs_mixed_with_plain(codec):
    P = 6
    plain, parts = _segments(P, 3, "text", seed=codec, max_recs=3000)
    segs, raws = [], []
    for i, s in enumerate(plain):
        if i % 2 == 0:
            z, r = _compressed(codec, s)
            segs.append(z)
            raws.append(r)
        else:
            segs.append(s)
            raws.append(len(s) - 4)
    with T.GpuMerger(segs, partitions=parts, num_partitions=P, concat=True, codec=codec, raw_lens=raws) as m:
        out, index, st = _write_partitions(m)
        assert m.parse_info()[0] == 3
        assert [(k, v) for k, v, _ in m.records()] == [r for p in range(P) for r in UM.records([s for s, q in zip(plain, parts) if q == p])]
    pos = 0
    for p in range(P):
        exp_seg, raw, _ = UM.concat_segment([s for s, q in zip(plain, parts) if q == p])
        if not exp_seg:
            assert index[p] == (0, 0, 0)
            continue
        exp_z, _ = _compressed(codec, exp_seg)
        assert index[p] == (pos, raw, len(exp_z))
        assert out[pos:pos + len(exp_z)] == exp_z
        pos += len(exp_z)
    assert pos == len(out)


def test_concat_errors_name_their_segment_or_call():
    good = [O.write_ifile([(b"a", b"1"), (b"b", b"2")])[0] for _ in range(3)]
    bad_crc = bytearray(good[1])
    bad_crc[-1] ^= 1
    with pytest.raises(_lib.TezGpuError) as e:
        T.GpuMerger([good[0], bytes(bad_crc), good[2]], concat=True)
    assert e.value.code == T.E_FORMAT and "segment 1" in str(e.value)
    body = good[2][4:-6]                               # records without the EOF marker, with a valid checksum
    no_eof = b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")
    with pytest.raises(_lib.TezGpuError) as e:
        T.GpuMerger([good[0], good[1], no_eof], concat=True)
    assert e.value.code == T.E_FORMAT and "segment 2" in str(e.value) and "EOF" in str(e.value)
    with pytest.raises(_lib.TezGpuError) as e:
        T.GpuMerger([good[0], good[1][:-3]], concat=True)          # truncated
    assert e.value.code == T.E_FORMAT and "segment 1" in str(e.value)
    with T.GpuMerger(good, concat=True) as m:
        with pytest.raises(_lib.TezGpuError) as e:
            m.write_ifile(rle=True)
        assert e.value.code == T.E_INVALID and "rle" in str(e.value)
        with pytest.raises(_lib.TezGpuError) as e:
            m.set_combiner(T.COMBINE_SUM_INT)
        assert e.value.code == T.E_STATE and "tezgpu_merge_set_combiner" in str(e.value)
        with pytest.raises(_lib.TezGpuError) as e:
            m.set_check_for_same_keys(False)
        assert e.value.code == T.E_STATE
        m.reopen(good[:2])                              # reopen keeps the mode
        seg, _, _, _ = m.write_ifile()
        assert seg == UM.concat_segment(good[:2])[0] and m.parse_info()[0] == 3


# ------------------------------------------------------------------------------------------------ plugin mirror
TEXT_CONF = {"tez.runtime.key.class": "org.apache.hadoop.io.Text", "tez.runtime.value.class": "org.apache.hadoop.io.IntWritable"}


def _produce(tmp_path, recs, P, conf=None, cls=UnorderedPartitionedKVOutput, uid="attempt_p_0", mb=None, scale=1.0):
    c = dict(TEXT_CONF, **(conf or {}))
    if mb is not None:
        c["tez.runtime.unordered.output.buffer.size-mb"] = mb
    ctx = OutputContext(conf=c, work_dir=str(tmp_path), unique_identifier=uid, memory_scale=scale)
    out = cls(ctx, P)
    out.initialize()
    out.start()
    w = out.getWriter()
    for k, v in recs:
        w.write(k, v)
    return out, out.close()


def _words(n, seed, vocab=50000):
    rng = random.Random(seed)
    return [(O.text("w%d" % rng.randrange(vocab)), O.int_writable(i)) for i in range(n)]


def _index_of(path, P):
    b = open(path, "rb").read()
    return [tuple(int.from_bytes(b[24 * p + 8 * j:24 * p + 8 * j + 8], "big") for j in range(3)) for p in range(P)]


def _spill_records(out, P):
    """{spill: {partition: records}} of a producer run with the final merge off: its spill files stay in place"""
    res = {}
    for s in range(out.num_spills):
        f = "%s/output/%s_%d/file.out" % (out.context.work_dir, out.context.unique_identifier, s)
        res[s] = UM.partition_records(open(f, "rb").read(), _index_of(f + ".index", P))
    return res


@pytest.mark.parametrize("spills", [1, 2, 5])
def test_unordered_partitioned_output_spills(tmp_path, spills):
    P = 8
    n = 40000 * spills
    recs = _words(n, spills)
    # one spill per ~1 MiB buffer: 40,000 records of ~12 bytes are ~0.5 MiB; a 0.5 scale grant makes 1 MiB hold them
    scale = 0.5 if spills > 1 else 1.0
    out, events = _produce(tmp_path / "merged", recs, P, mb=1, scale=scale)
    assert (out.num_spills > 1) == (spills > 1)
    data = open(out.final_output_file, "rb").read()
    want = {}
    for k, v in recs:
        want.setdefault(O.partition_of(O.CMP_TEXT, k, P), []).append((k, v))
    _, exp_index = UM.concat_file([O.write_ifile(want.get(p, []))[0] for p in range(P)], list(range(P)), P)
    index = _index_of(out.final_index_file, P)
    assert index == exp_index
    got = UM.partition_records(data, index)          # every segment: header, EOF and CRC verified by the oracle
    # The same records with the final merge off spill at the same points and leave every spill in place: the final
    # merge must be mergeAll's order, per partition the current buffer (the last spill), then spills 0 .. n-2.
    kept, _ = _produce(tmp_path / "spills", recs, P, conf={"tez.runtime.enable.final-merge.in.output": False}, mb=1,
                       scale=scale)
    ns = kept.num_spills
    assert ns == out.num_spills
    sp = _spill_records(kept, P)
    for p in range(P):
        exp = [r for s in [ns - 1] + list(range(ns - 1)) for r in sp[s].get(p, [])]
        assert got.get(p, []) == exp, "partition %d" % p
        assert sorted(exp) == sorted(want.get(p, []))
        if ns == 1 and p in want:
            assert got[p] == want[p][::-1], "one buffer: newest first"
    assert out.counter("OUTPUT_RECORDS") == n
    assert out.counter("OUTPUT_BYTES") == sum(len(k) + len(v) for k, v in recs)
    # the current buffer's records are not counted as spilled (UnorderedPartitionedKVWriter.finalSpill)
    assert out.counter("SPILLED_RECORDS") == n - sum(len(r) for r in sp[ns - 1].values())
    kinds = [e.type for e in events]
    assert kinds == ["VertexManagerEvent", "CompositeDataMovementEvent"]
    dm = parse_proto(events[1].payload)
    assert events[1].count == P and 9 not in dm and dm[4][0] == b"attempt_p_0"


def test_unordered_input_reads_spills_in_spill_id_order(tmp_path):
    """A pipelined producer's spill events arrive out of order, interleaved with another source: UnorderedKVInput reads
    the sources in delivery order and one source's spills in spill-id order."""
    P = 3
    recs = _words(120000, 8)
    piped, _ = _produce(tmp_path / "a", recs, P, conf={"tez.runtime.pipelined-shuffle.enabled": True}, mb=1, scale=0.5,
                        uid="attempt_a_0")
    ns = piped.num_spills
    assert ns >= 3
    whole, _ = _produce(tmp_path / "b", _words(5000, 9), P, uid="attempt_b_0")
    sp = _spill_records(piped, P)
    for p in range(P):
        def spill_event(s):
            f = "%s/output/attempt_a_0_%d/file.out" % (tmp_path / "a", s)
            return LocalOutput(0, f, f + ".index", p, spill_id=s, last_event=s == ns - 1)
        events = [spill_event(ns - 1), LocalOutput(1, whole.final_output_file, whole.final_index_file, p)]
        events += [spill_event(s) for s in range(ns - 2, -1, -1)]
        got, inp = _consume_events(tmp_path / ("c%d" % p), events, 2)
        exp = [r for s in range(ns) for r in sp[s].get(p, [])]
        exp += UM.partition_records(open(whole.final_output_file, "rb").read(), _index_of(whole.final_index_file, P)).get(p, [])
        assert got == exp, "partition %d" % p


def test_unordered_pipelined_shuffle_events(tmp_path):
    P = 4
    recs = _words(120000, 3)
    out, events = _produce(tmp_path, recs, P, conf={"tez.runtime.pipelined-shuffle.enabled": True}, mb=1, scale=0.5)
    ns = out.num_spills
    assert ns > 1
    dms = [parse_proto(e.payload) for e in events if e.type == "CompositeDataMovementEvent"]
    assert [d[9][0] for d in dms] == list(range(ns))
    assert [d[8][0] for d in dms] == [0] * (ns - 1) + [1]
    assert [d[4][0] for d in dms] == [("attempt_p_0_%d" % s).encode() for s in range(ns)]


def _consume(tmp_path, outputs, partition, uid):
    """UnorderedKVInput over the final output of every source; returns the records it reads."""
    return _consume_events(tmp_path, [LocalOutput(i, o.final_output_file, o.final_index_file, partition)
                                      for i, o in enumerate(outputs)], len(outputs), uid)


def _consume_events(tmp_path, events, sources, uid="attempt_c_0"):
    ctx = InputContext(conf=dict(TEXT_CONF), work_dir=str(tmp_path), unique_identifier=uid)
    inp = UnorderedKVInput(ctx, sources)
    inp.initialize()
    inp.start()
    inp.handleEvents(events)
    r = inp.getReader()
    got = []
    while r.next():
        got.append((r.getCurrentKey(), r.getCurrentValue()))
    assert inp.counter("INPUT_RECORDS_PROCESSED") == len(got)
    return got, inp


def test_broadcast_into_two_consumers(tmp_path):
    recs = _words(30000, 4)
    out, events = _produce(tmp_path / "p", recs, 2, cls=UnorderedKVOutput)
    dm = parse_proto(events[-1].payload)
    assert events[-1].count == 1 and dm[10][0] == len(recs)    # one writer partition, num_record
    for c in range(2):
        got, inp = _consume(tmp_path / ("c%d" % c), [out], 0, "attempt_c_%d" % c)
        assert got == recs[::-1]
        assert inp.counter("SHUFFLE_BYTES") == len(open(out.final_output_file, "rb").read())


CODECS = {None: {}, "default": {"tez.runtime.compress": True, "tez.runtime.compress.codec": "org.apache.hadoop.io.compress.DefaultCodec"},
          "lz4": {"tez.runtime.compress": True, "tez.runtime.compress.codec": "org.apache.hadoop.io.compress.Lz4Codec"},
          "zstd": {"tez.runtime.compress": True, "tez.runtime.compress.codec": "org.apache.hadoop.io.compress.ZStandardCodec"}}


@pytest.mark.parametrize("codec", list(CODECS))
def test_hash_join_through_partitioned_and_broadcast_edges(tmp_path, codec):
    """HashJoinExample's shape: the big side over an unordered-partitioned edge, the small side broadcast."""
    P = 3
    rng = random.Random(7)
    big = [O.text("k%d" % rng.randrange(20000)) for _ in range(50000)]
    small = sorted({O.text("k%d" % rng.randrange(40000)) for _ in range(3000)})
    conf = dict(CODECS[codec], **{"tez.runtime.value.class": "org.apache.hadoop.io.NullWritable"})
    big_out, _ = _produce(tmp_path / "big", [(k, b"") for k in big], P, conf=conf, mb=1, scale=0.3, uid="attempt_big_0")
    small_out, _ = _produce(tmp_path / "small", [(k, b"") for k in small], 1, conf=conf, cls=UnorderedKVOutput, uid="attempt_small_0")
    joined = set()
    for c in range(P):
        ctx = dict(TEXT_CONF, **conf)
        ins = []
        for name, o, part in (("s", small_out, 0), ("b", big_out, c)):
            inp = UnorderedKVInput(InputContext(conf=ctx, work_dir=str(tmp_path / ("c%d%s" % (c, name)))), 1)
            inp.initialize()
            inp.start()
            inp.handleEvents([LocalOutput(0, o.final_output_file, o.final_index_file, part)])
            ins.append(inp)
        r = ins[0].getReader()
        table = set()
        while r.next():
            table.add(r.getCurrentKey())
        r = ins[1].getReader()
        while r.next():
            if r.getCurrentKey() in table:
                joined.add(r.getCurrentKey())
    assert joined == set(big) & set(small)

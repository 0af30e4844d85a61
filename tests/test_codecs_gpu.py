"""GPU: the cases every IFile codec on the device shares, each run for the codecs of codec_table that have it.  Every
compressed segment the device writes is checked against the uncompressed output of the oracle (or of the same merge
without the codec): header, CRC of the stream, its decode, index triple, and byte for byte against the host emulation
of the writer.  The sorter runs every comparator, RLE, empty partitions, combiners and fixed-width records; the merger
reads foreign-written streams mixed with plain segments, fixed-width runs, partitions on the device, one segment of
hundreds of blocks and malformed or wrong-codec segments; the plugin classes run spills, the pipelined shuffle and
OrderedWordCount through the codec.  The cases of one stream format are in that codec's own suite."""
import random
import zlib

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import native
from tez_b200._lib import TezGpuError
from tez_b200.runtime_library import (BYTES_WRITABLE, INT_WRITABLE, TEXT, TEZ_BYTES_COMPARATOR, InputContext, LocalOutput,
                                      OrderedGroupedKVInput)
import codec_model as CM
import codec_table as CT
import combine_model as CBM
import lz4_model as L4
import snappy_model as SN
import zstd_model as ZS
from plugin_runs import consume, read_index, run_output

pytestmark = pytest.mark.gpu
ALL = list(CT.CODECS)
RUN_TABLE = ["default", "lz4", "zstd"]          # fixed-width run-table mode and reopen; fetch-verified
LARGE = ["lz4", "zstd", "snappy"]               # one segment of hundreds of blocks or frames
PLUGIN = [n for n, c in CT.CODECS.items() if c.plugin is not None]


def _codec(name):
    return CT.CODECS[name]


# ------------------------------------------------------------------------------------------------ sorter
@pytest.mark.parametrize("cmp_kind", [O.CMP_TEXT, O.CMP_BYTES, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG])
@pytest.mark.parametrize("P", [1, 64])
@pytest.mark.parametrize("codec", ALL)
def test_sorter_collect_batch_every_comparator(codec, P, cmp_kind):
    _, _, st = CT.sort_case(_codec(codec), CT.records(cmp_kind, 30000, seed=cmp_kind * 7 + P), P, cmp_kind)
    assert st["output_bytes_physical"] < st["output_bytes_with_overhead"]


@pytest.mark.parametrize("rle", [T.RLE_AUTO, T.RLE_OFF, T.RLE_ON])
@pytest.mark.parametrize("send_empty", [True, False])
@pytest.mark.parametrize("codec", ALL)
def test_sorter_rle_and_empty_partitions(codec, send_empty, rle):
    recs = CT.records(O.CMP_TEXT, 20000, seed=rle + 5)
    part = [zlib.crc32(k) % 5 * 3 for k, _ in recs]      # partitions 0, 3, 6, 9, 12 of 16: the others are empty
    CT.sort_case(_codec(codec), recs, 16, O.CMP_TEXT, rle=rle, send_empty=send_empty, partition=part)


@pytest.mark.parametrize("codec", ALL)
def test_sorter_no_records(codec):
    CT.sort_case(_codec(codec), [], 8, O.CMP_TEXT, send_empty=False)
    CT.sort_case(_codec(codec), [], 8, O.CMP_TEXT, send_empty=True)


@pytest.mark.parametrize("codec", ALL)
def test_sorter_unordered_handle(codec):
    CT.sort_case(_codec(codec), CT.records(O.CMP_TEXT, 20000, seed=9), 32, O.CMP_TEXT, unordered=True)


@pytest.mark.parametrize("combiner", [T.COMBINE_SUM_INT, T.COMBINE_SUM_LONG])
@pytest.mark.parametrize("codec", ALL)
def test_sorter_with_combiner(codec, combiner):
    rng = random.Random(combiner)
    w = 4 if combiner == T.COMBINE_SUM_INT else 8
    recs = [(k, rng.getrandbits(8 * w).to_bytes(w, "big")) for k, _ in CT.records(O.CMP_TEXT, 30000, seed=combiner)]
    _, _, st = CT.sort_case(_codec(codec), recs, 16, O.CMP_TEXT, combiner=combiner)
    assert st["spilled_records"] < 30000


@pytest.mark.parametrize("path,kind,n", [("collect_fixed", "c2", 100000), ("collect_fixed", "longs", 300000),
                                         ("device", "c2", 10 ** 7), ("device", "longs", 10 ** 6)])
@pytest.mark.parametrize("codec", ALL)
def test_sorter_fixed_width(codec, path, kind, n):
    c = _codec(codec)
    kl, vl = (16, 64) if kind == "c2" else (8, 8)
    P = 64
    kv = CT.fixed_kv(kind, n, seed=n)
    exp = O.pipelined_sort_fixed(O.sorter_conf(P, cmp_kind=O.CMP_BYTES if kind == "c2" else O.CMP_LONG), kv, kl, vl)
    with T.GpuSorter(P, comparator=T.CMP_BYTES if kind == "c2" else T.CMP_LONG, fixed=(kl, vl), codec=c.id) as s:
        if path == "collect_fixed":
            s.collect_fixed(kv)
            out, _, index, st = s.flush_to_memory()
            out = bytes(out)
        else:
            d_kv = torch.from_numpy(kv).cuda()
            cap = c.zcap(n * (kl + vl + 2) + 10 * P + 64, P)
            assert s.output_bound() <= cap
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            ln, index, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
            out = d_out[:ln].cpu().numpy().tobytes()
    CT.check_file(c, out, index, exp["file_out"], exp["index"])
    ratio = len(out) / len(exp["file_out"])
    assert ratio < c.ratio[0] if kind == "c2" else ratio < c.ratio[1]


@pytest.mark.parametrize("codec", ALL)
def test_set_codec_errors(codec):
    with T.GpuSorter(4) as s:
        with pytest.raises(TezGpuError, match="codec 7") as e:
            s.set_codec(7)
        assert e.value.code == T.E_UNSUPPORTED
        s.collect(b"\x01a\x00\x00\x00\x01", [0], [2], [4])
        with pytest.raises(TezGpuError) as e:
            s.set_codec(_codec(codec).id)
        assert e.value.code == T.E_STATE


@pytest.mark.parametrize("codec", ALL)
def test_codec_survives_reset(codec):
    c = _codec(codec)
    recs = CT.records(O.CMP_TEXT, 5000, seed=3)
    kv, ko, kl, vl, vo = CBM.pack(recs)
    exp = O.pipelined_sort(O.sorter_conf(4, cmp_kind=O.CMP_TEXT), kv, ko, kl, vl)
    with T.GpuSorter(4, comparator=T.CMP_TEXT, codec=c.id) as s:
        for _ in range(2):
            s.collect(kv, ko.astype(np.uint32), vo, vl)
            out, _, index, _ = s.flush_to_memory()
            CT.check_file(c, out, index, exp["file_out"], exp["index"])
            s.reset()


# ------------------------------------------------------------------------------------------------ merger
def _foreign(codec, mode, i, body):
    """(segment, rawLength) of the i-th compressed input of test_merger_inputs_mixed_with_plain"""
    c = _codec(codec)
    if codec == "default":
        level, strategy = mode
        return CM.compressed_segment(body, level, strategy, members=1 + (i % 2))
    if mode in ("java_fast", "java_hc"):
        z = L4.java_stream(L4.ifile_writes(body), compress=lambda d: L4.java_chunk(d, hc=mode == "java_hc"))
    elif mode == "java":
        z = SN.java_stream(SN.ifile_writes(body), compress=SN.java_chunk)
    else:                       # "device", and zstd's "hadoop", whose Hadoop-written segments come from the fixture
        z = c.emulate(body)
    return c.segment(z), len(body) + 4


def _merged(flat):
    """the same merge without the codec: its IFile and record count"""
    with T.GpuMerger(flat, comparator=T.CMP_TEXT) as m:
        return m.write_ifile(rle=False)[0], m.counts()[0]


ZSTD_HADOOP = ("wordcount_level1", "wordcount_checksum", "wordcount_oneshot", "two_frames_skippable")
MIXED = ([("default", (level, strategy), level * 10 + strategy)
          for level, strategy in [(0, 0), (1, 0), (6, 0), (9, 0), (6, zlib.Z_FIXED), (6, zlib.Z_HUFFMAN_ONLY), (6, zlib.Z_RLE),
                                  (6, zlib.Z_FILTERED)]]
         + [("lz4", m, len(m)) for m in ("device", "java_fast", "java_hc")] + [("zstd", m, len(m)) for m in ("device", "hadoop")]
         + [("snappy", m, len(m)) for m in ("device", "java")])


@pytest.mark.parametrize("codec,mode,seed", MIXED, ids=["%s-%s" % (c, "-".join(map(str, m)) if isinstance(m, tuple) else m)
                                                        for c, m, _ in MIXED])
def test_merger_inputs_mixed_with_plain(codec, mode, seed):
    """every third segment stays uncompressed; the others are written by a foreign writer or the device's own"""
    c = _codec(codec)
    plain = CT.c3(6, seed=seed)
    segs, raws, flat = [], [], list(plain)
    for i, s in enumerate(plain):
        if i % 3 == 2:
            segs.append(s)
            raws.append(0)
        else:
            z, raw = _foreign(codec, mode, i, CM.body_of(s))
            segs.append(z)
            raws.append(raw)
    if mode == "hadoop":
        for name, s, r in ZS.fixture():
            if name in ZSTD_HADOOP:
                segs.append(s)
                raws.append(r)
                flat.append(CT.plain(c.emulated_read(s[4:-4], r - 4)))
    exp, n = _merged(flat)
    if mode != "hadoop":      # the oracle's merge of the Hadoop-written fixture segments is not the device's length
        oracle = O.merge(flat, O.CMP_TEXT)
        assert exp == oracle["ifile"] and n == len(oracle["records"])
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=c.id, raw_lens=raws) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
        assert m.counts()[0] == n
    CT.check_merged(c, seg, raw, part, exp)
    with T.GpuMerger(segs[:2], comparator=T.CMP_TEXT, codec=c.id, raw_lens=raws[:2]) as m:
        m.reopen(segs[2:], raw_lens=raws[2:])
        seg, raw, part, _ = m.write_ifile(rle=False)
    exp, _ = _merged(flat[2:])
    if mode != "hadoop":
        assert exp == O.merge(flat[2:], O.CMP_TEXT)["ifile"]
    CT.check_merged(c, seg, raw, part, exp)


@pytest.mark.parametrize("codec", RUN_TABLE)
def test_merger_fixed_width_run_table_mode_and_reopen(codec):
    c = _codec(codec)
    plain = [O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 20000, seed=s), 16, 64)["file_out"] for s in (1, 2, 3)]
    exp = O.merge(plain, O.CMP_BYTES)
    zs = [CT.input_segment(c, CM.body_of(s), level=1) for s in plain]
    with T.GpuMerger([z for z, _ in zs], fixed=(16, 64), codec=c.id, raw_lens=[r for _, r in zs]) as m:
        assert m.parse_info()[0] == 0
        seg, raw, part, _ = m.write_ifile(rle=False)
        CT.check_merged(c, seg, raw, part, exp["ifile"])
        m.reopen([z for z, _ in zs[:2]], raw_lens=[r for _, r in zs[:2]])
        seg, raw, part, _ = m.write_ifile(rle=False)
        CT.check_merged(c, seg, raw, part, O.merge(plain[:2], O.CMP_BYTES)["ifile"])


@pytest.mark.parametrize("codec", ALL)
def test_merger_write_partitions_device_and_combiner(codec):
    c = _codec(codec)
    P = 4
    outs = []
    for seed in (11, 12):
        recs = CT.records(O.CMP_TEXT, 8000, seed=seed, vocab=500)
        kv, ko, kl, vl, vo = CBM.pack(recs)
        r = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT, rle_policy=0), kv, ko, kl, vl)
        outs.append((r["file_out"], r["index"]))
    segs, parts, raws, flat = [], [], [], []
    for fo, idx in outs:
        for p in range(P):
            s0, raw, part = (int(x) for x in idx[p])
            if part == 0:
                continue
            seg = fo[s0:s0 + part]
            z, r = CT.input_segment(c, CM.body_of(seg))
            segs.append(z); parts.append(p); raws.append(r); flat.append(seg)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P, codec=c.id, raw_lens=raws) as m:
        cap = m.output_bound()
        d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        ln, index, st = m.write_partitions_device(d_out.data_ptr(), cap)
        out = d_out[:ln].cpu().numpy().tobytes()
    assert st["file_out_bytes"] == ln
    # the same merge over the uncompressed segments, without the codec
    with T.GpuMerger(flat, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P) as m:
        cap = m.output_bound()
        d_ref = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        rln, rindex, _ = m.write_partitions_device(d_ref.data_ptr(), cap)
        ref = d_ref[:rln].cpu().numpy().tobytes()
    CT.check_file(c, out, index, ref, rindex)
    with T.GpuMerger(segs[:2], comparator=T.CMP_TEXT, codec=c.id, raw_lens=raws[:2], combiner=T.COMBINE_SUM_INT) as m:
        seg, raw, part, _ = m.write_ifile()
    with T.GpuMerger(flat[:2], comparator=T.CMP_TEXT, combiner=T.COMBINE_SUM_INT) as m:
        eseg = m.write_ifile()[0]
    CT.check_merged(c, seg, raw, part, eseg)


@pytest.mark.parametrize("codec", LARGE)
def test_merger_one_segment_of_hundreds_of_blocks(codec):
    """>= 64 MiB in one segment: about 1,000 blocks or frames decoded by as many warps, then merged with a small
    segment"""
    c = _codec(codec)
    big = O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 850000, seed=41), 16, 64)["file_out"]
    small = O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 1000, seed=42), 16, 64)["file_out"]
    assert len(big) >= 64 << 20
    zb = c.emulate(CM.body_of(big))
    assert c.units(zb) >= 1000
    segs = [c.segment(zb), c.segment(c.emulate(CM.body_of(small)))]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=c.id, raw_lens=[len(big) - 4, len(small) - 4]) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
    with T.GpuMerger([big, small], comparator=T.CMP_BYTES) as m:
        CT.check_merged(c, seg, raw, part, m.write_ifile(rle=False)[0])


@pytest.mark.parametrize("codec", ALL)
def test_merger_rejects_malformed_segments(codec):
    """wrong rawLength, a flipped checksum byte, no raw lengths, no codec, and every other codec's stream (the
    stream-level cases are in the codec's own suite)"""
    c = _codec(codec)
    bodies, segs, raws = CT.malformed_inputs(c)
    with pytest.raises(IOError, match="compressed segment 2"):
        CT.opened(c.id, segs, raws[:2] + [raws[2] + 1])
    with pytest.raises(IOError, match="checksum mismatch in segment 1"):
        CT.opened(c.id, [segs[0], segs[1][:-1] + bytes([segs[1][-1] ^ 1]), segs[2]], raws)
    with pytest.raises(TezGpuError) as e:
        CT.opened(c.id, segs, None)
    assert e.value.code == T.E_INVALID
    # without a codec the compressed flag is still refused
    with pytest.raises(IOError, match="compressed"):
        T.GpuMerger(segs, comparator=T.CMP_TEXT)
    # each other codec's stream given to this codec's merger, and this codec's streams given to each other codec's
    for other in CT.CODECS.values():
        if other is c:
            continue
        with pytest.raises(IOError, match="compressed segment 0"):
            CT.opened(c.id, [CT.input_segment(other, bodies[0])[0]] + segs[1:], raws)
        with pytest.raises(IOError, match="compressed segment 0"):
            CT.opened(other.id, segs, raws)


# ------------------------------------------------------------------------------------------------ transport
@pytest.mark.parametrize("codec", RUN_TABLE)
def test_fetch_verified_then_open_codec_and_wire_round_trip(codec):
    c = _codec(codec)
    P, n = 8, 200000
    kv = CT.fixed_kv("longs", n, seed=4)
    with T.GpuSorter(P, comparator=T.CMP_LONG, fixed=(8, 8), codec=c.id) as s:
        d_kv = torch.from_numpy(kv).cuda()
        cap = c.zcap(n * 18 + 10 * P + 64, P)
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ln, index, _ = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
        exp = O.pipelined_sort_fixed(O.sorter_conf(P, cmp_kind=O.CMP_LONG), kv, 8, 8)
        host = d_out[:ln].cpu().numpy().tobytes()
        CT.check_file(c, host, index, exp["file_out"], exp["index"])
        live = [p for p in range(P) if index[p][2] > 0]
        dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        table = [(d_out.data_ptr() + int(index[p][0]), dst.data_ptr() + int(index[p][0]), int(index[p][2])) for p in live]
        T.fetch_segments_verified(table)
        dsegs = [(dst.data_ptr() + int(index[p][0]), int(index[p][2])) for p in live]
        with T.GpuMerger(dsegs, comparator=T.CMP_LONG, device_ptrs=True, verified=[True] * len(live), codec=c.id,
                         raw_lens=[int(index[p][1]) for p in live]) as m:
            seg, raw, part, _ = m.write_ifile()
        plain = [exp["file_out"][int(exp["index"][p][0]):int(exp["index"][p][0] + exp["index"][p][2])] for p in live]
        with T.GpuMerger(plain, comparator=T.CMP_LONG) as m:   # the same merge without the codec
            CT.check_merged(c, seg, raw, part, m.write_ifile()[0])
        got = native.shuffle_receive(native.shuffle_serve(d_out.data_ptr(), index, "attempt_1", 0, P))
        wsegs = [g[3] for g in got if len(g[3])]
        wraws = [g[2] for g in got if len(g[3])]
        assert len(wsegs) == len(live)
        with T.GpuMerger(wsegs, comparator=T.CMP_LONG, codec=c.id, raw_lens=wraws) as m:
            seg2, raw2, part2, _ = m.write_ifile()
        assert seg2 == seg and raw2 == raw


# ------------------------------------------------------------------------------------------------ plugin classes
@pytest.mark.parametrize("n,spills", [(5000, 1), (20000, 2), (60000, 4)])
@pytest.mark.parametrize("codec", PLUGIN)
def test_output_spills_and_final_merge_compressed(tmp_path, codec, n, spills):
    """Unique keys: the final file.out is the single sort's, every segment compressed.  Spills follow the raw bytes
    against tez.runtime.io.sort.mb, whatever the codec."""
    c = _codec(codec)
    P = 8
    kv = O.gen_c2(0, n, seed=n)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = dict(c.plugin, **{"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
                             "tez.runtime.io.sort.mb": 1})
    out, events = run_output(tmp_path, conf, recs, P)
    assert out.num_spills >= spills if spills == 4 else out.num_spills == spills
    exp = O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, 64)
    got = open(out.final_output_file, "rb").read()
    CT.check_file(c, got, read_index(out.final_index_file, P), exp["file_out"], exp["index"])
    assert out.counter("OUTPUT_BYTES_PHYSICAL") == len(got)
    assert out.counter("OUTPUT_BYTES_WITH_OVERHEAD") == int(exp["index"][:, 1].sum())
    assert out.counter("OUTPUT_RECORDS") == n
    assert out.counter("SPILLED_RECORDS") == (n if out.num_spills == 1 else 2 * n)


@pytest.mark.parametrize("codec", PLUGIN)
def test_pipelined_shuffle_compressed_spills_reach_the_input(tmp_path, codec):
    c = _codec(codec)
    n, P = 40000, 4
    kv = O.gen_c2(0, n, seed=23)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = dict(c.plugin, **{"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
                             "tez.runtime.io.sort.mb": 1, "tez.runtime.enable.final-merge.in.output": False})
    out, events = run_output(tmp_path, conf, recs, P)
    S = out.num_spills
    assert S >= 3
    uid = out.context.unique_identifier
    files = [str(tmp_path / "output" / ("%s_%d" % (uid, s)) / "file.out") for s in range(S)]
    for f in files:
        data, idx = open(f, "rb").read(), read_index(f + ".index", P)
        for s0, raw, part in idx:
            if part:
                seg = data[s0:s0 + part]
                assert seg[:4] == b"TIF\x01" and len(c.decode(seg[4:-4], raw - 4)) == raw - 4
    p = 2
    inp = OrderedGroupedKVInput(InputContext(conf, str(tmp_path / "r")), 1)
    inp.initialize()
    inp.start()
    inp.handleEvents([LocalOutput(0, files[s], files[s] + ".index", p, spill_id=s, last_event=(s == S - 1)) for s in range(S)])
    r = inp.getReader()
    got = []
    while r.next():
        got.append((r.getCurrentKey(), list(r.getCurrentValues())))
    mine = sorted((k, v) for k, v in recs if O.partition_of(O.CMP_BYTES, k, P) == p)
    assert [(k, vs[0]) for k, vs in got] == mine
    # random records: stored chunks or raw blocks, a few bytes of framing per chunk over the raw length.  LZ4 is not
    # held to it: a block of random bytes is all literals, one length byte per 255 bytes over the raw length.
    if codec != "lz4":
        assert 0 < inp.counter("SHUFFLE_BYTES") <= 1.001 * inp.counter("SHUFFLE_BYTES_DECOMPRESSED") + 32 * S


@pytest.mark.parametrize("codec", PLUGIN)
def test_ordered_word_count_known_answer_compressed(tmp_path, codec):
    """TestTezJobs.testOrderedWordCount's answer with both edges compressed; the compressible word stream shuffles
    fewer bytes than it decompresses to."""
    plugin = _codec(codec).plugin
    words = []
    for i in range(1, 11):
        words += ["a_%d" % i] * (22 - 2 * i) * 50
    random.Random(3).shuffle(words)
    P = 4
    conf1 = dict(plugin, **{"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE})
    producers = [run_output(tmp_path / ("t%d" % t), conf1, [(O.text(w), O.int_writable(1)) for w in words[t::3]], P,
                            uid="attempt_1_0001_1_00_%06d_0_10001" % t) for t in range(3)]
    for prod, _ in producers:
        assert open(prod.final_output_file, "rb").read(4) in (b"TIF\x01", b"")
    counts = {}
    shuffled = decompressed = 0
    for p in range(P):
        inp, groups = consume(tmp_path / ("s%d" % p), conf1, producers, p, P)
        for k, vals in groups:
            counts[k[1:].decode()] = sum(int.from_bytes(v, "big") for v in vals)
        shuffled += inp.counter("SHUFFLE_BYTES")
        decompressed += inp.counter("SHUFFLE_BYTES_DECOMPRESSED")
    assert counts == {"a_%d" % i: (22 - 2 * i) * 50 for i in range(1, 11)}
    assert 0 < shuffled < decompressed
    conf2 = dict(plugin, **{"tez.runtime.key.class": INT_WRITABLE, "tez.runtime.value.class": TEXT})
    prod2 = [run_output(tmp_path / "sum", conf2, [(O.int_writable(c), O.text(w)) for w, c in counts.items()], 1,
                        uid="attempt_1_0001_1_01_000000_0_10001")]
    _, groups = consume(tmp_path / "sorter", conf2, prod2, 0, 1)
    final = [(int.from_bytes(k, "big", signed=True), v[0][1:].decode()) for k, v in groups]
    assert final == [((22 - 2 * i) * 50, "a_%d" % i) for i in range(10, 0, -1)]

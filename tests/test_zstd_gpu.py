"""GPU: ZStandardCodec on the device.  Every compressed segment the device writes is checked against the uncompressed
output of the oracle (or of the same merge without the codec): header, CRC of the stream, its decode (libzstd where it
can be loaded, else the emulated reader), index triple, and byte for byte against the host emulation of the writer.
The reader is fed the Hadoop-written fixture, device-written streams, mixes of compressed and plain segments, one
segment of about 1,000 frames (one warp per frame), a one-frame segment of several MB (one warp per segment), malformed
and wrong-codec streams; the plugin classes run spills, the pipelined shuffle and OrderedWordCount through
ZStandardCodec."""
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
import combine_model as CBM
import lz4_model as L4
import zstd_model as M
from test_codec_gpu import _c3, _fixed_kv, _plain, _records
from test_runtime_library_gpu import _consume, _run_output

pytestmark = pytest.mark.gpu
Z = T.CODEC_ZSTD
LCONF = {"tez.runtime.compress": True, "tez.runtime.compress.codec": "org.apache.hadoop.io.compress.ZStandardCodec",
         "io.compression.codec.zstd.level": 9}


def check_segment(seg, body, model=None):
    """one device-written zstd segment against its uncompressed body, decoded by libzstd where it can be loaded, else by
    the emulated reader (checked against libzstd on the CPU)"""
    if model is None:
        model = M.libzstd() is not None
    assert seg[:4] == b"TIF\x01"
    assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])
    assert (M.hadoop_read if model else M.decompress_emulate)(seg[4:-4], len(body)) == body
    assert seg[4:-4] == M.compress_emulate(body), "device bytes differ from the host emulation"


def check_file(out, index, exp_file, exp_index):
    """Device file.out / index with the codec against the oracle's uncompressed file.out / index."""
    out = bytes(out)
    pos = 0
    for p in range(len(exp_index)):
        s, raw, part = (int(x) for x in index[p])
        es, eraw, epart = (int(x) for x in exp_index[p])
        assert raw == eraw, p
        if epart == 0:
            assert part == 0 and s in (0, pos), p
            continue
        assert s == pos, p
        seg = out[s:s + part]
        assert len(seg) == part
        check_segment(seg, exp_file[es + 4:es + epart - 4])
        pos += part
    assert pos == len(out)


def _check_merged(seg, raw, part, exp_ifile, model=None):
    assert part == len(seg) and raw == len(exp_ifile) - 4
    check_segment(seg, exp_ifile[4:-4], model)


def _zcap(raw, P):
    return raw + 10 * (raw // M.ZSTD_BLOCK_BYTES + P + 1) + 64


def _sort_case(recs, P, cmp_kind, rle=-1, send_empty=True, partition=None, combiner=0, unordered=False):
    kv, ko, kl, vl, vo = CBM.pack(recs)
    part_mode = T.PART_GIVEN if partition is not None else T.PART_HASH
    if combiner:
        exp = CBM.sort_combine(P, cmp_kind, combiner, kv, ko, kl, vl, partition, send_empty=send_empty)
    else:
        conf = O.sorter_conf(P, cmp_kind=cmp_kind, partitioner=part_mode, send_empty=send_empty, rle_policy=rle)
        exp = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl, partition)
    with T.GpuSorter(P, comparator=cmp_kind, partitioner=part_mode, rle_policy=rle, send_empty=send_empty,
                     combiner=combiner, codec=Z, unordered=unordered) as s:
        if len(recs):
            s.collect(kv, ko.astype(np.uint32), vo, vl, None if partition is None else np.asarray(partition, np.int32))
        out, index_bytes, index, st = s.flush_to_memory()
    check_file(out, index, exp["file_out"], exp["index"])
    assert st["output_bytes_physical"] == st["file_out_bytes"] == len(out)
    assert st["output_bytes_with_overhead"] == int(exp["index"][:, 1].sum())
    return out, index, st


# ------------------------------------------------------------------------------------------------ sorter
@pytest.mark.parametrize("cmp_kind", [O.CMP_TEXT, O.CMP_BYTES, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG])
@pytest.mark.parametrize("P", [1, 64])
def test_sorter_collect_batch_every_comparator(cmp_kind, P):
    _, _, st = _sort_case(_records(cmp_kind, 30000, seed=cmp_kind * 7 + P), P, cmp_kind)
    assert st["output_bytes_physical"] < st["output_bytes_with_overhead"]


@pytest.mark.parametrize("rle", [T.RLE_AUTO, T.RLE_OFF, T.RLE_ON])
@pytest.mark.parametrize("send_empty", [True, False])
def test_sorter_rle_and_empty_partitions(rle, send_empty):
    recs = _records(O.CMP_TEXT, 20000, seed=rle + 5)
    part = [zlib.crc32(k) % 5 * 3 for k, _ in recs]
    _sort_case(recs, 16, O.CMP_TEXT, rle=rle, send_empty=send_empty, partition=part)


def test_sorter_no_records_and_unordered():
    _sort_case([], 8, O.CMP_TEXT, send_empty=False)
    _sort_case([], 8, O.CMP_TEXT, send_empty=True)
    _sort_case(_records(O.CMP_TEXT, 20000, seed=9), 32, O.CMP_TEXT, unordered=True)


@pytest.mark.parametrize("combiner", [T.COMBINE_SUM_INT, T.COMBINE_SUM_LONG])
def test_sorter_with_combiner(combiner):
    rng = random.Random(combiner)
    w = 4 if combiner == T.COMBINE_SUM_INT else 8
    recs = [(k, rng.getrandbits(8 * w).to_bytes(w, "big")) for k, _ in _records(O.CMP_TEXT, 30000, seed=combiner)]
    _, _, st = _sort_case(recs, 16, O.CMP_TEXT, combiner=combiner)
    assert st["spilled_records"] < 30000


@pytest.mark.parametrize("path,kind,n", [("collect_fixed", "c2", 100000), ("collect_fixed", "longs", 300000),
                                         ("device", "c2", 10 ** 7), ("device", "longs", 10 ** 6)])
def test_sorter_fixed_width(path, kind, n):
    kl, vl = (16, 64) if kind == "c2" else (8, 8)
    P = 64
    kv = _fixed_kv(kind, n, seed=n)
    exp = O.pipelined_sort_fixed(O.sorter_conf(P, cmp_kind=O.CMP_BYTES if kind == "c2" else O.CMP_LONG), kv, kl, vl)
    with T.GpuSorter(P, comparator=T.CMP_BYTES if kind == "c2" else T.CMP_LONG, fixed=(kl, vl), codec=Z) as s:
        if path == "collect_fixed":
            s.collect_fixed(kv)
            out, _, index, st = s.flush_to_memory()
            out = bytes(out)
        else:
            d_kv = torch.from_numpy(kv).cuda()
            cap = _zcap(n * (kl + vl + 2) + 10 * P + 64, P)
            assert s.output_bound() <= cap
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            ln, index, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
            out = d_out[:ln].cpu().numpy().tobytes()
    check_file(out, index, exp["file_out"], exp["index"])
    ratio = len(out) / len(exp["file_out"])
    assert ratio < 1.01 if kind == "c2" else ratio < 0.75


def test_set_codec_errors_and_reset():
    with T.GpuSorter(4) as s:
        with pytest.raises(TezGpuError) as e:
            s.set_codec(7)
        assert e.value.code == T.E_UNSUPPORTED
        s.collect(b"\x01a\x00\x00\x00\x01", [0], [2], [4])
        with pytest.raises(TezGpuError) as e:
            s.set_codec(Z)
        assert e.value.code == T.E_STATE
    recs = _records(O.CMP_TEXT, 5000, seed=3)
    kv, ko, kl, vl, vo = CBM.pack(recs)
    exp = O.pipelined_sort(O.sorter_conf(4, cmp_kind=O.CMP_TEXT), kv, ko, kl, vl)
    with T.GpuSorter(4, comparator=T.CMP_TEXT, codec=Z) as s:
        for _ in range(2):
            s.collect(kv, ko.astype(np.uint32), vo, vl)
            out, _, index, _ = s.flush_to_memory()
            check_file(out, index, exp["file_out"], exp["index"])
            s.reset()


# ------------------------------------------------------------------------------------------------ merger
def test_merger_hadoop_written_fixture():
    """The fixture's segments (libzstd streams at levels 1, 3 and 19, a checksum, a one-shot frame, a 2^27 window with
    long-distance matching, a 700,000-byte value, a skippable frame between two frames): the same records and output
    as the merge over the emulator-decoded segments (compared with libzstd on the CPU)."""
    fx = M.fixture()
    segs, raws = [s for _, s, _ in fx], [r for _, _, r in fx]
    plain = [_plain(M.decompress_emulate(s[4:-4], r - 4)) for s, r in zip(segs, raws)]
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        exp_recs = list(m.records())
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        exp_ifile = m.write_ifile(rle=False)[0]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=raws) as m:
        assert list(m.records()) == exp_recs
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=raws) as m:
        seg, raw, part, st = m.write_ifile(rle=False)
    _check_merged(seg, raw, part, exp_ifile)
    assert st["file_out_bytes"] == part


@pytest.mark.parametrize("mode", ["device", "hadoop"])
def test_merger_zstd_inputs_mixed_with_plain(mode):
    """device-written segments, or the fixture's Hadoop-written segments with Text keys, mixed with plain ones"""
    plain = _c3(6, seed=len(mode))
    segs, raws, flat = [], [], []
    for i, s in enumerate(plain):
        if i % 3 == 2:
            segs.append(s)
            raws.append(0)
            flat.append(s)
            continue
        body = CM.body_of(s)
        segs.append(M.segment(M.compress_emulate(body)))
        raws.append(len(body) + 4)
        flat.append(s)
    if mode == "hadoop":
        for name, s, r in M.fixture():
            if name in ("wordcount_level1", "wordcount_checksum", "wordcount_oneshot", "two_frames_skippable"):
                segs.append(s)
                raws.append(r)
                flat.append(_plain(M.decompress_emulate(s[4:-4], r - 4)))
    with T.GpuMerger(flat, comparator=T.CMP_TEXT) as m:
        exp_ifile = m.write_ifile(rle=False)[0]
        n = m.counts()[0]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=Z, raw_lens=raws) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
        assert m.counts()[0] == n
    _check_merged(seg, raw, part, exp_ifile)


def test_merger_fixed_width_run_table_mode_and_reopen():
    plain = [O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 20000, seed=s), 16, 64)["file_out"] for s in (1, 2, 3)]
    exp = O.merge(plain, O.CMP_BYTES)
    zs = [(M.segment(M.compress_emulate(CM.body_of(s))), len(s) - 4) for s in plain]
    with T.GpuMerger([z for z, _ in zs], fixed=(16, 64), codec=Z, raw_lens=[r for _, r in zs]) as m:
        assert m.parse_info()[0] == 0
        seg, raw, part, _ = m.write_ifile(rle=False)
        _check_merged(seg, raw, part, exp["ifile"])
        m.reopen([z for z, _ in zs[:2]], raw_lens=[r for _, r in zs[:2]])
        seg, raw, part, _ = m.write_ifile(rle=False)
        _check_merged(seg, raw, part, O.merge(plain[:2], O.CMP_BYTES)["ifile"])


def test_merger_write_partitions_device_and_combiner():
    P = 4
    outs = []
    for seed in (11, 12):
        recs = _records(O.CMP_TEXT, 8000, seed=seed, vocab=500)
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
            segs.append(M.segment(M.compress_emulate(CM.body_of(seg)))); parts.append(p); raws.append(raw); flat.append(seg)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P, codec=Z, raw_lens=raws) as m:
        cap = m.output_bound()
        d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        ln, index, st = m.write_partitions_device(d_out.data_ptr(), cap)
        out = d_out[:ln].cpu().numpy().tobytes()
    assert st["file_out_bytes"] == ln
    with T.GpuMerger(flat, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P) as m:
        cap = m.output_bound()
        d_ref = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        rln, rindex, _ = m.write_partitions_device(d_ref.data_ptr(), cap)
        ref = d_ref[:rln].cpu().numpy().tobytes()
    check_file(out, index, ref, rindex)
    with T.GpuMerger(segs[:2], comparator=T.CMP_TEXT, codec=Z, raw_lens=raws[:2], combiner=T.COMBINE_SUM_INT) as m:
        seg, raw, part, _ = m.write_ifile()
    with T.GpuMerger(flat[:2], comparator=T.CMP_TEXT, combiner=T.COMBINE_SUM_INT) as m:
        eseg = m.write_ifile()[0]
    _check_merged(seg, raw, part, eseg)


def test_merger_one_segment_of_hundreds_of_frames():
    """>= 64 MiB in one segment: about 1,000 frames decoded by as many warps, then merged with a small segment."""
    big = O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 850000, seed=41), 16, 64)["file_out"]
    small = O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 1000, seed=42), 16, 64)["file_out"]
    assert len(big) >= 64 << 20
    zb = M.compress_emulate(CM.body_of(big))
    assert len(M.frames(zb)) >= 1000
    segs = [M.segment(zb), M.segment(M.compress_emulate(CM.body_of(small)))]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=[len(big) - 4, len(small) - 4]) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
    with T.GpuMerger([big, small], comparator=T.CMP_BYTES) as m:
        _check_merged(seg, raw, part, m.write_ifile(rle=False)[0])


def test_merger_one_frame_segment_of_several_mb():
    """The Java shape: one frame of many blocks without Frame_Content_Size, decoded by one warp walking it; merged with
    device-written segments."""
    plain = [O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, n, seed=s), 16, 64)["file_out"] for n, s in ((60000, 51), (3000, 52))]
    big = CM.body_of(plain[0])
    z = M.one_frame(M.compress_emulate(big))
    assert len(big) >= 4 << 20 and len(M.frames(z)) == 1 and M.frames(z)[0][2] is None and len(M.frames(z)[0][3]) >= 70
    segs = [M.segment(z), M.segment(M.compress_emulate(CM.body_of(plain[1])))]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=[len(p) - 4 for p in plain]) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        _check_merged(seg, raw, part, m.write_ifile(rle=False)[0])


def test_merger_rejects_malformed_and_wrong_codec_segments():
    plain = _c3(3, seed=5)
    bodies = [CM.body_of(s) for s in plain]
    segs = [M.segment(M.compress_emulate(b)) for b in bodies]
    raws = [len(b) + 4 for b in bodies]

    def opened(segs_, raws_, codec=Z):
        with T.GpuMerger(segs_, comparator=T.CMP_TEXT, codec=codec, raw_lens=raws_) as m:
            return m.counts()

    # the first frame's reserved bit (the frame walk sends the segment to the serial path), checksum recomputed
    z = bytearray(segs[1][4:-4])
    z[4] |= 0x08
    with pytest.raises(IOError, match="compressed segment 1: reserved bit set"):
        opened([segs[0], M.segment(bytes(z)), segs[2]], raws)
    # a compressed block's literals section made treeless with no table: the frame walk passes, the frame's warp fails
    # and the serial path names the error
    z = bytearray(segs[2][4:-4])
    ip = 0
    for f, fhd, fcs, blocks in M.frames(z):
        if blocks[0][0] == 2:
            q = ip + (7 if fcs >= 256 else 6) + 3
            z[q] |= 3
            break
        ip += len(f)
    else:
        pytest.fail("no compressed frame")
    with pytest.raises(IOError, match="compressed segment 2: "):
        opened([segs[0], segs[1], M.segment(bytes(z))], raws)
    # wrong rawLength
    with pytest.raises(IOError, match="compressed segment 2"):
        opened(segs, raws[:2] + [raws[2] + 1])
    # bytes after the last frame
    with pytest.raises(IOError, match="compressed segment 0: bytes after the last frame"):
        opened([M.segment(segs[0][4:-4] + b"\0\0\0\0")] + segs[1:], raws)
    # checksum of the stream
    with pytest.raises(IOError, match="checksum mismatch in segment 1"):
        opened([segs[0], segs[1][:-1] + bytes([segs[1][-1] ^ 1]), segs[2]], raws)
    # no raw lengths for compressed segments
    with pytest.raises(TezGpuError) as e:
        opened(segs, None)
    assert e.value.code == T.E_INVALID
    # zlib and LZ4 streams given to a zstd merger, and a zstd stream given to DefaultCodec and Lz4Codec mergers
    zseg, zraw = CM.compressed_segment(bodies[0], 6)
    with pytest.raises(IOError, match="compressed segment 0: bad frame magic"):
        opened([zseg] + segs[1:], [zraw] + raws[1:])
    with pytest.raises(IOError, match="compressed segment 1: bad frame magic"):
        opened([segs[0], L4.segment(L4.compress_emulate(bodies[1])), segs[2]], raws)
    with pytest.raises(IOError, match="compressed segment 0"):
        opened(segs, raws, codec=T.CODEC_DEFAULT)
    with pytest.raises(IOError, match="compressed segment 0"):
        opened(segs, raws, codec=T.CODEC_LZ4)


# ------------------------------------------------------------------------------------------------ transport
def test_fetch_verified_then_open_codec_and_wire_round_trip():
    P, n = 8, 200000
    kv = _fixed_kv("longs", n, seed=4)
    with T.GpuSorter(P, comparator=T.CMP_LONG, fixed=(8, 8), codec=Z) as s:
        d_kv = torch.from_numpy(kv).cuda()
        cap = _zcap(n * 18 + 10 * P + 64, P)
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ln, index, _ = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
        exp = O.pipelined_sort_fixed(O.sorter_conf(P, cmp_kind=O.CMP_LONG), kv, 8, 8)
        host = d_out[:ln].cpu().numpy().tobytes()
        check_file(host, index, exp["file_out"], exp["index"])
        live = [p for p in range(P) if index[p][2] > 0]
        dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        table = [(d_out.data_ptr() + int(index[p][0]), dst.data_ptr() + int(index[p][0]), int(index[p][2])) for p in live]
        T.fetch_segments_verified(table)
        dsegs = [(dst.data_ptr() + int(index[p][0]), int(index[p][2])) for p in live]
        with T.GpuMerger(dsegs, comparator=T.CMP_LONG, device_ptrs=True, verified=[True] * len(live), codec=Z,
                         raw_lens=[int(index[p][1]) for p in live]) as m:
            seg, raw, part, _ = m.write_ifile()
        plain = [exp["file_out"][int(exp["index"][p][0]):int(exp["index"][p][0] + exp["index"][p][2])] for p in live]
        with T.GpuMerger(plain, comparator=T.CMP_LONG) as m:
            _check_merged(seg, raw, part, m.write_ifile()[0])
        got = native.shuffle_receive(native.shuffle_serve(d_out.data_ptr(), index, "attempt_1", 0, P))
        wsegs = [g[3] for g in got if len(g[3])]
        wraws = [g[2] for g in got if len(g[3])]
        assert len(wsegs) == len(live)
        with T.GpuMerger(wsegs, comparator=T.CMP_LONG, codec=Z, raw_lens=wraws) as m:
            seg2, raw2, part2, _ = m.write_ifile()
        assert seg2 == seg and raw2 == raw


# ------------------------------------------------------------------------------------------------ plugin classes
def _index(path, P):
    return np.frombuffer(open(path, "rb").read()[:-8], dtype=">i8").reshape(P, 3)


@pytest.mark.parametrize("n,spills", [(5000, 1), (20000, 2), (60000, 4)])
def test_output_spills_and_final_merge_compressed(tmp_path, n, spills):
    P = 8
    kv = O.gen_c2(0, n, seed=n)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = dict(LCONF, **{"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
                          "tez.runtime.io.sort.mb": 1})
    out, events = _run_output(tmp_path, conf, recs, P)
    assert out.num_spills >= spills if spills == 4 else out.num_spills == spills
    exp = O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, 64)
    got = open(out.final_output_file, "rb").read()
    check_file(got, _index(out.final_index_file, P), exp["file_out"], exp["index"])
    assert out.counter("OUTPUT_BYTES_PHYSICAL") == len(got)
    assert out.counter("OUTPUT_RECORDS") == n


def test_pipelined_shuffle_compressed_spills_reach_the_input(tmp_path):
    n, P = 40000, 4
    kv = O.gen_c2(0, n, seed=23)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = dict(LCONF, **{"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
                          "tez.runtime.io.sort.mb": 1, "tez.runtime.enable.final-merge.in.output": False})
    out, events = _run_output(tmp_path, conf, recs, P)
    S = out.num_spills
    assert S >= 3
    uid = out.context.unique_identifier
    files = [str(tmp_path / "output" / ("%s_%d" % (uid, s)) / "file.out") for s in range(S)]
    for f in files:
        data, idx = open(f, "rb").read(), _index(f + ".index", P)
        for s0, raw, part in idx:
            if part:
                seg = data[s0:s0 + part]
                assert seg[:4] == b"TIF\x01" and len(M.decompress_emulate(seg[4:-4], raw - 4)) == raw - 4
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


def test_ordered_word_count_known_answer_over_two_zstd_edges(tmp_path):
    words = []
    for i in range(1, 11):
        words += ["a_%d" % i] * (22 - 2 * i) * 50
    random.Random(3).shuffle(words)
    P = 4
    conf1 = dict(LCONF, **{"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE})
    producers = [_run_output(tmp_path / ("t%d" % t), conf1, [(O.text(w), O.int_writable(1)) for w in words[t::3]], P,
                             uid="attempt_1_0001_1_00_%06d_0_10001" % t) for t in range(3)]
    counts = {}
    shuffled = decompressed = 0
    for p in range(P):
        inp, groups = _consume(tmp_path / ("s%d" % p), conf1, producers, p, P)
        for k, vals in groups:
            counts[k[1:].decode()] = sum(int.from_bytes(v, "big") for v in vals)
        shuffled += inp.counter("SHUFFLE_BYTES")
        decompressed += inp.counter("SHUFFLE_BYTES_DECOMPRESSED")
    assert counts == {"a_%d" % i: (22 - 2 * i) * 50 for i in range(1, 11)}
    assert 0 < shuffled < decompressed
    conf2 = dict(LCONF, **{"tez.runtime.key.class": INT_WRITABLE, "tez.runtime.value.class": TEXT})
    prod2 = [_run_output(tmp_path / "sum", conf2, [(O.int_writable(c), O.text(w)) for w, c in counts.items()], 1,
                         uid="attempt_1_0001_1_01_000000_0_10001")]
    _, groups = _consume(tmp_path / "sorter", conf2, prod2, 0, 1)
    final = [(int.from_bytes(k, "big", signed=True), v[0][1:].decode()) for k, v in groups]
    assert final == [((22 - 2 * i) * 50, "a_%d" % i) for i in range(10, 0, -1)]

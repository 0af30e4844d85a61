"""GPU: merges under a device budget through the plugin classes (tez.runtime.gpu.merge.device.budget.mb), compressed
inputs included.  tezgpu_decode_segments turns compressed segments into the uncompressed segments an IFile.Writer
writes for the same records, in groups that fit the budget; the input decodes and then merges in key-range steps, the
output's final merge runs in steps, and both return exactly what they return without the key."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import _lib, native
from tez_b200._lib import TezGpuError
from tez_b200.runtime_library import (INT_WRITABLE, TEXT, InputContext, LocalOutput, OrderedGroupedKVInput, OutputContext,
                                      UnorderedKVInput, UnorderedPartitionedKVOutput)
import combine_model as CBM
import lz4_model as L4M
import zstd_model as ZSM
from plugin_runs import run_output

pytestmark = pytest.mark.gpu
KEY = "tez.runtime.gpu.merge.device.budget.mb"
FLOOR = 16 << 20
CODECS = {T.CODEC_DEFAULT: "org.apache.hadoop.io.compress.DefaultCodec",
          T.CODEC_LZ4: "org.apache.hadoop.io.compress.Lz4Codec",
          T.CODEC_ZSTD: "org.apache.hadoop.io.compress.ZStandardCodec"}
WC = {"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE}


def _codec_conf(codec):
    return {"tez.runtime.compress": True, "tez.runtime.compress.codec": CODECS[codec]} if codec else {}


def _words(n, seed, vocab=20000):
    rng = random.Random(seed)
    return [(O.text("w%07x" % rng.randrange(vocab)), O.int_writable(1)) for _ in range(n)]


def _device_segments(codec, recs, P):
    """file.out of the device sorter with `codec` and the oracle's uncompressed file.out for the same records: the
    compressed segments, their raw lengths and the expected uncompressed segments, one per non-empty partition."""
    kv, ko, kl, vl, vo = CBM.pack(recs)
    exp = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT), kv, ko, kl, vl, None)
    with T.GpuSorter(P, comparator=T.CMP_TEXT, codec=codec) as s:
        s.collect(kv, ko.astype(np.uint32), vo, vl)
        out, _, index, _ = s.flush_to_memory()
    out = bytes(out)
    segs, raws, plain = [], [], []
    for p in range(P):
        s0, raw, part = (int(x) for x in index[p])
        es, _, epart = (int(x) for x in exp["index"][p])
        if part:
            segs.append(out[s0:s0 + part])
            raws.append(raw)
            plain.append(exp["file_out"][es:es + epart])
    return segs, raws, plain


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_decode_device_written_segments(codec):
    """16 segments of ~1.2 MiB raw each (keys nearly unique: no run-length encoding): one group at 1 GiB, several at the
    16 MiB floor; every image is the oracle's uncompressed segment byte for byte."""
    segs, raws, plain = _device_segments(codec, _words(1300000, seed=codec, vocab=1 << 28), 16)
    assert len(segs) == 16 and all(s[:4] == b"TIF\x01" for s in segs) and sum(raws) > 18 << 20
    peaks = {}
    for budget in (1 << 30, FLOOR):
        imgs, peak = native.decode_segments(segs, raws, codec, budget)
        assert imgs == plain
        assert peak <= budget
        peaks[budget] = peak
    assert peaks[1 << 30] > FLOOR   # the whole set does not fit the floor: the floor took several groups


@pytest.mark.parametrize("codec,model", [(T.CODEC_LZ4, L4M), (T.CODEC_ZSTD, ZSM)])
def test_decode_java_framed_fixtures(codec, model):
    """The fixtures' segments (Java block / frame cutting), eight times over: the image's body is the model's decode, its
    trailer the CRC-32 of that body; at 1 GiB one group, at the floor several."""
    fx = model.fixture() * 8
    segs, raws = [s for _, s, _ in fx], [r for _, _, r in fx]
    decode = L4M.decode_stream if codec == T.CODEC_LZ4 else ZSM.hadoop_read
    bodies = [decode(s[4:-4], r - 4) for s, r in zip(segs, raws)]
    peaks = []
    for budget in (1 << 30, FLOOR):
        imgs, peak = native.decode_segments(segs, raws, codec, budget)
        for img, body, r in zip(imgs, bodies, raws):
            assert len(img) == r + 4 and img[:4] == b"TIF\x00" and img[4:-4] == body
            assert int.from_bytes(img[-4:], "big") == zlib.crc32(body)
        assert peak <= budget
        peaks.append(peak)
    assert peaks[0] > FLOOR


def _decode_raw(segs, raws, codec, budget, sentinel=0xA5):
    """tezgpu_decode_segments with an output buffer for every segment, filled with `sentinel`: (rc, message, outputs)"""
    L = _lib.load()
    keep = [np.frombuffer(bytes(s), dtype=np.uint8) for s in segs]
    arr = (_lib.Segment * len(keep))()
    bufs = [np.full(max(len(s), r + 4), sentinel, dtype=np.uint8) for s, r in zip(segs, raws)]
    out = (C.c_void_p * len(keep))()
    for i, a in enumerate(keep):
        arr[i].data, arr[i].len, arr[i].flags = a.ctypes.data, a.size, T.SEG_HAS_HEADER
        out[i] = bufs[i].ctypes.data
    rl = (C.c_int64 * len(raws))(*raws)
    cf = native.make_conf(1, partitioner=T.PART_GIVEN)
    peak = C.c_uint64()
    rc = L.tezgpu_decode_segments(C.byref(cf), arr, rl, len(keep), codec, budget, out, C.byref(peak))
    return rc, L.tezgpu_last_error().decode(), [b.tobytes() for b in bufs]


def test_decode_errors_name_the_callers_segment():
    codec = T.CODEC_LZ4
    segs, raws, plain = _device_segments(codec, _words(60000, seed=5), 3)
    # plain segments in the list are not written
    mixed, mraw = [plain[0]] + segs[1:], [len(plain[0]) - 4] + raws[1:]
    rc, _, outs = _decode_raw(mixed, mraw, codec, 1 << 30)
    assert rc == 0 and outs[0] == bytes([0xA5]) * len(outs[0])
    assert outs[1][:mraw[1] + 4] == plain[1] and outs[2][:mraw[2] + 4] == plain[2]
    # a flipped byte: the checksum of segment 2
    bad = bytearray(segs[2])
    bad[len(bad) // 2] ^= 0x40
    with pytest.raises(TezGpuError) as e:
        native.decode_segments(segs[:2] + [bytes(bad)], raws, codec, 1 << 30)
    assert e.value.code == T.E_FORMAT and "checksum mismatch in segment 2" in str(e.value)
    # the same byte with a checksum that matches: the stream of segment 1 is refused
    bad = bytearray(segs[1])
    bad[12] ^= 0xFF
    bad[-4:] = zlib.crc32(bytes(bad[4:-4])).to_bytes(4, "big")
    with pytest.raises(TezGpuError) as e:
        native.decode_segments([segs[0], bytes(bad), segs[2]], raws, codec, 1 << 30)
    assert e.value.code == T.E_FORMAT and "compressed segment 1" in str(e.value)


def test_decode_segment_larger_than_the_budget():
    codec = T.CODEC_ZSTD
    small, sraw, _ = _device_segments(codec, _words(20000, seed=7), 1)
    big, braw, _ = _device_segments(codec, _words(1500000, seed=8, vocab=1 << 28), 1)
    assert braw[0] > FLOOR
    with pytest.raises(TezGpuError) as e:
        native.decode_segments(small + big, sraw + braw, codec, FLOOR)
    msg = str(e.value)
    assert e.value.code == T.E_NOMEM
    assert "segment 1 (%d compressed bytes, %d raw bytes)" % (len(big[0]), braw[0]) in msg and str(FLOOR) in msg


# ------------------------------------------------------------------------------------------------ input
def _producers(tmp_path, codecs, n):
    return [run_output(tmp_path / ("t%d" % t), dict(WC, **_codec_conf(c)), _words(n, seed=100 + t), 1,
                        uid="attempt_1_0001_1_00_%06d_0_10001" % t) for t, c in enumerate(codecs)]


def _read(tmp, conf, producers):
    inp = OrderedGroupedKVInput(InputContext(conf, str(tmp)), len(producers))
    inp.initialize()
    inp.start()
    inp.handleEvents([LocalOutput(i, out.final_output_file, out.final_index_file, 0) for i, (out, _) in enumerate(producers)])
    r = inp.getReader()
    groups = []
    while r.next():
        groups.append((r.getCurrentKey(), b"".join(r.getCurrentValues())))
    counters = {k: inp.counter(k) for k in ("SHUFFLE_BYTES", "SHUFFLE_BYTES_DECOMPRESSED", "SHUFFLE_BYTES_DISK_DIRECT",
                                           "MERGED_MAP_OUTPUTS", "NUM_SHUFFLED_INPUTS", "REDUCE_INPUT_GROUPS",
                                           "REDUCE_INPUT_RECORDS")}
    return groups, counters, inp.merge_info()


@pytest.mark.parametrize("codecs", [(0, 0, 0), (T.CODEC_DEFAULT,) * 3, (T.CODEC_LZ4,) * 3, (T.CODEC_ZSTD,) * 3,
                                    (T.CODEC_LZ4, 0, T.CODEC_LZ4)], ids=["none", "default", "lz4", "zstd", "mixed"])
def test_input_under_budget_reads_what_it_reads_without(tmp_path, codecs):
    """An OrderedWordCount-shaped reduce: three producers of 120000 words each; at 16 and 64 MiB the merge takes
    several steps and returns the groups, values and counters of the merge without the key."""
    producers = _producers(tmp_path, codecs, 120000)
    conf = dict(WC, **_codec_conf(max(codecs)))
    exp_groups, exp_counters, exp_info = _read(tmp_path / "r", conf, producers)
    assert exp_info == (1, 0, 0) and exp_counters["REDUCE_INPUT_RECORDS"] == 360000
    for mb in (16, 64):
        groups, counters, (steps, peak, h2d) = _read(tmp_path / ("r%d" % mb), dict(conf, **{KEY: mb}), producers)
        assert groups == exp_groups and counters == exp_counters, mb
        assert steps > 1 and 0 < peak <= mb << 20 and h2d > 0, (mb, steps, peak)


# ------------------------------------------------------------------------------------------------ output
def _output(tmp, conf, recs):
    out, events = run_output(tmp, conf, recs, 4)
    with open(out.final_output_file, "rb") as f, open(out.final_index_file, "rb") as fi:
        return out, f.read(), fi.read()


@pytest.mark.parametrize("combine", [None, 1, 100], ids=["no_combiner", "combine_at_final_merge", "combine_spills_only"])
def test_output_final_merge_under_budget_writes_the_same_files(tmp_path, combine):
    conf = dict(WC, **{"tez.runtime.io.sort.mb": 1})
    if combine is not None:
        conf.update({"tez.runtime.combiner.class": "org.apache.tez.mapreduce.combine.MRCombiner",
                     "mapred.combiner.class": "org.apache.hadoop.mapreduce.lib.reduce.IntSumReducer",
                     "tez.runtime.combine.min.spills": combine})
    recs = _words(400000, seed=11)
    out0, f0, i0 = _output(tmp_path / "plain", conf, recs)
    assert out0.num_spills >= 3 and out0.merge_info() == (1, 0, 0)
    out1, f1, i1 = _output(tmp_path / "budget", dict(conf, **{KEY: 16}), recs)
    assert f1 == f0 and i1 == i0
    steps, peak, h2d = out1.merge_info()
    assert steps > 1 and 0 < peak <= FLOOR and h2d > 0
    for k in ("OUTPUT_RECORDS", "SPILLED_RECORDS", "OUTPUT_BYTES_PHYSICAL", "OUTPUT_BYTES_WITH_OVERHEAD",
              "COMBINE_INPUT_RECORDS", "COMBINE_OUTPUT_RECORDS"):
        assert out1.counter(k) == out0.counter(k), k


def test_output_with_codec_keeps_its_one_step_merge(tmp_path):
    conf = dict(WC, **_codec_conf(T.CODEC_LZ4), **{"tez.runtime.io.sort.mb": 1})
    recs = _words(400000, seed=12)
    out0, f0, i0 = _output(tmp_path / "plain", conf, recs)
    out1, f1, i1 = _output(tmp_path / "budget", dict(conf, **{KEY: 16}), recs)
    assert out0.num_spills >= 3 and f1 == f0 and i1 == i0 and f1[:4] == b"TIF\x01"
    assert out1.merge_info() == (1, 0, 0)


# ------------------------------------------------------------------------------------------------ unordered
def test_unordered_edges_ignore_the_key(tmp_path):
    recs = _words(150000, seed=13)
    files, readouts = [], []
    for name, extra in (("unset", {}), ("set", {KEY: 16})):
        conf = dict(WC, **{"tez.runtime.unordered.output.buffer.size-mb": 1}, **extra)
        ctx_dir = tmp_path / name
        o = UnorderedPartitionedKVOutput(OutputContext(conf, str(ctx_dir)), 3)
        o.initialize()
        o.start()
        w = o.getWriter()
        for k, v in recs:
            w.write(k, v)
        o.close()
        assert o.num_spills > 1
        files.append((open(o.final_output_file, "rb").read(), open(o.final_index_file, "rb").read()))
        inp = UnorderedKVInput(InputContext(conf, str(ctx_dir / "r")), 1)
        inp.initialize()
        inp.start()
        inp.handleEvents([LocalOutput(0, o.final_output_file, o.final_index_file, 1)])
        r = inp.getReader()
        got = []
        while r.next():
            got.append((r.getCurrentKey(), r.getCurrentValue()))
        readouts.append(got)
        assert inp.merge_info() == (1, 0, 0)
    assert files[0] == files[1] and readouts[0] == readouts[1] and len(readouts[0]) > 0

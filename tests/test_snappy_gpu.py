"""GPU: SnappyCodec on the device.  Every compressed segment the device writes is checked against the uncompressed
output of the oracle (or of the same merge without the codec): header, CRC of the stream, the strict model's decode,
libsnappy's decode where pyarrow imports, index triple, and byte for byte against the host emulation of the writer.
The reader is fed the Java-framed fixture (multi-chunk blocks included), device-written streams, mixes of compressed
and plain segments, one segment of about 1,100 blocks, hand-made chunks, a mutant corpus and wrong-codec streams,
through merge_open_codec, concat_open, decode_segments and next_batch_device."""
import random
import zlib

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import native
from tez_b200._lib import TezGpuError
import codec_model as CM
import combine_model as CBM
import lz4_model as L4
import snappy_model as M
import zstd_model as ZS
from test_codec_gpu import _c3, _fixed_kv, _plain, _records

pytestmark = pytest.mark.gpu
Z = T.CODEC_SNAPPY


def check_segment(seg, body, model=None):
    """one device-written Snappy segment against its uncompressed body.  The Python model decodes bodies up to 4 MiB;
    the emulated reader (checked against the model on the CPU) decodes larger ones."""
    if model is None:
        model = len(body) <= 4 << 20
    assert seg[:4] == b"TIF\x01"
    assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])
    assert (M.decode_stream if model else M.decompress_emulate)(seg[4:-4], len(body)) == body
    assert seg[4:-4] == M.compress_emulate(body), "device bytes differ from the host emulation"
    if M.pyarrow() is not None and model:
        assert M.decode_stream(seg[4:-4], len(body), M.libsnappy_chunk) == body


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
    return raw + 14 * (raw // T.SNAPPY_BLOCK_BYTES + P + 1) + 64


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
    assert ratio < 1.01 if kind == "c2" else ratio < 0.8


@pytest.mark.parametrize("unordered", [False, True])
def test_sorter_sort_device_variable_length(unordered):
    recs = _records(O.CMP_TEXT, 40000, seed=31) + [(O.text("big"), bytes(range(256)) * 300)]
    kv, ko, kl, vl, vo = CBM.pack(recs)
    P = 8
    conf = O.sorter_conf(P, cmp_kind=O.CMP_TEXT)
    exp = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl)
    n, kv_bytes = len(recs), int(kv.size)
    d_kv = torch.from_numpy(np.concatenate([kv, np.zeros(16, np.uint8)])).cuda()
    d_ko = torch.from_numpy(ko.astype(np.int64)).cuda()
    d_vo = torch.from_numpy(vo.astype(np.int64)).cuda()
    d_vl = torch.from_numpy(vl.astype(np.int32)).cuda()
    with T.GpuSorter(P, comparator=T.CMP_TEXT, codec=Z, unordered=unordered) as s:
        cap = s.device_output_bound(n, kv_bytes)
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ln, index, _ = s.sort_device(d_kv.data_ptr(), kv_bytes, d_ko.data_ptr(), d_vo.data_ptr(), d_vl.data_ptr(), n,
                                     d_out.data_ptr(), cap)
        out = d_out[:ln].cpu().numpy().tobytes()
    check_file(out, index, exp["file_out"], exp["index"])


def test_set_codec_errors_and_reset():
    with T.GpuSorter(4) as s:
        with pytest.raises(TezGpuError, match="codec 7") as e:
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
def _fixture():
    """the Java-framed segments of the fixture (its crafted segments decode to bytes that are not records)"""
    fx = [f for f in M.fixture() if not f[0].startswith("crafted_")]
    return [s for _, s, _ in fx], [r for _, _, r in fx]


def test_merger_java_framed_fixture_merge_and_concat():
    """The fixture's segments (Java block cutting, libsnappy chunks, a block of several chunks, hand-made chunks)
    merge and concatenate to what the model-decoded segments give."""
    segs, raws = _fixture()
    plain = [_plain(M.decode_stream(s[4:-4], r - 4)) for s, r in zip(segs, raws)]
    for concat in (False, True):
        kw = dict(concat=True) if concat else dict(comparator=T.CMP_BYTES)
        with T.GpuMerger(plain, **kw) as m:
            exp_recs = list(m.records())
        with T.GpuMerger(plain, **kw) as m:
            exp_ifile = m.write_ifile(rle=False)[0]
        with T.GpuMerger(segs, codec=Z, raw_lens=raws, **kw) as m:
            assert list(m.records()) == exp_recs
        with T.GpuMerger(segs, codec=Z, raw_lens=raws, **kw) as m:
            seg, raw, part, st = m.write_ifile(rle=False)
        _check_merged(seg, raw, part, exp_ifile)
        assert st["file_out_bytes"] == part


@pytest.mark.parametrize("mode", ["device", "java"])
def test_merger_snappy_inputs_mixed_with_plain(mode):
    plain = _c3(6, seed=len(mode))
    exp = O.merge(plain, O.CMP_TEXT)
    segs, raws = [], []
    for i, s in enumerate(plain):
        if i % 3 == 2:
            segs.append(s)
            raws.append(0)
            continue
        body = CM.body_of(s)
        z = M.compress_emulate(body) if mode == "device" else M.java_stream(M.ifile_writes(body), compress=_java_chunk)
        segs.append(M.segment(z))
        raws.append(len(body) + 4)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=Z, raw_lens=raws) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
        assert m.counts()[0] == len(exp["records"])
    _check_merged(seg, raw, part, exp["ifile"])
    with T.GpuMerger(segs[:2], comparator=T.CMP_TEXT, codec=Z, raw_lens=raws[:2]) as m:
        m.reopen(segs[2:], raw_lens=raws[2:])
        seg, raw, part, _ = m.write_ifile(rle=False)
    _check_merged(seg, raw, part, O.merge(plain[2:], O.CMP_TEXT)["ifile"])


def _java_chunk(d):
    """libsnappy's chunk where pyarrow imports, else an all-literal chunk (the block framing is Java's either way)"""
    if M.pyarrow() is not None:
        return M.snappy_compress(d)
    return M.varint(len(d)) + M.lit(bytes(d))


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


def test_next_batch_device_on_a_snappy_handle():
    segs, raws = _fixture()
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=raws) as m:
        want = list(m.records())
    got = []
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=raws) as m:
        for kv, ko, vo, vl, sk in m.records_device(batch_records=997, batch_bytes=1 << 20):
            b = kv.cpu().numpy().tobytes()
            got += [(b[a:c], b[c:c + d], bool(s)) for a, c, d, s in zip(ko.tolist(), vo.tolist(), vl.tolist(), sk.tolist())]
    assert got == want and len(got) > 1000


def test_merger_one_segment_of_a_thousand_blocks():
    """about 70 MB in one segment: about 1,100 chunks decoded by as many warps, then merged with a small segment"""
    big = O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 850000, seed=41), 16, 64)["file_out"]
    small = O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 1000, seed=42), 16, 64)["file_out"]
    zb = M.compress_emulate(CM.body_of(big))
    assert len(M.blocks(zb)) >= 1000
    segs = [M.segment(zb), M.segment(M.compress_emulate(CM.body_of(small)))]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=Z, raw_lens=[len(big) - 4, len(small) - 4]) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
    with T.GpuMerger([big, small], comparator=T.CMP_BYTES) as m:
        _check_merged(seg, raw, part, m.write_ifile(rle=False)[0])


@pytest.mark.parametrize("budget", [1 << 30, 16 << 20])
def test_decode_segments_one_group_and_several(budget):
    fx = M.fixture() * (1 if budget > 1 << 29 else 6)
    plain = _c3(2, seed=8)
    segs, raws = [s for _, s, _ in fx] + plain, [r for _, _, r in fx] + [0, 0]
    imgs, peak = native.decode_segments(segs, raws, Z, budget)
    for s, r, img in zip(segs, raws, imgs):
        if r == 0:
            assert img is None
            continue
        body = M.decode_stream(s[4:-4], r - 4)
        assert img == b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")
    assert 0 < peak <= budget


def test_merger_rejects_malformed_and_wrong_codec_segments():
    plain = _c3(3, seed=5)
    bodies = [CM.body_of(s) for s in plain]
    segs = [M.segment(M.compress_emulate(b)) for b in bodies]
    raws = [len(b) + 4 for b in bodies]

    def opened(segs_, raws_, codec=Z):
        with T.GpuMerger(segs_, comparator=T.CMP_TEXT, codec=codec, raw_lens=raws_) as m:
            return m.counts()

    z = bytearray(segs[1][4:-4])
    z[0:4] = (int.from_bytes(z[0:4], "big") - 1).to_bytes(4, "big")
    with pytest.raises(IOError, match="compressed segment 1: chunks decode past"):
        opened([segs[0], M.segment(bytes(z)), segs[2]], raws)
    with pytest.raises(IOError, match="compressed segment 2"):
        opened(segs, raws[:2] + [raws[2] + 1])
    with pytest.raises(IOError, match="compressed segment 0: bytes after the last block"):
        opened([M.segment(segs[0][4:-4] + b"\0\0\0\0")] + segs[1:], raws)
    with pytest.raises(IOError, match="checksum mismatch in segment 1"):
        opened([segs[0], segs[1][:-1] + bytes([segs[1][-1] ^ 1]), segs[2]], raws)
    with pytest.raises(TezGpuError) as e:
        opened(segs, None)
    assert e.value.code == T.E_INVALID
    # zlib, LZ4 and zstd streams given to a Snappy merger, and a Snappy stream given to each of theirs
    others = {T.CODEC_DEFAULT: CM.compressed_segment(bodies[0], 6)[0], T.CODEC_LZ4: L4.segment(L4.compress_emulate(bodies[0])),
              T.CODEC_ZSTD: ZS.segment(ZS.compress_emulate(bodies[0]))}
    for codec, other in others.items():
        with pytest.raises(IOError, match="compressed segment 0"):
            opened([other] + segs[1:], raws)
        with pytest.raises(IOError, match="compressed segment 0"):
            opened(segs, raws, codec=codec)


# ------------------------------------------------------------------------------------------------ 32-lane paths
def _cases():
    """(name, stream, expect): the hand-made chunks alone, as one block of several, and the CPU suite's malformed
    streams"""
    from test_snappy_cpu import MALFORMED
    cr = M.crafted_chunks()
    res = [("crafted_" + n, M.one_block([c]), M.preamble(c)[0]) for n, c in cr]
    res.append(("crafted_all_in_one_block", M.one_block([c for _, c in cr]), sum(M.preamble(c)[0] for _, c in cr)))
    res += [("malformed_" + k, z, e) for k, (z, e, _) in sorted(MALFORMED.items())]
    return res


def _decode_all(cases):
    """every case through one decode_segments call: each must give the emulation's bytes or its reason; a batch with
    a bad segment names the first bad index"""
    segs = [M.segment(z) for _, z, _ in cases]
    raws = [e + 4 for _, _, e in cases]
    verdicts = []
    for _, z, e in cases:
        try:
            verdicts.append(M.decompress_emulate(z, e))
        except TezGpuError as err:
            assert err.code == T.E_FORMAT
            verdicts.append(str(err).split("compressed segment 0: ")[-1])
    good = [i for i, v in enumerate(verdicts) if isinstance(v, bytes)]
    if good:
        imgs, _ = native.decode_segments([segs[i] for i in good], [raws[i] for i in good], Z, 1 << 30)
        for i, img in zip(good, imgs):
            assert img[4:-4] == verdicts[i], cases[i][0]
    bad = [i for i, v in enumerate(verdicts) if isinstance(v, str)]
    for i in bad:
        with pytest.raises(TezGpuError) as err:
            native.decode_segments([segs[i]], [raws[i]], Z, 1 << 30)
        assert err.value.code == T.E_FORMAT and str(err.value).endswith("compressed segment 0: " + verdicts[i]), cases[i][0]
    if bad and good:
        g = good[0]
        batch = [segs[g]] * 3 + [segs[bad[0]]] + [segs[g]] * 2
        with pytest.raises(TezGpuError, match="compressed segment 3: " + verdicts[bad[0]]):
            native.decode_segments(batch, [raws[g]] * 3 + [raws[bad[0]]] + [raws[g]] * 2, Z, 1 << 30)
    return len(good), len(bad)


@pytest.mark.parametrize("order", ["forward", "reversed"])
def test_crafted_and_malformed_cases_on_32_lanes(order):
    cases = _cases()
    if order == "reversed":
        cases = cases[::-1]
    good, bad = _decode_all(cases)
    assert good >= 5 and bad >= 20


@pytest.mark.parametrize("order", ["forward", "reversed"])
def test_mutant_corpus_on_32_lanes(order):
    from test_snappy_cpu import corpus_streams
    muts = M.mutants(corpus_streams(), 3000, seed=4321)
    cases = [("mutant_%d" % i, z, e) for i, (z, e) in enumerate(muts) if e >= 2 and len(z) >= 2]
    if order == "reversed":
        cases = cases[::-1]
    # the good ones in one call; every bad one alone (its reason)
    good, bad = _decode_all(cases)
    assert good > 100 and bad > 300

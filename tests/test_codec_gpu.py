"""GPU: DefaultCodec on the device.  Every compressed segment the device writes is checked against the uncompressed
output of the oracle (or of the same merge without the codec) (header, CRC of the compressed bytes, zlib.decompress of the stream, index triple) and byte for
byte against the host emulation of the writer.  The reader is fed the reference fixture, zlib-made streams, mixes of
compressed and uncompressed segments and malformed streams."""
import random
import zlib

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import native
from tez_b200._lib import TezGpuError
import codec_model as M
import combine_model as CM
from test_codec_cpu import FIXTURE_COMPRESSED, FIXTURE_RAWS, GOLDEN

pytestmark = pytest.mark.gpu
Z = T.CODEC_DEFAULT


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
        assert len(seg) == part and seg[:4] == b"TIF\x01"
        assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])
        body = exp_file[es + 4:es + epart - 4]
        assert zlib.decompress(seg[4:-4]) == body
        assert seg[4:-4] == M.deflate_emulate(body), "device bytes differ from the host emulation"
        pos += part
    assert pos == len(out)


def _zcap(raw, P):
    """capacity for a compressed file.out whose uncompressed form is at most raw bytes (every chunk stored)"""
    return raw + 5 * (raw // M.CHUNK + P + 1) + 11 * P + 64


def _key(cmp_kind, x):
    if cmp_kind == O.CMP_TEXT:
        return O.text("w%d" % x)
    if cmp_kind == O.CMP_BYTESWRITABLE:
        b = x.to_bytes(4, "big").lstrip(b"\0") * (1 + x % 3)
        return len(b).to_bytes(4, "big") + b
    if cmp_kind == O.CMP_INT:
        return O.int_writable(x - 1000)
    if cmp_kind == O.CMP_LONG:
        return O.long_writable(-x * 999983)
    return x.to_bytes(5, "big").lstrip(b"\0") or b"\0"


def _records(cmp_kind, n, seed, vocab=3000):
    rng = random.Random(seed)
    return [(_key(cmp_kind, min(int(rng.paretovariate(1.1)), vocab)), O.int_writable(1)) for _ in range(n)]


def _sort_case(recs, P, cmp_kind, rle=-1, send_empty=True, partition=None, combiner=0, unordered=False):
    kv, ko, kl, vl, vo = CM.pack(recs)
    part_mode = T.PART_GIVEN if partition is not None else T.PART_HASH
    if combiner:
        exp = CM.sort_combine(P, cmp_kind, combiner, kv, ko, kl, vl, partition, send_empty=send_empty)
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
    part = [zlib.crc32(k) % 5 * 3 for k, _ in recs]      # partitions 0, 3, 6, 9, 12 of 16: the others are empty
    _sort_case(recs, 16, O.CMP_TEXT, rle=rle, send_empty=send_empty, partition=part)


def test_sorter_no_records():
    _sort_case([], 8, O.CMP_TEXT, send_empty=False)
    _sort_case([], 8, O.CMP_TEXT, send_empty=True)


def test_sorter_unordered_handle():
    _sort_case(_records(O.CMP_TEXT, 20000, seed=9), 32, O.CMP_TEXT, unordered=True)


@pytest.mark.parametrize("combiner", [T.COMBINE_SUM_INT, T.COMBINE_SUM_LONG])
def test_sorter_with_combiner(combiner):
    rng = random.Random(combiner)
    w = 4 if combiner == T.COMBINE_SUM_INT else 8
    recs = [(k, rng.getrandbits(8 * w).to_bytes(w, "big")) for k, _ in _records(O.CMP_TEXT, 30000, seed=combiner)]
    _, _, st = _sort_case(recs, 16, O.CMP_TEXT, combiner=combiner)
    assert st["spilled_records"] < 30000


def _fixed_kv(kind, n, seed):
    if kind == "c2":
        return O.gen_c2(0, n, seed=seed, threads=8)
    rng = np.random.default_rng(seed)
    k = np.minimum(rng.zipf(1.3, n), 1 << 20).astype(">i8").view(np.uint8).reshape(n, 8)
    v = np.ones(n, dtype=">i8").view(np.uint8).reshape(n, 8)
    return np.ascontiguousarray(np.concatenate([k, v], axis=1)).reshape(-1)


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
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            ln, index, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
            out = d_out[:ln].cpu().numpy().tobytes()
    check_file(out, index, exp["file_out"], exp["index"])
    ratio = len(out) / len(exp["file_out"])
    assert ratio < 1.001 if kind == "c2" else ratio < 0.5


def test_set_codec_errors():
    with T.GpuSorter(4) as s:
        with pytest.raises(TezGpuError) as e:
            s.set_codec(7)
        assert e.value.code == T.E_UNSUPPORTED
        s.collect(b"\x01a\x00\x00\x00\x01", [0], [2], [4])
        with pytest.raises(TezGpuError) as e:
            s.set_codec(Z)
        assert e.value.code == T.E_STATE


def test_codec_survives_reset():
    recs = _records(O.CMP_TEXT, 5000, seed=3)
    kv, ko, kl, vl, vo = CM.pack(recs)
    exp = O.pipelined_sort(O.sorter_conf(4, cmp_kind=O.CMP_TEXT), kv, ko, kl, vl)
    with T.GpuSorter(4, comparator=T.CMP_TEXT, codec=Z) as s:
        for _ in range(2):
            s.collect(kv, ko.astype(np.uint32), vo, vl)
            out, _, index, _ = s.flush_to_memory()
            check_file(out, index, exp["file_out"], exp["index"])
            s.reset()


# ------------------------------------------------------------------------------------------------ merger
def _fixture():
    data = open(GOLDEN + "/TestIFile_concatenated_compressed.bin", "rb").read()
    segs, pos = [], 0
    for c in FIXTURE_COMPRESSED:
        segs.append(data[pos:pos + c])
        pos += c
    return segs


def _plain(body):
    return b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")


def _check_merged(seg, raw, part, exp_ifile):
    assert seg[:4] == b"TIF\x01" and part == len(seg) and raw == len(exp_ifile) - 4
    assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])
    body = exp_ifile[4:-4]
    assert zlib.decompress(seg[4:-4]) == body
    assert seg[4:-4] == M.deflate_emulate(body)


def test_merger_fixture_segments():
    """The reference's five compressed segments (written by the real IFile.Writer; their keys are not in comparator
    order, so the expectation is the same merge over the decompressed segments, and the oracle's records)."""
    segs = _fixture()
    plain = [_plain(zlib.decompress(s[4:-4])) for s in segs]
    oracle = sorted((k, v) for p in plain for _, k, v in O.read_ifile(p))
    with T.GpuMerger(plain, comparator=T.CMP_TEXT) as m:
        exp_recs = list(m.records())
    with T.GpuMerger(plain, comparator=T.CMP_TEXT) as m:
        exp_ifile = m.write_ifile(rle=False)[0]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=Z, raw_lens=FIXTURE_RAWS) as m:
        got = list(m.records())
    assert got == exp_recs
    assert sorted((k, v) for k, v, _ in got) == oracle
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=Z, raw_lens=FIXTURE_RAWS) as m:
        seg, raw, part, st = m.write_ifile(rle=False)
    _check_merged(seg, raw, part, exp_ifile)
    assert st["file_out_bytes"] == part


def _c3(nseg, seed=3):
    segs, _ = O.gen_c3_segments(nseg, 1 << 17, seed=seed, threads=8)
    return [s.tobytes() for s in segs]


@pytest.mark.parametrize("level,strategy", [(0, 0), (1, 0), (6, 0), (9, 0), (6, zlib.Z_FIXED), (6, zlib.Z_HUFFMAN_ONLY),
                                            (6, zlib.Z_RLE), (6, zlib.Z_FILTERED)])
def test_merger_zlib_inputs_mixed_with_plain(level, strategy):
    plain = _c3(6, seed=level * 10 + strategy)
    exp = O.merge(plain, O.CMP_TEXT)
    segs, raws = [], []
    for i, s in enumerate(plain):
        if i % 3 == 2:             # every third segment stays uncompressed
            segs.append(s)
            raws.append(0)
        else:
            z, raw = M.compressed_segment(M.body_of(s), level, strategy, members=1 + (i % 2))
            segs.append(z)
            raws.append(raw)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=Z, raw_lens=raws) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
        assert m.counts()[0] == len(exp["records"])
    _check_merged(seg, raw, part, exp["ifile"])


def test_merger_fixed_width_reaches_run_table_mode_and_reopen():
    plain = [O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, 20000, seed=s), 16, 64)["file_out"] for s in (1, 2, 3)]
    exp = O.merge(plain, O.CMP_BYTES)
    zs = [M.compressed_segment(M.body_of(s), 1) for s in plain]
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
        kv, ko, kl, vl, vo = CM.pack(recs)
        r = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT, rle_policy=0), kv, ko, kl, vl)
        outs.append((r["file_out"], r["index"]))
    segs, parts, raws, plain, flat = [], [], [], {p: [] for p in range(P)}, []
    for fo, idx in outs:
        for p in range(P):
            s0, raw, part = (int(x) for x in idx[p])
            if part == 0:
                continue
            seg = fo[s0:s0 + part]
            z, r = M.compressed_segment(M.body_of(seg), 6)
            segs.append(z); parts.append(p); raws.append(r); plain[p].append(seg); flat.append(seg)
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P, codec=Z, raw_lens=raws) as m:
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
    check_file(out, index, ref, rindex)
    with T.GpuMerger(segs[:2], comparator=T.CMP_TEXT, codec=Z, raw_lens=raws[:2], combiner=T.COMBINE_SUM_INT) as m:
        seg, raw, part, _ = m.write_ifile()
    with T.GpuMerger(flat[:2], comparator=T.CMP_TEXT, combiner=T.COMBINE_SUM_INT) as m:
        eseg = m.write_ifile()[0]
    _check_merged(seg, raw, part, eseg)


def test_merger_rejects_malformed_compressed_segments():
    plain = _c3(3, seed=5)
    zs = [M.compressed_segment(M.body_of(s), 6) for s in plain]
    segs, raws = [z for z, _ in zs], [r for _, r in zs]

    def opened(segs_, raws_):
        with T.GpuMerger(segs_, comparator=T.CMP_TEXT, codec=Z, raw_lens=raws_) as m:
            return m.counts()

    # a flipped bit in the stream, checksum recomputed: the inflate fails
    z = bytearray(segs[1][4:-4])
    z[len(z) // 2] ^= 0x10
    bad = b"TIF\x01" + bytes(z) + zlib.crc32(bytes(z)).to_bytes(4, "big")
    with pytest.raises(IOError, match="compressed segment 1"):
        opened([segs[0], bad, segs[2]], raws)
    # wrong rawLength
    with pytest.raises(IOError, match="compressed segment 2"):
        opened(segs, raws[:2] + [raws[2] + 1])
    # checksum of the compressed bytes
    with pytest.raises(IOError, match="checksum mismatch in segment 1"):
        opened([segs[0], segs[1][:-1] + bytes([segs[1][-1] ^ 1]), segs[2]], raws)
    # no raw lengths for compressed segments
    with pytest.raises(TezGpuError) as e:
        opened(segs, None)
    assert e.value.code == T.E_INVALID
    # without a codec the compressed flag is still refused
    with pytest.raises(IOError, match="compressed"):
        T.GpuMerger(segs, comparator=T.CMP_TEXT)


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
        with T.GpuMerger(plain, comparator=T.CMP_LONG) as m:   # the same merge without the codec
            _check_merged(seg, raw, part, m.write_ifile()[0])
        got = native.shuffle_receive(native.shuffle_serve(d_out.data_ptr(), index, "attempt_1", 0, P))
        wsegs = [g[3] for g in got if len(g[3])]
        wraws = [g[2] for g in got if len(g[3])]
        assert len(wsegs) == len(live)
        with T.GpuMerger(wsegs, comparator=T.CMP_LONG, codec=Z, raw_lens=wraws) as m:
            seg2, raw2, part2, _ = m.write_ifile()
        assert seg2 == seg and raw2 == raw

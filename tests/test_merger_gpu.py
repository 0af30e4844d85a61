"""GPU parity tests of the reduce-side k-way merge (libtezgpu through the C ABI) against the CPU oracle's restatement
of TezMerger.MergeQueue, on the reference's own known-answer tables (TestTezMerger) and on seeded random runs."""
import random
import zlib

import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
from test_oracle_golden import MERGER_TABLES, _ifile_with_text_data

pytestmark = pytest.mark.gpu


def _gpu_merge(segs, cmp_kind, has_header=True, fixed=None, writer_rle=False, check_for_same_keys=True):
    with T.GpuMerger(segs, comparator=cmp_kind, has_header=has_header, fixed=fixed) as m:
        if not check_for_same_keys:
            m.set_check_for_same_keys(False)
        nrec, kvb = m.counts()
        recs = list(m.records(batch_records=1000, batch_bytes=1 << 16))
        assert len(recs) == nrec
        assert sum(len(k) + len(v) for k, v, _ in recs) == kvb
        seg, raw, part, st = m.write_ifile(rle=writer_rle)
        assert part == len(seg) == raw + 4
        assert st["kernel_launches"] > 0
    return recs, seg


@pytest.mark.parametrize("name", sorted(MERGER_TABLES))
def test_tez_merger_known_answer_tables_on_gpu(name):
    """RLT/common/sort/impl/TestTezMerger.java:185-552 -- (key, SAME_KEY/DIFF_KEY) streams."""
    files, expected = MERGER_TABLES[name]
    segs = [_ifile_with_text_data(keys, i) for i, keys in enumerate(files)]
    recs, seg = _gpu_merge(segs, T.CMP_BYTES)  # keys are Text bytes with equal-length prefixes: raw byte order == expected order
    assert [(k[1:].decode(), same) for k, _, same in recs] == expected
    assert sorted(v for _, v, _ in recs) == sorted(v for s in segs for _, _, v in O.read_ifile(s))
    back = O.read_ifile(seg)
    assert [(ks == O.SAME_KEY) for ks, _, _ in back] == [s for _, s in expected]
    assert int.from_bytes(seg[-4:], "big") == zlib.crc32(seg[4:-4])


def _random_runs(rng, nseg, per_seg, key_fn, val_fn, rle_inputs=True):
    segs = []
    for s in range(nseg):
        keys = sorted((key_fn(rng) for _ in range(rng.randint(0, per_seg))), key=lambda kb: kb[1])
        segs.append(O.write_ifile([(kb[0], val_fn(kb[0])) for kb in keys], rle=rle_inputs)[0])
    return segs


@pytest.mark.parametrize("nseg,per_seg", [(1, 50), (2, 2000), (7, 500), (40, 300), (256, 40)])
def test_int_keys_merge_bit_exact_vs_oracle(nseg, per_seg):
    """testMerge grid (TestTezMerger.java:110-154) shape: IntWritable keys (signed order), value = f(key)."""
    rng = random.Random(nseg * 1000 + per_seg)

    def key_fn(r):
        v = r.randint(-300, 300)
        return (O.int_writable(v), v)

    segs = _random_runs(rng, nseg, per_seg, key_fn, lambda k: O.long_writable(zlib.crc32(k)))
    for writer_rle in (False, True):
        exp = O.merge(segs, O.CMP_INT, factor=100, writer_rle=writer_rle)
        recs, seg = _gpu_merge(segs, T.CMP_INT, writer_rle=writer_rle)
        assert [(k, v) for k, v, _ in recs] == [(k, v) for k, v, _ in exp["records"]]
        assert [s for _, _, s in recs] == [s for _, _, s in exp["records"]]
        assert seg == exp["ifile"]


def test_text_keys_variable_length_bit_exact():
    """BASELINE config 3 shape (small): Text keys of length U[4,24], value 8 B = f(key)."""
    rng = random.Random(33)

    def key_fn(r):
        w = "".join(r.choice("abcdefghijklmnop") for _ in range(r.randint(4, 24)))
        return (O.text(w), w.encode())

    segs = _random_runs(rng, 16, 3000, key_fn, lambda k: zlib.crc32(k).to_bytes(4, "big") * 2, rle_inputs=False)
    exp = O.merge(segs, O.CMP_TEXT, factor=100)
    recs, seg = _gpu_merge(segs, T.CMP_TEXT)
    assert seg == exp["ifile"]
    assert [(k, v, s) for k, v, s in recs] == exp["records"]


def test_in_memory_segments_without_header():
    rng = random.Random(5)

    def key_fn(r):
        b = bytes(r.getrandbits(3) for _ in range(r.randint(1, 6)))
        return (b, b)

    # (empty keys are never run-length encoded by IFile.Writer, so repeated empty keys INSIDE one segment make the
    #  reference's SAME/DIFF flags depend on its heap's tie order -- DESIGN.md "parity caveats"; one per segment is fine)
    segs = _random_runs(rng, 5, 400, key_fn, lambda k: k[::-1])
    segs = [O.write_ifile([(b"", b"empty")] + [(k, v) for _, k, v in O.read_ifile(s)], rle=True)[0] if i % 2 == 0 else s
            for i, s in enumerate(segs)]
    inmem = [s[4:] for s in segs]                     # body + crc (OG/InMemoryWriter.java:55-77)
    exp = O.merge(segs, O.CMP_BYTES, factor=100, writer_rle=True)
    recs, seg = _gpu_merge(inmem, T.CMP_BYTES, has_header=False, writer_rle=True)
    assert [(k, v) for k, v, _ in recs] == [(k, v) for k, v, _ in exp["records"]]
    assert seg == exp["ifile"]
    # fetched MEMORY segments end in 4 slack bytes instead of a checksum: still readable (InMemoryReader stops at EOF)
    slack = [s[:-4] + b"\0\0\0\0" for s in inmem]
    recs2, seg2 = _gpu_merge(slack, T.CMP_BYTES, has_header=False, writer_rle=True)
    assert seg2 == seg


def test_merge_of_gpu_sorted_fixed_width_partitions():
    """Reduce side of the multi-GPU flow: G producers' segments of one partition -> one merged segment."""
    segs, all_rows = [], []
    for g in range(4):
        kv = O.gen_c2(g * 100000, 20000 + g, seed=4 + g)
        with T.GpuSorter(1, fixed=(16, 64)) as s:
            s.collect_fixed(kv)
            out, _, _, _ = s.flush_to_memory()
        segs.append(bytes(out))
        all_rows += [bytes(r) for r in kv.reshape(-1, 80)]
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    for fixed in (None, (16, 64)):
        recs, seg = _gpu_merge(segs, T.CMP_BYTES, fixed=fixed)
        assert seg == exp["ifile"]
    assert [k + v for k, v, _ in recs] == sorted(all_rows, key=lambda b: b[:16])


def test_corrupt_segments_are_rejected():
    seg = O.write_ifile([(O.text("a"), O.text("1")), (O.text("b"), O.text("2"))])[0]
    ok = O.write_ifile([(O.text("c"), O.text("3"))])[0]
    bad_crc = seg[:-1] + bytes([seg[-1] ^ 0xFF])
    with pytest.raises(IOError, match="checksum"):
        T.GpuMerger([ok, bad_crc], comparator=T.CMP_TEXT)
    bad_hdr = b"XIF\0" + seg[4:]
    with pytest.raises(IOError, match="ifile header"):
        T.GpuMerger([bad_hdr], comparator=T.CMP_TEXT)
    with pytest.raises(IOError):
        T.GpuMerger([seg[:7]], comparator=T.CMP_TEXT)
    # body with a record running past the end, checksum made consistent
    body = b"\x7f\x01" + b"xy" + b"\xff\xff"
    trunc = b"TIF\0" + body + zlib.crc32(body).to_bytes(4, "big")
    with pytest.raises(IOError, match="malformed"):
        T.GpuMerger([trunc], comparator=T.CMP_TEXT)
    compressed = b"TIF\x01" + seg[4:]
    with pytest.raises(IOError, match="compressed"):
        T.GpuMerger([compressed], comparator=T.CMP_TEXT)


def test_empty_inputs():
    empty = O.write_ifile([])[0]
    recs, seg = _gpu_merge([empty, empty, empty], T.CMP_BYTES)
    assert recs == [] and seg == empty
    recs, seg = _gpu_merge([], T.CMP_BYTES)
    assert recs == [] and seg == empty


def test_batched_multi_partition_merge_matches_per_partition_oracle():
    """Reduce side of the multi-GPU shuffle: segments of several partitions from several producers, one device pass."""
    import torch
    P, G = 6, 3
    outs = []
    for g in range(G):
        kv = O.gen_c2(g * 50000, 30000, seed=4)
        r = O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, 64)
        outs.append(r)
    segs, parts = [], []
    for g in range(G):
        for p in range(P):
            start, raw, part = (int(x) for x in outs[g]["index"][p])
            if part:
                segs.append(outs[g]["file_out"][start:start + part])
                parts.append(p)
    for fixed in ((16, 64), None):
        with T.GpuMerger(segs, comparator=T.CMP_BYTES, partitions=parts, num_partitions=P, fixed=fixed) as m:
            cap = m.output_bound()
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            n, index, st = m.write_partitions_device(d_out.data_ptr(), cap)
            out = d_out[:n].cpu().numpy().tobytes()
        off = 0
        for p in range(P):
            mine = [s for s, q in zip(segs, parts) if q == p]
            exp = O.merge(mine, O.CMP_BYTES, factor=100)["ifile"]
            start, raw, part = (int(x) for x in index[p])
            assert start == off and part == len(exp)
            assert out[start:start + part] == exp
            off += part
        assert off == n


def test_merger_reopen_and_large_runs_through_the_staged_parser():
    """Few large runs (the staged warp parser walks ~1e5 records per segment) and handle reuse."""
    rng = random.Random(77)
    segs = []
    for s in range(3):
        keys = sorted({rng.getrandbits(48).to_bytes(6, "big") + bytes([s]) for _ in range(40000)})
        segs.append(O.write_ifile([(k, (zlib.crc32(k) & 0xFFFF).to_bytes(2, "big") * (1 + k[0] % 3)) for k in keys])[0])
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    with T.GpuMerger(segs[:1], comparator=T.CMP_BYTES) as m:
        first, _, _, _ = m.write_ifile()
        assert first == O.merge(segs[:1], O.CMP_BYTES)["ifile"]
        m.reopen(segs)
        seg, raw, part, _ = m.write_ifile()
        assert seg == exp["ifile"]
        assert m.counts()[0] == len(exp["records"])


@pytest.mark.parametrize("inputs_rle", [False, True])
@pytest.mark.parametrize("dup_pct", [1, 5, 9, 30])
def test_check_for_same_keys_and_writer_rle_grid(inputs_rle, dup_pct):
    """MergeQueue(checkForSameKeys) x IFile.Writer(rle) (SORT/TezMerger.java:560-573,597-652; callers
    SORT/PipelinedSorter.java:797-814): duplicate keys inside and across >= 3 segments, value = f(key).  With
    checkForSameKeys off, isSameKey() is only what the input segments' own run-length encoding says."""
    rng = random.Random(1000 * dup_pct + inputs_rle)
    nseg, per = 5, 4000
    # Two kinds of duplicates, kept apart on purpose: keys SHARED by several segments occur at most once per segment, and
    # keys repeated INSIDE a segment are private to it.  When one key is both repeated inside a segment and present in
    # another one, the reference's SAME/DIFF flags depend on which of the two segments its heap (Hadoop PriorityQueue,
    # strict lessThan) happens to hold on top -- "parity unpinned" in DESIGN.md 6 -- and no canonical order reproduces it.
    shared_pool = [b"S" + rng.getrandbits(56).to_bytes(7, "big") for _ in range(nseg * per // 2)]
    segs = []
    for s in range(nseg):
        ndup = per * dup_pct // 100
        mine = set(b"P" + bytes([s]) + rng.getrandbits(48).to_bytes(6, "big") for _ in range(per // 2))
        keys = list(mine) + list(set(shared_pool[rng.randrange(len(shared_pool))] for _ in range(per // 2 + ndup)))
        private = sorted(mine)
        keys += [private[rng.randrange(len(private))] for _ in range(ndup)]          # repeats inside the segment
        keys.sort()
        segs.append(O.write_ifile([(k, zlib.crc32(k).to_bytes(4, "big") * (1 + k[1] % 3)) for k in keys], rle=inputs_rle)[0])
    shared = set(k for _, k, _ in O.read_ifile(segs[0]) if k) & set(k for _, k, _ in O.read_ifile(segs[1]))
    for check in (True, False):
        for writer_rle in (False, True):
            exp = O.merge(segs, O.CMP_BYTES, factor=100, check_for_same_keys=check, writer_rle=writer_rle)
            recs, seg = _gpu_merge(segs, T.CMP_BYTES, writer_rle=writer_rle, check_for_same_keys=check)
            assert [(k, v) for k, v, _ in recs] == [(k, v) for k, v, _ in exp["records"]]
            assert [s for _, _, s in recs] == [s for _, _, s in exp["records"]], (check, writer_rle)
            assert seg == exp["ifile"], (check, writer_rle)
            if not check and not writer_rle and not inputs_rle:   # nothing is a repeat: no RLE / V_END markers in the output
                assert not any(s for _, _, s in recs)
                assert all(ks == O.NEW_KEY for ks, _, _ in O.read_ifile(seg))
            if check and shared:                                  # equal keys of different segments ARE flagged
                assert any(s for _, _, s in recs)


def test_write_ifile_on_a_multi_partition_merger_is_rejected():
    segs = [O.write_ifile([(b"a", b"1")])[0], O.write_ifile([(b"b", b"2")])[0]]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, partitions=[0, 1], num_partitions=2) as m:
        with pytest.raises(IOError, match="num_partitions"):
            m.write_ifile()


@pytest.mark.parametrize("nseg,seg_kb,id_bits", [(16, 512, 14), (16, 8192, 22), (64, 256, 12)])
def test_config3_shape_text_merge_bit_exact(nseg, seg_kb, id_bits):
    """BASELINE config 3 shape: k-way merge of sorted IFile segments with Text keys of length U[4,24] drawn from a small
    word space (so every word occurs in many segments: large groups of EQUAL keys, REPEAT_KEY output).  Exercises the
    parallel window parser, the alphabet-compressed sort word and the equal-group shortcut; the merged IFile must equal
    the oracle's TezMerger.writeFile byte for byte."""
    segs, nrec = O.gen_c3_segments(nseg, seg_kb << 10, seed=3, threads=8, id_bits=id_bits)
    exp, n, _ = O.merge_ifile(segs, O.CMP_TEXT, factor=100)
    with T.GpuMerger([s.tobytes() for s in segs], comparator=T.CMP_TEXT) as m:
        assert m.counts()[0] == n == sum(nrec)
        mode, by_hand = m.parse_info()
        assert mode == 1, (mode, by_hand)                  # the window parser, not the sequential walker
        assert by_hand * 32768 * 50 <= sum(a.size for a in segs) + 50 * 32768 * nseg, by_hand   # guesses are right for > 98 % of the windows
        seg, raw, part, st = m.write_ifile()
    assert part == exp.size
    assert np.array_equal(np.frombuffer(seg, dtype=np.uint8), exp)
    # and without the cross-segment check (PipelinedSorter's final merge when the last spill saw few duplicates)
    exp2, _, _ = O.merge_ifile(segs, O.CMP_TEXT, factor=100, check_for_same_keys=False)
    with T.GpuMerger([s.tobytes() for s in segs], comparator=T.CMP_TEXT) as m:
        m.set_check_for_same_keys(False)
        seg2, _, part2, _ = m.write_ifile()
    assert np.array_equal(np.frombuffer(seg2, dtype=np.uint8), exp2)


@pytest.mark.parametrize("shape", ["binary_values", "rle_runs", "long_records", "ff_bytes"])
def test_window_parser_on_multi_window_segments(shape):
    """parse_windows.cuh: segments of many 32 KiB windows whose bytes invite wrong walks -- random binary values (every
    byte value is a plausible vint), long run-length encoded runs (windows that begin inside a run), records longer
    than a window, values full of 0xFF (EOF look-alikes).  Whatever route open() takes (window parser, or the sequential
    walker for malformed input) the merge must equal TezMerger's; well-formed input always takes the window parser, whose
    chase walks by hand whatever the guesses got wrong."""
    rng = random.Random(zlib.crc32(shape.encode()))
    rs = np.random.default_rng(11)
    segs = []
    for sidx in range(5):
        recs = []
        if shape == "binary_values":
            keys = sorted({rng.getrandbits(40).to_bytes(5, "big") for _ in range(30000)})
            for k in keys:
                recs.append((k, rs.integers(0, 256, 1 + k[4] % 23, dtype=np.uint8).tobytes() if sidx == 0 else bytes([k[3]]) * (1 + k[4] % 23)))
            # values must be a function of the key across segments: segment 0 keeps private keys
            if sidx == 0:
                recs = [(b"\x00" + k, v) for k, v in recs]
            else:
                recs = [(b"\x01" + k, v) for k, v in recs]
        elif shape == "rle_runs":
            keys = sorted({rng.getrandbits(24).to_bytes(3, "big") + bytes([sidx]) for _ in range(300)})
            for k in keys:
                for _ in range(1 + (k[0] * 7) % 900):       # runs of up to 900 repeats (tens of KB: whole windows inside one run)
                    recs.append((k, (zlib.crc32(k) & 0xFFFFFF).to_bytes(3, "big") * (1 + k[1] % 9)))
        elif shape == "long_records":
            keys = sorted({rng.getrandbits(32).to_bytes(4, "big") + bytes([sidx]) for _ in range(40)})
            for k in keys:
                recs.append((k, bytes([k[0]]) * (20000 + 1000 * (k[1] % 50))))
        else:
            keys = sorted({b"\xff" * (1 + rng.randint(0, 3)) + rng.getrandbits(32).to_bytes(4, "big") + bytes([sidx]) for _ in range(20000)})
            for k in keys:
                recs.append((k, b"\xff" * (2 + k[-2] % 30)))
        segs.append(O.write_ifile(recs, rle=True)[0])
    assert min(len(x) for x in segs) > 3 * 32768
    exp = O.merge(segs, O.CMP_BYTES, factor=100)
    with T.GpuMerger(segs, comparator=T.CMP_BYTES) as m:
        mode, by_hand = m.parse_info()
        assert mode == 1, (mode, by_hand)
        assert m.counts()[0] == len(exp["records"])
        seg, raw, part, _ = m.write_ifile()
    assert seg == exp["ifile"]


@pytest.mark.parametrize("val_len,n", [(4096, 6000), (256, 60000)])
def test_config5_shape_zipf_keys_sort_and_merge_bit_exact(val_len, n):
    """BASELINE config 5 shape: Zipf(1.1) keys (one key holds ~7 % of the records), large values = f(key), so the map side
    turns run-length encoding on, the reduce side parses RLE segments of multi-KB records, meets tie groups of thousands
    of equal keys, and writes REPEAT_KEY runs.  Map side vs the PipelinedSorter oracle, reduce side vs TezMerger."""
    from tez_b200 import synth
    P, G = 8, 3
    outs = []
    for g in range(G):
        kv = synth.gen_c5(g * n, n, seed=5, val_len=val_len, device="cuda").cpu().numpy()
        exp = O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, val_len)
        with T.GpuSorter(P, fixed=(16, val_len)) as s:
            s.collect_fixed(kv)
            out, index_bytes, index, st = s.flush_to_memory()
        assert st["rle_used"] and exp["rle_used"]
        assert np.array_equal(np.frombuffer(bytes(out), dtype=np.uint8), np.frombuffer(exp["file_out"], dtype=np.uint8))
        assert index_bytes == exp["index_out"]
        outs.append((bytes(out), index))
    segs, parts = [], []
    for g in range(G):
        for p in range(P):
            a, raw, ln = (int(x) for x in outs[g][1][p])
            if ln:
                segs.append(outs[g][0][a:a + ln])
                parts.append(p)
    import torch
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, partitions=parts, num_partitions=P, fixed=(16, val_len)) as m:
        cap = m.output_bound()
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        nbytes, index, st = m.write_partitions_device(d_out.data_ptr(), cap)
        merged = d_out[:nbytes].cpu().numpy()
    for p in range(P):
        mine = [sg for sg, q in zip(segs, parts) if q == p]
        a, raw, ln = (int(x) for x in index[p])
        if not mine:
            continue
        exp, _, _ = O.merge_ifile(mine, O.CMP_BYTES, factor=100)
        assert ln == exp.size and np.array_equal(merged[a:a + ln], exp), "partition %d" % p


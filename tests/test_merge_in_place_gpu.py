"""GPU: merges of segments that already sit in device memory and are read where they are (TEZGPU_SEG_DEVICE on every
segment: no staging copy, the segment table is relative to the lowest segment address rounded down to 16, and every
clamped load clamps to the whole span, not to one segment).

Every case places the same segments in device buffers several ways -- all starts 16-aligned with descending addresses,
one start residue 1..15 per segment across two allocations, back to back at odd offsets -- and fills the bytes around
them with 0xFF (EOF look-alikes, maximum sort bytes, -1 vints), with copies of another segment's body (plausible records
right behind each segment's end), or with seeded random bytes.  The merge over each placement must equal, bit for bit,
the same merge over the segments as host buffers (records, counts, the merged IFile, write_partitions_device's bytes and
index) and report the record-finding mode the case is meant to reach.  The host merge is checked against the oracle and,
where every value is its record's global index (big-endian), against the stable merge model of DESIGN.md section 6, so a
moved, lost or duplicated record is visible.

Run as a script (`python tests/test_merge_in_place_gpu.py serial-walker`, with TEZGPU_PARSE_SERIAL=1) it prints the
digests of the sequential walker's merges of the window-parser inputs; the switch is latched per process, so
test_sequential_walker_equals_the_window_parser runs it in a subprocess."""
import hashlib
import json
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200._lib import TezGpuError  # noqa: E402

import codec_model as CM  # noqa: E402
import combine_model as CBM  # noqa: E402
import lz4_model as L4  # noqa: E402
import unordered_model as UM  # noqa: E402
import zstd_model as ZS  # noqa: E402
from merge_model import GUARD, LAYOUTS, POISONS, check_oracle, partition_segments, place, run  # noqa: E402

pytestmark = pytest.mark.gpu

WINDOW = 32768     # the window parser's window (parse_windows.cuh)
PARSE_WIN = 4096   # the sequential walker's staging window (merger.cuh)


def check_in_place(segs, mode, layouts=tuple(LAYOUTS), poisons=tuple(POISONS), **kw):
    """The merge over every placement x poison equals the host merge, which reaches `mode`.  Returns the host merge."""
    host = run([bytes(s) for s in segs], **kw)
    assert host["mode"] == mode, "host merge took mode %d, not %d" % (host["mode"], mode)
    for k, layout in enumerate(layouts):
        for poison in poisons:
            ptrs, keep = place(segs, layout, poison, seed=k)
            dev = run(ptrs, device_ptrs=True, **kw)
            del keep
            for key in host:
                assert dev[key] == host[key], "%s differs from the host merge (layout %s, poison %s)" % (key, layout, poison)
    return host


# ------------------------------------------------------------------------------------------------ inputs
def fixed_segments(klen, vlen, G, P, n, seed, rle=False):
    """G producers' fixed-width records sorted by GpuSorter into P partitions (given ids); every value is the record's
    global index.  Keys come from a shared pool, each at most once per producer, so equal keys meet across segments
    only.  Returns (segments, partitions) in (producer, partition) order: partitions interleave."""
    rng = random.Random(seed)
    pool = [rng.randbytes(klen) for _ in range(n * 3 // 2)]
    segs, parts, gidx = [], [], 0
    for g in range(G):
        keys = rng.sample(pool, n)
        kv = b"".join(k + (gidx + j).to_bytes(vlen, "big") for j, k in enumerate(keys))
        gidx += n
        part = np.array([rng.randrange(P) for _ in range(n)], dtype=np.int32)
        with T.GpuSorter(P, fixed=(klen, vlen), partitioner=T.PART_GIVEN, rle_policy=T.RLE_ON if rle else T.RLE_OFF) as s:
            s.collect_fixed(np.frombuffer(kv, dtype=np.uint8), partition=part)
            out, _, index, _ = s.flush_to_memory()
        out = bytes(out)
        for p in range(P):
            start, _, ln = (int(x) for x in index[p])
            if ln:
                segs.append(out[start:start + ln])
                parts.append(p)
    return segs, parts


def rle_fixed_segments(nseg, n, seed):
    """fixed 16/64 records with runs of equal keys inside each segment (keys private to it), written run-length
    encoded: not the plain fixed framing"""
    rng = random.Random(seed)
    segs, gidx = [], 0
    for s in range(nseg):
        heads = sorted(bytes([s]) + rng.randbytes(15) for _ in range(n // 4))
        keys = sorted(rng.choice(heads) for _ in range(n))
        segs.append(O.write_ifile([(k, (gidx + j).to_bytes(64, "big")) for j, k in enumerate(keys)], rle=True)[0])
        gidx += n
    return segs


def window_segments(shape, nseg=3):
    """test_merger_gpu's multi-window shapes, every value ending in its record's global index"""
    rng = random.Random(zlib.crc32(shape.encode()))
    rs = np.random.default_rng(11)
    segs, gidx = [], 0
    for sidx in range(nseg):
        recs = []
        if shape == "binary_values":
            keys = sorted({bytes([sidx == 0]) + rng.getrandbits(40).to_bytes(5, "big") for _ in range(9000)})
            recs = [(k, rs.integers(0, 256, 1 + k[5] % 23, dtype=np.uint8).tobytes()) for k in keys]
        elif shape == "rle_runs":
            for k in sorted({rng.getrandbits(24).to_bytes(3, "big") + bytes([sidx]) for _ in range(90)}):
                recs += [(k, bytes([k[1]]) * (1 + k[1] % 9))] * (1 + (k[0] * 7) % 300)
        elif shape == "long_records":
            for k in sorted({rng.getrandbits(32).to_bytes(4, "big") + bytes([sidx]) for _ in range(12)}):
                recs.append((k, bytes([k[0]]) * (20000 + 1000 * (k[1] % 50))))
        else:
            keys = sorted({b"\xff" * (1 + rng.randint(0, 3)) + rng.getrandbits(32).to_bytes(4, "big") + bytes([sidx])
                           for _ in range(6000)})
            recs = [(k, b"\xff" * (2 + k[-2] % 30)) for k in keys]
        recs = [(k, v + (gidx + j).to_bytes(4, "big")) for j, (k, v) in enumerate(recs)]
        gidx += len(recs)
        segs.append(O.write_ifile(recs, rle=True)[0])
    assert min(len(s) for s in segs) > 3 * WINDOW
    return segs


def _vint_len(v):
    return 1 if -112 <= v <= 127 else 1 + (max(v, ~v).bit_length() + 7) // 8


def straddle_segments():
    """Two segments whose record headers straddle the sequential walker's PARSE_WIN staging window: the walk stages
    [wbase, wbase + PARSE_WIN) and restages at a record start rounded down to 16 when a header does not fit, and
    records are sized from a restatement of that rule so that two-byte key-length vints start on a window's last byte.
    Records longer than a window lie in between."""
    segs, gidx = [], 0
    for sidx in range(2):
        recs, off, wbase, j, straddles = [], 4, 4, 0, 0   # segment offset of the next record, of the staged window

        def header_at(h):
            nonlocal wbase, straddles
            if off + h > wbase + PARSE_WIN:
                straddles += off < wbase + PARSE_WIN
                wbase = off & ~15
        while straddles < 8:
            key = bytes([0x10 + sidx]) + j.to_bytes(3, "big")
            header_at(4)                                    # one-byte key length, three-byte value length
            pad = wbase + PARSE_WIN - 1 - off - 4 - len(key) - 4
            if pad < 256:
                pad += 2 * PARSE_WIN                        # too close: the next header restages the window
            val = bytes([j & 0xFF]) * pad + (gidx + j).to_bytes(4, "big")
            assert _vint_len(len(val)) == 3
            recs.append((key, val))
            off += 4 + len(key) + len(val)
            j += 1
            key = bytes([0x10 + sidx]) + j.to_bytes(3, "big") + bytes(126 + j % 5)   # 130..134 bytes: 2-byte vint
            val = bytes(3 + 7000 * (j % 3)) + (gidx + j).to_bytes(4, "big")        # some longer than the window
            header_at(_vint_len(len(key)) + _vint_len(len(val)))
            recs.append((key, val))
            off += _vint_len(len(key)) + _vint_len(len(val)) + len(key) + len(val)
            j += 1
        gidx += j
        segs.append(O.write_ifile(recs, rle=False)[0])
    return segs


def walker_inputs():
    """name -> (segments, merge kwargs) of the record-finder comparison (window parser vs sequential walker)"""
    res = {s: (window_segments(s), dict(comparator=T.CMP_BYTES)) for s in ("binary_values", "rle_runs", "long_records", "ff_bytes")}
    res["straddle"] = (straddle_segments(), dict(comparator=T.CMP_BYTES))
    return res


def walker_digests(mode):
    """sha256 of every output of the merges of walker_inputs(), host and in place; asserts the record-finding mode"""
    digests = {}
    for name, (segs, kw) in walker_inputs().items():
        for where in ("host", "device"):
            if where == "host":
                out = run([bytes(s) for s in segs], **kw)
            else:
                ptrs, keep = place(segs, "packed", "body")
                out = run(ptrs, device_ptrs=True, **kw)
                del keep
            assert out.pop("mode") == mode, (name, where)
            digests["%s/%s" % (name, where)] = hashlib.sha256(repr(sorted(out.items())).encode()).hexdigest()
    return digests


def text_segments(nseg, n, seed, vocab=3000, value=None):
    """sorted Text-key segments; a word at most once per segment; value = global index (4 bytes) unless given"""
    rng = random.Random(seed)
    segs, gidx = [], 0
    for s in range(nseg):
        words = sorted({"w%d" % rng.randrange(vocab) for _ in range(rng.randint(1, n))}, key=lambda w: w.encode())
        recs = [(O.text(w), value(w) if value else (gidx + j).to_bytes(4, "big")) for j, w in enumerate(words)]
        gidx += len(recs)
        segs.append(O.write_ifile(recs)[0])
    return segs


def compressed(codec, plain):
    body = CM.body_of(plain)
    if codec == T.CODEC_DEFAULT:
        z = CM.deflate_emulate(body)
    elif codec == T.CODEC_LZ4:
        z = L4.compress_emulate(body)
    else:
        z = ZS.compress_emulate(body)
    return b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big"), len(plain) - 4


# ------------------------------------------------------------------------------------------------ run table, mode 0
@pytest.mark.parametrize("klen,vlen,G,P,n", [(16, 64, 2, 1, 3000), (16, 64, 8, 5, 1500), (32, 480, 3, 2, 600),
                                              (10, 7, 4, 3, 2000)])
def test_run_table_merge_in_place(klen, vlen, G, P, n):
    """k_stage's run-table path and the fixed-width emit (k_emit_fast4u for 16/64, FastUnaligned for 32/480, the
    general emit for 10/7, whose stride is no multiple of 16) over GpuSorter segments, 2 to 40 of them."""
    segs, parts = fixed_segments(klen, vlen, G, P, n, seed=klen * 100 + G)
    assert 2 <= len(segs) <= 40
    host = check_in_place(segs, 0, P=P, parts=parts, fixed=(klen, vlen))
    check_oracle(host, segs, parts, P, O.CMP_BYTES)


@pytest.mark.parametrize("writer_rle", [False, True])
def test_run_length_encoded_fixed_width_falls_back_in_place(writer_rle):
    """fixed 16/64 segments written run-length encoded: the run table meets a framing mismatch and the window parser
    takes over (mode 1); the REPEAT_KEY output equals the oracle's"""
    segs = rle_fixed_segments(4, 1200, seed=7)
    host = check_in_place(segs, 1, fixed=(16, 64), writer_rle=writer_rle)
    check_oracle(host, segs, None, 1, O.CMP_BYTES, writer_rle=writer_rle)


# ------------------------------------------------------------------------------------------------ window parser, mode 1
@pytest.mark.parametrize("check", [True, False])
def test_config3_text_merge_in_place(check):
    """config-3 shape: Text keys, segments of several 32 KiB windows; byte-exact against the oracle (values are a
    function of the word and a word occurs once per segment, so the oracle's order is pinned)"""
    segs, nrec = O.gen_c3_segments(5, 160 << 10, seed=3, threads=8, id_bits=14)
    segs = [s.tobytes() for s in segs]
    assert min(len(s) for s in segs) > 3 * WINDOW
    host = check_in_place(segs, 1, comparator=T.CMP_TEXT, check=check)
    exp, n, _ = O.merge_ifile(segs, O.CMP_TEXT, factor=100, check_for_same_keys=check)
    assert host["counts"][0] == n == sum(nrec)
    assert host["ifile"] == exp.tobytes()


@pytest.mark.parametrize("check", [True, False])
@pytest.mark.parametrize("shape", ["binary_values", "rle_runs", "long_records", "ff_bytes"])
def test_window_parser_shapes_in_place(shape, check):
    segs = window_segments(shape)
    host = check_in_place(segs, 1, comparator=T.CMP_BYTES, check=check)
    check_oracle(host, segs, None, 1, O.CMP_BYTES, check=check)


def test_in_memory_segments_in_place():
    """header-less segments: body + CRC (InMemoryWriter), and body + 4 slack bytes (fetched MEMORY segments)"""
    segs = text_segments(5, 800, seed=21)
    inmem = [s[4:] for s in segs]
    host = check_in_place(inmem, 1, comparator=T.CMP_TEXT, has_header=False)
    check_oracle(host, inmem, None, 1, O.CMP_TEXT, has_header=False)
    slack = [s[:-4] + b"\0\0\0\0" for s in inmem]
    host2 = check_in_place(slack, 1, comparator=T.CMP_TEXT, has_header=False)
    assert host2["ifile"] == host["ifile"] and host2["records"] == host["records"]


# ------------------------------------------------------------------------------------------------ checksums
def test_checksums_in_place_and_the_segment_a_mismatch_names():
    """unverified device segments have their CRC checked where they are (64 KiB pieces at odd base alignment);
    verified ones are not read for it.  A flipped bit names the segment by its index in the caller's list, not by its
    place after the partition-major reorder."""
    P = 3
    parts = [2, 0, 1, 0, 2, 1]
    segs = text_segments(len(parts), 30000, seed=5, vocab=200000)
    assert max(len(s) for s in segs) > 2 * 65536
    host = check_in_place(segs, 1, comparator=T.CMP_TEXT, P=P, parts=parts)
    check_oracle(host, segs, parts, P, O.CMP_TEXT)
    check_in_place(segs, 1, layouts=("residues",), comparator=T.CMP_TEXT, P=P, parts=parts, verified=[True] * len(segs))
    for k in (0, 4, 5):
        bad = [bytearray(s) for s in segs]
        bad[k][len(bad[k]) // 2 + 1] ^= 0x08
        for layout in LAYOUTS:
            ptrs, keep = place(bad, layout, "body")
            with pytest.raises(IOError, match="checksum mismatch in segment %d\\b" % k):
                T.GpuMerger(ptrs, device_ptrs=True, comparator=T.CMP_TEXT, partitions=parts, num_partitions=P)
            del keep


# ------------------------------------------------------------------------------------------------ combiner
def test_sum_long_combiner_in_place():
    """COMBINE_SUM_LONG over 8/8 records with duplicate keys (inside and across segments), partitions interleaved:
    write_partitions_device equals the dict-of-sums model"""
    rng = random.Random(8)
    P, gidx = 3, 0
    segs, parts, flat, fparts = [], [], [], []
    pool = [rng.randbytes(8) for _ in range(400)]
    for s in range(9):
        recs = sorted((rng.choice(pool), 0) for _ in range(700))
        recs = [(k, (gidx + j).to_bytes(8, "big")) for j, (k, _) in enumerate(recs)]
        gidx += len(recs)
        segs.append(O.write_ifile(recs, rle=False)[0])
        parts.append(s % P)
        flat += recs
        fparts += [s % P] * len(recs)
    host = check_in_place(segs, 0, P=P, parts=parts, fixed=(8, 8), combiner=T.COMBINE_SUM_LONG)
    model = CBM.model(flat, fparts, O.CMP_BYTES, CBM.SUM_LONG, P)
    got = partition_segments(host)
    for p in range(P):
        assert [(k, v) for _, k, v in O.read_ifile(got[p])] == model[p], "partition %d" % p


# ------------------------------------------------------------------------------------------------ codec mix
@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_codec_segments_mixed_with_plain_in_place(codec):
    """open_codec over unverified compressed device segments (staged, checked, decoded into an internal buffer) mixed
    with plain device segments read in place: the span then covers two allocations.  Equal to the plain merge of the
    same bodies; the compressed output equals the same merge's over host segments."""
    plain = text_segments(6, 2500, seed=40 + codec)
    segs, raws = [], []
    for i, s in enumerate(plain):
        if i % 2:
            segs.append(s)
            raws.append(0)
        else:
            z, raw = compressed(codec, s)
            segs.append(z)
            raws.append(raw)
    ref = run(plain, comparator=T.CMP_TEXT)
    host = check_in_place(segs, 1, layouts=("residues", "packed"), comparator=T.CMP_TEXT, codec=codec, raw_lens=raws)
    assert host["records"] == ref["records"] and host["counts"] == ref["counts"]
    check_oracle(ref, plain, None, 1, O.CMP_TEXT)


# ------------------------------------------------------------------------------------------------ concatenation, mode 3
@pytest.mark.parametrize("kind", ["fixed", "text"])
def test_concatenation_in_place(kind):
    if kind == "fixed":
        segs, parts = fixed_segments(16, 64, 4, 3, 800, seed=3)
        kw = dict(fixed=(16, 64))
    else:
        segs = text_segments(9, 600, seed=9)
        parts = [i % 3 for i in range(len(segs))]
        kw = {}
    host = check_in_place(segs, 3, P=3, parts=parts, concat=True, **kw)
    exp_out, exp_index = UM.concat_file(segs, parts, 3)
    assert host["file"] == exp_out
    assert [tuple(r) for r in host["index"]] == exp_index
    order = [r for p in range(3) for r in UM.records([s for s, q in zip(segs, parts) if q == p])]
    assert [(k, v) for k, v, _ in host["records"]] == order


# ------------------------------------------------------------------------------------------------ span over 4 GiB
def test_span_over_4_gib():
    """A handful of small segments in one 4 GiB + 64 MiB buffer, near offset 0, across 2^31 and past 2^32 + 4093, listed
    out of address order with partitions interleaved: every offset relative to the base (segment table, run table,
    record offsets, emit sources, checksum pieces) needs more than 32 bits.  Only the 4 KiB around each segment is
    written; no kernel may read the rest."""
    free, _ = torch.cuda.mem_get_info(0)
    if free < (6 << 30):
        pytest.skip("needs 6 GiB free on cuda:0 for a 4 GiB + 64 MiB buffer; %.1f GiB free" % (free / 2 ** 30))
    big = torch.empty((4 << 30) + (64 << 20), dtype=torch.uint8, device="cuda:0")
    # listed out of address order; segments across 2^31 and 2^32, two past 2^32 + 4093; >= 8 KiB between segments
    offsets = [(1 << 32) + 12285, GUARD + 1, (1 << 31) - 1500, (1 << 32) + 100003, (1 << 31) + 70001, (1 << 32) - 800]
    rng = np.random.default_rng(4)
    try:
        for kind in ("fixed", "text"):
            if kind == "fixed":
                segs, parts = fixed_segments(16, 64, 3, 2, 40, seed=6)
                kw, mode = dict(fixed=(16, 64)), 0
            else:
                segs = text_segments(6, 100, seed=66)
                parts = [0, 1, 0, 1, 0, 1]
                kw, mode = dict(comparator=T.CMP_TEXT), 1
            segs, parts = segs[:len(offsets)], parts[:len(offsets)]
            assert max(len(s) for s in segs) < 4096 and len(segs) >= 5
            for o, s in zip(offsets, segs):
                a, b = o - GUARD, o + len(s) + GUARD
                img = rng.integers(0, 256, b - a, dtype=np.uint8)
                img[GUARD:GUARD + len(s)] = np.frombuffer(s, dtype=np.uint8)
                big[a:b].copy_(torch.from_numpy(img))
            ptrs = [(big.data_ptr() + o, len(s)) for o, s in zip(offsets, segs)]
            host = run(segs, P=2, parts=parts, **kw)
            assert host["mode"] == mode
            check_oracle(host, segs, parts, 2, O.CMP_TEXT if kind == "text" else O.CMP_BYTES)
            dev = run(ptrs, device_ptrs=True, P=2, parts=parts, **kw)
            for key in host:
                assert dev[key] == host[key], "%s: %s differs from the host merge" % (kind, key)
    finally:
        del big
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ sequential walker
def test_sequential_walker_equals_the_window_parser():
    """TEZGPU_PARSE_SERIAL=1 sends every merge to k_parse_segments (mode 2); the switch is read once per process, so a
    subprocess runs the window-parser inputs through it, host and in place, and prints the digests of every output.
    They must equal this process's window-parser merges (mode 1), which equal the oracle."""
    env = dict(os.environ, TEZGPU_PARSE_SERIAL="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "serial-walker"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    serial = json.loads(r.stdout.strip().splitlines()[-1])
    parallel = walker_digests(1)
    assert sorted(serial) == sorted(parallel)
    for name in parallel:
        assert serial[name] == parallel[name], name + ": the sequential walker's merge differs from the window parser's"
    segs = walker_inputs()["straddle"][0]
    host = run(segs, comparator=T.CMP_BYTES)
    check_oracle(host, segs, None, 1, O.CMP_BYTES)


# ------------------------------------------------------------------------------------------------ output alignment
@pytest.mark.parametrize("combiner", [T.COMBINE_NONE, T.COMBINE_SUM_LONG])
def test_misaligned_device_output_is_refused_then_the_handle_writes(combiner):
    """tezgpu_merge_write_*_device store 16-byte words: a misaligned d_out is TEZGPU_E_INVALID before anything is
    written, and the same handle then writes the right output into an aligned buffer"""
    segs = text_segments(4, 500, seed=77, value=lambda w: zlib.crc32(w.encode()).to_bytes(8, "big"))
    ptrs, keep = place(segs, "residues", "ff")
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, combiner=combiner) as m:
        exp = m.write_ifile()[0]
    with T.GpuMerger(ptrs, device_ptrs=True, comparator=T.CMP_TEXT, combiner=combiner) as m:
        cap = m.output_bound()
        d = torch.full((cap + 64,), 0x5A, dtype=torch.uint8, device="cuda:0")
        for shift in (1, 4, 8, 15):
            with pytest.raises(TezGpuError) as e:
                m.write_ifile_device(d.data_ptr() + shift, cap)
            assert e.value.code == T.E_INVALID
            with pytest.raises(TezGpuError) as e:
                m.write_partitions_device(d.data_ptr() + shift, cap)
            assert e.value.code == T.E_INVALID
        assert bool((d == 0x5A).all()), "a refused write changed the output buffer"
        raw, part, _ = m.write_ifile_device(d.data_ptr(), cap)
        assert d[:part].cpu().numpy().tobytes() == exp
        n, index, _ = m.write_partitions_device(d.data_ptr() + 16, cap)
        assert d[16:16 + n].cpu().numpy().tobytes() == exp
    del keep


if __name__ == "__main__":
    if sys.argv[1:] == ["serial-walker"]:
        print(json.dumps(walker_digests(2)))

"""GPU: ZStandardCodec's own cases on the device (the cases every codec shares are in test_codecs_gpu.py): the
Hadoop-written fixture through the merger, a one-frame segment of several MB (one warp per segment), and zstd streams
the reader refuses."""
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
import codec_model as CM
import codec_table as CT
import lz4_model as L4
import zstd_model as M

pytestmark = pytest.mark.gpu
C = CT.CODECS["zstd"]


def test_merger_hadoop_written_fixture():
    """The fixture's segments (libzstd streams at levels 1, 3 and 19, a checksum, a one-shot frame, a 2^27 window with
    long-distance matching, a 700,000-byte value, a skippable frame between two frames): the same records and output
    as the merge over the emulator-decoded segments (compared with libzstd on the CPU)."""
    fx = M.fixture()
    segs, raws = [s for _, s, _ in fx], [r for _, _, r in fx]
    plain = [CT.plain(M.decompress_emulate(s[4:-4], r - 4)) for s, r in zip(segs, raws)]
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        exp_recs = list(m.records())
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        exp_ifile = m.write_ifile(rle=False)[0]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=C.id, raw_lens=raws) as m:
        assert list(m.records()) == exp_recs
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=C.id, raw_lens=raws) as m:
        seg, raw, part, st = m.write_ifile(rle=False)
    CT.check_merged(C, seg, raw, part, exp_ifile)
    assert st["file_out_bytes"] == part


def test_merger_one_frame_segment_of_several_mb():
    """The Java shape: one frame of many blocks without Frame_Content_Size, decoded by one warp walking it; merged with
    device-written segments."""
    plain = [O.pipelined_sort_fixed(O.sorter_conf(1), O.gen_c2(0, n, seed=s), 16, 64)["file_out"] for n, s in ((60000, 51), (3000, 52))]
    big = CM.body_of(plain[0])
    z = M.one_frame(M.compress_emulate(big))
    assert len(big) >= 4 << 20 and len(M.frames(z)) == 1 and M.frames(z)[0][2] is None and len(M.frames(z)[0][3]) >= 70
    segs = [M.segment(z), M.segment(M.compress_emulate(CM.body_of(plain[1])))]
    with T.GpuMerger(segs, comparator=T.CMP_BYTES, codec=C.id, raw_lens=[len(p) - 4 for p in plain]) as m:
        seg, raw, part, _ = m.write_ifile(rle=False)
    with T.GpuMerger(plain, comparator=T.CMP_BYTES) as m:
        CT.check_merged(C, seg, raw, part, m.write_ifile(rle=False)[0])


def test_merger_rejects_malformed_streams():
    bodies, segs, raws = CT.malformed_inputs(C)
    # the first frame's reserved bit (the frame walk sends the segment to the serial path), checksum recomputed
    z = bytearray(segs[1][4:-4])
    z[4] |= 0x08
    with pytest.raises(IOError, match="compressed segment 1: reserved bit set"):
        CT.opened(C.id, [segs[0], M.segment(bytes(z)), segs[2]], raws)
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
        CT.opened(C.id, [segs[0], segs[1], M.segment(bytes(z))], raws)
    # bytes after the last frame
    with pytest.raises(IOError, match="compressed segment 0: bytes after the last frame"):
        CT.opened(C.id, [M.segment(segs[0][4:-4] + b"\0\0\0\0")] + segs[1:], raws)
    # zlib and LZ4 streams: no frame magic
    zseg, zraw = CM.compressed_segment(bodies[0], 6)
    with pytest.raises(IOError, match="compressed segment 0: bad frame magic"):
        CT.opened(C.id, [zseg] + segs[1:], [zraw] + raws[1:])
    with pytest.raises(IOError, match="compressed segment 1: bad frame magic"):
        CT.opened(C.id, [segs[0], L4.segment(L4.compress_emulate(bodies[1])), segs[2]], raws)

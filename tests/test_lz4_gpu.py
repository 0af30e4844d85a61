"""GPU: Lz4Codec's own cases on the device (the cases every codec shares are in test_codecs_gpu.py): the Java-framed
fixture through the merger, and LZ4 streams the reader refuses."""
import pytest

import tez_b200 as T
import codec_table as CT
import lz4_model as M

pytestmark = pytest.mark.gpu
C = CT.CODECS["lz4"]


def test_merger_java_framed_fixture():
    """The fixture's segments (Java block cutting, liblz4 chunks at acceleration 1 and 8 and HC, a block of several
    chunks): the same records and output as the merge over the model-decoded segments."""
    fx = M.fixture()
    segs, raws = [s for _, s, _ in fx], [r for _, _, r in fx]
    plain = [CT.plain(M.decode_stream(s[4:-4], r - 4)) for s, r in zip(segs, raws)]
    with T.GpuMerger(plain, comparator=T.CMP_TEXT) as m:
        exp_recs = list(m.records())
    with T.GpuMerger(plain, comparator=T.CMP_TEXT) as m:
        exp_ifile = m.write_ifile(rle=False)[0]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=C.id, raw_lens=raws) as m:
        assert list(m.records()) == exp_recs
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=C.id, raw_lens=raws) as m:
        seg, raw, part, st = m.write_ifile(rle=False)
    CT.check_merged(C, seg, raw, part, exp_ifile)
    assert st["file_out_bytes"] == part


def test_merger_rejects_malformed_streams():
    _, segs, raws = CT.malformed_inputs(C)
    # the first block's raw length one short of what its chunk decodes to, checksum recomputed
    z = bytearray(segs[1][4:-4])
    z[0:4] = (int.from_bytes(z[0:4], "big") - 1).to_bytes(4, "big")
    with pytest.raises(IOError, match="compressed segment 1: chunks decode past"):
        CT.opened(C.id, [segs[0], M.segment(bytes(z)), segs[2]], raws)
    # bytes after the last block
    with pytest.raises(IOError, match="compressed segment 0: bytes after the last block"):
        CT.opened(C.id, [M.segment(segs[0][4:-4] + b"\0\0\0\0")] + segs[1:], raws)

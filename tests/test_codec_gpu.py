"""GPU: DefaultCodec's own cases on the device (the cases every codec shares are in test_codecs_gpu.py): the reference's
compressed fixture through the merger, and a zlib stream the inflate refuses."""
import zlib

import pytest

from oracle import tez_oracle as O
import tez_b200 as T
import codec_model as M
import codec_table as CT

pytestmark = pytest.mark.gpu
C = CT.CODECS["default"]


def test_merger_fixture_segments():
    """The reference's five compressed segments (written by the real IFile.Writer; their keys are not in comparator
    order, so the expectation is the same merge over the decompressed segments, and the oracle's records)."""
    segs, raws = zip(*M.fixture())
    plain = [CT.plain(zlib.decompress(s[4:-4])) for s in segs]
    oracle = sorted((k, v) for p in plain for _, k, v in O.read_ifile(p))
    with T.GpuMerger(plain, comparator=T.CMP_TEXT) as m:
        exp_recs = list(m.records())
    with T.GpuMerger(plain, comparator=T.CMP_TEXT) as m:
        exp_ifile = m.write_ifile(rle=False)[0]
    with T.GpuMerger(list(segs), comparator=T.CMP_TEXT, codec=C.id, raw_lens=list(raws)) as m:
        got = list(m.records())
    assert got == exp_recs
    assert sorted((k, v) for k, v, _ in got) == oracle
    with T.GpuMerger(list(segs), comparator=T.CMP_TEXT, codec=C.id, raw_lens=list(raws)) as m:
        seg, raw, part, st = m.write_ifile(rle=False)
    CT.check_merged(C, seg, raw, part, exp_ifile)
    assert st["file_out_bytes"] == part


def test_merger_rejects_malformed_streams():
    """a flipped bit in the stream, checksum recomputed: the inflate fails"""
    _, segs, raws = CT.malformed_inputs(C)
    z = bytearray(segs[1][4:-4])
    z[len(z) // 2] ^= 0x10
    with pytest.raises(IOError, match="compressed segment 1"):
        CT.opened(C.id, [segs[0], M.segment(bytes(z)), segs[2]], raws)

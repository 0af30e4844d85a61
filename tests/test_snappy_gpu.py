"""GPU: SnappyCodec's own cases on the device (the cases every codec shares are in test_codecs_gpu.py): the
Java-framed fixture (multi-chunk blocks included) through merge_open_codec, concat_open and next_batch_device,
sort_device of variable-length records, decode_segments in one group and several, Snappy streams the reader refuses,
and hand-made chunks and a mutant corpus on the 32-lane paths."""
import zlib

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import native
from tez_b200._lib import TezGpuError
import codec_table as CT
import combine_model as CBM
import snappy_model as M

pytestmark = pytest.mark.gpu
C = CT.CODECS["snappy"]
Z = C.id


# ------------------------------------------------------------------------------------------------ sorter
@pytest.mark.parametrize("unordered", [False, True])
def test_sorter_sort_device_variable_length(unordered):
    recs = CT.records(O.CMP_TEXT, 40000, seed=31) + [(O.text("big"), bytes(range(256)) * 300)]
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
    CT.check_file(C, out, index, exp["file_out"], exp["index"])


# ------------------------------------------------------------------------------------------------ merger
def _fixture():
    """the Java-framed segments of the fixture (its crafted segments decode to bytes that are not records)"""
    fx = [f for f in M.fixture() if not f[0].startswith("crafted_")]
    return [s for _, s, _ in fx], [r for _, _, r in fx]


def test_merger_java_framed_fixture_merge_and_concat():
    """The fixture's segments (Java block cutting, libsnappy chunks, a block of several chunks, hand-made chunks)
    merge and concatenate to what the model-decoded segments give."""
    segs, raws = _fixture()
    plain = [CT.plain(M.decode_stream(s[4:-4], r - 4)) for s, r in zip(segs, raws)]
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
        CT.check_merged(C, seg, raw, part, exp_ifile)
        assert st["file_out_bytes"] == part


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


@pytest.mark.parametrize("budget", [1 << 30, 16 << 20])
def test_decode_segments_one_group_and_several(budget):
    fx = M.fixture() * (1 if budget > 1 << 29 else 6)
    plain = CT.c3(2, seed=8)
    segs, raws = [s for _, s, _ in fx] + plain, [r for _, _, r in fx] + [0, 0]
    imgs, peak = native.decode_segments(segs, raws, Z, budget)
    for s, r, img in zip(segs, raws, imgs):
        if r == 0:
            assert img is None
            continue
        body = M.decode_stream(s[4:-4], r - 4)
        assert img == b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")
    assert 0 < peak <= budget


def test_merger_rejects_malformed_streams():
    _, segs, raws = CT.malformed_inputs(C)
    z = bytearray(segs[1][4:-4])
    z[0:4] = (int.from_bytes(z[0:4], "big") - 1).to_bytes(4, "big")
    with pytest.raises(IOError, match="compressed segment 1: chunks decode past"):
        CT.opened(Z, [segs[0], M.segment(bytes(z)), segs[2]], raws)
    with pytest.raises(IOError, match="compressed segment 0: bytes after the last block"):
        CT.opened(Z, [M.segment(segs[0][4:-4] + b"\0\0\0\0")] + segs[1:], raws)


# ------------------------------------------------------------------------------------------------ 32-lane paths
def _cases():
    """(name, stream, expect): the hand-made chunks alone, as one block of several, and the CPU suite's malformed
    streams"""
    cr = M.crafted_chunks()
    res = [("crafted_" + n, M.one_block([c]), M.preamble(c)[0]) for n, c in cr]
    res.append(("crafted_all_in_one_block", M.one_block([c for _, c in cr]), sum(M.preamble(c)[0] for _, c in cr)))
    res += [("malformed_" + k, z, e) for k, (z, e, _) in sorted(M.malformed().items())]
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
    muts = M.mutants(M.corpus_streams(), 3000, seed=4321)
    cases = [("mutant_%d" % i, z, e) for i, (z, e) in enumerate(muts) if e >= 2 and len(z) >= 2]
    if order == "reversed":
        cases = cases[::-1]
    # the good ones in one call; every bad one alone (its reason)
    good, bad = _decode_all(cases)
    assert good > 100 and bad > 300

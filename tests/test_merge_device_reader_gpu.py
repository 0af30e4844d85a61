"""GPU: tezgpu_merge_next_batch_device, the record iterator whose batches stay in device memory.

Every read is checked against tezgpu_merge_next_batch on a second handle over the same inputs, batch for batch: the
same record bytes, record boundaries and isSameKey flags, at the same caps.  Each device batch must start its table at
0 with records back to back, and the poisoned bytes after kv_bytes and after the table's last entry must come back
untouched.  The routes are the seeded scenarios of tests/merge_scenarios.py (five comparators, both framings,
run-length encoded inputs, checkForSameKeys 0 and 1, P > 1, host and device segments), concatenations, the three
codecs and a bounded merge that takes several steps.  Then the batch edges, the refusals, one batch past 4 GiB, and
OrderedWordCount's two ordered edges run on the device from sort to reducer."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import _lib, synth
from tez_b200._lib import KvIndex, TezGpuError

import merge_scenarios as MS
from merge_model import place, stable_model
from test_merge_in_place_gpu import compressed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
POISON = 0xA5
GUARD = 4096
FLOOR = 16 << 20                                   # TEZGPU_MERGE_BUDGET_MIN
ROUTE_SEEDS = tuple(range(0, 100, 3))              # every comparator and axis value (test_merge_device_reader_cpu)
SHAPES = ((997, 1 << 17), (1 << 14, 1 << 22))      # (idx_cap, kv_cap): above the 65,536-byte Text keys


# ------------------------------------------------------------------------------------------------ readers
def host_batch(m, idx_cap, cap):
    """one tezgpu_merge_next_batch: (bytes, [(key_off, key_len, val_off, val_len, same_key)])"""
    buf = np.empty(max(1, cap), dtype=np.uint8)
    idx = (KvIndex * max(1, idx_cap))()
    n = C.c_uint32()
    _lib.check(m.L.tezgpu_merge_next_batch(m.h, buf.ctypes.data, cap, idx, idx_cap, C.byref(n)))
    ents = [(e.key_off, e.key_len, e.val_off, e.val_len, e.same_key) for e in idx[:n.value]]
    end = ents[-1][2] + ents[-1][3] if ents else 0
    return buf[:end].tobytes(), ents


class DevBufs:
    """kv and table buffers with poisoned guards after their capacities"""

    def __init__(self, kv_cap, idx_cap):
        self.kv_cap, self.idx_cap = kv_cap, idx_cap
        self.kv = torch.full((kv_cap + GUARD,), POISON, dtype=torch.uint8, device=DEV)
        self.ko = torch.full((idx_cap + GUARD // 8,), -7, dtype=torch.int64, device=DEV)
        self.vo = torch.full((idx_cap + GUARD // 8,), -7, dtype=torch.int64, device=DEV)
        self.vl = torch.full((idx_cap + GUARD // 4,), -7, dtype=torch.int32, device=DEV)
        self.sk = torch.full((idx_cap + GUARD,), POISON, dtype=torch.uint8, device=DEV)

    def poison(self):
        self.kv.fill_(POISON)
        for t in (self.ko, self.vo, self.vl):
            t.fill_(-7)
        self.sk.fill_(POISON)

    def untouched_from(self, b, n):
        return (bool((self.kv[b:] == POISON).all()) and bool((self.ko[n:] == -7).all()) and bool((self.vo[n:] == -7).all())
                and bool((self.vl[n:] == -7).all()) and bool((self.sk[n:] == POISON).all()))

    def read(self, m, idx_cap=None, kv_cap=None, kv_ptr=None, same=True):
        torch.cuda.synchronize()   # the poison fills run on torch's stream, the batch on the merger's
        return m.next_batch_device(self.kv.data_ptr() if kv_ptr is None else kv_ptr,
                                   self.kv_cap if kv_cap is None else kv_cap, self.ko.data_ptr(), self.vo.data_ptr(),
                                   self.vl.data_ptr(), self.sk.data_ptr() if same else None,
                                   self.idx_cap if idx_cap is None else idx_cap)


def dev_batch(m, bufs, idx_cap=None, kv_cap=None):
    """one next_batch_device, checked for its table invariants and its guards: host_batch's shape"""
    bufs.poison()
    n, b = bufs.read(m, idx_cap, kv_cap)
    assert bufs.untouched_from(b, n), "bytes written past kv_bytes or past the table"
    if n == 0:
        assert b == 0
        return b"", []
    ko, vo = bufs.ko[:n].cpu().numpy(), bufs.vo[:n].cpu().numpy()
    vl, sk = bufs.vl[:n].cpu().numpy().astype(np.int64), bufs.sk[:n].cpu().numpy()
    assert ko[0] == 0 and np.array_equal(ko[1:], vo[:-1] + vl[:-1]) and vo[-1] + vl[-1] == b, "records not back to back"
    assert np.all(vo >= ko) and set(np.unique(sk).tolist()) <= {0, 1}
    ents = [(int(a), int(c - a), int(c), int(d), int(s)) for a, c, d, s in zip(ko, vo, vl, sk)]
    return bufs.kv[:b].cpu().numpy().tobytes(), ents


def read_all(m, idx_cap, cap, device):
    bufs = DevBufs(cap, idx_cap) if device else None
    out = []
    while True:
        batch = dev_batch(m, bufs) if device else host_batch(m, idx_cap, cap)
        if not batch[1]:
            return out
        out.append(batch)


def records_of(batches):
    return [(b[ko:ko + kl], b[vo:vo + vl], bool(s)) for b, ents in batches for ko, kl, vo, vl, s in ents]


def same_stream(open_merger, shapes=SHAPES, check=None):
    """the device batches equal the host batches at every shape; returns the records"""
    recs = None
    for idx_cap, cap in shapes:
        got = []
        for device in (False, True):
            with open_merger() as m:
                if check is not None and not check:
                    m.set_check_for_same_keys(False)
                got.append(read_all(m, idx_cap, cap, device))
        assert len(got[0]) == len(got[1]), "batch counts differ at %r" % ((idx_cap, cap),)
        for i, (h, d) in enumerate(zip(*got)):
            assert d[1] == h[1], "batch %d: record boundaries or isSameKey differ at %r" % (i, (idx_cap, cap))
            assert d[0] == h[0], "batch %d: bytes differ at %r" % (i, (idx_cap, cap))
        r = records_of(got[1])
        assert recs is None or r == recs
        recs = r
    return recs


# ------------------------------------------------------------------------------------------------ 1. every route
@pytest.mark.parametrize("seed", ROUTE_SEEDS, ids=MS.scenario_id)
def test_routes_equal_the_host_iterator(seed):
    sc = MS.scenario(seed)
    kw = MS.merge_kwargs(sc)
    model = [r for p in stable_model(sc["segs"], sc["parts"], sc["P"], sc["cmp"], sc["has_header"], sc["check"]) for r in p]
    recs = same_stream(lambda: T.GpuMerger(sc["segs"], fixed=sc["fixed"], **kw), check=sc["check"])
    assert recs == model, "records or isSameKey flags differ from the stable merge"
    ptrs, keep = place(sc["segs"], "residues", "body", seed=seed)
    assert same_stream(lambda: T.GpuMerger(ptrs, device_ptrs=True, **kw), SHAPES[:1], check=sc["check"]) == model
    del keep


def _text_segments(nseg, n, seed):
    rng = random.Random(seed)
    segs, gidx = [], 0
    for _ in range(nseg):
        words = sorted({O.text(b"w%d" % rng.randrange(4 * n)) for _ in range(rng.randint(1, n))}, key=lambda w: w[1:])
        recs = [(w, (gidx + j).to_bytes(4, "big") + b"v" * (j % 23)) for j, w in enumerate(words)]
        gidx += len(recs)
        segs.append(O.write_ifile(recs, rle=False)[0])
    return segs


def test_concatenation():
    segs = _text_segments(9, 800, seed=1)
    parts = [i % 3 for i in range(len(segs))]
    recs = same_stream(lambda: T.GpuMerger(segs, partitions=parts, num_partitions=3, concat=True))
    with T.GpuMerger(segs, partitions=parts, num_partitions=3, concat=True) as m:
        assert recs == list(m.records())


@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_codecs_host_and_device_segments(codec):
    plain = _text_segments(6, 1500, seed=codec)
    segs, raws = [], []
    for i, s in enumerate(plain):
        z, r = compressed(codec, s) if i % 2 == 0 else (s, len(s) - 4)
        segs.append(z)
        raws.append(r)
    model = [r for p in stable_model(plain, None, 1, O.CMP_TEXT) for r in p]
    assert same_stream(lambda: T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=codec, raw_lens=raws)) == model
    # device-resident compressed segments: checksums verified and streams decoded in place
    ptrs, keep = place(segs, "residues", "body", seed=codec)
    assert same_stream(lambda: T.GpuMerger(ptrs, device_ptrs=True, comparator=T.CMP_TEXT, codec=codec, raw_lens=raws),
                       SHAPES[:1]) == model
    del keep
    assert same_stream(lambda: T.GpuMerger(segs, concat=True, codec=codec, raw_lens=raws), SHAPES[:1]) == \
        [(k, v, False) for s in plain for _, k, v in O.read_ifile(s)]


def test_bounded_merge_in_several_steps():
    seed = next(s for s in MS.SEEDS if MS.shape(s)["large"] and not MS.shape(s)["fixed"])
    sc = MS.scenario(seed)
    kw = MS.merge_kwargs(sc)
    with T.GpuMerger(sc["segs"], device_budget=FLOOR, **kw) as m:
        assert len(records_of(read_all(m, 4093, 1 << 20, True))) == sc["nrec"]
        assert m.bounded_info()[0] > 1, "the floor budget took one step"
    model = [r for p in stable_model(sc["segs"], sc["parts"], sc["P"], sc["cmp"], sc["has_header"], sc["check"]) for r in p]
    assert same_stream(lambda: T.GpuMerger(sc["segs"], device_budget=FLOOR, **kw), ((4093, 1 << 20),),
                       check=sc["check"]) == model


def test_long_records_among_short_ones():
    """Batches of short records size their lane groups at one or two lanes, which then copy a few long records (up to
    1,100 bytes longer than the rest) on their own: every length near 256 and 512 bytes, at every source alignment,
    among 3,000 short records."""
    rng = random.Random(17)
    segs, gidx = [], 0
    for s in range(3):
        keys = sorted({rng.randbytes(rng.randint(1, 6)) for _ in range(1000)})
        recs = []
        for j, k in enumerate(keys):
            extra = rng.choice((0,) * 400 + tuple(range(248, 258)) + tuple(range(504, 514)) + (1100,))
            recs.append((k, gidx.to_bytes(4, "big") + bytes((gidx + t) & 0xFF for t in range(extra + j % 16))))
            gidx += 1
        segs.append(O.write_ifile(recs)[0])
    model = [r for p in stable_model(segs, None, 1, O.CMP_BYTES) for r in p]
    assert same_stream(lambda: T.GpuMerger(segs), ((1 << 14, 1 << 22), (301, 1 << 17))) == model


# ------------------------------------------------------------------------------------------------ records_device
def test_records_device_with_an_asynchronous_consumer():
    """Each batch is read by torch work that is still queued behind a long kernel when the next batch is asked for; the
    generator must not overwrite the views under it.  A record larger than batch_bytes makes the buffer grow."""
    segs = _text_segments(5, 2000, seed=23)
    segs.append(O.write_ifile([(O.text(b"w~big"), b"B" * 70000)])[0])
    with T.GpuMerger(segs, comparator=T.CMP_TEXT) as m:
        want = list(m.records())
    assert max(len(k) + len(v) for k, v, _ in want) > 1 << 16
    copies = []
    with T.GpuMerger(segs, comparator=T.CMP_TEXT) as m:
        for kv, ko, vo, vl, sk in m.records_device(batch_records=211, batch_bytes=1 << 16):
            torch.cuda._sleep(20_000_000)   # the consumer's stream is busy well past the next call
            copies.append((kv.clone(), ko.clone(), vo.clone(), vl.clone(), sk.clone()))
    torch.cuda.synchronize()
    got = []
    for kv, ko, vo, vl, sk in copies:
        b = kv.cpu().numpy().tobytes()
        got += [(b[a:c], b[c:c + d], bool(s)) for a, c, d, s in zip(ko.tolist(), vo.tolist(), vl.tolist(), sk.tolist())]
    assert len(copies) > 20 and got == want


# ------------------------------------------------------------------------------------------------ 2. batch edges
def _small():
    return _text_segments(4, 300, seed=5)


def _open():
    return T.GpuMerger(_small(), comparator=T.CMP_TEXT)


def _all_records():
    with _open() as m:
        return records_of(read_all(m, 1 << 16, 1 << 22, False))


def test_kv_cap_at_and_below_a_batch():
    recs = _all_records()
    k = 37
    exact = sum(len(key) + len(v) for key, v, _ in recs[:k])
    bufs = DevBufs(1 << 20, 1 << 12)
    for cap, want in ((exact, k), (exact - 1, k - 1)):
        with _open() as m:
            _, ents = dev_batch(m, bufs, kv_cap=cap)
            assert len(ents) == want and ents[-1][2] + ents[-1][3] == sum(len(a) + len(b) for a, b, _ in recs[:want])
    with _open() as m:
        first = len(recs[0][0]) + len(recs[0][1])
        bufs.poison()
        with pytest.raises(TezGpuError) as e:
            bufs.read(m, kv_cap=first - 1)
        assert e.value.code == T.E_NOMEM and e.value.needed == first
        assert bufs.untouched_from(0, 0), "a refused batch wrote"
        assert records_of(read_all(m, 1 << 12, 1 << 20, True)) == recs, "the cursor moved"


def test_one_record_per_batch_and_the_end():
    recs = _all_records()
    with _open() as m:
        got = read_all(m, 1, 1 << 20, True)
        assert all(len(ents) == 1 for _, ents in got) and records_of(got) == recs
        bufs = DevBufs(1 << 10, 4)
        for _ in range(2):
            assert bufs.read(m) == (0, 0)


def test_interleaved_with_the_host_iterator():
    recs = _all_records()
    bufs = DevBufs(1 << 12, 50)
    with _open() as m:
        got, i = [], 0
        while True:
            b = dev_batch(m, bufs) if i % 2 else host_batch(m, 50 + i % 7, 1 << 12)
            if not b[1]:
                break
            got.append(b)
            i += 1
    assert i > 4 and records_of(got) == recs


# ------------------------------------------------------------------------------------------------ 3. refusals
def test_refusals_write_nothing():
    recs = _all_records()
    bufs = DevBufs(1 << 20, 1 << 12)
    with _open() as m:
        for ptr in (bufs.kv.data_ptr() + 1, bufs.kv.data_ptr() + 8):
            bufs.poison()
            with pytest.raises(TezGpuError, match="16-byte aligned") as e:
                bufs.read(m, kv_ptr=ptr)
            assert e.value.code == T.E_INVALID and bufs.untouched_from(0, 0)
        n, b = C.c_uint32(7), C.c_uint64(7)
        assert m.L.tezgpu_merge_next_batch_device(m.h, bufs.kv.data_ptr(), 1 << 20, None, bufs.vo.data_ptr(), bufs.vl.data_ptr(),
                                                  None, 100, C.byref(n), C.byref(b)) == T.E_INVALID
        assert n.value == 0 and b.value == 0 and bufs.untouched_from(0, 0)
        assert records_of(read_all(m, 1 << 12, 1 << 20, True)) == recs
    segs = [O.write_ifile([(O.text(b"k%d" % i), O.int_writable(i)) for i in range(50)])[0]]
    with T.GpuMerger(segs, comparator=T.CMP_TEXT, combiner=T.COMBINE_SUM_INT) as m:
        bufs.poison()
        with pytest.raises(TezGpuError, match="combiner") as e:
            bufs.read(m)
        assert e.value.code == T.E_STATE and bufs.untouched_from(0, 0)


# ------------------------------------------------------------------------------------------------ 4. past 4 GiB
VLEN = 1 << 20

@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.mem_get_info(0)[0] < (13 << 30),
                    reason="needs 13 GiB of free device memory")
def test_one_batch_past_4_gib():
    """4,160 records of 1 MiB values in three header-less segments built on the device: one batch of 4.36e9 bytes.
    Keys are unique, so the oracle's merge of the same keys with short values fixes every record's position."""
    nrec, nseg = 4160, 3
    rng = random.Random(71)
    keys = rng.sample(range(1 << 32), nrec)
    seg_of = [rng.randrange(nseg) for _ in range(nrec)]
    pattern = torch.arange(VLEN + 256, device=DEV, dtype=torch.int64).remainder(251).to(torch.uint8)
    segs_dev, small = [], []
    for s in range(nseg):
        mine = sorted((keys[r].to_bytes(4, "big"), r) for r in range(nrec) if seg_of[r] == s)
        hdr = [O.vint(4) + O.vint(VLEN) + k for k, _ in mine]
        size = sum(len(h) + VLEN for h in hdr) + 2 + 4
        d = torch.empty(size, dtype=torch.uint8, device=DEV)
        at = 0
        for h, (_, r) in zip(hdr, mine):
            d[at:at + len(h)] = torch.frombuffer(bytearray(h), dtype=torch.uint8).to(DEV)
            at += len(h)
            d[at:at + VLEN] = pattern[r % 251:r % 251 + VLEN]
            at += VLEN
        d[at:] = torch.tensor([0xFF, 0xFF, 0, 0, 0, 0], dtype=torch.uint8, device=DEV)
        segs_dev.append(d)
        small.append(O.write_ifile([(k, r.to_bytes(4, "big")) for k, r in mine])[0])
    order = [int.from_bytes(v, "big") for _, v, _ in O.merge(small, O.CMP_BYTES, factor=100)["records"]]
    total = nrec * (4 + VLEN)
    assert total > 1 << 32
    kv = torch.empty(total, dtype=torch.uint8, device=DEV)
    ko, vo = torch.empty(nrec, dtype=torch.int64, device=DEV), torch.empty(nrec, dtype=torch.int64, device=DEV)
    vl, sk = torch.empty(nrec, dtype=torch.int32, device=DEV), torch.empty(nrec, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()   # the segments are written on torch's stream
    with T.GpuMerger([(d.data_ptr(), d.numel()) for d in segs_dev], device_ptrs=True, has_header=False) as m:
        n, b = m.next_batch_device(kv.data_ptr(), total, ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), sk.data_ptr(), nrec)
        assert (n, b) == (nrec, total)
        assert m.next_batch_device(kv.data_ptr(), total, ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), None, nrec) == (0, 0)
    del segs_dev
    ko_h, vo_h = ko.cpu().numpy(), vo.cpu().numpy()
    assert np.array_equal(ko_h, np.arange(nrec, dtype=np.int64) * (4 + VLEN)) and bool((vl == VLEN).all())
    assert np.array_equal(vo_h, ko_h + 4) and not bool(sk.any()) and ko_h[-1] > 1 << 32
    for i in sorted(set(random.Random(73).sample(range(nrec), 40)) | {nrec - 1}):
        r = order[i]
        rec = kv[int(ko_h[i]):int(vo_h[i]) + VLEN]
        assert rec[:4].cpu().numpy().tobytes() == keys[r].to_bytes(4, "big"), "record %d: key" % i
        assert torch.equal(rec[4:], pattern[r % 251:r % 251 + VLEN]), "record %d: value" % i


# ------------------------------------------------------------------------------------------------ 5. OrderedWordCount
def _sort_on_device(P, cmp, kv, kv_bytes, ko, vo, vl, n, rle):
    with T.GpuSorter(P, comparator=cmp, rle_policy=rle) as s:
        cap = s.device_output_bound(n, kv_bytes)
        out = torch.empty(cap + 16, dtype=torch.uint8, device=DEV)
        torch.cuda.synchronize()   # the inputs come from torch's stream, the sort runs on the sorter's
        ln, index, _ = s.sort_device(kv.data_ptr(), kv_bytes, ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), n,
                                     out.data_ptr(), cap)
    return out, ln, index


def _merge_on_device(outs, cmp):
    """one merge over partition 0 of each device file.out, read as one device batch"""
    segs = [(out.data_ptr() + int(index[0][0]), int(index[0][2])) for out, _, index in outs]
    with T.GpuMerger(segs, device_ptrs=True, comparator=cmp) as m:
        total = m.counts()
        kv = torch.empty(total[1] + 16, dtype=torch.uint8, device=DEV)
        ko, vo = torch.empty(total[0], dtype=torch.int64, device=DEV), torch.empty(total[0], dtype=torch.int64, device=DEV)
        vl, sk = torch.empty(total[0], dtype=torch.int32, device=DEV), torch.empty(total[0], dtype=torch.uint8, device=DEV)
        torch.cuda.synchronize()
        n, b = m.next_batch_device(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), sk.data_ptr(),
                                   total[0])
        assert (n, b) == total
    return kv, ko, vo, vl, sk, n, b


def _be32(kv, off):
    """the big-endian int32 at every offset"""
    x = torch.zeros(off.numel(), dtype=torch.int64, device=DEV)
    for j in range(4):
        x = x * 256 + kv[off + j].to(torch.int64)
    return torch.where(x >= 1 << 31, x - (1 << 32), x)


def _host_records(kv, ko, vo, vl):
    b = kv.cpu().numpy().tobytes()
    return [(b[a:c], b[c:c + d]) for a, c, d in zip(ko.tolist(), vo.tolist(), vl.tolist())]


def test_ordered_word_count_two_edges_on_the_device():
    n, vocab = 120000, 3000
    maps = [synth.gen_words(i * n, n, seed=11, vocab=vocab, device=DEV) for i in range(2)]
    # edge 1: each map's words sorted on the device, the two outputs merged and read on the device
    outs = [_sort_on_device(1, T.CMP_TEXT, kv, kv.numel(), ko, vo, vl, n, T.RLE_ON) for kv, ko, vo, vl in maps]
    kv, ko, vo, vl, sk, m1, b1 = _merge_on_device(outs, T.CMP_TEXT)
    # reducer: a segment sum over the isSameKey runs
    first = sk == 0
    gid = torch.cumsum(first.to(torch.int64), 0) - 1
    counts = torch.zeros(int(first.sum()), dtype=torch.int64, device=DEV).index_add_(0, gid, _be32(kv, vo))
    wko, wvo = ko[first], vo[first]
    wlen = wvo - wko
    # edge 2: (IntWritable count, Text word) records built in device memory
    rlen = 4 + wlen
    ko2 = torch.cumsum(rlen, 0) - rlen
    kv2 = torch.empty(int(rlen.sum()) + 16, dtype=torch.uint8, device=DEV)
    for j in range(4):
        kv2[ko2 + j] = ((counts >> (24 - 8 * j)) & 0xFF).to(torch.uint8)
    rep = torch.repeat_interleave(torch.arange(wlen.numel(), device=DEV), wlen)
    pos = torch.arange(rep.numel(), device=DEV) - (torch.cumsum(wlen, 0) - wlen)[rep]
    kv2[ko2[rep] + 4 + pos] = kv[wko[rep] + pos]
    nw = counts.numel()
    out2 = _sort_on_device(1, T.CMP_INT, kv2, int(rlen.sum()), ko2, ko2 + 4, wlen.to(torch.int32), nw, T.RLE_OFF)
    kv3, ko3, vo3, vl3, _, m2, _ = _merge_on_device([out2], T.CMP_INT)
    got = _host_records(kv3, ko3, vo3, vl3)

    # the oracle's two edges on the same records rebuilt on the CPU
    segs = []
    for kvh, koh, voh, vlh in maps:
        kvh, koh, voh = kvh.cpu().numpy(), koh.cpu().numpy().astype(np.uint64), voh.cpu().numpy().astype(np.uint64)
        conf = O.sorter_conf(1, cmp_kind=O.CMP_TEXT, rle_policy=1)
        segs.append(O.pipelined_sort(conf, kvh, koh, (voh - koh).astype(np.uint32), vlh.cpu().numpy().astype(np.uint32))["file_out"])
    exp1 = O.merge(segs, O.CMP_TEXT, factor=100)["records"]
    got1 = [(k, v, s) for (k, v), s in zip(_host_records(kv, ko, vo, vl), sk.cpu().tolist())]
    assert got1 == [(k, v, int(s)) for k, v, s in exp1], "edge 1: the merged stream differs from the oracle's"
    words = {}
    for k, v, _ in exp1:
        words[k] = words.get(k, 0) + int.from_bytes(v, "big", signed=True)
    assert [k for k, _ in _host_records(kv, wko, wvo, torch.zeros_like(wlen))] == list(words)
    assert counts.cpu().tolist() == list(words.values()) and sum(words.values()) == 2 * n
    recs2 = [(O.int_writable(c), w) for w, c in words.items()]
    kvx = np.frombuffer(b"".join(k + v for k, v in recs2), dtype=np.uint8)
    kl2 = np.full(len(recs2), 4, np.uint32)
    vl2 = np.array([len(v) for _, v in recs2], dtype=np.uint32)
    ko_x = np.zeros(len(recs2), np.uint64)
    ko_x[1:] = np.cumsum(kl2.astype(np.uint64) + vl2)[:-1]
    seg2 = O.pipelined_sort(O.sorter_conf(1, cmp_kind=O.CMP_INT, rle_policy=0), kvx, ko_x, kl2, vl2)["file_out"]
    exp2 = O.merge([seg2], O.CMP_INT, factor=100)["records"]

    def canon(recs):   # words of equal count: their order is the sort's tie order, which the contract leaves open
        out = {}
        for k, v in recs:
            out.setdefault(k, []).append(v)
        return [(k, sorted(v)) for k, v in out.items()]
    assert [k for k, _ in got] == [k for k, _, _ in exp2] and canon(got) == canon([(k, v) for k, v, _ in exp2])
    assert m2 == len(words)

    # a merged batch's table straight into sort_device: file.out equals the oracle's for the same records
    P = 8
    out, ln, index = _sort_on_device(P, T.CMP_TEXT, kv, b1, ko, vo, vl, m1, T.RLE_AUTO)
    recs1 = _host_records(kv, ko, vo, vl)
    kvy = np.frombuffer(b"".join(k + v for k, v in recs1), dtype=np.uint8)
    kly = np.array([len(k) for k, _ in recs1], np.uint32)
    vly = np.array([len(v) for _, v in recs1], np.uint32)
    koy = np.zeros(len(recs1), np.uint64)
    koy[1:] = np.cumsum(kly.astype(np.uint64) + vly)[:-1]
    e = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT), kvy, koy, kly, vly)
    assert out[:ln].cpu().numpy().tobytes() == e["file_out"] and np.array_equal(index, e["index"])

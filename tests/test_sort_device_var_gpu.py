"""GPU: tezgpu_sorter_sort_device, the one-call sort of variable-length records that are already in device memory.

Every case runs the same records twice: through the host path (collect_batch + flush_to_memory, records packed in
collection order) and through sort_device (records anywhere in a device buffer, 64-bit offsets).  file.out and the index
must be byte-identical; uncompressed cases are also checked against the CPU oracle (pipelined_sort / unordered_write,
with the combiner model for combined cases).  The refusals are argument checks: the validating kernel rejects the
records before any byte outside them is read, d_out keeps its sentinel and the handle serves the next call."""
import random
import zlib

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import synth
from tez_b200._lib import TezGpuError

import combine_model as CM
import total_order_model as TO
from test_record_sizes_gpu import fill, serialize, size_mix

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 0xA5


def _pack(recs):
    """[(key, value)] in collection order -> host kv, key_off u64, key_len u32, val_len u32 (back to back)"""
    kl = np.array([len(k) for k, _ in recs], dtype=np.uint64)
    vl = np.array([len(v) for _, v in recs], dtype=np.uint64)
    ko = np.zeros(len(recs), dtype=np.uint64)
    if len(recs):
        ko[1:] = np.cumsum(kl + vl)[:-1]
    kv = np.frombuffer(b"".join(k + v for k, v in recs), dtype=np.uint8) if recs else np.zeros(0, np.uint8)
    return kv, ko, kl.astype(np.uint32), vl.astype(np.uint32)


def _scatter(recs, seed, gap=24, lead=48):
    """The records in a shuffled placement with gaps of 0..gap filler bytes between them: (host buffer, key_off u64,
    val_off u64, val_len u32) indexed by collection order"""
    rng = random.Random(seed)
    order = list(range(len(recs)))
    rng.shuffle(order)
    parts, ko, vo = [rng.randbytes(lead)], np.zeros(len(recs), np.uint64), np.zeros(len(recs), np.uint64)
    at = lead
    for i in order:
        k, v = recs[i]
        ko[i], vo[i] = at, at + len(k)
        parts.append(k + v)
        g = rng.randint(0, gap)
        parts.append(rng.randbytes(g))
        at += len(k) + len(v) + g
    vl = np.array([len(v) for _, v in recs], dtype=np.uint32)
    return np.frombuffer(b"".join(parts), dtype=np.uint8), ko, vo, vl


def _dev(a, dtype=None):
    return torch.from_numpy(np.array(a, dtype=dtype)).to(DEV)


def _sorter_kw(P, cmp, part, rle=T.RLE_AUTO, combiner=0, codec=0, unordered=False, splits=None):
    kw = dict(comparator=cmp, partitioner=part, rle_policy=rle, combiner=combiner, codec=codec, unordered=unordered)
    if part == T.PART_TOTAL_ORDER:
        kw["split_points"] = splits
    return kw


def _host_path(recs, P, kw, part_ids):
    kv, ko, kl, vl = _pack(recs)
    with T.GpuSorter(P, **kw) as s:
        if len(recs):
            s.collect(kv, ko.astype(np.uint32), (ko + kl).astype(np.uint32), vl, part_ids)
        out, _, index, st = s.flush_to_memory()
    return bytes(out), index, st


def _device_path(P, kw, d_kv, kv_bytes, d_ko, d_vo, d_vl, n, d_part=None, out_cap=None, kv_ptr=None):
    with T.GpuSorter(P, **kw) as s:
        cap = s.device_output_bound(n, kv_bytes) if out_cap is None else out_cap
        d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device=DEV)
        out_len, index, st = s.sort_device(d_kv.data_ptr() if kv_ptr is None else kv_ptr, kv_bytes, d_ko.data_ptr(),
                                           d_vo.data_ptr(), d_vl.data_ptr(), n, d_out.data_ptr(), cap,
                                           None if d_part is None else d_part.data_ptr())
    tail = d_out[out_len:]
    assert bool((tail == SENTINEL).all()), "bytes written past out_len"
    return d_out[:out_len].cpu().numpy().tobytes(), index, st


def _oracle(recs, P, cmp, part_ids, rle, combiner, unordered):
    kv, ko, kl, vl = _pack(recs)
    if combiner:
        e = CM.sort_combine(P, cmp, combiner, kv, ko, kl, vl, part_ids)
        return e["file_out"], e["index"]
    conf = O.sorter_conf(P, cmp_kind=cmp, partitioner=O.PART_GIVEN if part_ids is not None else O.PART_HASH,
                         rle_policy=0 if unordered else rle)
    e = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl, part_ids)
    return e["file_out"], e["index"]


def _case(recs, P, cmp, part=T.PART_HASH, rle=T.RLE_AUTO, combiner=0, codec=0, unordered=False, seed=0, splits=None):
    """host path == sort_device on a shuffled placement with gaps (== oracle when uncompressed)"""
    rng = random.Random(seed)
    part_ids = None
    if part == T.PART_GIVEN:
        part_ids = np.array([rng.randrange(P) for _ in recs], dtype=np.int32)
    kw = _sorter_kw(P, cmp, part, rle, combiner, codec, unordered, splits)
    exp, exp_idx, exp_st = _host_path(recs, P, kw, part_ids)
    buf, ko, vo, vl = _scatter(recs, seed + 1)
    got, idx, st = _device_path(P, kw, _dev(buf), buf.size, _dev(ko, np.int64), _dev(vo, np.int64),
                                _dev(vl, np.int32), len(recs), None if part_ids is None else _dev(part_ids))
    assert got == exp, "sort_device file.out differs from collect_batch + flush_to_memory"
    assert np.array_equal(idx, exp_idx)
    assert st["output_bytes"] == exp_st["output_bytes"] and st["output_records"] == exp_st["output_records"]
    assert st["rle_used"] == exp_st["rle_used"]
    if not codec:
        if part == T.PART_TOTAL_ORDER:
            part_ids = np.array(TO.partitions([k for k, _ in recs], splits, cmp), dtype=np.int32)
        o_out, o_idx = _oracle(recs, P, cmp, part_ids, rle, combiner, unordered)
        assert got == o_out, "sort_device file.out differs from the oracle"
        assert np.array_equal(idx, o_idx)
    return st


def _content(rng, cmp):
    if cmp == O.CMP_INT:
        return rng.randbytes(4)
    if cmp == O.CMP_LONG:
        return rng.randbytes(8)
    return bytes(rng.choice(b"abcdefgh\x00\xff") for _ in range(rng.randint(0, 14)))


def _records(cmp, n, seed):
    """values are a function of their key: the order inside a group of equal keys, which the contract does not pin,
    cannot change a byte"""
    rng = random.Random(seed)
    pool = [serialize(cmp, _content(rng, cmp)) for _ in range(n // 3)]
    recs = []
    for _ in range(n):
        k = rng.choice(pool)
        recs.append((k, fill(k, zlib.crc32(k) % 41)))
    return recs


@pytest.mark.parametrize("part", [T.PART_HASH, T.PART_GIVEN, T.PART_TOTAL_ORDER])
@pytest.mark.parametrize("cmp", [O.CMP_TEXT, O.CMP_BYTESWRITABLE, O.CMP_BYTES, O.CMP_INT, O.CMP_LONG])
def test_comparators_and_partitioners(cmp, part):
    recs = _records(cmp, 20000, seed=cmp * 10 + part)
    P = 7
    splits = TO.quantile_splits([k for k, _ in recs], P, cmp) if part == T.PART_TOTAL_ORDER else None
    _case(recs, P, cmp, part, rle=T.RLE_OFF, seed=cmp + 3 * part, splits=splits)


def _word_records(n, seed=7, first=0):
    kv, ko, vo, vl = synth.gen_words(first, n, seed=seed, vocab=5000)
    b, ko, vo = kv.numpy().tobytes(), ko.numpy(), vo.numpy()
    return [(b[ko[i]:vo[i]], b[vo[i]:vo[i] + 4]) for i in range(n)]


def test_rle_auto_on_duplicate_heavy_words():
    st = _case(_word_records(100000), 16, O.CMP_TEXT, rle=T.RLE_AUTO, seed=5)
    assert st["rle_used"] == 1


@pytest.mark.parametrize("combiner", [T.COMBINE_SUM_INT, T.COMBINE_SUM_LONG])
def test_combiners(combiner):
    recs = _word_records(60000, seed=9)
    if combiner == T.COMBINE_SUM_LONG:
        recs = [(k, O.long_writable(len(k) * 1000003 - 7)) for k, _ in recs]
    _case(recs, 8, O.CMP_TEXT, combiner=combiner, rle=T.RLE_OFF, seed=11)


@pytest.mark.parametrize("codec", [T.CODEC_DEFAULT, T.CODEC_LZ4, T.CODEC_ZSTD])
def test_codecs(codec):
    _case(_word_records(80000, seed=13), 8, O.CMP_TEXT, codec=codec, seed=17)


def test_unordered_handle():
    _case(_records(O.CMP_TEXT, 30000, seed=21), 5, O.CMP_TEXT, part=T.PART_GIVEN, unordered=True, seed=23)


@pytest.mark.parametrize("cmp", [O.CMP_TEXT, O.CMP_BYTES])
def test_empty_keys_and_values_larger_than_the_emit_image(cmp):
    # CMP_BYTES: keys of 0 bytes; CMP_TEXT: empty Text keys (the 1-byte vint 0)
    recs = size_mix(cmp, seed=31, n_small=1500) + [(serialize(cmp, b""), b"v" * 300)] * 5
    _case(recs, 3, cmp, rle=T.RLE_AUTO, seed=33)


def test_records_generated_on_the_device_match_the_host_generator():
    """gen_words on the GPU writes the bytes the CPU generator writes, and sort_device sorts them in place"""
    n = 200000
    kv, ko, vo, vl = synth.gen_words(1000, n, seed=3, vocab=20000, device=DEV)
    h = synth.gen_words(1000, n, seed=3, vocab=20000)
    assert torch.equal(kv.cpu(), h[0]) and torch.equal(ko.cpu(), h[1]) and torch.equal(vo.cpu(), h[2])
    b = h[0].numpy().tobytes()
    recs = [(b[a:c], b[c:c + 4]) for a, c in zip(h[1].tolist(), h[2].tolist())]
    kw = _sorter_kw(32, O.CMP_TEXT, T.PART_HASH)
    exp, exp_idx, _ = _host_path(recs, 32, kw, None)
    got, idx, _ = _device_path(32, kw, kv, kv.numel(), ko, vo, vl, n)
    assert got == exp and np.array_equal(idx, exp_idx)


def test_records_end_exactly_at_kv_bytes_before_poisoned_bytes():
    """kv_bytes is not a multiple of 16 and the allocation goes on with bytes that must not reach the output"""
    recs = _records(O.CMP_TEXT, 5000, seed=41)
    kv, ko, kl, vl = _pack(recs)
    kv = np.concatenate([kv, np.frombuffer(b"\x01xyz", np.uint8)])    # one more record ends at kv_bytes
    recs.append((b"\x01x", b"yz"))
    ko, kl, vl = np.append(ko, kv.size - 4), np.append(kl, 2).astype(np.uint32), np.append(vl, 2).astype(np.uint32)
    if kv.size % 16 == 0:
        kv, ko = np.concatenate([np.zeros(1, np.uint8), kv]), ko + 1
    kw = _sorter_kw(4, O.CMP_TEXT, T.PART_HASH, rle=T.RLE_OFF)
    exp, exp_idx, _ = _host_path(recs, 4, kw, None)
    outs = []
    for poison in (0xFF, 0x00, 0x7F):
        d = torch.full((kv.size + 4096,), poison, dtype=torch.uint8, device=DEV)
        d[:kv.size] = _dev(kv)
        got, idx, _ = _device_path(4, kw, d, kv.size, _dev(ko, np.int64), _dev(ko + kl, np.int64),
                                   _dev(vl, np.int32), len(recs))
        outs.append(got)
        assert got == exp and np.array_equal(idx, exp_idx)
    assert outs[0] == outs[1] == outs[2]


def test_records_past_4_gib():
    """Records on both sides of the 4 GiB offset of a 4.5 GiB buffer, one across it and one ending at kv_bytes, placed in
    shuffled order: 64-bit offsets all the way"""
    recs = _records(O.CMP_TEXT, 4000, seed=51)
    kv_bytes = (9 << 29) + 5                     # 4.5 GiB + 5
    rng = random.Random(53)
    order = list(range(len(recs)))
    rng.shuffle(order)
    ko, vo = np.zeros(len(recs), np.uint64), np.zeros(len(recs), np.uint64)
    d = torch.zeros(kv_bytes, dtype=torch.uint8, device=DEV)
    half = len(order) // 2
    last = order[-1]
    tail_len = len(recs[last][0]) + len(recs[last][1])
    # region starts: low half at 1 MiB, the straddler just below 4 GiB, the high half past it, the last record at the end
    regions = [((1 << 20) + 3, order[:half]), ((1 << 32) - 7, order[half:half + 1]), ((1 << 32) + (1 << 20) + 9, order[half + 1:-1]),
               (kv_bytes - tail_len, [last])]
    for at, members in regions:
        blob = bytearray()
        for i in members:
            k, v = recs[i]
            ko[i], vo[i] = at + len(blob), at + len(blob) + len(k)
            blob += k + v + rng.randbytes(rng.randint(0, 9))
        blob = blob[:kv_bytes - at]
        if blob:
            d[at:at + len(blob)] = torch.frombuffer(blob, dtype=torch.uint8).to(DEV)
    vl = np.array([len(v) for _, v in recs], dtype=np.uint32)
    assert (ko > (1 << 32)).sum() > 1000 and (ko < (1 << 32)).sum() > 1000 and int(vo[last]) + len(recs[last][1]) == kv_bytes
    kw = _sorter_kw(5, O.CMP_TEXT, T.PART_HASH)
    exp, exp_idx, _ = _host_path(recs, 5, kw, None)
    payload = sum(len(k) + len(v) for k, v in recs)
    got, idx, _ = _device_path(5, kw, d, kv_bytes, _dev(ko, np.int64), _dev(vo, np.int64), _dev(vl, np.int32),
                               len(recs), out_cap=payload + 12 * len(recs) + 10 * 5 + 64)
    del d
    assert got == exp and np.array_equal(idx, exp_idx)
    o_out, o_idx = _oracle(recs, 5, O.CMP_TEXT, None, T.RLE_AUTO, 0, False)
    assert got == o_out and np.array_equal(idx, o_idx)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_leave_d_out_untouched_and_the_handle_usable():
    P, n = 6, 3000
    recs = _records(O.CMP_TEXT, n, seed=61)
    part = np.array([zlib.crc32(k) % P for k, _ in recs], dtype=np.int32)
    kv, ko, kl, vl = _pack(recs)
    kv = np.concatenate([kv, np.zeros(64, np.uint8)])
    kv_bytes = int(ko[-1]) + int(kl[-1]) + int(vl[-1])
    kw = _sorter_kw(P, O.CMP_TEXT, T.PART_GIVEN)
    exp, exp_idx, _ = _host_path(recs, P, kw, part)
    d_kv, d_ko, d_vo = _dev(kv), _dev(ko, np.int64), _dev(ko + kl, np.int64)
    d_vl, d_part = _dev(vl, np.int32), _dev(part)
    s = T.GpuSorter(P, **kw)
    cap = s.device_output_bound(n, kv_bytes)
    d_out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device=DEV)

    def call(kv_ptr=None, kvb=kv_bytes, ko_=None, vo_=None, part_=None, nn=n, out_ptr=None, h=s):
        return h.sort_device(d_kv.data_ptr() if kv_ptr is None else kv_ptr, kvb, (d_ko if ko_ is None else ko_).data_ptr(),
                             (d_vo if vo_ is None else vo_).data_ptr(), d_vl.data_ptr(), nn, d_out.data_ptr() if out_ptr is None else out_ptr,
                             cap, (d_part if part_ is None else part_).data_ptr())

    def refused(code, match, **a):
        with pytest.raises(TezGpuError, match=match) as e:
            call(**a)
        assert e.value.code == code
        assert bool((d_out == SENTINEL).all()), "a refused call wrote d_out"
        ln, idx, _ = call()                                            # the handle serves the next valid call
        assert d_out[:ln].cpu().numpy().tobytes() == exp and np.array_equal(idx, exp_idx)
        d_out.fill_(SENTINEL)

    refused(T.E_INVALID, "16-byte aligned", kv_ptr=d_kv.data_ptr() + 1)
    refused(T.E_INVALID, "16-byte aligned", out_ptr=d_out.data_ptr() + 8)
    bad_ko = d_ko.clone()
    bad_ko[1234] = d_vo[1234] + 1
    bad_ko[2000] = d_vo[2000] + 1
    refused(T.E_INVALID, "record 1234: key offset after value offset", ko_=bad_ko)
    short = int(ko[2500])                                              # records from 2500 on end past it
    refused(T.E_INVALID, "record 2500: value ends past kv_bytes", kvb=short)
    bad_part = d_part.clone()
    bad_part[77] = P
    bad_part[78] = -1
    refused(T.E_INVALID, "record 77: Illegal partition", part_=bad_part)
    refused(T.E_INVALID, "2\\^30-1", nn=1 << 30)
    with T.GpuSorter(P, fixed=(16, 64), partitioner=T.PART_GIVEN) as f:
        refused(T.E_STATE, "fixed-width", h=f)
    s.collect(kv[:kv_bytes], ko.astype(np.uint32), (ko + kl).astype(np.uint32), vl, part)
    with pytest.raises(TezGpuError, match="reset it first") as e:
        call()
    assert e.value.code == T.E_STATE and bool((d_out == SENTINEL).all())
    s.reset()
    refused(T.E_INVALID, "16-byte aligned", kv_ptr=d_kv.data_ptr() + 4)   # after the reset the handle takes device records again
    s.close()

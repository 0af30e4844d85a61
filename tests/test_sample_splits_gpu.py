"""GPU: the device sampler (tezgpu_sample_keys) and split selection (tezgpu_select_split_points) against
tests/sample_splits_model.py: the sampled set at every rate with and without the cap, ties in h, records in any order
with gaps and poisoned bytes after the last one, the refusal of a bad record, sampling in halves, the split points of
writePartitionFile's rule for the five comparators and both search orders, those splits fed to a TOTAL_ORDER sort
against the oracle, a skewed sample's out-of-order splits, and the capacity errors."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import _lib, native
import sample_splits_model as SM
import sort_order_model as M
import total_order_model as TO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
CMPS = [O.CMP_BYTES, O.CMP_TEXT, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG]


def _content(rng, cmp, pool):
    if cmp in M.FIXED_LEN:
        return bytes(rng.randrange(256) for _ in range(M.FIXED_LEN[cmp])) if rng.random() < 0.5 else rng.choice(pool)[:M.FIXED_LEN[cmp]].ljust(M.FIXED_LEN[cmp], b"\0")
    return rng.choice(pool) if rng.random() < 0.5 else bytes(rng.randrange(97, 100) for _ in range(rng.randrange(0, 9)))


def _keys(rng, cmp, n):
    pool = [bytes(rng.randrange(256) for _ in range(rng.randrange(0, 12))) for _ in range(max(1, n // 20))]
    return [M.make_key(cmp, _content(rng, cmp, pool)) for _ in range(n)]


class DeviceRecords:
    """records in a device buffer in shuffled order with gaps; kv_bytes ends exactly at the last record's value, the
    bytes after it are poisoned"""

    def __init__(self, keys, rng, poison=0xEE):
        n = len(keys)
        vals = [bytes(rng.randrange(256) for _ in range(rng.randrange(0, 6))) for _ in range(n)]
        order = list(range(n))
        rng.shuffle(order)
        buf = bytearray()
        ko, vo, vl = [0] * n, [0] * n, [0] * n
        for i in order:
            buf += bytes([poison]) * rng.randrange(0, 3)
            ko[i] = len(buf)
            buf += keys[i]
            vo[i] = len(buf)
            buf += vals[i]
            vl[i] = len(vals[i])
        self.kv_bytes = len(buf)
        buf += bytes([poison]) * 64
        self.kv = torch.tensor(list(buf), dtype=torch.uint8, device=DEV)
        self.ko = torch.tensor(ko, dtype=torch.int64, device=DEV)
        self.vo = torch.tensor(vo, dtype=torch.int64, device=DEV)
        self.vl = torch.tensor(vl, dtype=torch.int32, device=DEV)
        self.keys, self.n = keys, n
        torch.cuda.synchronize()

    def args(self, lo=0, hi=None):
        hi = self.n if hi is None else hi
        return (self.kv.data_ptr(), self.kv_bytes, self.ko.data_ptr() + 8 * lo, self.vo.data_ptr() + 8 * lo,
                self.vl.data_ptr() + 4 * lo, hi - lo)


def _check_sample(s, expected, keys, gid_base=0):
    assert s.gid.tolist() == [g for _, g in expected]
    assert s.h.tolist() == [h for h, _ in expected]
    assert native.sample_key_list(s) == [keys[g - gid_base] for _, g in expected]
    assert s.key_off.tolist() == (np.cumsum(s.key_len, dtype=np.uint64) - s.key_len).tolist()


@pytest.mark.parametrize("freq", [0.0, 1e-4, 0.1, 1.0])
@pytest.mark.parametrize("cap", [40, 1 << 20])
def test_sample_equals_model(freq, cap):
    rng = random.Random(int(freq * 1000) + cap)
    n = 30000
    keys = _keys(rng, O.CMP_TEXT, n)
    d = DeviceRecords(keys, rng)
    s = native.sample_keys(*d.args(), seed=77, freq=freq, max_samples=cap, gid_base=123)
    exp = SM.sample(n, 77, freq, cap, gid_base=123)
    _check_sample(s, exp, keys, gid_base=123)
    if freq >= 0.1:
        assert (len(exp) == cap) == (cap == 40)      # the cap is hit exactly when it is the small one


def test_sample_ties_in_h_break_by_gid():
    L = _lib.load()
    rng = random.Random(5)
    keys = _keys(rng, O.CMP_BYTES, 5000)
    d = DeviceRecords(keys, rng)
    mask = 0xF << 60
    old = L.tezgpu_debug_set_sample_hash_mask(mask)
    try:
        for freq, cap in ((1.0, 700), (0.5, 333), (1.0, 1)):
            s = native.sample_keys(*d.args(), seed=3, freq=freq, max_samples=cap)
            exp = SM.sample(5000, 3, freq, cap, mask=mask)
            assert len({h for h, _ in exp}) < len(exp) or cap == 1
            _check_sample(s, exp, keys)
    finally:
        L.tezgpu_debug_set_sample_hash_mask(old)


def test_bad_record_refused_by_index_before_anything_is_written():
    L = _lib.load()
    rng = random.Random(6)
    keys = _keys(rng, O.CMP_BYTES, 3000)
    d = DeviceRecords(keys, rng)
    d.vo[2100] = d.kv_bytes + 1          # value past kv_bytes
    d.ko[1900] = d.vo[1900] + 1          # key after value
    torch.cuda.synchronize()
    m = 64
    ko, kl = np.full(m, 7, np.uint64), np.full(m, 7, np.uint32)
    h, gid = np.full(m, 7, np.uint64), np.full(m, 7, np.uint64)
    keys_out = np.full(4096, 7, np.uint8)
    cnt, need = C.c_uint32(9), C.c_uint64(9)
    rc = L.tezgpu_sample_keys(0, *d.args(), 0, 1, 1.0, m, keys_out.ctypes.data, keys_out.size, ko.ctypes.data, kl.ctypes.data,
                              h.ctypes.data, gid.ctypes.data, C.byref(cnt), C.byref(need))
    assert rc == T.E_INVALID
    assert L.tezgpu_last_error().startswith(b"record 1900: key offset after value offset")
    assert (keys_out == 7).all() and (ko == 7).all() and (kl == 7).all() and (h == 7).all() and (gid == 7).all()
    d.ko[1900] = d.vo[1900]
    torch.cuda.synchronize()
    with pytest.raises(_lib.TezGpuError, match="record 2100: value ends past kv_bytes"):
        native.sample_keys(*d.args(), seed=1, freq=0.0, max_samples=m)


def test_nomem_reports_the_bytes_and_writes_nothing():
    L = _lib.load()
    rng = random.Random(7)
    keys = _keys(rng, O.CMP_TEXT, 4000)
    d = DeviceRecords(keys, rng)
    exp = SM.sample(4000, 5, 0.25, 300)
    need_bytes = sum(len(keys[g]) for _, g in exp)
    m = 300
    ko, kl = np.full(m, 7, np.uint64), np.full(m, 7, np.uint32)
    h, gid = np.full(m, 7, np.uint64), np.full(m, 7, np.uint64)
    keys_out = np.full(need_bytes, 7, np.uint8)
    cnt, need = C.c_uint32(9), C.c_uint64(9)
    rc = L.tezgpu_sample_keys(0, *d.args(), 0, 5, 0.25, m, keys_out.ctypes.data, need_bytes - 1, ko.ctypes.data, kl.ctypes.data,
                              h.ctypes.data, gid.ctypes.data, C.byref(cnt), C.byref(need))
    assert rc == T.E_NOMEM and need.value == need_bytes and cnt.value == 0
    assert (keys_out == 7).all() and (ko == 7).all() and (h == 7).all() and (gid == 7).all()
    rc = L.tezgpu_sample_keys(0, *d.args(), 0, 5, 0.25, m, keys_out.ctypes.data, need_bytes, ko.ctypes.data, kl.ctypes.data,
                              h.ctypes.data, gid.ctypes.data, C.byref(cnt), C.byref(need))
    assert rc == 0 and cnt.value == len(exp) and need.value == need_bytes
    # the split points: NOMEM with the bytes they need
    s = native.sample_keys(*d.args(), seed=5, freq=0.25, max_samples=m)
    splits = native.select_split_points(s, 8, m, T.CMP_TEXT)
    total = sum(len(x) for x in splits)
    so, sl, out = np.zeros(7, np.uint64), np.zeros(7, np.uint32), np.full(total, 7, np.uint8)
    rc = L.tezgpu_select_split_points(0, T.CMP_TEXT, T.CMP_TEXT, 8, m, s.keys.ctypes.data, s.key_off.ctypes.data,
                                      s.key_len.ctypes.data, s.h.ctypes.data, s.gid.ctypes.data, s.gid.size, out.ctypes.data,
                                      total - 1, so.ctypes.data, sl.ctypes.data, C.byref(need), None)
    assert rc == T.E_NOMEM and need.value == total and (out == 7).all() and (sl == 0).all()


def test_halves_with_gid_base_give_the_whole_sets_splits():
    rng = random.Random(8)
    n, cap, P = 20000, 1500, 37
    keys = _keys(rng, O.CMP_TEXT, n)
    d = DeviceRecords(keys, rng)
    whole = native.sample_keys(*d.args(), seed=9, freq=0.2, max_samples=cap)
    a = native.sample_keys(*d.args(0, 7000), seed=9, freq=0.2, max_samples=cap)
    b = native.sample_keys(*d.args(7000), seed=9, freq=0.2, max_samples=cap, gid_base=7000)
    assert native.select_split_points([a, b], P, cap, T.CMP_TEXT) == native.select_split_points(whole, P, cap, T.CMP_TEXT)
    assert native.select_split_points([b, a], P, cap, T.CMP_TEXT, with_chosen=True)[1].tolist() == \
        native.select_split_points(whole, P, cap, T.CMP_TEXT, with_chosen=True)[1].tolist()


def _host_sample(keys, seed):
    gid = np.arange(len(keys), dtype=np.uint64) * 3 + 11
    h = np.array([SM.splitmix64(seed ^ int(g)) for g in gid], dtype=np.uint64)
    kv, ko, kl = native._pack_keys(keys)
    return native.KeySample(kv, ko, kl, h, gid)


ORDERS = [(c, c) for c in CMPS] + [(O.CMP_BYTES, O.CMP_TEXT), (O.CMP_BYTES, O.CMP_BYTESWRITABLE)]


@pytest.mark.parametrize("cmp,order", ORDERS)
def test_split_points_equal_the_model(cmp, order):
    rng = random.Random(cmp * 10 + order)
    key_cmp = order if cmp == O.CMP_BYTES and order != cmp else cmp      # natural order: Text / BytesWritable keys
    keys = _keys(rng, key_cmp, 12000)
    s = _host_sample(keys, 21)
    entries = list(zip(s.h.tolist(), s.gid.tolist(), keys))
    for P, cap in ((1, 5000), (2, 5000), (3, 5000), (64, 5000), (1024, 9000), (4097, 12000), (4097, 3000), (50, 20)):
        try:
            exp, exp_k = SM.select(entries, P, cap, cmp)
        except SM.SplitIndexError:
            with pytest.raises(_lib.TezGpuError, match="ArrayIndexOutOfBoundsException"):
                native.select_split_points(s, P, cap, cmp, order)
            continue
        got, got_k = native.select_split_points(s, P, cap, cmp, order, with_chosen=True)
        assert got_k.tolist() == exp_k, (P, cap)
        assert got == exp, (P, cap)


def test_sample_smaller_than_p_and_empty_sample():
    keys = [O.text(bytes([97 + i])) for i in range(5)]
    s = _host_sample(keys, 1)
    entries = list(zip(s.h.tolist(), s.gid.tolist(), keys))
    for P in (2, 3, 5, 6, 9, 40):
        try:
            exp = SM.select(entries, P, 100, O.CMP_TEXT)[0]
        except SM.SplitIndexError:
            with pytest.raises(_lib.TezGpuError, match="ArrayIndexOutOfBoundsException") as e:
                native.select_split_points(s, P, 100, O.CMP_TEXT)
            assert e.value.code == T.E_INVALID
            continue
        assert native.select_split_points(s, P, 100, O.CMP_TEXT) == exp
    empty = _host_sample([], 1)
    with pytest.raises(_lib.TezGpuError, match="empty sample"):
        native.select_split_points(empty, 2, 100, O.CMP_TEXT)
    assert native.select_split_points(empty, 1, 100, O.CMP_TEXT) == []


def test_skewed_sample_split_is_returned_and_refused_by_set_split_points():
    keys = [O.text(c) for c in (b"A", b"A", b"B", b"B", b"B", b"B", b"C")]
    s = _host_sample(keys, 2)
    splits, ks = native.select_split_points(s, 9, 100, O.CMP_TEXT, with_chosen=True)
    srt = sorted(keys, key=lambda k: M.content(O.CMP_TEXT, k))
    assert ks.tolist() == [1, 2, 3, 4, 5, 6, 5, 6] and splits == [srt[k] for k in ks]
    with pytest.raises(_lib.TezGpuError, match="Split points are out of order"):
        T.GpuSorter(9, comparator=T.CMP_TEXT, partitioner=T.PART_TOTAL_ORDER, split_points=splits)
    dup = [O.text(c) for c in [b"x"] * 2 + [b"y"] * 6]
    splits = native.select_split_points(_host_sample(dup, 3), 8, 100, O.CMP_TEXT)
    assert splits == [dup[0]] + [dup[2]] * 6
    with pytest.raises(_lib.TezGpuError, match="Split points are out of order"):
        T.GpuSorter(8, comparator=T.CMP_TEXT, partitioner=T.PART_TOTAL_ORDER, split_points=splits)


@pytest.mark.parametrize("P", [2, 16, 300])
def test_sampled_splits_sort_equals_the_oracle(P):
    """BytesWritable keys of the reference Sort's shape, distinct, so that every P gets increasing splits"""
    rng = random.Random(P)
    n = 40000
    keys = [M.make_key(O.CMP_BYTESWRITABLE, rng.randbytes(rng.randrange(4, 20))) for _ in range(n)]
    d = DeviceRecords(keys, rng)
    s = native.sample_keys(*d.args(), seed=4, freq=0.05, max_samples=1500)
    splits = native.select_split_points(s, P, 1500, T.CMP_BYTESWRITABLE)
    with T.GpuSorter(P, comparator=T.CMP_BYTESWRITABLE, partitioner=T.PART_TOTAL_ORDER, split_points=splits) as sorter:
        cap = sorter.device_output_bound(n, d.kv_bytes)
        out = torch.empty(cap, dtype=torch.uint8, device=DEV)
        out_len, index, _ = sorter.sort_device(*d.args(), out.data_ptr(), cap)
    hkv, hko, hvo, hvl = (t.cpu().numpy() for t in (d.kv, d.ko, d.vo, d.vl))
    part = np.array(TO.partitions(keys, splits, O.CMP_BYTESWRITABLE), dtype=np.int32)
    assert len(set(part.tolist())) == P
    exp = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_BYTESWRITABLE, partitioner=O.PART_GIVEN), hkv[:d.kv_bytes],
                           hko.astype(np.uint64), (hvo - hko).astype(np.uint32), hvl.astype(np.uint32), part)
    assert out[:out_len].cpu().numpy().tobytes() == exp["file_out"]
    assert np.array_equal(index, exp["index"])

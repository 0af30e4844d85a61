"""CPU: the sampler's model (Math.round(float), writePartitionFile's rule on skewed samples, the candidate rule and the
cap) and the argument checks of tezgpu_sample_keys and tezgpu_select_split_points, without a device."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest
import torch

import tez_b200 as T
from tez_b200 import _lib, synth

import sample_splits_model as SM


def test_splitmix64_matches_the_generators():
    xs = [0, 1, 2, 12345, (1 << 63) - 1, 1 << 63, (1 << 64) - 1]
    got = synth.splitmix64(torch.tensor([x - (1 << 64) if x >= 1 << 63 else x for x in xs], dtype=torch.int64))
    assert [int(v) & SM.MASK64 for v in got] == [SM.splitmix64(x) for x in xs]


@pytest.mark.parametrize("x,exp", [(0.5, 1), (1.5, 2), (2.5, 3), (0.49999997, 0), (-0.5, 0), (-1.5, -1), (3.4999998, 3),
                                   (4194303.5, 4194304), (8388607.0, 8388607), (8388608.0, 8388608), (16777215.0, 16777215), (16777216.0, 16777216),
                                   (16777218.0, 16777218)])
def test_java_round_float(x, exp):
    assert float(np.float32(x)) == x or abs(x) < 1e7
    assert SM.java_round(np.float32(x)) == exp


def test_java_round_has_no_double_rounding():
    # 0.49999997f + 0.5f rounds to 1.0f in float; Math.round gives 0
    x = np.float32(0.49999997)
    assert np.float32(x + np.float32(0.5)) == np.float32(1.0)
    assert SM.java_round(x) == 0
    # floats in [2^22, 2^23) are integers and halves (halves round up), from 2^23 on every float is an integer
    for v in (2 ** 22 + 0.5, 2 ** 22 + 1.5, 2 ** 23 - 0.5, 2 ** 23 + 1, 2 ** 24 + 2):
        assert float(np.float32(v)) == v
        assert SM.java_round(np.float32(v)) == int(v + 0.5)
    assert float(np.float32(2 ** 24 + 1)) == 2 ** 24


def test_step_is_float_arithmetic():
    # stepSize = n / (float) P in float: 2^24 + 1 samples round to 2^24 before the division
    assert np.float32(np.float32(2 ** 24 + 1) / np.float32(2)) == np.float32(2 ** 23)
    assert SM.pick([bytes([i % 256, i // 256]) for i in range(10)], 4) == [3, 5, 8]


def test_pick_steps_past_a_run_it_lands_in():
    # samples a a a a b c: P = 3 -> step 2; k = 2 ("a"), then round(4) = 4 ("b")
    assert SM.pick([b"a"] * 4 + [b"b", b"c"], 3) == [2, 4]
    # P = 5 on 6 samples: step 1.2 -> k = 1, 2 (same run as 1? k > last, no loop), 4, 5
    assert SM.pick([b"a"] * 4 + [b"b", b"c"], 5) == [1, 2, 4, 5]


def test_skewed_sample_writes_a_split_below_the_one_before():
    # 7 samples, P = 9, step 7/9: the loop steps i = 3..6 past "B"s to last = 6 ("C"); i = 7 rounds 5.44 to 5 <= last,
    # and samples[5] = "B" differs from samples[6], so the loop stops there and "B" is written after "C"
    keys = [b"A", b"A", b"B", b"B", b"B", b"B", b"C"]
    ks = SM.pick(keys, 9)
    assert ks == [1, 2, 3, 4, 5, 6, 5, 6]
    splits = [keys[k] for k in ks]
    assert splits[6] < splits[5]                  # "B" after "C": TotalOrderPartitioner refuses these splits


def test_k_past_the_end_raises():
    with pytest.raises(SM.SplitIndexError):
        SM.pick([b"a", b"b", b"b"], 4)
    with pytest.raises(SM.SplitIndexError):
        SM.pick([], 2)
    assert SM.pick([], 1) == []


def test_duplicate_split_when_round_lands_inside_the_previous_run():
    # keys x x y y y y y y, P = 8: step 1 -> k = 1 (x), 2 (y), 3 (y) ... splits repeat "y": Java writes them
    keys = [b"x"] * 2 + [b"y"] * 6
    ks = SM.pick(keys, 8)
    assert ks == [1, 2, 3, 4, 5, 6, 7]
    assert [keys[k] for k in ks].count(b"y") == 6


def test_threshold_is_exact():
    assert SM.threshold(0.0) == 0 and SM.threshold(1.0) is None
    assert SM.threshold(0.5) == 1 << 63
    assert SM.threshold(1e-4) == -(-Fraction(1e-4) * (1 << 64) // 1)
    assert SM.threshold(2.0 ** -70) == 1          # a fraction of one hash step still admits h = 0


def test_sample_cap_keeps_the_smallest_hashes_and_is_a_function_of_gid():
    full = SM.sample(2000, 9, 0.5, 100)
    assert len(full) == 100
    assert [g for _, g in full] == sorted(g for _, g in full)
    hs = sorted(SM.splitmix64(9 ^ g) for g in range(2000) if SM.splitmix64(9 ^ g) < 1 << 63)
    assert sorted(h for h, _ in full) == hs[:100]
    a, b = SM.sample(700, 9, 0.5, 100), SM.sample(1300, 9, 0.5, 100, gid_base=700)
    assert sorted(a + b)[:100] == sorted(full)


def test_sample_ties_in_h_break_by_gid():
    got = SM.sample(500, 3, 1.0, 50, mask=0xF << 60)
    hs = sorted((SM.splitmix64(3 ^ g) & (0xF << 60), g) for g in range(500))[:50]
    assert sorted(got) == hs
    assert len({h for h, _ in got}) < len(got)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_device_both_calls_fail_with_cuda_error():
    L = _lib.load()
    cnt, need = C.c_uint32(), C.c_uint64()
    buf = np.zeros(16, dtype=np.uint64)
    assert L.tezgpu_sample_keys(0, None, 0, None, None, None, 0, 0, 1, 0.5, 4, None, 0, buf.ctypes.data, buf.ctypes.data,
                                buf.ctypes.data, buf.ctypes.data, C.byref(cnt), C.byref(need)) == T.E_CUDA
    kv = np.frombuffer(b"ab", dtype=np.uint8)
    ko, kl = np.zeros(2, dtype=np.uint64), np.ones(2, dtype=np.uint32)
    ko[1] = 1
    h, g = np.array([5, 6], dtype=np.uint64), np.array([0, 1], dtype=np.uint64)
    out, so, sl = np.zeros(16, np.uint8), np.zeros(2, np.uint64), np.zeros(2, np.uint32)
    assert L.tezgpu_select_split_points(0, T.CMP_BYTES, T.CMP_BYTES, 2, 10, kv.ctypes.data, ko.ctypes.data, kl.ctypes.data,
                                        h.ctypes.data, g.ctypes.data, 2, out.ctypes.data, out.size, so.ctypes.data,
                                        sl.ctypes.data, C.byref(need), None) == T.E_CUDA


def test_sample_keys_argument_checks():
    L = _lib.load()
    cnt, need = C.c_uint32(), C.c_uint64()
    a = np.zeros(16, dtype=np.uint64)
    p = a.ctypes.data

    def call(freq=0.5, n=4, d=p, count=True, idx=p, max_samples=4):
        return L.tezgpu_sample_keys(0, d, 64, d, d, d, n, 0, 1, freq, max_samples, p, 64, idx, idx, idx, idx,
                                    C.byref(cnt) if count else None, C.byref(need))
    for freq in (-0.1, 1.0000001, float("nan"), float("inf")):
        assert call(freq=freq) == T.E_INVALID
        assert b"freq" in L.tezgpu_last_error()
    assert call(d=None) == T.E_INVALID
    assert call(count=False) == T.E_INVALID
    assert call(idx=None) == T.E_INVALID
    assert call(n=1 << 32) == T.E_INVALID


def test_select_split_points_argument_checks():
    L = _lib.load()
    need = C.c_uint64()
    a = np.zeros(16, dtype=np.uint64)
    p = a.ctypes.data

    def call(cmp=T.CMP_BYTES, order=T.CMP_BYTES, P=2, keys=p, out_len=True, max_samples=10):
        return L.tezgpu_select_split_points(0, cmp, order, P, max_samples, keys, p, p, p, p, 2, p, 64, p, p,
                                            C.byref(need) if out_len else None, None)
    assert call(cmp=9) == T.E_UNSUPPORTED
    assert call(cmp=T.CMP_TEXT, order=T.CMP_BYTES) == T.E_INVALID
    assert call(P=0) == T.E_INVALID
    assert call(keys=None) == T.E_INVALID
    assert call(out_len=False) == T.E_INVALID
    assert call(max_samples=1 << 30) == T.E_INVALID

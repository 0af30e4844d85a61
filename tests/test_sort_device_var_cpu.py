"""CPU: the device-resident variable-length sort without a device, its output bound, and the word generator.

tezgpu_sorter_device_output_bound must cover what the sort writes before the sort has run: here it is compared with the
files the CPU oracle writes for random record sets (uncompressed), and with those files' segments compressed by the host
runs of the device codecs (tezgpu_debug_*_compress_emulate) -- the bytes the device writes, as the codec tests show."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import _lib, synth
from tez_b200._lib import TezGpuError

import codec_model as CM
import lz4_model as L4
import zstd_model as ZS


def _bound(P, codec, n, kv_bytes):
    return _lib.load().tezgpu_debug_device_output_bound(P, codec, n, kv_bytes)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_device_both_calls_fail_with_cuda_error():
    for call in (lambda s: s.sort_device(0, 0, 0, 0, 0, 0, 0, 0), lambda s: s.device_output_bound(10, 100)):
        with pytest.raises(TezGpuError, match="no CUDA device") as e:
            call(T.GpuSorter(4, comparator=T.CMP_TEXT))
        assert e.value.code == T.E_CUDA
    # without a handle: an argument error, and a bound of 0
    L = _lib.load()
    out_len = C.c_uint64()
    assert L.tezgpu_sorter_sort_device(None, None, 0, None, None, None, None, 0, None, 0, C.byref(out_len), None, None) == T.E_INVALID
    assert L.tezgpu_sorter_device_output_bound(None, 10, 100) == 0


def test_debug_bound_refuses_bad_arguments():
    assert _bound(0, T.CODEC_NONE, 1, 1) == 0
    assert _bound(1, 9, 1, 1) == 0
    assert _bound(3, T.CODEC_NONE, 0, 0) == 30 + 64


def _random_records(rng, n):
    pool = [O.text(bytes(rng.choice(b"abcde") for _ in range(rng.randint(0, 12)))) for _ in range(max(1, n // 4))]
    return [(rng.choice(pool), rng.randbytes(rng.choice((0, 1, 4, 30, 200, 70000)) if rng.random() < 0.01 else rng.randint(0, 20)))
            for _ in range(n)]


def _pack(recs):
    kl = np.array([len(k) for k, _ in recs], dtype=np.uint64)
    vl = np.array([len(v) for _, v in recs], dtype=np.uint64)
    ko = np.zeros(len(recs), dtype=np.uint64)
    if recs:
        ko[1:] = np.cumsum(kl + vl)[:-1]
    kv = np.frombuffer(b"".join(k + v for k, v in recs) + b"\0", dtype=np.uint8)
    return kv, ko, kl.astype(np.uint32), vl.astype(np.uint32)


COMPRESS = {T.CODEC_DEFAULT: CM.deflate_emulate, T.CODEC_LZ4: L4.compress_emulate, T.CODEC_ZSTD: ZS.compress_emulate}


@pytest.mark.parametrize("seed", range(6))
def test_bound_covers_what_is_written(seed):
    rng = random.Random(seed)
    n = rng.choice((0, 1, 7, 300, 5000, 40000))
    P = rng.choice((1, 2, 13, 200))
    recs = _random_records(rng, n)
    kv, ko, kl, vl = _pack(recs)
    kv_bytes = int(sum(len(k) + len(v) for k, v in recs))          # the tightest buffer: records back to back
    for rle, unordered in ((0, False), (1, False), (-1, False), (0, True)):
        conf = O.sorter_conf(P, cmp_kind=O.CMP_TEXT, rle_policy=rle)
        res = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl)
        assert len(res["file_out"]) <= _bound(P, T.CODEC_NONE, n, kv_bytes)
        if rle != 0:
            continue
        for codec, compress in COMPRESS.items():
            written = 0
            for start, _, part in res["index"].tolist():
                if part:
                    seg = res["file_out"][start:start + part]
                    written += 4 + len(compress(seg[4:-4])) + 4     # TIF\x01 + stream + CRC-32
            assert written <= _bound(P, codec, n, kv_bytes), (codec, n, P)


def test_gen_words_is_a_function_of_index_and_seed():
    kv, ko, vo, vl = synth.gen_words(0, 5000, seed=3, vocab=1000)
    kv2, ko2, vo2, _ = synth.gen_words(1234, 2000, seed=3, vocab=1000)
    a, b = int(ko[1234]), int(ko[3234])
    assert kv2.numpy().tobytes() == kv.numpy().tobytes()[a:b]
    assert torch.equal(ko2 + a, ko[1234:3234]) and torch.equal(vo2 + a, vo[1234:3234])
    assert kv.numpy().tobytes() != synth.gen_words(0, 5000, seed=4, vocab=1000)[0].numpy().tobytes()
    data = kv.numpy().tobytes()
    counts = {}
    assert torch.equal(vl, torch.full((5000,), 4, dtype=torch.int32))
    assert int(vo[-1]) + 4 == kv.numel() and torch.equal(ko[1:], vo[:-1] + 4)
    for k0, v0 in zip(ko.tolist(), vo.tolist()):
        key, val = data[k0:v0], data[v0:v0 + 4]
        assert 3 <= key[0] <= 12 and len(key) == 1 + key[0] and all(97 <= c <= 122 for c in key[1:])
        assert val == O.int_writable(1)
        counts[key] = counts.get(key, 0) + 1
    top = sorted(counts.values(), reverse=True)
    assert top[0] > 5 * top[min(len(top) - 1, 50)]                    # Zipf: the head words dominate

"""Device selection at the C ABI boundary: every call runs on its handle's conf.device (or its device argument) and
returns with the calling thread's CUDA context current again.  Handles on device 1, driven from a thread whose current
device is 0, write the bytes the same runs write on device 0; a thread that never used CUDA gets no context on device 0.
Threads that touch a device for the first time together all sort with its checksum tables."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200 import native  # noqa: E402
from tez_b200._lib import TezGpuError  # noqa: E402

import codec_model as CM  # noqa: E402
import lz4_model as L4  # noqa: E402

pytestmark = pytest.mark.gpu
P = 4
REC = 80   # config-2 records: 16-byte keys, 64-byte values


def _need_two_devices():
    if T._lib.load().tezgpu_device_count() < 2:
        pytest.skip("needs two visible CUDA devices")


def _call(fn, *args, **kw):
    """one library call from a thread whose current device is 0, which it must leave at 0"""
    torch.cuda.set_device(0)
    out = fn(*args, **kw)
    assert torch.cuda.current_device() == 0, "%s changed the current device" % getattr(fn, "__name__", fn)
    return out


# ------------------------------------------------------------------------------------------------ sorter
def _sort_fixed(device, kv):
    s = _call(T.GpuSorter, P, fixed=(16, 64), device=device)
    half = len(kv) // 2 // REC * REC
    _call(s.collect_fixed, kv[:half])
    _call(s.collect_fixed, kv[half:])
    out, index_bytes, index, st = _call(s.flush_to_memory)
    _call(s.close)
    return bytes(out), index_bytes, st


def _variable_batches(seed, batches=3, n=20000):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(batches):
        klen = rng.integers(1, 25, n)
        vlen = rng.integers(0, 61, n)
        key_off = np.zeros(n, dtype=np.uint32)
        key_off[1:] = np.cumsum(klen + vlen)[:-1]
        kv = rng.integers(0, 256, int((klen + vlen).sum()), dtype=np.uint8)
        out.append((kv, key_off, key_off + klen.astype(np.uint32), vlen.astype(np.uint32)))
    return out


def _sort_variable(device, batches, tmp):
    s = _call(T.GpuSorter, P, comparator=T.CMP_BYTES, device=device)
    for b in batches:
        _call(s.collect, *b)
    f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
    index, st = _call(s.flush, f, fi)
    _call(s.close)
    return open(f, "rb").read(), open(fi, "rb").read(), index.tolist(), st


def _sort_device_resident(device, kv):
    """sort_device_fixed on this device's buffers, then the shuffle response of every partition from the sorted file"""
    dev = torch.device("cuda", device)
    n = len(kv) // REC
    cap = len(kv) + 12 * n + 10 * P + 64
    d_kv = torch.from_numpy(kv).to(dev)
    d_out = torch.empty(cap, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    s = _call(T.GpuSorter, P, fixed=(16, 64), device=device)
    out_len, index, st = _call(s.sort_device_fixed, d_kv.data_ptr(), n, d_out.data_ptr(), cap)
    torch.cuda.synchronize(dev)
    body = _call(native.shuffle_serve, d_out.data_ptr(), index, "attempt_1_0001_m_000000_0", 0, P, device=device)
    _call(s.close)
    return d_out[:out_len].cpu().numpy().tobytes(), index.tolist(), body, st


def test_sorter_on_device_1_driven_from_device_0(tmp_path):
    _need_two_devices()
    kv = O.gen_c2(0, 200000, seed=7)
    batches = _variable_batches(3)
    for run in (lambda d: _sort_fixed(d, kv), lambda d: _sort_variable(d, batches, str(tmp_path)),
                lambda d: _sort_device_resident(d, kv)):
        out0, out1 = run(0), run(1)
        assert out1[:-1] == out0[:-1], "device 1 wrote other bytes than device 0"
        assert out1[-1]["ms_total"] > 0, "no device time measured on device 1: its events are not on its device"


# ------------------------------------------------------------------------------------------------ merger
def _fixed_segments(G=3, n=20000):
    """the P partition segments of G config-2 sorts (several bounded-merge steps at the 16 MiB floor)"""
    segs, parts = [], []
    for g in range(G):
        r = O.pipelined_sort_fixed(O.sorter_conf(P), O.gen_c2(g * 2 * n, n, seed=9 + g), 16, 64)
        for p in range(P):
            start, _, part = (int(x) for x in r["index"][p])
            if part:
                segs.append(bytes(r["file_out"][start:start + part]))
                parts.append(p)
    return segs, parts


def _merge(device, segs, parts, tmp, **kw):
    m = _call(T.GpuMerger, segs, partitions=parts, num_partitions=P, device=device, **kw)
    recs = []
    torch.cuda.set_device(0)
    for r in m.records(batch_records=997, batch_bytes=1 << 16):
        assert torch.cuda.current_device() == 0, "next_batch changed the current device"
        recs.append(r)
    f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
    index, st = _call(m.write_partitions, f, fi)
    counts = _call(m.counts)
    steps = _call(m.bounded_info)[0] if m.bounded else 1
    _call(m.close)
    return recs, open(f, "rb").read(), open(fi, "rb").read(), index.tolist(), counts, steps, st


@pytest.mark.parametrize("route", ["host", "lz4", "concat", "bounded"])
def test_merger_on_device_1_driven_from_device_0(route, tmp_path):
    _need_two_devices()
    segs, parts = _fixed_segments()
    kw = {"comparator": T.CMP_BYTES}
    if route == "lz4":
        kw.update(codec=T.CODEC_LZ4, raw_lens=[len(s) - 4 for s in segs])
        segs = [L4.segment(L4.compress_emulate(CM.body_of(s))) for s in segs]
    elif route == "concat":
        kw.update(concat=True)
    elif route == "bounded":
        kw.update(device_budget=16 << 20)
    out0 = _merge(0, segs, parts, str(tmp_path), **kw)
    out1 = _merge(1, segs, parts, str(tmp_path), **kw)
    assert out1[:-1] == out0[:-1], "device 1 merged other records or bytes than device 0"
    if route == "bounded":
        assert out1[5] > 1, "the bounded merge took one step"
    assert out1[-1]["ms_total"] > 0, "no device time measured on device 1: its events are not on its device"


# ------------------------------------------------------------------------------------------------ device argument
def test_device_argument_calls_leave_the_current_device():
    _need_two_devices()
    buf = _call(T.PeerBuffer, 1 << 20, device=1)
    _call(buf.close)
    dev = torch.device("cuda", 1)
    seg = O.write_ifile([(b"k%05d" % i, b"v" * (i % 50)) for i in range(3000)])[0]
    src = torch.frombuffer(bytearray(seg), dtype=torch.uint8).to(dev)
    dst = torch.zeros(len(seg) + 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    _call(T.fetch_ranges, [(src.data_ptr(), dst.data_ptr(), len(seg))], device=1)
    assert dst[:len(seg)].cpu().numpy().tobytes() == seg
    dst.zero_()
    torch.cuda.synchronize(dev)
    _call(T.fetch_segments_verified, [(src.data_ptr(), dst.data_ptr(), len(seg))], device=1)
    assert dst[:len(seg)].cpu().numpy().tobytes() == seg


# ------------------------------------------------------------------------------------------------ first touch
def _sort_c2_on_device_0(kv):
    with T.GpuSorter(64, fixed=(16, 64), device=0) as s:
        s.collect_fixed(kv)
        out, index_bytes, _, _ = s.flush_to_memory()
    return bytes(out), index_bytes


def _first_touch_worker():
    """four threads create their sorters at once, before anything else in this process touched device 0"""
    kv = O.gen_c2(0, 100000, seed=4)
    start = threading.Barrier(4)
    outs, errors = [None] * 4, []

    def sort(i):
        try:
            start.wait()
            outs[i] = _sort_c2_on_device_0(kv)
        except Exception as e:   # reported by the parent
            errors.append(repr(e))

    threads = [threading.Thread(target=sort, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    one = _sort_c2_on_device_0(kv)
    assert all(o == one for o in outs), "a thread that first touched the device wrote other bytes"
    print("first-touch ok")


def _worker(mode):
    """runs this file's worker `mode` in a fresh process, where nothing has touched a device yet"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), mode], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and mode + " ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_threads_that_first_touch_a_device_together():
    _worker("first-touch")


# ------------------------------------------------------------------------------------------------ the caller's context
def _cuda_driver():
    cu = C.CDLL("libcuda.so.1")
    assert cu.cuInit(0) == 0
    return cu


def _primary_context_active(cu, ordinal):
    dev, flags, active = C.c_int(), C.c_uint(), C.c_int()
    assert cu.cuDeviceGet(C.byref(dev), ordinal) == 0
    assert cu.cuDevicePrimaryCtxGetState(dev, C.byref(flags), C.byref(active)) == 0
    return bool(active.value)


def _own_context_worker():
    """a thread whose current context is one it created has that context current again after every call"""
    cu = _cuda_driver()
    dev, own, cur = C.c_int(), C.c_void_p(), C.c_void_p()
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuCtxCreate_v2(C.byref(own), 0, dev) == 0

    def call(fn, *args, **kw):
        out = fn(*args, **kw)
        assert cu.cuCtxGetCurrent(C.byref(cur)) == 0 and cur.value == own.value, "the caller's context is not current after %s" % fn
        return out

    kv = O.gen_c2(0, 50000, seed=5)
    s = call(T.GpuSorter, P, fixed=(16, 64), device=0)
    call(s.collect_fixed, kv)
    out = call(s.flush_to_memory)[0]
    call(s.close)
    buf = call(T.PeerBuffer, 1 << 20, device=0)
    call(buf.close)
    assert bytes(out) == O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, 64)["file_out"]
    assert cu.cuCtxDestroy_v2(own) == 0
    print("own-context ok")


def test_the_callers_own_context_is_current_after_every_call():
    _worker("own-context")


def _no_context_worker():
    """a thread that never used CUDA sorts on device 1: no context appears on device 0"""
    cu = _cuda_driver()
    assert not _primary_context_active(cu, 0)
    with T.GpuSorter(P, fixed=(16, 64), device=1) as s:
        s.collect_fixed(O.gen_c2(0, 50000, seed=5))
        s.flush_to_memory()
    assert _primary_context_active(cu, 1)
    assert not _primary_context_active(cu, 0), "a call on device 1 created a context on device 0"
    print("no-context ok")


def test_a_thread_without_a_context_gets_none_on_device_0():
    _need_two_devices()
    _worker("no-context")


# ------------------------------------------------------------------------------------------------ bad ordinals
def test_bad_device_ordinals():
    """handle and device-argument calls refuse an ordinal outside [0, device count) before touching a device"""
    dev = torch.device("cuda", 0)
    seg = O.write_ifile([(b"k", b"v")])[0]
    src = torch.frombuffer(bytearray(seg), dtype=torch.uint8).to(dev)
    dst = torch.zeros(len(seg) + 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    rng = [(src.data_ptr(), dst.data_ptr(), len(seg))]
    index = np.array([[0, len(seg) - 4, len(seg)]], dtype=np.int64)
    calls = [lambda d: T.GpuSorter(P, device=d), lambda d: T.GpuMerger([seg], device=d), lambda d: T.PeerBuffer(16, device=d),
             lambda d: T.fetch_ranges(rng, device=d), lambda d: T.fetch_segments_verified(rng, device=d),
             lambda d: native.shuffle_serve(src.data_ptr(), index, "m", 0, 1, device=d)]
    for d in (-1, T._lib.load().tezgpu_device_count()):
        for call in calls:
            with pytest.raises(TezGpuError, match="bad device ordinal") as e:
                call(d)
            assert e.value.code == T.E_INVALID
    assert dst.count_nonzero().item() == 0


if __name__ == "__main__":
    workers = {"first-touch": _first_touch_worker, "own-context": _own_context_worker, "no-context": _no_context_worker}
    workers[sys.argv[1]]()

"""Device budgets without a device: tez.runtime.gpu.merge.device.budget.mb validation, the new symbols, and the argument
checks of tezgpu_decode_segments, which has no CPU fallback."""
import ctypes as C

import pytest

import tez_b200 as T
from tez_b200 import _lib
from tez_b200.native import make_conf
from tez_b200.runtime_library import (INT_WRITABLE, TEXT, InputContext, OrderedGroupedKVInput, OrderedPartitionedKVOutput,
                                      OutputContext, UnorderedKVInput)
from tez_b200._lib import TezGpuError
from oracle import tez_oracle as O
import codec_model as CM

E_INVALID, E_CUDA, E_UNSUPPORTED = -1, -2, -6
KEY = "tez.runtime.gpu.merge.device.budget.mb"
CONF = {"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE}


def _plain_seg():
    return O.write_ifile([(b"\x01a", b"\x00\x00\x00\x01"), (b"\x01b", b"\x00\x00\x00\x02")])[0]


def _decode(segs, raw, codec=T.CODEC_DEFAULT, budget=64 << 20, flags=T.SEG_HAS_HEADER, outs=None, conf=True):
    """tezgpu_decode_segments through ctypes; outs[i] None passes a NULL output.  Returns (rc, message)."""
    L = _lib.load()
    keep = [bytes(s) for s in segs]
    arr = (_lib.Segment * max(1, len(keep)))()
    for i, s in enumerate(keep):
        arr[i].data = C.cast(C.c_char_p(s), C.c_void_p)
        arr[i].len = len(s)
        arr[i].flags = flags
    bufs = [C.create_string_buffer(max(1, r + 4)) for r in (raw or [0] * len(keep))]
    out = (C.c_void_p * max(1, len(keep)))()
    for i in range(len(keep)):
        out[i] = None if outs is not None and outs[i] is None else C.cast(bufs[i], C.c_void_p)
    rl = None if raw is None else (C.c_int64 * len(raw))(*raw)
    cf = make_conf(1, partitioner=T.PART_GIVEN)
    peak = C.c_uint64()
    rc = L.tezgpu_decode_segments(C.byref(cf) if conf else None, arr, rl, len(keep), codec, budget, out, C.byref(peak))
    return rc, L.tezgpu_last_error().decode()


@pytest.mark.parametrize("value", [1, 15, -1])
def test_budget_key_below_the_floor_fails_at_initialize(tmp_path, value):
    conf = dict(CONF, **{KEY: value})
    for make in (lambda: OrderedGroupedKVInput(InputContext(conf, str(tmp_path)), 1),
                 lambda: UnorderedKVInput(InputContext(conf, str(tmp_path)), 1),
                 lambda: OrderedPartitionedKVOutput(OutputContext(conf, str(tmp_path)), 2)):
        with pytest.raises(TezGpuError) as e:
            make().initialize()
        assert e.value.code == E_INVALID and KEY in str(e.value) and str(value) in str(e.value)


@pytest.mark.parametrize("value", [0, 16, 4096])
def test_budget_key_accepted(tmp_path, value):
    conf = dict(CONF, **{KEY: value})
    inp = OrderedGroupedKVInput(InputContext(conf, str(tmp_path)), 1)
    inp.initialize()
    assert inp.merge_info() == (0, 0, 0)   # no merge has run
    out = OrderedPartitionedKVOutput(OutputContext(conf, str(tmp_path)), 2)
    out.initialize()
    assert out.merge_info() == (0, 0, 0)


def test_new_symbols_resolve():
    L = _lib.load()
    for name in ("tezgpu_decode_segments", "tezrt_input_merge_info", "tezrt_output_merge_info"):
        assert getattr(L, name) is not None


def test_decode_argument_checks():
    plain = _plain_seg()
    z, raw = CM.compressed_segment(CM.body_of(plain))
    assert _decode([z], [raw], conf=False)[0] == E_INVALID
    for codec in (7, T.CODEC_NONE, -1):
        rc, msg = _decode([z], [raw], codec=codec)
        assert rc == E_UNSUPPORTED and "codec %d" % codec in msg
    rc, msg = _decode([z], [raw], budget=(16 << 20) - 1)
    assert rc == E_INVALID and "below the floor" in msg
    rc, msg = _decode([z], None)
    assert rc == E_INVALID and "raw_len" in msg
    rc, msg = _decode([z], [raw], flags=T.SEG_HAS_HEADER | T.SEG_DEVICE)
    assert rc == E_INVALID and "host segments only" in msg
    assert _decode([plain, z], [len(plain) - 4, raw], outs=[None, 1])[0] in (0, E_CUDA)   # plain: out may be NULL
    rc, msg = _decode([plain, z], [len(plain) - 4, raw], outs=[1, None])
    assert rc == E_INVALID and "segment 1 is compressed" in msg and "out[1]" in msg


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
def test_decode_has_no_cpu_fallback():
    z, raw = CM.compressed_segment(CM.body_of(_plain_seg()))
    for codec_seg in ([z], [_plain_seg()], []):
        rc, msg = _decode(codec_seg, [raw] * len(codec_seg))
        assert rc == E_CUDA and "no CUDA device" in msg
    with pytest.raises(IOError):
        T.native.decode_segments([z], [raw], T.CODEC_DEFAULT, 64 << 20)

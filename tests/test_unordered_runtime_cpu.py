"""CPU checks of the unordered edge: the checksum algebra of tezgpu_concat_open (host emulation against zlib), the
refusals of UnorderedPartitionedKVOutput that come before any device call, and the model the GPU tests use."""
import ctypes as C
import random
import zlib

import pytest

from oracle import tez_oracle as O
import tez_b200 as T
from tez_b200 import _lib
from tez_b200.runtime_library import OutputContext, UnorderedKVOutput, UnorderedPartitionedKVOutput

import unordered_model as UM


def _emulate(bodies):
    L = _lib.load()
    arrs = [(C.c_uint8 * max(1, len(b))).from_buffer_copy(b.ljust(1, b"\0")) for b in bodies]
    ptrs = (C.c_void_p * max(1, len(bodies)))(*[C.addressof(a) for a in arrs])
    lens = (C.c_uint64 * max(1, len(bodies)))(*[len(b) for b in bodies])
    crc = C.c_uint32()
    _lib.check(L.tezgpu_debug_crc_concat_emulate(ptrs, lens, len(bodies), C.byref(crc)))
    return crc.value


def _expected(bodies):
    return zlib.crc32(b"".join(b[:-2] for b in bodies) + b"\xff\xff")


@pytest.mark.parametrize("case", ["one_empty", "all_empty", "one_byte_records", "mixed", "large"])
def test_crc_concat_emulate_equals_zlib(case):
    rng = random.Random(zlib.crc32(case.encode()))
    eof = b"\xff\xff"
    if case == "one_empty":
        bodies = [eof]
    elif case == "all_empty":
        bodies = [eof] * 7
    elif case == "one_byte_records":
        bodies = [bytes([rng.randrange(256)]) + eof for _ in range(300)]
    elif case == "mixed":
        bodies = [rng.randbytes(rng.choice([0, 1, 2, 3, 15, 16, 17, 4095, 4096, 65537])) + eof for _ in range(120)]
    else:
        bodies = [rng.randbytes(rng.randint(1, 4 << 20)) + eof for _ in range(3)] + [eof, rng.randbytes(5) + eof]
    assert _emulate(bodies) == _expected(bodies)


@pytest.mark.parametrize("n", [1, 2, 9, 64, 300])
def test_crc_concat_emulate_segment_counts(n):
    rng = random.Random(n)
    bodies = [rng.randbytes(rng.randint(0, 3000)) + b"\xff\xff" for _ in range(n)]
    assert _emulate(bodies) == _expected(bodies)


def test_crc_concat_emulate_refuses_a_body_without_eof_marker():
    with pytest.raises(_lib.TezGpuError) as e:
        _emulate([b"ab\xff\xff", b"abc\xff"])
    assert e.value.code == T.E_FORMAT and "body 1" in str(e.value)


@pytest.mark.parametrize("cls", [UnorderedPartitionedKVOutput, UnorderedKVOutput])
@pytest.mark.parametrize("mb", [0, -1])
def test_buffer_size_mb_must_be_positive(tmp_path, cls, mb):
    ctx = OutputContext(conf={"tez.runtime.unordered.output.buffer.size-mb": mb}, work_dir=str(tmp_path))
    out = cls(ctx, 4)
    with pytest.raises(_lib.TezGpuError) as e:
        out.initialize()
    assert e.value.code == T.E_INVALID and "tez.runtime.unordered.output.buffer.size-mb should be larger than 0" in str(e.value)


def test_buffer_size_mb_is_the_memory_request(tmp_path):
    ctx = OutputContext(conf={"tez.runtime.unordered.output.buffer.size-mb": 7}, work_dir=str(tmp_path))
    out = UnorderedPartitionedKVOutput(ctx, 4)
    out.initialize()
    assert out.requested_memory == 7 << 20


def test_model_matches_dict_of_lists():
    rng = random.Random(11)
    P = 5
    segs, parts, want = [], [], {}
    for p in range(P):
        for _ in range(rng.randint(0, 3)):
            recs = [(rng.randbytes(rng.randint(0, 9)), rng.randbytes(rng.randint(0, 30))) for _ in range(rng.randint(0, 6))]
            segs.append(O.write_ifile(recs)[0])
            parts.append(p)
            want.setdefault(p, []).extend(recs)
    out, index = UM.concat_file(segs, parts, P)
    got = UM.partition_records(out, index)
    assert got == {p: r for p, r in want.items() if r}
    for p in range(P):
        if not want.get(p):
            assert index[p] == (0, 0, 0)
    pos = 0
    for p in range(P):
        if index[p][2]:
            assert index[p][0] == pos and out[pos:pos + 4] == b"TIF\x00"
            pos += index[p][2]
    assert pos == len(out)

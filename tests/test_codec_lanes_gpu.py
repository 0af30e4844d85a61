"""GPU: the compressed-segment readers of DefaultCodec, Lz4Codec and ZStandardCodec on their 32-lane paths.

The CPU suites check the decoders through the host emulation, which runs the same code with one lane.  Here the device
decodes the crafted streams of codec_lanes_model through decode_segments (TIF\\x00 + body + CRC-32 of the body, no
record parsing), so the lane-only code runs: overlapping match copies in rounds of min(distance, 32) bytes, the lane-0
branch of short copies, strided stored blocks, literal runs and raw / RLE blocks, the lane-split Adler-32, zstd literals
staged at the end of a block's room, and the unit pass (one warp per LZ4 block or zstd frame) with its fallback to the
serial pass.  Every image must equal the library's bytes; every corrupted stream must get the emulation's verdict: the
same bytes, or a refusal with the same reason."""
import time
import zlib

import numpy as np
import pytest
import torch

import tez_b200 as T
from tez_b200 import native
from tez_b200._lib import TezGpuError
import codec_lanes_model as M
import codec_model as CM
import lz4_model as L4
import zstd_model as ZS

pytestmark = pytest.mark.gpu
CODECS = ["default", "lz4", "zstd"]
WARPS = {"default": 4, "lz4": 4, "zstd": 2}      # warps per CTA of k_zinflate, k_l4blocks / k_l4serial, k_zsframes / k_zsserial
BUDGET = 16 << 30
GiB = 1 << 30
_CACHE = {}


def _cases(codec):
    if ("cases", codec) not in _CACHE:
        _CACHE[("cases", codec)] = M.cases(codec)
    return _CACHE[("cases", codec)]


def _corpus(codec):
    if ("corpus", codec) not in _CACHE:
        _CACHE[("corpus", codec)] = M.corrupt(codec, n=1000)
    return _CACHE[("corpus", codec)]


def _decode(codec, items):
    """items [(stream, body length)] decoded in one call: the images"""
    segs = [M.segment(z) for z, _ in items]
    imgs, _ = native.decode_segments(segs, [n + 4 for _, n in items], M.CODECS[codec], BUDGET)
    return imgs


def _refusal(codec, items):
    with pytest.raises(TezGpuError) as e:
        _decode(codec, items)
    assert e.value.code == T.E_FORMAT, str(e.value)
    return str(e.value)


# ------------------------------------------------------------------------------------------------ well-formed streams
@pytest.mark.parametrize("order", ["forward", "reversed", "not_a_warp_multiple"])
@pytest.mark.parametrize("codec", CODECS)
def test_crafted_streams_decode_to_the_library_bytes(codec, order):
    cs = list(_cases(codec))
    if order == "reversed":
        cs = cs[::-1]
    elif order == "not_a_warp_multiple":
        k = len(cs) - 1
        while k % WARPS[codec] == 0:
            k -= 1
        cs = cs[1:k + 1]
    assert {c.path for c in cs} == ({"serial"} if codec == "default" else {"unit", "serial"})
    imgs = _decode(codec, [(c.stream, len(c.body)) for c in cs])
    bad = [c.name for c, img in zip(cs, imgs) if img != M.image(c.body)]
    assert not bad, bad


def test_lz4_short_block_leaves_the_unit_pass_and_is_refused():
    """a one-chunk block that decodes validly to one byte fewer than its raw length: the unit pass sees no error in the
    chunk, so only its length check sends the segment to the serial pass, which refuses it"""
    z, raw = M.lz4_short_block()
    _, reason = M.emulate("lz4", z, raw)
    assert reason == "truncated block header"
    assert _refusal("lz4", [(z, raw)]).endswith("compressed segment 0: " + reason)
    good = [c for c in _cases("lz4") if c.path == "unit"][:6]
    items = [(c.stream, len(c.body)) for c in good]
    assert _refusal("lz4", items[:3] + [(z, raw)] + items[3:]).endswith("compressed segment 3: " + reason)


# ------------------------------------------------------------------------------------------------ corrupted streams
@pytest.mark.parametrize("codec", CODECS)
def test_corrupted_streams_the_emulation_accepts_decode_to_its_bytes(codec):
    ok = [(z, n, got) for z, n, got, _ in _corpus(codec) if got is not None]
    assert ok
    for a in range(0, len(ok), 200):
        part = ok[a:a + 200]
        imgs = _decode(codec, [(z, n) for z, n, _ in part])
        bad = [a + i for i, ((_, _, got), img) in enumerate(zip(part, imgs)) if img != M.image(got)]
        assert not bad, bad


@pytest.mark.parametrize("codec", CODECS)
def test_corrupted_streams_the_emulation_refuses_fail_with_its_reason(codec):
    refused = [(z, n, reason) for z, n, got, reason in _corpus(codec) if got is None]
    assert refused
    wrong = []
    for i, (z, n, reason) in enumerate(refused):
        try:
            _decode(codec, [(z, n)])
            wrong.append((i, "accepted", reason))
        except TezGpuError as e:
            if e.code != T.E_FORMAT or not str(e).endswith("compressed segment 0: " + reason):
                wrong.append((i, str(e), reason))
    assert not wrong, wrong[:10]


def _malformed(codec):
    """the malformed-stream tables of the CPU suites: [(name, stream, body length)]"""
    if codec == "default":
        cases, n = CM.malformed()
        return [(k, z, n) for k, z in sorted(cases.items())]
    if codec == "lz4":
        return [(k, z, n) for k, (z, n) in sorted(L4.malformed().items())]
    return [(k, z, n) for k, (z, n, _) in sorted(ZS.malformed().items())]


@pytest.mark.parametrize("codec", CODECS)
def test_malformed_tables_fail_on_the_device_with_the_emulation_reason(codec):
    seen = 0
    for name, z, n in _malformed(codec):
        if len(M.segment(z)) < 10:
            continue          # shorter than a compressed segment's header and trailer: not taken as compressed
        got, reason = M.emulate(codec, z, n)
        assert got is None, name
        msg = _refusal(codec, [(z, n)])
        assert msg.endswith("compressed segment 0: " + reason), (name, msg, reason)
        seen += 1
    assert seen >= len(_malformed(codec)) - 1


@pytest.mark.parametrize("codec", CODECS)
def test_one_bad_segment_in_a_batch_is_named(codec):
    good = [(c.stream, len(c.body)) for c in _cases(codec)[:11]]
    z, n, _, reason = next(m for m in _corpus(codec) if m[2] is None)
    for k in (0, 5, 11):
        items = good[:k] + [(z, n)] + good[k:]
        assert _refusal(codec, items).endswith("compressed segment %d: %s" % (k, reason))


# ------------------------------------------------------------------------------------------------ output past 4 GiB
LARGE_BODY = (1 << 32) + 4099
# On one H100 80GB HBM3 the call's peak was 4.05 GiB of device memory (staged stream and image); the host holds the
# 4 GiB image twice while decode_segments copies it out, plus the 46 MB stream and a 64 MiB comparison tile.
LARGE_DEVICE_NEED = 9 * GiB // 2
LARGE_HOST_NEED = 9 * GiB


def _host_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def test_default_codec_body_past_4_gib_in_one_serial_stream():
    """One zlib member of 2^32 + 4,099 bytes: a 4 KiB random block, then matches of 258 bytes at distance 4,096 (never
    distance 1, which would copy one byte per round).  Output offsets past 2^32 in a single warp."""
    free, _ = torch.cuda.mem_get_info(0)
    if free < LARGE_DEVICE_NEED or _host_available() < LARGE_HOST_NEED:
        pytest.skip("needs %.0f GiB free on cuda:0 and %.0f GiB of host memory; %.1f / %.1f GiB available"
                    % (LARGE_DEVICE_NEED / GiB, LARGE_HOST_NEED / GiB, free / GiB, _host_available() / GiB))
    block = np.random.default_rng(4096).integers(0, 256, 4096, dtype=np.uint8).tobytes()
    z = M.deflate_large(block, LARGE_BODY)
    t0 = time.perf_counter()
    imgs, peak = native.decode_segments([M.segment(z)], [LARGE_BODY + 4], T.CODEC_DEFAULT, BUDGET)
    dt = time.perf_counter() - t0
    img = imgs[0]
    print("\nlarge DefaultCodec segment: %d compressed bytes, %.1f s, peak device bytes %.2f GiB" % (len(z), dt, peak / GiB))
    assert len(img) == LARGE_BODY + 8 and img[:4] == b"TIF\x00"
    big = np.tile(np.frombuffer(block, dtype=np.uint8), 16384).tobytes()       # 64 MiB, a whole number of blocks
    view = memoryview(img)[4:4 + LARGE_BODY]
    crc, bad = 0, []
    for a in range(0, LARGE_BODY, len(big)):
        part = view[a:a + len(big)]
        crc = zlib.crc32(part, crc)
        if part != big[:len(part)]:
            bad.append(a)
    assert not bad, bad[:5]
    assert int.from_bytes(img[-4:], "big") == crc

"""GPU: the three device walkers of IFile bodies agree on edge inputs.  Every case is merged three ways:

  default   the window parser (parse_windows.cuh), which hands malformed segments to the sequential walker;
  serial    the sequential walker k_parse_segments alone (TEZGPU_PARSE_SERIAL=1, latched per process: a subprocess
            runs this file as a script, `python tests/test_ifile_walkers_gpu.py serial-walker`, and prints its results);
  bounded   a bounded merge at the 16 MiB floor, whose window scan and cut (k_step_walk) read every segment before
            the Merger does; the valid filler segments make the inputs too large for its one-step shortcut.

Valid cases must give the oracle's records, written segment and counts on every path; malformed ones the same
TEZGPU_E_FORMAT message on every path, naming the caller's segment index."""
import functools
import hashlib
import json
import os
import subprocess
import sys
import zlib

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200._lib import TezGpuError  # noqa: E402

pytestmark = pytest.mark.gpu

FLOOR = 16 << 20
HDR = 4
STAGE = 4096       # the sequential walker's and the bounded walk's shared-memory staging window (ifile_walk.cuh)
WINDOW = 32768     # the window parser's window (parse_windows.cuh)


def _filler():
    """about 200 KB of valid segments"""
    segs = []
    for s in range(4):
        keys = sorted(b"f%02d%06d" % (s, (i * 7919) % 100000) for i in range(1700))
        segs.append(O.write_ifile([(k, b"filler-%02d-%010d" % (s, i)) for i, k in enumerate(keys)])[0])
    return segs


def _framed(body):
    return b"TIF\0" + body + zlib.crc32(body).to_bytes(4, "big")


def _rec(k, v):
    return O.vint(len(k)) + O.vint(len(v)) + k + v


def _rle_segment(tag, lead):
    """key "a<tag>" with a value of `lead` bytes, a REPEAT_KEY run of "bb", then "cc" (its V_END_MARKER FD, key length
    and 2-byte value length vint) and a run of "dd".  Values are a function of their key: the order inside a group of
    equal keys from several segments is not part of the contract."""
    recs = [(b"a" + tag, b"x" * lead)] + [(b"bb", b"bb-value")] * 3
    recs += [(b"cc", b"c" * 200), (b"dd", b"dd"), (b"dd", b"dd"), (b"ee", b"e")]
    return O.write_ifile(recs, rle=True)[0]


def _marker_at(target, tag):
    """an RLE segment whose V_END_MARKER is at segment offset `target`, or None where the vint width of the lead
    value's length skips that offset"""
    pat = b"\xfd" + O.vint(2) + O.vint(200) + b"cc"
    lead = max(0, target - 50)
    for _ in range(4):
        seg = _rle_segment(tag, lead)
        at = seg.index(pat)
        if at == target:
            return seg
        lead += target - at
        if lead < 0:
            return None
    return None


@functools.lru_cache(maxsize=None)
def cases():
    """name -> (segments, expected): expected is the segment list the oracle merges, or the index of the malformed
    segment"""
    fill = _filler()
    out = {}
    rle = []
    for edge in (HDR + STAGE, HDR + WINDOW, HDR + 2 * STAGE):
        for d in range(-6, 3):
            seg = _marker_at(edge + d, b"%05d" % (edge + d))
            assert seg is not None and seg[edge + d] == 0xFD
            rle.append(seg)
    out["rle_markers_on_window_edges"] = (fill + rle, fill + rle)
    good = _rec(b"k1", b"v1") + _rec(b"k2", b"v2")
    eof = b"\xff\xff"
    out["value_past_body_end"] = (fill + [_framed(good + O.vint(2) + O.vint(100) + b"k3" + b"v" * 10)], len(fill))
    out["vint_past_body_end"] = (fill[:2] + [_framed(good + b"\x8e\x01")] + fill[2:], 2)
    out["body_starts_with_repeat"] = (fill[:2] + [_framed(b"\xfe" + O.vint(1) + b"v" + b"\xfd" + eof)] + fill[2:], 2)
    out["key_length_minus_4"] = (fill[:2] + [_framed(good + b"\xfc" + O.vint(1) + b"v" + eof)] + fill[2:], 2)
    big = O.vint(2 ** 31)
    assert len(big) == 5
    out["length_above_2^31-1"] = (fill[:2] + [_framed(good + big + O.vint(1) + b"k" + b"v" + eof)] + fill[2:], 2)
    # EOF markers before the body end, followed by the bytes of more records: the reader stops at the first markers
    early = _framed(good + eof + _rec(b"k3", b"v3") + eof)
    out["eof_markers_before_the_body_end"] = (fill[:2] + [early] + fill[2:],
                                              fill[:2] + [O.write_ifile([(b"k1", b"v1"), (b"k2", b"v2")])[0]] + fill[2:])
    return out


def _digest(recs, seg, counts):
    h = hashlib.sha256()
    for k, v, same in recs:
        h.update(len(k).to_bytes(4, "little") + k + len(v).to_bytes(4, "little") + v + bytes([same]))
    return {"records": h.hexdigest(), "ifile": hashlib.sha256(seg).hexdigest(), "counts": list(counts)}


def run(segs, budget=None):
    """the merge's digest and parse mode, or {"error": message} when the open or a read raises"""
    try:
        with T.GpuMerger(segs, comparator=T.CMP_BYTES, device_budget=budget) as m:
            mode = m.parse_info()[0] if budget is None else None
            recs = list(m.records(batch_records=997, batch_bytes=1 << 16))
            if budget is not None:
                assert m.bounded_info()[0] >= 1
            seg = m.write_ifile(rle=False)[0]
            counts = m.counts()
    except TezGpuError as e:
        assert e.code == T.E_FORMAT, str(e)
        return {"error": str(e)}
    return dict(_digest(recs, seg, counts), mode=mode)


def expected(exp):
    if isinstance(exp, int):
        return {"error": "tezgpu error %d: malformed IFile segment %d" % (T.E_FORMAT, exp)}
    o = O.merge(exp, O.CMP_BYTES, factor=100)
    recs = o["records"]
    return _digest(recs, o["ifile"], (len(recs), sum(len(k) + len(v) for k, v, _ in recs)))


def _without_mode(r):
    return {k: v for k, v in r.items() if k != "mode"}


# the record-finding mode of the default path: the window parser, except where a segment is malformed or has EOF
# markers before its end -- the parser then hands the whole merge to the sequential walker
DEFAULT_MODE = {"rle_markers_on_window_edges": 1, "eof_markers_before_the_body_end": 2}


@pytest.mark.parametrize("name", sorted(cases()))
def test_window_parser_and_bounded_walk(name):
    segs, exp = cases()[name]
    want = expected(exp)
    got = run(segs)
    assert _without_mode(got) == want, name
    if "error" not in want:
        assert got["mode"] == DEFAULT_MODE[name]
    assert sum(len(s) for s in segs) > 150000
    assert _without_mode(run(segs, budget=FLOOR)) == want, name


def test_sequential_walker():
    env = dict(os.environ, TEZGPU_PARSE_SERIAL="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "serial-walker"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    serial = json.loads(r.stdout.strip().splitlines()[-1])
    cs = cases()
    assert sorted(serial) == sorted(cs)
    for name, (segs, exp) in cs.items():
        want = expected(exp)
        assert _without_mode(serial[name]) == want, name
        if "error" not in want:
            assert serial[name]["mode"] == 2


if __name__ == "__main__":
    if sys.argv[1:] == ["serial-walker"]:
        print(json.dumps({name: run(segs) for name, (segs, _) in cases().items()}))

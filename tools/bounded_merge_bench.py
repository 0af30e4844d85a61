"""Merges larger than a device budget: tezgpu_merge_open_bounded + write_ifile over config-3 segments in pinned host
memory, at several budgets and unbounded (one-step tezgpu_merge_open), plain and Lz4Codec-compressed.  One JSON line
per run.

  plain: the segments are merged as they are (key-range steps at a budget, one step without).
  lz4:   the same records as Lz4Codec segments (written by the device writer); a budgeted run decodes them with
         tezgpu_decode_segments under the budget, then merges the images in steps; the unbounded run is
         tezgpu_merge_open_codec, which decodes and merges in one step.

Times: host clock around calls that end in a device synchronise (open, decode and write all return synchronised), one
warm-up run per case first, --reps runs per case.  h2d_gbps is the step loop's uploaded bytes over the run time, next
to the pinned H2D copy rate measured in the same process (tools/pcie_probe.py's measurement).  Parity, outside the
timed region: every run's output has the CRC-32 trailer of its body, every uncompressed output the unbounded plain run's
bytes (trailer and length; the one-step codec merge writes an Lz4Codec segment), and a sample of the
segments merged under a 64 MiB budget is byte-exact against the oracle's TezMerger.  The card name and power limit are
read in the same run.

  --write-codec none,default,lz4,zstd,snappy: instead, the bounded merge's compressed write (write_codec_arm).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200 import _lib, native  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def pinned(a):
    """a copy of the uint8 array in pinned host memory, as a numpy view"""
    t = torch.empty(a.size, dtype=torch.uint8, pin_memory=True)
    t.numpy()[:] = a
    return t.numpy()


def h2d_ceiling(nbytes=1 << 30, reps=5):
    """pinned host -> device copy rate, GB/s"""
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    return nbytes * reps / (time.perf_counter() - t0) / 1e9


def write(m, out):
    """tezgpu_merge_write_ifile into out, written as config 3 writes (rle = 0); returns the segment's length"""
    raw, part = C.c_int64(), C.c_int64()
    _lib.check(_lib.load().tezgpu_merge_write_ifile(m.h, None, out.ctypes.data, out.size, 0, C.byref(raw), C.byref(part), None))
    return part.value


def decode(segs, raws, budget, imgs):
    """tezgpu_decode_segments of the Lz4Codec segments into the host buffers imgs; returns the peak device bytes"""
    arr = (_lib.Segment * len(segs))()
    out = (C.c_void_p * len(segs))()
    for i, (a, img) in enumerate(zip(segs, imgs)):
        arr[i].data, arr[i].len, arr[i].flags = a.ctypes.data, a.size, T.SEG_HAS_HEADER
        out[i] = img.ctypes.data
    rl = (C.c_int64 * len(raws))(*raws)
    conf = native.make_conf(1, partitioner=T.PART_GIVEN)
    peak = C.c_uint64()
    _lib.check(_lib.load().tezgpu_decode_segments(C.byref(conf), arr, rl, len(segs), T.CODEC_LZ4, budget, out, C.byref(peak)))
    return peak.value


def run(variant, budget, segs, raws, out, imgs):
    """one merge: (seconds, output length, steps, h2d bytes, peak device bytes)"""
    t0 = time.perf_counter()
    decode_peak = 0
    if variant == "lz4" and budget:
        decode_peak = decode(segs, raws, budget, imgs)
        segs = imgs
    if budget:
        m = T.GpuMerger(segs, comparator=T.CMP_TEXT, device_budget=budget)
    elif variant == "lz4":
        m = T.GpuMerger(segs, comparator=T.CMP_TEXT, codec=T.CODEC_LZ4, raw_lens=raws)
    else:
        m = T.GpuMerger(segs, comparator=T.CMP_TEXT)
    with m:
        n = write(m, out)
        secs = time.perf_counter() - t0
        steps, peak, h2d = m.bounded_info() if budget else (1, 0, sum(s.size for s in segs))
    return secs, n, steps, h2d, max(peak, decode_peak)


WRITE_CODECS = {"none": None, "default": T.CODEC_DEFAULT, "lz4": T.CODEC_LZ4, "zstd": T.CODEC_ZSTD, "snappy": T.CODEC_SNAPPY}


def write_codec_arm(args, plain, in_bytes, nseg, nrec, out):
    """--write-codec: the compressed write of the bounded merge (tezgpu_merge_open_bounded_write_codec) at every budget,
    beside the bounded uncompressed write at the same budgets and a one-step tezgpu_merge_open_codec write of the
    whole input (which fits the device unbounded).  Times: host clock around open + write_ifile (rle = 0), one
    warm-up run per arm, --reps runs.  GB/s are of the uncompressed output (rawLength); ratio = rawLength / partLength.
    Parity: every bounded compressed write equals the one-step write of its codec byte for byte."""
    name = card()
    budgets = sorted((int(float(g) * (1 << 30)) for g in args.budgets_gib.split(",")), reverse=True)
    for arm in [c for c in args.write_codec.split(",") if c]:
        codec = WRITE_CODECS[arm]
        ref, warm = None, False
        for budget in ([0] if codec else []) + budgets:
            def once():
                t0 = time.perf_counter()
                if budget:
                    m = T.GpuMerger(plain, comparator=T.CMP_TEXT, device_budget=budget, write_codec=codec)
                else:
                    m = T.GpuMerger(plain, comparator=T.CMP_TEXT, codec=codec)
                with m:
                    raw, part = C.c_int64(), C.c_int64()
                    _lib.check(_lib.load().tezgpu_merge_write_ifile(m.h, None, out.ctypes.data, out.size, 0, C.byref(raw),
                                                                    C.byref(part), None))
                    secs = time.perf_counter() - t0
                    steps, peak, _ = m.bounded_info() if budget else (1, None, None)
                return secs, raw.value, part.value, steps, peak
            times = []
            try:
                if not warm:
                    once()                                               # warm-up
                    warm = True
                for _ in range(args.reps):
                    secs, raw, part, steps, peak = once()
                    times.append(secs)
            except _lib.TezGpuError as e:   # the one-step write of the whole input needs more than the device holds
                if budget:
                    raise
                print(json.dumps({"bench": "bounded_merge_write_codec", "write_codec": arm, "open": "open_codec one step",
                                  "input_bytes": in_bytes, "error": str(e), "card": name}), flush=True)
                continue
            digest = zlib.crc32(out[:part])
            if ref is None:
                ref = digest
            s = sum(times) / len(times)
            print(json.dumps({
                "bench": "bounded_merge_write_codec", "write_codec": arm,
                "open": "bounded_write_codec" if (budget and codec) else ("bounded" if budget else "open_codec one step"),
                "budget_bytes": budget or None, "input_bytes": in_bytes, "segments": nseg, "records": int(sum(nrec)),
                "raw_bytes": raw, "written_bytes": part, "crc32": digest, "ratio": round(raw / part, 3),
                "ms_per_run": round(s * 1e3, 1), "ms_runs": [round(t * 1e3, 1) for t in times],
                "raw_gbps": round(raw / s / 1e9, 3), "steps": steps, "peak_device_bytes": peak, "card": name,
                "parity": {"same_bytes_as_one_step_write": digest == ref if codec else None}}), flush=True)
            assert not codec or digest == ref, "bounded compressed write differs from the one-step write"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=8.0, help="input bytes in GiB (config-3 segments)")
    ap.add_argument("--segment-mb", type=int, default=32)
    ap.add_argument("--budgets-gib", default="1,2,4")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample-segments", type=int, default=8)
    ap.add_argument("--write-codec", default="",
                    help="comma-separated arms (none,default,lz4,zstd,snappy; none = the bounded uncompressed write): measure "
                         "the bounded merge's compressed write instead of the plain and lz4 variants")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bounded_merge_bench measures the device path: no GPU, no numbers"
    torch.cuda.set_device(0)
    nseg = max(2, int(args.gib * 1024 / args.segment_mb))
    gen, nrec = O.gen_c3_segments(nseg, args.segment_mb << 20, seed=3, threads=min(os.cpu_count() or 1, 64))
    plain = [pinned(a) for a in gen]
    del gen
    in_bytes = sum(a.size for a in plain)
    kv_bytes = in_bytes - 10 * nseg - 2 * sum(nrec)
    if args.write_codec:
        write_codec_arm(args, plain, in_bytes, nseg, nrec, np.empty(in_bytes + (1 << 20), dtype=np.uint8))
        return
    # the same records as Lz4Codec segments, written by the device writer (a one-segment merge with the codec)
    lz4, raws = [], []
    for a in plain:
        with T.GpuMerger([a], comparator=T.CMP_TEXT, codec=T.CODEC_LZ4) as m:
            seg, raw, _, _ = m.write_ifile(rle=False)
        lz4.append(pinned(np.frombuffer(seg, dtype=np.uint8)))
        raws.append(raw)
    lz4_bytes = sum(a.size for a in lz4)
    out = np.empty(in_bytes + (1 << 20), dtype=np.uint8)
    imgs = [pinned(np.zeros(r + 4, dtype=np.uint8)) for r in raws]   # where a budgeted lz4 run decodes to
    ceiling = round(h2d_ceiling(), 2)
    budgets = [int(float(g) * (1 << 30)) for g in args.budgets_gib.split(",")] + [0]
    name = card()
    ref = None
    for variant, segs in (("plain", plain), ("lz4", lz4)):
        for budget in sorted(budgets, key=lambda b: b or 1 << 62, reverse=True):
            run(variant, budget, segs, raws, out, imgs)                   # warm-up
            times = []
            for _ in range(args.reps):
                secs, n, steps, h2d, peak = run(variant, budget, segs, raws, out, imgs)
                times.append(secs)
            crc_ok = int.from_bytes(out[n - 4:n].tobytes(), "big") == zlib.crc32(out[4:n - 4])
            # the one-step codec merge writes through its codec: only the uncompressed outputs compare
            compressed = variant == "lz4" and not budget
            sig = None if compressed else (n, out[n - 4:n].tobytes())
            if ref is None:
                ref = sig
            s = sum(times) / len(times)
            print(json.dumps({
                "bench": "bounded_merge", "variant": variant, "budget_bytes": budget or None,
                "input_bytes": in_bytes, "compressed_bytes": lz4_bytes if variant == "lz4" else None, "segments": nseg,
                "records": int(sum(nrec)), "ms_per_run": round(s * 1e3, 1), "ms_runs": [round(t * 1e3, 1) for t in times],
                "steps": steps, "h2d_bytes": h2d, "peak_device_bytes": peak or None,
                "kv_gbps": round(kv_bytes / s / 1e9, 3), "h2d_gbps": round(h2d / s / 1e9, 3) if budget else None,
                "h2d_ceiling_gbps": ceiling, "card": name,
                "output": "Lz4Codec segment" if compressed else "uncompressed segment",
                "parity": {"crc32_of_full_output_matches_zlib": bool(crc_ok),
                           "same_output_as_unbounded_plain_run": None if compressed else sig == ref}}),
                flush=True)
            assert crc_ok and (compressed or sig == ref), "bounded merge output differs"
    # byte-exact against the oracle on a sample, merged in steps under a small budget
    k = max(2, min(nseg, args.sample_segments))
    exp, _, _ = O.merge_ifile([a for a in plain[:k]], O.CMP_TEXT, factor=100)
    with T.GpuMerger(plain[:k], comparator=T.CMP_TEXT, device_budget=64 << 20) as m:
        n = write(m, out)
        steps = m.bounded_info()[0]
    exact = bool(n == exp.size and np.array_equal(out[:n], exp))
    print(json.dumps({"bench": "bounded_merge", "parity": "sample", "segments": k, "budget_bytes": 64 << 20, "steps": steps,
                      "bit_exact_vs_oracle": exact}))
    assert exact and steps > 1


if __name__ == "__main__":
    main()

"""Final merge of an unordered edge on the device: tezgpu_concat_open against tezgpu_merge_open over the same segments.

Prints one JSON line per case:
  1. --spills spills x 64 partitions of config-2 records (16-byte key, 64-byte value), --spill-gb of records per spill
     (default 4 x 2 GB = 8 GB), write_partitions_device;
  2. --read-segments x 4 MiB Text segments (default 256) read through next_batch into host memory;
  3. case 1 with LZ4 and zstd inputs and output, at a quarter of case 1's records per spill (compressing the spills
     first is the slow part of the set-up, not of the measurement).
Times are medians of --reps runs of open + write (or open + the whole read), CUDA events around the host calls, so
they include the host side of the calls.  Rates are input bytes over that time; `concat_of_peak` is the bytes the
concatenating write moves (input read twice -- checksum at open, copy -- and output written once) over 3.35 TB/s.
"""
import argparse
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tez_b200 as T  # noqa: E402

PEAK = 3.35e12


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception:
        return torch.cuda.get_device_name(0)


def spills(n_spill, recs, P, codec):
    """device-resident unordered spills of random config-2 records: [(device buffer, index)]"""
    out = []
    for s in range(n_spill):
        kv = torch.randint(0, 256, (recs * 80,), dtype=torch.uint8, device="cuda", generator=torch.Generator("cuda").manual_seed(s))
        with T.GpuSorter(P, fixed=(16, 64), unordered=True, codec=codec) as srt:
            cap = int(recs * 84 * 1.05) + (1 << 20)   # every record framed, the codec's worst case, segment overhead
            buf = torch.empty(cap, dtype=torch.uint8, device="cuda")
            n, index, _ = srt.sort_device_fixed(kv.data_ptr(), recs, buf.data_ptr(), cap)
        out.append((buf, index))
        del kv
    return out


def timed(fn, reps):
    ts = []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts[1:]))


def case_final_merge(n_spill, recs, P, codec, reps, name):
    sp = spills(n_spill, recs, P, codec)
    segs, parts, raws = [], [], []
    for p in range(P):                        # mergeAll's order: current buffer (the last spill) first, then the others
        for s in [n_spill - 1] + list(range(n_spill - 1)):
            buf, index = sp[s]
            start, raw, part = (int(x) for x in index[p])
            if part:
                segs.append((buf.data_ptr() + start, part))
                parts.append(p)
                raws.append(raw)
    in_bytes = sum(n for _, n in segs)
    res = {}
    outputs = {}
    for mode in ("concat", "merge"):
        m = T.GpuMerger(segs, device_ptrs=True, partitions=parts, num_partitions=P, codec=codec, raw_lens=raws,
                        concat=mode == "concat", verified=[False] * len(segs))
        m.close()
        cap = None

        def run():
            nonlocal cap
            mm = T.GpuMerger(segs, device_ptrs=True, partitions=parts, num_partitions=P, codec=codec, raw_lens=raws,
                             concat=mode == "concat")
            if cap is None:
                cap = mm.output_bound()
                outputs[mode] = torch.empty(cap, dtype=torch.uint8, device="cuda")
            n, index, _ = mm.write_partitions_device(outputs[mode].data_ptr(), cap)
            mm.close()
            res[mode + "_out"] = n
        res[mode + "_ms"] = timed(run, reps)
        del outputs[mode]
    moved = 2 * in_bytes + res["concat_out"]
    return {"case": name, "gpu": gpu_name(), "input_bytes": in_bytes, "segments": len(segs),
            "concat_ms": res["concat_ms"], "merge_ms": res["merge_ms"],
            "concat_GBps": in_bytes / res["concat_ms"] / 1e6, "merge_GBps": in_bytes / res["merge_ms"] / 1e6,
            "concat_of_peak": moved / (res["concat_ms"] * 1e-3) / PEAK, "speedup": res["merge_ms"] / res["concat_ms"]}


def text_segment(seg_bytes, seed):
    """one IFile segment of (Text "w" + 7 digits, IntWritable) records, built with numpy: 15 bytes a record"""
    rng = np.random.default_rng(seed)
    n = seg_bytes // 15
    a = np.empty((n, 15), dtype=np.uint8)
    a[:, 0], a[:, 1], a[:, 2], a[:, 3] = 9, 4, 8, ord("w")   # vint klen, vint vlen, Text length, "w"
    ids = rng.integers(0, 10 ** 7, n)
    for d in range(7):
        a[:, 4 + d] = 48 + (ids // 10 ** (6 - d)) % 10
    a[:, 11:15] = np.frombuffer(np.full(n, seed, dtype=">i4").tobytes(), dtype=np.uint8).reshape(n, 4)
    body = a.tobytes() + b"\xff\xff"
    return b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")


def case_read(nseg, seg_bytes, reps):
    segs = [text_segment(seg_bytes, s) for s in range(nseg)]
    res = {}
    for mode in ("concat", "merge"):
        def run():
            m = T.GpuMerger(segs, comparator=T.CMP_TEXT, concat=mode == "concat")
            buf = np.empty(64 << 20, dtype=np.uint8)
            idx = (T._lib.KvIndex * (1 << 20))()
            import ctypes as C
            n = C.c_uint32()
            while True:
                T._lib.check(m.L.tezgpu_merge_next_batch(m.h, buf.ctypes.data, buf.size, idx, 1 << 20, C.byref(n)))
                if n.value == 0:
                    break
            m.close()
        res[mode] = timed(run, reps)
    b = sum(len(s) for s in segs)
    return {"case": "read_%dx%dMiB_text" % (nseg, seg_bytes >> 20), "gpu": gpu_name(), "input_bytes": b,
            "concat_ms": res["concat"], "merge_ms": res["merge"], "concat_GBps": b / res["concat"] / 1e6,
            "merge_GBps": b / res["merge"] / 1e6, "speedup": res["merge"] / res["concat"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spill-gb", type=float, default=2.0, help="bytes of records per spill (4 spills: 8 GB in all)")
    ap.add_argument("--spills", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--read-segments", type=int, default=256)
    a = ap.parse_args()
    recs = int(a.spill_gb * 1e9 / 80)
    print(json.dumps(case_final_merge(a.spills, recs, 64, T.CODEC_NONE, a.reps, "final_merge_c2")), flush=True)
    print(json.dumps(case_read(a.read_segments, 4 << 20, a.reps)), flush=True)
    for c, nm in ((T.CODEC_LZ4, "lz4"), (T.CODEC_ZSTD, "zstd")):
        print(json.dumps(case_final_merge(a.spills, recs // 4, 64, c, a.reps, "final_merge_c2_" + nm)), flush=True)


if __name__ == "__main__":
    main()

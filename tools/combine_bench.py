"""Device combiner benchmark: device-resident LongWritable key + LongWritable value records (16-byte stride) through
tezgpu_sorter_sort_device_fixed, P = 64, with and without the LongSumReducer combine, over three key spaces.

    python tools/combine_bench.py [--n 100000000] [--steps 10] [--warmup 3]

Every (key space, combiner) configuration runs in a fresh process.  Prints one JSON line: per configuration the step
time (median / min / max over the timed steps, host clock around the call, which ends in a device synchronise), the
records and bytes written, and the share of the step the combine took (device events: ms_total minus the stage, sort,
tie and emit phases).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPACES = {"k2^10": 1 << 10, "k2^20": 1 << 20, "unique": 0}


def one(n, space, combiner, steps, warmup):
    import torch
    sys.path.insert(0, ROOT)
    import tez_b200 as T
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randperm(n, device="cuda", generator=g) if SPACES[space] == 0 else \
        torch.randint(0, SPACES[space], (n,), device="cuda", generator=g)
    be = lambda x: x.to(torch.int64).contiguous().view(torch.uint8).view(n, 8).flip(1)   # LongWritable: big-endian
    kv = torch.cat([be(keys), be(torch.ones(n, dtype=torch.int64, device="cuda"))], dim=1).contiguous()
    del keys
    P = 64
    cap = n * 28 + 10 * P + 64
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with T.GpuSorter(P, comparator=T.CMP_LONG, fixed=(8, 8), combiner=combiner) as s:
        times, combine_ms, device_ms, st, ln = [], [], [], None, 0
        for i in range(warmup + steps):
            t0 = time.perf_counter()
            ln, _, st = s.sort_device_fixed(kv.data_ptr(), n, out.data_ptr(), cap)
            dt = (time.perf_counter() - t0) * 1e3
            if i >= warmup:
                times.append(dt)
                device_ms.append(st["ms_total"])
                combine_ms.append(st["ms_total"] - st["ms_stage"] - st["ms_sort"] - st["ms_ties"] - st["ms_emit"])
    return dict(space=space, combiner=bool(combiner), n=n, step_ms_median=statistics.median(times), step_ms_min=min(times),
                step_ms_max=max(times), records_written=st["spilled_records"], bytes_written=ln,
                device_ms_total_median=statistics.median(device_ms),
                combine_ms_median=statistics.median(combine_ms) if combiner else 0.0,
                combine_share=(statistics.median(combine_ms) / statistics.median(times)) if combiner else 0.0,
                emit_ms=st["ms_emit"], sort_ms=st["ms_sort"], ties_ms=st["ms_ties"], steps=steps)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--one", nargs=2, metavar=("SPACE", "COMBINER"))
    a = ap.parse_args()
    if a.one:
        print(json.dumps(one(a.n, a.one[0], int(a.one[1]), a.steps, a.warmup)))
        return
    results = []
    for space in SPACES:
        for comb in (0, 2):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--n", str(a.n), "--steps", str(a.steps),
                                "--warmup", str(a.warmup), "--one", space, str(comb)], stdout=subprocess.PIPE, text=True)
            if r.returncode != 0:
                raise SystemExit("configuration %s / combiner %d failed" % (space, comb))
            results.append(json.loads(r.stdout.strip().splitlines()[-1]))
    print(json.dumps(dict(gpu=gpu_info(), workload="sort_device_fixed LongWritable/LongWritable P=64", results=results)))


if __name__ == "__main__":
    main()

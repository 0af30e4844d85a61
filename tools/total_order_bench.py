"""What TotalOrderPartitioner costs on the device: the map-side sort with the partition from the split search, against
the HashPartitioner and against partitions computed on the host and passed in (PART_GIVEN).

    python tools/total_order_bench.py [--records N] [--text-records N] [--steps K] [--warmup W]

Arms, alternated inside every step so that clock and neighbour noise falls on all of them alike:
  config 2 shape (N x 16 B key / 64 B value, sort_device_fixed) at P = 64 and P = 1024: HASH, TOTAL_ORDER with P - 1
  splits at the quantiles of a seeded sample, GIVEN with the same partitions computed on the host;
  Text keys (10 content bytes) with 8-byte values, variable width through collect, P = 64: HASH, TOTAL_ORDER, GIVEN.
Prints one JSON line per run with the GPU's name and power limit, read in the same call, and per arm the min, the
spread (max - min) and every timed step of ms_total and ms_stage."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def quantile_splits(keys, P, rng):
    """P - 1 distinct keys at the quantiles of a seeded sample (keys: numpy 'S' array, bytes order)"""
    sample = np.unique(keys[rng.choice(len(keys), size=min(len(keys), 64 * P), replace=False)])
    return sample[(np.arange(1, P) * len(sample)) // P]


def fixed_arms(n, P, rng):
    kv = O.gen_c2(0, n, seed=2)
    keys = kv.reshape(n, 80)[:, :16].copy().view("S16").ravel()
    splits = quantile_splits(keys, P, rng)
    part = np.searchsorted(splits, keys, side="right").astype(np.int32)
    d_kv = torch.from_numpy(kv).cuda()
    d_part = torch.from_numpy(part).cuda()
    cap = n * 82 + 10 * P + 4096
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    split_list = [bytes(s).ljust(16, b"\0") for s in splits]
    handles = {
        "hash": (T.GpuSorter(P, fixed=(16, 64)), None),
        "total_order": (T.GpuSorter(P, fixed=(16, 64), partitioner=T.PART_TOTAL_ORDER, split_points=split_list), None),
        "given": (T.GpuSorter(P, fixed=(16, 64), partitioner=T.PART_GIVEN), d_part.data_ptr()),
    }

    def run(arm):
        s, dp = handles[arm]
        _, _, st = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap, dp)
        return st
    return handles, run


def text_arms(n, P, rng):
    content = rng.integers(97, 123, size=(n, 10), dtype=np.uint8)
    rec = np.concatenate([np.full((n, 1), 10, np.uint8), content, rng.integers(0, 256, size=(n, 8), dtype=np.uint8)], axis=1)
    kv = rec.ravel()
    ko = np.arange(n, dtype=np.uint32) * 19
    vo, vl = ko + 11, np.full(n, 8, np.uint32)
    keys = content.copy().view("S10").ravel()
    splits = quantile_splits(keys, P, rng)
    part = np.searchsorted(splits, keys, side="right").astype(np.int32)
    split_list = [O.text(bytes(s).ljust(10, b"\0")) for s in splits]
    kw = dict(comparator=T.CMP_TEXT, rle_policy=T.RLE_OFF)
    handles = {
        "hash": (T.GpuSorter(P, **kw), None),
        "total_order": (T.GpuSorter(P, partitioner=T.PART_TOTAL_ORDER, split_points=split_list, **kw), None),
        "given": (T.GpuSorter(P, partitioner=T.PART_GIVEN, **kw), part),
    }

    def run(arm):
        s, p = handles[arm]
        s.reset()
        s.collect(kv, ko, vo, vl, p)
        return s.flush_to_memory()[3]
    return handles, run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=100_000_000)
    ap.add_argument("--text-records", type=int, default=20_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    name, power = gpu_info()
    rng = np.random.default_rng(7)
    for label, make, n, P in (("c2_fixed", fixed_arms, a.records, 64), ("c2_fixed", fixed_arms, a.records, 1024),
                              ("text_variable", text_arms, a.text_records, 64)):
        handles, run = make(n, P, rng)
        arms = list(handles)
        times = {arm: {"ms_total": [], "ms_stage": []} for arm in arms}
        for step in range(a.warmup + a.steps):
            for arm in (arms if step % 2 == 0 else arms[::-1]):
                st = run(arm)
                if step >= a.warmup:
                    times[arm]["ms_total"].append(st["ms_total"])
                    times[arm]["ms_stage"].append(st["ms_stage"])
        # every step's time is kept, so that a spread says whether one step or all of them moved
        res = {arm: {k: {"min": round(min(v), 4), "spread": round(max(v) - min(v), 4), "steps": [round(x, 3) for x in v]}
                     for k, v in t.items()} for arm, t in times.items()}
        print(json.dumps({"case": label, "records": n, "partitions": P, "gpu": name, "power_limit": power,
                          "steps": a.steps, "warmup": a.warmup, "arms": res}), flush=True)
        for s, _ in handles.values():
            s.close()
        del handles, run
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""Total-order sort across the GPUs of a box (DESIGN §5, §7): every rank generates records on its device, the ranks
agree on split points sampled on the devices (shuffle.total_order_splits: sample, all-gather, select), sort with
TotalOrderPartitioner into an exported buffer (sort_device), pull their blocks of partitions (PeerExchange, checksum
verified in flight) and merge them in place.  Rank 0's merged output, then rank 1's, ... is one sorted sequence.

    python -m torch.distributed.run --nproc-per-node N tools/total_order_sort_bench.py [--workload sort|words] [--records R]

Workloads: "sort", the reference Sort's shape (BytesWritable keys of 10..25 bytes and values of 0..31, generated on the
device from splitmix64); "words", OrderedWordCount's Text records (synth.gen_words, Zipf), whose hot keys cannot be split.
Rank 0 prints one JSON line: the seconds of each phase (max over ranks), GB/s of KV over their sum, the imbalance of
records and bytes across owners (max / mean), and the card name and power limit read in the same run.  After the timed
region it checks that the last key of rank g is <= the first key of rank g + 1, that every rank's splits have rank 0's
digest, and that one owned partition of each rank equals the oracle byte for byte; a failed check exits non-zero.
Ranks use cuda:(local rank % devices); with one device the ranks share it (CUDA IPC maps a buffer of the same device)."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200 import shuffle, synth  # noqa: E402
from total_order_sort_worker import gen_bytes  # noqa: E402

SEED = 17


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["sort", "words"], default="sort")
    ap.add_argument("--records", type=int, default=4_000_000, help="records per rank")
    ap.add_argument("--partitions", type=int, default=0, help="P (default 64 per rank)")
    ap.add_argument("--freq", type=float, default=0.01)
    ap.add_argument("--samples", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev_id = int(os.environ.get("LOCAL_RANK", "0")) % torch.cuda.device_count()
    torch.cuda.set_device(dev_id)
    dev = torch.device("cuda", dev_id)
    P = a.partitions or 64 * world
    n = a.records
    cmp = T.CMP_BYTESWRITABLE if a.workload == "sort" else T.CMP_TEXT
    table = synth.word_table(50000, SEED) if a.workload == "words" else None

    def records(g):
        if a.workload == "words":
            return synth.gen_words(g * n, n, seed=SEED, device=dev, table=table)
        return gen_bytes(g * n, n, dev)

    kv, ko, vo, vl = records(rank)
    torch.cuda.synchronize()
    cap = None
    px = sorter = merger = None
    best = None
    for rep in range(a.reps + 1):          # rep 0 warms every shape up
        ph = {}
        dist.barrier()
        splits = shuffle.total_order_splits((kv, ko, vo, vl), P, a.freq, a.samples, seed=5, comparator=cmp, device=dev_id,
                                            timings=ph)
        uniq = [s for i, s in enumerate(splits) if i == 0 or s != splits[i - 1]]   # Zipf heads: Java repeats splits
        Pe = len(uniq) + 1
        if sorter is None or sorter.P != Pe:
            sorter = T.GpuSorter(Pe, comparator=cmp, partitioner=T.PART_TOTAL_ORDER, split_points=uniq, device=dev_id)
            cap = sorter.device_output_bound(n, kv.numel())
            if px is None:
                px = shuffle.PeerExchange(cap, dev_id)
        else:
            sorter.set_split_points(uniq)
        t0 = time.perf_counter()
        _, index, _ = sorter.sort_device(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), n,
                                         px.out_ptr(rep), cap)
        t1 = time.perf_counter()
        segs = px.exchange(rep, index, Pe)
        t2 = time.perf_counter()
        p0, p1 = shuffle.owner_ranges(Pe, world)[rank]
        seg_list, parts = [(ptr, ln) for ptr, ln, _, _ in segs], [p for _, _, p, _ in segs]
        if merger is None:
            merger = T.GpuMerger(seg_list, comparator=cmp, device_ptrs=True, partitions=parts, num_partitions=max(1, p1 - p0),
                                 verified=px.last_verified, device=dev_id)
        else:
            merger.reopen(seg_list, parts, verified=px.last_verified)
        d_merged = torch.empty(merger.output_bound() + 64, dtype=torch.uint8, device=dev)
        mlen, mindex, _ = merger.write_partitions_device(d_merged.data_ptr(), d_merged.numel())
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        ph.update(sort=t1 - t0, exchange=t2 - t1, merge=t3 - t2)
        allph = [None] * world
        dist.all_gather_object(allph, ph)
        ph = {k: max(p[k] for p in allph) for k in ph}
        if rep and (best is None or sum(ph.values()) < sum(best.values())):
            best = ph
    # ---- checks, outside the timed region
    got = d_merged[:mlen].cpu().numpy().tobytes()
    recs, nbytes = merger.counts()
    empty = len(O.write_ifile([])[0])
    nonempty = [q for q in range(p1 - p0) if int(mindex[q][2]) > empty]
    first = last = None
    if nonempty:
        q0, q1 = nonempty[0], nonempty[-1]
        first = O.read_ifile(got[int(mindex[q0][0]):int(mindex[q0][0]) + int(mindex[q0][2])])[0][1]
        last = O.read_ifile(got[int(mindex[q1][0]):int(mindex[q1][0]) + int(mindex[q1][2])])[-1][1]
    digest = hashlib.sha256(b"".join(len(s).to_bytes(8, "little") + s for s in splits)).hexdigest()
    info = [None] * world
    dist.all_gather_object(info, (first, last, digest, recs, nbytes, kv.numel()))
    ok_order = True
    prev_last = None
    for f, l, _, _, _, _ in info:
        if f is None:
            continue
        if prev_last is not None and O.compare(cmp, prev_last, f) > 0:
            ok_order = False
        prev_last = l
    ok_digest = all(d == info[0][2] for _, _, d, _, _, _ in info)
    # oracle: the first non-empty owned partition, from every producer's records of that partition
    ok_oracle = True
    if nonempty:
        p = p0 + nonempty[0]
        runs = []
        for g in range(world):
            hkv, hko, hvo, hvl = (t.cpu().numpy() for t in records(g))
            keys = [hkv[x:y].tobytes() for x, y in zip(hko.tolist(), hvo.tolist())]
            part = np.asarray(T.debug_total_order(keys, uniq, cmp))
            sel = np.nonzero(part == p)[0]
            if sel.size == 0:
                continue
            res = O.pipelined_sort(O.sorter_conf(1, cmp_kind=cmp, partitioner=O.PART_GIVEN), hkv, hko[sel].astype(np.uint64),
                                   (hvo - hko)[sel].astype(np.uint32), hvl[sel].astype(np.uint32), np.zeros(sel.size, np.int32))
            runs.append(res["file_out"][int(res["index"][0][0]):int(res["index"][0][0]) + int(res["index"][0][2])])
        q = nonempty[0]
        ok_oracle = got[int(mindex[q][0]):int(mindex[q][0]) + int(mindex[q][2])] == O.merge(runs, cmp, factor=100)["ifile"]
    oks = [None] * world
    dist.all_gather_object(oks, ok_oracle)
    if rank == 0:
        rec = np.array([i[3] for i in info], dtype=np.float64)
        byt = np.array([i[4] for i in info], dtype=np.float64)
        kv_total = sum(i[5] for i in info)
        tot = sum(best.values())
        print(json.dumps({
            "workload": a.workload, "gpus": world, "devices": torch.cuda.device_count(), "records_per_rank": n,
            "partitions": P, "partitions_used": Pe, "freq": a.freq, "max_samples": a.samples,
            "phase_s": {k: round(v, 6) for k, v in best.items()}, "total_s": round(tot, 6),
            "kv_gbps": round(kv_total / tot / 1e9, 3),
            "imbalance_records": round(float(rec.max() / rec.mean()), 4), "imbalance_bytes": round(float(byt.max() / byt.mean()), 4),
            "sample_select_over_sort": round((best["sample"] + best["select"]) / best["sort"], 4),
            "card": card(), "checks": {"global_order": ok_order, "digest": ok_digest, "oracle": all(oks)}}))
    merger.close()
    px.close()
    sorter.close()
    dist.destroy_process_group()
    sys.exit(0 if (ok_order and ok_digest and all(oks)) else 1)


if __name__ == "__main__":
    main()

"""Multi-GPU shuffle of variable-length records: OrderedWordCount-shaped map output (Text word, IntWritable 1) that each
GPU generates in its own HBM (synth.gen_words), weak scaling, one rank per GPU.

step = sort_device (partition + sort by Text key, straight from device memory, into the exported file.out buffer)
       -> verified NVLink pull of the owned partitions (PeerExchange) -> in-place k-way merge of the pulled
       variable-framed segments (GpuMerger, write_partitions_device).

Prints one JSON line: records and KV bytes per GPU, sort / exchange / merge ms (mean, min, max over the timed steps), KV
GB/s, the transport, the GPU's name, power limit and SM clocks read in the same run.  At N=1 it also times collect_batch
+ flush_to_memory (the host-buffer path, pinned host memory) on the same records, so the gain from keeping the records
on the device is measured on the same machine.  After the timed region every rank checks one owned partition byte for
byte: the producers' records are rebuilt on the CPU, sorted by the oracle, and the oracle's merge of their runs of that
partition must equal the merged segment.

    python tools/multigpu_text_bench.py --records 16777216 --steps 10 --warmup 3                  # one GPU
    python -m torch.distributed.run --nproc-per-node 8 tools/multigpu_text_bench.py --records ...  # eight GPUs
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tez_b200 as T  # noqa: E402
from tez_b200 import shuffle, synth  # noqa: E402


def gpu_state(local):
    """name, power limit and SM clocks as nvidia-smi reports them (read only)"""
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        return dict(zip(q.split(","), vals)) if len(vals) == 5 else {"name": torch.cuda.get_device_name(local)}
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(local)}


def spread(xs):
    return {"mean": round(float(np.mean(xs)), 3), "min": round(float(np.min(xs)), 3), "max": round(float(np.max(xs)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 24, help="records per GPU")
    ap.add_argument("--partitions", type=int, default=64)
    ap.add_argument("--vocab", type=int, default=100000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if "RANK" not in os.environ:   # plain `python tools/multigpu_text_bench.py`: a group of one
        os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1")
        os.environ.setdefault("MASTER_PORT", str(29500 + os.getpid() % 1000))
    if not torch.cuda.is_available():
        raise SystemExit("multigpu_text_bench: no CUDA device (the measurement has no CPU fallback)")
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    n, P = args.records, args.partitions
    table = synth.word_table(args.vocab, args.seed)
    d_kv, d_ko, d_vo, d_vl = synth.gen_words(rank * n, n, seed=args.seed, device=dev, table=table)
    kv_bytes = d_kv.numel()
    torch.cuda.synchronize()   # the library works on its own stream
    sorter = T.GpuSorter(P, comparator=T.CMP_TEXT, device=local)
    cap = sorter.device_output_bound(n, n * (1 + synth.WORD_MAX + 4))   # the same on every rank: every record at its longest
    px = shuffle.PeerExchange(cap, local)
    transport = "peer: index all-gather (NCCL) + one verified fetch kernel over CUDA IPC mappings; own partitions merged in place"
    d_merged = torch.empty(int(cap * 1.3) + (1 << 20), dtype=torch.uint8, device=dev)
    p0, p1 = shuffle.owner_ranges(P, world)[rank]
    merger = [None]
    state = {"k": 0, "last": None}
    ph = {"sort": [], "exchange": [], "merge": [], "step": []}

    def step(timed):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        k = state["k"]
        state["k"] += 1
        _, index, _ = sorter.sort_device(d_kv.data_ptr(), kv_bytes, d_ko.data_ptr(), d_vo.data_ptr(), d_vl.data_ptr(), n,
                                         px.out_ptr(k), cap)
        e[1].record()
        segs = px.exchange(k, index, P)
        e[2].record()
        torch.cuda.current_stream().synchronize()
        seg_list = [(ptr, ln) for ptr, ln, _, _ in segs]
        parts = [p for _, _, p, _ in segs]
        if merger[0] is None:
            merger[0] = T.GpuMerger(seg_list, comparator=T.CMP_TEXT, device=local, device_ptrs=True, partitions=parts,
                                    num_partitions=max(1, p1 - p0), verified=px.last_verified)
        else:
            merger[0].reopen(seg_list, parts, verified=px.last_verified)
        mlen, mindex, _ = merger[0].write_partitions_device(d_merged.data_ptr(), d_merged.numel())
        state["last"] = (k, index, segs, mindex)
        e[3].record()
        if timed:
            torch.cuda.synchronize()
            for name, a, b in (("sort", 0, 1), ("exchange", 1, 2), ("merge", 2, 3), ("step", 0, 3)):
                ph[name].append(e[a].elapsed_time(e[b]))

    before = gpu_state(local)
    for _ in range(args.warmup):
        step(False)
    dist.barrier()
    for _ in range(args.steps):
        step(True)
    dist.barrier()
    after = gpu_state(local)
    step_ms = torch.tensor([float(np.mean(ph["step"]))], device=dev, dtype=torch.float64)
    dist.all_reduce(step_ms, op=dist.ReduceOp.MAX)
    total_kv = torch.tensor([float(kv_bytes)], device=dev, dtype=torch.float64)
    dist.all_reduce(total_kv)

    # ---- N=1: the host-buffer path on the same records (collect_batch + flush_to_memory from pinned memory)
    host = None
    if world == 1:
        h_kv = d_kv.cpu().pin_memory().numpy()
        h_ko = d_ko.to(torch.int32).cpu().pin_memory().numpy().view(np.uint32)
        h_vo = d_vo.to(torch.int32).cpu().pin_memory().numpy().view(np.uint32)
        h_vl = d_vl.cpu().pin_memory().numpy().view(np.uint32)
        h_out = torch.empty(sorter.device_output_bound(n, kv_bytes), dtype=torch.uint8).pin_memory().numpy()
        hs = T.GpuSorter(P, comparator=T.CMP_TEXT, device=local)
        host_ms, host_out = [], None
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            hs.collect(h_kv, h_ko, h_vo, h_vl)
            out, _, index, _ = hs.flush_to_memory(h_out)
            t1 = time.perf_counter()
            hs.reset()
            if i >= args.warmup:
                host_ms.append((t1 - t0) * 1e3)
            host_out = (bytes(out), index)
        hs.close()
        k, index, _, _ = state["last"]
        dev_out = torch.empty(int(index[-1, 0] + index[-1, 2]), dtype=torch.uint8, device=dev)
        T.fetch_ranges([(px.out_ptr(k), dev_out.data_ptr(), dev_out.numel())], local)
        same = dev_out.cpu().numpy().tobytes() == host_out[0] and np.array_equal(index, host_out[1])
        assert same, "sort_device and collect_batch + flush_to_memory wrote different file.out bytes"
        host = {"what": "collect_batch + flush_to_memory, pinned host buffers, host clock around each call pair",
                "ms": spread(host_ms), "kv_GBps": round(kv_bytes / (np.mean(host_ms) * 1e-3) / 1e9, 2),
                "sort_device_kv_GBps": round(kv_bytes / (np.mean(ph["sort"]) * 1e-3) / 1e9, 2),
                "sort_device_speedup": round(float(np.mean(host_ms) / np.mean(ph["sort"])), 2), "same_file_out": same}

    # ---- outside the timed region: one owned partition per rank against the oracle
    from oracle import tez_oracle as O
    checked = torch.zeros(1, device=dev, dtype=torch.float64)
    k, _, segs, mindex = state["last"]
    owned = sorted({p for _, _, p, _ in segs})
    if owned:
        lp = owned[(rank * 7) % len(owned)]
        step_first = [g * n for g in range(world)]
        runs = []
        for g in range(world):
            kv, ko, vo, vl = (t.numpy() for t in synth.gen_words(step_first[g], n, seed=args.seed, table=table))
            res = O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT), kv, ko.astype(np.uint64), (vo - ko).astype(np.uint32),
                                   vl.astype(np.uint32))
            a, _, ln = (int(x) for x in res["index"][p0 + lp])
            if ln:
                runs.append(res["file_out"][a:a + ln])
        a, _, ln = (int(x) for x in mindex[lp])
        merged = d_merged[a:a + ln].cpu().numpy().tobytes()
        assert merged == O.merge(runs, O.CMP_TEXT, factor=100)["ifile"], "rank %d partition %d differs from the oracle" % (rank, p0 + lp)
        checked[0] = 1
    dist.all_reduce(checked)
    if rank == 0:
        ms = float(step_ms.item())
        line = {"metric": "sort_device + NVLink pull + merge of Text / IntWritable records", "unit": "GB/s of KV",
                "value": round(float(total_kv.item()) / (ms * 1e-3) / 1e9, 3), "n_gpus": world,
                "records_per_gpu": n, "kv_bytes_per_gpu": kv_bytes, "partitions": P, "vocab": args.vocab,
                "steps": args.steps, "warmup": args.warmup, "ms_per_step_max_over_ranks": round(ms, 3),
                "phases_ms_rank0": {name: spread(v) for name, v in ph.items()},
                "transport": transport, "gpu_before": before, "gpu_after": after, "host_path": host,
                "parity_check": {"ranks_checked": int(checked.item()),
                                 "what": "one owned partition per rank: the oracle's merge of the producers' oracle runs "
                                         "(records rebuilt on the CPU) equals the merged segment byte for byte"}}
        print(json.dumps(line))
    dist.barrier()
    merger[0].close()
    px.close()
    sorter.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

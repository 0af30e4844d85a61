"""Multi-GPU arm of bench.py: BASELINE config 4 shape, weak scaling, one rank per GPU.

step = local partition+sort (P partitions) -> all-to-all of the partition segments to their owners over NVLink
       -> batched k-way merge of the G runs of every owned partition into the final segments.
"""
import json
import os
import time

import numpy as np
import torch
import torch.distributed as dist

def run(args, workload_config, ClockSampler, hbm_peak, run_cpu, host_cores, verify_partition=None):
    """verify_partition(run_bytes_list, merged_segment_bytes) -> None or raises: the caller's checker (bench.py passes the
    CPU oracle's TezMerger restatement); run on every rank for one owned partition AFTER the timed region."""
    import tez_b200 as T
    from tez_b200 import shuffle, synth
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    # point-to-point (send/recv) all-to-all: let NCCL use many channels per peer over NVLink
    os.environ.setdefault("NCCL_MIN_P2P_NCHANNELS", "32")
    os.environ.setdefault("NCCL_MAX_P2P_NCHANNELS", "32")
    os.environ.setdefault("NCCL_NCHANNELS_PER_PEER", "32")
    dist.init_process_group("nccl", device_id=dev)
    config = getattr(args, "config", 4)
    if config == 5:
        # BASELINE config 5: Zipf(1.1) keys, 4 KB values, 256 partitions -- partition imbalance, run-length encoded
        # segments (the producers' AUTO rule turns RLE on), general parse / merge / emit on the reduce side
        KEY_LEN, VAL_LEN, P = 16, 4096, 256
        REC, OUT_REC = KEY_LEN + VAL_LEN, KEY_LEN + VAL_LEN + 4      # vint(16) = 1 byte, vint(4096) = 3 bytes
        n = args.records
        d_kv = synth.gen_c5(rank * n, n, seed=5, val_len=VAL_LEN, device=dev)
    else:
        KEY_LEN, VAL_LEN, P = 16, 64, 1024
        REC, OUT_REC = KEY_LEN + VAL_LEN, KEY_LEN + VAL_LEN + 2
        n = args.records
        d_kv = synth.gen_c2(rank * n, n, seed=4, device=dev)
    torch.cuda.synchronize()   # the library works on its own stream
    sorter = T.GpuSorter(P, fixed=(KEY_LEN, VAL_LEN), device=local)
    cap = n * OUT_REC + 10 * P + 4096
    # shuffle transport: "peer" = consumers pull file.out ranges out of the producers' HBM with libtezgpu's fetch kernel
    # (CUDA IPC mappings over NVLink); "nccl" = one variable-size all-to-all of NCCL send/recv pairs (the baseline)
    transport = os.environ.get("TEZ_SHUFFLE", "peer")
    px = None
    if transport == "peer":
        try:
            px = shuffle.PeerExchange(cap, local)
        except RuntimeError as e:   # raised on every rank or on none (consensus inside)
            transport = "nccl (%s)" % e
    d_out = None if px else torch.empty(cap, dtype=torch.uint8, device=dev)
    step_no = [0]
    d_merged = torch.empty(int(cap * 1.3) + (1 << 20), dtype=torch.uint8, device=dev)
    p0, p1 = shuffle.owner_ranges(P, world)[rank]
    launches = [0]
    merger = [None]
    phase_ms = {"sort": [], "exchange": [], "merge": []}
    fetch_ms = []
    last_step = [None, None, 0]

    def step(timed):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        k = step_no[0]
        step_no[0] += 1
        out_ptr = px.out_ptr(k) if px else d_out.data_ptr()
        out_len, index, st = sorter.sort_device_fixed(d_kv.data_ptr(), n, out_ptr, cap)
        e[1].record()
        if px:
            segs = px.exchange(k, index, P)   # returns once the pulled bytes have landed
            seg_list = [(ptr, ln) for ptr, ln, _, _ in segs]
            if timed:
                fetch_ms.append(px.last_fetch_ms)
        else:
            recv, segs = shuffle.exchange_partitions(d_out[:out_len], index, P)
            base = recv.data_ptr()
            seg_list = [(base + off, ln) for off, ln, _, _ in segs]
        e[2].record()
        # the library works on its own stream: the received bytes must have landed before it reads them
        torch.cuda.current_stream().synchronize()
        parts = [p for _, _, p, _ in segs]
        verified = px.last_verified if px else None
        if merger[0] is None:
            merger[0] = T.GpuMerger(seg_list, comparator=T.CMP_BYTES, device=local, device_ptrs=True,
                                    fixed=(KEY_LEN, VAL_LEN), partitions=parts, num_partitions=p1 - p0, verified=verified)
        else:
            merger[0].reopen(seg_list, parts, verified=verified)
        m = merger[0]
        mlen, mindex, mst = m.write_partitions_device(d_merged.data_ptr(), d_merged.numel())
        nrec, _ = m.counts()
        last_step[:] = [segs, mindex, mlen]
        e[3].record()
        if timed:
            torch.cuda.synchronize()
            launches[0] += st["kernel_launches"] + mst["kernel_launches"]
            phase_ms["sort"].append(e[0].elapsed_time(e[1]))
            phase_ms["exchange"].append(e[1].elapsed_time(e[2]))
            phase_ms["merge"].append(e[2].elapsed_time(e[3]))
        return nrec, mlen

    # TEZ_SHUFFLE_OVERLAP=1 (opt-in, written at the end of round 1, not yet measured): the NVLink-bound pull of batch k
    # runs concurrently with the HBM-bound sort of batch k+1 (second host thread, own stream).  The sort of batch k+1
    # starts only after the index all-gather of batch k returned: by then every peer has finished pulling batch k-1,
    # whose buffer the sort rewrites.  Every iteration still performs one sort, one exchange and one merge.
    overlap = px is not None and os.environ.get("TEZ_SHUFFLE_OVERLAP", "0") == "1"
    if overlap:
        import threading
        # a pull grid that fills every SM serialises with the sort kernels instead of overlapping (exchange = sort +
        # pull); about one CTA per SM keeps NVLink busy and leaves the other half of each SM to the sort
        os.environ.setdefault("TEZGPU_FETCH_CTAS", str(torch.cuda.get_device_properties(dev).multi_processor_count))
        pull_stream = torch.cuda.Stream(device=dev)
        pending = {}

        def sort_batch(k):
            out_len, index, st = sorter.sort_device_fixed(d_kv.data_ptr(), n, px.out_ptr(k), cap)
            pending[k] = (index, st)

        sort_batch(0)          # batch 0 is sorted before the pipeline starts; batch K is sorted inside it

        def step(timed):       # noqa: F811 -- replaces the sequential step
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            k = step_no[0]
            step_no[0] += 1
            index, st = pending.pop(k)
            all_idx = px.gather(index)
            th = threading.Thread(target=sort_batch, args=(k + 1,))
            th.start()
            segs = px.pull(k, all_idx, P, stream=pull_stream.cuda_stream)
            th.join()
            e[1].record()
            seg_list = [(ptr, ln) for ptr, ln, _, _ in segs]
            parts = [p for _, _, p, _ in segs]
            verified = px.last_verified
            if merger[0] is None:
                merger[0] = T.GpuMerger(seg_list, comparator=T.CMP_BYTES, device=local, device_ptrs=True,
                                        fixed=(KEY_LEN, VAL_LEN), partitions=parts, num_partitions=p1 - p0, verified=verified)
            else:
                merger[0].reopen(seg_list, parts, verified=verified)
            m = merger[0]
            mlen, mindex, mst = m.write_partitions_device(d_merged.data_ptr(), d_merged.numel())
            nrec, _ = m.counts()
            last_step[:] = [segs, mindex, mlen]
            e[2].record()
            if timed:
                torch.cuda.synchronize()
                launches[0] += st["kernel_launches"] + mst["kernel_launches"]
                fetch_ms.append(px.last_fetch_ms)
                phase_ms["sort"].append(0.0)
                phase_ms["exchange"].append(e[0].elapsed_time(e[1]))   # gather + max(pull k, sort k+1)
                phase_ms["merge"].append(e[1].elapsed_time(e[2]))
            return nrec, mlen

    for _ in range(args.warmup):
        step(False)
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    dist.barrier()
    torch.cuda.synchronize()
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        nrec, mlen = step(True)
    t1.record()
    torch.cuda.synchronize()
    dist.barrier()
    ms = torch.tensor([t0.elapsed_time(t1) / args.steps], device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    tot = torch.tensor([float(nrec), float(launches[0])], device=dev, dtype=torch.float64)
    dist.all_reduce(tot)
    ms_step = float(ms.item())
    ph = torch.tensor([sum(phase_ms[k]) / max(1, len(phase_ms[k])) for k in ("sort", "exchange", "merge")] +
                      [sum(fetch_ms) / max(1, len(fetch_ms))], device=dev, dtype=torch.float64)
    ph_max, ph_min = ph.clone(), ph.clone()
    dist.all_reduce(ph_max, op=dist.ReduceOp.MAX)
    dist.all_reduce(ph_min, op=dist.ReduceOp.MIN)
    clk = clocks.stop() if rank == 0 else None
    # ---- outside the timed region: every rank checks one partition it owns, byte for byte -- the G runs it merged
    # (device memory: the local slot or the receive buffer) through the caller's checker against its merged segment,
    # and the segment's CRC32 trailer with zlib
    checked = torch.zeros(1, device=dev, dtype=torch.float64)
    if verify_partition is not None and last_step[0] is not None:
        import zlib
        segs_l, mindex_l, _ = last_step
        owned = sorted({p for _, _, p, _ in segs_l})
        if owned:
            lp = owned[(rank * 7) % len(owned)]                      # a different local partition on every rank

            def dev_bytes(ptr, ln):   # raw device address -> host bytes, through the library's own copy kernel
                t = torch.empty(ln + 32, dtype=torch.uint8, device=dev)
                torch.cuda.synchronize()
                off = (ptr - t.data_ptr()) % 16
                T.fetch_ranges([(ptr, t.data_ptr() + off, ln)], local)
                return t[off:off + ln].cpu().numpy().tobytes()

            runs = [dev_bytes(ptr, ln) for ptr, ln, p, _ in segs_l if p == lp]
            a, _, ln = (int(x) for x in mindex_l[lp])
            merged = d_merged[a:a + ln].cpu().numpy().tobytes()
            assert int.from_bytes(merged[-4:], "big") == zlib.crc32(merged[4:-4]), "CRC32 trailer of the merged segment"
            verify_partition(runs, merged)
            checked[0] = 1
    dist.all_reduce(checked)
    # partition imbalance: merged bytes this rank ends up owning (max / mean over the ranks)
    own = torch.tensor([float(last_step[2])], device=dev, dtype=torch.float64)
    own_max, own_sum = own.clone(), own.clone()
    dist.all_reduce(own_max, op=dist.ReduceOp.MAX)
    dist.all_reduce(own_sum)
    if rank == 0:
        total_records = n * world
        assert int(tot[0].item()) == total_records, "records lost in the shuffle"
        value = total_records * REC / (ms_step * 1e-3) / 1e9
        peak, peak_src = hbm_peak()
        avg = {k: round(sum(v) / len(v), 3) for k, v in phase_ms.items()}
        sent = int(n * OUT_REC * (world - 1) / world)
        line = {"metric": "sorted KV GB/s (16B key / %dB val)" % VAL_LEN, "value": round(value, 3), "unit": "GB/s",
                "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_step, 4),
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
                "config": workload_config(world, n, config) if config == 5 else workload_config(world, n), "clocks": clk, "gpu_launches": int(tot[1].item()),
                "e2e": None,
                "phases_ms_rank0": avg,
                "phases_ms_over_ranks": {k: [round(float(ph_min[i]), 3), round(float(ph_max[i]), 3)]
                                         for i, k in enumerate(("sort", "exchange", "merge", "fetch_kernel"))},
                "nvlink": {"bytes_sent_per_gpu_per_step": sent,
                           "achieved_GBps_per_gpu": round(sent / (avg["exchange"] * 1e-3) / 1e9, 1) if avg["exchange"] else None,
                           "fetch_kernel_ms": round(sum(fetch_ms) / len(fetch_ms), 3) if fetch_ms else None,
                           "fetch_kernel_GBps_per_gpu": round(sent / (sum(fetch_ms) / len(fetch_ms) * 1e-3) / 1e9, 1) if fetch_ms and sum(fetch_ms) else None,
                           "transport": transport + (" + sort(k+1) overlapped with pull(k)" if overlap else ""),
                           "note": ("peer pull: index all-gather (NCCL) + one fetch kernel over CUDA IPC mappings; own partitions merged in place"
                                    if px else "variable-size all-to-all (NCCL send/recv) incl. index all-gather")},
                "roofline": {"bound": "hbm", "achieved": round(n * (2 * (REC + OUT_REC)) / (ms_step * 1e-3) / 1e9, 1), "peak": peak,
                             "unit": "GB/s", "frac": round(n * (2 * (REC + OUT_REC)) / (ms_step * 1e-3) / 1e9 / peak, 4),
                             "traffic": None, "peak_source": peak_src,
                             "note": "per GPU: sort (read key+value, write framed record) + merge (read + write the framed "
                                     "records) algorithmic bytes over the whole step, without run-length savings"},
                "imbalance": {"max_owned_bytes": int(own_max.item()), "mean_owned_bytes": int(own_sum.item() / world),
                              "max_over_mean": round(float(own_max.item()) / max(1.0, own_sum.item() / world), 3)},
                "parity_check": {"ranks_checked": int(checked.item()),
                                 "what": "after the timed region every rank compared one owned partition's merged segment with the CPU "
                                         "oracle's TezMerger over the G runs it merged (byte-exact) and its CRC32 trailer with zlib"},
                "cpu_baseline": None}
        print(json.dumps(line))
    if px:
        dist.barrier()
        px.close()
    dist.destroy_process_group()
    return 0

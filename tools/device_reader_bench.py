"""The merged stream read on the device (tezgpu_merge_next_batch_device) next to the same stream read into pinned host
memory (tezgpu_merge_next_batch), on three inputs.  One JSON line per input.

  c3:    config-3-shaped Text segments (oracle generator), merged in place from device memory
  fixed: 16 B key / 64 B value records (config-2 records, oracle-sorted runs), merged in place with the fixed framing
  words: OrderedWordCount map outputs (synth.gen_words) sorted on the device by tezgpu_sorter_sort_device, then merged
         in place

The merge itself (open) is timed on its own and kept out of the read times: the run-length encoded Text merge takes far
longer than reading its result, and would hide the reader.  Every pass opens a fresh merger and reads the whole stream
in batches of --batch-bytes / --batch-records:
  device_call_ms  host clock around every next_batch_device call (each returns once its batch is written), summed
  host_call_ms    the same for next_batch into pinned host memory on the merger's stream
  gather_ms       the k_gather_batch kernels of one device pass (every launch of the pass), from torch.profiler's CUDA
                  activity in a pass of its own.  CUDA events cannot bracket the kernel alone: it runs inside the
                  library call, between the batch search and the call's own synchronise, on the merger's stream
  gather_gbps     moved_bytes() over gather_ms, and its share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
The device and host passes must hand out the same records (checked on a sample of batches).  The card's name and power
limit are read in the same run.  Without a CUDA device the measurement fails; --help and the byte accounting do not need
one.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12      # bytes/s, H100 SXM data sheet
META_READ = 4 + 8 + 8 + 8 + 4 + 4 + 4 + 1   # per record: order, kv_off, key_off, val_off, key_len, val_len, tag, same


def moved_bytes(kv_bytes, records, same_key):
    """Bytes one batch must move at least: its key + value bytes read from the segments and written to the batch, the
    table it writes (64-bit key and value offsets, 32-bit value length, the isSameKey byte when asked for) and the
    per-record metadata the gather reads (META_READ)."""
    return 2 * kv_bytes + records * (8 + 8 + 4 + (1 if same_key else 0)) + records * META_READ


def share_of_peak(nbytes, seconds):
    """nbytes moved in seconds, over the data-sheet HBM3 bandwidth"""
    return nbytes / seconds / HBM_PEAK


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


# ------------------------------------------------------------------------------------------------ inputs
def input_c3(torch, O, T, scale):
    segs, _ = O.gen_c3_segments(8, int(96 * scale) << 20, seed=3, threads=8)
    dev = [torch.from_numpy(s).to("cuda") for s in segs]
    return dict(segments=[(d.data_ptr(), d.numel()) for d in dev], keep=dev, kw=dict(comparator=T.CMP_TEXT))


def input_fixed(torch, O, T, scale):
    n = int((1 << 21) * scale)
    dev = []
    for s in range(4):
        kv = O.gen_c2(s * n, n, seed=2)
        seg = O.pipelined_sort_fixed(O.sorter_conf(1), kv, 16, 64)["file_out"]
        dev.append(torch.frombuffer(bytearray(seg), dtype=torch.uint8).to("cuda"))
    return dict(segments=[(d.data_ptr(), d.numel()) for d in dev], keep=dev, kw=dict(comparator=T.CMP_BYTES, fixed=(16, 64)))


def input_words(torch, O, T, scale):
    from tez_b200 import synth
    n = int((1 << 23) * scale)
    dev, segs = [], []
    for i in range(2):
        kv, ko, vo, vl = synth.gen_words(i * n, n, seed=7, vocab=50000, device="cuda")
        with T.GpuSorter(1, comparator=T.CMP_TEXT, rle_policy=T.RLE_ON) as s:
            cap = s.device_output_bound(n, kv.numel())
            out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
            _, index, _ = s.sort_device(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), n,
                                        out.data_ptr(), cap)
        dev.append(out)
        segs.append((out.data_ptr() + int(index[0][0]), int(index[0][2])))
    return dict(segments=segs, keep=dev, kw=dict(comparator=T.CMP_TEXT))


INPUTS = {"c3": input_c3, "fixed": input_fixed, "words": input_words}


# ------------------------------------------------------------------------------------------------ passes
def open_merger(T, inp):
    t0 = time.perf_counter()
    m = T.GpuMerger(inp["segments"], device_ptrs=True, **inp["kw"])
    n, kv = m.counts()
    return m, (time.perf_counter() - t0) * 1e3, n, kv


def device_pass(torch, m, bufs, batch_records, sample):
    kv, ko, vo, vl, sk = bufs
    calls, ms, total, got = 0, 0.0, 0, []
    while True:
        t0 = time.perf_counter()
        n, b = m.next_batch_device(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), sk.data_ptr(),
                                   batch_records)
        ms += (time.perf_counter() - t0) * 1e3
        if n == 0:
            return calls, ms, total, got
        if calls in sample:
            got.append((kv[:b].cpu().numpy().tobytes(), vl[:n].cpu().numpy().tolist(), sk[:n].cpu().numpy().tolist()))
        calls += 1
        total += b


def host_pass(T, m, buf, batch_records, sample):
    from tez_b200 import _lib
    from tez_b200._lib import KvIndex
    idx = (KvIndex * batch_records)()
    n = C.c_uint32()
    calls, ms, total, got = 0, 0.0, 0, []
    while True:
        t0 = time.perf_counter()
        _lib.check(m.L.tezgpu_merge_next_batch(m.h, buf.data_ptr(), buf.numel(), idx, batch_records, C.byref(n)))
        ms += (time.perf_counter() - t0) * 1e3
        if n.value == 0:
            return calls, ms, total, got
        e = idx[n.value - 1]
        b = e.val_off + e.val_len
        if calls in sample:
            got.append((buf[:b].numpy().tobytes(), [x.val_len for x in idx[:n.value]], [x.same_key for x in idx[:n.value]]))
        calls += 1
        total += b


def gather_kernel_ms(torch, m, bufs, batch_records):
    """k_gather_batch time of one device pass, from the profiler's CUDA activity"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device_pass(torch, m, bufs, batch_records, ())
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if "k_gather_batch" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
    return sum(e.device_time for e in evs) / 1e3, len(evs)


def run_input(torch, O, T, name, args):
    inp = INPUTS[name](torch, O, T, args.scale)
    dev = torch.device("cuda")
    bufs = (torch.empty(args.batch_bytes, dtype=torch.uint8, device=dev),
            torch.empty(args.batch_records, dtype=torch.int64, device=dev),
            torch.empty(args.batch_records, dtype=torch.int64, device=dev),
            torch.empty(args.batch_records, dtype=torch.int32, device=dev),
            torch.empty(args.batch_records, dtype=torch.uint8, device=dev))
    pinned = torch.empty(args.batch_bytes, dtype=torch.uint8, pin_memory=True)
    sample = {0, 1, 5}
    res = dict(input=name, card=card(), batch_bytes=args.batch_bytes, batch_records=args.batch_records)
    opens, dcall, hcall, gms = [], [], [], []
    for rep in range(args.warmup + args.reps):
        m, t_open, n, kv = open_merger(T, inp)
        calls, d_ms, d_bytes, d_got = device_pass(torch, m, bufs, args.batch_records, sample)
        m.close()
        m, _, _, _ = open_merger(T, inp)
        g_ms, launches = gather_kernel_ms(torch, m, bufs, args.batch_records)
        m.close()
        m, _, _, _ = open_merger(T, inp)
        hcalls, h_ms, h_bytes, h_got = host_pass(T, m, pinned, args.batch_records, sample)
        m.close()
        assert d_bytes == h_bytes == kv and calls == hcalls == launches, (d_bytes, h_bytes, kv, calls, hcalls, launches)
        assert d_got == h_got, "device and host batches differ"
        if rep >= args.warmup:
            opens.append(t_open)
            dcall.append(d_ms)
            hcall.append(h_ms)
            gms.append(g_ms)
    moved = moved_bytes(kv, n, True)
    g = min(gms)
    res.update(records=n, kv_bytes=kv, batches=calls, open_ms=opens, device_call_ms=dcall, host_call_ms=hcall,
               gather_ms=gms, moved_bytes=moved, gather_gbps=moved / g / 1e6,
               gather_share_of_hbm_peak=share_of_peak(moved, g / 1e3),
               device_call_gbps=kv / min(dcall) / 1e6, host_call_gbps=kv / min(hcall) / 1e6)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--inputs", default="c3,fixed,words", help="comma-separated subset of %s" % ",".join(INPUTS))
    ap.add_argument("--scale", type=float, default=1.0, help="input size factor (1.0: about 0.75-1 GB of records each)")
    ap.add_argument("--batch-bytes", type=int, default=256 << 20)
    ap.add_argument("--batch-records", type=int, default=1 << 22)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("device_reader_bench: no CUDA device (nothing here is measured without one)")
    from oracle import tez_oracle as O
    import tez_b200 as T
    for name in args.inputs.split(","):
        print(json.dumps(run_input(torch, O, T, name, args)), flush=True)


if __name__ == "__main__":
    main()

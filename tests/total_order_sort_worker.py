"""Worker of tests/test_total_order_sort_gpu.py: one of G processes sharing cuda:0, rendezvous over gloo.  Each rank
generates records on the device, the ranks agree on split points sampled on the devices (shuffle.total_order_splits),
each sorts its records with TOTAL_ORDER into its exported buffer, pulls its block of partitions with the checksum
verified in flight and merges them in place.  The ranks' merged outputs, concatenated in rank order, must equal the
oracle's sort of every record, partition by partition.  argv: n P kind (words | bytes)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200 import shuffle, synth  # noqa: E402

SEED, VOCAB = 17, 20000


def gen_bytes(first, n, device):
    """the reference Sort's records: BytesWritable keys of 10..25 content bytes and values of 0..31, from splitmix64 counters"""
    i = torch.arange(first, first + n, device=device, dtype=torch.int64)
    h = synth.splitmix64(i ^ (SEED << 40))
    klen = 4 + 10 + (h & 15)
    vlen = 4 + ((h >> 8) & 31)
    size = klen + vlen
    ko = torch.cumsum(size, 0) - size
    total = int(size.sum().item())
    kv = torch.empty(total, dtype=torch.uint8, device=device)
    pos = torch.arange(total, device=device, dtype=torch.int64)
    rec = torch.searchsorted(ko, pos, right=True) - 1
    j = pos - ko[rec]
    word = synth.splitmix64((i[rec] << 6) ^ (j >> 3))
    kv[:] = ((word >> ((7 - (j & 7)) * 8)) & 0xFF).to(torch.uint8)
    for lens, base in ((klen, ko), (vlen, ko + klen)):       # 4-byte big-endian length prefixes of key and value
        ln = lens - 4
        for b in range(4):
            kv[base + b] = ((ln >> (8 * (3 - b))) & 0xFF).to(torch.uint8)
    vo = ko + klen
    return kv, ko, vo, vlen.to(torch.int32)


def main():
    n, P, kind = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    cmp = T.CMP_TEXT if kind == "words" else T.CMP_BYTESWRITABLE
    table = synth.word_table(VOCAB, SEED) if kind == "words" else None

    def records(g, device):
        if kind == "words":
            return synth.gen_words(g * n, n, seed=SEED, device=device, table=table)
        return gen_bytes(g * n, n, device)

    kv, ko, vo, vl = records(rank, dev)
    torch.cuda.synchronize()
    splits = shuffle.total_order_splits((kv, ko, vo, vl), P, 0.02, 4000, seed=5, comparator=cmp)
    # words: a Zipf head word can fill several steps of the sample, and Java's rule then repeats a split, which
    # TotalOrderPartitioner refuses; every rank drops the repeats the same way and runs with fewer partitions
    if any(a == b for a, b in zip(splits, splits[1:])):
        splits = [s for i, s in enumerate(splits) if i == 0 or s != splits[i - 1]]
        P = len(splits) + 1
    sorter = T.GpuSorter(P, comparator=cmp, partitioner=T.PART_TOTAL_ORDER, split_points=splits)
    cap = sorter.device_output_bound(n, kv.numel())
    px = shuffle.PeerExchange(cap, 0)
    out_len, index, _ = sorter.sort_device(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), n,
                                           px.out_ptr(0), cap)
    segs = px.exchange(0, index, P)
    p0, p1 = shuffle.owner_ranges(P, world)[rank]
    merger = T.GpuMerger([(ptr, ln) for ptr, ln, _, _ in segs], comparator=cmp, device_ptrs=True,
                         partitions=[p for _, _, p, _ in segs], num_partitions=max(1, p1 - p0), verified=px.last_verified)
    d_merged = torch.empty(merger.output_bound() + 64, dtype=torch.uint8, device=dev)
    mlen, mindex, _ = merger.write_partitions_device(d_merged.data_ptr(), d_merged.numel())
    got = d_merged[:mlen].cpu().numpy().tobytes()
    # the oracle: every rank's records sorted with the same splits by the oracle's PipelinedSorter, then TezMerger over
    # the producers' runs of each owned partition (rank order breaks ties, as in the pull's segment table)
    outs = []
    for g in range(world):
        hkv, hko, hvo, hvl = (t.cpu().numpy() for t in records(g, "cpu"))
        keys = [hkv[a:b].tobytes() for a, b in zip(hko.tolist(), hvo.tolist())]
        part = np.array(T.debug_total_order(keys, splits, cmp), dtype=np.int32)
        outs.append(O.pipelined_sort(O.sorter_conf(P, cmp_kind=cmp, partitioner=O.PART_GIVEN), hkv, hko.astype(np.uint64),
                                     (hvo - hko).astype(np.uint32), hvl.astype(np.uint32), part))
    for p in range(p0, p1):
        runs = []
        for g in range(world):
            a, _, ln = (int(x) for x in outs[g]["index"][p])
            if ln:
                runs.append(outs[g]["file_out"][a:a + ln])
        a, _, ln = (int(x) for x in mindex[p - p0])
        if not runs:
            assert ln == 0 or got[a:a + ln] == O.write_ifile([])[0], "empty partition %d" % p
            continue
        assert got[a:a + ln] == O.merge(runs, cmp, factor=100)["ifile"], "rank %d partition %d differs from the oracle" % (rank, p)
    dist.barrier()
    merger.close()
    px.close()
    sorter.close()
    dist.destroy_process_group()
    print("total order worker %d ok" % rank)


if __name__ == "__main__":
    main()

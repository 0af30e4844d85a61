"""Worker of tests/test_peer_fetch_var_gpu.py: one of G processes sharing cuda:0 (CUDA IPC maps a buffer of the same
device), rendezvous over gloo.  OrderedWordCount-shaped records generated on the device -> sort_device (Text keys,
HashPartitioner) into the exported file.out buffer -> verified pull of the owned partitions -> merge of the pulled
variable-framed segments in place, checked partition by partition against the oracle's TezMerger over the producers'
oracle runs."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402
from tez_b200 import shuffle, synth  # noqa: E402

SEED, VOCAB = 11, 3000


def main():
    n, P, steps = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    table = synth.word_table(VOCAB, SEED)
    sorter = T.GpuSorter(P, comparator=T.CMP_TEXT)
    cap = sorter.device_output_bound(n, n * (1 + synth.WORD_MAX + 4))    # every record at its longest
    px = shuffle.PeerExchange(cap, 0)
    p0, p1 = shuffle.owner_ranges(P, world)[rank]
    merger = None
    for k in range(steps):
        first = [g * n + 1000 * k for g in range(world)]
        d_kv, d_ko, d_vo, d_vl = synth.gen_words(first[rank], n, seed=SEED, device=dev, table=table)
        torch.cuda.synchronize()   # the sorter works on its own stream
        out_len, index, _ = sorter.sort_device(d_kv.data_ptr(), d_kv.numel(), d_ko.data_ptr(), d_vo.data_ptr(),
                                               d_vl.data_ptr(), n, px.out_ptr(k), cap)
        segs = px.exchange(k, index, P)
        seg_list = [(ptr, ln) for ptr, ln, _, _ in segs]
        parts = [p for _, _, p, _ in segs]
        if merger is None:
            merger = T.GpuMerger(seg_list, comparator=T.CMP_TEXT, device_ptrs=True, partitions=parts,
                                 num_partitions=max(1, p1 - p0), verified=px.last_verified)
        else:
            merger.reopen(seg_list, parts, verified=px.last_verified)
        assert px.last_verified is not None and sum(px.last_verified) == sum(1 for _, _, _, g in segs if g != rank)
        d_merged = torch.empty(merger.output_bound() + 64, dtype=torch.uint8, device=dev)
        mlen, mindex, _ = merger.write_partitions_device(d_merged.data_ptr(), d_merged.numel())
        got = d_merged[:mlen].cpu().numpy().tobytes()
        # oracle: every producer's file.out from the same records rebuilt on the CPU, then TezMerger per owned partition
        outs = []
        for g in range(world):
            kv, ko, vo, vl = (t.numpy() for t in synth.gen_words(first[g], n, seed=SEED, table=table))
            outs.append(O.pipelined_sort(O.sorter_conf(P, cmp_kind=O.CMP_TEXT), kv, ko.astype("uint64"),
                                         (vo - ko).astype("uint32"), vl.astype("uint32")))
        for p in range(p0, p1):
            runs = []
            for g in range(world):
                a, _, ln = (int(x) for x in outs[g]["index"][p])
                if ln:
                    runs.append(outs[g]["file_out"][a:a + ln])
            a, raw, ln = (int(x) for x in mindex[p - p0])
            if not runs:
                assert ln == 0 or got[a:a + ln] == O.write_ifile([])[0], "empty partition %d" % p
                continue
            exp = O.merge(runs, O.CMP_TEXT, factor=100)["ifile"]
            assert got[a:a + ln] == exp, "rank %d step %d partition %d differs from the oracle merge" % (rank, k, p)
    dist.barrier()
    merger.close()
    px.close()
    sorter.close()
    dist.destroy_process_group()
    print("peer var worker %d ok" % rank)


if __name__ == "__main__":
    main()

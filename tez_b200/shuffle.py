"""Scatter-gather shuffle between the GPUs of one box -- what ScatterGatherEdgeManager + ShuffleHandler +
FetcherOrderedGrouped do over HTTP in the reference (DAG/dag/app/dag/impl/ScatterGatherEdgeManager.java:108-131,
OG/FetcherOrderedGrouped.java:437-632): consumer p pulls partition p from every producer.

Here every rank is one producer and owns a contiguous block of partitions (owner(p) = p * G // P).  Because a
producer's file.out already stores its partitions in partition order, the bytes destined to one owner are ONE
contiguous range of file.out: the exchange is a single variable-size all-to-all (NCCL send/recv pairs over NVLink)
with no repacking, preceded by an all-gather of the TezSpillRecord index (P x 3 int64 per rank).

exchange_partitions() is pure torch.distributed plumbing: works on CUDA tensors over NCCL and on CPU tensors over
gloo (tests).  PeerExchange is the fast path on an NVSwitch box: every producer keeps file.out in an exported device
buffer, consumers map it once and pull their byte ranges with libtezgpu's fetch kernel (all SMs, 128-bit words);
a rank's own partitions are merged in place, they never move.
"""
import numpy as np
import torch
import torch.distributed as dist


def owner_ranges(num_partitions, world):
    """[p0, p1) of every rank for owner(p) = p * world // num_partitions (contiguous blocks)."""
    bounds = [(num_partitions * g + world - 1) // world for g in range(world + 1)]
    return [(bounds[g], bounds[g + 1]) for g in range(world)]


def exchange_partitions(file_out, index, num_partitions, group=None):
    """file_out: uint8 tensor with this rank's file.out bytes (device or CPU); index: [P,3] int64 numpy
    (start, rawLength, partLength).  Returns (recv uint8 tensor, segments) where segments is a list of
    (offset_in_recv, length, local_partition, source_rank) for every non-empty segment this rank now owns."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = file_out.device
    idx = torch.from_numpy(np.ascontiguousarray(index, dtype=np.int64)).to(dev)
    all_idx = [torch.empty_like(idx) for _ in range(world)]
    dist.all_gather(all_idx, idx, group=group)
    all_idx = torch.stack(all_idx).cpu().numpy()  # [world, P, 3]
    ranges = owner_ranges(num_partitions, world)
    part_len = all_idx[:, :, 2]
    # what I send to g: my segments of g's partitions (contiguous in my file.out)
    send_sizes = [int(part_len[rank, a:b].sum()) for a, b in ranges]
    p0, p1 = ranges[rank]
    recv_sizes = [int(part_len[g, p0:p1].sum()) for g in range(world)]
    send_off0 = int(all_idx[rank, ranges[0][0], 0]) if num_partitions else 0
    send = file_out[send_off0:send_off0 + sum(send_sizes)]
    recv = torch.empty(max(1, sum(recv_sizes)), dtype=torch.uint8, device=dev)
    dist.all_to_all_single(recv[:sum(recv_sizes)], send, output_split_sizes=recv_sizes, input_split_sizes=send_sizes,
                           group=group)
    segments = []
    off = 0
    for g in range(world):
        for p in range(p0, p1):
            ln = int(part_len[g, p])
            if ln:
                segments.append((off, ln, p - p0, g))
            off += ln
    return recv, segments


def _gather_index(index, group, device):
    """all-gather of the [P,3] spill index -> [world, P, 3] numpy (device tensors over NCCL, CPU tensors over gloo)."""
    world = dist.get_world_size(group)
    on_dev = dist.get_backend(group) == "nccl"
    idx = torch.from_numpy(np.ascontiguousarray(index, dtype=np.int64))
    if on_dev:
        idx = idx.to(device)
    out = [torch.empty_like(idx) for _ in range(world)]
    dist.all_gather(out, idx, group=group)
    return torch.stack(out).cpu().numpy()


def pull_plan(all_idx, rank, num_partitions, peer_ptrs):
    """What rank `rank` pulls: all_idx is the gathered [world, P, 3] spill index, peer_ptrs[g] the address of rank g's
    file.out in this process.  Returns (ranges, seg_src, need): ranges = [(g, src_address, offset_in_receive_buffer,
    nbytes)], one per producer, in ring order starting at rank+1 (the classic all-to-all schedule: at any moment every
    producer's HBM / NVLink egress serves one consumer instead of all consumers pulling from rank 0 first);
    seg_src[g] = (receive offset, file offset) of g's range; need = receive buffer bytes.  Receive offsets agree
    with the source address modulo 16 so the copy moves 128-bit words (the receive buffer is 16-byte aligned)."""
    world = all_idx.shape[0]
    p0, p1 = owner_ranges(num_partitions, world)[rank]
    ranges, seg_src, need = [], {}, 0
    for step_g in range(1, world):
        g = (rank + step_g) % world
        if p1 <= p0:
            continue
        a = int(all_idx[g, p0, 0])
        ln = int(all_idx[g, p0:p1, 2].sum())
        src = peer_ptrs[g] + a
        off = (need + 15) // 16 * 16 + (src & 15)
        seg_src[g] = (off, a)
        need = off + ln
        if ln:
            ranges.append((g, src, off, ln))
    return ranges, seg_src, need


def pull_segments(all_idx, rank, num_partitions, peer_ptrs, seg_src, recv_base):
    """Segment table after the pull: [(address, length, local_partition, source_rank)] ordered by (source_rank,
    partition) -- the order TezMerger breaks ties in.  Own runs stay where the sorter wrote them.  (The merge sorts by
    (partition, key) and breaks ties by position in this table, i.e. by source rank inside a partition.)"""
    world = all_idx.shape[0]
    p0, p1 = owner_ranges(num_partitions, world)[rank]
    starts = all_idx[:, p0:p1, 0]
    lens = all_idx[:, p0:p1, 2]
    bases = np.zeros((world, 1), dtype=np.int64)
    for g in range(world):
        if g == rank:
            bases[g, 0] = peer_ptrs[g]
        elif g in seg_src:
            off, a = seg_src[g]
            bases[g, 0] = recv_base + off - a
    ptrs = starts + bases
    gs, ps = np.nonzero(lens)                          # row-major: ordered by (source_rank, partition)
    return list(zip(ptrs[gs, ps].tolist(), lens[gs, ps].tolist(), ps.tolist(), gs.tolist()))


def ring_order(segs, rank, world):
    """The remote rows of a pull_segments table in the order they are pulled: producer rank+1 first, then rank+2, ...
    (partitions of one producer keep their order)."""
    return sorted((t for t in segs if t[3] != rank), key=lambda t: (t[3] - rank) % world)


def total_order_splits(records, num_partitions, freq, max_samples, seed, group=None, comparator=None, order=None, device=0,
                       timings=None):
    """TotalOrderPartitioner split points shared by every rank, sampled on the devices: records = (kv, key_off, val_off,
    val_len), this rank's device tensors in GpuSorter.sort_device's layout (synth.gen_words returns them).  The records
    are numbered across ranks (gid_base = the records of the lower ranks, from an all-gather of the counts), each rank
    samples its own (native.sample_keys), the samples are all-gathered, and every rank selects the same splits from their
    union (native.select_split_points).  With these splits on every rank's TOTAL_ORDER sorter and owner_ranges' blocks of
    partitions, rank 0's merged output, then rank 1's, ... is one sorted sequence.  A failure on any rank, or splits
    whose digest differs from rank 0's, raise on every rank.  timings: an optional dict that receives the seconds of the
    phases sample, all-gather and select."""
    import hashlib
    import time

    from . import native
    from .constants import CMP_BYTES
    cmp = CMP_BYTES if comparator is None else comparator
    kv, ko, vo, vl = records
    n = int(ko.numel())
    world, rank = dist.get_world_size(group), dist.get_rank(group)

    def agree(ok, payload, what):
        got = [None] * world
        dist.all_gather_object(got, (ok, payload), group=group)
        bad = [g for g, (o, _) in enumerate(got) if not o]
        if bad:
            raise RuntimeError("total_order_splits: rank %d could not %s (%s)" % (bad[0], what, got[bad[0]][1]))
        return [p for _, p in got]

    t0 = time.perf_counter()
    counts = agree(True, n, "count its records")
    sample, err = None, None
    try:
        sample = native.sample_keys(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(), n, seed, freq,
                                    max_samples, gid_base=sum(counts[:rank]), device=device)
    except Exception as e:  # noqa: BLE001 -- reported on every rank by agree()
        err = e
    t1 = time.perf_counter()
    samples = agree(err is None, sample if err is None else str(err), "sample its keys")
    t2 = time.perf_counter()
    splits, err = None, None
    try:
        splits = native.select_split_points(samples, num_partitions, max_samples, cmp, order, device=device)
    except Exception as e:  # noqa: BLE001
        err = e
    digest = hashlib.sha256(b"".join(len(s).to_bytes(8, "little") + s for s in splits)).hexdigest() if err is None else None
    digests = agree(err is None, digest if err is None else str(err), "select the split points")
    if any(d != digests[0] for d in digests):
        raise RuntimeError("total_order_splits: the split points of rank %d differ from rank 0's"
                           % next(g for g, d in enumerate(digests) if d != digests[0]))
    t3 = time.perf_counter()
    if timings is not None:
        timings.update(sample=t1 - t0, all_gather=t2 - t1, select=t3 - t2)
    return splits


class PeerExchange:
    """NVLink pull shuffle.  Each rank owns `slots` exported file.out buffers used round-robin (step k writes slot
    k % slots): with two slots the index all-gather of step k+1 is the only synchronisation needed -- a peer has
    finished pulling step k's bytes before it enters that all-gather, and slot k % 2 is not rewritten before step k+2."""

    def __init__(self, out_capacity, device, group=None, slots=2):
        from . import native
        self.group, self.device = group, device
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.capacity = int(out_capacity)
        self.slots, self._maps, self.peers = [], [], []
        self._recv = None
        self.last_fetch_ms = 0.0
        self.last_verified = None
        import os
        self.verify = os.environ.get("TEZ_SHUFFLE_VERIFY_IN_FETCH", "1") != "0"
        # every phase ends in a consensus (all-reduce MIN of a success flag): either all ranks get the peer transport
        # or all of them raise, so a caller can fall back to exchange_partitions() without a collective mismatch
        err = None
        try:
            self.slots = [native.PeerBuffer(out_capacity, device) for _ in range(slots)]
        except Exception as e:  # noqa: BLE001 -- reported through the consensus below
            err = e
        self._consensus(err, "allocate an exportable file.out buffer")
        handles = [None] * self.world
        dist.all_gather_object(handles, [b.handle for b in self.slots], group=group)
        try:
            for g in range(self.world):   # peers[g][slot] -> device address of rank g's slot in this process
                if g == self.rank:
                    self.peers.append([b.ptr for b in self.slots])
                else:
                    maps = [native.PeerMapping(h, device) for h in handles[g]]
                    self._maps += maps
                    self.peers.append([m.ptr for m in maps])
        except Exception as e:  # noqa: BLE001
            err = e
        self._consensus(err, "map a peer's file.out buffer")

    def _consensus(self, err, what):
        on_dev = dist.get_backend(self.group) == "nccl"
        flag = torch.tensor([0 if err is not None else 1], dtype=torch.int32,
                            device=torch.device("cuda", self.device) if on_dev else torch.device("cpu"))
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            self.close()
            raise RuntimeError("peer pull unavailable: some rank could not %s%s" % (what, (" (%s)" % err) if err else ""))

    def out_ptr(self, step):
        return self.slots[step % len(self.slots)].ptr

    def exchange(self, step, index, num_partitions):
        """index: this rank's [P,3] spill index of the file.out it just wrote into slot `step`.
        Returns segments [(device_ptr, length, local_partition, source_rank)] ordered by (source_rank, partition):
        own segments point into the local slot, the others into the receive buffer the pull kernel filled."""
        return self.pull(step, self.gather(index), num_partitions)

    def gather(self, index):
        """The collective half of exchange(): all-gather of the spill index.  When it returns, every rank has entered
        it, i.e. has finished pulling the previous step."""
        return _gather_index(index, self.group, torch.device("cuda", self.device))

    def pull(self, step, all_idx, num_partitions, stream=None):
        """The data half of exchange(): one fetch kernel (on `stream`, a raw cudaStream_t handle, default stream when
        None) pulls this rank's partitions of step `step` from every peer; returns the segment table once they landed."""
        from . import native
        slot = step % len(self.slots)
        peer_ptrs = [self.peers[g][slot] for g in range(self.world)]
        ranges, seg_src, need = pull_plan(all_idx, self.rank, num_partitions, peer_ptrs)
        if self._recv is None or self._recv.numel() < need + 64:
            self._recv = torch.empty(int(need * 1.25) + 4096, dtype=torch.uint8, device=torch.device("cuda", self.device))
        base = self._recv.data_ptr()
        segs = pull_segments(all_idx, self.rank, num_partitions, peer_ptrs, seg_src, base)
        if self.verify:
            # one kernel moves the remote segments AND verifies each one's CRC32 trailer on the bytes in flight, like
            # IFile.Reader.readToMemory on a fetch to memory (SORT/IFile.java:764-809); own runs are verified by the merge
            p0 = owner_ranges(num_partitions, self.world)[self.rank][0]
            src_of = {g: (peer_ptrs[g] + a) - (base + off) for g, (off, a) in seg_src.items()}   # src - dst per producer
            # ring order, like pull_plan: producer rank+1 first, so that at any moment a producer serves one consumer
            # (the segment table itself is ordered by source rank -- pulling in THAT order sends all consumers to rank 0
            # first, and every rank but the first waits for the others)
            remote = [(ptr + src_of[g], ptr, ln) for ptr, ln, _, g in ring_order(segs, self.rank, self.world)]
            self.last_fetch_ms = native.fetch_segments_verified(remote, self.device, stream)
            self.last_verified = [g != self.rank for _, _, _, g in segs]
        else:
            self.last_fetch_ms = native.fetch_ranges([(src, base + off, ln) for _, src, off, ln in ranges], self.device, stream)
            self.last_verified = None
        return segs

    def close(self):
        for m in self._maps:
            m.close()
        for b in self.slots:
            b.close()
        self._maps, self.slots = [], []

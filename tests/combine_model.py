"""Reference combine for the tests: MRCombiner running IntSumReducer / LongSumReducer, restated over the CPU oracle.

The oracle sorts (or merges) the records as PipelinedSorter / TezMerger do; this module then walks every partition's
segment with IFile.Reader semantics, groups adjacent records whose keys compare equal under the comparator
(ValuesIterator, RL/common/ValuesIterator.java:178-197), replaces each group by (key, big-endian wrapped sum) and
writes the segment again through the oracle's IFile.Writer.  The sums do not depend on the order of equal keys, so
the result is exact even where the oracle's tie order is not pinned.
"""
import numpy as np

from oracle import tez_oracle as O

SUM_INT, SUM_LONG = 1, 2
WIDTH = {SUM_INT: 4, SUM_LONG: 8}


class BadWidth(ValueError):
    pass


def combine_records(records, cmp_kind, combiner):
    """records: [(key, value)] of one partition in sorted order -> [(key, sum bytes)], one per group."""
    w = WIDTH[combiner]
    mask = (1 << (8 * w)) - 1
    out = []
    for k, v in records:
        if len(v) != w:
            raise BadWidth("value of %d bytes, combiner needs %d" % (len(v), w))
        x = int.from_bytes(v, "big")
        if out and O.compare(cmp_kind, out[-1][0], k) == 0:
            out[-1][1] = (out[-1][1] + x) & mask
        else:
            out.append([k, x])
    return [(k, s.to_bytes(w, "big")) for k, s in out]


def _segment_records(seg):
    return [(k, v) for _, k, v in O.read_ifile(seg)]


def recombine_file(file_out, index, cmp_kind, combiner):
    """file.out + index (P x 3) of a sort -> (combined file.out, index (P x 3), index file bytes, records in, out)."""
    P = len(index)
    out = bytearray()
    idx = np.zeros((P, 3), dtype=np.int64)
    n_in = n_out = 0
    for p in range(P):
        start, raw, part = (int(x) for x in index[p])
        if part == 0:                      # no segment at all (empty partition, sent through the event)
            idx[p] = (len(out), 0, 0)
            continue
        recs = _segment_records(bytes(file_out[start:start + part]))
        comb = combine_records(recs, cmp_kind, combiner)
        n_in += len(recs)
        n_out += len(comb)
        seg, raw_len, part_len = O.write_ifile(comb)
        idx[p] = (len(out), raw_len, part_len)
        out += seg
    return bytes(out), idx, O.spill_record_bytes(idx.reshape(-1)), n_in, n_out


def sort_combine(P, cmp_kind, combiner, kv, key_off, key_len, val_len, partition=None, send_empty=True):
    """PipelinedSorter flush with the combiner: dict(file_out, index, index_out, combine_input, combine_output)."""
    part_mode = O.PART_GIVEN if partition is not None else O.PART_HASH
    conf = O.sorter_conf(P, cmp_kind=cmp_kind, partitioner=part_mode, send_empty=send_empty, rle_policy=0)
    res = O.pipelined_sort(conf, kv, key_off, key_len, val_len, partition)
    f, idx, ib, n_in, n_out = recombine_file(res["file_out"], res["index"], cmp_kind, combiner)
    return dict(file_out=f, index=idx, index_out=ib, combine_input=n_in, combine_output=n_out)


def merge_combine(segments, cmp_kind, combiner, has_header=True):
    """TezMerger.merge over IFile segments into a combining writer -> (segment bytes, rawLen, partLen)."""
    res = O.merge(segments, cmp_kind, has_header=has_header)
    comb = combine_records([(k, v) for k, v, _ in res["records"]], cmp_kind, combiner)
    return O.write_ifile(comb)


def model(records, partitions, cmp_kind, combiner, P):
    """Independent model: {(partition, key): wrapped sum}, then every partition's keys in comparator order.
    Returns [[(key, sum bytes)] per partition]."""
    import functools
    w = WIDTH[combiner]
    mask = (1 << (8 * w)) - 1
    sums = {}
    for (k, v), p in zip(records, partitions):
        if len(v) != w:
            raise BadWidth("value of %d bytes, combiner needs %d" % (len(v), w))
        sums[(p, bytes(k))] = (sums.get((p, bytes(k)), 0) + int.from_bytes(v, "big")) & mask
    out = [[] for _ in range(P)]
    for (p, k), s in sums.items():
        out[p].append((k, s.to_bytes(w, "big")))
    key = functools.cmp_to_key(lambda a, b: O.compare(cmp_kind, a[0], b[0]))
    return [sorted(o, key=key) for o in out]


def pack(records):
    """[(key, value)] -> (kv uint8, key_off u64, key_len u32, val_len u32, val_off u32) for the oracle and the sorter."""
    kv = bytearray()
    ko, kl, vl = [], [], []
    for k, v in records:
        ko.append(len(kv))
        kv += k
        kl.append(len(k))
        kv += v
        vl.append(len(v))
    ko = np.array(ko, np.uint64)
    kl = np.array(kl, np.uint32)
    return (np.frombuffer(bytes(kv), dtype=np.uint8) if kv else np.zeros(0, np.uint8), ko, kl,
            np.array(vl, np.uint32), (ko + kl).astype(np.uint32))

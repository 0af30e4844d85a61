"""Model of the unordered edge over the oracle's IFile reader and writer: what tezgpu_concat_open writes and iterates
(UnorderedPartitionedKVWriter.mergeAll, RL/common/writers/UnorderedPartitionedKVWriter.java:1058-1144, and
UnorderedKVReader, RL/common/readers/UnorderedKVReader.java:119-230)."""
from oracle import tez_oracle as O


def records(segments, has_header=True):
    """The records of the segments in (segment, position) order: [(key, value)]."""
    out = []
    for s in segments:
        out += [(k, v) for _, k, v in O.read_ifile(bytes(s), has_header=has_header)]
    return out


def concat_segment(segments, has_header=True):
    """One output segment: the oracle's IFile writer (rle = false) over the records of the inputs in order.
    (b"", 0, 0) when they hold no record (mergeAll writes nothing for such a partition, :1087-1091)."""
    recs = records(segments, has_header)
    if not recs:
        return b"", 0, 0
    return O.write_ifile(recs, rle=False)


def concat_file(segments, partitions, P, has_header=True):
    """file.out and its index (P triples) of write_partitions over segments tagged with their partitions; each
    partition's inputs in the order they appear."""
    out = bytearray()
    index = []
    for p in range(P):
        seg, raw, part = concat_segment([s for s, q in zip(segments, partitions) if q == p], has_header)
        index.append((len(out), raw, part) if seg else (0, 0, 0))
        out += seg
    return bytes(out), index


def partition_records(file_out, index):
    """{partition: [(key, value)]} of a file.out, read with the oracle (checksums verified)."""
    return {p: records([file_out[s:s + n]]) for p, (s, _, n) in enumerate(index) if n}

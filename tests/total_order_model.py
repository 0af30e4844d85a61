"""Model of Hadoop's TotalOrderPartitioner for the tests: the partition of a key restated as bisect_right over comparison
keys, split points at the quantiles of a sample, and a writer of the partition file (a SequenceFile, version 6).

No partition file written by Java exists here.  The file format is restated from the SequenceFile layout:
  header  "SEQ" 0x06, key class and value class (vint length + UTF-8 each), compressed byte, block-compressed byte,
          the codec class (same encoding) when compressed, metadata (int32 count, then that many Text pairs), 16 sync
          bytes;
  record  int32 record length (key + stored value bytes), int32 key length, key bytes, value bytes; a record length
          of -1 is a sync escape followed by the 16 sync bytes.
Record compression (what InputSampler writes by default) compresses each value alone (DefaultCodec: one zlib stream);
keys stay plain.  Block compression stores blocks of keys and values and is refused by the reader under test."""
import bisect
import random
import struct
import zlib

from oracle import tez_oracle as O
import sort_order_model as M

TEXT = "org.apache.hadoop.io.Text"
BYTES_WRITABLE = "org.apache.hadoop.io.BytesWritable"
INT_WRITABLE = "org.apache.hadoop.io.IntWritable"
LONG_WRITABLE = "org.apache.hadoop.io.LongWritable"
NULL_WRITABLE = "org.apache.hadoop.io.NullWritable"
DEFAULT_CODEC = "org.apache.hadoop.io.compress.DefaultCodec"
NEW_API = "org.apache.hadoop.mapreduce.lib.partition.TotalOrderPartitioner"
OLD_API = "org.apache.hadoop.mapred.lib.TotalOrderPartitioner"


def search_key(order, key):
    """Comparison key of a serialized key under a search order (a CMP_*): its normalised content bytes."""
    return M.content(order, key)


def partitions(keys, splits, order):
    """The number of split points <= key in the search order (BinarySearchNode.findPartition)."""
    sk = [search_key(order, s) for s in splits]
    return [bisect.bisect_right(sk, search_key(order, k)) for k in keys]


def quantile_splits(sample, P, cmp):
    """P - 1 distinct keys at the quantiles of a sample, increasing under the comparator (InputSampler.writePartitionFile)."""
    uniq = sorted(set(sample), key=lambda k: search_key(cmp, k))
    assert len(uniq) >= P - 1, "sample too small for %d partitions" % P
    step = len(uniq) / P
    out = [uniq[int(round(step * (i + 1)))] for i in range(P - 1)]
    assert all(search_key(cmp, a) < search_key(cmp, b) for a, b in zip(out, out[1:]))
    return out


def pack_keys(keys):
    """(kv bytes, key_off, key_len) of keys back to back"""
    off, kv = [], bytearray()
    for k in keys:
        off.append(len(kv))
        kv += k
    return bytes(kv), off, [len(k) for k in keys]


def random_content(rng, max_len=14, alphabet=None):
    ln = rng.randrange(max_len + 1)
    if alphabet is None:
        return bytes(rng.randrange(256) for _ in range(ln))
    return bytes(rng.choice(alphabet) for _ in range(ln))


def _text_string(s):
    b = s.encode("utf-8")
    return O.vint(len(b)) + b


def sequence_file(keys, key_class, value_class=NULL_WRITABLE, compression="none", sync_every=3, values=None, seed=0):
    """Bytes of a SequenceFile holding the serialized keys.  compression: "none", "record" (zlib values) or "block".
    A sync escape follows every sync_every records (0: none)."""
    rng = random.Random(seed)
    sync = bytes(rng.randrange(256) for _ in range(16))
    out = bytearray(b"SEQ\x06")
    out += _text_string(key_class) + _text_string(value_class)
    out += bytes([compression != "none", compression == "block"])
    if compression != "none":
        out += _text_string(DEFAULT_CODEC)
    out += struct.pack(">i", 1) + O.text("creator") + O.text("total_order_model")
    out += sync
    values = values if values is not None else [b""] * len(keys)
    if compression == "block":
        # one block: sync escape, then vint record count and four length-prefixed (zlib) buffers
        def buf(parts):
            z = zlib.compress(b"".join(parts))
            return O.vint(len(z)) + z
        out += struct.pack(">i", -1) + sync + O.vint(len(keys))
        out += buf([O.vint(len(k)) for k in keys]) + buf(keys) + buf([O.vint(len(v)) for v in values]) + buf(values)
        return bytes(out)
    for i, (k, v) in enumerate(zip(keys, values)):
        if sync_every and i and i % sync_every == 0:
            out += struct.pack(">i", -1) + sync
        stored = zlib.compress(v) if compression == "record" else v
        out += struct.pack(">ii", len(k) + len(stored), len(k)) + k + stored
    return bytes(out)

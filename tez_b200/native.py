"""Thin object wrappers over the C ABI (include/tezgpu.h) -- what the JNI shim does in a Tez task JVM.

GpuSorter  ~ ExternalSorter seam (SORT/ExternalSorter.java:74-92): write/collect -> flush -> close.
GpuMerger  ~ TezMerger.merge(...) -> TezRawKeyValueIterator (SORT/TezMerger.java:717-912).
"""
import collections
import ctypes as C
import os
import tempfile

import numpy as np

from . import _lib
from .constants import *  # noqa: F401,F403
from ._lib import Conf, KvIndex, Segment, Stats, check


def _ptr(a):
    return None if a is None else a.ctypes.data


def make_conf(num_partitions, comparator=CMP_BYTES, partitioner=PART_HASH, rle_policy=RLE_AUTO, send_empty=True,
              fixed=None, device=0, legacy=False, mem_budget=0, unordered=False):
    c = Conf()
    c.abi_version = ABI_VERSION
    c.device = device
    c.num_partitions = num_partitions
    c.comparator = comparator
    c.partitioner = partitioner
    c.rle_policy = rle_policy
    c.send_empty_partition_details = 1 if send_empty else 0
    c.sorter_impl = SORTER_UNORDERED if unordered else (SORTER_LEGACY if legacy else SORTER_PIPELINED)
    c.fixed_key_len, c.fixed_val_len = fixed if fixed else (0, 0)
    c.mem_budget_bytes = mem_budget
    return c


def _pack_keys(keys):
    """Serialized keys -> (bytes uint8, offsets uint64, lengths uint32), back to back."""
    kl = np.array([len(k) for k in keys], dtype=np.uint32)
    ko = np.zeros(len(keys), dtype=np.uint64)
    if len(keys):
        ko[1:] = np.cumsum(kl[:-1], dtype=np.uint64)
    return np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8).copy(), ko, kl


def debug_total_order(keys, split_points, comparator, order=None):
    """Partitions TotalOrderPartitioner gives the serialized keys with these split points, computed on the host with the
    device's checks and search (tezgpu_debug_total_order_emulate).  order: search order (default: the comparator)."""
    L = _lib.load()
    kv, ko, kl = _pack_keys(keys)
    sv, so, sl = _pack_keys(split_points)
    part = np.zeros(max(1, len(keys)), dtype=np.int32)
    check(L.tezgpu_debug_total_order_emulate(_ptr(kv), _ptr(ko), _ptr(kl), len(keys), _ptr(sv), _ptr(so), _ptr(sl),
                                             len(split_points), comparator, comparator if order is None else order,
                                             _ptr(part)))
    return part[:len(keys)]


def debug_stitched_compress(codec, body, cuts):
    """The codec stream a bounded merge's compressed write gives one partition body that its steps cut at the offsets
    `cuts`, computed on the host with the device path's chunk grid, carry and folds (tezgpu_debug_stitched_compress_emulate).
    It equals the codec's stream of the uncut body."""
    L = _lib.load()
    body = bytes(body)
    c = np.ascontiguousarray(cuts, dtype=np.uint64)
    cap = len(body) + len(body) // 255 + 16 * (len(body) // 32768 + 2) + 64
    out = np.empty(cap, dtype=np.uint8)
    n = C.c_uint64()
    check(L.tezgpu_debug_stitched_compress_emulate(codec, body, len(body), _ptr(c) if c.size else None, c.size, _ptr(out), cap,
                                                   C.byref(n)))
    return out[:n.value].tobytes()


KeySample = collections.namedtuple("KeySample", "keys key_off key_len h gid")
KeySample.__doc__ = """A sample of tezgpu_sample_keys, in gid order (numpy): keys uint8 (the keys back to back), key_off uint64,
key_len uint32, h uint64 (splitmix64(seed ^ gid)), gid uint64 (the records' global numbers)."""


def sample_keys(d_kv, kv_bytes, d_key_off, d_val_off, d_val_len, n, seed, freq, max_samples, gid_base=0, device=0):
    """RandomSampler on the device (tezgpu_sample_keys): a sample of the keys of device-resident records given as
    GpuSorter.sort_device's input (raw device pointers as ints).  Record i is numbered gid_base + i; it is a candidate
    when splitmix64(seed ^ gid) < freq * 2^64, and of more than max_samples candidates those with the smallest
    (h, gid) are kept.  Returns a KeySample."""
    L = _lib.load()
    m = max(1, int(max_samples))
    ko, kl = np.empty(m, dtype=np.uint64), np.empty(m, dtype=np.uint32)
    h, gid = np.empty(m, dtype=np.uint64), np.empty(m, dtype=np.uint64)
    count, need = C.c_uint32(), C.c_uint64()
    keys = np.empty(max(4096, min(int(n), m) * 32), dtype=np.uint8)
    while True:
        rc = L.tezgpu_sample_keys(device, d_kv, kv_bytes, d_key_off, d_val_off, d_val_len, n, gid_base, seed, float(freq),
                                  max_samples, _ptr(keys), keys.size, _ptr(ko), _ptr(kl), _ptr(h), _ptr(gid), C.byref(count),
                                  C.byref(need))
        if rc == E_NOMEM and need.value > keys.size:
            keys = np.empty(need.value, dtype=np.uint8)
            continue
        check(rc)
        c = count.value
        return KeySample(keys[:need.value].copy(), ko[:c].copy(), kl[:c].copy(), h[:c].copy(), gid[:c].copy())


def concat_samples(samples):
    """The union of several KeySamples as one (keys rebased), e.g. every rank's sample."""
    samples = list(samples)
    if len(samples) == 1:
        return samples[0]
    base = np.cumsum([0] + [s.keys.size for s in samples[:-1]]).astype(np.uint64)
    return KeySample(np.concatenate([s.keys for s in samples]).astype(np.uint8),
                     np.concatenate([s.key_off + b for s, b in zip(samples, base)]).astype(np.uint64),
                     np.concatenate([s.key_len for s in samples]).astype(np.uint32),
                     np.concatenate([s.h for s in samples]).astype(np.uint64),
                     np.concatenate([s.gid for s in samples]).astype(np.uint64))


def sample_key_list(sample):
    """The keys of a KeySample as a list of bytes."""
    raw = sample.keys.tobytes()
    return [raw[o:o + ln] for o, ln in zip(sample.key_off.tolist(), sample.key_len.tolist())]


def select_split_points(samples, num_partitions, max_samples, comparator, order=None, device=0, with_chosen=False):
    """InputSampler.writePartitionFile on the device (tezgpu_select_split_points): the union of the KeySamples capped to
    the max_samples smallest (h, gid), sorted under `comparator` on the device, and the num_partitions - 1 split points
    picked by writePartitionFile's rule.  Returns the serialized split keys, the list GpuSorter(partitioner=PART_TOTAL_ORDER,
    split_points=...) takes, searched in `order` (None = the comparator); with_chosen also their indices in the sorted
    sample."""
    L = _lib.load()
    s = concat_samples([samples] if isinstance(samples, KeySample) else samples)
    P = int(num_partitions)
    so, sl = np.empty(max(1, P - 1), dtype=np.uint64), np.empty(max(1, P - 1), dtype=np.uint32)
    chosen = np.empty(max(1, P - 1), dtype=np.uint64)
    need = C.c_uint64()
    out = np.empty(max(16, int(s.key_len.max(initial=0)) * max(0, P - 1)), dtype=np.uint8)   # every split at the longest key
    check(L.tezgpu_select_split_points(device, comparator, comparator if order is None else order, P, max_samples,
                                       _ptr(s.keys if s.keys.size else np.zeros(1, np.uint8)), _ptr(s.key_off), _ptr(s.key_len),
                                       _ptr(s.h), _ptr(s.gid), s.gid.size, _ptr(out), out.size, _ptr(so), _ptr(sl),
                                       C.byref(need), _ptr(chosen)))
    raw = out[:need.value].tobytes()
    splits = [raw[o:o + ln] for o, ln in zip(so[:P - 1].tolist(), sl[:P - 1].tolist())]
    return (splits, chosen[:P - 1].copy()) if with_chosen else splits


def decode_segments(segs, raw_lens, codec, budget, device=0):
    """The compressed (TIF\\x01) host segments among segs decoded on the device under a budget of device bytes
    (tezgpu_decode_segments).  Returns (images, peak device bytes): images[i] is segment i's uncompressed IFile segment
    (TIF\\x00, body, CRC-32 of the body; raw_lens[i] + 4 bytes) or None for a segment that is not compressed."""
    L = _lib.load()
    keep = [np.ascontiguousarray(np.frombuffer(s, dtype=np.uint8) if isinstance(s, (bytes, bytearray)) else s, dtype=np.uint8)
            for s in segs]
    arr = (Segment * max(1, len(keep)))()
    imgs = [None] * len(keep)
    out = (C.c_void_p * max(1, len(keep)))()
    for i, a in enumerate(keep):
        arr[i].data = a.ctypes.data if a.size else None
        arr[i].len = a.size
        arr[i].flags = SEG_HAS_HEADER
        if raw_lens is not None and a.size >= 10 and bytes(a[:4]) == b"TIF\x01":
            imgs[i] = np.empty(int(raw_lens[i]) + 4, dtype=np.uint8)
            out[i] = imgs[i].ctypes.data
    raw = None if raw_lens is None else np.ascontiguousarray(raw_lens, dtype=np.int64)
    conf = make_conf(1, partitioner=PART_GIVEN, device=device)
    peak = C.c_uint64()
    check(L.tezgpu_decode_segments(C.byref(conf), arr, _ptr(raw), len(keep), codec, int(budget), out, C.byref(peak)))
    return [None if m is None else m.tobytes() for m in imgs], peak.value


class GpuSorter:
    def __init__(self, num_partitions, combiner=COMBINE_NONE, codec=CODEC_NONE, split_points=None, split_order=None, **kw):
        """combiner: COMBINE_SUM_INT / COMBINE_SUM_LONG runs MRCombiner with IntSumReducer / LongSumReducer on every
        flush (tezgpu_sorter_set_combiner).  codec: CODEC_DEFAULT writes zlib-compressed segments, CODEC_LZ4 Lz4Codec
        segments (blocks of LZ4_BLOCK_BYTES raw bytes, one chunk each), CODEC_ZSTD ZStandardCodec segments (one frame per
        ZSTD_BLOCK_BYTES raw bytes), CODEC_SNAPPY SnappyCodec segments (blocks of SNAPPY_BLOCK_BYTES raw bytes, one chunk
        each) (tezgpu_sorter_set_codec).  split_points: the serialized split keys of a
        partitioner=PART_TOTAL_ORDER handle, searched in split_order (a CMP_*; None = the handle's comparator)
        (tezgpu_sorter_set_split_points)."""
        self.L = _lib.load()
        self.conf = make_conf(num_partitions, **kw)
        self.P = num_partitions
        self.h = C.c_void_p()
        check(self.L.tezgpu_sorter_create(C.byref(self.conf), C.byref(self.h)))
        try:
            if combiner:
                self.set_combiner(combiner)
            if codec:
                self.set_codec(codec)
            if split_points is not None:
                self.set_split_points(split_points, split_order)
        except Exception:
            self.close()
            raise

    def set_combiner(self, combiner):
        """Before the first collect (or after reset); survives reset."""
        check(self.L.tezgpu_sorter_set_combiner(self.h, combiner))

    def set_codec(self, codec):
        """CODEC_NONE / CODEC_DEFAULT / CODEC_LZ4 / CODEC_ZSTD / CODEC_SNAPPY; before the first collect (or after reset); survives reset."""
        check(self.L.tezgpu_sorter_set_codec(self.h, codec))

    def set_split_points(self, split_points, order=None):
        """TotalOrderPartitioner split keys; before the first collect (or after reset); survives reset."""
        kv, ko, kl = _pack_keys(split_points)
        check(self.L.tezgpu_sorter_set_split_points(self.h, _ptr(kv), _ptr(ko), _ptr(kl), len(split_points),
                                                    self.conf.comparator if order is None else order))

    def close(self):
        if self.h:
            self.L.tezgpu_sorter_destroy(self.h)
            self.h = C.c_void_p()

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def collect(self, kv, key_off, val_off, val_len, partition=None):
        kv = np.ascontiguousarray(np.frombuffer(kv, dtype=np.uint8) if isinstance(kv, (bytes, bytearray)) else kv,
                                  dtype=np.uint8)
        key_off = np.ascontiguousarray(key_off, dtype=np.uint32)
        val_off = np.ascontiguousarray(val_off, dtype=np.uint32)
        val_len = np.ascontiguousarray(val_len, dtype=np.uint32)
        if partition is not None:
            partition = np.ascontiguousarray(partition, dtype=np.int32)
        check(self.L.tezgpu_sorter_collect_batch(self.h, _ptr(kv), kv.size, _ptr(key_off), _ptr(val_off),
                                                 _ptr(val_len), _ptr(partition), len(key_off)))

    def collect_fixed(self, kv, partition=None, n=None):
        if isinstance(kv, int):  # raw host pointer (pinned memory)
            p = kv
        else:
            kv = np.ascontiguousarray(kv, dtype=np.uint8)
            p = kv.ctypes.data
            if n is None:
                n = kv.size // (self.conf.fixed_key_len + self.conf.fixed_val_len)
        if partition is not None:
            partition = np.ascontiguousarray(partition, dtype=np.int32)
        check(self.L.tezgpu_sorter_collect_fixed(self.h, p, _ptr(partition), n))

    def reset(self):
        check(self.L.tezgpu_sorter_reset(self.h))

    def output_bound(self):
        return self.L.tezgpu_sorter_output_bound(self.h)

    def flush_to_memory(self, out=None):
        """Returns (file_out uint8 array view, index_bytes, index[P,3], stats dict)."""
        if out is None:
            out = np.empty(self.output_bound(), dtype=np.uint8)
        cap = out.size
        n = C.c_uint64()
        index = np.zeros((self.P, 3), dtype=np.int64)
        index_bytes = np.zeros(self.P * 24 + 8, dtype=np.uint8)
        st = Stats()
        check(self.L.tezgpu_sorter_flush_to_memory(self.h, _ptr(out), cap, C.byref(n), _ptr(index_bytes), _ptr(index),
                                                   C.byref(st)))
        return out[:n.value], index_bytes.tobytes(), index, st.as_dict()

    def flush(self, out_path, index_path):
        index = np.zeros((self.P, 3), dtype=np.int64)
        st = Stats()
        check(self.L.tezgpu_sorter_flush(self.h, out_path.encode(), index_path.encode(), _ptr(index), C.byref(st)))
        return index, st.as_dict()

    def sort_device_fixed(self, d_kv, n, d_out, out_cap, d_partition=None):
        """Device-resident records (raw device pointers as ints). Returns (out_len, index, stats)."""
        out_len = C.c_uint64()
        index = np.zeros((self.P, 3), dtype=np.int64)
        st = Stats()
        check(self.L.tezgpu_sorter_sort_device_fixed(self.h, d_kv, d_partition, n, d_out, out_cap, C.byref(out_len),
                                                     _ptr(index), C.byref(st)))
        return out_len.value, index, st.as_dict()

    def sort_device(self, d_kv, kv_bytes, d_key_off, d_val_off, d_val_len, n, d_out, out_cap, d_partition=None):
        """Device-resident variable-length records (raw device pointers as ints): record i's key is
        kv[key_off[i] .. val_off[i]) and its value kv[val_off[i] .. + val_len[i]) with uint64 offsets, uint32 value
        lengths and optional int32 partition ids, all on the handle's device.  Sorts in one call into d_out.  Returns
        (out_len, index, stats)."""
        out_len = C.c_uint64()
        index = np.zeros((self.P, 3), dtype=np.int64)
        st = Stats()
        check(self.L.tezgpu_sorter_sort_device(self.h, d_kv, kv_bytes, d_key_off, d_val_off, d_val_len, d_partition, n, d_out,
                                               out_cap, C.byref(out_len), _ptr(index), C.byref(st)))
        return out_len.value, index, st.as_dict()

    def device_output_bound(self, n, kv_bytes):
        """out_cap that sort_device always fits for n records in a buffer of kv_bytes."""
        return self.L.tezgpu_sorter_device_output_bound(self.h, n, kv_bytes)

    def stream(self):
        return self.L.tezgpu_sorter_stream(self.h)


class GpuMerger:
    def __init__(self, segments, comparator=CMP_BYTES, device=0, has_header=True, device_ptrs=False, fixed=None,
                 partitions=None, num_partitions=1, send_empty=True, verified=None, combiner=COMBINE_NONE,
                 codec=CODEC_NONE, raw_lens=None, concat=False, device_budget=None, write_codec=None):
        """segments: list of bytes / uint8 arrays (host) or (ptr, len) tuples when device_ptrs.
        verified: optional per-segment booleans -- the transport already checked that segment's checksum
        (TEZGPU_SEG_VERIFIED: fetch_segments_verified), the merge does not read it again to verify.
        combiner: COMBINE_SUM_INT / COMBINE_SUM_LONG combines the merged stream in write_* (tezgpu_merge_set_combiner).
        codec: CODEC_DEFAULT (zlib), CODEC_LZ4 (Lz4Codec), CODEC_ZSTD (ZStandardCodec) or CODEC_SNAPPY (SnappyCodec) reads
        compressed (TIF\\x01) segments of that codec and writes compressed output (tezgpu_merge_open_codec); raw_lens: per-segment rawLength, required for the compressed
        segments.
        concat: UnorderedPartitionedKVWriter.mergeAll / UnorderedKVReader (tezgpu_concat_open): records leave in
        (segment, position) order, the writes copy the record bytes (rle must be False).
        device_budget: bytes of device memory the merge may hold (tezgpu_merge_open_bounded; 0 = the free memory):
        host segments larger than that merge in key-range steps, with the same stream and output.
        write_codec (with device_budget): the bounded merge of uncompressed host segments writes segments of this codec
        (tezgpu_merge_open_bounded_write_codec), byte for byte what GpuMerger(codec=write_codec) writes."""
        self.h = C.c_void_p()
        if write_codec is not None and device_budget is None:
            raise ValueError("write_codec is the codec of a bounded merge's writes: it needs device_budget (codec= otherwise)")
        self.L = _lib.load()
        self.conf = make_conf(num_partitions, comparator=comparator, partitioner=PART_GIVEN, device=device, fixed=fixed,
                              send_empty=send_empty)
        self.P = num_partitions
        self._has_header, self._device_ptrs = has_header, device_ptrs
        arr = self._segments(segments, partitions, verified)
        self.h = C.c_void_p()
        self.bounded = device_budget is not None
        if write_codec is not None:
            check(self.L.tezgpu_merge_open_bounded_write_codec(C.byref(self.conf), arr, len(segments), write_codec,
                                                               int(device_budget), C.byref(self.h)))
        elif self.bounded:
            check(self.L.tezgpu_merge_open_bounded(C.byref(self.conf), arr, _ptr(self._raw(raw_lens)), len(segments), codec,
                                                   int(device_budget), C.byref(self.h)))
        elif concat:
            check(self.L.tezgpu_concat_open(C.byref(self.conf), arr, _ptr(self._raw(raw_lens)), len(segments), codec,
                                            C.byref(self.h)))
        elif codec:
            check(self.L.tezgpu_merge_open_codec(C.byref(self.conf), arr, _ptr(self._raw(raw_lens)), len(segments), codec,
                                                 C.byref(self.h)))
        else:
            check(self.L.tezgpu_merge_open(C.byref(self.conf), arr, len(segments), C.byref(self.h)))
        self.codec = codec
        if combiner:
            try:
                self.set_combiner(combiner)
            except Exception:
                self.close()
                raise

    def set_combiner(self, combiner):
        """Combines in write_*; the record iterator is then unavailable (TEZGPU_E_STATE)."""
        check(self.L.tezgpu_merge_set_combiner(self.h, combiner))

    def _segments(self, segments, partitions, verified=None):
        self._keep = []
        arr = (Segment * max(1, len(segments)))()
        flags = (SEG_HAS_HEADER if self._has_header else 0) | (SEG_DEVICE if self._device_ptrs else 0)
        if self._device_ptrs and len(segments) > 64:
            # many device-resident runs (the reduce side of the multi-GPU shuffle): fill the table through numpy
            tab = np.zeros(len(segments), dtype=np.dtype([("data", "<u8"), ("len", "<u8"), ("flags", "<u4"), ("partition", "<u4")]))
            sp = np.asarray(segments, dtype=np.uint64).reshape(-1, 2)
            tab["data"], tab["len"], tab["flags"] = sp[:, 0], sp[:, 1], flags
            if verified is not None:
                tab["flags"] |= np.where(np.asarray(verified, dtype=bool), SEG_VERIFIED, 0).astype(np.uint32)
            if partitions is not None:
                tab["partition"] = np.asarray(partitions, dtype=np.uint32)
            self._keep.append(tab)
            return C.cast(tab.ctypes.data, C.POINTER(Segment))
        for i, s in enumerate(segments):
            if self._device_ptrs:
                arr[i].data, arr[i].len = s
            else:
                a = np.ascontiguousarray(np.frombuffer(s, dtype=np.uint8) if isinstance(s, (bytes, bytearray)) else s)
                self._keep.append(a)
                arr[i].data = a.ctypes.data if a.size else None
                arr[i].len = a.size
            arr[i].flags = flags | (SEG_VERIFIED if (verified is not None and verified[i]) else 0)
            arr[i].partition = 0 if partitions is None else int(partitions[i])
        return arr

    def _raw(self, raw_lens):
        self._raw_keep = None if raw_lens is None else np.ascontiguousarray(raw_lens, dtype=np.int64)
        return self._raw_keep

    def reopen(self, segments, partitions=None, verified=None, raw_lens=None):
        """New merge through the same handle (device allocations are kept)."""
        arr = self._segments(segments, partitions, verified)
        if self.codec:
            check(self.L.tezgpu_merge_reopen_codec(self.h, arr, _ptr(self._raw(raw_lens)), len(segments)))
        else:
            check(self.L.tezgpu_merge_reopen(self.h, arr, len(segments)))

    def close(self):
        if self.h:
            self.L.tezgpu_merge_close(self.h)
            self.h = C.c_void_p()

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_check_for_same_keys(self, on):
        """MergeQueue's checkForSameKeys (SORT/TezMerger.java:560-573); default True."""
        check(self.L.tezgpu_merge_set_check_for_same_keys(self.h, 1 if on else 0))

    def parse_info(self):
        """(mode, windows walked by hand) of the last open: 0 records addressed in place, 1 window parser, 2 sequential walker."""
        m, r = C.c_int32(), C.c_int32()
        check(self.L.tezgpu_merge_parse_info(self.h, C.byref(m), C.byref(r)))
        return m.value, r.value

    def bounded_info(self):
        """(steps, peak device bytes, bytes uploaded from the host) of a merger opened with device_budget."""
        steps, peak, h2d = C.c_int32(), C.c_uint64(), C.c_uint64()
        check(self.L.tezgpu_merge_bounded_info(self.h, C.byref(steps), C.byref(peak), C.byref(h2d)))
        return steps.value, peak.value, h2d.value

    def counts(self):
        r, b = C.c_uint64(), C.c_uint64()
        check(self.L.tezgpu_merge_counts(self.h, C.byref(r), C.byref(b)))
        return r.value, b.value

    def records(self, batch_records=1 << 16, batch_bytes=1 << 24):
        """Iterates (key, value, is_same_key) like TezRawKeyValueIterator.next/getKey/getValue/isSameKey.  The batch
        buffer grows to fit a record larger than batch_bytes."""
        buf = np.empty(batch_bytes, dtype=np.uint8)
        idx = (KvIndex * batch_records)()
        n = C.c_uint32()
        while True:
            rc = self.L.tezgpu_merge_next_batch(self.h, _ptr(buf), buf.size, idx, batch_records, C.byref(n))
            if rc == E_NOMEM and n.value == 0 and idx[0].key_len + idx[0].val_len > buf.size:
                buf = np.empty(idx[0].key_len + idx[0].val_len, dtype=np.uint8)
                continue
            check(rc)
            if n.value == 0:
                return
            raw = buf.tobytes()
            for i in range(n.value):
                e = idx[i]
                yield (raw[e.key_off:e.key_off + e.key_len], raw[e.val_off:e.val_off + e.val_len], bool(e.same_key))

    def next_batch_device(self, d_kv, kv_cap, d_key_off, d_val_off, d_val_len, d_same_key=None, idx_cap=1 << 16):
        """The next records of the merged stream written into device memory (raw device pointers as ints, on the
        handle's device; d_kv 16-byte aligned): record i's key is kv[key_off[i] .. val_off[i]) and its value
        kv[val_off[i] .. + val_len[i]), with uint64 offsets, uint32 value lengths and uint8 isSameKey flags, packed back
        to back from kv[0] (tezgpu_merge_next_batch_device).  Returns (n, kv_bytes) once the batch is written; n = 0 at
        the end of the stream.  A record larger than kv_cap raises TezGpuError(E_NOMEM) whose `needed` is the bytes it
        needs; the stream stays where it was.  The call runs on the merger's own stream (stream()), which nothing orders
        after the caller's: work the caller queued on the buffers must be complete, or waited for, before the call."""
        n, kvb = C.c_uint32(), C.c_uint64()
        rc = self.L.tezgpu_merge_next_batch_device(self.h, d_kv, kv_cap, d_key_off, d_val_off, d_val_len, d_same_key,
                                                   idx_cap, C.byref(n), C.byref(kvb))
        try:
            check(rc)
        except _lib.TezGpuError as e:
            e.needed = kvb.value if rc == E_NOMEM else 0
            raise
        return n.value, kvb.value

    def records_device(self, batch_records=1 << 16, batch_bytes=1 << 24):
        """The device twin of records(): yields one batch at a time as torch CUDA tensor views (kv uint8, key_off int64,
        val_off int64, val_len int32, same_key uint8) over buffers the next batch reuses; the offsets are the uint64 /
        uint32 values of next_batch_device.  The kv buffer grows to fit a record larger than batch_bytes.  Work the
        consumer queues on the views on torch's current stream may still be running when it asks for the next batch:
        the merger's stream waits for that stream before it writes the buffers again."""
        import torch
        dev = torch.device("cuda", self.conf.device)
        mine = torch.cuda.ExternalStream(self.stream(), device=dev)
        kv = torch.empty(batch_bytes, dtype=torch.uint8, device=dev)
        ko = torch.empty(batch_records, dtype=torch.int64, device=dev)
        vo = torch.empty(batch_records, dtype=torch.int64, device=dev)
        vl = torch.empty(batch_records, dtype=torch.int32, device=dev)
        sk = torch.empty(batch_records, dtype=torch.uint8, device=dev)
        while True:
            mine.wait_stream(torch.cuda.current_stream(dev))
            try:
                n, b = self.next_batch_device(kv.data_ptr(), kv.numel(), ko.data_ptr(), vo.data_ptr(), vl.data_ptr(),
                                              sk.data_ptr(), batch_records)
            except _lib.TezGpuError as e:
                if e.code != E_NOMEM or e.needed <= kv.numel():
                    raise
                kv = torch.empty(e.needed, dtype=torch.uint8, device=dev)
                continue
            if n == 0:
                return
            yield kv[:b], ko[:n], vo[:n], vl[:n], sk[:n]

    def output_bound(self):
        return self.L.tezgpu_merge_output_bound(self.h)

    def write_ifile(self, rle=False, path=None):
        """TezMerger.writeFile into an IFile.Writer(rle). Returns (segment bytes or None, rawLen, partLen, stats)."""
        raw, part = C.c_int64(), C.c_int64()
        st = Stats()
        if path is not None:
            check(self.L.tezgpu_merge_write_ifile(self.h, path.encode(), None, 0, 1 if rle else 0, C.byref(raw),
                                                  C.byref(part), C.byref(st)))
            return None, raw.value, part.value, st.as_dict()
        bound = self.output_bound()
        if bound == 0 and self.bounded:
            # a merge in several steps knows its output size only once it has run: write through a file
            with tempfile.TemporaryDirectory() as d:
                f = os.path.join(d, "merged")
                _, raw_len, part_len, stats = self.write_ifile(rle, f)
                with open(f, "rb") as fh:
                    return fh.read(), raw_len, part_len, stats
        out = np.empty(bound, dtype=np.uint8)
        check(self.L.tezgpu_merge_write_ifile(self.h, None, _ptr(out), out.size, 1 if rle else 0, C.byref(raw),
                                              C.byref(part), C.byref(st)))
        return out[:part.value].tobytes(), raw.value, part.value, st.as_dict()

    def write_ifile_device(self, d_out, out_cap, rle=False):
        raw, part = C.c_int64(), C.c_int64()
        st = Stats()
        check(self.L.tezgpu_merge_write_ifile_device(self.h, d_out, out_cap, 1 if rle else 0, C.byref(raw),
                                                     C.byref(part), C.byref(st)))
        return raw.value, part.value, st.as_dict()

    def write_partitions(self, out_path, index_path, rle=False):
        """file.out + file.out.index of the merged partitions. Returns (index[P,3], stats)."""
        index = np.zeros((self.P, 3), dtype=np.int64)
        st = Stats()
        check(self.L.tezgpu_merge_write_partitions(self.h, out_path.encode(), index_path.encode(), 1 if rle else 0,
                                                   _ptr(index), C.byref(st)))
        return index, st.as_dict()

    def write_partitions_device(self, d_out, out_cap, rle=False):
        """Batched reduce side: P merged segments back to back. Returns (out_len, index[P,3], stats)."""
        n = C.c_uint64()
        index = np.zeros((self.P, 3), dtype=np.int64)
        st = Stats()
        check(self.L.tezgpu_merge_write_partitions_device(self.h, d_out, out_cap, 1 if rle else 0, C.byref(n), _ptr(index),
                                                          C.byref(st)))
        return n.value, index, st.as_dict()

    def stream(self):
        return self.L.tezgpu_merge_stream(self.h)


class PeerBuffer:
    """Device buffer other processes of the box can map (tezgpu_peer_alloc): where a producer keeps file.out."""

    def __init__(self, nbytes, device=0):
        self.L = _lib.load()
        self.device, self.nbytes = device, int(nbytes)
        p = C.c_void_p()
        handle = (C.c_uint8 * 64)()
        check(self.L.tezgpu_peer_alloc(device, self.nbytes, C.byref(p), handle))
        self.ptr, self.handle = p.value, bytes(handle)

    def close(self):
        if self.ptr:
            check(self.L.tezgpu_peer_free(self.device, self.ptr))
            self.ptr = None


class PeerMapping:
    """A peer's exported buffer mapped into this process (tezgpu_peer_open)."""

    def __init__(self, handle, device=0):
        self.L = _lib.load()
        self.device = device
        p = C.c_void_p()
        buf = (C.c_uint8 * 64).from_buffer_copy(handle)
        check(self.L.tezgpu_peer_open(device, buf, C.byref(p)))
        self.ptr = p.value

    def close(self):
        if self.ptr:
            check(self.L.tezgpu_peer_close(self.device, self.ptr))
            self.ptr = None


FETCH_SEG_DTYPE = np.dtype([("src", "<u8"), ("dst", "<u8"), ("len", "<u8"), ("flags", "<u4"), ("reserved", "<u4")])


def fetch_segments_verified(segs, device=0, stream=None, has_header=True):
    """segs: iterable of (src_ptr, dst_ptr, nbytes) -- one IFile segment each.  One launch copies them and verifies every
    segment's CRC32 trailer on the bytes in flight (IFile.Reader.readToMemory); raises TezGpuError(TEZGPU_E_FORMAT) on a
    mismatch.  Returns the copy kernel's time in ms."""
    L = _lib.load()
    tab = np.zeros(len(segs), dtype=FETCH_SEG_DTYPE)
    if len(segs):
        a = np.asarray(segs, dtype=np.uint64).reshape(-1, 3)
        tab["src"], tab["dst"], tab["len"] = a[:, 0], a[:, 1], a[:, 2]
        tab["flags"] = SEG_HAS_HEADER if has_header else 0
    ms = C.c_float()
    check(L.tezgpu_fetch_segments_verified(device, tab.ctypes.data, len(segs), stream, C.byref(ms)))
    return ms.value


def fetch_ranges(ranges, device=0, stream=None):
    """ranges: list of (src_ptr, dst_ptr, nbytes) device addresses; one launch, returns the kernel time in ms."""
    L = _lib.load()
    arr = (_lib.CopyRange * max(1, len(ranges)))()
    for i, (s, d, n) in enumerate(ranges):
        arr[i].src, arr[i].dst, arr[i].len = s, d, n
    ms = C.c_float()
    check(L.tezgpu_fetch_ranges(device, arr, len(ranges), stream, C.byref(ms)))
    return ms.value


# ---------------------------------------------------------------- SURVEY 8 f-2: ShuffleHandler <-> fetcher wire format
def shuffle_header(map_id, part_len, raw_len, reduce):
    """ShuffleHeader.write (OG/ShuffleHeader.java:101-106) -> bytes."""
    L = _lib.load()
    mid = map_id.encode("utf-8")
    buf = (C.c_uint8 * (len(mid) + 64))()
    n = C.c_uint64()
    check(L.tezgpu_shuffle_header_write(mid, part_len, raw_len, reduce, buf, len(buf), C.byref(n)))
    assert n.value == L.tezgpu_shuffle_header_size(mid, part_len, raw_len, reduce)
    return bytes(buf[:n.value])


def read_shuffle_header(data):
    """ShuffleHeader.readFields -> (map_id, part_len, raw_len, reduce, header bytes consumed)."""
    L = _lib.load()
    mid = C.create_string_buffer(1008)
    pl, rl, rd, used = C.c_int64(), C.c_int64(), C.c_int32(), C.c_uint64()
    raw = bytes(data)
    check(L.tezgpu_shuffle_header_read(raw, len(raw), mid, len(mid), C.byref(pl), C.byref(rl), C.byref(rd), C.byref(used)))
    return mid.value.decode("utf-8"), pl.value, rl.value, rd.value, used.value


def shuffle_serve(d_file_out, index, map_id, reduce0, nreduce, device=0, stream=None):
    """Response body ShuffleHandler sends for reducers [reduce0, reduce0 + nreduce) of one map output whose file.out is in
    device memory (d_file_out = device pointer, index = (P, 3) int64 spill index) -> bytes."""
    L = _lib.load()
    idx = np.ascontiguousarray(index, dtype=np.int64)
    mid = map_id.encode("utf-8")
    cap = L.tezgpu_shuffle_serve_bound(mid, idx.ctypes.data, reduce0, nreduce)
    out = np.empty(max(1, cap), dtype=np.uint8)
    n = C.c_uint64()
    check(L.tezgpu_shuffle_serve(device, d_file_out, idx.ctypes.data, mid, reduce0, nreduce, out.ctypes.data, cap, C.byref(n), stream))
    return out[:n.value].tobytes()


def shuffle_receive(body):
    """Splits a response body into [(map_id, reduce, raw_len, segment bytes)] the way FetcherOrderedGrouped.copyMapOutput
    walks it (header, then compressedLength bytes)."""
    L = _lib.load()
    raw = bytes(body)
    n = C.c_uint32()
    cap = 64
    while True:
        tab = (_lib.WireSegment * cap)()
        rc = L.tezgpu_shuffle_receive(raw, len(raw), tab, cap, C.byref(n))
        if rc != 0 and n.value > cap:
            cap = n.value
            continue
        check(rc)
        break
    return [(s.map_id.decode("utf-8"), s.reduce, s.raw_len, raw[s.offset:s.offset + s.part_len]) for s in tab[:n.value]]

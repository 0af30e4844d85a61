"""Shared helpers of the map-side radix sort tests (test_radix_edges_cpu.py, test_radix_edges_gpu.py): record builders,
digit-shaped key sets, the host reference of the sort (a stable numpy sort on (partition, normalised key)), the file.out
it implies, and a device checker for sorts too large for the host.

Keys are handled as their *normalised* value: the unsigned integer whose order is the comparator's order.  CMP_BYTES keys
serialize it big-endian; CMP_INT / CMP_LONG keys flip its top bit (the sign).  Every record's value is a 4-byte
big-endian word, by default the record's collection index, so that the permutation and the order of ties can be read
back from file.out."""
import zlib

import numpy as np

from oracle import tez_oracle as O

# the 32-bit onesweep pass (radix_sort.cuh): 384 threads x 16 keys per tile, 75,840 bytes of shared memory and 80
# registers per thread
RADIX_THREADS, RADIX_IPT = 384, 16
TILE = RADIX_THREADS * RADIX_IPT
RADIX_SMEM, RADIX_REGS = 75840, 80
RADIX_MAX_N = (1 << 30) - 1
EOF_CRC = zlib.crc32(b"\xff\xff")

CONST_SHAPES = ["const%x" % m for m in range(16)]   # bit b of m: byte b (pass b, least significant first) is constant
SHAPES = CONST_SHAPES + ["zeros", "ones", "alternating", "ascending", "descending", "outlier_first", "outlier_last",
                         "ff_last", "zipf", "uniform"]
LOW_SHAPES = ["uniform", "outlier"]                  # the low word of 8-byte keys


def resident_ctas(props):
    """Onesweep CTAs one SM holds at once: threads, shared memory and registers of the 32-bit pass."""
    return min(props.max_threads_per_multi_processor // RADIX_THREADS,
               props.shared_memory_per_multiprocessor // (RADIX_SMEM + 1024),
               props.regs_per_multiprocessor // (RADIX_THREADS * RADIX_REGS))


def wave_records(props):
    """Records one full wave of onesweep tiles covers on this device."""
    return props.multi_processor_count * resident_ctas(props) * TILE


# ------------------------------------------------------------------------------------------------ key shapes
def _rng(seed, *salt):
    return np.random.default_rng([seed] + [int(s) for s in salt])


def _bytes_of(rng, shape, lo, hi):
    """n x 4 bytes in [lo, hi] composed into uint32 values, byte 3 most significant"""
    b = rng.integers(lo, hi + 1, shape + (4,), dtype=np.uint64)
    return ((b[..., 3] << 24) | (b[..., 2] << 16) | (b[..., 1] << 8) | b[..., 0]).astype(np.uint32)


def shape_keys(shape, n, seed):
    """n normalised 32-bit keys (uint32) of one digit shape; a function of (shape, n, seed) alone."""
    r = _rng(seed, SHAPES.index(shape), n)
    i = np.arange(n, dtype=np.int64)
    u = r.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    if shape in CONST_SHAPES:
        mask = int(shape[5:], 16)
        c = r.integers(0, 256, 4, dtype=np.uint32)
        for b in range(4):
            if (mask >> b) & 1:
                u = (u & np.uint32(~(0xFF << (8 * b)) & 0xFFFFFFFF)) | np.uint32(int(c[b]) << (8 * b))
        return u
    if shape == "zeros":
        return np.zeros(n, dtype=np.uint32)
    if shape == "ones":
        return np.full(n, 0xFFFFFFFF, dtype=np.uint32)
    if shape == "alternating":
        a = _bytes_of(r, (), 0x80, 0xFF)
        b = _bytes_of(r, (), 0x00, 0x7F)   # differs from a in every byte, and sorts first
        return np.where(i % 2 == 0, a, b).astype(np.uint32)
    if shape == "ascending":
        return np.sort(u)
    if shape == "descending":
        return np.sort(u)[::-1].copy()
    if shape in ("outlier_first", "outlier_last"):
        # every key equal except one per tile, at the tile's first (or last real) slot, differing in every byte: it
        # travels to the other end of the order (last for outlier_first, first for outlier_last)
        c = np.uint32(0x80808080)
        if shape == "outlier_first":
            o = _bytes_of(r, (n,), 0x81, 0xFF)
            at = i % TILE == 0
        else:
            o = _bytes_of(r, (n,), 0x00, 0x7F)
            at = (i % TILE == TILE - 1) | (i == n - 1)
        return np.where(at, o, c).astype(np.uint32)
    if shape == "ff_last":
        # no byte is 0xFF except in the last record, which is all 0xFF: digit 255 holds one key in every pass
        k = _bytes_of(r, (n,), 0x00, 0xFE)
        if n:
            k[-1] = 0xFFFFFFFF
        return k
    if shape == "zipf":
        ids = np.minimum(r.zipf(1.2, n), 1 << 20).astype(np.uint64)
        return ((ids * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    if shape == "uniform":
        return u
    raise ValueError(shape)


def shape_keys64(shape, low, n, seed):
    """n normalised 64-bit keys (uint64): the high word has the 32-bit shape, the low word is uniform or (outlier) one
    constant except for a smaller value in the last record, so one refinement digit holds all keys but one."""
    hi = shape_keys(shape, n, seed).astype(np.uint64)
    r = _rng(seed, 1000 + LOW_SHAPES.index(low), n)
    if low == "uniform":
        lo = r.integers(0, 1 << 32, n, dtype=np.uint64)
    else:
        lo = np.full(n, 0x80808080, dtype=np.uint64)
        if n:
            lo[-1] = 0x7F7F7F7F
    return (hi << np.uint64(32)) | lo


def distinct_keys(n, width, seed):
    """n distinct normalised keys of 4 or 8 bytes in random order (an odd multiplier is a bijection modulo 2^bits)"""
    r = _rng(seed, 77, n, width)
    bits = 8 * width
    mask = (1 << bits) - 1
    base = int(r.integers(0, 1 << 62)) & mask
    mul = (int(r.integers(0, 1 << 62)) * 2 + 1) & mask
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        k = (i * np.uint64(mul) + np.uint64(base))
    return (k & np.uint64(mask)).astype(np.uint32 if width == 4 else np.uint64)


def words(n, seed, distinct=True):
    """n lower-case words of 1-12 letters (distinct when asked), as bytes"""
    r = _rng(seed, 91, n)
    out, seen = [], set()
    while len(out) < n:
        ln = int(r.integers(1, 13))
        w = bytes(r.integers(97, 123, ln, dtype=np.uint8))
        if distinct and w in seen:
            continue
        seen.add(w)
        out.append(w)
    return out


# ------------------------------------------------------------------------------------------------ records
def serialize(norm, width, cmp):
    """uint8 [n, width]: the serialized keys of these normalised values"""
    dt = ">u4" if width == 4 else ">u8"
    v = np.asarray(norm).astype(np.uint32 if width == 4 else np.uint64)
    if cmp in (O.CMP_INT, O.CMP_LONG):
        v = v ^ (np.uint32(1 << 31) if width == 4 else np.uint64(1 << 63))
    return v.astype(dt).view(np.uint8).reshape(-1, width)


def key_hash_values(norm, width):
    """tie-blind values: a 32-bit function of the whole key (records with equal keys are equal records)"""
    v = np.asarray(norm).astype(np.uint64)
    with np.errstate(over="ignore"):
        h = (v * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(32)
    return h.astype(np.uint32)


def fixed_records(norm, width, cmp, values=None):
    """uint8 [n, width + 4]: serialized key, then a 4-byte big-endian value (default: the collection index)"""
    n = len(norm)
    v = np.arange(n, dtype=np.uint32) if values is None else np.asarray(values, dtype=np.uint32)
    rec = np.empty((n, width + 4), dtype=np.uint8)
    rec[:, :width] = serialize(norm, width, cmp)
    rec[:, width:] = v.astype(">u4").view(np.uint8).reshape(-1, 4)
    return rec


def var_keys(contents, cmp):
    """serialized Text / BytesWritable keys of these contents"""
    if cmp == O.CMP_TEXT:
        return [O.text(c) for c in contents]
    assert cmp == O.CMP_BYTESWRITABLE
    return [len(c).to_bytes(4, "big") + c for c in contents]


def var_batch(keys, values=None):
    """(kv, key_off, val_off, val_len) of collect_batch for keys with 4-byte values (default: the collection index)"""
    n = len(keys)
    vals = [int(i).to_bytes(4, "big") for i in (range(n) if values is None else values)]
    kv = b"".join(k + v for k, v in zip(keys, vals))
    kl = np.array([len(k) for k in keys], dtype=np.uint32)
    key_off = (np.cumsum(kl + 4, dtype=np.uint64) - (kl + 4)).astype(np.uint32)
    return kv, key_off, key_off + kl, np.full(n, 4, dtype=np.uint32)


def framed_fixed(rec):
    """(framed bytes, record offsets) of fixed-width records: vint(klen) vint(vlen) key value, back to back"""
    n, w = rec.shape
    klen = w - 4
    fr = np.empty((n, w + 2), dtype=np.uint8)
    fr[:, 0], fr[:, 1] = klen, 4     # both lengths are below 128: one-byte vints
    fr[:, 2:] = rec
    return fr.reshape(-1), np.arange(n + 1, dtype=np.int64) * (w + 2)


def framed_var(keys, values=None):
    n = len(keys)
    vals = [int(i).to_bytes(4, "big") for i in (range(n) if values is None else values)]
    recs = [O.vint(len(k)) + O.vint(4) + k + v for k, v in zip(keys, vals)]
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(r) for r in recs])
    return np.frombuffer(b"".join(recs), dtype=np.uint8), off


# ------------------------------------------------------------------------------------------------ partition widths
KINDS = ["fixed4", "fixed8", "text", "bytes"]


def width_cases():
    """P = 2^k and 2^k + 1 for k = 1..24 (pbits 1..25), each with an ordered and an unordered handle.  The key kind,
    comparator, partitioner and send_empty rotate with k so that every one meets every handle at low and high pbits."""
    out = []
    for k in range(1, 25):
        for j, P in enumerate((1 << k, (1 << k) + 1)):
            for u in (False, True):
                kind = KINDS[(k + j + 1 + (2 if u else 0)) % 4]
                hashed = (k + j + u) % 2 == 0
                cmp = {"fixed4": O.CMP_INT if k % 2 else O.CMP_BYTES, "fixed8": O.CMP_LONG if k % 2 else O.CMP_BYTES,
                       "text": O.CMP_TEXT, "bytes": O.CMP_BYTESWRITABLE}[kind]
                out.append(dict(P=P, kind=kind, cmp=cmp, hashed=hashed, unordered=u, send_empty=(k + u) % 3 != 0))
    return out


def case_id(c):
    return "P%d-%s-%s-%s-%s" % (c["P"], c["kind"], "hash" if c["hashed"] else "given",
                                "unordered" if c["unordered"] else "ordered", "empty" if c["send_empty"] else "noempty")


def width_case_data(c, n, seed):
    """(records uint8 [n, w] or serialized keys, partitions, given ids or None) of one partition-width case: distinct
    keys (the oracle's order of equal keys is not the stable one) whose sort words collide within a partition"""
    P = c["P"]
    if c["kind"] in ("fixed4", "fixed8"):
        w = 4 if c["kind"] == "fixed4" else 8
        data = fixed_records(distinct_keys(n, w, seed), w, c["cmp"])
        keys = data[:, :w]
    else:
        data = keys = var_keys(words(n, seed), c["cmp"])
    given = None if c["hashed"] else given_partitions(n, P, seed)
    return data, partitions(keys, c["cmp"], P, given), given


# ------------------------------------------------------------------------------------------------ host reference
def partitions(keys, cmp, P, given=None):
    """HashPartitioner's partition of every serialized key (given: the ids themselves)"""
    if given is not None:
        return np.asarray(given, dtype=np.int64)
    return np.array([O.partition_of(cmp, bytes(k), P) for k in keys], dtype=np.int64)


def given_partitions(n, P, seed):
    """partition ids crowding a few partitions (0, 1, P/2, P-1: the top id sets the highest partition bit) and spread
    over the rest"""
    r = _rng(seed, 55, n, P)
    few = np.array([0, 1 % P, P // 2, P - 1], dtype=np.int64)
    return np.where(r.random(n) < 0.5, few[r.integers(0, 4, n)], r.integers(0, P, n)).astype(np.int64)


def stable_order(norm, parts):
    """the sorted permutation: by partition, then normalised key, ties in collection order"""
    return np.lexsort((np.asarray(norm), np.asarray(parts)))


def stable_order_var(contents, parts):
    return np.array(sorted(range(len(contents)), key=lambda i: (int(parts[i]), contents[i])), dtype=np.int64)


def unordered_order(parts):
    """UnorderedPartitionedKVWriter: by partition, newest record first"""
    n = len(parts)
    return np.lexsort((np.arange(n)[::-1], np.asarray(parts)))


def spill_file(framed, rec_off, order, parts, P, send_empty=True, unordered=False):
    """(file.out as uint8, index int64 [P, 3]) of records written in `order`: one IFile segment per partition ("TIF\\0",
    the framed records, the EOF marker 0xFF 0xFF, the CRC-32 of records and marker).  Partitions without records have
    no segment when send_empty (start = the running offset, lengths 0), an empty one when not; the unordered writer
    never writes them and leaves their index entry all zero."""
    order = np.asarray(order, dtype=np.int64)
    parts = np.asarray(parts, dtype=np.int64)
    if P <= 4096:
        return _spill_file_loop(framed, rec_off, order, parts, P, send_empty, unordered)
    lens = np.diff(rec_off)[order]
    ps = parts[order]
    cnt = np.bincount(ps, minlength=P)
    body = np.bincount(ps, weights=lens, minlength=P).astype(np.int64)
    present = (cnt > 0) if (send_empty or unordered) else np.ones(P, dtype=bool)
    seg = np.where(present, body + 10, 0)
    start = np.cumsum(seg) - seg
    index = np.zeros((P, 3), dtype=np.int64)
    index[:, 0] = np.where(present, start, 0) if unordered else start
    index[:, 1] = np.where(present, seg - 4, 0)
    index[:, 2] = seg
    out = np.empty(int(seg.sum()), dtype=np.uint8)
    B = int(lens.sum())
    if B:
        sorted_off = np.cumsum(lens) - lens
        src = np.repeat(rec_off[:-1][order] - sorted_off, lens) + np.arange(B)
        before = np.cumsum(present) - present      # segments in front of each partition's
        out[np.arange(B) + np.repeat(10 * before[ps] + 4, lens)] = framed[src]
    s = start[present]
    e = s + seg[present]
    for j, b in enumerate(b"TIF\x00"):
        out[s + j] = b
    out[e - 6] = 0xFF
    out[e - 5] = 0xFF
    crc = np.full(P, EOF_CRC, dtype=np.int64)
    for p in np.nonzero(cnt)[0]:
        crc[p] = zlib.crc32(out[start[p] + 4:start[p] + seg[p] - 4])
    cp = crc[present]
    for j in range(4):
        out[e - 4 + j] = (cp >> (24 - 8 * j)) & 0xFF
    return out, index


def _spill_file_loop(framed, rec_off, order, parts, P, send_empty, unordered):
    """spill_file segment by segment (few partitions, many records)"""
    lens = np.diff(rec_off)
    ps = parts[order]
    bounds = np.searchsorted(ps, np.arange(P + 1))
    rows = framed.reshape(-1, int(lens[0]))[order] if lens.size and bool((lens == lens[0]).all()) else None
    pieces, index, off = [], np.zeros((P, 3), dtype=np.int64), 0
    for p in range(P):
        a, b = bounds[p], bounds[p + 1]
        if a == b and (send_empty or unordered):
            index[p, 0] = 0 if unordered else off
            continue
        if rows is not None:
            body = rows[a:b].tobytes()
        else:
            body = b"".join(framed[rec_off[i]:rec_off[i + 1]].tobytes() for i in order[a:b])
        body += b"\xff\xff"
        pieces.append(b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big"))
        index[p] = (off, len(body) + 4, len(body) + 8)
        off += len(body) + 8
    return np.frombuffer(b"".join(pieces), dtype=np.uint8), index


def reference_fixed(rec, cmp, P, parts, send_empty=True, unordered=False):
    """file.out and index of fixed-width records (fixed_records) sorted by the map side"""
    width = rec.shape[1] - 4
    norm = normalised(rec[:, :width], cmp)
    order = unordered_order(parts) if unordered else stable_order(norm, parts)
    framed, off = framed_fixed(rec)
    return spill_file(framed, off, order, parts, P, send_empty, unordered)


def reference_var(keys, cmp, P, parts, values=None, send_empty=True, unordered=False):
    contents = [_content(cmp, k) for k in keys]
    order = unordered_order(parts) if unordered else stable_order_var(contents, parts)
    framed, off = framed_var(keys, values)
    return spill_file(framed, off, order, parts, P, send_empty, unordered)


def _content(cmp, k):
    if cmp == O.CMP_TEXT:
        _, used = O.read_vint(k)
        return k[used:]
    if cmp == O.CMP_BYTESWRITABLE:
        return k[4:]
    raise ValueError(cmp)


def normalised(keys, cmp):
    """normalised values (uint64) of serialized fixed keys uint8 [n, 4 or 8]"""
    w = keys.shape[1]
    v = np.zeros(keys.shape[0], dtype=np.uint64)
    for j in range(w):
        v = (v << np.uint64(8)) | keys[:, j].astype(np.uint64)
    if cmp in (O.CMP_INT, O.CMP_LONG):
        v ^= np.uint64(1 << (8 * w - 1))
    return v


def oracle_run(rec_or_keys, cmp, P, parts=None, send_empty=True, unordered=False, values=None):
    """the oracle's file.out and index for fixed records (uint8 [n, w]) or variable keys (list of bytes) with RLE off;
    parts None = HashPartitioner"""
    if isinstance(rec_or_keys, np.ndarray):
        n, w = rec_or_keys.shape
        kv = rec_or_keys.reshape(-1)
        ko = np.arange(n, dtype=np.uint64) * w
        kl = np.full(n, w - 4, dtype=np.uint32)
    else:
        keys = rec_or_keys
        n = len(keys)
        kvb, koff, voff, _ = var_batch(keys, values)
        kv = np.frombuffer(kvb + b"\0", dtype=np.uint8)
        ko, kl = koff.astype(np.uint64), (voff - koff).astype(np.uint32)
    vl = np.full(n, 4, dtype=np.uint32)
    conf = O.sorter_conf(P, cmp_kind=cmp, partitioner=O.PART_HASH if parts is None else O.PART_GIVEN,
                         send_empty=send_empty, rle_policy=0)
    pa = None if parts is None else np.asarray(parts, dtype=np.int32)
    r = (O.unordered_write if unordered else O.pipelined_sort)(conf, kv, ko, kl, vl, pa)
    return r["file_out"], r["index"]


# ------------------------------------------------------------------------------------------------ device checker
def _ord_key(k, width, cmp):
    """int64 tensor whose signed order is the comparator order of the big-endian keys k (uint8 [m, width])"""
    import torch
    k = k.to(torch.int64)
    v = torch.zeros(k.shape[0], dtype=torch.int64, device=k.device)
    for j in range(width):
        v = (v << 8) | k[:, j]
    if width == 4:
        return v ^ (1 << 31) if cmp == O.CMP_INT else v
    return v if cmp == O.CMP_LONG else v ^ (-1 << 63)


def _host_crc(d, a, b, pinned):
    crc = 0
    step = pinned.numel()
    for x in range(a, b, step):
        m = min(step, b - x)
        pinned[:m].copy_(d[x:x + m])
        crc = zlib.crc32(pinned[:m].numpy(), crc)
    return crc


def check_device(d_out, out_len, index, n, width, cmp, part_of=None, chunk=1 << 25):
    """Checks a sort of n fixed-width records (fixed_records: width-byte key, 4-byte index value, RLE off) from its output
    on the device, chunk by chunk, carrying state across chunk and segment edges: every segment's header, EOF marker
    and CRC-32; every record's framing and partition (part_of: serialized keys uint8 [m, width] -> partition ids; None
    = one partition); keys non-decreasing in comparator order inside a partition; the values a permutation of 0..n-1
    (a byte map on the device); indices ascending inside every run of equal keys.  Together these say the output is
    the stable sort, without a reference order.  Returns the number of records seen."""
    import torch
    dev = d_out.device
    P = index.shape[0]
    rec = width + 6
    seen = torch.zeros(n, dtype=torch.bool, device=dev)
    pinned = torch.empty(1 << 26, dtype=torch.uint8).pin_memory()
    total, off = 0, 0
    for p in range(P):
        start, raw, part = (int(x) for x in index[p])
        assert start == off, "partition %d starts at %d, expected %d" % (p, start, off)
        if part == 0:
            assert raw == 0
            continue
        assert part == raw + 4
        off += part
        head = d_out[start:start + 4].cpu().numpy().tobytes()
        tail = d_out[start + part - 6:start + part].cpu().numpy().tobytes()
        assert head == b"TIF\x00" and tail[:2] == b"\xff\xff", "partition %d: header or EOF marker" % p
        assert (raw - 6) % rec == 0, "partition %d: %d body bytes" % (p, raw - 6)
        assert int.from_bytes(tail[2:], "big") == _host_crc(d_out, start + 4, start + part - 4, pinned), \
            "partition %d: CRC-32" % p
        cnt = (raw - 6) // rec
        prev_k = prev_i = None
        for a in range(0, cnt, chunk):
            m = min(chunk, cnt - a)
            r = d_out[start + 4 + a * rec:start + 4 + (a + m) * rec].view(m, rec)
            assert bool((r[:, 0] == width).all()) and bool((r[:, 1] == 4).all()), "partition %d: framing" % p
            keys = r[:, 2:2 + width]
            if part_of is None:
                assert P == 1
            else:
                assert bool((part_of(keys) == p).all()), "partition %d: a record of another partition" % p
            k = _ord_key(keys, width, cmp)
            v = r[:, 2 + width:].to(torch.int64)
            idx = (v[:, 0] << 24) | (v[:, 1] << 16) | (v[:, 2] << 8) | v[:, 3]
            del r, keys, v
            assert bool((idx < n).all()), "partition %d: value out of range" % p
            seen[idx] = True
            if prev_k is not None:
                k = torch.cat([prev_k, k])
                idx = torch.cat([prev_i, idx])
            lo, hi = k[:-1], k[1:]
            assert bool((lo <= hi).all()), "partition %d: keys out of order near record %d" % (p, a)
            tie = lo == hi
            assert bool((idx[:-1][tie] < idx[1:][tie]).all()), "partition %d: ties out of collection order near record %d" % (p, a)
            prev_k, prev_i = k[-1:].clone(), idx[-1:].clone()
            del k, idx, lo, hi, tie
        total += cnt
    assert off == out_len, "segments cover %d of %d bytes" % (off, out_len)
    assert total == n, "%d records written, %d sorted" % (total, n)
    assert bool(seen.all()), "some record index is missing (and another one repeated)"
    del seen
    return total

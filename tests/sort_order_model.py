"""Shared helpers of the sort-order tests: the normalised key content of every comparator (the bytes whose unsigned
lexicographic order is the RawComparator's order), the host run of the map side's sort word build
(tezgpu_debug_sort_words_emulate) and key sets aimed at the branches of the alphabet table (SymTable)."""
import ctypes as C

import numpy as np

from oracle import tez_oracle as O
from tez_b200 import _lib

CMPS = [O.CMP_BYTES, O.CMP_TEXT, O.CMP_BYTESWRITABLE, O.CMP_INT, O.CMP_LONG]
FIXED_LEN = {O.CMP_INT: 4, O.CMP_LONG: 8}     # IntWritable / LongWritable keys have one length
SYM_MAX_POS = 16


def pbits_of(P):
    return (P - 1).bit_length()


def _vint_decode_size(b0):
    v = b0 - 256 if b0 >= 128 else b0
    return 1 if v >= -112 else (-119 - v if v < -120 else -111 - v)


def content(cmp, key):
    """Normalised content bytes of a serialized key: comparator order == bytes order (shorter prefix first)."""
    if cmp == O.CMP_TEXT:
        return key[min(_vint_decode_size(key[0]), len(key)):] if key else b""
    if cmp == O.CMP_BYTESWRITABLE:
        return key[min(4, len(key)):]
    if cmp in (O.CMP_INT, O.CMP_LONG) and key:
        return bytes([key[0] ^ 0x80]) + key[1:]
    return key


def make_key(cmp, c):
    """Serialized key whose normalised content is c (inverse of content())."""
    if cmp == O.CMP_TEXT:
        return O.text(c)
    if cmp == O.CMP_BYTESWRITABLE:
        return len(c).to_bytes(4, "big") + c
    if cmp in (O.CMP_INT, O.CMP_LONG):
        assert len(c) == FIXED_LEN[cmp]
        return bytes([c[0] ^ 0x80]) + c[1:]
    return c


def sort_words(keys, cmp, P, partition=None, use_sym=True):
    """(words uint32[n], npos, table used) the variable-width map side gives these keys."""
    L = _lib.load()
    n = len(keys)
    kv = np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8).copy()
    kl = np.array([len(k) for k in keys], dtype=np.uint32)
    ko = np.zeros(n, dtype=np.uint64)
    if n:
        ko[1:] = np.cumsum(kl[:-1], dtype=np.uint64)
    part = None if partition is None else np.ascontiguousarray(partition, dtype=np.int32)
    words = np.zeros(max(n, 1), dtype=np.uint32)
    npos, used = C.c_uint32(), C.c_int32()
    _lib.check(L.tezgpu_debug_sort_words_emulate(kv.ctypes.data, ko.ctypes.data, kl.ctypes.data, n, cmp, P,
                                                 None if part is None else part.ctypes.data, 1 if use_sym else 0,
                                                 words.ctypes.data, C.byref(npos), C.byref(used)))
    return words[:n], npos.value, bool(used.value)


def table_layout(contents, P):
    """Plain restatement of the table's size rule: position q needs ceil(log2(#values at q + 1)) bits (rank 0 = the key
    ended), positions are packed while they fit the (32 - pbits)-bit field, and the table is used when it packs more
    positions than the raw prefix's (32 - pbits) // 8 bytes.  Returns (npos, used, depth0)."""
    avail = 32 - pbits_of(P)
    used_bits, npos = 0, 0
    while npos < SYM_MAX_POS:
        vals = {c[npos] for c in contents if len(c) > npos}
        if not vals:
            break
        bits = len(vals).bit_length()       # smallest b with 2^b >= count + 1
        if used_bits + bits > avail:
            break
        used_bits += bits
        npos += 1
    used = npos > avail // 8
    return npos, used, (npos if used else avail // 8)


def sample_values(rng, c):
    """c distinct byte values; the extremes 0x00 and 0xFF are always among them when c >= 2."""
    if c >= 256:
        return list(range(256))
    vals = {0, 255} if c >= 2 else {rng.randrange(256)}
    while len(vals) < c:
        vals.add(rng.randrange(256))
    return sorted(vals)


def alphabet_contents(rng, cmp, c, q, other="small", n=None):
    """Normalised key contents with exactly c byte values at content position q, every one of them occurring.
    other="small": the other positions use {a, b} below position 4 and {a} beyond, so the table packs many positions;
    other="wide": the other positions take any byte, so the table packs no more than the raw prefix.
    Lengths: longer than SYM_MAX_POS, exactly SYM_MAX_POS, ending before q, empty, and (Text) 128+ bytes, whose vint
    header is two bytes."""
    fixed = FIXED_LEN.get(cmp)
    vals = sample_values(rng, c)
    n = n or (1024 if other == "wide" else max(3 * c, 240))

    def other_byte(p):
        if other == "wide":
            return rng.randrange(256)
        return rng.choice(b"ab") if p < 4 else ord("a")

    out = []
    for i in range(n):
        if fixed:
            ln = fixed
        else:
            r = rng.random()
            ln = (20 if r < 0.35 else SYM_MAX_POS if r < 0.6 else rng.randrange(0, q + 1) if r < 0.75 else
                  0 if r < 0.78 else 130 + rng.randrange(40) if (r < 0.83 and cmp == O.CMP_TEXT) else rng.randrange(q + 1, 24))
            if i < len(vals):
                ln = max(ln, q + 1)            # every value occurs at q
        b = bytearray(other_byte(p) for p in range(ln))
        if ln > q:
            b[q] = vals[i] if i < len(vals) else rng.choice(vals)
        out.append(bytes(b))
    return out


def check_words(keys, cmp, P, words, depth0, used, partition=None):
    """The two properties the sort relies on, against the oracle comparator:
    word(a) < word(b)  =>  (partition a, a) < (partition b, b);
    word(a) == word(b) =>  same partition and equal normalised content on the first depth0 bytes (both ended there
    count as equal; the raw prefix pads an ended key with zero bytes)."""
    n = len(keys)
    parts = (np.asarray(partition, dtype=np.int64) if partition is not None
             else np.array([O.partition_of(cmp, k, P) for k in keys], dtype=np.int64))
    cont = [content(cmp, k) for k in keys]

    def head(c):
        h = c[:depth0]
        return h if used else h.ljust(depth0, b"\0")

    order = sorted(range(n), key=lambda i: (int(words[i]), parts[i], cont[i]))
    # inside every word group: one partition and one head; between groups: the last key of a group is below the first
    # of the next (Python order, confirmed by the oracle comparator), which by transitivity covers every pair
    prev_last = None
    g0 = 0
    while g0 < n:
        g1 = g0
        w = words[order[g0]]
        while g1 < n and words[order[g1]] == w:
            g1 += 1
        first, last = order[g0], order[g1 - 1]
        hd = head(cont[first])
        for i in order[g0:g1]:
            assert parts[i] == parts[first], "equal sort words 0x%08x, partitions %d and %d" % (w, parts[first], parts[i])
            assert head(cont[i]) == hd, "equal sort words 0x%08x for keys %s and %s (depth %d)" % (
                w, keys[first].hex(), keys[i].hex(), depth0)
        if prev_last is not None:
            a, b = prev_last, first
            assert (parts[a], cont[a]) < (parts[b], cont[b]), (
                "sort word 0x%08x of key %s (partition %d) is below 0x%08x of key %s (partition %d)" % (
                    words[a], keys[a].hex(), parts[a], words[b], keys[b].hex(), parts[b]))
            if parts[a] == parts[b]:
                assert O.compare(cmp, keys[a], keys[b]) < 0, (keys[a].hex(), keys[b].hex())
        prev_last = last
        g0 = g1

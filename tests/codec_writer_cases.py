"""Crafted partition bodies for the device codec writers: lengths at the edges of every codec's lane, slice and chunk
schedule, and contents that drive each writer down a chosen path (stored / raw output, longest matches, matches one
slice back, literal runs across lanes, Huffman against raw literals, degenerate and length-limited Huffman codes).

Each case is one partition holding one record, so its body vint(kl) vint(vl) key payload FF FF has an exact length and
chosen content: the key (0-2 bytes) absorbs the steps of the vint widths.  A body of 2 bytes is an empty partition,
written when send_empty_partition_details is off.  The cases need no device."""
import functools
import random

from oracle import tez_oracle as O
import tez_b200 as T

EOF_MARKER = b"\xff\xff"


class Geometry:
    """a codec's chunk writer: threads (lanes) per chunk, bytes each lane parses (slice), body bytes per chunk"""

    def __init__(self, name, codec, lanes, chunk):
        self.name, self.codec, self.lanes, self.chunk = name, codec, lanes, chunk
        self.slice = chunk // lanes
        assert self.slice * lanes == chunk


GEOMETRY = {
    "default": Geometry("default", T.CODEC_DEFAULT, 16, 32768),
    "lz4": Geometry("lz4", T.CODEC_LZ4, 32, T.LZ4_BLOCK_BYTES),
    "snappy": Geometry("snappy", T.CODEC_SNAPPY, 32, T.SNAPPY_BLOCK_BYTES),
    "zstd": Geometry("zstd", T.CODEC_ZSTD, 32, T.ZSTD_BLOCK_BYTES),
}
assert GEOMETRY["lz4"].slice == GEOMETRY["snappy"].slice == GEOMETRY["zstd"].slice == 2032
assert GEOMETRY["default"].slice == 2048


def lengths(g):
    """body lengths at the edges of g's schedule (and of the LZ4, Snappy and zstd format rules)"""
    s, c, n = g.slice, g.chunk, g.lanes
    out = {2}                                   # an empty partition
    out.update(range(4, 18))                    # LZ4's 5 last literals and 12-byte match limit; fewer bytes than lanes
    out.update((n - 1, n, n + 1))               # one byte per lane
    out.update((60, 61, 62, 63))                # Snappy: literals of 60 bytes and less take one tag byte, of 61 two
    out.update((4095, 4096, 4097))              # zstd: 2- and 3-byte literals section headers
    out.update((s - 1, s, s + 1, (n - 1) * s - 1, (n - 1) * s + 1, c - 1, c, c + 1, 2 * c, 3 * c + 7))
    return sorted(out)


# ------------------------------------------------------------------------------------------------ contents
def _random(rng, n, g):
    return bytes(rng.getrandbits(8) for _ in range(n))


def _one_value(rng, n, g):
    return b"\x61" * n


def _slice_periodic(rng, n, g):
    """one random slice repeated: a lane's first match in a chunk reaches exactly one slice back, into the bytes its
    hash table is seeded with"""
    s = _random(rng, g.slice, g)
    return (s * (n // g.slice + 1))[:n]


def _one_lane_matches(rng, n, g):
    """random bytes except the slice of one lane, which repeats an 8-byte word: the literal runs before and after it
    cross many lanes"""
    b = bytearray(_random(rng, n, g))
    lane = min(g.lanes // 2, max(0, n // g.slice - 1))
    a = lane * g.slice
    e = min(n, a + g.slice)
    w = _random(rng, 8, g)
    b[a:e] = (w * (g.slice // 8 + 1))[:e - a]
    return bytes(b)


GAPS = (15, 60, 61, 270, 525)   # LZ4 literal lengths 15, 270, 525 (a length byte each); Snappy's 60 / 61 literal tags


def _literal_gaps(rng, n, g):
    """a run of one byte value with random gaps (no byte of that value) of GAPS bytes, each straddling a lane
    boundary: each gap is one literal run of exactly its length, split between two lanes"""
    b = bytearray(b"\x61" * n)
    for i, gap in enumerate(GAPS):
        edge = (2 * i + 2) * g.slice
        a = edge - (gap // 2 + i)
        if edge >= g.chunk or a + gap + 32 > n:
            break
        b[a:a + gap] = bytes(rng.choice(range(0x62, 0x100)) for _ in range(gap))
    return bytes(b)


def _below_128(rng, n, g):
    """words over bytes 0-127 with repeats: matches, and literals that zstd codes with Huffman"""
    words = [bytes(rng.randrange(128) for _ in range(rng.randint(3, 9))) for _ in range(400)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) if rng.random() < 0.5 else bytes([rng.randrange(128)])
    return bytes(out[:n])


def _below_128_one_128(rng, n, g):
    """_below_128 with one byte of 128 in its middle: zstd's literals of every frame that holds it stay raw"""
    b = bytearray(_below_128(rng, n, g))
    if n:
        b[n // 2] = 128
    return bytes(b)


def _two_symbols(rng, n, g):
    """random over two byte values: two literal symbols beside the matches"""
    return bytes(rng.choice(b"\x41\x42") for _ in range(n))


def _fibonacci(rng, n, g):
    """per chunk: 16 byte values with counts 1, 1, 2, 3, 5, ..., 987 and 4 more of count 1 among random bytes of 64
    other values, shuffled: an unlimited Huffman code of the literals would be deeper than 15 bits"""
    fib = [1, 1]
    while len(fib) < 16:
        fib.append(fib[-1] + fib[-2])
    sym = [i for i in range(16) for _ in range(fib[i])] + [16, 17, 18, 19]
    out = bytearray()
    while len(out) < n:
        c = sym + [rng.randrange(192, 256) for _ in range(g.chunk - len(sym))]
        rng.shuffle(c)
        out += bytes(c)
    return bytes(out[:n])


def _records_text(rng, n, g):
    """real record bytes: a word-count body (Text keys, IntWritable values) as the payload"""
    words = [b"w%x%s" % (i, b"abcdefgh"[:i % 7]) for i in range(3000)]
    out = bytearray()
    while len(out) < n:
        w = rng.choice(words)
        out += O.vint(len(w) + 1) + b"\x04" + bytes([len(w)]) + w + b"\x00\x00\x00\x01"
    return bytes(out[:n])


CONTENTS = {
    "random": _random,
    "one_value": _one_value,
    "slice_periodic": _slice_periodic,
    "one_lane_matches": _one_lane_matches,
    "literal_gaps": _literal_gaps,
    "below_128": _below_128,
    "below_128_one_128": _below_128_one_128,
    "two_symbols": _two_symbols,
    "fibonacci": _fibonacci,
    "records_text": _records_text,
}
LARGE = ("random", "one_value", "slice_periodic", "literal_gaps", "below_128", "below_128_one_128", "fibonacci", "records_text")   # also at a chunk and more


# ------------------------------------------------------------------------------------------------ bodies
def record_for(content, length):
    """(key, value) of the one record whose body vint(kl) vint(vl) key value FF FF is `length` bytes and equals
    content outside its vints; None for length 2 (no record)"""
    if length == 2:
        return None
    n = length - 2
    for kl in range(3):
        for w in range(1, 6):
            vl = n - 1 - kl - w
            if vl >= 0 and len(O.vint(vl)) == w:
                h = 1 + w
                return content[h:h + kl], content[h + kl:n]
    raise AssertionError("no record of %d bytes" % length)


def body_of_record(rec):
    if rec is None:
        return EOF_MARKER
    k, v = rec
    return O.vint(len(k)) + O.vint(len(v)) + k + v + EOF_MARKER


class Case:
    def __init__(self, name, content, length, rec, body):
        self.name, self.content, self.length, self.rec, self.body = name, content, length, rec, body

    def __repr__(self):
        return "Case(%s)" % self.name


def make_case(g, content, length, seed=0):
    rng = random.Random("%s/%s/%d/%d" % (g.name, content, length, seed))
    raw = CONTENTS[content](rng, max(0, length - 2), g)
    rec = record_for(raw, length)
    body = body_of_record(rec)
    assert len(body) == length and body.endswith(EOF_MARKER)
    if rec is not None:
        h = len(body) - 2 - len(rec[0]) - len(rec[1])
        assert h in (2, 3, 4, 5, 6) and len(rec[0]) <= 2
        assert body[h:-2] == raw[h:], "the body is the content outside its vints"
        seg = O.write_ifile([rec], rle=False)[0]
        assert seg[4:-4] == body, "the oracle's IFile writer frames the record the same way"
    return Case("%s/%s/%d" % (g.name, content, length), content, length, rec, body)


@functools.lru_cache(maxsize=None)
def cases(g):
    """every content class at every length of g (the large lengths for LARGE only), the empty partition once"""
    res = [make_case(g, "random", 2)]
    big = g.chunk - 1
    for content in CONTENTS:
        for n in lengths(g):
            if n == 2 or (n >= big and content not in LARGE):
                continue
            res.append(make_case(g, content, n))
    return tuple(res)


def sorted_records(g, n=3000, seed=1):
    """ordinary sorted multi-record partitions: a word count's records (Text keys, IntWritable values)"""
    rng = random.Random(seed)
    words = [O.text("w%d%s" % (i, "xyz"[: i % 4])) for i in range(n // 3)]
    return sorted((rng.choice(words), rng.getrandbits(32).to_bytes(4, "big")) for _ in range(n))

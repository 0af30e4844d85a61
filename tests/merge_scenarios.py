"""Seeded merge problems for the route tests (tests/test_merge_routes_gpu.py, tests/test_merge_scenarios_cpu.py).

scenario(seed) returns one merge: a comparator, P partitions and the IFile segments (written by the oracle writer,
run-length encoded or plain, with or without the TIF header) of each, listed with their partitions interleaved;
fixed or variable framing; checkForSameKeys, the writer's RLE, a sum combiner or none; and whether the merge is
"large", i.e. more records than the 16 MiB floor budget of the bounded merge holds in one step.  shape(seed) is the
part that needs no data (the pytest ids).

Every value is its record's global index (big-endian, padded to one length per scenario; a few records of some
scenarios are longer than the 32 KiB parse window), or with a combiner a 4- or 8-byte signed summand.  Duplicates keep
the oracle's isSameKey flags pinned (DESIGN.md section 6): a key shared by several segments of a partition occurs at
most once in each of them, and a key repeated inside a segment is private to it.  Keys come from a palette per
comparator where raw byte order and comparator order disagree (PALETTES), mixed with random keys."""
import functools
import random

from oracle import tez_oracle as O
import sort_order_model as SOM

CMP_NAMES = {O.CMP_BYTES: "tezbytes", O.CMP_TEXT: "text", O.CMP_BYTESWRITABLE: "byteswritable", O.CMP_INT: "int",
             O.CMP_LONG: "long"}
PS = (1, 2, 7, 64)
SEEDS = tuple(range(100))
FIXED_KLEN = {O.CMP_INT: 4, O.CMP_LONG: 8, O.CMP_BYTES: 16}   # the comparators with a fixed-framing scenario
SUM_INT, SUM_LONG = 1, 2                                      # COMBINE_SUM_INT / COMBINE_SUM_LONG
COMBINER_WIDTH = {SUM_INT: 4, SUM_LONG: 8}
LARGE_RECORDS = 60000   # 320 B of workspace per record (DESIGN.md section 3): far more than one 16 MiB step holds
WINDOW = 32768          # the window parser's window (parse_windows.cuh)
SOLO_LEN = 1024         # keys at least this long occur once per scenario (Text contents around 65,536 bytes)


# ------------------------------------------------------------------------------------------------ palettes
def _ints():
    vals = [-2 ** 31, -2 ** 31 + 1, -256, -1, 0, 1, 255, 256, 2 ** 31 - 1]
    for x in (5, 0x7F, 0x80, 0x12345678, 0x7FFFFE01):
        vals += [x, x ^ 0x80000000]
    return [O.int_writable(v) for v in vals]


def _longs():
    vals = [-2 ** 63, -2 ** 63 + 1, -1, 0, 1, 2 ** 63 - 1, -2 ** 32, 2 ** 32 - 1, 2 ** 32]
    for x in (0x7F, 0x0123456789ABCDEF, 2 ** 40 + 3):
        vals += [x, x ^ 2 ** 63]
    for high in (0, 1, -5, 0x7FFFFFFF, -2 ** 31):   # equal high 32 bits: the 4-byte sort word ties, the tail decides
        vals += [(high << 32) | low for low in (0, 1, 0x7F000000, 0x80000000, 0xFFFFFFFF)]
    return list(dict.fromkeys(O.long_writable(v) for v in vals))


HEAD = bytes(range(0x30, 0x44))   # 20 shared bytes: more than the 16 positions the alphabet sort word covers


def _tezbytes():
    return ([b"", b"\x00", b"\x00\x00", b"\x00" * 7, b"\x00\x01", b"\x01", b"\x7f", b"\x80", b"\xff", b"\xff\xff",
             b"\xff" * 9, b"\xff\x00", b"\x00\xff", b"a", b"ab", b"abc", b"abcd", b"abcd\x00", b"abcd\xff", b"abcde"]
            + [HEAD + t for t in (b"", b"\x00", b"\x01", b"\x7f", b"\x80", b"\xff", b"\xff\xff", b"zz")])


def _tezbytes16():
    return ([b"\x00" * 16, b"\xff" * 16, b"\x00" * 15 + b"\x01", b"\xff" * 15 + b"\xfe", b"\x80" + b"\x00" * 15,
             b"\x7f" + b"\xff" * 15, b"abcd" + b"\x00" * 12, b"abcd" + b"\xff" * 12, b"abcdefgh" + b"\x00" * 8,
             b"abcdefgh" + b"\x80" * 8]
            + [HEAD[:12] + t for t in (b"\x00" * 4, b"\x00\x00\x00\x01", b"\x7f\xff\xff\xff", b"\x80\x00\x00\x00",
                                       b"\xff" * 4)])


def _text():
    contents = [b"", b"b", b"\x00", b"\xff", b"\x00\x00", b"\xff\xff", b"a\x00", b"a\xff", b"ab", b"abc"]
    for n in (1, 127, 128, 255, 256, 65535, 65536, 65537):   # vint prefixes of 1 to 4 bytes
        contents += [b"a" * n, b"a" * (n - 1) + b"b"]
    return [O.text(c) for c in dict.fromkeys(contents)]


def _byteswritable():
    contents = [b"", b"a", b"b", b"aa", b"ab", b"ba", b"\x00", b"\xff", b"\x00\x00", b"\xff" * 40, b"a" * 40,
                b"abcde" * 8, b"zz", b"z" + b"\x00" * 30]
    contents += [b"abcdefgh" + t for t in (b"", b"\x00", b"\xff", b"i", b"ij")]
    contents += [b"m" * n for n in range(0, 41, 5)]
    return [len(c).to_bytes(4, "big") + c for c in dict.fromkeys(contents)]


PALETTES = {O.CMP_BYTES: _tezbytes(), O.CMP_TEXT: _text(), O.CMP_BYTESWRITABLE: _byteswritable(), O.CMP_INT: _ints(),
            O.CMP_LONG: _longs()}
FIXED_PALETTES = {O.CMP_BYTES: _tezbytes16(), O.CMP_INT: PALETTES[O.CMP_INT], O.CMP_LONG: PALETTES[O.CMP_LONG]}


def _random_key(rng, cmp, fixed):
    """one random serialized key of the comparator (fixed: of the fixed key length)"""
    if cmp == O.CMP_INT:
        return rng.randbytes(4)
    if cmp == O.CMP_LONG:
        if rng.random() < 0.3:      # a high half shared with palette keys: the tie path of fixed framing
            return rng.choice((b"\x00" * 4, b"\x00\x00\x00\x01", b"\xff\xff\xff\xfb")) + rng.randbytes(4)
        return rng.randbytes(8)
    small = b"\x00\x01ab\x7f\x80\xfe\xff"   # a small alphabet: prefixes of each other and common heads

    def content(n):
        return bytes(rng.choice(small) for _ in range(n)) if rng.random() < 0.5 else rng.randbytes(n)
    if cmp == O.CMP_BYTES:
        if fixed:
            return (rng.choice((b"", HEAD[:8], b"abcd")) + rng.randbytes(16))[:16]
        return rng.choice((b"", b"", HEAD)) + content(rng.randint(0, 12))
    if cmp == O.CMP_TEXT:
        n = rng.randint(120, 300) if rng.random() < 0.05 else rng.randint(0, 20)
        return O.text(content(n))
    c = content(rng.randint(0, 40))
    return len(c).to_bytes(4, "big") + c


class _Keys:
    """distinct keys of one partition: the palette first (shuffled), then random ones"""

    def __init__(self, rng, cmp, fixed):
        self.rng, self.cmp, self.fixed = rng, cmp, fixed
        pal = list(dict.fromkeys((FIXED_PALETTES if fixed else PALETTES)[cmp]))
        rng.shuffle(pal)
        self.palette = [k for k in pal if len(k) < SOLO_LEN]
        self.used = set()

    def take(self, n, palette=True):
        out = []
        if palette:
            while self.palette and len(out) < n:
                k = self.palette.pop()
                self.used.add(k)
                out.append(k)
        while len(out) < n:
            k = _random_key(self.rng, self.cmp, self.fixed)
            if k not in self.used and len(k) < SOLO_LEN:
                self.used.add(k)
                out.append(k)
        return out


# ------------------------------------------------------------------------------------------------ scenarios
def shape(seed):
    """The axes of scenario(seed), derived from the seed alone.  The seeds cycle the comparators; j = seed // 5 runs
    through 20 patterns of the other axes, so every comparator meets every axis value."""
    cmp = SOM.CMPS[seed % 5]
    j = seed // 5
    fixed = cmp in FIXED_KLEN and j % 3 == 0
    combiner = (SUM_INT if j % 2 else SUM_LONG) if j % 7 in (2, 5) else 0
    return dict(seed=seed, cmp=cmp, P=PS[j % 4], check=j // 2 % 2 == 0, writer_rle=(j % 4 + j // 4) % 2 == 1,
                has_header=j % 5 != 3, fixed=fixed, combiner=combiner, large=j in (1, 5, 11, 18),
                encode=(j % 2 == 1) if fixed else j % 4 != 2,
                long_values=not fixed and not combiner and j % 4 == 3)


def scenario_id(seed):
    s = shape(seed)
    return "%03d-%s-P%d-%s-chk%d-wrle%d-%s-%s-%s" % (
        seed, CMP_NAMES[s["cmp"]], s["P"], "fixed" if s["fixed"] else "var", s["check"], s["writer_rle"],
        "hdr" if s["has_header"] else "nohdr", ("sum%d" % (8 * COMBINER_WIDTH[s["combiner"]])) if s["combiner"] else "nocomb",
        "large" if s["large"] else "small")


def _segments_per_partition(rng, P):
    if P == 1:
        return [rng.choice((1, 2, rng.randint(3, 40), 40))]
    if P == 2:
        return [rng.randint(1, 24), rng.randint(0, 24)]
    if P == 7:
        return [rng.choice((0, 1, rng.randint(2, 8))) for _ in range(P)]
    return [rng.choice((0, 0, 1, 2, 3)) for _ in range(P)]


@functools.lru_cache(maxsize=8)
def scenario(seed):
    """dict: shape(seed) + segs (bytes, header stripped when not has_header), parts, fixed as (klen, vlen) or None,
    vlen, encoded (some input holds a REPEAT_KEY record), nrec"""
    s = shape(seed)
    rng = random.Random(seed * 7919 + 1)
    cmp, P = s["cmp"], s["P"]
    counts = _segments_per_partition(rng, P)
    if not any(counts):
        counts[rng.randrange(P)] = 1
    total = (LARGE_RECORDS + rng.randint(0, 4000)) if s["large"] else rng.randint(300, 5000)
    nseg_all = sum(counts)
    # records per segment: random weights, some segments hold only the EOF marker
    weights = [0.0 if rng.random() < 0.1 else rng.random() + 0.05 for _ in range(nseg_all)]
    if not any(weights):
        weights[0] = 1.0
    wsum = sum(weights)
    sizes = [int(total * w / wsum) for w in weights]

    width = COMBINER_WIDTH.get(s["combiner"])
    if s["fixed"]:
        vlen = width or rng.choice((4, 8, 12, 64))
    else:
        vlen = width or rng.choice((4, 5, 9, 16, 30))
    solo = [key for key in PALETTES[cmp] if len(key) >= SOLO_LEN and not s["fixed"]]
    segs_recs = []   # [(partition, [keys sorted], rle)]
    k = 0
    for p in range(P):
        keys = _Keys(rng, cmp, s["fixed"])
        mine = sizes[k:k + counts[p]]
        k += counts[p]
        if not mine:
            continue
        frac = [rng.uniform(0.3, 0.8) if len(mine) > 1 else 0.0 for _ in mine]
        pool = keys.take(max(1, int(max(n * f for n, f in zip(mine, frac)) * 1.4)))
        for n, f in zip(mine, frac):
            shared = rng.sample(pool, min(len(pool), int(n * f)))
            rest = n - len(shared)
            distinct = keys.take(max(0, rest - rest // 4), palette=len(mine) == 1)
            seg_keys = shared + distinct
            if distinct:                          # repeats of private keys only
                seg_keys += [rng.choice(distinct) for _ in range(rest - len(distinct))]
            if solo and n and rng.random() < 0.5:
                seg_keys.append(solo.pop())
            seg_keys.sort(key=lambda key: SOM.content(cmp, key))
            rle = s["encode"] and rng.random() < 0.6
            segs_recs.append((p, seg_keys, rle))
    rng.shuffle(segs_recs)                        # partitions interleave in the caller's list
    if s["encode"]:                               # at least one input holds an encoded repeat when any can
        reps = [i for i, (_, ks, _) in enumerate(segs_recs) if any(a == b and a for a, b in zip(ks, ks[1:]))]
        if reps:
            i = max(reps, key=lambda i: len(segs_recs[i][1]))
            segs_recs[i] = segs_recs[i][:2] + (True,)

    nrec = sum(len(ks) for _, ks, _ in segs_recs)
    longs = set(rng.sample(range(nrec), min(3, nrec))) if s["long_values"] else set()
    segs, parts, gidx = [], [], 0
    for p, ks, rle in segs_recs:
        recs = []
        for key in ks:
            if width:
                v = rng.randint(-2 ** (8 * width - 1), 2 ** (8 * width - 1) - 1).to_bytes(width, "big", signed=True)
            else:
                v = gidx.to_bytes(vlen + (WINDOW + 1000 * (gidx % 7) if gidx in longs else 0), "big")
            recs.append((key, v))
            gidx += 1
        seg = O.write_ifile(recs, rle=rle)[0]
        segs.append(seg if s["has_header"] else seg[4:])
        parts.append(p)
    encoded = any(ks == O.SAME_KEY for seg in segs for ks, _, _ in O.read_ifile(seg, has_header=s["has_header"]))
    out = dict(s, segs=segs, parts=parts, vlen=vlen, encoded=encoded, nrec=nrec,
               fixed=(FIXED_KLEN[cmp], vlen) if s["fixed"] else None)
    return out


def merge_kwargs(sc):
    """GpuMerger keyword arguments of a scenario (without a combiner)"""
    return dict(comparator=sc["cmp"], has_header=sc["has_header"], partitions=sc["parts"], num_partitions=sc["P"])

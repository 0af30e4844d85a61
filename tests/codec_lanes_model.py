"""Stream builders and references of the codec lane tests (test_codec_lanes_cpu.py / test_codec_lanes_gpu.py).

The device decodes a compressed segment with one warp whose 32 lanes share match copies, stored blocks, literal runs and
the Adler-32; the host emulation runs the same code with one lane.  The builders here place exactly the structures where
the two differ: DEFLATE (length, distance) pairs, stored-block lengths and code lengths; LZ4 (literal run, match length,
offset) sequences in Java block framing; Zstandard raw / RLE blocks, hand-made sequence blocks and libzstd frames.  Each
case carries its intended body; the references are the libraries (zlib, liblz4, libzstd) and the one-lane emulation.
Parsers read the structure back from every stream, so a case is checked to be what its name says."""
import ctypes as C
import random
import zlib

import numpy as np

from tez_b200._lib import TezGpuError
from tez_b200.constants import CODEC_DEFAULT, CODEC_LZ4, CODEC_ZSTD, E_FORMAT
import codec_model as CM
import lz4_model as L4
import zstd_model as ZS


class Case:
    """One well-formed stream: `stream` decodes to `body`; `path` is the device pass that takes it ("unit": every LZ4
    block one chunk / every zstd frame with Frame_Content_Size; "serial": the one-warp-per-segment decoder)."""

    def __init__(self, name, stream, body, path="serial"):
        self.name, self.stream, self.body, self.path = name, bytes(stream), bytes(body), path

    def __repr__(self):
        return "Case(%s, %d -> %d bytes, %s)" % (self.name, len(self.stream), len(self.body), self.path)


def segment(stream):
    """TIF\\x01 + stream + CRC-32 of the stream (IFile.Writer's compressed segment)"""
    return b"TIF\x01" + bytes(stream) + zlib.crc32(bytes(stream)).to_bytes(4, "big")


def image(body):
    """the uncompressed IFile segment decode_segments returns for a body: TIF\\x00 + body + CRC-32 of the body"""
    return b"TIF\x00" + bytes(body) + zlib.crc32(bytes(body)).to_bytes(4, "big")


def _rand(rng, n, alphabet=None):
    if alphabet is None:
        return bytes(rng.getrandbits(8) for _ in range(n))
    return bytes(rng.choice(alphabet) for _ in range(n))


# ================================================================================================ DEFLATE
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30
# a complete code-length code over all 19 symbols (13 of 4 bits, 6 of 5 bits): any length list can be sent with it
CL_LENS = [4] * 13 + [5] * 6


def len_sym(n):
    assert 3 <= n <= 258
    if n == 258:
        return 285, 0, 0
    i = max(k for k in range(28) if LBASE[k] <= n)
    return 257 + i, n - LBASE[i], LEXT[i]


def dist_sym(d):
    assert 1 <= d <= 32768
    i = max(k for k in range(30) if DBASE[k] <= d)
    return i, d - DBASE[i], DEXT[i]


def canonical(lengths):
    """RFC 1951 3.2.2: the code of every symbol with a nonzero length"""
    mx = max(lengths) if lengths else 0
    count = [0] * (mx + 2)
    for n in lengths:
        if n:
            count[n] += 1
    code, nxt = 0, [0] * (mx + 2)
    for b in range(1, mx + 1):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    codes = {}
    for s, n in enumerate(lengths):
        if n:
            codes[s] = (nxt[n], n)
            nxt[n] += 1
    return codes


def flat_lengths(symbols, total):
    """a complete prefix code over `symbols` (two or more) with lengths b - 1 and b, in a list of `total` lengths"""
    k = len(symbols)
    b = max(1, (k - 1).bit_length())
    out = [0] * total
    for i, s in enumerate(sorted(symbols)):
        out[s] = b - 1 if i < (1 << b) - k else b
    return out


class BitW:
    """LSB-first bit writer (Huffman codes are given MSB first, as RFC 1951 writes them)"""

    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def huff(self, code, n):
        self.put(int(format(code, "0%db" % n)[::-1], 2), n)

    def align(self):
        if self.n:
            self.out.append(self.acc & 255)
            self.acc, self.n = 0, 0


def M(length, dist):
    """a match token"""
    return ("m", length, dist)


def _expand(out, tokens):
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
            continue
        _, n, d = t
        assert 1 <= d <= len(out), (d, len(out))
        while n:
            k = min(n, d)
            out += out[len(out) - d:len(out) - d + k]
            n -= k


def rle_lengths(lens):
    """code-length tokens (symbol, extra bits value) for a combined length list: 17 / 18 for zero runs, 16 for repeats
    of the previous length"""
    toks, i = [], 0
    while i < len(lens):
        v, j = lens[i], i
        while j < len(lens) and lens[j] == v:
            j += 1
        run = j - i
        if v == 0 and run >= 3:
            while run >= 11:
                r = min(run, 138)
                toks.append((18, r - 11))
                run -= r
            if run >= 3:
                toks.append((17, run - 3))
                run = 0
            toks += [(0, None)] * run
        else:
            toks.append((v, None))
            run -= 1
            while run >= 3:
                r = min(run, 6)
                toks.append((16, r - 3))
                run -= r
            toks += [(v, None)] * run
        i = j
    return toks


def deflate_member(blocks, cinfo=7):
    """One zlib member of the given blocks and its body.  A block is ("stored", data), ("fixed", tokens) or
    ("dynamic", tokens, lit_lengths, dist_lengths); tokens are literal byte values and M(length, distance)."""
    w = BitW()
    w.out += CM.zhdr(cinfo)
    body = bytearray()
    for bi, blk in enumerate(blocks):
        w.put(int(bi + 1 == len(blocks)), 1)
        if blk[0] == "stored":
            data = bytes(blk[1])
            w.put(0, 2)
            w.align()
            w.put(len(data), 16)
            w.put(len(data) ^ 0xFFFF, 16)
            w.out += data
            body += data
            continue
        if blk[0] == "fixed":
            w.put(1, 2)
            lit, dist = FIXED_LIT, FIXED_DIST
        else:
            lit, dist = blk[2], blk[3]
            w.put(2, 2)
            w.put(len(lit) - 257, 5)
            w.put(len(dist) - 1, 5)
            w.put(15, 4)
            for s in CL_ORDER:
                w.put(CL_LENS[s], 3)
            cl = canonical(CL_LENS)
            for s, e in rle_lengths(list(lit) + list(dist)):
                w.huff(*cl[s])
                if s >= 16:
                    w.put(e, {16: 2, 17: 3, 18: 7}[s])
        lc, dc = canonical(lit), canonical(dist)
        for t in blk[1]:
            if isinstance(t, int):
                w.huff(*lc[t])
            else:
                s, e, eb = len_sym(t[1])
                w.huff(*lc[s])
                w.put(e, eb)
                s, e, eb = dist_sym(t[2])
                w.huff(*dc[s])
                w.put(e, eb)
        w.huff(*lc[256])
        _expand(body, blk[1])
    w.align()
    w.out += zlib.adler32(bytes(body)).to_bytes(4, "big")
    return bytes(w.out), bytes(body)


class _BitR:
    def __init__(self, b, pos=0):
        self.b, self.pos = b, pos       # pos in bits

    def get(self, n):
        v = 0
        for i in range(n):
            v |= ((self.b[self.pos >> 3] >> (self.pos & 7)) & 1) << i
            self.pos += 1
        return v

    def sym(self, codes):
        code, n = 0, 0
        while True:
            code = (code << 1) | self.get(1)
            n += 1
            if (code, n) in codes:
                return codes[(code, n)]
            assert n < 16, "no such code"


def inflate_walk(z):
    """The structure of a well-formed zlib stream (one or more members): per member its CINFO and its blocks, each a
    dict with "type" and, for stored blocks, "len"; for Huffman blocks "matches" [(length, distance)] (and "literals",
    the literal count), "end_bit" (the bit offset in its byte where the block ends) and, for dynamic blocks, "max_len"
    (longest literal/length code), "hlit", "ndist_codes" (distance codes with a length) and "cl" (the code-length
    symbols in order, with the list index each starts at)."""
    z, pos, members = bytes(z), 0, []
    while pos < len(z):
        cinfo = z[pos] >> 4
        r = _BitR(z, 8 * (pos + 2))
        blocks = []
        while True:
            final, typ = r.get(1), r.get(2)
            if typ == 0:
                r.pos = (r.pos + 7) & ~7
                n = r.get(16)
                r.get(16)
                blocks.append({"type": "stored", "len": n})
                r.pos += 8 * n
            else:
                b = {"type": "fixed" if typ == 1 else "dynamic", "matches": [], "literals": 0}
                if typ == 1:
                    lit, dist = FIXED_LIT, FIXED_DIST
                else:
                    hlit, hdist, hclen = r.get(5) + 257, r.get(5) + 1, r.get(4) + 4
                    cll = [0] * 19
                    for i in range(hclen):
                        cll[CL_ORDER[i]] = r.get(3)
                    clc = {v: s for s, v in canonical(cll).items()}
                    lens, cl = [], []
                    while len(lens) < hlit + hdist:
                        s = r.sym(clc)
                        cl.append((s, len(lens)))
                        if s < 16:
                            lens.append(s)
                        elif s == 16:
                            lens += [lens[-1]] * (3 + r.get(2))
                        elif s == 17:
                            lens += [0] * (3 + r.get(3))
                        else:
                            lens += [0] * (11 + r.get(7))
                    lit, dist = lens[:hlit], lens[hlit:]
                    b.update(max_len=max(lit), hlit=hlit, ndist_codes=sum(1 for x in dist if x), cl=cl)
                lc = {v: s for s, v in canonical(lit).items()}
                dc = {v: s for s, v in canonical(dist).items()}
                while True:
                    s = r.sym(lc)
                    if s < 256:
                        b["literals"] += 1
                        continue
                    if s == 256:
                        break
                    n = LBASE[s - 257] + r.get(LEXT[s - 257])
                    d = r.sym(dc)
                    b["matches"].append((n, DBASE[d] + r.get(DEXT[d])))
                b["end_bit"] = r.pos & 7
                blocks.append(b)
            if final:
                break
        pos = ((r.pos + 7) >> 3) + 4
        members.append({"cinfo": cinfo, "blocks": blocks})
    return members


def _fixed_case(name, tokens, prefix=b"", cinfo=7):
    z, body = deflate_member([("fixed", list(prefix) + list(tokens))], cinfo)
    return Case(name, z, body)


DIST_SET = list(range(1, 41)) + [63, 64, 65, 32767, 32768]
LEN_SET = [3, 31, 32, 33, 63, 64, 65, 257, 258]


def deflate_cases(seed=1):
    rng = random.Random(seed)
    cases = []
    # every distance, each with every length in one fixed block (a literal between the matches)
    for d in DIST_SET:
        toks = list(_rand(rng, d))
        for n in LEN_SET:
            toks += [M(n, d), rng.getrandbits(8)]
        cases.append(_fixed_case("dist_%d" % d, toks))
    # back-to-back long matches, no literal between them
    toks = list(_rand(rng, 50)) + [M(258, 1), M(64, 3), M(100, 17), M(33, 31), M(40, 50), M(258, 32), M(31, 2), M(32, 9),
                                   M(257, 5), M(65, 29)]
    cases.append(_fixed_case("back_to_back_long", toks))
    # a long match that reads lane 0's literals, a short one (lane 0) that reads bytes the lanes have just written
    toks = list(b"abcdefg") + [M(64, 7), M(5, 3), M(31, 13), M(40, 2), M(3, 1), ord("z"), M(33, 30), M(31, 33)]
    cases.append(_fixed_case("short_reads_long", toks))
    # stored blocks of every edge length between Huffman blocks; the match after each reads back into it
    for n in (0, 1, 31, 32, 33, 65535):
        data = _rand(rng, n)
        back = [M(min(n, 258), min(n, 32768))] if n >= 3 else [M(3, n + 4)]
        z, body = deflate_member([("fixed", list(b"head")), ("stored", data), ("fixed", back + list(b"tail"))])
        cases.append(Case("stored_%d" % n, z, body))
    # a stored block after a fixed block that ends at bit offset 0..7 (so 0..6 whole bytes are still buffered)
    for b in range(8):
        nine = (b - 2) % 8                  # 3 + 8a + 9c + 7 bits from bit 16: ends at (2 + c) mod 8
        toks = list(b"ab") + [200 + k for k in range(nine)]
        data = _rand(rng, 40)
        z, body = deflate_member([("fixed", toks), ("stored", data), ("fixed", [M(40, 40), M(33, 7)])])
        cases.append(Case("stored_after_bit_%d" % b, z, body))
    # dynamic: codes of 1..15 bits (the walk past the first-level table), literals with the longest codes
    lits = list(b"abcdefghijklmn")
    lit = [0] * 258
    for i, s in enumerate(lits):
        lit[s] = i + 1
    lit[256], lit[257] = 15, 15
    dist = [0] * 5
    dist[0], dist[4] = 1, 1
    toks = lits + lits[::-1] + [M(3, 1), ord("n"), ord("m"), M(3, 5), ord("n")] * 3
    z, body = deflate_member([("dynamic", toks, lit, dist)])
    cases.append(Case("dynamic_15_bit_codes", z, body))
    # dynamic: exactly one distance code (25..32, incomplete), long matches at distances below 32
    toks = list(_rand(rng, 40)) + [M(40, 25), M(258, 31), M(32, 28), ord("q"), M(100, 32)]
    used = sorted({t for t in toks if isinstance(t, int)} | {256} | {len_sym(t[1])[0] for t in toks if not isinstance(t, int)})
    dist = [0] * 10
    dist[9] = 1
    z, body = deflate_member([("dynamic", toks, flat_lengths(used, 286), dist)])
    cases.append(Case("dynamic_one_distance_code", z, body))
    # dynamic: no distance codes at all (a literal-only block)
    toks = list(_rand(rng, 300, b"etaoin shrdlu"))
    used = sorted(set(toks) | {256})
    z, body = deflate_member([("dynamic", toks, flat_lengths(used, 257), [0])])
    cases.append(Case("dynamic_no_distance_codes", z, body))
    # dynamic: repeat codes at the list edges: 18 first, a 16 run across the literal/distance boundary, 17 or 16 last
    for tail in (4, 0):
        lit = [0] * 264
        for s in list(range(97, 105)) + list(range(256, 264)):
            lit[s] = 4
        dist = [4] * 16 + [0] * tail
        toks = list(b"abcdefgh") + [M(3, 1), M(9, 8), ord("a"), M(5, 3), M(4, 9)]
        z, body = deflate_member([("dynamic", toks, lit, dist)])
        cases.append(Case("dynamic_repeat_edges_%s" % ("17" if tail else "16"), z, body))
    # dynamic: HLIT = 286 (every length symbol) and HDIST = 30
    toks = list(_rand(rng, 64))
    for n in (3, 10, 11, 18, 19, 34, 35, 66, 67, 130, 131, 226, 227, 257, 258):
        toks += [M(n, rng.randrange(1, 60)), rng.getrandbits(8)]
    prefix = list(_rand(rng, 25000))
    toks = prefix + toks + [M(40, d) for d in (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025,
                                                1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577)]
    z, body = deflate_member([("dynamic", toks, flat_lengths(range(286), 286), flat_lengths(range(30), 30))])
    cases.append(Case("dynamic_hlit_286", z, body))
    # window bits 8..15 in the header (CINFO 0..7), distances within the window
    for cinfo in range(8):
        toks = list(_rand(rng, 100)) + [M(64, 100), M(200, 33), ord("w"), M(31, 129)]
        cases.append(_fixed_case("window_bits_%d" % (cinfo + 8), toks, cinfo=cinfo))
    # bodies that set the Adler-32 lane split: empty lanes below 32 bytes, 5552 / 5553 around zlib's NMAX
    for n in (2, 3, 31, 32, 33, 5552, 5553, 65537):
        body = _rand(rng, n, b"abcd\x00\xff")
        cases.append(Case("adler_body_%d" % n, zlib.compress(body, 6), body))
        z, b2 = deflate_member([("stored", body[:65535]), ("stored", body[65535:])] if n > 65535 else [("stored", body)])
        cases.append(Case("adler_stored_%d" % n, z, b2))
    # 1..7 members, empty members among them, and a 2-byte last member
    for m in range(1, 8):
        parts = [_rand(rng, rng.choice([0, 1, 40, 500, 3000]), b"xyz\x01") for _ in range(m - 1)] + [b"\xff\xff"]
        if m >= 3:
            parts[1] = b""
        cases.append(Case("members_%d" % m, b"".join(zlib.compress(p, 6) for p in parts), b"".join(parts)))
    return cases


def deflate_large(block, total):
    """One zlib member of `total` bytes: `block` (len 4096) as literals, then matches at distance 4096 (258 bytes each)
    and a final shorter one.  Built by repeating the 23-byte pattern of eight 23-bit matches.  Returns the stream and the
    body's Adler-32 (computed by repetition)."""
    d = len(block)
    assert d == 4096 and total > d + 258 * 64
    w = BitW()
    w.out += CM.zhdr(7)
    w.put(1, 1)
    w.put(1, 2)
    lc, dc = canonical(FIXED_LIT), canonical(FIXED_DIST)

    def match(n):
        s, e, eb = len_sym(n)
        w.huff(*lc[s])
        w.put(e, eb)
        s, e, eb = dist_sym(d)
        w.huff(*dc[s])
        w.put(e, eb)

    for c in block:
        w.huff(*lc[c])
    rest = total - d
    full, last = divmod(rest, 258)
    if last and last < 3:
        full, last = full - 1, last + 258      # 259 / 260: two matches
    groups, tail = divmod(full, 8)
    for _ in range(8):
        match(258)
    a = len(w.out)
    for _ in range(8):
        match(258)
    pattern = bytes(w.out[a:])
    assert len(pattern) == 23
    w.out += pattern * (groups - 2)
    for _ in range(tail):
        match(258)
    while last:
        n = last if last <= 258 else last - 3
        match(n)
        last -= n
    w.huff(*lc[256])
    w.align()
    tile = np.frombuffer(block, dtype=np.uint8)
    big = np.tile(tile, 16384).tobytes()       # 64 MiB
    adler, left = 1, total
    while left:
        k = min(left, len(big))
        adler = zlib.adler32(big[:k], adler)
        left -= k
    w.out += adler.to_bytes(4, "big")
    return bytes(w.out)


# ================================================================================================ LZ4
def _ext(n):
    r, out = n - 15, b""
    while r >= 255:
        out += b"\xff"
        r -= 255
    return out + bytes([r])


def l4_chunk(seqs, last):
    """One raw LZ4 block: sequences (literals, offset, match length) then the last literals.  Returns the chunk and the
    bytes it decodes to."""
    out, body = bytearray(), bytearray()
    for lit, off, ml in seqs:
        L, m = len(lit), ml - 4
        assert ml >= 4 and 0 < off < 65536
        out.append(min(L, 15) << 4 | min(m, 15))
        if L >= 15:
            out += _ext(L)
        out += lit
        out += off.to_bytes(2, "little")
        if m >= 15:
            out += _ext(m)
        body += lit
        _expand(body, [M(ml, off)])
    L = len(last)
    out.append(min(L, 15) << 4)
    if L >= 15:
        out += _ext(L)
    out += last
    body += last
    return bytes(out), bytes(body)


def l4_block(raw, *chunks):
    return raw.to_bytes(4, "big") + b"".join(len(c).to_bytes(4, "big") + c for c in chunks)


def l4_pair(name, chunk, body):
    """the chunk as one block of one chunk (unit pass) and twice in one block (serial pass)"""
    return [Case(name, l4_block(len(body), chunk), body, "unit"),
            Case(name + "_twice", l4_block(2 * len(body), chunk, chunk), body * 2, "serial")]


def l4_sequences(chunk):
    """(literal length, offset, match length) of every sequence of a chunk; the last has offset None"""
    ip, seqs = 0, []
    while True:
        tok = chunk[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                s = chunk[ip]
                ip += 1
                lit += s
                if s != 255:
                    break
        ip += lit
        if ip == len(chunk):
            seqs.append((lit, None, None))
            return seqs
        off = chunk[ip] | chunk[ip + 1] << 8
        ip += 2
        m = tok & 15
        if m == 15:
            while True:
                s = chunk[ip]
                ip += 1
                m += s
                if s != 255:
                    break
        seqs.append((lit, off, m + 4))


L4_OFFSETS = list(range(1, 41)) + [64, 65535]
L4_CAP = L4.CHUNK_CAP


def lz4_cases(seed=2):
    rng = random.Random(seed)
    cases = []

    def add(name, seqs, last):
        cases.extend(l4_pair(name, *l4_chunk(seqs, last)))

    for L in (14, 15, 15 + 255, 15 + 2 * 255):
        add("literal_run_%d" % L, [(_rand(rng, L), 3, 20), (_rand(rng, L), L + 1, 5)], _rand(rng, 5))
    add("match_lengths_4_to_19", [(_rand(rng, 3), 3, m) for m in range(4, 20)], _rand(rng, 6))
    add("match_lengths_19_plus_255k", [(_rand(rng, 3), 3, 19 + 255 * k) for k in (1, 2, 3)], _rand(rng, 5))
    for off in L4_OFFSETS:
        seqs = [(_rand(rng, off), off, 4)] + [(_rand(rng, 1), off, m) for m in (31, 32, 33, 64, 100, 4, 270)]
        add("offset_%d" % off, seqs, _rand(rng, 5))
    # a match that ends exactly 5 bytes before the 262,144-byte cap, then exactly 5 last literals: a chunk of the cap
    add("chunk_of_cap_lastliterals", [(b"ab", 2, L4_CAP - 2 - 5)], _rand(rng, 5))
    # a literal run that ends exactly 12 bytes before the cap (MFLIMIT), then a 7-byte match and 5 last literals
    add("literal_run_at_mflimit", [(b"x", 1, L4_CAP - 113), (_rand(rng, 100), 9, 7)], _rand(rng, 5))
    # liblz4's own chunks: fast (accelerations 1, 8, 65537) and HC, over record-shaped and repetitive bodies
    if L4.liblz4() is not None:
        bodies = [CM.wordcount_body(n=15000, seed=7), CM.int_long_body(n=8000, seed=8), b"xy" * 40000 + _rand(rng, 3000),
                  bytes(range(7)) * 9000]
        for mode, accel in (("fast", 1), ("fast", 8), ("fast", 65537), ("hc", 0)):
            for i, body in enumerate(bodies):
                body = body[:L4.MAX_INPUT]
                name = "liblz4_%s%d_body%d" % (mode, accel, i)
                cases.append(Case(name, l4_block(len(body), L4.lz4_compress(body, mode, accel)), body, "unit"))
                step = 20000 + 997 * i
                chunks = [L4.lz4_compress(body[a:a + step], mode, accel) for a in range(0, len(body), step)]
                cases.append(Case(name + "_chunks", l4_block(len(body), *chunks), body, "serial"))
    # the device writer's own blocks (one chunk each)
    for i, body in enumerate([CM.wordcount_body(n=12000, seed=9), _rand(rng, 70000, b"ab\x00")]):
        cases.append(Case("device_writer_%d" % i, L4.compress_emulate(body), body, "unit"))
    return cases


def lz4_short_block(seed=3):
    """A block whose one chunk decodes validly to one byte fewer than the block's raw length (and the raw length the
    segment declares): the unit pass must hand it to the serial pass, which refuses it."""
    rng = random.Random(seed)
    chunk, body = l4_chunk([(_rand(rng, 9), 4, 40)], _rand(rng, 6))
    return l4_block(len(body) + 1, chunk), len(body) + 1


def lz4_library_stream(z, expect):
    """BlockDecompressorStream over liblz4: each block's chunks decoded by LZ4_decompress_safe until its raw length; the
    bytes, or None where liblz4 fails, a block over-decodes or the stream is not exactly `expect` bytes"""
    z, ip, out = bytes(z), 0, bytearray()
    while ip < len(z):
        if ip + 4 > len(z):
            return None
        raw = int.from_bytes(z[ip:ip + 4], "big")
        ip += 4
        if raw == 0:
            return None
        got = 0
        while got < raw:
            if ip + 4 > len(z):
                return None
            c = int.from_bytes(z[ip:ip + 4], "big")
            ip += 4
            if c > len(z) - ip or c > L4_CAP:
                return None
            d = L4.lz4_decompress_safe(z[ip:ip + c])
            if d is None or got + len(d) > raw:
                return None
            out += d
            got += len(d)
            ip += c
    return bytes(out) if len(out) == expect else None


# ================================================================================================ Zstandard
_P1, _P2, _P3, _P4, _P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261
_M64 = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M64


def _xround(acc, v):
    return (_rotl((acc + v * _P2) & _M64, 31) * _P1) & _M64


def xxh64(data, seed=0):
    """XXH64 (the Content_Checksum hash of RFC 8878 takes its low 32 bits)"""
    data, n, p = bytes(data), len(data), 0
    le = lambda a, k: int.from_bytes(data[a:a + k], "little")
    if n >= 32:
        v = [(seed + _P1 + _P2) & _M64, (seed + _P2) & _M64, seed, (seed - _P1) & _M64]
        while p + 32 <= n:
            v = [_xround(v[i], le(p + 8 * i, 8)) for i in range(4)]
            p += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M64
        for x in v:
            h = ((h ^ _xround(0, x)) * _P1 + _P4) & _M64
    else:
        h = (seed + _P5) & _M64
    h = (h + n) & _M64
    while p + 8 <= n:
        h = (_rotl(h ^ _xround(0, le(p, 8)), 27) * _P1 + _P4) & _M64
        p += 8
    if p + 4 <= n:
        h = (_rotl(h ^ ((le(p, 4) * _P1) & _M64), 23) * _P2 + _P3) & _M64
        p += 4
    while p < n:
        h = (_rotl(h ^ ((data[p] * _P5) & _M64), 11) * _P1) & _M64
        p += 1
    h ^= h >> 33
    h = (h * _P2) & _M64
    h ^= h >> 29
    h = (h * _P3) & _M64
    return h ^ (h >> 32)


def zs_bh(last, bt, size):
    return (int(last) | bt << 1 | size << 3).to_bytes(3, "little")


def zs_window_byte(need):
    """the smallest Window_Descriptor whose window holds `need` bytes"""
    for wd in range(256):
        base = 1 << (10 + (wd >> 3))
        if base + (base >> 3) * (wd & 7) >= need:
            return wd
    raise ValueError(need)


def zs_frame(blocks, content, fcs=True, checksum=False, window=None):
    """A Zstandard frame of the given block bytes whose content is `content`: with Frame_Content_Size in a
    Single_Segment frame (fcs=True), else with a Window_Descriptor (`window` bytes, default the content's size)."""
    n = len(content)
    fhd = 4 if checksum else 0
    if fcs and window is None:
        fhd |= 0x20
        if n < 256:
            h = bytes([n])
        elif n < 65536 + 256:
            fhd |= 1 << 6
            h = (n - 256).to_bytes(2, "little")
        else:
            fhd |= 2 << 6
            h = n.to_bytes(4, "little")
    else:
        h = bytes([zs_window_byte(max(window or n, 1))])
        if fcs:
            fhd |= 2 << 6
            h += n.to_bytes(4, "little")
    ck = (xxh64(content) & 0xFFFFFFFF).to_bytes(4, "little") if checksum else b""
    return ZS.MAGIC + bytes([fhd]) + h + b"".join(blocks) + ck


def zs_raw(data, last=False):
    return zs_bh(last, 0, len(data)) + bytes(data)


def zs_rle(byte, n, last=False):
    return zs_bh(last, 1, n) + bytes([byte])


def _lit_header(lt, size):
    if size < 32:
        return bytes([size << 3 | lt])
    if size < 4096:
        return bytes([(size & 15) << 4 | 1 << 2 | lt, size >> 4])
    return bytes([(size & 15) << 4 | 3 << 2 | lt, (size >> 4) & 255, size >> 12])


LL_BASE = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024,
           2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771,
                                65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]


def _code(base, bits, v):
    i = max(k for k in range(len(base)) if base[k] <= v)
    assert v - base[i] < (1 << bits[i])
    return i, v - base[i], bits[i]


def zs_seq_block(literals, seqs, rle_literal=None, last=False):
    """A compressed block whose sequences all share one literal-length, offset and match-length code (RLE mode for all
    three tables): `seqs` [(literal length, offset, match length)], offsets new (no repeat codes).  Literals raw from
    `literals`, or rle_literal * len(literals) (RLE literals, staged by the decoder at the end of the block's room)."""
    n = len(literals)
    if rle_literal is None:
        lit = _lit_header(0, n) + bytes(literals)
    else:
        lit = _lit_header(1, n) + bytes([rle_literal])
    codes, fields = set(), []
    for ll, off, ml in seqs:
        lc, le, lb = _code(LL_BASE, LL_BITS, ll)
        mc, me, mb = _code(ML_BASE, ML_BITS, ml)
        ov = off + 3
        oc = ov.bit_length() - 1
        codes.add((lc, oc, mc))
        fields.append(((ov - (1 << oc), oc), (me, mb), (le, lb)))   # read order: offset, match length, literal length
    assert len(codes) == 1, codes
    lc, oc, mc = codes.pop()
    acc, nb = 0, 0
    for f in reversed(fields):
        for v, b in reversed(f):
            acc |= v << nb
            nb += b
    acc |= 1 << nb
    bits = acc.to_bytes(nb // 8 + 1, "little")
    ns = len(seqs)
    hdr = bytes([ns]) if ns < 128 else bytes([(ns >> 8) + 0x80, ns & 255])
    content = lit + hdr + bytes([0x54, lc, oc, mc]) + bits
    return zs_bh(last, 2, len(content)) + content


def zs_decode_seqs(lit_bytes, seqs, prefix=b""):
    """the output of sequences over literals after `prefix` (earlier output of the frame): the block's bytes"""
    out, lp = bytearray(prefix), 0
    for ll, off, ml in seqs:
        out += lit_bytes[lp:lp + ll]
        lp += ll
        _expand(out, [M(ml, off)])
    out += lit_bytes[lp:]
    return bytes(out[len(prefix):])


def zstd_walk(z):
    """Every frame of a stream: ("skippable", length) or a dict with fcs (None when absent), checksum, window and
    blocks [(type, size, literals kind or None, (LL, OF, ML) modes or None)].  Literals kinds: "raw", "rle", "huf1",
    "huf4", "treeless1", "treeless4"; modes 0 predefined, 1 RLE, 2 FSE, 3 repeat."""
    z, ip, res = bytes(z), 0, []
    while ip < len(z):
        magic = int.from_bytes(z[ip:ip + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            n = int.from_bytes(z[ip + 4:ip + 8], "little")
            res.append(("skippable", n))
            ip += 8 + n
            continue
        assert z[ip:ip + 4] == ZS.MAGIC
        fhd = z[ip + 4]
        single, fcs_flag, did = (fhd >> 5) & 1, fhd >> 6, fhd & 3
        q = ip + 5
        window = None
        if not single:
            wd = z[q]
            base = 1 << (10 + (wd >> 3))
            window = base + (base >> 3) * (wd & 7)
            q += 1
        q += [0, 1, 2, 4][did]
        fsz = [single, 2, 4, 8][fcs_flag]
        fcs = int.from_bytes(z[q:q + fsz], "little") + (256 if fsz == 2 else 0) if fsz else None
        q += fsz
        blocks = []
        while True:
            bh = int.from_bytes(z[q:q + 3], "little")
            bt, bs = (bh >> 1) & 3, bh >> 3
            lk = modes = None
            if bt == 2:
                b = z[q + 3:q + 3 + bs]
                lt, sf = b[0] & 3, (b[0] >> 2) & 3
                if lt < 2:
                    hs = {0: 1, 1: 2, 2: 1, 3: 3}[sf]
                    size = int.from_bytes(b[:hs], "little") >> (3 if hs == 1 else 4)
                    end = hs + (size if lt == 0 else 1)
                    lk = "raw" if lt == 0 else "rle"
                else:
                    hs, nbits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
                    end = hs + (int.from_bytes(b[:hs], "little") >> (4 + nbits) & ((1 << nbits) - 1))
                    lk = ("huf" if lt == 2 else "treeless") + ("1" if sf == 0 else "4")
                nb = b[end]
                e = end + (1 if nb < 128 else 3 if nb == 255 else 2)
                if nb:
                    modes = (b[e] >> 6, (b[e] >> 4) & 3, (b[e] >> 2) & 3)
            blocks.append((bt, bs, lk, modes))
            q += 3 + (1 if bt == 1 else bs)
            if bh & 1:
                break
        q += 4 if fhd & 4 else 0
        res.append({"fcs": fcs, "checksum": bool(fhd & 4), "window": window, "single": bool(single), "blocks": blocks})
        ip = q
    return res


def zstd_lib_frame(body, level=3, checksum=False, window_log=0, ldm=False, content_size=True, buf=None):
    """libzstd's frame of body through ZSTD_compressStream2 with the given parameters; with content_size the whole body
    goes in one ZSTD_e_end call, so the frame carries Frame_Content_Size, else it is flushed every `buf` bytes"""
    if not content_size:
        return ZS.hadoop_stream(body, level=level, checksum=checksum, window_log=window_log, ldm=ldm, buf=buf or ZS.IN_SIZE)
    L = ZS.libzstd()
    body = bytes(body)
    cctx = L.ZSTD_createCCtx()
    try:
        for p, v in ((ZS.C_LEVEL, level), (ZS.C_CHECKSUM, int(checksum)), (ZS.C_WINDOWLOG, window_log), (ZS.C_LDM, int(ldm)),
                     (ZS.C_CONTENTSIZE, 1)):
            assert not L.ZSTD_isError(L.ZSTD_CCtx_setParameter(cctx, p, v))
        src = C.create_string_buffer(body, len(body))
        inb = ZS._In(C.cast(src, C.c_void_p), len(body), 0)
        obuf = C.create_string_buffer(1 << 17)
        res = bytearray()
        while True:
            outb = ZS._Out(C.cast(obuf, C.c_void_p), len(obuf), 0)
            r = L.ZSTD_compressStream2(cctx, C.byref(outb), C.byref(inb), ZS.E_END)
            assert not L.ZSTD_isError(r)
            res += obuf.raw[:outb.pos]
            if r == 0:
                return bytes(res)
    finally:
        L.ZSTD_freeCCtx(cctx)


def zstd_cases(seed=4):
    rng = random.Random(seed)
    cases = []

    def both(name, blocks, content, **kw):
        """the same blocks in a frame with Frame_Content_Size (unit pass) and in one without it (serial pass)"""
        cases.append(Case(name, zs_frame(blocks, content, fcs=True, **kw), content, "unit"))
        cases.append(Case(name + "_nofcs", zs_frame(blocks, content, fcs=False, **kw), content, "serial"))

    # raw and RLE blocks, an empty raw block among them, an RLE block of Block_Maximum_Size
    a, b = _rand(rng, 100), _rand(rng, 50)
    both("raw_blocks", [zs_raw(a), zs_raw(b""), zs_raw(b, True)], a + b)
    c = _rand(rng, 33)
    both("rle_blocks", [zs_rle(0x78, 1000), zs_raw(c), zs_rle(0, 5, True)], b"x" * 1000 + c + b"\0" * 5)
    both("rle_block_maximum", [zs_rle(7, 131072, True)], b"\x07" * 131072, window=131072)
    # hand-made sequence blocks: offsets below 32 with matches of 131..258 bytes after varied raw-block content
    pre = _rand(rng, 64)
    for oc, offs in ((2, [1, 2, 3, 4]), (3, [5, 8, 12, 9]), (4, [13, 20, 28, 17]), (5, [29, 31, 30, 60])):
        seqs = [(8, o, 131 + 37 * i) for i, o in enumerate(offs)]
        lits = _rand(rng, 8 * len(seqs) + 5)
        blk = zs_seq_block(lits, seqs, last=True)
        both("seq_offsets_code_%d" % oc, [zs_raw(pre), blk], pre + zs_decode_seqs(lits, seqs, pre))
        # RLE literals: staged at the end of the block's room; long runs of them with short matches after
        seqs = [(20 + k, o, 3 + 4 * k) for k, o in enumerate(offs)][:1] * 3
        lits = b"q" * (sum(s[0] for s in seqs) + 40)
        blk = zs_seq_block(lits, seqs, rle_literal=ord("q"), last=True)
        both("seq_rle_literals_code_%d" % oc, [zs_raw(pre), blk], pre + zs_decode_seqs(lits, seqs, pre))
    # literals staged at the room's end where the room is the segment's end: a frame without Frame_Content_Size and a
    # small window is the last of its segment in the serial pass; the same block first in a two-frame segment
    seqs = [(12, 9, 40)] * 4
    lits = b"r" * (48 + 7)
    blk = zs_seq_block(lits, seqs, rle_literal=ord("r"), last=True)
    body = pre + zs_decode_seqs(lits, seqs, pre)
    f1 = zs_frame([zs_raw(pre), blk], body, fcs=False, window=1024)
    f2 = zs_frame([zs_raw(b"tail!", True)], b"tail!", fcs=False)
    cases.append(Case("staged_literals_at_segment_end", f1, body, "serial"))
    cases.append(Case("staged_literals_before_next_frame", f1 + f2, body + b"tail!", "serial"))
    # the device writer's frames (one warp per frame) and the same blocks as one frame without Frame_Content_Size
    for i, body in enumerate([CM.wordcount_body(n=9000, seed=11), bytes(rng.getrandbits(7) for _ in range(70000))]):
        z = ZS.compress_emulate(body)
        cases.append(Case("device_writer_%d" % i, z, body, "unit"))
        cases.append(Case("device_writer_%d_one_frame" % i, ZS.one_frame(z), body, "serial"))
    if ZS.libzstd() is None:
        return cases
    # libzstd: every literals type and sequence mode, repeat offsets (levels 3, 9, 19), window logs 10..27, checksums
    wc = CM.wordcount_body(n=20000, vocab=2000, seed=12)
    bodies = {
        "text": wc,
        "short_text": wc[:200],
        "rle_literals": b"".join(b"a" + bytes(rng.getrandbits(8) for _ in range(12)) * 3 for _ in range(400)),
        "random_mix": _rand(rng, 30000) + wc[:30000],
        "periodic": bytes(range(23)) * 5000 + b"." * 3000,
    }
    for name, body in sorted(bodies.items()):
        for level in (3, 9, 19):
            cases.append(Case("lib_%s_l%d" % (name, level), zstd_lib_frame(body, level), body, "unit"))
            cases.append(Case("lib_%s_l%d_stream" % (name, level),
                              zstd_lib_frame(body, level, content_size=False, buf=4096, checksum=True), body, "serial"))
    big = wc * 6
    for wlog in range(10, 28):
        ldm = wlog % 3 == 0
        cases.append(Case("lib_window_log_%d" % wlog, zstd_lib_frame(big, 3, window_log=wlog, ldm=ldm, content_size=False), big,
                          "serial"))
        cases.append(Case("lib_window_log_%d_fcs" % wlog, zstd_lib_frame(big, 3, window_log=wlog, ldm=ldm), big, "unit"))
    # several frames: with Frame_Content_Size (unit) and without (serial), skippable frames between, checksums
    parts = [wc[:5000], wc[5000:5001], wc[5001:30000], b"\xff\xff"]
    fr = [zstd_lib_frame(parts[0], 3, checksum=True), ZS.skippable(b"hello"), zstd_lib_frame(parts[1], 1),
          ZS.skippable(b""), zstd_lib_frame(parts[2], 19), zs_frame([zs_raw(parts[3], True)], parts[3], checksum=True)]
    cases.append(Case("frames_fcs_skippable_checksum", b"".join(fr), b"".join(parts), "unit"))
    fr = [zstd_lib_frame(parts[0], 3, content_size=False), ZS.skippable(b"x" * 40), zstd_lib_frame(parts[1], 1),
          zstd_lib_frame(parts[2], 9, content_size=False, checksum=True), zs_frame([zs_raw(parts[3], True)], parts[3], fcs=False)]
    cases.append(Case("frames_mixed_skippable_checksum", b"".join(fr), b"".join(parts), "serial"))
    return cases


# ================================================================================================ references
CODECS = {"default": CODEC_DEFAULT, "lz4": CODEC_LZ4, "zstd": CODEC_ZSTD}


def cases(codec):
    return {"default": deflate_cases, "lz4": lz4_cases, "zstd": zstd_cases}[codec]()


def library(codec, stream, body_len):
    """the reference library's bytes (DecompressorStream over zlib, BlockDecompressorStream over liblz4,
    ZStandardDecompressor over libzstd) or None where it refuses the stream or the length differs"""
    if codec == "default":
        try:
            out = CM.hadoop_inflate(stream)
        except zlib.error:
            return None
        return out if len(out) == body_len else None
    if codec == "lz4":
        return lz4_library_stream(stream, body_len)
    return zstd_library_stream(stream, body_len)


def zstd_library_stream(z, expect):
    """libzstd's streaming decoder frame after frame: the bytes, or None where it fails, a frame is left unfinished or
    the output is not exactly `expect` bytes.  Unlike zstd_model.hadoop_read it stops once the input is used up and the
    last frame is complete, also when that frame's content ends exactly at the end of an output buffer."""
    L = ZS.libzstd()
    z = bytes(z)
    dctx = L.ZSTD_createDCtx()
    try:
        src = C.create_string_buffer(z, len(z))
        inb = ZS._In(C.cast(src, C.c_void_p), len(z), 0)
        obuf = C.create_string_buffer(L.ZSTD_DStreamOutSize())
        res, r = bytearray(), 0
        while True:
            outb = ZS._Out(C.cast(obuf, C.c_void_p), len(obuf), 0)
            r = L.ZSTD_decompressStream(dctx, C.byref(outb), C.byref(inb))
            if L.ZSTD_isError(r):
                return None
            res += obuf.raw[:outb.pos]
            if len(res) > expect:
                return None
            if inb.pos == inb.size and (r == 0 or outb.pos < outb.size):
                break
        return bytes(res) if r == 0 and len(res) == expect else None
    finally:
        L.ZSTD_freeDCtx(dctx)


_EMULATE = {"default": CM.inflate_emulate, "lz4": L4.decompress_emulate, "zstd": ZS.decompress_emulate}


def emulate(codec, stream, body_len):
    """the one-lane emulation's verdict: (bytes, None), or (None, reason) with the reason string of its TezGpuError"""
    try:
        return _EMULATE[codec](stream, body_len), None
    except TezGpuError as e:
        assert e.code == E_FORMAT, str(e)
        return None, str(e).split(": ")[-1]


def reference(codec, stream, body_len):
    """(library bytes or None, emulation bytes or None, emulation reason or None)"""
    got, reason = emulate(codec, stream, body_len)
    return library(codec, stream, body_len), got, reason


def _sources(codec, rng):
    """small well-formed streams the mutants start from: device-written, library-written and crafted"""
    bodies = [CM.wordcount_body(n=60, vocab=20, seed=s) for s in range(3)] + [bytes(rng.getrandbits(7) for _ in range(300))]
    src = []
    if codec == "default":
        for b in bodies:
            src += [(CM.deflate_emulate(b), b), (zlib.compress(b, 9), b), (zlib.compress(b, 1) + zlib.compress(b[:7], 0), b + b[:7])]
        keep = ("dist_3", "dist_31", "back_to_back_long", "short_reads_long", "stored_33", "stored_after_bit_5",
                "dynamic_one_distance_code", "dynamic_repeat_edges_17", "dynamic_15_bit_codes", "members_4")
    elif codec == "lz4":
        for b in bodies:
            src.append((L4.compress_emulate(b), b))
            if L4.liblz4() is not None:
                src.append((l4_block(len(b), *[L4.lz4_compress(b[a:a + 97]) for a in range(0, len(b), 97)]), b))
        keep = ("literal_run_270", "match_lengths_4_to_19", "offset_7", "offset_7_twice", "offset_31", "offset_33")
    else:
        for b in bodies:
            src.append((ZS.compress_emulate(b), b))
            if ZS.libzstd() is not None:
                src += [(zstd_lib_frame(b, 3, content_size=False, buf=97), b), (zstd_lib_frame(b, 19, checksum=True), b)]
        keep = ("raw_blocks", "rle_blocks_nofcs", "seq_offsets_code_3", "seq_rle_literals_code_4_nofcs",
                "staged_literals_before_next_frame")
    byname = {c.name: c for c in cases(codec)}
    src += [(byname[k].stream, byname[k].body) for k in keep]
    return src


def _repair_adler(zz, blen):
    """a flipped single-member zlib stream whose raw DEFLATE data still decodes, with the Adler-32 and the body length
    of what it decodes to (so the mutant is accepted and its bytes differ from the source's); other streams unchanged"""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(bytes(zz[2:]))
    except zlib.error:
        return zz, blen
    if not d.eof or len(d.unused_data) != 4 or len(out) < 2:
        return zz, blen
    return zz[:-4] + zlib.adler32(out).to_bytes(4, "big"), len(out)


def corrupt(codec, n=1000, seed=99):
    """n seeded mutants [(stream, body_len, emulated bytes or None, emulated reason or None)]: single- and multi-bit
    flips (anywhere, or in the first 24 bytes), truncations and rawLength - 4 off by one, of small device-written,
    library and crafted streams.  Half the flipped zlib streams get the Adler-32 and length of what they now decode to,
    as zlib's checksum would refuse nearly every flip otherwise."""
    rng = random.Random(seed)
    src = _sources(codec, rng)
    res = []
    for i in range(n):
        z, body = src[i % len(src)]
        zz, blen = bytearray(z), len(body)
        kind = i % 5
        if kind <= 1:
            for _ in range(1 if kind == 0 else rng.randrange(2, 5)):
                bit = rng.randrange(len(zz) * 8)
                zz[bit // 8] ^= 1 << (bit % 8)
            if codec == "default" and i % 2 == 0:
                zz, blen = _repair_adler(zz, blen)
        elif kind == 2:
            zz = zz[:rng.randrange(2, len(zz))]
        elif kind == 3:
            bit = rng.randrange(min(len(zz), 24) * 8)      # headers: the first bytes
            zz[bit // 8] ^= 1 << (bit % 8)
        else:
            blen += rng.choice([-1, 1]) if blen > 2 else 1
        got, reason = emulate(codec, bytes(zz), blen)
        res.append((bytes(zz), blen, got, reason))
    return res

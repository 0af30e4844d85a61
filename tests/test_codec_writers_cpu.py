"""The crafted partition bodies of codec_writer_cases without a device: every case is what its name says (length,
record framing, the path it drives the writer down), and the host run of every codec writer on it decodes to the body
through a reader that is not the device's (Python zlib, liblz4 or the LZ4 model, the Snappy model and libsnappy where
it loads, libzstd)."""
import zlib

import pytest

import tez_b200 as T
import codec_model as M
import codec_table as CT
import codec_writer_cases as W
import lz4_model as L4
import snappy_model as SN
import zstd_model as ZS

# ------------------------------------------------------------------------------------------------ stream parsers
def lz4_sequences(chunk):
    """[(literals, offset, match length)] of one raw LZ4 block; the last sequence has offset 0 and no match"""
    ip, res = 0, []
    while True:
        tok = chunk[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                lit += chunk[ip]
                ip += 1
                if chunk[ip - 1] != 255:
                    break
        ip += lit
        if ip == len(chunk):
            res.append((lit, 0, 0))
            return res
        off = chunk[ip] | chunk[ip + 1] << 8
        ip += 2
        m = tok & 15
        if m == 15:
            while True:
                m += chunk[ip]
                ip += 1
                if chunk[ip - 1] != 255:
                    break
        res.append((lit, off, m + 4))


def snappy_elements(chunk):
    """[(literals, offset, copy length)] of one raw Snappy block, one per element"""
    ip = SN.preamble(chunk)[1]
    res = []
    while ip < len(chunk):
        tag = chunk[ip]
        ip += 1
        t = tag & 3
        if t == 0:
            n = tag >> 2
            if n >= 60:
                n, ip = int.from_bytes(chunk[ip:ip + n - 59], "little"), ip + n - 59
            res.append((n + 1, 0, 0))
            ip += n + 1
        elif t == 1:
            res.append((0, ((tag >> 5) << 8) | chunk[ip], ((tag >> 2) & 7) + 4))
            ip += 1
        else:
            eb = 2 if t == 2 else 4
            res.append((0, int.from_bytes(chunk[ip:ip + eb], "little"), (tag >> 2) + 1))
            ip += eb
    return res


def block_chunks(z, codec):
    """the raw chunks of a Lz4Codec / SnappyCodec stream in order (each block holds one)"""
    res = []
    for raw, chunks in (L4 if codec == T.CODEC_LZ4 else SN).blocks(z):
        assert len(chunks) == 1
        res.append(chunks[0])
    return res


class Bits:
    """LSB-first bit reader over a deflate stream"""

    def __init__(self, data, pos):
        self.data, self.bit = data, pos * 8

    def get(self, n):
        v = 0
        for i in range(n):
            v |= ((self.data[self.bit >> 3] >> (self.bit & 7)) & 1) << i
            self.bit += 1
        return v


def _huff_decode_table(lengths):
    """canonical Huffman code lengths -> {(length, code): symbol} (codes MSB-first)"""
    tab, code = {}, 0
    for ln in range(1, 16):
        for s, l in enumerate(lengths):
            if l == ln:
                tab[(ln, code)] = s
                code += 1
        code <<= 1
    return tab


def dynamic_lengths(br):
    """after a dynamic block's 3 header bits: the literal/length and distance code lengths"""
    hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
    order = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
    cl = [0] * 19
    for i in range(hclen):
        cl[order[i]] = br.get(3)
    tab = _huff_decode_table(cl)
    lens = []
    while len(lens) < hlit + hdist:
        code, ln = 0, 0
        while (ln, code) not in tab:
            code = (code << 1) | br.get(1)
            ln += 1
        s = tab[(ln, code)]
        if s < 16:
            lens.append(s)
        elif s == 16:
            lens += [lens[-1]] * (3 + br.get(2))
        elif s == 17:
            lens += [0] * (3 + br.get(3))
        else:
            lens += [0] * (11 + br.get(7))
    return lens[:hlit], lens[hlit:]


def zlib_chunks(z):
    """[(BTYPE, max literal/length code length or None)] of every chunk of a device-written zlib stream (78 01, chunks,
    Adler-32).  A chunk ends with its stored data, at the end of the stream, or with the sync-flush marker behind which
    the stream decodes to the chunk grid."""
    assert z[:2] == b"\x78\x01"
    chunk = W.GEOMETRY["default"].chunk
    res, pos, k = [], 2, 0
    while True:
        h = z[pos]
        final, btype = h & 1, (h >> 1) & 3
        maxlen = None
        if btype == 2:
            br = Bits(z, pos)
            br.get(3)
            maxlen = max(dynamic_lengths(br)[0])
        res.append((btype, maxlen))
        k += 1
        if final:
            return res
        if btype == 0:
            pos += 5 + int.from_bytes(z[pos + 1:pos + 3], "little")
            continue
        q = pos
        while True:
            q = z.index(b"\x00\x00\xff\xff", q + 1)
            d = zlib.decompressobj()
            if len(d.decompress(z[:q + 4])) == k * chunk:
                break
        pos = q + 4


# ------------------------------------------------------------------------------------------------ the cases
@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_lengths_cover_every_schedule_edge(name):
    g = W.GEOMETRY[name]
    ls = W.lengths(g)
    for n in (2, 4, 17, g.lanes - 1, g.slice - 1, g.slice, g.slice + 1, (g.lanes - 1) * g.slice - 1,
              (g.lanes - 1) * g.slice + 1, g.chunk - 1, g.chunk, g.chunk + 1, 2 * g.chunk, 3 * g.chunk + 7, 4095, 4096):
        assert n in ls
    cs = W.cases(g)
    assert len({c.name for c in cs}) == len(cs)
    for content in W.LARGE:
        assert {g.chunk - 1, g.chunk, g.chunk + 1, 2 * g.chunk, 3 * g.chunk + 7} <= {c.length for c in cs if c.content == content}


def test_record_framing_absorbs_every_vint_width():
    """every length from 4 up to past the 3-byte vints is one record of a 0-2 byte key"""
    for n in list(range(4, 300)) + list(range(65530, 65545)):
        rec = W.record_for(bytes(n), n)
        assert len(W.body_of_record(rec)) == n and len(rec[0]) <= 2


@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_host_writer_decodes_to_every_body(name):
    g = W.GEOMETRY[name]
    for c in W.cases(g):
        z = CT.CODECS[name].emulate(c.body)
        assert CT.CODECS[name].independent(z, len(c.body)) == c.body, c


@pytest.mark.parametrize("name", list(W.GEOMETRY))
def test_random_bodies_are_stored_literal_or_raw(name):
    g = W.GEOMETRY[name]
    for n in (g.slice + 1, g.chunk, 3 * g.chunk + 7):
        c = W.make_case(g, "random", n)
        z = CT.CODECS[name].emulate(c.body)
        if g.codec == T.CODEC_DEFAULT:
            # every chunk is stored, except a last chunk of a few bytes, which is smaller as a fixed-Huffman block
            types = [t for t, _ in zlib_chunks(z)]
            sizes = [min(g.chunk, n - k * g.chunk) for k in range(-(-n // g.chunk))]
            assert len(types) == len(sizes), c
            stored = [t for t, sz in zip(types, sizes) if sz >= 64]
            assert stored and stored == [0] * len(stored), c
        elif g.codec == T.CODEC_ZSTD:
            assert [b[0] for f in ZS.frames(z) for b in f[3]] == [0] * -(-n // g.chunk), c
        else:
            chunks = block_chunks(z, g.codec)
            assert len(chunks) == -(-n // g.chunk)
            for ch in chunks:
                parse = lz4_sequences(ch) if g.codec == T.CODEC_LZ4 else snappy_elements(ch)
                assert all(off == 0 for _, off, _ in parse), c


@pytest.mark.parametrize("name", ["lz4", "snappy"])
def test_slice_periodic_matches_reach_one_slice_back(name):
    """in every chunk, every lane after the first finds its first match exactly one slice back"""
    g = W.GEOMETRY[name]
    c = W.make_case(g, "slice_periodic", 2 * g.chunk + 100)
    z = CT.CODECS[name].emulate(c.body)
    for k, ch in enumerate(block_chunks(z, g.codec)):
        parse = lz4_sequences(ch) if g.codec == T.CODEC_LZ4 else snappy_elements(ch)
        pos, first = 0, {}
        for lit, off, m in parse:
            pos += lit
            if off:
                first.setdefault(pos // g.slice, off)
                pos += m
        clen = min(g.chunk, len(c.body) - k * g.chunk)
        lanes = [l for l in range(1, g.lanes) if (l + 1) * g.slice <= clen - 16]
        assert lanes or k == 2
        for l in lanes:
            assert first.get(l) == g.slice, (k, l, first.get(l))


def test_literal_gaps_are_literal_runs_across_lane_edges():
    """LZ4: literal runs of exactly 15, 60, 61, 270 and 525 bytes, each split between two lanes (the parse extends the
    match behind a gap back to its end); Snappy, which does not extend back: runs of at most 8 bytes more, one- and
    two-byte literal tags"""
    for name in ("lz4", "snappy"):
        g = W.GEOMETRY[name]
        c = W.make_case(g, "literal_gaps", g.chunk)
        z = CT.CODECS[name].emulate(c.body)
        ch = block_chunks(z, g.codec)[0]
        if name == "lz4":
            lits = [lit for lit, off, _ in lz4_sequences(ch) if off]
        else:
            lits = [lit for lit, off, _ in snappy_elements(ch) if not off]
        for gap in W.GAPS:
            if name == "lz4":
                assert gap in lits, (name, gap, lits)
            else:
                assert any(gap <= n <= gap + 8 for n in lits), (name, gap, lits)
        if name == "snappy":
            assert min(lits) <= 60 < max(lits)


def test_zlib_block_types_per_chunk():
    g = W.GEOMETRY["default"]
    one = zlib_chunks(M.deflate_emulate(W.make_case(g, "one_value", 3 * g.chunk + 7).body))
    assert len(one) == 4 and all(t in (1, 2) for t, _ in one)
    fib = zlib_chunks(M.deflate_emulate(W.make_case(g, "fibonacci", 2 * g.chunk).body))
    assert fib == [(2, 15)] * 2, "a Fibonacci-skewed chunk gets a dynamic code at the 15-bit length limit"
    gaps = zlib_chunks(M.deflate_emulate(W.make_case(g, "literal_gaps", 2 * g.chunk).body))
    assert len(gaps) == 2 and all(t in (1, 2) for t, _ in gaps)


def test_zstd_block_and_literals_types():
    """below 128 with matches: a compressed block with Huffman literals; one byte of 128 makes them raw; random: a
    raw block"""
    g = W.GEOMETRY["zstd"]

    def kinds(content, n):
        res = []
        for f, fhd, fcs, blocks in ZS.frames(ZS.compress_emulate(W.make_case(g, content, n).body)):
            assert len(blocks) == 1
            bt = blocks[0][0]
            single = (fhd >> 5) & 1
            hdr = 4 + 1 + (0 if single else 1) + [0, 1, 2, 4][fhd & 3] + [single, 2, 4, 8][fhd >> 6] + 3
            res.append((bt, f[hdr] & 3 if bt == 2 else None))
        return res

    # the first frame holds the record's value length (a vint with bytes of 128 and more), the last one FF FF
    assert kinds("below_128", 3 * g.chunk + 7) == [(2, 0), (2, 2), (2, 2), (0, None)]
    assert kinds("below_128_one_128", 3 * g.chunk + 7) == [(2, 0), (2, 0), (2, 2), (0, None)]
    assert kinds("random", 4096) == [(0, None)]

"""Regenerates the SnappyCodec fixture of tests/golden/ and its checksums (SNAPPY_SHA256SUMS).  Run it on a build machine
that has pyarrow (which bundles libsnappy); the tests read the committed files and need no pyarrow.

  snappy_segments.bin / snappy_segments.json  -- SnappyCodec IFile segments (TIF\\x01, stream, CRC-32 of the stream)
      written the way Java's IFile.Writer drives BlockCompressorStream over SnappyCompressor at the default buffer size:
      the bodies come from the oracle's IFile writer, the block cutting follows the Java rules (tests/lz4_model.py
      java_stream, MAX_INPUT_SIZE 218,422), the chunks are libsnappy's.  One segment holds a value of 700,000 bytes:
      a block of several chunks.  The "crafted_*" segments hold one block each of hand-made chunks with elements
      libsnappy never writes (tests/snappy_model.py crafted_chunks).  The manifest gives each segment's name, rawLength
      and length.
"""
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]


def snappy_fixture():
    import codec_model as CM
    import snappy_model as M
    from oracle import tez_oracle as O

    def long_value_body():
        pat = b"".join(b"row %06d of a long compressible value;" % i for i in range(400))
        big = (pat * (700000 // len(pat) + 1))[:700000]
        recs = [(O.text("alpha%d" % i), O.int_writable(i)) for i in range(50)]
        recs += [(O.text("beta"), big)] + [(O.text("gamma%d" % i), O.int_writable(i)) for i in range(50)]
        out, _, _ = O.write_ifile(recs, rle=False)
        return CM.body_of(out)

    def incompressible_body():
        rng = random.Random(14)
        recs = sorted((O.text("k%06d" % i), rng.randbytes(rng.randint(100, 3000))) for i in range(60))
        out, _, _ = O.write_ifile(recs, rle=False)
        return CM.body_of(out)

    bodies = [
        ("wordcount", CM.wordcount_body(n=60000, vocab=3000, seed=11)),
        ("c3", CM.c3_body(seg_bytes=300000, seed=13)),
        ("incompressible", incompressible_body()),
        ("long_value", long_value_body()),
    ]
    data, man = b"", []

    def add(name, z, body):
        seg = M.segment(z)
        assert M.decode_stream(z, len(body)) == body == M.decode_stream(z, len(body), M.libsnappy_chunk)
        man.append({"name": name, "raw_length": len(body) + 4, "part_length": len(seg)})
        return seg

    for name, body in bodies:
        data += add(name, M.java_stream(M.ifile_writes(body)), body)
    for name, chunk in M.crafted_chunks():
        body = M.decode_chunk(chunk)
        data += add("crafted_" + name, M.one_block([chunk]), body)
    open(M.FIXTURE, "wb").write(data)
    json.dump({"segments": man}, open(M.MANIFEST, "w"), indent=1)
    open(M.MANIFEST, "a").write("\n")
    return [M.FIXTURE, M.MANIFEST]


if __name__ == "__main__":
    sums = []
    for f in snappy_fixture():
        h = hashlib.sha256(open(f, "rb").read()).hexdigest()
        sums.append("%s  %s\n" % (h, os.path.basename(f)))
        print(h, os.path.getsize(f), os.path.basename(f))
    open(os.path.join(HERE, "SNAPPY_SHA256SUMS"), "w").write("".join(sums))

"""Regenerates the Lz4Codec fixture of tests/golden/ and its checksums (LZ4_SHA256SUMS).  Run it on a build machine
that has the system liblz4; the tests read the committed files and need no liblz4.

  lz4_segments.bin / lz4_segments.json  -- Lz4Codec IFile segments (TIF\\x01, stream, CRC-32 of the stream) written the
      way Java's IFile.Writer drives BlockCompressorStream over Lz4Compressor at the default buffer size: the bodies come
      from the oracle's IFile writer, the block cutting follows the Java rules (tests/lz4_model.py java_stream), the
      chunks are liblz4's (acceleration 1 and 8, HC level 9).  The manifest gives each segment's name, rawLength and
      length.  One segment holds a value longer than 261,100 bytes: a block of several chunks.
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]


def lz4_fixture():
    import codec_model as CM
    import lz4_model as M
    from oracle import tez_oracle as O

    def long_value_body():
        pat = b"".join(b"row %06d of a long compressible value;" % i for i in range(400))
        big = (pat * (700000 // len(pat) + 1))[:700000]
        recs = [(O.text("alpha%d" % i), O.int_writable(i)) for i in range(50)]
        recs += [(O.text("beta"), big)] + [(O.text("gamma%d" % i), O.int_writable(i)) for i in range(50)]
        out, _, _ = O.write_ifile(recs, rle=False)
        return CM.body_of(out)

    cases = [
        ("wordcount_accel1", CM.wordcount_body(n=60000, vocab=3000, seed=11), lambda d: M.lz4_compress(d, accel=1)),
        ("wordcount_accel8", CM.wordcount_body(n=60000, vocab=3000, seed=12), lambda d: M.lz4_compress(d, accel=8)),
        ("c3_hc", CM.c3_body(seg_bytes=300000, seed=13), lambda d: M.lz4_compress(d, mode="hc")),
        ("long_value_accel1", long_value_body(), lambda d: M.lz4_compress(d, accel=1)),
    ]
    data, man = b"", []
    for name, body, fn in cases:
        seg = M.segment(M.java_stream(M.ifile_writes(body), fn))
        assert M.decode_stream(seg[4:-4], len(body)) == body
        man.append({"name": name, "raw_length": len(body) + 4, "part_length": len(seg)})
        data += seg
    open(M.FIXTURE, "wb").write(data)
    json.dump({"segments": man}, open(M.MANIFEST, "w"), indent=1)
    open(M.MANIFEST, "a").write("\n")
    return [M.FIXTURE, M.MANIFEST]


if __name__ == "__main__":
    sums = []
    for f in lz4_fixture():
        h = hashlib.sha256(open(f, "rb").read()).hexdigest()
        sums.append("%s  %s\n" % (h, os.path.basename(f)))
        print(h, os.path.getsize(f), os.path.basename(f))
    open(os.path.join(HERE, "LZ4_SHA256SUMS"), "w").write("".join(sums))

"""Regenerates the ZStandardCodec fixture of tests/golden/ and its checksums (ZSTD_SHA256SUMS).  Run it on a build
machine that has the system libzstd; the tests read the committed files and need no libzstd.

  zstd_segments.bin / zstd_segments.json  -- ZStandardCodec IFile segments (TIF\\x01, stream, CRC-32 of the stream)
      written the way Java's IFile.Writer drives CompressorStream over ZStandardCompressor (tests/zstd_model.py
      hadoop_stream): the bodies come from the oracle's IFile writer, the frames are libzstd's.  The manifest gives each
      segment's name, rawLength and length.  Cases: streams at levels 1, 3 and 19; Content_Checksum on; a one-shot frame
      with Frame_Content_Size; a 2^27 window with long-distance matching; a 700,000-byte value; two frames with a
      skippable frame between them.
"""
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]


def zstd_fixture():
    import codec_model as CM
    import zstd_model as M
    from oracle import tez_oracle as O

    def body_of(recs):
        out, _, _ = O.write_ifile(recs, rle=False)
        return CM.body_of(out)

    def long_value_body():
        pat = b"".join(b"row %06d of a long compressible value;" % i for i in range(400))
        big = (pat * (700000 // len(pat) + 1))[:700000]
        recs = [(O.text("alpha%d" % i), O.int_writable(i)) for i in range(50)]
        return body_of(recs + [(O.text("beta"), big)] + [(O.text("gamma%d" % i), O.int_writable(i)) for i in range(50)])

    def far_repeat_body():
        # 400 KB of values drawn from four letters, then the same values again: matches 400 KB back
        rng = random.Random(7)
        vals = [bytes(rng.choice(b"acgt") for _ in range(1000)) for _ in range(400)]
        recs = [(O.text("k%04d" % i), v) for i, v in enumerate(vals)]
        return body_of(recs + [(O.text("k%04d" % (i + 400)), v) for i, v in enumerate(vals)])

    wc = CM.wordcount_body(n=60000, vocab=3000, seed=21)
    half = wc.index(b"\x00", len(wc) // 2)   # any cut: frames need not end on a record
    cases = [
        ("wordcount_level1", CM.wordcount_body(n=60000, vocab=3000, seed=22), lambda b: M.hadoop_stream(b, level=1)),
        ("wordcount_level3", CM.wordcount_body(n=60000, vocab=3000, seed=23), lambda b: M.hadoop_stream(b, level=3)),
        ("int_long_level19", CM.int_long_body(n=20000, seed=24), lambda b: M.hadoop_stream(b, level=19)),
        ("wordcount_checksum", CM.wordcount_body(n=20000, vocab=2000, seed=25), lambda b: M.hadoop_stream(b, checksum=True)),
        ("wordcount_oneshot", CM.wordcount_body(n=20000, vocab=2000, seed=26), lambda b: M.hadoop_stream(b, oneshot=True)),
        ("far_repeat_window27_ldm", far_repeat_body(), lambda b: M.hadoop_stream(b, window_log=27, ldm=True)),
        ("long_value_level3", long_value_body(), lambda b: M.hadoop_stream(b, level=3)),
        ("two_frames_skippable", wc, lambda b: M.hadoop_stream(b[:half]) + M.skippable(b"tez") + M.hadoop_stream(b[half:])),
    ]
    data, man = b"", []
    for name, body, fn in cases:
        seg = M.segment(fn(body))
        assert M.hadoop_read(seg[4:-4], len(body)) == body, name
        man.append({"name": name, "raw_length": len(body) + 4, "part_length": len(seg)})
        data += seg
    open(M.FIXTURE, "wb").write(data)
    json.dump({"segments": man}, open(M.MANIFEST, "w"), indent=1)
    open(M.MANIFEST, "a").write("\n")
    return [M.FIXTURE, M.MANIFEST]


if __name__ == "__main__":
    sums = []
    for f in zstd_fixture():
        h = hashlib.sha256(open(f, "rb").read()).hexdigest()
        sums.append("%s  %s\n" % (h, os.path.basename(f)))
        print(h, os.path.getsize(f), os.path.basename(f))
    open(os.path.join(HERE, "ZSTD_SHA256SUMS"), "w").write("".join(sums))

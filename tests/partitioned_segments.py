"""Partitioned segments for the bounded merge's write tests (tests/test_merge_bounded_gpu.py,
tests/test_merge_bounded_codec_gpu.py): partitions that span many steps at the 16 MiB floor budget, next to small and
empty ones."""
import random

from oracle import tez_oracle as O


def partitioned(P=16, G=3, seed=1):
    """G producers' segments of P partitions: three large partitions (each spans many steps at the floor), small ones,
    and empty ones first, inside and last.  Returns the segments, their partitions and the large partitions."""
    rng = random.Random(seed)
    recs = [0, 40000, 300, 0, 3000, 45000, 0, 0, 200, 2500, 50000, 10, 1, 0, 700, 0]
    segs, parts = [], []
    for g in range(G):
        for p in range(P):
            if not recs[p]:
                continue
            keys = sorted(b"k%09d" % rng.randrange(10 ** 9) for _ in range(recs[p]))
            segs.append(O.write_ifile([(k, b"v%d" % (i % 97) * (1 + i % 3)) for i, k in enumerate(keys)])[0])
            parts.append(p)
    return segs, parts, [p for p in range(P) if recs[p] >= 40000]

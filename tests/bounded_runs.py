"""The bounded merge runs the bounded-merge GPU tests share: one merge handle's outputs, and a bounded merge with
compressed output at several budgets checked against the one-step merge with the same codec."""
import os

import tez_b200 as T

FLOOR = 16 << 20


def run(segs, tmp=None, P=1, parts=None, rle=False, check_same=True, combiner=0, iterate=False, **kw):
    """written bytes (P = 1: segment, rawLength, partLength; else file.out, file.out.index, index), records, counts,
    output_bound, bounded_info (None unbounded)"""
    with T.GpuMerger(segs, partitions=parts, num_partitions=P, **kw) as m:
        if not check_same:
            m.set_check_for_same_keys(False)
        if combiner:
            m.set_combiner(combiner)
        recs = list(m.records(batch_records=997, batch_bytes=1 << 16)) if iterate else None
        if P == 1:
            seg, raw, part, _ = m.write_ifile(rle=rle)
            assert part == len(seg)
            out = (seg, raw, part)
        else:
            f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
            index, _ = m.write_partitions(f, fi, rle=rle)
            out = (open(f, "rb").read(), open(fi, "rb").read(), index.tolist())
        info = m.bounded_info() if "device_budget" in kw else None
        return out, recs, m.counts(), m.output_bound(), info


def check(segs, codec, tmp=None, mid=4, **kw):
    """the one-step codec merge; the bounded handle at the default budget (one step) and at the floor and need // mid
    (several steps, at most the budget): the same outputs.  Returns {budget: (outputs, steps)} of the bounded runs."""
    exp = run(segs, tmp=tmp, codec=codec, **kw)
    one = run(segs, tmp=tmp, device_budget=0, write_codec=codec, **kw)
    assert one[4][0] == 1
    assert one[:4] == exp[:4]
    need = one[4][1]
    got = {}
    for b in sorted({FLOOR, max(FLOOR, need // mid)}, reverse=True):
        r = run(segs, tmp=tmp, device_budget=b, write_codec=codec, **kw)
        steps, peak, _ = r[4]
        assert peak <= b, (b, peak)
        assert steps > 1, (b, need)
        assert r[0] == exp[0], b
        assert r[1] == exp[1] and r[2] == exp[2], b
        assert r[3] >= len(r[0][0])           # output_bound bounds the compressed bytes once the counts are known
        got[b] = (r[0], steps)
    return got

"""Shared helpers of the merge tests: placing segments in device memory, running one merge through every output it
hands out, and the reference checks of a merge -- the oracle's TezMerger per partition and the stable merge model of
DESIGN.md section 6, records, isSameKey flags and the written IFile."""
import random

import numpy as np
import torch

from oracle import tez_oracle as O
import tez_b200 as T

import sort_order_model as SOM

GUARD = 4096       # controlled bytes before the first and after the last segment of every buffer


# ------------------------------------------------------------------------------------------------ placement
# A layout maps n segments to (address order, per-segment slot).  A slot is (buffer, residue, gap): the segment starts
# `gap` bytes after the previous segment of its buffer, then rounded up to 16 plus `residue`; residue None starts it
# exactly `gap` bytes after the previous one (back to back when 0).
def _layout_aligned(n):
    """every start 16-aligned, addresses descending against the caller's order"""
    return list(range(n))[::-1], [(0, 0, 16 * (1 + i % 4)) for i in range(n)]


def _layout_residues(n):
    """residues 1..15, one per segment, in two allocations, addresses in a shuffled order"""
    order = list(range(n))
    random.Random(n).shuffle(order)
    return order, [(i % 2, 1 + i % 15, 16 + (7 * i) % 48) for i in range(n)]


def _layout_packed(n):
    """back to back from an odd offset, in the caller's order (each start inherits the previous lengths)"""
    return list(range(n)), [(0, 3 if i == 0 else None, 0) for i in range(n)]


LAYOUTS = {"aligned": _layout_aligned, "residues": _layout_residues, "packed": _layout_packed}
POISONS = ["ff", "body", "random"]


def _body(seg):
    return bytes(seg[4:]) if bytes(seg[:3]) == b"TIF" else bytes(seg)


def place(segs, layout, poison, seed=0):
    """Copies segs into cuda:0 buffers laid out by `layout`, every other byte of the buffers set by `poison`.  Returns
    ([(ptr, len)] in the caller's order, the buffers to keep alive)."""
    n = len(segs)
    order, slots = LAYOUTS[layout](n)
    starts, ends = [0] * n, {}
    for i in order:
        b, res, gap = slots[i]
        end = ends.get(b)
        if end is None:
            start = GUARD + (res or 0)
        elif res is None:
            start = end + gap
        else:
            start = (end + gap + 15) // 16 * 16 + res
        starts[i] = start
        ends[b] = start + len(segs[i])
    bufs = {}
    for b, end in ends.items():
        size = end + GUARD
        rng = np.random.default_rng(seed * 31 + b)
        mine = [i for i in order if slots[i][0] == b]
        if poison == "ff":
            img = np.full(size, 0xFF, dtype=np.uint8)
        elif poison == "random":
            img = rng.integers(0, 256, size, dtype=np.uint8)
        else:
            donor = np.frombuffer(_body(segs[(mine[0] + 1) % n]), dtype=np.uint8)
            img = np.resize(donor, size).copy()
            for i in mine:   # right behind every segment: the start of another segment's records
                d = np.frombuffer(_body(segs[(i + 1) % n]), dtype=np.uint8)
                e = starts[i] + len(segs[i])
                img[e:e + min(len(d), size - e)] = d[:size - e]
        for i in mine:
            img[starts[i]:starts[i] + len(segs[i])] = np.frombuffer(bytes(segs[i]), dtype=np.uint8)
        bufs[b] = torch.from_numpy(img).to("cuda:0")
    return [(bufs[slots[i][0]].data_ptr() + starts[i], len(segs[i])) for i in range(n)], bufs


# ------------------------------------------------------------------------------------------------ merge
def run(segs, device_ptrs=False, P=1, parts=None, check=True, writer_rle=False, combiner=T.COMBINE_NONE, **kw):
    """Everything a merge hands out: mode, the merged IFile (P = 1), write_partitions_device's bytes and index, counts
    and records (without a combiner)."""
    out = {}
    with T.GpuMerger(segs, device_ptrs=device_ptrs, partitions=parts, num_partitions=P, combiner=combiner, **kw) as m:
        if not check:
            m.set_check_for_same_keys(False)
        out["mode"] = m.parse_info()[0]
        if P == 1:
            out["ifile"] = m.write_ifile(rle=writer_rle)[0]
        cap = m.output_bound()
        d = torch.full((cap + 32,), 0xA5, dtype=torch.uint8, device="cuda:0")
        n, index, _ = m.write_partitions_device(d.data_ptr(), cap, rle=writer_rle)
        out["file"] = d[:n].cpu().numpy().tobytes()
        out["index"] = index.tolist()
        if not combiner:
            out["counts"] = m.counts()
            out["records"] = list(m.records(batch_records=1 << 14, batch_bytes=1 << 22))
    return out


def partition_segments(out):
    """[IFile segment bytes or b""] per partition of a write_partitions_device result"""
    return [out["file"][s:s + n] for s, _, n in out["index"]]


# ------------------------------------------------------------------------------------------------ reference checks
def stable_model(segs, parts, P, cmp, has_header=True, check=True):
    """The device's merge contract: per partition, the stable sort of its segments' records (caller order) by key, as
    [(key, value, isSameKey)].  A record is isSameKey when its key equals the previous record's of its partition and
    it was read as SAME_KEY from its own segment or -- checkForSameKeys -- that previous record comes from another
    segment (emit_is_repeat, DESIGN.md section 6)."""
    res = []
    for p in range(P):
        recs = [(SOM.content(cmp, k), s, ks == O.SAME_KEY, k, v) for s, q in enumerate(parts or [0] * len(segs)) if q == p
                for ks, k, v in O.read_ifile(bytes(segs[s]), has_header=has_header)]
        recs.sort(key=lambda r: r[0])
        out = []
        for j, (c, s, repeat, k, v) in enumerate(recs):
            prev = recs[j - 1] if j else None
            same = prev is not None and prev[0] == c and (repeat or (check and prev[1] != s))
            out.append((k, v, same))
        res.append(out)
    return res


def model_ifile(model_part, writer_rle=False):
    """The IFile the merge writes for one partition of stable_model: flagged records as REPEAT_KEY, and the writer's
    own run-length test on top when writer_rle"""
    return O.write_ifile([(None if same else k, v) for k, v, same in model_part], rle=writer_rle)[0]


def _canon(records):
    """IFile records grouped by key: (key, key states, values sorted).  The oracle's order inside a group of equal keys
    from different segments is its heap's (parity unpinned, DESIGN.md section 6); keys, states and values are pinned."""
    out = []
    for ks, k, v in records:
        if out and out[-1][0] == k:
            out[-1][1].append(ks)
            out[-1][2].append(v)
        else:
            out.append((k, [ks], [v]))
    return [(k, s, sorted(v)) for k, s, v in out]


def check_oracle(host, segs, parts, P, cmp, check=True, writer_rle=False, has_header=True):
    """host merge vs the oracle's TezMerger (factor 100) per partition, and record for record, flag for flag and byte
    for byte against the stable merge model (every value is its record's global index, or the records of a key group
    are otherwise told apart)"""
    got = partition_segments(host)
    model = stable_model(segs, parts, P, cmp, has_header, check)
    for p in range(P):
        if P > 1 and not model[p]:   # send_empty_partition_details: a partition without records writes no segment
            assert got[p] == b"", "partition %d has no records but %d bytes" % (p, len(got[p]))
            continue
        mine = [bytes(s) for s, q in zip(segs, parts or [0] * len(segs)) if q == p]
        exp = O.merge(mine, cmp, factor=100, check_for_same_keys=check, writer_rle=writer_rle, has_header=has_header)
        assert len(got[p]) == len(exp["ifile"]), "partition %d: %d bytes, oracle %d" % (p, len(got[p]), len(exp["ifile"]))
        mine_recs = O.read_ifile(got[p])
        assert _canon(mine_recs) == _canon(O.read_ifile(exp["ifile"])), "partition %d differs from the oracle" % p
        assert [(k, v) for _, k, v in mine_recs] == [(k, v) for k, v, _ in model[p]], "partition %d: not the stable merge" % p
        assert got[p] == model_ifile(model[p], writer_rle), "partition %d: not the stable merge's IFile" % p
    if P == 1:
        assert host["ifile"] == host["file"]
        exp = O.merge([bytes(s) for s in segs], cmp, factor=100, check_for_same_keys=check, writer_rle=writer_rle,
                      has_header=has_header)
        assert [(k, s) for k, _, s in host["records"]] == [(k, s) for k, _, s in exp["records"]]
    assert host["records"] == [r for m in model for r in m], "records or isSameKey flags differ from the stable merge"
    assert host["counts"][0] == len(host["records"]) == sum(len(m) for m in model)

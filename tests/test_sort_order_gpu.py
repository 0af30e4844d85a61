"""GPU: the ORDER of records with equal or colliding keys.  Every record carries a distinct value (its collection index,
big-endian), so a record that is lost, written twice or moved inside a group of equal keys changes the output.

Contract (DESIGN.md section 6): the map side writes every partition as the stable sort of its records by the
comparator -- equal keys stay in collection order; the merger emits the stable sort of its segments' concatenation,
equal keys in (segment, position) order.  The reference model is a plain Python / numpy stable sort by
(partition, normalised key bytes, record index); segment bytes come from the oracle's IFile writer, the index must
equal the oracle sorter's (segment lengths do not depend on the order inside a group of equal keys)."""
import collections
import random
import zlib

import numpy as np
import pytest

from oracle import tez_oracle as O
import tez_b200 as T
import sort_order_model as M

pytestmark = pytest.mark.gpu

VW = 4   # value width of the variable-width cases: the record index, big-endian


def _pack(keys, vals):
    kv = bytearray()
    ko, vo, vl = [], [], []
    for k, v in zip(keys, vals):
        ko.append(len(kv))
        kv += k
        vo.append(len(kv))
        kv += v
        vl.append(len(v))
    return (np.frombuffer(bytes(kv), dtype=np.uint8) if kv else np.zeros(0, np.uint8),
            np.array(ko, np.uint32), np.array(vo, np.uint32), np.array(vl, np.uint32))


def _decode(out, index):
    """Per partition: [(key, value)] read back from the device's file.out."""
    res = []
    for p in range(index.shape[0]):
        start, _, part = (int(x) for x in index[p])
        res.append([(k, v) for _, k, v in O.read_ifile(out[start:start + part])] if part else [])
    return res


def _check_sample_order(cmp, keys, rng, pairs=300):
    """The Python sort key (normalised content) agrees with the oracle comparator on a sample."""
    for _ in range(pairs):
        a, b = rng.choice(keys), rng.choice(keys)
        ca, cb = M.content(cmp, a), M.content(cmp, b)
        got = O.compare(cmp, a, b)
        assert (got > 0) - (got < 0) == (ca > cb) - (ca < cb), (a.hex(), b.hex())


def _sort_and_check(keys, cmp, P, rle, partition=None, path=None, what=""):
    """Sorts keys (value = record index) on the device and checks: no record lost or duplicated, every partition in
    stable comparator order, file.out equal to the oracle writer's segments, index equal to the oracle sorter's.
    path: "table" / "raw" asserts which sort word the device builds (the host run of the same decision)."""
    n = len(keys)
    vals = [i.to_bytes(VW, "big") for i in range(n)]
    kv, ko, vo, vl = _pack(keys, vals)
    part_mode = O.PART_GIVEN if partition is not None else O.PART_HASH
    if path is not None:
        _, _, used = M.sort_words(keys, cmp, P, partition=partition)
        assert used == (path == "table"), "%s: the keys do not take the %s path" % (what, path)
    with T.GpuSorter(P, comparator=cmp, partitioner=part_mode, rle_policy=rle) as s:
        s.collect(kv, ko, vo, vl, None if partition is None else np.asarray(partition, np.int32))
        out, _, index, st = s.flush_to_memory()
    out = bytes(out)
    got = _decode(out, index)
    flat = sorted(r for seg in got for r in seg)
    assert flat == sorted(zip(keys, vals)), "%s: records lost or duplicated (%d read back, %d collected)" % (
        what, sum(len(g) for g in got), n)

    parts = list(partition) if partition is not None else [O.partition_of(cmp, k, P) for k in keys]
    cont = [M.content(cmp, k) for k in keys]
    order = sorted(range(n), key=lambda i: (parts[i], cont[i], i))
    exp = [[] for _ in range(P)]
    for i in order:
        exp[parts[i]].append((keys[i], vals[i]))
    for p in range(P):
        if got[p] != exp[p]:
            j = next(j for j in range(min(len(got[p]), len(exp[p]))) if got[p][j] != exp[p][j])
            raise AssertionError("%s: partition %d differs at position %d: expected record %d (key %s), got record %d (key %s)"
                                 % (what, p, j, int.from_bytes(exp[p][j][1], "big"), exp[p][j][0].hex(),
                                    int.from_bytes(got[p][j][1], "big"), got[p][j][0].hex()))
    segs = [O.write_ifile(e, rle=rle == T.RLE_ON)[0] for e in exp if e]
    assert out == b"".join(segs), what + ": file.out differs from the oracle writer's segments"
    ref = O.pipelined_sort(O.sorter_conf(P, cmp_kind=cmp, partitioner=part_mode, rle_policy=rle), kv, ko.astype(np.uint64),
                           vo - ko, vl, partition)
    assert np.array_equal(index, ref["index"]), what + ": index differs from the oracle sorter's"
    return st


# ------------------------------------------------------------------------------------------------ 1. alphabet saturation
@pytest.mark.parametrize("P", [1, 64])
@pytest.mark.parametrize("c", [255, 256])
@pytest.mark.parametrize("cmp", [O.CMP_BYTES, O.CMP_TEXT])
def test_saturated_alphabet_position_sorts_in_order(cmp, c, P):
    """All 256 (or 255) byte values at one content position, tiny alphabets elsewhere: the alphabet table packs that
    position with 9 (8) bit ranks; keys with byte 0xFF there belong after every other value, not before."""
    rng = random.Random(c * 10 + P + cmp)
    for q in (0, 1, 5, 15):
        contents = M.alphabet_contents(rng, cmp, c, q)
        keys = [M.make_key(cmp, x) for x in contents]
        _check_sample_order(cmp, keys, rng, 50)
        _sort_and_check(keys, cmp, P, T.RLE_OFF, path="table", what="c=%d q=%d" % (c, q))


def _stable_merge_expected(segs_recs, cmp):
    """Stable sort of the segments' concatenation: equal keys in (segment, position) order."""
    allr = [(k, v, s, j) for s, recs in enumerate(segs_recs) for j, (k, v) in enumerate(recs)]
    return sorted(allr, key=lambda r: (M.content(cmp, r[0]), r[2], r[3]))


def _gpu_merge(segs, cmp, check=True, writer_rle=False):
    with T.GpuMerger(segs, comparator=cmp) as m:
        if not check:
            m.set_check_for_same_keys(False)
        recs = list(m.records(batch_records=4096, batch_bytes=1 << 20))
    with T.GpuMerger(segs, comparator=cmp) as m:
        if not check:
            m.set_check_for_same_keys(False)
        seg, _, _, _ = m.write_ifile(rle=writer_rle)
    return recs, seg


@pytest.mark.parametrize("c", [255, 256])
def test_saturated_alphabet_position_merges_in_order(c):
    """The merger builds the same sort word: sorted Text runs whose first content byte takes all 256 (255) values."""
    rng = random.Random(c)
    vals = M.sample_values(rng, c)
    segs_recs, nrec = [], 0
    for s in range(8):
        contents = [bytes([rng.choice(vals)]) + bytes(rng.choice(b"ab") for _ in range(rng.randrange(0, 8)))
                    for _ in range(200)]
        if s == 0:
            contents += [bytes([v]) + b"ab" for v in vals]
        keys = sorted((M.make_key(O.CMP_TEXT, x) for x in contents), key=lambda k: M.content(O.CMP_TEXT, k))
        segs_recs.append([(k, (nrec + j).to_bytes(VW, "big")) for j, k in enumerate(keys)])
        nrec += len(keys)
    segs = [O.write_ifile(r, rle=False)[0] for r in segs_recs]
    exp = _stable_merge_expected(segs_recs, O.CMP_TEXT)
    recs, seg = _gpu_merge(segs, O.CMP_TEXT, check=False)
    assert sorted((k, v) for k, v, _ in recs) == sorted((k, v) for r in segs_recs for k, v in r), "records lost or duplicated"
    assert [(k, v) for k, v, _ in recs] == [(k, v) for k, v, _, _ in exp], "merged order differs from the stable sort"
    assert seg == O.write_ifile([(k, v) for k, v, _, _ in exp], rle=False)[0]


# ------------------------------------------------------------------------------------------------ 2. tie-group sizes
def _group_keys(rng, g, kind, path, ngroups):
    """ngroups sort-word collision groups of g records each plus filler keys, shuffled.  Returns (keys, group of every
    key, -1 for filler).
    equal: one key per group; distinct: a shared 16-byte head (longer than any sort word covers) and distinct tails;
    mixed: a shared head and tails from about g / 3 values, so equal sub-runs sit inside a group of different keys."""
    alpha = b"abcdefgh" if path == "table" else bytes(range(256))
    groups = []
    for _ in range(ngroups):
        head = bytes(rng.choice(alpha) for _ in range(16))
        if kind == "equal":
            groups.append([head + b"xyz"] * g)
        elif kind == "distinct":
            groups.append([head + j.to_bytes(3, "big") + bytes(rng.choice(alpha) for _ in range(rng.randrange(3)))
                           for j in rng.sample(range(1 << 20), g)])
        else:
            tails = [bytes(rng.choice(alpha) for _ in range(rng.randrange(0, 5))) for _ in range(max(1, g // 3))]
            groups.append([head + rng.choice(tails) for _ in range(g)])
    keys = [k for grp in groups for k in grp]
    gid = [i for i, grp in enumerate(groups) for _ in grp]
    nfill = max(200, len(keys) // 4)
    keys += [bytes(rng.choice(alpha) for _ in range(rng.randrange(1, 20))) for _ in range(nfill)]
    gid += [-1] * nfill
    perm = list(range(len(keys)))
    rng.shuffle(perm)
    return [keys[j] for j in perm], [gid[j] for j in perm]


@pytest.mark.parametrize("path", ["table", "raw"])
@pytest.mark.parametrize("g", [2, 3, 15, 16, 17, 18, 64, 5000])
def test_tie_groups_keep_collection_order(g, path, monkeypatch):
    """Collision groups of exactly g records at and around TIE_SMALL_MAX (16, ordered in place by k_tie_fix), larger
    ones (k_group_equal for all-equal groups, refinement rounds for the rest), on the alphabet-table and the raw-prefix
    sort word, RLE off and on.  One partition, so that the partition bits of the word cannot split a group; the host run
    of the word build confirms every group is one sort word that no other record shares."""
    if path == "raw":
        monkeypatch.setenv("TEZGPU_NO_SYM", "1")
    rng = random.Random(g * 7 + (path == "raw"))
    ngroups = max(2, min(60, 6000 // g))
    for kind in ("equal", "distinct", "mixed"):
        keys, gid = _group_keys(rng, g, kind, path, ngroups)
        words, _, used = M.sort_words(keys, O.CMP_BYTES, 1, use_sym=path == "table")
        assert used == (path == "table"), "g=%d %s: the keys do not take the %s path" % (g, kind, path)
        per_word = collections.Counter(words.tolist())
        group_words = collections.defaultdict(set)
        for w, grp in zip(words.tolist(), gid):
            if grp >= 0:
                group_words[grp].add(w)
        for grp in range(ngroups):
            (w,) = group_words[grp]          # one sort word per group ...
            assert per_word[w] == g, "g=%d %s: group %d collides with %d records" % (g, kind, grp, per_word[w])
        for rle in (T.RLE_OFF, T.RLE_ON):
            _sort_and_check(keys, O.CMP_BYTES, 1, rle, what="g=%d %s %s rle=%d" % (g, kind, path, rle))


# ------------------------------------------------------------------------------------------------ 3. refinement depth
@pytest.mark.parametrize("path", ["table", "raw"])
@pytest.mark.parametrize("cmp", [O.CMP_BYTES, O.CMP_TEXT])
def test_refinement_depth_prefixes_and_zero_padding(cmp, path, monkeypatch):
    """Keys that share prefixes of depth0 + 3k + {-1, 0, +1} bytes (k up to 45: past the 127-byte cap of the length
    tag), proper prefixes of each other, zero bytes right after a key's end (the refinement pads its last 3-byte chunk
    with zeros), and a group of > 16 keys equal on the next three bytes that differ only later."""
    if path == "raw":
        monkeypatch.setenv("TEZGPU_NO_SYM", "1")
    rng = random.Random(cmp * 3 + (path == "raw"))
    alpha = b"abcd" if path == "table" else bytes(range(1, 256))
    base = bytes(rng.choice(alpha) for _ in range(200))
    depth0 = 16 if path == "table" else 4      # at least the bytes the sort word covers (the refinement starts there)
    contents = []
    for k in range(0, 46):
        for d in (-1, 0, 1):
            ln = depth0 + 3 * k + d
            if ln <= 0:
                continue
            pre = base[:ln]
            contents += [pre, pre + b"\0", pre + b"\0\0", pre + b"\0\0\0", pre + b"\0\x01", pre + b"\0\0\0\0",
                         pre + bytes([alpha[0]]), pre[:-1]]
            contents += [pre + bytes(rng.choice(alpha) for _ in range(rng.randrange(0, 8))) for _ in range(6)]
    # > 16 keys equal on depth0 .. depth0 + 2, different later
    contents += [base[:depth0 + 3] + bytes(rng.choice(alpha) for _ in range(rng.randrange(1, 6))) for _ in range(40)]
    contents = contents * 2                      # every key twice: equal pairs inside the groups
    rng.shuffle(contents)
    keys = [M.make_key(cmp, x) for x in contents]
    _check_sample_order(cmp, keys, rng)
    for rle in (T.RLE_OFF, T.RLE_ON):
        _sort_and_check(keys, cmp, 1, rle, path=None if path == "raw" else "table", what="%s rle=%d" % (path, rle))


# ------------------------------------------------------------------------------------------------ 4. tile edges
@pytest.mark.parametrize("n", [6143, 6144, 6145, 12289])
def test_record_counts_at_radix_tile_edges(n):
    """The 32-bit onesweep tile holds 384 x 16 = 6144 words: record counts around it, keys with many collisions."""
    rng = random.Random(n)
    heads = [bytes(rng.getrandbits(8) for _ in range(4)) for _ in range(n // 8)]
    keys = [rng.choice(heads) + bytes(rng.getrandbits(2) for _ in range(rng.randrange(0, 3))) for _ in range(n)]
    _sort_and_check(keys, O.CMP_BYTES, 1, T.RLE_OFF, path="raw", what="n=%d" % n)
    _sort_and_check(keys, O.CMP_BYTES, 64, T.RLE_ON, what="n=%d P=64" % n)


@pytest.mark.parametrize("m", [5119, 5120, 5121, 15361])
def test_tied_sets_at_refinement_tile_edges(m):
    """m records with one sort word (the 64-bit refinement sort's tile holds 512 x 10 = 5120): distinct and repeated
    tails, so the rounds have work at every depth."""
    rng = random.Random(m)
    tails = [bytes(rng.getrandbits(8) for _ in range(rng.randrange(0, 7))) for _ in range(m // 3)]
    keys = [b"HEAD" + rng.choice(tails) for _ in range(m)]
    keys += [bytes(rng.getrandbits(8) for _ in range(6)) for _ in range(1000)]
    rng.shuffle(keys)
    _sort_and_check(keys, O.CMP_BYTES, 1, T.RLE_OFF, path="raw", what="m=%d" % m)


def test_groups_straddling_tie_fix_and_scan_tiles(monkeypatch):
    """One partition, groups placed at sorted positions around 2048 j (the k_tie_fix and tie scan tiles), small (in
    place) and large (refinement), equal and distinct keys."""
    rng = random.Random(2048)
    spans = [(2040, 2060, "distinct"), (4090, 4100, "equal"), (6140, 6150, "distinct"), (8180, 8230, "mixed"),
             (10230, 10250, "equal"), (12285, 12290, "distinct")]
    n = 14000
    keys, i = [], 0
    while i < n:        # unique position i: sort word 2 i; a group at positions [a, b): sort word 2 a + 1
        sp = next((s for s in spans if s[0] == i), None)
        if sp is None:
            keys.append((2 * i).to_bytes(4, "big") + bytes(rng.getrandbits(8) for _ in range(rng.randrange(0, 3))))
            i += 1
            continue
        a, b, kind = sp
        for j in range(b - a):
            tail = {"equal": b"", "distinct": j.to_bytes(2, "big"), "mixed": bytes([j % 4])}[kind]
            keys.append((2 * a + 1).to_bytes(4, "big") + tail)
        i = b
    order = list(range(len(keys)))
    rng.shuffle(order)
    keys = [keys[j] for j in order]
    for path in ("table", "raw"):
        if path == "raw":
            monkeypatch.setenv("TEZGPU_NO_SYM", "1")
        for rle in (T.RLE_OFF, T.RLE_ON):
            _sort_and_check(keys, O.CMP_BYTES, 1, rle, path="table" if path == "table" else None,
                            what="straddling groups, %s rle=%d" % (path, rle))


# ------------------------------------------------------------------------------------------------ 5. fixed width at scale
def _np_hash_partition(keys, P):
    """HashPartitioner over WritableComparator.hashBytes of every row of keys (uint8 [n, klen])."""
    h = np.ones(keys.shape[0], dtype=np.uint32)
    for j in range(keys.shape[1]):
        h = h * np.uint32(31) + keys[:, j].astype(np.int8).astype(np.int32).astype(np.uint32)
    return ((h & np.uint32(0x7FFFFFFF)) % np.uint32(P)).astype(np.int64)


def _np_long_partition(keys, P):
    v = keys.astype(np.uint64)
    x = np.zeros(keys.shape[0], dtype=np.uint64)
    for j in range(8):
        x = (x << np.uint64(8)) | v[:, j]
    h = ((x ^ (x >> np.uint64(32))) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return ((h & np.uint32(0x7FFFFFFF)) % np.uint32(P)).astype(np.int64)


def _np_expected_fixed(rows, klen, part, P, cmp):
    """file.out (RLE off) of fixed-width rows [n, klen + vlen] sorted stably by (partition, key)."""
    n = rows.shape[0]
    norm = rows[:, :klen].copy()
    if cmp == O.CMP_LONG:
        norm[:, 0] ^= 0x80
    cols = [np.arange(n)]
    for j in range(klen - 1, -1, -1):
        cols.append(norm[:, j])
    cols.append(part)
    order = np.lexsort(cols)
    hdr = np.array([klen, rows.shape[1] - klen], dtype=np.uint8)
    srt = rows[order]
    bounds = np.searchsorted(part[order], np.arange(P + 1))
    out = []
    for p in range(P):
        a, b = bounds[p], bounds[p + 1]
        if a == b:
            continue
        body = np.empty((b - a, 2 + rows.shape[1]), dtype=np.uint8)
        body[:, :2] = hdr
        body[:, 2:] = srt[a:b]
        body = body.tobytes() + b"\xff\xff"
        out.append(b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big"))
    return b"".join(out), order


def _fixed_check(rows, klen, P, cmp, device=False):
    n, width = rows.shape
    kv = np.ascontiguousarray(rows).reshape(-1)
    keys = rows[:, :klen]
    part = _np_long_partition(keys, P) if cmp == O.CMP_LONG else _np_hash_partition(keys, P)
    rng = random.Random(n)
    for i in rng.sample(range(n), 200):
        assert part[i] == O.partition_of(cmp, keys[i].tobytes(), P)
    exp, order = _np_expected_fixed(rows, klen, part, P, cmp)
    with T.GpuSorter(P, comparator=cmp, fixed=(klen, width - klen), rle_policy=T.RLE_OFF) as s:
        if device:
            import torch
            d_kv = torch.from_numpy(kv).cuda()
            cap = n * (width + 2) + 16 * P + 4096
            d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
            out_len, index, _ = s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), cap)
            out = d_out[:out_len].cpu().numpy()
        else:
            s.collect_fixed(kv)
            out, _, index, _ = s.flush_to_memory()
    out = np.asarray(out)
    # multiset: every value (the record index) exactly once, behind its own key
    body = []
    for p in range(P):
        start, _, plen = (int(x) for x in index[p])
        if plen:
            body.append(out[start + 4:start + plen - 6].reshape(-1, width + 2)[:, 2:])
    got = np.concatenate(body) if body else np.zeros((0, width), np.uint8)
    assert got.shape[0] == n, "records lost or duplicated: %d read back, %d collected" % (got.shape[0], n)
    vidx = np.zeros(n, dtype=np.int64)
    for j in range(width - klen):
        vidx = (vidx << 8) | got[:, klen + j].astype(np.int64)
    assert np.array_equal(np.sort(vidx), np.arange(n)), "records lost or duplicated"
    assert np.array_equal(got, rows[vidx]), "a value moved away from its key"
    if not np.array_equal(vidx, order):
        j = int(np.argmax(vidx != order))
        raise AssertionError("sorted position %d: expected record %d, got record %d" % (j, order[j], vidx[j]))
    assert out.tobytes() == exp, "file.out differs from the stable numpy model"
    ref = O.pipelined_sort_fixed(O.sorter_conf(P, cmp_kind=cmp, rle_policy=T.RLE_OFF), kv, klen, width - klen)
    assert np.array_equal(index, ref["index"])


def _index_values(n, vlen):
    v = np.zeros((n, vlen), dtype=np.uint8)
    idx = np.arange(n, dtype=np.uint64)
    for j in range(min(vlen, 8)):
        v[:, vlen - 1 - j] = ((idx >> np.uint64(8 * j)) & np.uint64(0xFF)).astype(np.uint8)
    return v


def test_fixed_width_one_giant_group_per_partition():
    """2e6 16-byte keys whose first 12 bytes are constant, 64 hash partitions: every partition is one group of
    distinct keys (refinement rounds over 2e6 records), 16-byte values on the 16-byte fast stage."""
    n = 2_000_000
    rng = np.random.default_rng(5)
    keys = np.empty((n, 16), dtype=np.uint8)
    keys[:, :12] = np.frombuffer(b"constantHEAD", dtype=np.uint8)
    keys[:, 12:] = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    _fixed_check(np.concatenate([keys, _index_values(n, 16)], axis=1), 16, 64, O.CMP_BYTES)


def test_fixed_width_ten_distinct_keys():
    """3e6 records over 10 distinct keys: large all-equal groups settled by k_group_equal without refinement."""
    n = 3_000_000
    rng = np.random.default_rng(6)
    pool = rng.integers(0, 256, (10, 16), dtype=np.uint8)
    keys = pool[rng.integers(0, 10, n)]
    _fixed_check(np.concatenate([keys, _index_values(n, 8)], axis=1), 16, 64, O.CMP_BYTES, device=True)


def test_fixed_width_long_keys_heavy_duplication():
    """LongWritable 8 + 8 (generic stage, sign flip), 1.5e6 records over 3000 values around zero."""
    n = 1_500_000
    rng = np.random.default_rng(7)
    v = rng.integers(-1500, 1500, n).astype(">i8")
    keys = np.frombuffer(v.tobytes(), dtype=np.uint8).reshape(n, 8)
    _fixed_check(np.concatenate([keys, _index_values(n, 8)], axis=1), 8, 16, O.CMP_LONG)


# ------------------------------------------------------------------------------------------------ 6. merger contract
def _merge_segments(rng, nseg, per_seg, nkeys, repeats):
    """Sorted Text runs over a small key space; repeats: a key may occur several times in one run."""
    words = sorted({"".join(rng.choice("abcdefgh") for _ in range(rng.randrange(1, 7))) for _ in range(nkeys)})
    segs_recs, nrec = [], 0
    for _ in range(nseg):
        if repeats:
            ks = [rng.choice(words) for _ in range(per_seg)]
        else:
            ks = rng.sample(words, min(per_seg, len(words)))
        ks.sort()
        segs_recs.append([(O.text(w), (nrec + j).to_bytes(VW, "big")) for j, w in enumerate(ks)])
        nrec += len(ks)
    return segs_recs


@pytest.mark.parametrize("nseg", [2, 7, 40])
def test_merge_is_stable_sort_of_concatenation(nseg):
    """Equal keys inside and across runs, all values distinct: records() is the stable sort of the concatenation in
    (segment, position) order; without checkForSameKeys the written IFile is the oracle writer's file of that
    sequence, with records that were SAME_KEY in their own (RLE) run written as repeats."""
    rng = random.Random(nseg)
    for rle_inputs in (False, True):
        segs_recs = _merge_segments(rng, nseg, 400, 150, repeats=True)
        segs = [O.write_ifile(r, rle=rle_inputs)[0] for r in segs_recs]
        exp = _stable_merge_expected(segs_recs, O.CMP_TEXT)
        recs, seg = _gpu_merge(segs, O.CMP_TEXT, check=False)
        assert sorted((k, v) for k, v, _ in recs) == sorted((k, v) for r in segs_recs for k, v in r), "records lost or duplicated"
        got = [(k, v) for k, v, _ in recs]
        want = [(k, v) for k, v, _, _ in exp]
        if got != want:
            j = next(j for j in range(len(want)) if got[j] != want[j])
            raise AssertionError("rle_inputs=%s: merged record %d: expected value %s, got %s" % (
                rle_inputs, j, want[j][1].hex(), got[j][1].hex()))
        # SAME_KEY in its own run: the key equals the previous record's of the same run (the writer's rule, nonempty keys)
        same_in_run = [j > 0 and segs_recs[s][j - 1][0] == k and rle_inputs for k, _, s, j in exp]
        assert [f for _, _, f in recs] == same_in_run
        written = O.write_ifile([(None if f else k, v) for (k, v), f in zip(want, same_in_run)], rle=False)[0]
        assert seg == written, "rle_inputs=%s: merged IFile differs from the oracle writer's" % rle_inputs


@pytest.mark.parametrize("nseg", [3, 40])
def test_merge_with_same_key_check_flags_equal_neighbours(nseg):
    """checkForSameKeys on, every key at most once per run: the order is still the stable sort, and a record is flagged
    SAME_KEY exactly when its key equals the previous record's (which comes from another run)."""
    rng = random.Random(100 + nseg)
    segs_recs = _merge_segments(rng, nseg, 120, 200, repeats=False)
    segs = [O.write_ifile(r, rle=False)[0] for r in segs_recs]
    exp = _stable_merge_expected(segs_recs, O.CMP_TEXT)
    want = [(k, v) for k, v, _, _ in exp]
    flags = [j > 0 and want[j - 1][0] == k for j, (k, _) in enumerate(want)]
    # the oracle's merge flags the same records (its order of equal keys may differ, its keys do not)
    ref = O.merge(segs, O.CMP_TEXT, factor=100, check_for_same_keys=True)["records"]
    assert [k for k, _, _ in ref] == [k for k, _ in want]
    assert [f for _, _, f in ref] == flags
    recs, _ = _gpu_merge(segs, O.CMP_TEXT, check=True)
    assert [(k, v) for k, v, _ in recs] == want, "merged order differs from the stable sort"
    assert [f for _, _, f in recs] == flags

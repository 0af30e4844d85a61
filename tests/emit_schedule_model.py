"""Shared helpers of the emit-schedule tests (test_emit_schedule_cpu.py, test_emit_schedule_gpu.py): a restatement of
the fixed-width emit's tile schedule, cases built to land on its edges, and the expected file.out of every case.

The source-oriented emit kernels (emit_fast.cuh, emit_pipe.cuh, emit_pipe_u.cuh) and k_emit<true> (sorter_kernels.cuh)
walk tiles of R records.  k_layout gives every partition a segment and its first tile, k_build_tiles gives every tile
its partition, first record, record count, first / last flags, file offset abs0 (its lead is abs0 & 15: the ragged
first chunk) and `after` (segment body bytes behind it).  Persistent groups take tiles g, g + G, g + 2G, ...; the
pipelined kernels park the partial checksums of FE4_PARKED (k_emit_fast4) or FE4_BATCH (k_emit_fast4u) tiles and fold a
batch when it is full or when the group has no next tile.  k_crc_combine folds the tiles of one segment that share a
32-lane warp with one atomic per run.

Given partitions fix every partition's record count, so a case is a list of counts: the builders below turn a target
(tiles per group, a batch position, a lead on a first or a continuation tile, a segment across a warp of the tile
array, ...) into counts, given R (tezgpu_debug_fixed_emit_plan) and the launch's group count G (on the device:
tezgpu_debug_emit_grid).  Every record holds its collection index, so a misplaced, lost or repeated record changes
file.out."""
import zlib

import numpy as np

from oracle import tez_oracle as O

import radix_model as RM

# kernels, numbered as tezgpu_debug_fixed_emit_plan numbers them
PIPE, FAST, PIPE_U, FAST_U, GENERAL = range(5)
PACKED, OFFSETS, RUNS = range(3)
BATCH = {PIPE: 4, PIPE_U: 8}        # FE4_PARKED, FE4_BATCH: parked tiles per checksum fold
WARP = 32                            # k_crc_combine: tiles per warp

# kernel key -> (planned kernel, record layout, framings (klen, vlen)); the first framing carries the tiles-per-group
# axis.  k_emit_fast4u and k_emit_fast<5, false> run on the reduce side only: every map-side entry point hands the emit
# packed, 16-byte aligned records (collect_fixed copies into its own buffer, sort_device_fixed refuses an unaligned
# one, the combiner packs its output), so the merger's run table (layout 2) and its explicit offsets (layout 1, once
# the record iterator has filled them) are the paths that reach them.
KERNELS = {
    "fast4": (PIPE, PACKED, [(16, 64), (8, 8), (16, 16), (16, 112), (0, 128), (128, 0)]),
    "fast5a": (FAST, PACKED, [(16, 128), (16, 496)]),
    "fast4u": (PIPE_U, RUNS, [(16, 64), (16, 16), (16, 128)]),
    "fast5u": (FAST_U, RUNS, [(16, 496), (128, 384)]),
    "general": (GENERAL, PACKED, [(8, 16), (8, 32), (8, 128)]),
}
MAP_SIDE = ("fast4", "fast5a", "general")

TPG_M = [0, 1, 2, 3, 4, 5, 7, 8, 9]
TPG_R = ["0", "1", "G-1"]
SPECIAL_TILES = ["1", "2", "2sms-1", "2sms+1"]


def plan(klen, vlen, layout_):
    """(kernel, records per tile R) the device plans for fixed-width records (tezgpu_debug_fixed_emit_plan)"""
    import ctypes as C
    from tez_b200 import _lib
    k, r = C.c_int32(), C.c_uint32()
    _lib.check(_lib.load().tezgpu_debug_fixed_emit_plan(klen, vlen, layout_, C.byref(k), C.byref(r)))
    return k.value, r.value


def vint_size(v):
    return 1 if v <= 127 else 2 if v < 1 << 8 else 3 if v < 1 << 16 else 4 if v < 1 << 24 else 5


def rec_size(klen, vlen):
    return vint_size(klen) + vint_size(vlen) + klen + vlen


def lead_step(rs):
    """the residues mod 16 a tile can start at are the multiples of this: segment lengths (c * rs + 10), the header
    (4) and whole tiles (R * rs) are all even when rs is"""
    return 2 if rs % 2 == 0 else 1


def leads(rs):
    return list(range(0, 16, lead_step(rs)))


# ------------------------------------------------------------------------------------------------ the restatement
def layout(cnt, rs, send_empty=True, unordered=False):
    """k_layout: (segment starts [P + 1], index int64 [P, 3]) of partitions holding cnt records of rs bytes"""
    cnt = np.asarray(cnt, dtype=np.int64)
    present = cnt > 0
    seg = np.where(present, 4 + cnt * rs + 2 + 4, 0 if (send_empty or unordered) else 10)
    start = np.zeros(len(cnt) + 1, dtype=np.int64)
    start[1:] = np.cumsum(seg)
    index = np.zeros((len(cnt), 3), dtype=np.int64)
    index[:, 0] = np.where(seg > 0, start[:-1], 0) if unordered else start[:-1]
    index[:, 1] = np.where(seg > 0, seg - 4, 0)
    index[:, 2] = seg
    return start, index


def tiles(cnt, R, rs, send_empty=True, unordered=False):
    """k_build_tiles: one row per tile -- dict of arrays p, r0, nr, flags (1 first, 2 last), abs0, lead, after"""
    cnt = np.asarray(cnt, dtype=np.int64)
    start, _ = layout(cnt, rs, send_empty, unordered)
    nt = (cnt + R - 1) // R
    T = int(nt.sum())
    p = np.repeat(np.arange(len(cnt)), nt)
    tile_start = np.concatenate([[0], np.cumsum(nt)])
    k = np.arange(T) - tile_start[p]
    ps = np.concatenate([[0], np.cumsum(cnt)])
    r0 = ps[p] + k * R
    nr = np.minimum(R, ps[p + 1] - r0)
    first, last = k == 0, r0 + nr == ps[p + 1]
    seg0 = start[p]
    abs0 = seg0 + np.where(first, 0, 4 + (r0 - ps[p]) * rs)
    tile_end = seg0 + 4 + (r0 - ps[p] + nr) * rs + np.where(last, 2, 0)
    after = start[p + 1] - 4 - tile_end
    return dict(p=p, r0=r0, nr=nr, flags=first.astype(np.int64) | 2 * last.astype(np.int64), abs0=abs0, lead=abs0 & 15,
                after=after)


def group_tiles(T, G):
    """the tiles of every persistent group: group g takes g, g + G, ... (groups without a tile return at once)"""
    return [list(range(g, T, G)) for g in range(min(G, T))]


def last_batch_positions(T, G, batch):
    """positions (1..batch) in its parked batch of every group's last tile: the size of the batch folded by `!has1`"""
    return {(len(ts) - 1) % batch + 1 for ts in group_tiles(T, G)}


def crosses_warp(tab):
    """a segment whose tiles lie in two warps of the tile array (k_crc_combine's runs meet at lane 31 / lane 0)"""
    p = tab["p"]
    if len(p) == 0:
        return False
    t = np.arange(len(p))
    same = p[1:] == p[:-1]
    return bool((same & (t[1:] % WARP == 0)).any())


# ------------------------------------------------------------------------------------------------ the case builders
def _split_tiles(T, R):
    """counts with T tiles in all: every 8 tiles a partition of 2R + 1 records (two full tiles and one of one record)
    and five of one record; the last T mod 8 tiles in one partition, its last tile half full"""
    cnt = [0]
    for _ in range(T // 8):
        cnt += [2 * R + 1] + [1] * 5
    if T % 8:
        cnt.append((T % 8 - 1) * R + R // 2 + 1)
    return cnt


def _lead_partitions(rs, R, targets, send_empty, size):
    """counts whose partitions of `size` records start at each residue of `targets`: a spacer partition of c records
    (c * rs + 10 bytes), or j spacers of one record, moves the next segment to the residue; with send_empty off an
    empty partition (10 bytes) takes part where it can"""
    cnt, off = [], 0
    for L in targets:
        c = next((c for c in range(1, 64) if (off + c * rs + 10) % 16 == L), None)
        j = next((j for j in range(2, 17) if (off + j * (rs + 10)) % 16 == L), None)
        if c is not None and not send_empty and c > 1 and (off + 10 + (c - 1) * rs + 10) % 16 == L:
            cnt += [0, c - 1]                      # the same residue through an empty segment
            off += 10 + (c - 1) * rs + 10
        elif c is not None:
            cnt.append(c)
            off += c * rs + 10
        elif j is not None:
            cnt += [1] * j
            off += j * (rs + 10)
        else:
            raise AssertionError("residue %d unreachable with %d-byte records" % (L, rs))
        assert off % 16 == L
        cnt.append(size)
        off += size * rs + 10
    return cnt


def build(case, R, grid, sms):
    """partition counts of a case.  grid(T) -> groups of the launch over T tiles; sms: the device's SMs."""
    klen, vlen = case["framing"]
    rs = rec_size(klen, vlen)
    axis, t = case["axis"], case["target"]
    if axis == "tpg":
        m, r = t
        G = grid(1 << 24)                          # the full-wave group count
        T = G * m + {"0": 0, "1": 1, "G-1": G - 1}[r]
        return _split_tiles(T, R)
    if axis == "tiles":
        T = {"1": 1, "2": 2, "2sms-1": 2 * sms - 1, "2sms+1": 2 * sms + 1}[t]
        return _split_tiles(T, R)
    if axis == "cuts":
        sizes = [0, 1, 2, R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1]
        return [0, 0] + sizes[1:4] + [0, 0, 0] + sizes[4:] + [0, 3, 0, 0, R]
    if axis == "warp":
        return [5, 33 * R, 1, 0, R + 2]
    if axis == "p65536":
        return [1] * 65536
    if axis == "leads":
        return _lead_partitions(rs, R, leads(rs), case["send_empty"], R + 3)
    if axis == "maxtile":
        return _lead_partitions(rs, R, [leads(rs)[-1]], case["send_empty"], R) + [1]
    raise ValueError(axis)


def reached(cnt, R, rs, send_empty, grid, batch):
    """what a case reaches: tiles, batch positions of the groups' last tiles, leads on first and continuation tiles,
    a warp crossing, the partition sizes, empty runs, and the first-and-last tiles of R records with their leads"""
    tab = tiles(cnt, R, rs, send_empty)
    T = len(tab["p"])
    G = grid(T) if T else 0
    first = tab["flags"] & 1 == 1
    cnt = list(cnt)
    nonempty = [i for i, c in enumerate(cnt) if c]
    empty_run = any(all(c == 0 for c in cnt[a + 1:b]) and b - a > 2 for a, b in zip(nonempty, nonempty[1:]))
    return dict(T=T, G=G, positions=last_batch_positions(T, G, batch) if (T and batch) else set(),
                first_leads=set(tab["lead"][first].tolist()), cont_leads=set(tab["lead"][~first].tolist()),
                warp=crosses_warp(tab), sizes=set(cnt), empty_run=empty_run,
                full_tile_leads=set(tab["lead"][(tab["flags"] == 3) & (tab["nr"] == R)].tolist()))


def claims(case, R, rs, grid, sms):
    """the classes a case's name claims, checked against reached()"""
    axis, t = case["axis"], case["target"]
    out = {}
    if axis == "tpg":
        m, r = t
        G = grid(1 << 24)
        out["T"] = G * m + {"0": 0, "1": 1, "G-1": G - 1}[r]
    elif axis == "tiles":
        out["T"] = {"1": 1, "2": 2, "2sms-1": 2 * sms - 1, "2sms+1": 2 * sms + 1}[t]
    elif axis == "cuts":
        out["sizes"] = {0, 1, 2, R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1}
        out["empty_run"] = True
    elif axis == "warp":
        out["warp"] = True
        out["sizes"] = {33 * R}
    elif axis == "p65536":
        out["T"] = 65536
    elif axis == "leads":
        out["first_leads"] = out["cont_leads"] = set(leads(rs))
    elif axis == "maxtile":
        out["full_tile_leads"] = {leads(rs)[-1]}
    return out


# ------------------------------------------------------------------------------------------------ the case list
def _case(kernel, framing, axis, target, entry, send_empty=True):
    c = dict(kernel=kernel, framing=framing, axis=axis, target=target, entry=entry, send_empty=send_empty)
    tid = "m%d-r%s" % target if axis == "tpg" else str(target) if target is not None else ""
    c["id"] = "-".join(x for x in (kernel, "%d+%d" % framing, axis, tid, entry, "" if send_empty else "noempty") if x)
    return c


def cases():
    """every case of the GPU file: the tiles-per-group axis on each kernel's first framing; cuts, a segment across a
    warp, every lead and the largest tile on every framing; 2^16 one-record partitions on each kernel; other entry
    points (collect_fixed, unordered handles, the merger's explicit offsets) on a few"""
    out = []
    for k, (_, layout_, framings) in KERNELS.items():
        main = "device" if layout_ == PACKED else "merge"
        f0 = framings[0]
        for m in TPG_M:
            for r in TPG_R:
                out.append(_case(k, f0, "tpg", (m, r), main))
        for t in SPECIAL_TILES:
            out.append(_case(k, f0, "tiles", t, main))
        out.append(_case(k, f0, "p65536", None, main))
        for f in framings:
            for se in (True, False):
                out.append(_case(k, f, "cuts", None, main, se))
                out.append(_case(k, f, "leads", None, main, se))
            out.append(_case(k, f, "warp", None, main))
            out.append(_case(k, f, "maxtile", None, main, False))
        if layout_ == PACKED:
            for axis in ("cuts", "leads", "warp"):
                out.append(_case(k, f0, axis, None, "collect", False))
                out.append(_case(k, f0, axis, None, "unordered"))
        else:
            for axis in ("cuts", "leads", "warp"):
                out.append(_case(k, f0, axis, None, "merge-offsets", False))
    return out


# ------------------------------------------------------------------------------------------------ records and files
def records(n, klen, vlen, seed):
    """(uint8 [n, klen + vlen], sort key uint64 [n] or None): distinct keys in random order -- their first 8 bytes, the
    rest a function of those -- and the collection index, big-endian, in the value's first 4 bytes (in key bytes 8..12
    when the value is shorter).  klen == 0: every key is empty and equal (sort key None)."""
    rng = np.random.default_rng([seed, n, klen, vlen])
    i = np.arange(n, dtype=np.uint64)
    rec = np.empty((n, klen + vlen), dtype=np.uint8)
    with np.errstate(over="ignore"):
        h = i * np.uint64(0x9E3779B97F4A7C15)
    for j in range(min(8, klen + vlen)):       # filler: bytes of a hash of the index, repeated along the record
        rec[:, j] = (h >> np.uint64(8 * j)).astype(np.uint8)
    for j in range(8, klen + vlen, 8):
        rec[:, j:j + 8] = rec[:, :min(8, klen + vlen - j)]
    key = None
    if klen:
        assert klen >= 8
        mul = np.uint64(int(rng.integers(0, 1 << 62)) * 2 + 1)
        base = np.uint64(int(rng.integers(0, 1 << 62)))
        with np.errstate(over="ignore"):
            key = i * mul + base
        rec[:, :8] = key.astype(">u8").view(np.uint8).reshape(-1, 8)
    at = klen if vlen >= 4 else 8
    assert at + 4 <= klen + vlen
    rec[:, at:at + 4] = i.astype(">u4").view(np.uint8).reshape(-1, 4)
    return rec, key


def partition_ids(cnt, seed):
    """partition id of every record, shuffled: partition p holds cnt[p] records"""
    ids = np.repeat(np.arange(len(cnt), dtype=np.int32), np.asarray(cnt, dtype=np.int64))
    np.random.default_rng([seed, len(ids)]).shuffle(ids)
    return ids


def framed(rec, klen, vlen):
    """uint8 [n, rs]: vint(klen) vint(vlen) key value"""
    hdr = np.frombuffer(O.vint(klen) + O.vint(vlen), dtype=np.uint8)
    out = np.empty((rec.shape[0], len(hdr) + rec.shape[1]), dtype=np.uint8)
    out[:, :len(hdr)] = hdr
    out[:, len(hdr):] = rec
    return out


def sorted_order(key, parts, unordered=False):
    """the emit order: by partition, then key (distinct keys; equal empty keys keep collection order); unordered: by
    partition, newest first"""
    if unordered:
        return RM.unordered_order(parts)
    return np.lexsort((key, parts)) if key is not None else np.lexsort((np.arange(len(parts)), parts))


def expected(fr, order, parts, P, send_empty=True, unordered=False):
    """(file.out, index) of the framed records written in `order` (radix_model.spill_file)"""
    rs = fr.shape[1]
    off = np.arange(fr.shape[0] + 1, dtype=np.int64) * rs
    return RM.spill_file(fr.reshape(-1), off, order, parts, P, send_empty, unordered)


def segment(rows):
    """one IFile segment of framed rows uint8 [m, rs]: TIF\\0, the records, EOF marker, CRC-32"""
    body = rows.tobytes() + b"\xff\xff"
    return b"TIF\x00" + body + zlib.crc32(body).to_bytes(4, "big")


def merge_inputs(fr, key, parts, P, runs=2):
    """the reduce side's input: every partition's records dealt round-robin into `runs` sorted runs, one IFile segment
    each; returns (segments, partition of each)"""
    segs, seg_part = [], []
    order = sorted_order(key, parts)
    sp = parts[order]
    bounds = np.searchsorted(sp, np.arange(P + 1))
    for p in range(P):
        mine = order[bounds[p]:bounds[p + 1]]
        for j in range(min(runs, len(mine))):
            segs.append(segment(fr[mine[j::runs]]))
            seg_part.append(p)
    return segs, seg_part


def expected_merge(segs, seg_part, P, send_empty=True):
    """(file.out, index) of the merged partitions: O.merge of every partition's segments, empty partitions as
    k_layout writes them.  A merge into one partition always writes its segment, empty or not (merger.cuh)."""
    send_empty = send_empty and P > 1
    by = [[] for _ in range(P)]
    for s, p in zip(segs, seg_part):
        by[p].append(s)
    pieces, index, off = [], np.zeros((P, 3), dtype=np.int64), 0
    empty = b"TIF\x00\xff\xff" + zlib.crc32(b"\xff\xff").to_bytes(4, "big")
    for p in range(P):
        if not by[p]:
            if send_empty:
                index[p] = (off, 0, 0)
                continue
            seg = empty
        else:
            seg = by[p][0] if len(by[p]) == 1 else O.merge(by[p], O.CMP_BYTES, factor=100)["ifile"]
        index[p] = (off, len(seg) - 4, len(seg))
        pieces.append(seg)
        off += len(seg)
    return np.frombuffer(b"".join(pieces), dtype=np.uint8), index

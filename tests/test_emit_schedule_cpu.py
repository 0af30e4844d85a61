"""CPU: the emit-schedule cases of test_emit_schedule_gpu.py.  The restatement of k_layout / k_build_tiles in
tests/emit_schedule_model.py gives the oracle's segment layout; every case reaches the class its name claims (tiles,
batch positions, leads, a warp crossing, partition sizes) at the group counts of a 132-SM H100 SXM and a 114-SM H100
PCIe; and every kernel meets every value of every axis in some case."""
import numpy as np
import pytest

from oracle import tez_oracle as O

import emit_schedule_model as M

SMS = (132, 114)
RESIDENT = range(1, 9)     # CTAs per SM of the one-group kernels: the device decides, so every plausible count


def grids(kernel, sms):
    """group counts of a launch over T tiles: k_emit_fast4 runs up to one CTA of two groups per SM, the other kernels
    `resident` one-group CTAs per SM"""
    if kernel == M.PIPE:
        return [lambda T: 2 * min(-(-T // 2), sms)]
    return [lambda T, k=k: min(T, sms * k) for k in RESIDENT]


def _R(kernel_key, framing):
    kid, layout_, _ = M.KERNELS[kernel_key]
    k, R = M.plan(*framing, layout_)
    assert k == kid, (kernel_key, framing, k)
    return R


@pytest.mark.parametrize("framing", [(16, 64), (8, 16), (16, 128), (0, 128)])
@pytest.mark.parametrize("send_empty", [True, False])
@pytest.mark.parametrize("unordered", [False, True])
def test_tile_table_is_the_oracles_segment_layout(framing, send_empty, unordered):
    klen, vlen = framing
    rs = M.rec_size(klen, vlen)
    R = 7
    cnt = M.build(dict(framing=framing, axis="cuts", target=None, send_empty=send_empty), R, None, 132)
    cnt += M.build(dict(framing=framing, axis="leads", target=None, send_empty=send_empty), R, None, 132)
    P, n = len(cnt), sum(cnt)
    rec, key = M.records(n, klen, vlen, seed=3)
    parts = M.partition_ids(cnt, seed=3)
    conf = O.sorter_conf(P, partitioner=O.PART_GIVEN, send_empty=send_empty, rle_policy=0)
    r = (O.unordered_write if unordered else O.pipelined_sort)(conf, rec.reshape(-1), np.arange(n, dtype=np.uint64) * (klen + vlen),
                                                               np.full(n, klen, np.uint32), np.full(n, vlen, np.uint32), parts)
    start, index = M.layout(cnt, rs, send_empty, unordered)
    assert np.array_equal(index, r["index"])
    fr = M.framed(rec, klen, vlen)
    out, exp_index = M.expected(fr, M.sorted_order(key, parts, unordered), parts, P, send_empty, unordered)
    assert np.array_equal(exp_index, r["index"])
    if key is not None or unordered:   # the oracle's order of equal (empty) keys is not the stable one the device keeps
        assert out.tobytes() == r["file_out"]
    # the tiles cover every segment's header, records and EOF marker exactly once, in order
    tab = M.tiles(cnt, R, rs, send_empty, unordered)
    at, seg_end = {}, {}
    for t in range(len(tab["p"])):
        p, fl, nr = int(tab["p"][t]), int(tab["flags"][t]), int(tab["nr"][t])
        a = int(tab["abs0"][t])
        assert a == (start[p] if fl & 1 else at[p])
        end = a + (4 if fl & 1 else 0) + nr * rs + (2 if fl & 2 else 0)
        assert int(tab["after"][t]) == start[p + 1] - 4 - end
        at[p] = end
        if fl & 2:
            seg_end[p] = end
    assert seg_end == {p: int(start[p + 1]) - 4 for p in range(P) if cnt[p]}
    assert out[start[:-1][np.asarray(cnt) > 0]].tolist() == [ord("T")] * sum(1 for c in cnt if c)


def test_merge_reference_is_the_sort_reference():
    """expected_merge (O.merge per partition) and the stable reference write the same file for the merge cases"""
    for framing, se in (((16, 64), True), ((16, 128), False)):
        cnt = M.build(dict(framing=framing, axis="cuts", target=None, send_empty=se), 5, None, 132)
        P, n = len(cnt), sum(cnt)
        rec, key = M.records(n, *framing, seed=5)
        parts = M.partition_ids(cnt, seed=5)
        fr = M.framed(rec, *framing)
        segs, seg_part = M.merge_inputs(fr, key, parts, P)
        out, index = M.expected_merge(segs, seg_part, P, se)
        exp_out, exp_index = M.expected(fr, M.sorted_order(key, parts), parts, P, se)
        assert np.array_equal(index, exp_index) and np.array_equal(out, exp_out)


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("case", [c for c in M.cases() if c["axis"] != "p65536"], ids=lambda c: c["id"])
def test_case_reaches_its_class(case, sms):
    kid = M.KERNELS[case["kernel"]][0]
    R = _R(case["kernel"], case["framing"])
    rs = M.rec_size(*case["framing"])
    for grid in grids(kid, sms):
        cnt = M.build(case, R, grid, sms)
        got = M.reached(cnt, R, rs, case["send_empty"], grid, M.BATCH.get(kid, 0))
        for k, v in M.claims(case, R, rs, grid, sms).items():
            if isinstance(v, set):
                assert v <= got[k], (k, sorted(v - got[k]))
            else:
                assert got[k] == v, (k, got[k], v)


def test_p65536_case():
    for k in M.KERNELS:
        cnt = M.build(dict(framing=M.KERNELS[k][2][0], axis="p65536", target=None, send_empty=True), 100, None, 132)
        tab = M.tiles(cnt, 100, 82)
        assert len(cnt) == 65536 and (tab["flags"] == 3).all() and len(tab["p"]) == 65536


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("kernel", list(M.KERNELS))
def test_every_kernel_meets_every_axis_value(kernel, sms):
    kid, layout_, framings = M.KERNELS[kernel]
    mine = [c for c in M.cases() if c["kernel"] == kernel]
    assert {c["target"] for c in mine if c["axis"] == "tpg"} == {(m, r) for m in M.TPG_M for r in M.TPG_R}
    assert {c["target"] for c in mine if c["axis"] == "tiles"} == set(M.SPECIAL_TILES)
    assert any(c["axis"] == "p65536" for c in mine)
    entries = {c["entry"] for c in mine}
    assert entries == ({"device", "collect", "unordered"} if layout_ == M.PACKED else {"merge", "merge-offsets"})
    for f in framings:
        rs = M.rec_size(*f)
        R = _R(kernel, f)
        got = {a: set() for a in ("first_leads", "cont_leads", "full_tile_leads", "sizes")}
        warp = empty_run = False
        for c in mine:
            if c["framing"] != f or c["axis"] not in ("cuts", "leads", "warp", "maxtile"):
                continue
            tab_cnt = M.build(c, R, None, sms)
            tab = M.tiles(tab_cnt, R, rs, c["send_empty"])
            first = tab["flags"] & 1 == 1
            got["first_leads"] |= set(tab["lead"][first].tolist())
            got["cont_leads"] |= set(tab["lead"][~first].tolist())
            got["full_tile_leads"] |= set(tab["lead"][(tab["flags"] == 3) & (tab["nr"] == R)].tolist())
            got["sizes"] |= set(tab_cnt)
            warp |= M.crosses_warp(tab)
            empty_run |= any(x == 0 for x in tab_cnt)
        assert got["first_leads"] == got["cont_leads"] == set(M.leads(rs)), f
        assert max(M.leads(rs)) in got["full_tile_leads"], f
        assert {0, 1, 2, R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1, 33 * R} <= got["sizes"], f
        assert warp and empty_run, f
        if rs % 2:
            assert len(M.leads(rs)) == 16
    # every position of the parked batch meets a group's last tile, at every plausible group count
    if kid in M.BATCH:
        B = M.BATCH[kid]
        R = _R(kernel, framings[0])
        for grid in grids(kid, sms):
            pos = set()
            for c in mine:
                if c["axis"] in ("tpg", "tiles"):
                    pos |= M.reached(M.build(c, R, grid, sms), R, M.rec_size(*framings[0]), True, grid, B)["positions"]
            assert pos == set(range(1, B + 1)), sorted(pos)


def test_odd_leads_reach_every_kernel():
    """a framing of three bytes (a length >= 128) makes record sizes odd, so tiles start at all 16 residues"""
    for k, (_, _, framings) in M.KERNELS.items():
        assert any(M.rec_size(*f) % 2 for f in framings), k

"""The seeded merge scenarios (tests/merge_scenarios.py) and the stable merge model (tests/merge_model.py) against the
CPU oracle, without a GPU: the palettes' comparator order, the model's records, isSameKey flags and IFile against
TezMerger per partition, the sum combiner's two references against each other, and the scenarios' coverage of every
comparator x axis value."""
import functools

import pytest

from oracle import tez_oracle as O

import combine_model as CBM
import merge_scenarios as MS
import sort_order_model as SOM
from merge_model import _canon, model_ifile, stable_model


def _sign(x):
    return (x > 0) - (x < 0)


@pytest.mark.parametrize("cmp", SOM.CMPS, ids=[MS.CMP_NAMES[c] for c in SOM.CMPS])
def test_palette_order_is_the_comparator_order(cmp):
    """for every pair of palette keys, the order of their normalised contents is the sign of the oracle comparator --
    and the palette holds pairs whose raw byte order says the opposite"""
    for pal in (MS.PALETTES[cmp], MS.FIXED_PALETTES.get(cmp)):
        if pal is None:
            continue
        disagree = 0
        for a in pal:
            for b in pal:
                ca, cb = SOM.content(cmp, a), SOM.content(cmp, b)
                want = _sign((ca > cb) - (ca < cb))
                assert _sign(O.compare(cmp, a, b)) == want, (a[:40].hex(), b[:40].hex())
                disagree += want != _sign((a > b) - (a < b))
        assert disagree > 0 or cmp == O.CMP_BYTES, "raw byte order is the comparator order on the whole palette"


def _partition(sc, p):
    return [s for s, q in zip(sc["segs"], sc["parts"]) if q == p]


@pytest.mark.parametrize("seed", MS.SEEDS, ids=MS.scenario_id)
def test_stable_model_against_the_oracle(seed):
    """per partition: the oracle's TezMerger (factor 100, same flags) has the model's keys and isSameKey flags record
    for record, and its IFile equals the model's up to the order of values inside a key group (the heap's tie order);
    with a combiner, the combined oracle merge equals the dict-of-sums model"""
    sc = MS.scenario(seed)
    P, cmp, hdr = sc["P"], sc["cmp"], sc["has_header"]
    model = stable_model(sc["segs"], sc["parts"], P, cmp, hdr, sc["check"])
    assert sum(len(m) for m in model) == sc["nrec"]
    for p in range(P):
        mine = _partition(sc, p)
        if not mine:
            assert not model[p]
            continue
        exp = O.merge(mine, cmp, factor=100, check_for_same_keys=sc["check"], writer_rle=sc["writer_rle"], has_header=hdr)
        assert [(k, s) for k, _, s in exp["records"]] == [(k, s) for k, _, s in model[p]], "partition %d" % p
        assert sorted(v for _, v, _ in exp["records"]) == sorted(v for _, v, _ in model[p]), "partition %d" % p
        mine_ifile = model_ifile(model[p], sc["writer_rle"])
        assert len(mine_ifile) == len(exp["ifile"]), "partition %d" % p
        assert _canon(O.read_ifile(mine_ifile)) == _canon(O.read_ifile(exp["ifile"])), "partition %d" % p
        if sc["combiner"]:
            got = CBM.merge_combine(mine, cmp, sc["combiner"], has_header=hdr)[0]
            want = CBM.model([(k, v) for k, v, _ in model[p]], [0] * len(model[p]), cmp, sc["combiner"], 1)[0]
            assert got == O.write_ifile(want)[0], "partition %d: combined merge" % p


@functools.lru_cache(maxsize=None)
def _facts(seed):
    """the data-dependent axis values of one scenario"""
    sc = MS.scenario(seed)
    per_part = [len(_partition(sc, p)) for p in range(sc["P"])]
    recs = [O.read_ifile(s, has_header=sc["has_header"]) for s in sc["segs"]]
    return dict(empty_partition=0 in per_part, eof_only=any(not r for r in recs), max_segs=max(per_part),
                encoded=sc["encoded"], long_record=any(len(v) > MS.WINDOW for r in recs for _, _, v in r),
                plain_repeat=any(a[1] == b[1] and b[0] == O.NEW_KEY for r in recs for a, b in zip(r, r[1:])),
                nrec=sc["nrec"], interleaved=sc["parts"] != sorted(sc["parts"]))


def test_scenarios_cover_every_comparator_and_axis_value():
    """every comparator meets every value of every axis somewhere among the seeds (fixed framing: the comparators
    with fixed-width keys); large scenarios hold LARGE_RECORDS records or more"""
    seen = {}
    for seed in MS.SEEDS:
        s, f = MS.shape(seed), _facts(seed)
        assert f["nrec"] >= MS.LARGE_RECORDS if s["large"] else f["nrec"] < MS.LARGE_RECORDS // 4, seed
        axes = dict(P=s["P"], fixed=s["fixed"], check=s["check"], writer_rle=s["writer_rle"], header=s["has_header"],
                    combiner=s["combiner"], large=s["large"], encoded=f["encoded"], long_record=f["long_record"],
                    plain_repeat=f["plain_repeat"], eof_only=f["eof_only"], many_segments=f["max_segs"] >= 20,
                    fixed_encoded=(f["encoded"] if s["fixed"] else None), fixed_P1=(s["P"] == 1 if s["fixed"] else None),
                    large_P=(s["P"] if s["large"] else None), large_fixed=(s["fixed"] if s["large"] else None),
                    large_combiner=(bool(s["combiner"]) if s["large"] else None))
        if s["P"] > 1:
            axes.update(empty_partition=f["empty_partition"], interleaved=f["interleaved"])
        for axis, value in axes.items():
            seen.setdefault((s["cmp"], axis), set()).add(value)
    want = dict(P=set(MS.PS), fixed={False, True}, check={False, True}, writer_rle={False, True}, header={False, True},
                combiner={0, MS.SUM_INT, MS.SUM_LONG}, large={False, True}, encoded={False, True},
                long_record={False, True}, plain_repeat={False, True}, eof_only={False, True},
                many_segments={False, True}, fixed_encoded={None, False, True}, fixed_P1={None, False, True},
                large_P={None} | set(MS.PS[1:]), large_fixed={None, False, True}, large_combiner={None, False, True},
                empty_partition={True}, interleaved={True})
    missing = []
    for cmp in SOM.CMPS:
        want_cmp = want if cmp in MS.FIXED_KLEN else dict(want, fixed={False}, fixed_encoded={None}, fixed_P1={None},
                                                          large_fixed={None, False})
        for axis, values in want_cmp.items():
            lost = values - seen.get((cmp, axis), set())
            if lost:
                missing.append("%s %s: %s" % (MS.CMP_NAMES[cmp], axis, sorted(lost, key=repr)))
    assert not missing, "\n".join(missing)

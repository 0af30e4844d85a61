"""GPU: every route of the reduce-side merge over the seeded scenarios of tests/merge_scenarios.py -- all five
comparators, P = 1 / 2 / 7 / 64 with empty partitions and EOF-only segments, fixed and variable framing,
checkForSameKeys and the writer's RLE on and off, header-less segments, sum combiners, and merges larger than one
step of the bounded merge's 16 MiB floor.

(a) host segments: checked against the oracle's TezMerger and the stable merge model (records, isSameKey flags, the
    written IFile of every partition, counts), the record iterator at two batch shapes;
(b) fixed framing (run table, parse_info mode 0, or mode 1 when an input is run-length encoded);
(c) the segments in device memory, read in place;
(d) the bounded merge in key-range steps at the one-step, floor and about a third of the one-step budgets;
(e) with a combiner, (a), (c) and (d) against the oracle's merge-then-combine per partition;
(f) the sequential walker (TEZGPU_PARSE_SERIAL=1, in a subprocess) over every variable-framing scenario.
Each route must give (a)'s bytes, index, counts and records.

Run as a script (`python tests/test_merge_routes_gpu.py serial-walker`, with TEZGPU_PARSE_SERIAL=1) it prints the
digests of route (a) of every variable-framing scenario."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import tez_b200 as T  # noqa: E402

import combine_model as CBM  # noqa: E402
import merge_scenarios as MS  # noqa: E402
from merge_model import check_oracle, partition_segments, place, run  # noqa: E402

pytestmark = pytest.mark.gpu

FLOOR = 16 << 20      # TEZGPU_MERGE_BUDGET_MIN
ITER_SHAPES = ((1 << 14, 1 << 22), (997, 1 << 16))   # run()'s batch shape first


def _run(sc, segs=None, **kw):
    return run(sc["segs"] if segs is None else segs, P=sc["P"], parts=sc["parts"], check=sc["check"],
               writer_rle=sc["writer_rle"], comparator=sc["cmp"], has_header=sc["has_header"], **kw)


def _records(sc, shape):
    with T.GpuMerger(sc["segs"], comparator=sc["cmp"], has_header=sc["has_header"], partitions=sc["parts"],
                     num_partitions=sc["P"]) as m:
        if not sc["check"]:
            m.set_check_for_same_keys(False)
        return list(m.records(batch_records=shape[0], batch_bytes=shape[1]))


def _bounded(sc, budget, tmp, combiner=T.COMBINE_NONE):
    """(records or None, file bytes, index or None, counts, bounded_info) of one bounded merger"""
    with T.GpuMerger(sc["segs"], comparator=sc["cmp"], has_header=sc["has_header"], partitions=sc["parts"],
                     num_partitions=sc["P"], fixed=sc["fixed"], device_budget=budget) as m:
        if not sc["check"]:
            m.set_check_for_same_keys(False)
        if combiner:
            m.set_combiner(combiner)
        recs = None if combiner else list(m.records(batch_records=ITER_SHAPES[1][0], batch_bytes=ITER_SHAPES[1][1]))
        if sc["P"] == 1:
            seg, raw, part, _ = m.write_ifile(rle=sc["writer_rle"])
            assert part == len(seg) == raw + 4
            out, index = seg, None
        else:
            f, fi = os.path.join(tmp, "file.out"), os.path.join(tmp, "file.out.index")
            index, _ = m.write_partitions(f, fi, rle=sc["writer_rle"])
            with open(f, "rb") as fh:
                out = fh.read()
            index = index.tolist()
        return recs, out, index, m.counts(), m.bounded_info()


def _budgets(sc, tmp, combiner=T.COMBINE_NONE):
    """the bounded merge at the one-step budget, at the floor and at about a third of the one-step need (as
    test_merge_bounded_gpu's _check_budgets picks them): [(budget, result)]"""
    one = _bounded(sc, 0, tmp, combiner)
    assert one[4][0] == 1, "the one-step budget took %d steps" % one[4][0]
    need = one[4][1]
    res = [(0, one)]
    for b in sorted({max(FLOOR, need // 3), FLOOR}, reverse=True):
        got = _bounded(sc, b, tmp, combiner)
        steps, peak, _ = got[4]
        assert peak <= b, "budget %d: peak %d device bytes" % (b, peak)
        if sc["large"]:
            assert steps > 1, "budget %d: one step for a large merge (need %d)" % (b, need)
        res.append((b, got))
    return res


def _digest(out):
    out = dict(out)
    out.pop("mode")
    return hashlib.sha256(repr(sorted(out.items())).encode()).hexdigest()


_DIGESTS = {}   # seed -> digest of route (a), from test_merge_routes


@pytest.mark.parametrize("seed", MS.SEEDS, ids=MS.scenario_id)
def test_merge_routes(seed, tmp_path):
    sc = MS.scenario(seed)
    P, fixed = sc["P"], sc["fixed"]

    # (a) host segments, window parser: the oracle and the stable merge model
    host = _run(sc)
    assert host["mode"] == 1, "(a) host merge took mode %d" % host["mode"]
    check_oracle(host, sc["segs"], sc["parts"], P, sc["cmp"], sc["check"], sc["writer_rle"], sc["has_header"])
    assert _records(sc, ITER_SHAPES[1]) == host["records"], "(a) records at %d records / %d bytes per batch" % ITER_SHAPES[1]
    if not fixed:
        _DIGESTS[seed] = _digest(host)

    # (b) fixed framing: the run table unless an input holds a REPEAT_KEY record
    if fixed:
        got = _run(sc, fixed=fixed)
        assert got.pop("mode") == (1 if sc["encoded"] else 0), "(b) fixed framing took the wrong record finder"
        for key in got:
            assert got[key] == host[key], "(b) fixed framing: %s differs from (a)" % key

    # (c) device-resident segments read in place
    ptrs, keep = place(sc["segs"], "residues", "body", seed=seed)
    dev = _run(sc, ptrs, device_ptrs=True)
    del keep
    for key in host:
        assert dev[key] == host[key], "(c) device-resident: %s differs from (a)" % key

    # (d) bounded merge in key-range steps
    for b, (recs, out, index, counts, _) in _budgets(sc, str(tmp_path)):
        assert recs == host["records"], "(d) budget %d: records differ from (a)" % b
        assert out == (host["ifile"] if P == 1 else host["file"]), "(d) budget %d: written bytes differ from (a)" % b
        assert index is None or index == host["index"], "(d) budget %d: index differs from (a)" % b
        assert counts == host["counts"], "(d) budget %d: counts differ from (a)" % b

    # (e) the combiner on (a), (c) and (d)
    if sc["combiner"]:
        want = []
        for p, (_, _, n) in enumerate(host["index"]):   # a partition without records writes no segment (P > 1)
            mine = [s for s, q in zip(sc["segs"], sc["parts"]) if q == p]
            want.append(CBM.merge_combine(mine, sc["cmp"], sc["combiner"], has_header=sc["has_header"])[0]
                        if n or P == 1 else b"")
        comb = _run(sc, combiner=sc["combiner"])
        assert partition_segments(comb) == want, "(e) host segments with the combiner"
        ptrs, keep = place(sc["segs"], "residues", "body", seed=seed)
        comb_dev = _run(sc, ptrs, device_ptrs=True, combiner=sc["combiner"])
        del keep
        assert comb_dev == comb, "(e) device-resident segments with the combiner"
        for b, (_, out, index, _, _) in _budgets(sc, str(tmp_path), sc["combiner"]):
            assert out == (comb["ifile"] if P == 1 else comb["file"]), "(e) bounded budget %d with the combiner" % b
            assert index is None or index == comb["index"], "(e) bounded budget %d: index" % b


def _variable_seeds():
    return [s for s in MS.SEEDS if not MS.shape(s)["fixed"]]


def walker_digests(mode):
    """digest of route (a) of every variable-framing scenario; asserts the record finder's mode"""
    out = {}
    for seed in _variable_seeds():
        got = _run(MS.scenario(seed))
        assert got["mode"] == mode, (seed, got["mode"])
        out[str(seed)] = _digest(got)
    return out


def test_sequential_walker_equals_the_window_parser():
    """(f) TEZGPU_PARSE_SERIAL=1 sends every merge to the sequential walker (mode 2); the switch is read once per
    process, so a subprocess merges every variable-framing scenario and prints the digests of route (a)"""
    env = dict(os.environ, TEZGPU_PARSE_SERIAL="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "serial-walker"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    serial = json.loads(r.stdout.strip().splitlines()[-1])
    assert sorted(serial) == sorted(str(s) for s in _variable_seeds())
    for seed in _variable_seeds():
        if seed not in _DIGESTS:
            got = _run(MS.scenario(seed))
            assert got["mode"] == 1
            _DIGESTS[seed] = _digest(got)
        assert serial[str(seed)] == _DIGESTS[seed], "%s: the sequential walker's merge differs" % MS.scenario_id(seed)


if __name__ == "__main__":
    if sys.argv[1:] == ["serial-walker"]:
        print(json.dumps(walker_digests(2)))

"""The host reference of the map-side radix sort tests (tests/radix_model.py) against the CPU oracle, without a GPU: for
every digit shape and every partition width the GPU tests use, the reference's file.out and index equal the oracle's
byte for byte; the shape generator is deterministic; the cases cover every subset of constant passes, both key widths
and both handles."""
import numpy as np
import pytest

from oracle import tez_oracle as O

import radix_model as RM

N_SHAPE = 2 * RM.TILE + 5
N_WIDTH = 600


def _ties_in_collection_order(rec, width, cmp, parts, out):
    """every run of equal (partition, key) in the reference's order lists its records by ascending index"""
    order = RM.stable_order(RM.normalised(rec[:, :width], cmp), parts)
    norm = RM.normalised(rec[order, :width], cmp)
    tie = (norm[1:] == norm[:-1]) & (np.asarray(parts)[order][1:] == np.asarray(parts)[order][:-1])
    assert (order[1:][tie] > order[:-1][tie]).all()


@pytest.mark.parametrize("cmp", [O.CMP_BYTES, O.CMP_INT], ids=["bytes", "int"])
@pytest.mark.parametrize("shape", RM.SHAPES)
def test_shape_reference_is_the_oracle_4byte(shape, cmp):
    """tie-blind values (a function of the key) make the oracle's order of equal keys unobservable: the bytes must
    agree exactly; with index values the reference orders ties by index"""
    norm = RM.shape_keys(shape, N_SHAPE, seed=1)
    rec = RM.fixed_records(norm, 4, cmp, values=RM.key_hash_values(norm, 4))
    parts = np.zeros(N_SHAPE, dtype=np.int64)
    out, index = RM.reference_fixed(rec, cmp, 1, parts)
    exp_out, exp_index = RM.oracle_run(rec, cmp, 1)
    assert out.tobytes() == exp_out
    assert np.array_equal(index, exp_index)
    _ties_in_collection_order(RM.fixed_records(norm, 4, cmp), 4, cmp, parts, out)


@pytest.mark.parametrize("low", RM.LOW_SHAPES)
@pytest.mark.parametrize("shape", RM.SHAPES)
def test_shape_reference_is_the_oracle_8byte(shape, low):
    cmp = O.CMP_LONG if RM.SHAPES.index(shape) % 2 else O.CMP_BYTES
    norm = RM.shape_keys64(shape, low, N_SHAPE, seed=2)
    rec = RM.fixed_records(norm, 8, cmp, values=RM.key_hash_values(norm, 8))
    out, index = RM.reference_fixed(rec, cmp, 1, np.zeros(N_SHAPE, dtype=np.int64))
    exp_out, exp_index = RM.oracle_run(rec, cmp, 1)
    assert out.tobytes() == exp_out
    assert np.array_equal(index, exp_index)


@pytest.mark.parametrize("case", RM.width_cases(), ids=RM.case_id)
def test_width_reference_is_the_oracle(case):
    """index values and distinct keys: the stable order is the oracle's order"""
    data, parts, given = RM.width_case_data(case, N_WIDTH, seed=case["P"])
    P, cmp = case["P"], case["cmp"]
    if isinstance(data, np.ndarray):
        out, index = RM.reference_fixed(data, cmp, P, parts, case["send_empty"], case["unordered"])
    else:
        out, index = RM.reference_var(data, cmp, P, parts, None, case["send_empty"], case["unordered"])
    exp_out, exp_index = RM.oracle_run(data, cmp, P, given, case["send_empty"], case["unordered"])
    assert np.array_equal(index, exp_index)
    assert out.tobytes() == exp_out


def test_both_spill_builders_agree():
    """the segment-by-segment builder (few partitions) and the vectorised one (many) write the same file"""
    for P, send_empty, unordered in ((7, True, False), (7, False, False), (3000, False, False), (3000, True, True)):
        rec = RM.fixed_records(RM.distinct_keys(2000, 4, 5), 4, O.CMP_BYTES)
        parts = RM.given_partitions(2000, P, 5)
        framed, off = RM.framed_fixed(rec)
        order = RM.stable_order(RM.normalised(rec[:, :4], O.CMP_BYTES), parts)
        a = RM._spill_file_loop(framed, off, order, parts, P, send_empty, unordered)
        big = P + 5000      # the same partitions among more, empty ones
        b = RM.spill_file(framed, off, order, parts, big, send_empty, unordered)
        assert np.array_equal(a[1], b[1][:P])
        assert a[0].tobytes() == b[0][:a[0].size].tobytes()


def test_shapes_are_deterministic_per_seed():
    for shape in RM.SHAPES:
        for n in (1, 6145):
            a, b = RM.shape_keys(shape, n, 3), RM.shape_keys(shape, n, 3)
            assert np.array_equal(a, b), shape
        for low in RM.LOW_SHAPES:
            assert np.array_equal(RM.shape_keys64(shape, low, 999, 3), RM.shape_keys64(shape, low, 999, 3))
    for shape in ("uniform", "zipf", "descending", "const5"):
        assert not np.array_equal(RM.shape_keys(shape, 6145, 3), RM.shape_keys(shape, 6145, 4)), shape
    assert RM.words(500, 1) == RM.words(500, 1) and len(set(RM.words(500, 1))) == 500
    assert np.array_equal(RM.given_partitions(500, 9, 1), RM.given_partitions(500, 9, 1))


def test_shapes_have_their_digits():
    """each shape is what its name says, pass by pass"""
    n = 3 * RM.TILE + 7

    def digits(k, b):
        return (k >> np.uint32(8 * b)) & np.uint32(0xFF)

    for m in range(16):
        k = RM.shape_keys("const%x" % m, n, 1)
        for b in range(4):
            distinct = np.unique(digits(k, b)).size
            assert (distinct == 1) == bool((m >> b) & 1), ("const%x" % m, b, distinct)
    assert (RM.shape_keys("zeros", n, 1) == 0).all() and (RM.shape_keys("ones", n, 1) == 0xFFFFFFFF).all()
    alt = RM.shape_keys("alternating", n, 1)
    assert np.unique(alt).size == 2 and all(np.unique(digits(alt, b)).size == 2 for b in range(4))
    asc = RM.shape_keys("ascending", n, 1)
    assert (np.diff(asc.astype(np.int64)) >= 0).all()
    assert (np.diff(RM.shape_keys("descending", n, 1).astype(np.int64)) <= 0).all()
    for shape, slot in (("outlier_first", 0), ("outlier_last", RM.TILE - 1)):
        k = RM.shape_keys(shape, n, 1)
        odd = np.nonzero(k != 0x80808080)[0]
        exp = [t * RM.TILE + slot for t in range(4) if t * RM.TILE + slot < n]
        if shape == "outlier_last":
            exp.append(n - 1)
        assert list(odd) == exp, shape
        assert all((digits(k[odd], b) != 0x80).all() for b in range(4))
    ff = RM.shape_keys("ff_last", n, 1)
    assert ff[-1] == 0xFFFFFFFF and all((digits(ff[:-1], b) != 0xFF).all() for b in range(4))
    lo = RM.shape_keys64("constf", "outlier", n, 1) & np.uint64(0xFFFFFFFF)
    assert np.unique(lo[:-1]).size == 1 and lo[-1] < lo[0]


def test_width_cases_cover_every_combination_axis():
    cases = RM.width_cases()
    pbits = lambda P: (P - 1).bit_length()   # noqa: E731
    assert sorted({pbits(c["P"]) for c in cases}) == list(range(1, 26))
    assert {c["P"] for c in cases} == {v for k in range(1, 25) for v in ((1 << k), (1 << k) + 1)}
    for u in (False, True):
        sub = [c for c in cases if c["unordered"] == u]
        assert {c["kind"] for c in sub} == set(RM.KINDS)
        assert {c["hashed"] for c in sub} == {True, False}
        assert {c["send_empty"] for c in sub} == {True, False}
        for kind in RM.KINDS:   # every key kind at low pbits and at pbits >= 17 (alphabet depth 1 or 0)
            ks = [pbits(c["P"]) for c in sub if c["kind"] == kind]
            assert min(ks) <= 8 and max(ks) >= 17, (u, kind, ks)
    # the alphabet table's covered depth reaches 0 (pbits 25) for a variable-width key on an ordered handle
    assert any(pbits(c["P"]) == 25 and c["kind"] in ("text", "bytes") and not c["unordered"] for c in cases)

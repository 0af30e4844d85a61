"""CPU: the 32-bit sort word of the variable-width map side and of the merger (SymTable alphabet packing or the raw
prefix, sorter_kernels.cuh stage_sort_word), run on the host with the device's code (tezgpu_debug_sort_words_emulate)
and checked against the oracle comparator: a smaller word must mean a smaller (partition, key), and equal words must
mean equal partitions and equal content on the bytes the word covers, which the tie refinement then skips."""
import random

import numpy as np
import pytest

from oracle import tez_oracle as O
from tez_b200 import _lib
import sort_order_model as M

ALPHABET_SIZES = [1, 2, 3, 4, 7, 8, 15, 16, 31, 32, 127, 128, 255, 256]
POSITIONS = [0, 1, 5, 15]
PARTITIONS = [1, 2, 64, 1000, 1024, 65537]     # (32 - pbits) = 32, 31, 26, 22, 22, 15 bits of key field


def _run_case(rng, cmp, c, q, P, other):
    contents = M.alphabet_contents(rng, cmp, c, q, other=other)
    keys = [M.make_key(cmp, x) for x in contents]
    words, npos, used = M.sort_words(keys, cmp, P)
    exp_npos, exp_used, depth0 = M.table_layout(contents, P)
    case = "cmp=%d c=%d q=%d P=%d other=%s" % (cmp, c, q, P, other)
    assert (npos, used) == (exp_npos, exp_used), case
    M.check_words(keys, cmp, P, words, depth0, used)
    return npos, used


@pytest.mark.parametrize("c", ALPHABET_SIZES)
@pytest.mark.parametrize("cmp", M.CMPS)
def test_alphabet_table_words_order_keys(cmp, c):
    """c byte values at content position q, the other positions from tiny alphabets: the table is used wherever keys
    are longer than the raw prefix, and packs position q itself whenever its bits fit.  c = 256 needs 9-bit ranks: a rank stored in a byte
    wraps 256 to 0 ("key ended") and sends every key with byte 0xFF at q in front of all others."""
    rng = random.Random(1000 * cmp + c)
    packed_q = 0
    for q in POSITIONS:
        if q >= M.FIXED_LEN.get(cmp, 1 << 30):
            continue
        for P in PARTITIONS:
            npos, used = _run_case(rng, cmp, c, q, P, "small")
            # (IntWritable keys have four bytes: with P = 1 the raw prefix already holds all of them)
            if M.FIXED_LEN.get(cmp, M.SYM_MAX_POS) > (32 - M.pbits_of(P)) // 8:
                assert used, "cmp=%d c=%d q=%d P=%d: the table is not used" % (cmp, c, q, P)
            packed_q += npos > q
    assert packed_q > 0, "no case packs the position under test"


@pytest.mark.parametrize("P", PARTITIONS)
@pytest.mark.parametrize("cmp", M.CMPS)
def test_raw_prefix_words_order_keys(cmp, P):
    """Arbitrary bytes everywhere: the table would pack no more positions than the raw prefix, so the sort word is the
    first (32 - pbits) / 8 normalised bytes (with zero padding after a key's end)."""
    rng = random.Random(7 * cmp + P)
    for c in (128, 256):
        for q in (0, 1):
            _, used = _run_case(rng, cmp, c, q, P, "wide")
            assert not used, "cmp=%d c=%d q=%d P=%d: the table is used" % (cmp, c, q, P)


@pytest.mark.parametrize("cmp", M.CMPS)
def test_table_switched_off_gives_raw_prefix(cmp):
    """use_sym = 0 (the TEZGPU_NO_SYM=1 switch) takes the raw prefix even where the table would pay."""
    rng = random.Random(cmp)
    contents = M.alphabet_contents(rng, cmp, 256, 0)
    keys = [M.make_key(cmp, x) for x in contents]
    for P in PARTITIONS:
        words, npos, used = M.sort_words(keys, cmp, P, use_sym=False)
        assert not used and npos == M.table_layout(contents, P)[0]
        M.check_words(keys, cmp, P, words, (32 - M.pbits_of(P)) // 8, False)


def test_saturated_first_byte_with_binary_tail():
    """One arbitrary byte followed by six letters from {a, b}, one partition: seven positions packed into 9 + 6 * 2 bits;
    the keys that start with 0xFF must sort last, not first."""
    rng = random.Random(1)
    keys = [bytes([b]) + bytes(rng.choice(b"ab") for _ in range(6)) for b in range(256) for _ in range(3)]
    words, npos, used = M.sort_words(keys, O.CMP_BYTES, 1)
    assert (npos, used) == (7, True)
    order = np.argsort(words, kind="stable")
    assert [keys[i][0] for i in order[:3]] == [0, 0, 0]
    assert [keys[i][0] for i in order[-3:]] == [0xFF, 0xFF, 0xFF]
    M.check_words(keys, O.CMP_BYTES, 1, words, 7, True)


def test_given_partitions_lead_the_word():
    """Given partition ids occupy the top pbits whatever the key; the key field keeps its order inside a partition."""
    rng = random.Random(5)
    contents = M.alphabet_contents(rng, O.CMP_TEXT, 256, 1)
    keys = [M.make_key(O.CMP_TEXT, x) for x in contents]
    for P in (2, 1000, 65537):
        part = [rng.randrange(P) for _ in keys]
        words, npos, used = M.sort_words(keys, O.CMP_TEXT, P, partition=part)
        assert used
        pb = M.pbits_of(P)
        assert np.array_equal(words >> np.uint32(32 - pb), np.array(part, dtype=np.uint32))
        M.check_words(keys, O.CMP_TEXT, P, words, npos, True, partition=part)


def test_illegal_given_partition_is_an_error():
    with pytest.raises(_lib.TezGpuError):
        M.sort_words([b"a", b"b"], O.CMP_BYTES, 4, partition=[0, 4])


@pytest.mark.parametrize("cmp", M.CMPS)
def test_normalised_content_order_equals_oracle_comparator(cmp):
    """The Python sort key of these tests (normalised content bytes) agrees with the oracle comparator."""
    rng = random.Random(11 + cmp)
    contents = M.alphabet_contents(rng, cmp, 7, 1) + M.alphabet_contents(rng, cmp, 256, 0, other="wide")
    keys = [M.make_key(cmp, x) for x in contents]
    assert all(M.content(cmp, k) == x for k, x in zip(keys, contents))
    for _ in range(3000):
        a, b = rng.choice(keys), rng.choice(keys)
        ca, cb = M.content(cmp, a), M.content(cmp, b)
        exp = (ca > cb) - (ca < cb)
        got = O.compare(cmp, a, b)
        assert (got > 0) - (got < 0) == exp, (a.hex(), b.hex())

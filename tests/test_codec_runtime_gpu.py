"""GPU: DefaultCodec through the plugin classes (tez.runtime.compress=true, tez.runtime.compress.codec=DefaultCodec):
compressed spills, a final merge that reads them and writes a compressed file.out, the pipelined shuffle and the
OrderedWordCount known answer read back through the input."""
import random
import zlib

import numpy as np
import pytest

from oracle import tez_oracle as O
from tez_b200.runtime_library import (BYTES_WRITABLE, INT_WRITABLE, TEXT, TEZ_BYTES_COMPARATOR, InputContext, LocalOutput,
                                      OrderedGroupedKVInput)
from test_codec_gpu import check_file
from test_runtime_library_gpu import _consume, _run_output

pytestmark = pytest.mark.gpu
ZCONF = {"tez.runtime.compress": True, "tez.runtime.compress.codec": "org.apache.hadoop.io.compress.DefaultCodec"}


def _index(path, P):
    return np.frombuffer(open(path, "rb").read()[:-8], dtype=">i8").reshape(P, 3)


@pytest.mark.parametrize("n,spills", [(5000, 1), (20000, 2), (60000, 3)])
def test_output_spills_and_final_merge_compressed(tmp_path, n, spills):
    """Unique keys: the final file.out is the single sort's, every segment compressed."""
    P = 8
    kv = O.gen_c2(0, n, seed=n)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = dict(ZCONF, **{"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
                          "tez.runtime.io.sort.mb": 1})
    out, events = _run_output(tmp_path, conf, recs, P)
    assert out.num_spills >= spills if spills == 3 else out.num_spills == spills
    exp = O.pipelined_sort_fixed(O.sorter_conf(P), kv, 16, 64)
    got = open(out.final_output_file, "rb").read()
    idx = _index(out.final_index_file, P)
    check_file(got, idx, exp["file_out"], exp["index"])
    assert out.counter("OUTPUT_BYTES_PHYSICAL") == len(got)
    assert out.counter("OUTPUT_BYTES_WITH_OVERHEAD") == int(exp["index"][:, 1].sum())
    assert out.counter("OUTPUT_RECORDS") == n
    assert out.counter("SPILLED_RECORDS") == (n if out.num_spills == 1 else 2 * n)


def test_pipelined_shuffle_compressed_spills_reach_the_input(tmp_path):
    n, P = 40000, 4
    kv = O.gen_c2(0, n, seed=23)
    recs = [(bytes(r[:16]), bytes(r[16:])) for r in kv.reshape(n, 80)]
    conf = dict(ZCONF, **{"tez.runtime.key.class": BYTES_WRITABLE, "tez.runtime.key.comparator.class": TEZ_BYTES_COMPARATOR,
                          "tez.runtime.io.sort.mb": 1, "tez.runtime.enable.final-merge.in.output": False})
    out, events = _run_output(tmp_path, conf, recs, P)
    S = out.num_spills
    assert S >= 3
    uid = out.context.unique_identifier
    files = [str(tmp_path / "output" / ("%s_%d" % (uid, s)) / "file.out") for s in range(S)]
    for f in files:
        data, idx = open(f, "rb").read(), _index(f + ".index", P)
        for s0, raw, part in idx:
            if part:
                seg = data[s0:s0 + part]
                assert seg[:4] == b"TIF\x01" and len(zlib.decompress(seg[4:-4])) == raw - 4
    p = 2
    inp = OrderedGroupedKVInput(InputContext(conf, str(tmp_path / "r")), 1)
    inp.initialize()
    inp.start()
    inp.handleEvents([LocalOutput(0, files[s], files[s] + ".index", p, spill_id=s, last_event=(s == S - 1)) for s in range(S)])
    r = inp.getReader()
    got = []
    while r.next():
        got.append((r.getCurrentKey(), list(r.getCurrentValues())))
    mine = sorted((k, v) for k, v in recs if O.partition_of(O.CMP_BYTES, k, P) == p)
    assert [(k, vs[0]) for k, vs in got] == mine
    # random records: stored chunks, a few bytes of framing per 32 KiB chunk over the raw length
    assert 0 < inp.counter("SHUFFLE_BYTES") <= 1.001 * inp.counter("SHUFFLE_BYTES_DECOMPRESSED") + 32 * S


def test_ordered_word_count_known_answer_compressed(tmp_path):
    """TestTezJobs.testOrderedWordCount's answer with both edges compressed; the compressible word stream shuffles
    fewer bytes than it decompresses to."""
    words = []
    for i in range(1, 11):
        words += ["a_%d" % i] * (22 - 2 * i) * 50
    random.Random(3).shuffle(words)
    P = 4
    conf1 = dict(ZCONF, **{"tez.runtime.key.class": TEXT, "tez.runtime.value.class": INT_WRITABLE})
    producers = [_run_output(tmp_path / ("t%d" % t), conf1, [(O.text(w), O.int_writable(1)) for w in words[t::3]], P,
                             uid="attempt_1_0001_1_00_%06d_0_10001" % t) for t in range(3)]
    for prod, _ in producers:
        assert open(prod.final_output_file, "rb").read(4) in (b"TIF\x01", b"")
    counts = {}
    shuffled = decompressed = 0
    for p in range(P):
        inp, groups = _consume(tmp_path / ("s%d" % p), conf1, producers, p, P)
        for k, vals in groups:
            counts[k[1:].decode()] = sum(int.from_bytes(v, "big") for v in vals)
        shuffled += inp.counter("SHUFFLE_BYTES")
        decompressed += inp.counter("SHUFFLE_BYTES_DECOMPRESSED")
    assert counts == {"a_%d" % i: (22 - 2 * i) * 50 for i in range(1, 11)}
    assert 0 < shuffled < decompressed
    conf2 = dict(ZCONF, **{"tez.runtime.key.class": INT_WRITABLE, "tez.runtime.value.class": TEXT})
    prod2 = [_run_output(tmp_path / "sum", conf2, [(O.int_writable(c), O.text(w)) for w, c in counts.items()], 1,
                         uid="attempt_1_0001_1_01_000000_0_10001")]
    _, groups = _consume(tmp_path / "sorter", conf2, prod2, 0, 1)
    final = [(int.from_bytes(k, "big", signed=True), v[0][1:].decode()) for k, v in groups]
    assert final == [((22 - 2 * i) * 50, "a_%d" % i) for i in range(10, 0, -1)]

"""The crafted streams of the codec lane tests, checked without a GPU: every case decodes to its intended body through
the reference library (zlib, liblz4, libzstd) and through the one-lane emulation of the device decoders, has the
structure its name says (parsed back from the stream), and is generated the same way every time."""
import pytest

import codec_lanes_model as M
import lz4_model as L4
import zstd_model as ZS

CODECS = ["default", "lz4", "zstd"]
_CACHE = {}


def _cases(codec):
    if codec not in _CACHE:
        _CACHE[codec] = {c.name: c for c in M.cases(codec)}
    return _CACHE[codec]


def _libs(codec):
    if codec == "lz4" and L4.liblz4() is None:
        pytest.skip("liblz4 cannot be loaded")
    if codec == "zstd" and ZS.libzstd() is None:
        pytest.skip("libzstd cannot be loaded")


@pytest.mark.parametrize("codec", CODECS)
def test_every_case_decodes_to_its_body_in_the_library_and_the_emulation(codec):
    _libs(codec)
    for c in _cases(codec).values():
        lib, emu, reason = M.reference(codec, c.stream, len(c.body))
        assert lib == c.body, c
        assert emu == c.body, (c, reason)
        assert len(c.body) >= 2 and len(M.segment(c.stream)) >= 10, c


@pytest.mark.parametrize("codec", CODECS)
def test_generation_is_deterministic(codec):
    _libs(codec)
    again = M.cases(codec)
    assert [(c.name, c.stream, c.body, c.path) for c in again] == \
        [(c.name, c.stream, c.body, c.path) for c in _cases(codec).values()]


# ------------------------------------------------------------------------------------------------ DefaultCodec
def _walk(name):
    return M.inflate_walk(_cases("default")[name].stream)


def _matches(members):
    return [m for mb in members for b in mb["blocks"] if b["type"] != "stored" for m in b["matches"]]


def test_deflate_every_distance_has_every_length_in_fixed_blocks():
    for d in M.DIST_SET:
        (mb,) = _walk("dist_%d" % d)
        assert [b["type"] for b in mb["blocks"]] == ["fixed"]
        assert _matches([mb]) == [(n, d) for n in M.LEN_SET], d


def test_deflate_back_to_back_and_short_after_long_matches():
    (mb,) = _walk("back_to_back_long")
    ms = _matches([mb])
    assert len(ms) == 10 and mb["blocks"][0]["literals"] == 50       # every literal before the first match
    assert sum(n >= 32 for n, _ in ms) >= 8 and any(d < 32 for n, d in ms if n >= 32)
    (mb,) = _walk("short_reads_long")
    ms = _matches([mb])
    assert ms[0] == (64, 7) and ms[1] == (5, 3)                      # long over lane 0's literals, then short over it


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 65535])
def test_deflate_stored_block_lengths_and_a_match_back_into_them(n):
    (mb,) = _walk("stored_%d" % n)
    assert [b["type"] for b in mb["blocks"]] == ["fixed", "stored", "fixed"]
    assert mb["blocks"][1]["len"] == n
    (length, dist), = mb["blocks"][2]["matches"]
    if n >= 3:
        assert dist <= n                                             # the match source lies in the stored block


def test_deflate_stored_blocks_after_every_bit_offset():
    ends = []
    for b in range(8):
        (mb,) = _walk("stored_after_bit_%d" % b)
        assert [x["type"] for x in mb["blocks"]] == ["fixed", "stored", "fixed"]
        ends.append(mb["blocks"][0]["end_bit"])
    assert ends == list(range(8))


def test_deflate_dynamic_blocks_have_their_shapes():
    (mb,) = _walk("dynamic_15_bit_codes")
    (b,) = mb["blocks"]
    assert b["type"] == "dynamic" and b["max_len"] == 15
    (b,) = _walk("dynamic_one_distance_code")[0]["blocks"]
    assert b["ndist_codes"] == 1 and any(n >= 32 and d < 32 for n, d in b["matches"])
    (b,) = _walk("dynamic_no_distance_codes")[0]["blocks"]
    assert b["ndist_codes"] == 0 and not b["matches"]
    for last in ("17", "16"):
        (b,) = _walk("dynamic_repeat_edges_" + last)[0]["blocks"]
        syms = [s for s, _ in b["cl"]]
        assert syms[0] == 18 and syms[-1] == int(last)
        hlit = b["hlit"]
        # a 16 that starts among the literal/length lengths and runs into the distance lengths
        starts = [i for s, i in b["cl"]] + [hlit + 10 ** 6]
        assert any(s == 16 and i < hlit < starts[k + 1] for k, (s, i) in enumerate(b["cl"]))
    (b,) = _walk("dynamic_hlit_286")[0]["blocks"]
    assert b["hlit"] == 286 and b["ndist_codes"] == 30


def test_deflate_window_bits_and_members():
    for cinfo in range(8):
        assert [m["cinfo"] for m in _walk("window_bits_%d" % (cinfo + 8))] == [cinfo]
    for m in range(1, 8):
        c = _cases("default")["members_%d" % m]
        assert len(M.inflate_walk(c.stream)) == m and c.body.endswith(b"\xff\xff")
        if m >= 3:
            assert M.zlib.compress(b"", 6) in c.stream                   # an empty member
        assert len(M.zlib.decompress(c.stream[-10:])) == 2               # the last member holds 2 bytes
    assert {len(c.body) for n, c in _cases("default").items() if n.startswith("adler_")} == {2, 3, 31, 32, 33, 5552, 5553, 65537}


# ------------------------------------------------------------------------------------------------ Lz4Codec
def _chunks(name):
    return [ch for _, chs in L4.blocks(_cases("lz4")[name].stream) for ch in chs]


def test_lz4_literal_runs_match_lengths_and_offsets():
    for L in (14, 15, 270, 525):
        assert M.l4_sequences(_chunks("literal_run_%d" % L)[0])[0][0] == L
    assert [s[2] for s in M.l4_sequences(_chunks("match_lengths_4_to_19")[0])[:-1]] == list(range(4, 20))
    assert [s[2] for s in M.l4_sequences(_chunks("match_lengths_19_plus_255k")[0])[:-1]] == [274, 529, 784]
    for off in M.L4_OFFSETS:
        seqs = M.l4_sequences(_chunks("offset_%d" % off)[0])
        assert {s[1] for s in seqs[:-1]} == {off}
        assert any(ml >= 32 for _, _, ml in seqs[:-1])


def test_lz4_end_of_chunk_limits_and_the_chunk_cap():
    c = _cases("lz4")["chunk_of_cap_lastliterals"]
    assert len(c.body) == L4.CHUNK_CAP
    seqs = M.l4_sequences(_chunks("chunk_of_cap_lastliterals")[0])
    assert seqs[-1][0] == 5                                          # LASTLITERALS: the match ends 5 bytes before the cap
    seqs = M.l4_sequences(_chunks("literal_run_at_mflimit")[0])
    op = seqs[0][0] + seqs[0][2] + seqs[1][0]
    assert op == L4.CHUNK_CAP - 12                                   # MFLIMIT: a literal run ending 12 bytes before the cap


def test_lz4_unit_and_serial_variants_of_every_crafted_chunk():
    cs = _cases("lz4")
    for name, c in cs.items():
        chunks_per_block = [len(chs) for _, chs in L4.blocks(c.stream)]
        if c.path == "unit":
            assert set(chunks_per_block) == {1}, name
            assert all(raw <= L4.CHUNK_CAP for raw, _ in L4.blocks(c.stream)), name
        else:
            assert max(chunks_per_block) > 1, name
        if name + "_twice" in cs:
            assert cs[name + "_twice"].body == c.body * 2
    if L4.liblz4() is not None:
        assert {n.split("_body")[0] for n in cs if n.startswith("liblz4_")} == {"liblz4_fast1", "liblz4_fast8", "liblz4_fast65537",
                                                                               "liblz4_hc0"}


def test_lz4_short_block_decodes_validly_to_fewer_bytes_than_its_raw_length():
    z, raw = M.lz4_short_block()
    ((blk_raw, (chunk,)),) = [(int.from_bytes(z[:4], "big"), [z[8:]])]
    assert blk_raw == raw and len(L4.decode_chunk(chunk)) == raw - 1
    lib, emu, reason = M.reference("lz4", z, raw)
    assert lib is None and emu is None and reason == "truncated block header"


# ------------------------------------------------------------------------------------------------ ZStandardCodec
def test_zstd_every_literals_type_and_sequence_mode_is_present():
    _libs("zstd")
    kinds, modes = set(), [set(), set(), set()]
    for c in _cases("zstd").values():
        for f in M.zstd_walk(c.stream):
            if isinstance(f, dict):
                for _, _, lk, md in f["blocks"]:
                    kinds.add(lk)
                    for t in range(3):
                        if md:
                            modes[t].add(md[t])
    assert kinds >= {"raw", "rle", "huf1", "huf4", "treeless1", "treeless4"}
    assert modes[0] == modes[1] == modes[2] == {0, 1, 2, 3}


def test_zstd_crafted_blocks_and_frames():
    cs = _cases("zstd")
    (f,) = M.zstd_walk(cs["rle_block_maximum"].stream)
    assert f["blocks"] == [(1, 131072, None, None)] and f["fcs"] == 131072
    for name, c in cs.items():
        fr = [f for f in M.zstd_walk(c.stream) if isinstance(f, dict)]
        assert c.path == ("unit" if all(f["fcs"] is not None for f in fr) else "serial"), name
        if name.startswith("seq_"):
            blk = fr[0]["blocks"][-1]
            assert blk[3] == (1, 1, 1) and blk[2] == ("rle" if "rle_literals" in name else "raw"), name
    for oc in (2, 3, 4, 5):
        assert cs["seq_offsets_code_%d" % oc].path == "unit" and cs["seq_offsets_code_%d_nofcs" % oc].path == "serial"
    walk = M.zstd_walk(cs["staged_literals_before_next_frame"].stream)
    assert len(walk) == 2 and walk[0]["fcs"] is None and walk[0]["blocks"][-1][2] == "rle"


def test_zstd_library_frames_windows_checksums_and_skippable_frames():
    _libs("zstd")
    cs = _cases("zstd")
    wins = {}
    for wlog in range(10, 28):
        (f,) = M.zstd_walk(cs["lib_window_log_%d" % wlog].stream)
        wins[wlog] = f["window"]
        assert f["fcs"] is None
        assert M.zstd_walk(cs["lib_window_log_%d_fcs" % wlog].stream)[0]["fcs"] == len(cs["lib_window_log_%d" % wlog].body)
    assert all(wins[w] <= 1 << w for w in wins) and wins[10] == 1024
    for name in ("frames_fcs_skippable_checksum", "frames_mixed_skippable_checksum"):
        walk = M.zstd_walk(cs[name].stream)
        assert sum(isinstance(f, tuple) for f in walk) >= 1
        assert any(isinstance(f, dict) and f["checksum"] for f in walk)
        assert sum(isinstance(f, dict) for f in walk) >= 4


def test_xxh64_matches_libzstd_checksums():
    _libs("zstd")
    for body in (b"", b"a", b"abcdefgh" * 5, bytes(range(256)) * 3):
        z = M.zstd_lib_frame(body, 3, checksum=True)
        assert int.from_bytes(z[-4:], "little") == M.xxh64(body) & 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ corrupted streams
@pytest.mark.parametrize("codec", CODECS)
def test_corruption_corpus_is_seeded_and_mixes_verdicts(codec):
    _libs(codec)
    a = M.corrupt(codec, n=200)
    assert a == M.corrupt(codec, n=200)
    refused = [m for m in a if m[2] is None]
    assert 20 < len(refused) < len(a)
    assert all(m[3] for m in refused) and all(m[3] is None for m in a if m[2] is not None)
    assert len({m[3] for m in refused}) >= 4
    # the library never accepts different bytes from the ones the emulation returns
    for z, n, got, _ in a:
        lib = M.library(codec, z, n)
        if got is not None and lib is not None:
            assert lib == got

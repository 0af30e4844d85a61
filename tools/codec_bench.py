"""DefaultCodec, Lz4Codec, ZStandardCodec and SnappyCodec cost on the device: one JSON line per case, no-codec, zlib,
LZ4, zstd and Snappy runs alternating in one process (the *_lz4 fields are Lz4Codec's, the *_zstd fields
ZStandardCodec's, the *_snappy fields SnappyCodec's).

  1. config-2 map side: 1e8 random 80-byte records, P = 64, sort_device_fixed (the stored / all-literal path)
  2. compressible map side: Text words drawn from a Zipf law with IntWritable 1 values, sort_device_fixed
  3. reduce side: config-3 segments compressed on the host (zlib level 1; LZ4, zstd and Snappy by the device writers' host
     emulations, zstd's frames taking the one-warp-per-frame path; zstd also as libzstd level-3 one-frame streams
     without content size, the one-warp-per-segment path, where libzstd can be loaded), reopen + write_ifile_device
  4. e2e through host buffers: collect_batch + flush_to_memory of the case-2 records

Times: host clock around fully synchronised library calls.  The card name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import tez_oracle as O  # noqa: E402
import tez_b200 as T  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def zcap(raw, P):
    """room for the zlib (every chunk stored), the LZ4 and Snappy (every block all literals) and the zstd (every frame
    raw) worst case"""
    return raw + raw // 255 + 10 * (raw // 32768 + P + 1) + 11 * P + 64


CODECS = (0, T.CODEC_LZ4, T.CODEC_ZSTD, T.CODEC_SNAPPY, T.CODEC_DEFAULT)   # zlib last: the compressible case reads its output back


def lz4_stream(body):
    """the device writer's LZ4 stream of one body, run on the host (tezgpu_debug_lz4_compress_emulate)"""
    L = T._lib.load()
    cap = len(body) + len(body) // 255 + 10 * (len(body) // T.LZ4_BLOCK_BYTES + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    T._lib.check(L.tezgpu_debug_lz4_compress_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def zstd_stream(body):
    """the device writer's zstd frames of one body, run on the host (tezgpu_debug_zstd_compress_emulate)"""
    L = T._lib.load()
    cap = len(body) + 10 * (len(body) // T.ZSTD_BLOCK_BYTES + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    T._lib.check(L.tezgpu_debug_zstd_compress_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def snappy_stream(body):
    """the device writer's Snappy stream of one body, run on the host (tezgpu_debug_snappy_compress_emulate)"""
    L = T._lib.load()
    cap = len(body) + 14 * (len(body) // T.SNAPPY_BLOCK_BYTES + 2) + 64
    out = (C.c_uint8 * cap)()
    n = C.c_uint64()
    T._lib.check(L.tezgpu_debug_snappy_compress_emulate(body, len(body), out, cap, C.byref(n)))
    return bytes(out[:n.value])


def libzstd_level3(body):
    """libzstd level 3, one frame without Frame_Content_Size (ZSTD_c_contentSizeFlag 0), or None without libzstd"""
    try:
        L = C.CDLL("libzstd.so.1")
    except OSError:
        return None
    L.ZSTD_createCCtx.restype = C.c_void_p
    L.ZSTD_compress2.restype = L.ZSTD_compressBound.restype = C.c_size_t
    L.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
    cctx = L.ZSTD_createCCtx()
    L.ZSTD_CCtx_setParameter(cctx, 100, 3)
    L.ZSTD_CCtx_setParameter(cctx, 200, 0)
    cap = L.ZSTD_compressBound(C.c_size_t(len(body)))
    out = C.create_string_buffer(cap)
    n = L.ZSTD_compress2(cctx, out, cap, body, len(body))
    L.ZSTD_freeCCtx(cctx)
    return out.raw[:n]


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def words_kv(n, seed=7):
    """n records of an 8-byte Text key (vint 7, 'w', 6 digits of a Zipf-drawn word id) and IntWritable 1"""
    rng = np.random.default_rng(seed)
    ids = np.minimum(rng.zipf(1.2, n), 999999)
    rec = np.empty((n, 12), dtype=np.uint8)
    rec[:, 0] = 7
    rec[:, 1] = ord("w")
    for d in range(6):
        rec[:, 7 - d] = ord("0") + (ids // 10 ** d) % 10
    rec[:, 8:11] = 0
    rec[:, 11] = 1
    return rec.reshape(-1)


def map_side(name, kv, kl, vl, cmp_kind, P, runs, out):
    n = kv.size // (kl + vl)
    d_kv = torch.from_numpy(kv).cuda()
    raw_cap = n * (kl + vl + 2) + 10 * P + 64
    d_out = torch.empty(zcap(raw_cap, P), dtype=torch.uint8, device="cuda")
    res = {c: [] for c in CODECS}
    lens = {}
    sorters = {c: T.GpuSorter(P, comparator=cmp_kind, fixed=(kl, vl), codec=c) for c in CODECS}
    for r in range(runs + 1):
        for c, s in sorters.items():
            ms, (ln, index, st) = timed(lambda: s.sort_device_fixed(d_kv.data_ptr(), n, d_out.data_ptr(), d_out.numel()))
            if r:
                res[c].append(ms)
            lens[c] = (ln, index)
    raw = lens[0][0]
    zlen, zindex = lens[T.CODEC_DEFAULT]
    line = dict(case=name, records=n, partitions=P, raw_bytes=raw, compressed_bytes=zlen, ratio=round(zlen / raw, 4),
                ms_no_codec=round(min(res[0]), 2), ms_codec=round(min(res[T.CODEC_DEFAULT]), 2),
                ms_runs_no_codec=[round(x, 2) for x in res[0]], ms_runs_codec=[round(x, 2) for x in res[T.CODEC_DEFAULT]])
    extra = line["ms_codec"] - line["ms_no_codec"]
    line["compress_gbps_derived"] = round(raw / extra / 1e6, 2) if extra > 0 else None
    llen = lens[T.CODEC_LZ4][0]
    line.update(compressed_bytes_lz4=llen, ratio_lz4=round(llen / raw, 4), ms_lz4=round(min(res[T.CODEC_LZ4]), 2),
                ms_runs_lz4=[round(x, 2) for x in res[T.CODEC_LZ4]])
    extra = line["ms_lz4"] - line["ms_no_codec"]
    line["compress_gbps_derived_lz4"] = round(raw / extra / 1e6, 2) if extra > 0 else None
    slen = lens[T.CODEC_ZSTD][0]
    line.update(compressed_bytes_zstd=slen, ratio_zstd=round(slen / raw, 4), ms_zstd=round(min(res[T.CODEC_ZSTD]), 2),
                ms_runs_zstd=[round(x, 2) for x in res[T.CODEC_ZSTD]])
    extra = line["ms_zstd"] - line["ms_no_codec"]
    line["compress_gbps_derived_zstd"] = round(raw / extra / 1e6, 2) if extra > 0 else None
    nlen = lens[T.CODEC_SNAPPY][0]
    line.update(compressed_bytes_snappy=nlen, ratio_snappy=round(nlen / raw, 4), ms_snappy=round(min(res[T.CODEC_SNAPPY]), 2),
                ms_runs_snappy=[round(x, 2) for x in res[T.CODEC_SNAPPY]])
    extra = line["ms_snappy"] - line["ms_no_codec"]
    line["compress_gbps_derived_snappy"] = round(raw / extra / 1e6, 2) if extra > 0 else None
    if name == "compressible":
        # zlib level 1 on the same bodies (the first 8 partitions)
        host = d_out[:zlen].cpu().numpy().tobytes()
        zsum = rsum = 0
        for p in range(8):
            s0, rl, pl = (int(x) for x in zindex[p])
            body = zlib.decompress(host[s0 + 4:s0 + pl - 4])
            zsum += pl - 8
            rsum += len(zlib.compress(body, 1))
        line["ratio_to_zlib1"] = round(zsum / rsum, 4)
    for s in sorters.values():
        s.close()
    del d_kv, d_out
    torch.cuda.empty_cache()
    out.append(line)


def reduce_side(nseg, seg_bytes, runs, out):
    plain, _ = O.gen_c3_segments(nseg, seg_bytes, seed=3, threads=16)
    plain = [p.tobytes() for p in plain]
    zsegs, raws = [], []
    for p in plain:
        z = zlib.compress(p[4:-4], 1)
        zsegs.append(b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big"))
        raws.append(len(p) - 4)
    with ThreadPoolExecutor(16) as ex:
        lsegs = [b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big") for z in ex.map(lambda p: lz4_stream(p[4:-4]), plain)]
        ssegs = [b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big") for z in ex.map(lambda p: zstd_stream(p[4:-4]), plain)]
        nsegs = [b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big") for z in ex.map(lambda p: snappy_stream(p[4:-4]), plain)]
        jz = list(ex.map(lambda p: libzstd_level3(p[4:-4]), plain))
    jsegs = None if jz[0] is None else [b"TIF\x01" + z + zlib.crc32(z).to_bytes(4, "big") for z in jz]
    if jsegs is None:
        print("note: libzstd cannot be loaded; the zstd one-warp-per-segment (libzstd level 3) arm is skipped", file=sys.stderr)
    mz = T.GpuMerger(zsegs, comparator=T.CMP_TEXT, codec=T.CODEC_DEFAULT, raw_lens=raws)
    ml = T.GpuMerger(lsegs, comparator=T.CMP_TEXT, codec=T.CODEC_LZ4, raw_lens=raws)
    ms_ = T.GpuMerger(ssegs, comparator=T.CMP_TEXT, codec=T.CODEC_ZSTD, raw_lens=raws)
    mn = T.GpuMerger(nsegs, comparator=T.CMP_TEXT, codec=T.CODEC_SNAPPY, raw_lens=raws)
    mp = T.GpuMerger(plain, comparator=T.CMP_TEXT)
    cap = max(mz.output_bound(), ml.output_bound(), ms_.output_bound(), mn.output_bound(), mp.output_bound())
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    res = {c: [] for c in CODECS + ("java",)}
    arms = [(0, mp, plain), (T.CODEC_DEFAULT, mz, zsegs), (T.CODEC_LZ4, ml, lsegs), (T.CODEC_ZSTD, ms_, ssegs), (T.CODEC_SNAPPY, mn, nsegs)]
    if jsegs is not None:
        arms.append(("java", ms_, jsegs))
    for r in range(runs + 1):
        for c, m, segs in arms:
            def step():
                if c:
                    m.reopen(segs, raw_lens=raws)
                else:
                    m.reopen(segs)
                return m.write_ifile_device(d_out.data_ptr(), cap)
            ms, (raw, part, st) = timed(step)
            if r:
                res[c].append(ms)
    raw_total, z_total = sum(len(p) for p in plain), sum(len(z) for z in zsegs)
    line = dict(case="reduce_c3_zlib1", segments=nseg, raw_bytes=raw_total, compressed_in_bytes=z_total,
                ms_plain=round(min(res[0]), 2), ms_codec=round(min(res[1]), 2),
                ms_runs_plain=[round(x, 2) for x in res[0]], ms_runs_codec=[round(x, 2) for x in res[1]],
                compressed_in_bytes_lz4=sum(len(z) for z in lsegs), ms_lz4=round(min(res[T.CODEC_LZ4]), 2),
                ms_runs_lz4=[round(x, 2) for x in res[T.CODEC_LZ4]],
                compressed_in_bytes_zstd=sum(len(z) for z in ssegs), ms_zstd=round(min(res[T.CODEC_ZSTD]), 2),
                ms_runs_zstd=[round(x, 2) for x in res[T.CODEC_ZSTD]],
                compressed_in_bytes_snappy=sum(len(z) for z in nsegs), ms_snappy=round(min(res[T.CODEC_SNAPPY]), 2),
                ms_runs_snappy=[round(x, 2) for x in res[T.CODEC_SNAPPY]],
                note="codec: reads compressed segments and writes a compressed merged segment")
    if jsegs is not None:
        line.update(compressed_in_bytes_zstd_libzstd3=sum(len(z) for z in jsegs), ms_zstd_libzstd3=round(min(res["java"]), 2),
                    ms_runs_zstd_libzstd3=[round(x, 2) for x in res["java"]])
    out.append(line)
    mz.close()
    ml.close()
    ms_.close()
    mn.close()
    mp.close()


def e2e(kv, kl, vl, cmp_kind, P, runs, out):
    """collect_batch (variable-width API, one batch) + flush_to_memory"""
    n = kv.size // (kl + vl)
    stride = kl + vl
    key_off = (np.arange(n, dtype=np.uint64) * stride).astype(np.uint32)
    val_off = key_off + np.uint32(kl)
    val_len = np.full(n, vl, dtype=np.uint32)
    res = {c: [] for c in CODECS}
    moved = {}
    for r in range(runs + 1):
        for c in CODECS:
            with T.GpuSorter(P, comparator=cmp_kind, codec=c) as s:
                def step():
                    s.collect(kv, key_off, val_off, val_len)
                    return s.flush_to_memory()
                ms, (o, _, _, _) = timed(step)
            if r:
                res[c].append(ms)
            moved[c] = len(o)
    out.append(dict(case="e2e_host_buffers", api="collect_batch + flush_to_memory", records=n, kv_bytes=kv.size,
                    down_bytes_no_codec=moved[0], down_bytes_codec=moved[1], ms_no_codec=round(min(res[0]), 1),
                    ms_codec=round(min(res[1]), 1), kv_gbps_no_codec=round(kv.size / min(res[0]) / 1e6, 2),
                    kv_gbps_codec=round(kv.size / min(res[1]) / 1e6, 2), down_bytes_lz4=moved[T.CODEC_LZ4],
                    ms_lz4=round(min(res[T.CODEC_LZ4]), 1), kv_gbps_lz4=round(kv.size / min(res[T.CODEC_LZ4]) / 1e6, 2),
                    down_bytes_zstd=moved[T.CODEC_ZSTD], ms_zstd=round(min(res[T.CODEC_ZSTD]), 1),
                    kv_gbps_zstd=round(kv.size / min(res[T.CODEC_ZSTD]) / 1e6, 2), down_bytes_snappy=moved[T.CODEC_SNAPPY],
                    ms_snappy=round(min(res[T.CODEC_SNAPPY]), 1), kv_gbps_snappy=round(kv.size / min(res[T.CODEC_SNAPPY]) / 1e6, 2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--c2-records", type=int, default=10 ** 8)
    ap.add_argument("--words-records", type=int, default=90 * 10 ** 6)
    ap.add_argument("--c3-segments", type=int, default=256)
    ap.add_argument("--c3-seg-bytes", type=int, default=1 << 22)
    a = ap.parse_args()
    dev = card()
    out = []
    map_side("config2_stored", O.gen_c2(0, a.c2_records, seed=2, threads=16), 16, 64, T.CMP_BYTES, 64, a.runs, out)
    words = words_kv(a.words_records)
    map_side("compressible", words, 8, 4, T.CMP_TEXT, 64, a.runs, out)
    reduce_side(a.c3_segments, a.c3_seg_bytes, a.runs, out)
    e2e(words[:12 * (a.words_records // 4)], 8, 4, T.CMP_TEXT, 64, a.runs, out)
    for line in out:
        line["device"] = dev
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

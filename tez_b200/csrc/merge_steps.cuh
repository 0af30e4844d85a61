// merge_steps.cuh -- k-way merge of host-resident segments under a device-memory budget, in key-range steps
// (tezgpu_merge_open_bounded).  The reference never fails a task because of data size: TezMerger merges any number of
// segments through one small buffer per segment (SORT/TezMerger.java:717-912).  Here a merge whose inputs and
// workspace do not fit the budget runs as a sequence of steps, each an ordinary Merger::open over device windows.
//
// A merge is a stable sort by (partition, key) with ties in (segment, position) order, so it can be cut at key
// boundaries without changing its output.  Each step uploads a window [c_i, c_i + W_i) of every unfinished segment i,
// finds the last complete record of every window (k_step_walk<false>), takes the smallest of those keys as the
// splitter S (k_step_splitter; a window that reaches its segment's EOF does not bound S), and cuts every window before
// its first record with key >= S (k_step_walk<true>).  The records before the cuts are exactly those with key < S, a
// prefix of every window, and the step merges them with the Merger reading the windows in place.  Every key group
// therefore lies inside one step: combiners and isSameKey never see a step boundary, and the first record of a step
// never equals the last one of the step before.  The record at a cut is always a full record (a repeat has the key of
// the record before it); a V_END_MARKER in front of it belongs to the step before, whose piece then ends in FD FF FF.
// Bytes after a cut are uploaded again by the next step.
//
// Writes stitch the pieces every step emits into the file the one-step merge writes, with or without a codec
// (tezgpu_merge_open_bounded_write_codec): the header (TIF\0; TIF\x01 with a codec, and 78 01 with zlib) only at the
// start of a partition, the FF FF EOF markers and the trailer only at its end.  One pass per step takes its pieces.
// Without a codec a piece is copied as it is.  A codec compresses it on the codec's chunk grid, counted from the
// start of each partition's body, so the stream is the one the one-step merge writes: a piece that closes its
// partition is compressed whole; of the partition the step leaves open only the whole chunks before the piece's last
// byte are, and the bytes after them (1 to one chunk) wait in a device carry buffer for the partition's next piece.
// zlib chunks of an open piece end with the sync-flush block like every inner chunk (ZSeg::open), and the Adler-32 at
// a partition's end is folded from the chunks' values.  The CRC-32 trailer is folded across steps from each piece's
// raw remainder (k_stitch_fold, k_stitch_trailers): a codec's chunk remainders, or, without one, the trailer the
// step's Merger wrote after the piece.
#pragma once
#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "codec.cuh"
#include "concat.cuh"
#include "merger.cuh"

namespace tezgpu {

// ---- workspace bound from which the windows are sized (DESIGN.md section 3, "Bounded-memory merge").  A step that merges n records with kv
//      key + value bytes out of windows of w bytes holds at most
//        STEP_BYTES_PER_WINDOW_BYTE * w + STEP_BYTES_PER_KV_BYTE * kv + STEP_BYTES_PER_RECORD * n + fixed(P, segments)
//      device bytes: the windows and the parse tables over them; the output image, the combiner's copy and one batch
//      of the record iterator; and per record the parse arrays (32 B), the sort words and order (16 B), the tie
//      refinement (<= 65 B), the emit's sizes, offsets and flags (13 B), the iterator's offsets and index (32 B), the
//      combiner's group arrays (<= 45 B) and the output framing (12 B), rounded up.  Buffers only grow, so the bound is
//      applied to the largest w, kv and n of all steps so far.
constexpr uint64_t STEP_BYTES_PER_WINDOW_BYTE = 2;
constexpr uint64_t STEP_BYTES_PER_KV_BYTE = 3;
constexpr uint64_t STEP_BYTES_PER_RECORD = 320;
constexpr uint64_t STEP_FIXED_BYTES = 8ull << 20;
constexpr uint64_t STEP_FIXED_PER_PARTITION = 256;
constexpr uint64_t STEP_FIXED_PER_SEGMENT = 512;
constexpr uint64_t STEP_MIN_SHARE = 256;          // smallest window the step loop gives a segment

struct StepWin {
  uint64_t off;         // window start in the window buffer (16-byte aligned)
  uint64_t len;         // window bytes
  uint32_t at_end;      // the window ends at its segment's body end
  uint32_t partition;
};
struct StepScan {
  uint64_t last_koff;   // window offset of the key of the last complete record (the full key a repeat refers to)
  uint64_t kv;          // key + value bytes of the complete records
  uint32_t last_klen;
  uint32_t nrec;        // complete records
  uint32_t eof;         // the EOF markers were read
  uint32_t bad;         // a malformed record, or the window reaches the body end inside a record
};
struct StepCut {
  uint64_t bytes;       // window bytes before the first record with key >= S (a V_END_MARKER in front of it included);
                        // at the EOF markers: the bytes before them
  uint64_t kv;
  uint32_t nrec;
  uint32_t pad;
};

// the merge order over (partition, key): the RawComparator order of compare_keys_from from byte 0
__device__ __forceinline__ int step_compare(int cmp, uint32_t pa, const uint8_t *a, uint32_t la, uint32_t pb,
                                            const uint8_t *b, uint32_t lb) {
  if (pa != pb) return pa < pb ? -1 : 1;
  const uint32_t sa = key_content_skip(cmp, a, la), sb = key_content_skip(cmp, b, lb);
  a += sa; b += sb; la -= sa; lb -= sb;
  const uint32_t nmin = la < lb ? la : lb;
  for (uint32_t i = 0; i < nmin; i++) {
    const uint32_t x = norm_byte(cmp, a, i), y = norm_byte(cmp, b, i);
    if (x != y) return x < y ? -1 : 1;
  }
  return la < lb ? -1 : (la == lb ? 0 : 1);
}

// Walks every window with IFile.Reader semantics, one warp per window (warp_window_walk).  A window ends wherever the
// bytes end, usually inside a record: the walk stops there (status REC_PAST_END).  CUT=false fills scan[] (complete
// records, the last complete key, EOF, malformed); CUT=true counts the records with (partition, key) < S, S being the
// last complete key of window *split (none when *split < 0), and fills cut[].
constexpr int STEP_AT_SPLIT = 4;   // k_step_walk<true> stopped at a record with key >= S
template <bool CUT>
__global__ void __launch_bounds__(PARSE_WARPS * 32)
    k_step_walk(const uint8_t *__restrict__ win, const StepWin *__restrict__ wins, uint32_t nw, int cmp,
                StepScan *__restrict__ scan, const int32_t *__restrict__ split, StepCut *__restrict__ cut) {
  __shared__ __align__(16) uint8_t s_win[PARSE_WARPS][PARSE_WIN];
  const int warp = threadIdx.x >> 5;
  const uint32_t s = blockIdx.x * PARSE_WARPS + warp;
  if (s >= nw) return;
  const StepWin sw = wins[s];
  const uint8_t *src = win + sw.off;
  const uint8_t *skey = nullptr;
  uint32_t sklen = 0, spart = 0;
  bool bounded = false;
  if (CUT && *split >= 0) {
    const StepScan q = scan[*split];
    skey = win + wins[*split].off + q.last_koff;
    sklen = q.last_klen;
    spart = wins[*split].partition;
    bounded = true;
  }
  uint64_t orig_koff = 0, orig_klen = 0, n = 0, kv = 0;
  const WalkEnd e = warp_window_walk(src, sw.len, 0, sw.len, s_win[warp], [&](const RecHdr &h) {
    uint64_t q = h.pos, ko = orig_koff, kfull = orig_klen;
    if (h.kl != -2) {
      if (q + (uint64_t)h.kl > sw.len) return REC_PAST_END;
      ko = q;
      kfull = (uint64_t)h.kl;
      q += (uint64_t)h.kl;
    } else if (n == 0) {
      return REC_BAD;   // a window starts at a full record: a repeat needs a previous key
    }
    if (q + (uint64_t)h.vl > sw.len) return REC_PAST_END;
    if (CUT && bounded && h.kl != -2 && step_compare(cmp, sw.partition, src + ko, (uint32_t)kfull, spart, skey, sklen) >= 0)
      return STEP_AT_SPLIT;
    orig_koff = ko;
    orig_klen = kfull;
    n++;
    kv += kfull + (uint64_t)h.vl;
    return REC_OK;
  });
  if ((threadIdx.x & 31) != 0) return;
  if (CUT) {
    StepCut c;
    c.bytes = e.status == REC_BAD ? 0 : e.stop;
    c.kv = kv;
    c.nrec = (uint32_t)n;
    c.pad = 0;
    cut[s] = c;
  } else {
    StepScan q;
    q.last_koff = orig_koff;
    q.kv = kv;
    q.last_klen = (uint32_t)orig_klen;
    q.nrec = (uint32_t)n;
    q.eof = e.status == REC_EOF;
    q.bad = e.status == REC_BAD || (e.status == REC_PAST_END && sw.at_end);
    scan[s] = q;
  }
}

// S = the smallest (partition, last complete key) of the windows that hold a complete record and do not end in their
// segment's EOF markers; *split = that window, or -1 when every window reaches EOF.  on_split[w]: window w's last
// complete key equals S (the windows a key group larger than them holds up).  One thread: there is one window per
// segment.
__global__ void k_step_splitter(const uint8_t *__restrict__ win, const StepWin *__restrict__ wins, uint32_t nw, int cmp,
                                const StepScan *__restrict__ scan, int32_t *__restrict__ split, uint8_t *__restrict__ on_split) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int32_t best = -1;
  auto bounds = [&](uint32_t s) { return scan[s].nrec > 0 && !(scan[s].eof && wins[s].at_end); };
  auto cmp_win = [&](uint32_t a, uint32_t b) {
    return step_compare(cmp, wins[a].partition, win + wins[a].off + scan[a].last_koff, scan[a].last_klen,
                        wins[b].partition, win + wins[b].off + scan[b].last_koff, scan[b].last_klen);
  };
  for (uint32_t s = 0; s < nw; s++)
    if (bounds(s) && (best < 0 || cmp_win(s, (uint32_t)best) < 0)) best = (int32_t)s;
  *split = best;
  for (uint32_t s = 0; s < nw; s++) on_split[s] = best >= 0 && bounds(s) && cmp_win(s, (uint32_t)best) == 0;
}

// the EOF markers FF FF after every cut, so that each window prefix reads as a header-less segment (the 4 bytes after
// them stand for the checksum an in-memory segment does not have)
__global__ void k_step_terminate(uint8_t *__restrict__ win, const StepWin *__restrict__ wins, const StepCut *__restrict__ cut,
                                 uint32_t nw) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nw) return;
  uint8_t *o = win + wins[s].off + cut[s].bytes;
  o[0] = 0xFF; o[1] = 0xFF; o[2] = 0; o[3] = 0; o[4] = 0; o[5] = 0;
}

// Checksums across steps: raw[w] is the remainder of the bytes window w consumed in this step; acc[segment] folds
// them with crc(A||B) = crc(A) * x^(8 len B) xor crc(B).  A segment whose last bytes went in this step is compared
// with its trailer (IFileInputStream at the end of its stream); a mismatch writes the caller's index + 1 to *bad.
struct StepCrcSeg {
  uint64_t len;         // bytes consumed in this step
  uint64_t total;       // body bytes of the segment
  uint32_t seg;         // caller's segment index
  uint32_t stored;      // big-endian trailer
  uint32_t last;        // the segment ends in this step
  uint32_t pad;
};
__global__ void k_step_crc_fold(const uint32_t *__restrict__ raw, const StepCrcSeg *__restrict__ cs, uint32_t nw,
                                const CrcTables *__restrict__ t, uint32_t *__restrict__ acc, int *__restrict__ bad) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nw) return;
  const StepCrcSeg c = cs[w];
  const uint32_t a = crc_shift_bytes(t, acc[c.seg], c.len) ^ raw[w];
  acc[c.seg] = a;
  if (c.last && crc_from_raw(t, a, c.total) != c.stored) atomicExch(bad, (int)c.seg + 1);
}

// ------------------------------------------------------------------------------------------------ stitched writes
// Room in front of a step's uncompressed image (DESIGN.md section 3): bytes [0, 2) hold the EOF markers an empty
// segment writes, a partition that closes without records of its own writes its carry and FF FF from [2, 4 + carry),
// and the carry of a continuing partition is put right in front of its piece in the image.
constexpr uint64_t STEP_CARRY_ROOM = 65536;
static_assert(STEP_CARRY_ROOM >= 4 + 4 + L4_BLOCK && L4_BLOCK == ZS_BLOCK && L4_BLOCK == SN_BLOCK && ZCHUNK < L4_BLOCK,
              "the room holds the EOF markers, the largest carry with its own, and a step image's first TIF header");
// workspace of one pass per chunk: its slot, its packed bytes (at most a slot), its size, offset, Adler-32, CRC
// descriptor, piece start and remainder; per partition: the piece table, the running CRC and Adler-32, the chunk
// bytes and the trailer; fixed: the carry, the room and the scan's block sums with the buffers' rounding
constexpr uint64_t STEP_CODEC_BYTES_PER_CHUNK_TABLE = 80;
constexpr uint64_t STEP_CODEC_BYTES_PER_PARTITION = 128;
constexpr uint64_t STEP_CODEC_FIXED_BYTES = 1ull << 20;

// One piece of a partition's body on the chunk grid: the piece's own n bytes lie at `off` in its source, the carry (the
// bytes of the partition after its last compressed chunk) right before them.
struct StitchPlan {
  uint64_t off;       // first byte compressed now (the carry's first byte)
  uint64_t len;       // bytes compressed now: whole chunks, or everything when the piece closes the partition
  uint64_t carry;     // bytes after them, kept for the partition's next piece (at most one chunk)
  uint32_t nchunks;
  uint32_t open;      // the partition continues: the last chunk is not the stream's last
};
inline StitchPlan plan_stitch_piece(uint64_t chunk, uint64_t carry, uint64_t off, uint64_t n, bool closes) {
  StitchPlan s;
  const uint64_t all = carry + n;
  s.off = off - carry;
  s.open = closes ? 0 : 1;
  if (closes) {
    s.nchunks = (uint32_t)std::max<uint64_t>(1, div_up(all, chunk));
    s.len = all;
  } else {
    // the chunk the piece ends in waits, also a whole one: only the close tells whether it is the stream's last (zlib
    // marks it final, and a closing piece of no bytes of its own must not add an empty chunk)
    s.nchunks = (uint32_t)(all ? (all - 1) / chunk : 0);
    s.len = (uint64_t)s.nchunks * chunk;
  }
  s.carry = all - s.len;
  return s;
}

// raw CRC remainder (zero initial value, no final xor) of n bytes, bitwise: the host check of the folds below
static inline uint32_t crc_raw_host(const uint8_t *p, uint64_t n) {
  uint32_t c = 0;
  for (uint64_t i = 0; i < n; i++) {
    c ^= p[i];
    for (int k = 0; k < 8; k++) c = (c & 1) ? CRC_POLY ^ (c >> 1) : (c >> 1);
  }
  return c;
}

// one chunk through the host run of a codec's device chunk writer, appended to out (zlib: *adler = its Adler-32)
class ChunkHost {
 public:
  explicit ChunkHost(int32_t codec) : codec_(codec), slot_(codec_layout(codec).slot) {
    switch (codec) {
      case TEZGPU_CODEC_LZ4: l4_.reset(new L4Shared()); break;
      case TEZGPU_CODEC_ZSTD: zs_.reset(new ZsShared()); break;
      case TEZGPU_CODEC_SNAPPY: sn_.reset(new SnShared()); break;
      default: z_.reset(new ZShared());
    }
  }
  void run(const uint8_t *p, uint32_t clen, bool last, std::vector<uint8_t> &out, uint32_t *adler) {
    uint32_t n;
    switch (codec_) {
      case TEZGPU_CODEC_LZ4: l4_compress_block_host(*l4_, p, clen, slot_.data()); n = 8 + l4_->bytes; break;
      case TEZGPU_CODEC_ZSTD: zs_compress_block_host(*zs_, p, clen, slot_.data()); n = zs_->bytes; break;
      case TEZGPU_CODEC_SNAPPY: sn_compress_block_host(*sn_, p, clen, slot_.data()); n = 8 + sn_->bytes; break;
      default:
        z_deflate_chunk_host(*z_, p, clen, last, slot_.data());
        n = z_->bytes;
        *adler = z_->adler;
    }
    out.insert(out.end(), slot_.begin(), slot_.begin() + n);
  }

 private:
  int32_t codec_;
  std::vector<uint8_t> slot_;
  std::unique_ptr<ZShared> z_;
  std::unique_ptr<L4Shared> l4_;
  std::unique_ptr<ZsShared> zs_;
  std::unique_ptr<SnShared> sn_;
};

// Host run of the compressed write across steps over one partition body cut into pieces at cuts[0, ncuts)
// (tezgpu_debug_stitched_compress_emulate): the carry, plan_stitch_piece, the open flag, the Adler-32 fold and the CRC
// fold of the device path, piece by piece.  Returns the codec stream (zlib: 78 01, chunks, Adler-32), which equals the
// stream of the uncut body.
static inline std::vector<uint8_t> stitched_compress_host(int32_t codec, const uint8_t *body, uint64_t len, const uint64_t *cuts,
                                                          uint32_t ncuts) {
  const CodecLayout L = codec_layout(codec);
  const bool zlib = codec == TEZGPU_CODEC_DEFAULT;
  ChunkHost ch(codec);
  std::vector<uint8_t> stream, src, carry, piece;
  if (zlib) stream = {0x78, 0x01};
  uint32_t adler = 1, raw = 0;   // the body's Adler-32 and the chunk bytes' CRC remainder, folded piece by piece
  for (uint32_t i = 0; i <= ncuts; i++) {
    const uint64_t a = i ? cuts[i - 1] : 0, b = i < ncuts ? cuts[i] : len;
    TG_CHECK(a <= b && b <= len, TEZGPU_E_INVALID, "cuts must be non-decreasing offsets into the body");
    const bool closes = i == ncuts;
    src = carry;
    src.insert(src.end(), body + a, body + b);
    const StitchPlan pl = plan_stitch_piece(L.chunk, carry.size(), carry.size(), b - a, closes);
    piece.clear();
    for (uint32_t k = 0; k < pl.nchunks; k++) {
      const uint64_t c0 = (uint64_t)k * L.chunk;
      const uint32_t clen = (uint32_t)std::min<uint64_t>(L.chunk, pl.len - c0);
      uint32_t ca = 1;
      ch.run(src.data() + pl.off + c0, clen, !pl.open && k + 1 == pl.nchunks, piece, &ca);
      if (zlib) adler = z_adler_combine(adler, ca, clen);
    }
    raw = crc_multmodp(raw, crc_host_xpow8(piece.size())) ^ crc_raw_host(piece.data(), piece.size());
    stream.insert(stream.end(), piece.begin(), piece.end());
    carry.assign(src.begin() + pl.off + pl.len, src.end());
  }
  const uint64_t h = zlib ? 2 : 0;
  TG_CHECK(raw == crc_raw_host(stream.data() + h, stream.size() - h), TEZGPU_E_INVALID,
           "the folded CRC differs from the CRC of the stitched stream");
  if (zlib)
    for (int b = 3; b >= 0; b--) stream.push_back((uint8_t)(adler >> (8 * b)));
  return stream;
}

// Per piece of one pass (the pieces of a pass are distinct partitions): the raw CRC remainder of its s.zlen bytes and,
// for zlib, its chunks' Adler-32 values folded into the partition's running values: acc[2p] = remainder of the
// partition's stream bytes so far, acc[2p + 1] = Adler-32 of its body so far.  A codec's piece is its chunk bytes, with
// remainder seg_crc[i].  Without a codec (seg_crc null) a piece is the image bytes at s.body_off taken whole: records R
// of a step (FF FF included when it closes the partition), or FF FF alone from the room (remainder eof_raw).  The
// remainder of R comes from the trailer crc(R || FF FF) the step's Merger wrote behind R || FF FF, through the identity
// of concat.cuh for an open piece, so the bytes are not read.
__global__ void k_stitch_fold(const ZSeg *__restrict__ segs, const uint32_t *__restrict__ part, uint32_t n,
                              const uint32_t *__restrict__ seg_crc, const uint32_t *__restrict__ cadler,
                              const uint8_t *__restrict__ img, const CrcTables *__restrict__ t, uint32_t *__restrict__ acc) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ZSeg s = segs[i];
  const uint32_t p = part[i];
  uint32_t raw = t->eof_raw;
  if (seg_crc) {
    raw = seg_crc[i];
  } else if (s.body_off >= STEP_CARRY_ROOM) {
    const uint64_t b = s.zlen + (s.open ? 2 : 0);   // R || FF FF
    raw = crc_to_raw(t, load_be32(img + s.body_off + b), b);
    if (s.open) raw = concat_records_raw(raw, *t);
  }
  acc[2 * p] = crc_shift_bytes(t, acc[2 * p], s.zlen) ^ raw;
  if (!cadler) return;
  uint32_t a = acc[2 * p + 1];
  for (uint32_t k = 0; k < s.nchunks; k++)
    a = z_adler_combine(a, cadler[s.chunk0 + k], z_min64(ZCHUNK, s.body_len - (uint64_t)k * ZCHUNK));
  acc[2 * p + 1] = a;
}

// per partition with a segment (zb[p]: its stream bytes): the CRC-32 trailer of its stream; zlib: of 78 01, the chunks
// and the big-endian Adler-32
__global__ void k_stitch_trailers(const uint32_t *__restrict__ acc, const uint64_t *__restrict__ zb, uint32_t P, int zlib,
                                  const CrcTables *__restrict__ t, uint32_t *__restrict__ crc) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P || !zb[p]) return;
  if (!zlib) {
    crc[p] = crc_from_raw(t, acc[2 * p], zb[p]);
    return;
  }
  uint32_t hraw = 0, araw = 0;
  hraw = t->slice[0][(hraw ^ 0x78) & 0xFF] ^ (hraw >> 8);
  hraw = t->slice[0][(hraw ^ 0x01) & 0xFF] ^ (hraw >> 8);
  const uint32_t adler = acc[2 * p + 1];
  for (int b = 3; b >= 0; b--) araw = t->slice[0][(araw ^ (adler >> (8 * b))) & 0xFF] ^ (araw >> 8);
  const uint32_t raw = crc_shift_bytes(t, hraw, zb[p] + 4) ^ crc_shift_bytes(t, acc[2 * p], 4) ^ araw;
  crc[p] = crc_from_raw(t, raw, zb[p] + 6);
}

// ------------------------------------------------------------------------------------------------ host loop
class BoundedMerge {
 public:
  Merger &m;
  uint64_t budget;
  DeviceTally &tally;                      // the handle's: every buffer it holds, the Merger's included
  std::vector<tezgpu_segment> in;          // the caller's host segments: read step by step until close
  std::vector<uint64_t> body0, body_end, consumed, grow;
  std::vector<uint32_t> stored;
  std::vector<uint8_t> check_crc, finished;
  uint64_t wtot0 = 0, wtot = 0;            // window bytes of a step (shared by the segments of its lowest partition)
  size_t n_lead = 1;                       // unfinished segments of the lowest partition in the last layout
  std::vector<uint32_t> pmajor;            // segments by partition, the caller's order inside one
  uint64_t max_w = 0, max_kv = 0, max_n = 0;   // largest step so far (the workspace bound is applied to these)
  bool single = false;                     // everything fits: the handle took one ordinary Merger::open
  int steps = 0;                           // steps of the current (or last) pass over the inputs
  uint64_t h2d = 0;                        // window bytes uploaded by all passes
  int iter = 0;                            // record iterator: 0 not started, 1 streaming, 2 ended
  bool in_step = false, have_counts = false;
  uint64_t pass_n = 0, pass_kv = 0, total_n = 0, total_kv = 0;
  DeviceBuffer d_win, d_wins, d_scan, d_cut, d_split, d_on_split, d_acc, d_crcseg, d_crcsd, d_bad;
  std::vector<StepWin> wins;
  std::vector<uint32_t> win_seg;           // window -> caller's segment
  std::vector<StepScan> scans;
  std::vector<StepCut> cuts;
  int32_t zcodec = TEZGPU_CODEC_NONE;      // the codec of the written segments (the steps' Merger writes uncompressed)
  DeviceBuffer d_carry, d_zout, d_piece_part, d_fold, d_stream_bytes, d_trailer;
  PinnedBuffer h_pass;

  BoundedMerge(Merger &mm, uint64_t b, DeviceTally &t) : m(mm), budget(b), tally(t) {}

  // device bytes of one compression pass per chunk (DESIGN.md section 3)
  uint64_t codec_chunk_bytes() const { return 2ull * codec_layout(zcodec).slot + STEP_CODEC_BYTES_PER_CHUNK_TABLE; }
  uint64_t fixed_bytes() const {
    const uint64_t P = (uint64_t)m.pipe.conf.num_partitions;
    uint64_t b = STEP_FIXED_BYTES + STEP_FIXED_PER_PARTITION * P + STEP_FIXED_PER_SEGMENT * (uint64_t)in.size();
    // a compressed write: the chunks no image byte pays for (one per piece, the carry's), the tables, room and carry
    if (zcodec)
      b += (P + 3) * codec_chunk_bytes() + STEP_CODEC_BYTES_PER_PARTITION * P + 2 * STEP_CARRY_ROOM + STEP_CODEC_FIXED_BYTES;
    return b;
  }
  uint64_t need(uint64_t w, uint64_t kv, uint64_t n) const {
    uint64_t b = STEP_BYTES_PER_WINDOW_BYTE * w + STEP_BYTES_PER_KV_BYTE * kv + STEP_BYTES_PER_RECORD * n + fixed_bytes();
    if (zcodec)   // the chunks of the step's uncompressed image
      b += div_up(SortPipeline::output_bound(n, kv, m.pipe.conf.num_partitions), codec_layout(zcodec).chunk) * codec_chunk_bytes();
    return b;
  }

  // m.pipe.codec on entry: the codec the writes compress with (NONE: uncompressed)
  void open(const tezgpu_segment *segs, uint32_t nseg) {
    TallyScope ts(&tally);
    zcodec = m.pipe.codec;
    uint64_t total = 0;
    in.assign(segs, segs + nseg);
    body0.resize(nseg); body_end.resize(nseg); stored.assign(nseg, 0); check_crc.assign(nseg, 0);
    for (uint32_t s = 0; s < nseg; s++) {
      const tezgpu_segment &sg = segs[s];
      TG_CHECK(!(sg.flags & TEZGPU_SEG_DEVICE), TEZGPU_E_INVALID, "tezgpu_merge_open_bounded takes host segments only");
      m.check_segment(sg);
      const bool hdr = sg.flags & TEZGPU_SEG_HAS_HEADER;
      const uint8_t *d = static_cast<const uint8_t *>(sg.data);
      if (hdr) {
        TG_CHECK(d[0] == 'T' && d[1] == 'I' && d[2] == 'F', TEZGPU_E_FORMAT, "Not a valid ifile header (segment " + std::to_string(s) + ")");
        TG_CHECK(d[3] == 0, TEZGPU_E_UNSUPPORTED, "compressed IFile segments are not supported by the bounded merge");
      }
      body0[s] = hdr ? 4 : 0;
      body_end[s] = sg.len - 4;
      stored[s] = load_be32(d + body_end[s]);
      check_crc[s] = hdr && !(sg.flags & TEZGPU_SEG_VERIFIED);
      total += align_up(sg.len, 16);
    }
    // one step when the inputs fit with the worst case of one record per byte
    single = need(total + 64, total, total) <= budget;
    if (single) {
      m.open(segs, nseg);   // with the write codec: what tezgpu_merge_open_codec does with uncompressed segments
      steps = 1;
      h2d = total;
      have_counts = true;
      total_n = m.n;
      total_kv = m.kv_bytes;
      in.clear();
      return;
    }
    TG_CHECK(budget > fixed_bytes() + STEP_BYTES_PER_WINDOW_BYTE * STEP_MIN_SHARE * nseg, TEZGPU_E_NOMEM,
             "device budget of " + std::to_string(budget) + " bytes is below the fixed workspace of " + std::to_string(nseg) +
                 " segments and " + std::to_string(m.pipe.conf.num_partitions) + " partitions");
    wtot0 = (budget - fixed_bytes()) / 2 / STEP_BYTES_PER_WINDOW_BYTE;
    pmajor.resize(nseg);
    for (uint32_t q = 0; q < nseg; q++) pmajor[q] = q;
    std::stable_sort(pmajor.begin(), pmajor.end(), [&](uint32_t a, uint32_t b) { return in[a].partition < in[b].partition; });
    d_bad.ensure(16);
    d_split.ensure(16);
    m.pipe.codec = TEZGPU_CODEC_NONE;   // the steps write uncompressed pieces; write compresses them
    // the first step runs here, as every other open parses its inputs before returning
    begin_pass();
    iter = 1;
    in_step = next_step();
    if (!in_step) iter = 2;
    if (std::all_of(finished.begin(), finished.end(), [](uint8_t f) { return f != 0; })) {
      // the first step took every record: the Merger holds the whole merge, as after a one-step open (the checksums
      // have been checked, the host segments are no longer read)
      single = true;
      m.pipe.codec = zcodec;
      end_pass();
      in.clear();
    }
  }

  void begin_pass() {
    const uint32_t nseg = (uint32_t)in.size();
    consumed = body0;
    finished.assign(nseg, 0);
    grow.assign(nseg, 0);
    wtot = wtot0;
    steps = 0;
    pass_n = pass_kv = 0;
    in_step = false;
    d_acc.ensure((size_t)std::max<uint32_t>(1, nseg) * 4);
    TG_CUDA(cudaMemsetAsync(d_acc.p, 0, (size_t)std::max<uint32_t>(1, nseg) * 4, m.pipe.stream));
    TG_CUDA(cudaMemsetAsync(d_bad.p, 0, 16, m.pipe.stream));
  }
  void end_pass() {
    have_counts = true;
    total_n = pass_n;
    total_kv = pass_kv;
  }

  // Lays out and uploads the windows of one step; returns their bytes.  The merge order is (partition, key), so only
  // the lowest unfinished partition can hold keys < S: its unfinished segments share the step's window bytes (a
  // segment whose key group outgrew its share keeps its grown window).  A later partition comes along only whole, and
  // only while every partition before it fit whole: no window of the step then ends before its segment does, and the
  // step takes them all.  Segments of later partitions are never uploaded ahead of their turn.
  uint64_t upload_windows() {
    cudaStream_t st = m.pipe.stream;
    wins.clear();
    win_seg.clear();
    uint64_t off = 0, bytes = 0;
    bool lead = true;
    std::vector<uint32_t> grp;
    for (size_t i = 0; i < pmajor.size();) {
      const uint32_t p = in[pmajor[i]].partition;
      grp.clear();
      uint64_t rest_sum = 0;
      for (; i < pmajor.size() && in[pmajor[i]].partition == p; i++) {
        const uint32_t s = pmajor[i];
        if (finished[s]) continue;
        grp.push_back(s);
        rest_sum += body_end[s] - consumed[s];
      }
      if (grp.empty()) continue;
      if (!lead && bytes + rest_sum > wtot) break;
      const uint64_t share = lead ? align_up(std::max<uint64_t>(STEP_MIN_SHARE, wtot / grp.size()), 16) : ~0ull;
      if (lead) n_lead = grp.size();
      bool whole = true;
      for (const uint32_t s : grp) {
        const uint64_t rest = body_end[s] - consumed[s];
        const uint64_t len = std::min(rest, std::max(share, grow[s]));
        StepWin w;
        w.off = off;
        w.len = len;
        w.at_end = len == rest;
        w.partition = in[s].partition;
        wins.push_back(w);
        win_seg.push_back(s);
        off = align_up(off + len + 6, 16);
        bytes += len;
        whole &= w.at_end != 0;
      }
      lead = false;
      if (!whole) break;
    }
    d_win.ensure(off + 16);
    for (size_t i = 0; i < wins.size(); i++) {
      const uint32_t s = win_seg[i];
      if (wins[i].len)
        TG_CUDA(cudaMemcpyAsync(d_win.as<uint8_t>() + wins[i].off, static_cast<const uint8_t *>(in[s].data) + consumed[s], wins[i].len, cudaMemcpyHostToDevice, st));
    }
    h2d += bytes;
    const size_t nw = std::max<size_t>(1, wins.size());
    d_wins.ensure(nw * sizeof(StepWin));
    d_scan.ensure(nw * sizeof(StepScan));
    d_cut.ensure(nw * sizeof(StepCut));
    d_on_split.ensure(nw);
    if (!wins.empty()) TG_CUDA(cudaMemcpyAsync(d_wins.p, wins.data(), wins.size() * sizeof(StepWin), cudaMemcpyHostToDevice, st));
    return bytes;
  }

  // Runs the next step: on return true, the Merger holds the step's merged records (possibly none).  false: every
  // segment is finished.
  bool next_step() {
    cudaStream_t st = m.pipe.stream;
    const int cmp = m.pipe.conf.comparator;
    while (true) {
      if (std::all_of(finished.begin(), finished.end(), [](uint8_t f) { return f != 0; })) return false;
      const uint64_t wbytes = upload_windows();
      const uint32_t nw = (uint32_t)wins.size();
      const uint32_t grid = (uint32_t)div_up(nw, PARSE_WARPS);
      k_step_walk<false><<<grid, PARSE_WARPS * 32, 0, st>>>(d_win.as<uint8_t>(), d_wins.as<StepWin>(), nw, cmp,
                                                            d_scan.as<StepScan>(), nullptr, nullptr);
      TG_CUDA(cudaGetLastError());
      scans.resize(nw);
      TG_CUDA(cudaMemcpyAsync(scans.data(), d_scan.p, nw * sizeof(StepScan), cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaStreamSynchronize(st));   // also: the host segments have been read
      uint64_t scan_n = 0, scan_kv = 0;
      bool stuck = false;
      for (uint32_t i = 0; i < nw; i++) {
        const uint32_t s = win_seg[i];
        TG_CHECK(!scans[i].bad, TEZGPU_E_FORMAT, "malformed IFile segment " + std::to_string(s));
        scan_n += scans[i].nrec;
        scan_kv += scans[i].kv;
        if (scans[i].nrec == 0 && !(scans[i].eof && wins[i].at_end)) {
          grow[s] = 2 * std::max(wins[i].len, (uint64_t)16);   // no complete record yet: the window must grow
          stuck = true;
        }
      }
      const uint64_t nd = need(std::max(max_w, wbytes), std::max(max_kv, scan_kv), std::max(max_n, scan_n));
      if (nd > budget) {
        if (wtot / n_lead > STEP_MIN_SHARE) {
          wtot = align_up(wtot / 2, 16);
          continue;
        }
        uint64_t held = 0;
        for (uint32_t i = 0; i < nw; i++) if (grow[win_seg[i]]) held += wins[i].len;   // the group's bytes seen so far
        TG_CHECK(false, TEZGPU_E_NOMEM, held ? "a key group of more than " + std::to_string(held) +
                                            " bytes does not fit the device budget of " + std::to_string(budget) + " bytes"
                                      : "the merge does not fit the device budget of " + std::to_string(budget) + " bytes");
      }
      if (stuck) continue;
      k_step_splitter<<<1, 32, 0, st>>>(d_win.as<uint8_t>(), d_wins.as<StepWin>(), nw, cmp, d_scan.as<StepScan>(),
                                        d_split.as<int32_t>(), d_on_split.as<uint8_t>());
      k_step_walk<true><<<grid, PARSE_WARPS * 32, 0, st>>>(d_win.as<uint8_t>(), d_wins.as<StepWin>(), nw, cmp,
                                                           d_scan.as<StepScan>(), d_split.as<int32_t>(), d_cut.as<StepCut>());
      TG_CUDA(cudaGetLastError());
      cuts.resize(nw);
      std::vector<uint8_t> on_split(nw);
      TG_CUDA(cudaMemcpyAsync(cuts.data(), d_cut.p, nw * sizeof(StepCut), cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaMemcpyAsync(on_split.data(), d_on_split.p, nw, cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaStreamSynchronize(st));
      uint64_t cut_n = 0;
      bool ends = false;
      for (uint32_t i = 0; i < nw; i++) {
        cut_n += cuts[i].nrec;
        ends |= scans[i].eof && wins[i].at_end && cuts[i].nrec == scans[i].nrec;
      }
      if (!cut_n && !ends) {
        // one key group is larger than the windows that hold it: grow them (the budget check above bounds them)
        for (uint32_t i = 0; i < nw; i++) if (on_split[i]) grow[win_seg[i]] = 2 * wins[i].len;
        continue;
      }
      run_step(wbytes);
      return true;
    }
  }

  // checksums of the consumed bytes, the EOF markers after the cuts, the Merger over the window prefixes
  void run_step(uint64_t wbytes) {
    cudaStream_t st = m.pipe.stream;
    const uint32_t nw = (uint32_t)wins.size();
    const CrcTables *d_crc = DeviceConstants::get(m.pipe.conf.device).d_crc;
    std::vector<uint64_t> take(nw);
    std::vector<uint8_t> ends(nw);
    for (uint32_t i = 0; i < nw; i++) {
      ends[i] = scans[i].eof && wins[i].at_end && cuts[i].nrec == scans[i].nrec;
      take[i] = ends[i] ? wins[i].len : cuts[i].bytes;
    }
    // ---- checksums: raw remainder of the consumed bytes of every checked window, folded per segment
    std::vector<SegDesc> cd;
    std::vector<StepCrcSeg> cs;
    for (uint32_t i = 0; i < nw; i++) {
      const uint32_t s = win_seg[i];
      if (!check_crc[s] || !take[i]) continue;
      SegDesc d;
      d.off = wins[i].off; d.len = take[i]; d.body0 = 0; d.body_end = take[i]; d.has_header = 1; d.partition = 0;
      cd.push_back(d);
      StepCrcSeg c;
      c.len = take[i]; c.total = body_end[s] - body0[s]; c.seg = s; c.stored = stored[s]; c.last = ends[i]; c.pad = 0;
      cs.push_back(c);
    }
    if (!cd.empty()) {
      const uint32_t nc = (uint32_t)cd.size();
      d_crcsd.ensure(nc * sizeof(SegDesc));
      d_crcseg.ensure(nc * sizeof(StepCrcSeg));
      TG_CUDA(cudaMemcpyAsync(d_crcsd.p, cd.data(), nc * sizeof(SegDesc), cudaMemcpyHostToDevice, st));
      TG_CUDA(cudaMemcpyAsync(d_crcseg.p, cs.data(), nc * sizeof(StepCrcSeg), cudaMemcpyHostToDevice, st));
      std::vector<uint32_t> piece_start;
      m.segment_remainders(d_win.as<uint8_t>(), cd, d_crcsd.as<SegDesc>(), [](const SegDesc &) { return true; }, piece_start, false);
      // (the m.open() below checks no checksum of its header-less segments, so d_seg_crc is not touched before the fold)
      k_step_crc_fold<<<(uint32_t)div_up(nc, 128), 128, 0, st>>>(m.d_seg_crc.as<uint32_t>(), d_crcseg.as<StepCrcSeg>(), nc, d_crc,
                                                                d_acc.as<uint32_t>(), d_bad.as<int>());
      TG_CUDA(cudaGetLastError());
      TG_CUDA(cudaStreamSynchronize(st));   // the host tables above live on this stack
    }
    // ---- the window prefixes as header-less device segments, merged in the caller's order
    k_step_terminate<<<(uint32_t)div_up(nw, 128), 128, 0, st>>>(d_win.as<uint8_t>(), d_wins.as<StepWin>(), d_cut.as<StepCut>(), nw);
    TG_CUDA(cudaGetLastError());
    std::vector<tezgpu_segment> ps;
    uint64_t step_kv = 0, step_n = 0;
    for (uint32_t i = 0; i < nw; i++) {
      const uint32_t s = win_seg[i];
      consumed[s] += take[i];
      finished[s] = ends[i];
      if (cuts[i].nrec) grow[s] = 0;
      step_n += cuts[i].nrec;
      step_kv += cuts[i].kv;
      if (!cuts[i].nrec) continue;
      tezgpu_segment sg;
      sg.data = d_win.as<uint8_t>() + wins[i].off;
      sg.len = cuts[i].bytes + 6;
      sg.flags = TEZGPU_SEG_DEVICE;
      sg.partition = wins[i].partition;
      ps.push_back(sg);
    }
    m.launches = 0;
    m.open(ps.data(), (uint32_t)ps.size());
    int bad = 0;
    TG_CUDA(cudaMemcpyAsync(&bad, d_bad.p, 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    TG_CHECK(bad == 0, TEZGPU_E_FORMAT, "IFile checksum mismatch in segment " + std::to_string(bad - 1));
    steps++;
    pass_n += m.n;
    pass_kv += m.kv_bytes;
    max_w = std::max(max_w, wbytes);
    max_n = std::max(max_n, step_n);
    max_kv = std::max(max_kv, step_kv);
    // windows grow back once a step needs less than a quarter of the budget
    if (wtot < wtot0 && need(max_w, max_kv, max_n) < budget / 4) wtot = std::min(wtot0, 2 * wtot);
  }

  // ---- record iterator across steps
  void next_batch(const BatchDest &d, uint64_t cap, uint32_t idx_cap, uint32_t *count) {
    TallyScope ts(&tally);
    *count = 0;
    if (d.kv_bytes) *d.kv_bytes = 0;
    TG_CHECK(!m.pipe.combiner, TEZGPU_E_STATE, "a merger with a combiner has no record iterator: use tezgpu_merge_write_*");
    if (idx_cap == 0 || iter == 2) return;
    if (iter == 0) {
      begin_pass();
      iter = 1;
    }
    while (true) {
      if (in_step && m.cursor < m.n) {
        m.next_batch(d, cap, idx_cap, count);
        if (*count) return;
      }
      in_step = next_step();
      if (!in_step) {
        iter = 2;
        end_pass();
        return;
      }
    }
  }

  // ---- writes (see the top of this file): the file and index the one-step merge with the write codec writes; out
  //      receives file.out, index the TezIndexRecord triples.  Every step that has records writes its uncompressed
  //      image behind STEP_CARRY_ROOM bytes of m.d_out and runs one pass over its pieces; one more pass after the last
  //      step closes what is left.
  struct StitchJob {
    uint32_t part;
    uint64_t off;       // the piece's own bytes in m.d_out (in the room, or in the step image behind it)
    uint64_t n;
    bool starts;        // the partition's first piece: the header in front of it
    bool closes;        // its last: the trailer after it
    bool bytes;         // false: a partition without records and without a segment (send_empty_partition_details 1)
  };

  void write(int rle, std::vector<uint8_t> &out, std::vector<int64_t> &index, tezgpu_stats *stats) {
    TallyScope ts(&tally);
    SortPipeline &pp = m.pipe;
    cudaStream_t st = pp.stream;
    const int P = pp.conf.num_partitions;
    const bool empty_segments = pp.conf.send_empty_partition_details == 0;   // as k_layout
    const bool zlib = zcodec == TEZGPU_CODEC_DEFAULT;
    const CodecLayout L = codec_layout(zcodec);   // with a codec only
    const CrcTables *d_crc = DeviceConstants::get(pp.conf.device).d_crc;
    static const uint8_t kEof[2] = {0xFF, 0xFF};
    const uint8_t head[6] = {'T', 'I', 'F', (uint8_t)(zcodec ? 1 : 0), 0x78, 0x01};
    const size_t head_len = zlib ? 6 : 4, trailer_len = zlib ? 8 : 4;   // zlib: 78 01; Adler-32 and CRC-32
    begin_pass();
    iter = 0;   // the windows are the write's now: a later next_batch starts from the beginning
    out.clear();
    index.assign((size_t)P * 3, 0);
    std::vector<uint64_t> raw((size_t)P, 0), slen((size_t)P, 0);   // per partition: record bytes, stream bytes
    std::vector<int64_t> at((size_t)P, 0);                          // file offset of its segment
    std::vector<uint32_t> acc((size_t)P * 2);                       // running CRC remainder and Adler-32 (k_stitch_fold)
    for (int p = 0; p < P; p++) { acc[2 * p] = 0; acc[2 * p + 1] = 1; }
    d_fold.ensure((size_t)P * 8);
    TG_CUDA(cudaMemcpyAsync(d_fold.p, acc.data(), (size_t)P * 8, cudaMemcpyHostToDevice, st));
    if (zcodec) d_carry.ensure(STEP_CARRY_ROOM);
    tezgpu_stats sum;
    memset(&sum, 0, sizeof(sum));
    int cur = -1;            // the last partition with records so far
    bool open = false;       // its segment continues in a later step
    uint64_t carry = 0;      // its body bytes after its last compressed chunk, in d_carry (always 0 without a codec)
    std::vector<StitchJob> jobs;
    std::vector<uint32_t> part;
    std::vector<uint32_t> seg_of;
    auto done = [&](uint32_t p) {   // every segment of partition p has been read to its end
      for (size_t s = 0; s < in.size(); s++)
        if (in[s].partition == p && !finished[s]) return false;
      return true;
    };
    auto close_open = [&] {   // the open partition has no records in this step: its carry and FF FF close it
      if (open) jobs.push_back({(uint32_t)cur, 2 + carry, 2, false, true, true});
      open = false;
    };
    auto skip_to = [&](int p) {   // partitions before p without records
      for (int q = cur + 1; q < p; q++) jobs.push_back({(uint32_t)q, 0, 2, true, true, empty_segments});
    };
    // one pass: the pieces of `jobs` compressed (plan_stitch_piece) or, without a codec, taken whole; their checksums
    // folded and their bytes appended to out
    auto pass = [&] {
      m.d_out.ensure(STEP_CARRY_ROOM);
      uint8_t *img = m.d_out.as<uint8_t>();
      pp.z_timer.reset();
      pp.z_timer.mark(st);
      int launches = 0;
      TG_CUDA(cudaMemcpyAsync(img, kEof, 2, cudaMemcpyHostToDevice, st));
      pp.z_host.ensure(jobs.size() * sizeof(ZSeg) + 64);
      ZSeg *hs = pp.z_host.as<ZSeg>();
      seg_of.assign(jobs.size(), ~0u);
      part.clear();
      uint32_t nseg = 0, nchunks = 0;
      uint64_t bytes = 0;   // the pass's bytes for h_pass
      for (size_t i = 0; i < jobs.size(); i++) {
        const StitchJob &j = jobs[i];
        if (!j.bytes) continue;
        const uint64_t c = j.starts ? 0 : carry;   // only the open partition continues
        if (c) TG_CUDA(cudaMemcpyAsync(img + j.off - c, d_carry.p, c, cudaMemcpyDeviceToDevice, st));
        if (j.off < STEP_CARRY_ROOM) TG_CUDA(cudaMemcpyAsync(img + j.off, kEof, 2, cudaMemcpyHostToDevice, st));
        ZSeg &s = hs[nseg];
        memset(&s, 0, sizeof(s));
        if (zcodec) {
          const StitchPlan pl = plan_stitch_piece(L.chunk, c, j.off, j.n, j.closes);
          if (pl.open) {
            carry = pl.carry;
            if (carry) TG_CUDA(cudaMemcpyAsync(d_carry.p, img + pl.off + pl.len, carry, cudaMemcpyDeviceToDevice, st));
          }
          if (!pl.nchunks) continue;
          s.body_off = pl.off;
          s.body_len = pl.len;
          s.chunk0 = nchunks;
          s.nchunks = pl.nchunks;
          s.open = pl.open;
          nchunks += pl.nchunks;
        } else {   // the piece whole: its bytes reach the host with the image
          s.body_off = s.zstart = j.off;
          s.zlen = j.n;
          s.open = !j.closes;
          bytes = std::max(bytes, j.off + j.n);
        }
        s.rank = nseg;
        seg_of[i] = nseg++;
        part.push_back(j.part);
      }
      if (nseg) {
        const uint8_t *src = img;
        if (zcodec) {
          bytes = pp.compress_chunks(zcodec, img, hs, nseg, nchunks, 0, 0, &launches);
          d_zout.ensure(bytes);
          k_zpack<<<nchunks, 256, 0, st>>>(pp.z_slots.as<uint8_t>(), pp.z_csize.as<uint32_t>(), pp.z_coff.as<uint64_t>(), pp.z_segs.as<ZSeg>(),
                                           nseg, L.slot, 0, d_zout.as<uint8_t>());
          src = d_zout.as<uint8_t>();
          launches++;
        } else {
          pp.z_segs.ensure((size_t)nseg * sizeof(ZSeg));
          TG_CUDA(cudaMemcpyAsync(pp.z_segs.p, hs, (size_t)nseg * sizeof(ZSeg), cudaMemcpyHostToDevice, st));
        }
        d_piece_part.ensure((size_t)nseg * 4);
        TG_CUDA(cudaMemcpyAsync(d_piece_part.p, part.data(), (size_t)nseg * 4, cudaMemcpyHostToDevice, st));
        k_stitch_fold<<<(uint32_t)div_up(nseg, 128), 128, 0, st>>>(pp.z_segs.as<ZSeg>(), d_piece_part.as<uint32_t>(), nseg,
                                                                   zcodec ? pp.z_crc.as<uint32_t>() : nullptr,
                                                                   zlib ? pp.z_cadler.as<uint32_t>() : nullptr, img, d_crc,
                                                                   d_fold.as<uint32_t>());
        launches++;
        TG_CUDA(cudaGetLastError());
        h_pass.ensure(bytes);
        TG_CUDA(cudaMemcpyAsync(h_pass.p, src, bytes, cudaMemcpyDeviceToHost, st));
      }
      pp.z_timer.mark(st);
      TG_CUDA(cudaStreamSynchronize(st));
      sum.ms_total += pp.z_timer.ms(0, 1);
      sum.kernel_launches += launches;
      for (size_t i = 0; i < jobs.size(); i++) {   // hs holds zstart / zlen of every piece with bytes in h_pass
        const StitchJob &j = jobs[i];
        const uint32_t p = j.part;
        if (!j.bytes) {
          index[3 * p] = (int64_t)out.size();
          continue;
        }
        if (j.starts) {
          at[p] = (int64_t)out.size();
          out.insert(out.end(), head, head + head_len);
        }
        if (seg_of[i] != ~0u) {
          const ZSeg &s = hs[seg_of[i]];
          const uint8_t *z = h_pass.as<uint8_t>() + s.zstart;
          out.insert(out.end(), z, z + s.zlen);
          slen[p] += s.zlen;
        }
        if (j.closes) {
          out.insert(out.end(), trailer_len, 0);   // from the folds below
          index[3 * p] = at[p];
          index[3 * p + 1] = (int64_t)raw[p] + 6;
          index[3 * p + 2] = (int64_t)out.size() - at[p];
        }
      }
      jobs.clear();
    };
    std::vector<int64_t> idx((size_t)P * 3);
    while ((in_step = next_step())) {
      if (!m.n) continue;
      m.d_out.ensure(STEP_CARRY_ROOM + m.output_bound());
      uint64_t len = 0;
      tezgpu_stats s;
      m.write_device(m.d_out.as<uint8_t>() + STEP_CARRY_ROOM, m.d_out.cap - STEP_CARRY_ROOM, rle, &len, idx.data(), &s);
      sum.output_records += s.output_records;
      sum.output_bytes += s.output_bytes;
      sum.spilled_records += s.spilled_records;
      sum.rle_used |= s.rle_used;
      sum.adjacent_equal_keys += s.adjacent_equal_keys;
      sum.tie_records += s.tie_records;
      sum.ms_stage += s.ms_stage; sum.ms_sort += s.ms_sort; sum.ms_ties += s.ms_ties; sum.ms_emit += s.ms_emit; sum.ms_total += s.ms_total;
      sum.kernel_launches += s.kernel_launches;
      for (int p = 0; p < P; p++) {
        const int64_t seglen = idx[3 * p + 2];
        if (seglen <= 10) continue;   // no records of p in this step
        const bool starts = p != cur;
        if (starts) {
          close_open();
          skip_to(p);
          cur = p;
        }
        const bool closes = done((uint32_t)p);
        const uint64_t body = (uint64_t)seglen - 10;
        jobs.push_back({(uint32_t)p, STEP_CARRY_ROOM + (uint64_t)idx[3 * p] + 4, body + (closes ? 2 : 0), starts, closes, true});
        raw[p] += body;
        open = !closes;
      }
      pass();
    }
    end_pass();
    close_open();
    skip_to(P);
    if (!jobs.empty()) pass();
    // ---- the trailers: CRC-32 of every segment's stream (and zlib's Adler-32) from the folded values
    d_stream_bytes.ensure((size_t)P * 8);
    d_trailer.ensure((size_t)P * 4);
    TG_CUDA(cudaMemcpyAsync(d_stream_bytes.p, slen.data(), (size_t)P * 8, cudaMemcpyHostToDevice, st));
    k_stitch_trailers<<<(uint32_t)div_up(P, 128), 128, 0, st>>>(d_fold.as<uint32_t>(), d_stream_bytes.as<uint64_t>(), (uint32_t)P,
                                                                 zlib ? 1 : 0, d_crc, d_trailer.as<uint32_t>());
    TG_CUDA(cudaGetLastError());
    std::vector<uint32_t> crc((size_t)P);
    TG_CUDA(cudaMemcpyAsync(acc.data(), d_fold.p, (size_t)P * 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaMemcpyAsync(crc.data(), d_trailer.p, (size_t)P * 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    for (int p = 0; p < P; p++) {
      if (!slen[p]) continue;
      uint8_t *e = out.data() + index[3 * p] + index[3 * p + 2];
      if (zlib) store_be32(e - 8, acc[2 * p + 1]);
      store_be32(e - 4, crc[p]);
    }
    for (int p = 0; p < P; p++) sum.output_bytes_with_overhead += index[3 * p + 1];
    sum.output_bytes_physical = sum.file_out_bytes = (int64_t)out.size();
    sum.num_spills = 1;
    sum.kernel_launches += 1;
    if (stats) *stats = sum;
  }
};

}  // namespace tezgpu

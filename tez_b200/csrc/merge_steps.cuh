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
// Writes stitch the pieces every step emits: TIF\0 only at the start of a partition, the FF FF EOF markers and the
// checksum only at its end; the checksum of a partition is folded from the trailers of its pieces (k_stitch_raw,
// k_crc_combine, k_stitch_finish), so the output is byte-identical to the one-step merge.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

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

// One piece = the records R one step wrote for one partition, between its TIF\0 header and its FF FF EOF markers.  Its
// trailer is crc(R || FF FF); with the identity of concat.cuh, raw(R || FF FF) = trailer ^ ~0 ^ (~0 * x^(8 len)), and
// raw(R || FF FF) ^ eof_raw = raw(R) * x^16, which k_crc_combine moves past the pieces after it in the partition.
struct StitchPiece {
  uint64_t body;        // bytes of R
  uint64_t after;       // bytes of the partition's pieces after this one
  uint32_t trailer;
  uint32_t partition;
};
__global__ void k_stitch_raw(const StitchPiece *__restrict__ pc, uint32_t n, const CrcTables *__restrict__ t,
                             TileCrc *__restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const StitchPiece c = pc[i];
  TileCrc tc;
  tc.raw = crc_to_raw(t, c.trailer, c.body + 2) ^ t->eof_raw;
  tc.p = c.partition;
  tc.after = c.after;
  out[i] = tc;
}
// checksum of every partition from the folded remainder of its records (0 without records) and their length
__global__ void k_stitch_finish(const uint32_t *__restrict__ part_raw, const uint64_t *__restrict__ part_body, uint32_t P,
                                const CrcTables *__restrict__ t, uint32_t *__restrict__ crc) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  crc[p] = crc_from_raw(t, part_raw[p] ^ t->eof_raw, part_body[p] + 2);
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
  DeviceBuffer d_pieces, d_piece_tc, d_part_raw, d_part_body, d_part_crc;
  std::vector<StepWin> wins;
  std::vector<uint32_t> win_seg;           // window -> caller's segment
  std::vector<StepScan> scans;
  std::vector<StepCut> cuts;

  BoundedMerge(Merger &mm, uint64_t b, DeviceTally &t) : m(mm), budget(b), tally(t) {}

  uint64_t fixed_bytes() const {
    return STEP_FIXED_BYTES + STEP_FIXED_PER_PARTITION * (uint64_t)m.pipe.conf.num_partitions +
           STEP_FIXED_PER_SEGMENT * (uint64_t)in.size();
  }
  uint64_t need(uint64_t w, uint64_t kv, uint64_t n) const {
    return STEP_BYTES_PER_WINDOW_BYTE * w + STEP_BYTES_PER_KV_BYTE * kv + STEP_BYTES_PER_RECORD * n + fixed_bytes();
  }

  void open(const tezgpu_segment *segs, uint32_t nseg) {
    TallyScope ts(&tally);
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
      m.open(segs, nseg);
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
    // the first step runs here, as every other open parses its inputs before returning
    begin_pass();
    iter = 1;
    in_step = next_step();
    if (!in_step) iter = 2;
    if (std::all_of(finished.begin(), finished.end(), [](uint8_t f) { return f != 0; })) {
      // the first step took every record: the Merger holds the whole merge, as after a one-step open (the checksums
      // have been checked, the host segments are no longer read)
      single = true;
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

  // ---- writes: every step's pieces stitched into one segment per partition.  out receives file.out, index the
  //      TezIndexRecord triples.
  void write(int rle, std::vector<uint8_t> &out, std::vector<int64_t> &index, tezgpu_stats *stats) {
    TallyScope ts(&tally);
    cudaStream_t st = m.pipe.stream;
    const int P = m.pipe.conf.num_partitions;
    const bool empty_segments = m.pipe.conf.send_empty_partition_details == 0;   // as k_layout
    static const uint8_t kHeader[4] = {'T', 'I', 'F', 0};
    begin_pass();
    iter = 0;   // the windows are the write's now: a later next_batch starts from the beginning
    out.clear();
    index.assign((size_t)P * 3, 0);
    std::vector<StitchPiece> pieces;
    std::vector<uint64_t> part_body((size_t)P, 0);
    std::vector<int64_t> part_at((size_t)P, -1);
    tezgpu_stats sum;
    memset(&sum, 0, sizeof(sum));
    int cur = -1;
    auto close_partition = [&](int p) {
      const uint8_t eof[6] = {0xFF, 0xFF, 0, 0, 0, 0};
      out.insert(out.end(), eof, eof + 6);
      index[3 * p + 0] = part_at[p];
      index[3 * p + 2] = (int64_t)out.size() - part_at[p];
      index[3 * p + 1] = index[3 * p + 2] - 4;
    };
    auto skip_to = [&](int p) {   // partitions before p without records
      for (int q = cur + 1; q < p; q++) {
        part_at[q] = (int64_t)out.size();
        index[3 * q] = part_at[q];
        if (!empty_segments) continue;
        out.insert(out.end(), kHeader, kHeader + 4);
        close_partition(q);
      }
    };
    std::vector<int64_t> idx((size_t)P * 3);
    while ((in_step = next_step())) {
      if (!m.n) continue;
      uint64_t len = 0;
      tezgpu_stats s;
      const uint8_t *img = m.write_host(rle, nullptr, 0, &len, idx.data(), &s);
      for (int p = 0; p < P; p++) {
        const int64_t seglen = idx[3 * p + 2];
        if (seglen <= 10) continue;   // no records of p in this step
        const uint8_t *seg = img + idx[3 * p];
        if (p != cur) {
          if (cur >= 0) close_partition(cur);
          skip_to(p);
          cur = p;
          part_at[p] = (int64_t)out.size();
          out.insert(out.end(), seg, seg + 4);
        }
        const uint64_t body = (uint64_t)seglen - 10;
        out.insert(out.end(), seg + 4, seg + 4 + body);
        StitchPiece pc;
        pc.body = body;
        pc.after = 0;
        pc.trailer = load_be32(seg + seglen - 4);
        pc.partition = (uint32_t)p;
        pieces.push_back(pc);
        part_body[p] += body;
      }
      sum.output_records += s.output_records;
      sum.output_bytes += s.output_bytes;
      sum.spilled_records += s.spilled_records;
      sum.rle_used |= s.rle_used;
      sum.adjacent_equal_keys += s.adjacent_equal_keys;
      sum.tie_records += s.tie_records;
      sum.ms_stage += s.ms_stage; sum.ms_sort += s.ms_sort; sum.ms_ties += s.ms_ties; sum.ms_emit += s.ms_emit; sum.ms_total += s.ms_total;
      sum.kernel_launches += s.kernel_launches;
    }
    end_pass();
    if (cur >= 0) close_partition(cur);
    skip_to(P);
    // ---- the checksum of every partition from the trailers of its pieces
    for (size_t i = pieces.size(); i-- > 0;) {
      if (i + 1 < pieces.size() && pieces[i + 1].partition == pieces[i].partition)
        pieces[i].after = pieces[i + 1].after + pieces[i + 1].body;
    }
    const CrcTables *d_crc = DeviceConstants::get(m.pipe.conf.device).d_crc;
    const uint32_t npc = (uint32_t)pieces.size();
    d_pieces.ensure(std::max<size_t>(1, npc) * sizeof(StitchPiece));
    d_piece_tc.ensure(std::max<size_t>(1, npc) * sizeof(TileCrc));
    d_part_raw.ensure((size_t)P * 4);
    d_part_body.ensure((size_t)P * 8);
    d_part_crc.ensure((size_t)P * 4);
    TG_CUDA(cudaMemsetAsync(d_part_raw.p, 0, (size_t)P * 4, st));
    TG_CUDA(cudaMemcpyAsync(d_part_body.p, part_body.data(), (size_t)P * 8, cudaMemcpyHostToDevice, st));
    if (npc) {
      TG_CUDA(cudaMemcpyAsync(d_pieces.p, pieces.data(), npc * sizeof(StitchPiece), cudaMemcpyHostToDevice, st));
      k_stitch_raw<<<(uint32_t)div_up(npc, 128), 128, 0, st>>>(d_pieces.as<StitchPiece>(), npc, d_crc, d_piece_tc.as<TileCrc>());
      k_crc_combine<<<(uint32_t)div_up(npc, 256), 256, 0, st>>>(d_piece_tc.as<TileCrc>(), npc, d_crc, d_part_raw.as<uint32_t>());
    }
    k_stitch_finish<<<(uint32_t)div_up(P, 128), 128, 0, st>>>(d_part_raw.as<uint32_t>(), d_part_body.as<uint64_t>(), (uint32_t)P,
                                                               d_crc, d_part_crc.as<uint32_t>());
    TG_CUDA(cudaGetLastError());
    std::vector<uint32_t> crc((size_t)P);
    TG_CUDA(cudaMemcpyAsync(crc.data(), d_part_crc.p, (size_t)P * 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    for (int p = 0; p < P; p++)
      if (index[3 * p + 2]) store_be32(out.data() + index[3 * p] + index[3 * p + 2] - 4, crc[p]);
    for (int p = 0; p < P; p++) sum.output_bytes_with_overhead += index[3 * p + 1];
    sum.output_bytes_physical = sum.file_out_bytes = (int64_t)out.size();
    sum.num_spills = 1;
    if (stats) *stats = sum;
  }
};

}  // namespace tezgpu

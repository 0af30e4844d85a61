// parse_windows.cuh -- parallel IFile parser for the reduce side (IFile.Reader semantics, SORT/IFile.java:877-1000).
//
// An IFile body is a chain: the position of record i+1 is only known once the vint lengths of record i are decoded,
// and the format has no sync markers.  The walker of merger.cuh follows that chain with ONE lane per segment
// (2.7 M dependent steps for a 64 MiB segment of 25-byte records).  Here every segment body is cut into windows of
// PW_WINDOW bytes that are walked at the same time:
//
//   1. guess    (k_parse_guess)       every window guesses where the reader LEAVES it without knowing where it enters
//                                      (k_parse_guess below); the guess of window w is the presumed entry of window w+1.
//   2. evaluate (k_parse_windows<1>)  every window is walked from its presumed entry: record count, last full key,
//                                      exit.  If the presumed entry is the true one, so are these.
//   3. chase    (k_parse_chase)       one warp per segment follows the TRUE chain from the body start: window after
//                                      window, "my entry equals the presumed entry" means the stored evaluation is the
//                                      sequential reader's (32 windows are compared per step); where it is not -- a
//                                      wrong guess, a few per thousand windows -- lane 0 walks that one window from
//                                      the true entry and the chase goes on with its exit.
//   4. emit     (k_parse_windows<2>)  entries are final; every window writes its records' metadata.
//
// EXACTNESS rests on step 3 alone: the chase reproduces the sequential reader by induction from the first window; the
// guesses only decide how many windows it has to walk by hand (all of them in the worst case, which is the sequential
// walker's cost).  A malformed record, EOF markers before the body's end or a body that does not end with them makes
// the chase give up and the merger takes the sequential walker, which reports the error the way IFile.Reader does.
//
// An earlier version iterated entry_{t+1}[w+1] = exit(walk from entry_t[w]) to a fixed point.  On word-count data a
// wrong guess starts a walk in the "previous record was a repeat" state that reads every byte it lands on as a value
// length, hops on without ever meeting the true chain or dying, and is handed from window to window one round at a
// time, forever ahead of the correction behind it: the iteration did not converge within any useful number of rounds.
//
// Cost: guess = one or two rounds of 32 concurrent candidate walks per window (a warp; most die at once, the survivors
// share their loads), evaluate 1 walk, emit 1 walk; chase ~(#windows / 32) steps per segment + the hand-walked windows.
#pragma once
#include "ifile_walk.cuh"

namespace tezgpu {

struct SegDesc;  // merger.cuh

constexpr uint32_t PW_WINDOW = 32768;
constexpr uint32_t PW_MAX_TRIES = 8192;   // candidate start offsets per window in the guess round (covers records up to 8 KiB)
constexpr int PW_THREADS = 128;
constexpr uint64_t PW_EOF = ~0ull;        // the reader met the EOF markers before this window
constexpr uint64_t PW_BAD = ~0ull - 1;    // the walk that produced this entry met a malformed record
constexpr uint32_t PW_TAIL = 2048;         // k_parse_guess looks for agreeing candidates in a window's last bytes first
constexpr uint32_t PW_TAIL_TRIES = 512;    // candidate offsets tried there
constexpr uint32_t PW_TAIL_MIN_RECS = 24;  // ... and the records a candidate walk must cover to count
constexpr uint32_t PW_ALT_WAIT = 4;        // rounds a strong exit that is not a plain-state agreement waits for one
constexpr uint32_t PW_STRONG = 6;          // records a candidate walk must cover for its exit to count as strong evidence
constexpr uint32_t PW_EMIT_GROUP = 8;      // lanes that walk one window together in the metadata pass (power of two)
constexpr int PW_GUESS_THREADS = 128;      // k_parse_guess: four windows per CTA, one warp each
constexpr int PW_CHASE_WARPS = 4;          // segments per CTA of k_parse_chase

struct PwSeg {
  uint64_t off;        // segment start in the data buffer
  uint64_t len;        // segment bytes
  uint64_t body0;      // first body byte (4 with header, 0 in-memory)
  uint64_t body_end;   // len - 4
  uint32_t win0;       // first window of the segment in the global window list
  uint32_t nwin;
  uint32_t partition;
  uint32_t pad;
};

// segment of window w: last s with segs[s].win0 <= w (segments are listed in window order; every segment has >= 1 window)
__device__ __forceinline__ uint32_t pw_seg_of(const PwSeg *__restrict__ segs, uint32_t nseg, uint32_t w) {
  uint32_t lo = 0, hi = nseg;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(&segs[mid].win0) <= w) lo = mid; else hi = mid;
  }
  return lo;
}

// per-segment record counts from the per-window offsets: counts[s] = wbase[win0 + nwin] - wbase[win0]
__global__ void k_parse_seg_counts(const PwSeg *__restrict__ segs, uint32_t nseg, const uint64_t *__restrict__ wbase,
                                   uint64_t *__restrict__ counts) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nseg) counts[s] = wbase[segs[s].win0 + segs[s].nwin] - wbase[segs[s].win0];
}

struct ParseArrays {
  uint64_t *key_off;
  uint64_t *val_off;
  uint32_t *key_len;
  uint32_t *val_len;
  uint32_t *tag;  // (segment << 1) | read as SAME_KEY (run-length encoded in the input)
  int32_t *partition;
};

struct PwWalk {
  uint64_t exit_v;      // (pos << 1) | state on leaving the window, PW_EOF, PW_BAD
  uint32_t n;           // records that start in the window
  uint64_t lk_off, lk_len;  // last full key seen (segment offset, length); lk_off = ~0 when none
  uint64_t bytes;       // EMIT: key + value bytes
  bool early_eof;       // the EOF markers were met before the last two bytes of the body
};

// the sequential reader over one window, from entry e
// EMIT: PW_EMIT_GROUP lanes walk the SAME window from the same entry (identical control flow, broadcast loads) and lane
// (record number mod PW_EMIT_GROUP) writes that record's metadata: consecutive records go out from consecutive lanes
// within a few iterations, so every 32-byte sector of the six output arrays is completed while it is still in L2.
// One THREAD per window keeps 483 k windows x 6 arrays = 2.9 M concurrent write streams open at config 3 -- 370 MB of
// partial cache lines, more than the L2; a whole warp per window avoids that but issues every walk instruction once
// per window instead of once per 32 windows.  Groups of eight lanes keep four windows per warp and ~230 k open lines
// (29 MB).
template <bool EMIT>
__device__ __forceinline__ PwWalk pw_walk(const uint8_t *__restrict__ seg, const PwSeg &sd, uint32_t s, uint64_t wend, bool last_win,
                                          uint64_t e, uint64_t base, uint64_t carry_off, uint64_t carry_len, const ParseArrays &out,
                                          uint32_t lane = 0) {  // lane: position inside the emit group
  PwWalk r;
  r.exit_v = e;
  r.n = 0;
  r.lk_off = ~0ull;
  r.lk_len = 0;
  r.bytes = 0;
  r.early_eof = false;
  if (e == PW_EOF || e == PW_BAD) return r;
  uint64_t pos = e >> 1;
  int state = (int)(e & 1u);        // 1: the previous record was a repeat
  // the key a repeat at the start of this window refers to: the last full key before the window (a window may begin
  // inside a run-length encoded run, or with the run's RLE marker right after the key)
  uint64_t orig_koff = carry_off, orig_klen = carry_len;
  bool have_key = EMIT && carry_off != ~0ull;
  int status = 0;                   // 0 running, 1 EOF, 2 malformed
  // records that START inside this window belong to it; the last window also owns whatever lies up to the body end
  while (pos < wend || last_win) {
    RecHdr h;
    const int d = decode_header(GlobalVlong{seg, sd.len, sd.body_end}, state == 1, pos, h);
    if (d == REC_EOF) { status = 1; r.early_eof = h.pos != sd.body_end; break; }
    if (d != REC_OK) { status = 2; break; }
    const int64_t kl = h.kl, vl = h.vl;
    uint64_t q = h.pos;
    if (kl != -2) {
      if (q + (uint64_t)kl > sd.body_end) { status = 2; break; }
      orig_koff = q;
      orig_klen = (uint64_t)kl;
      have_key = true;
      r.lk_off = q;
      r.lk_len = (uint64_t)kl;
      q += (uint64_t)kl;
    } else if (EMIT && !have_key) { status = 2; break; }                // a repeat needs a previous key
    if (q + (uint64_t)vl > sd.body_end) { status = 2; break; }
    if (EMIT) {
      const uint64_t rr = base + r.n;
      if (((uint32_t)rr & (PW_EMIT_GROUP - 1u)) == lane) {
        out.key_off[rr] = sd.off + orig_koff;
        out.val_off[rr] = sd.off + q;
        out.key_len[rr] = (uint32_t)orig_klen;
        out.val_len[rr] = (uint32_t)vl;
        out.tag[rr] = (s << 1) | (kl == -2 ? 1u : 0u);
        out.partition[rr] = (int32_t)sd.partition;
        r.bytes += orig_klen + (uint64_t)vl;
      }
    }
    r.n++;
    pos = q + (uint64_t)vl;
    state = (kl == -2) ? 1 : 0;
  }
  if (status == 1) r.exit_v = PW_EOF;
  else if (status == 2) r.exit_v = PW_BAD;
  else r.exit_v = (pos << 1) | (uint64_t)state;
  return r;
}

// When the caller declared fixed key / value lengths (tezgpu_conf.fixed_*_len) but the segments could not be addressed
// in place (run-length encoded inputs), the first bytes of a record are one of four known patterns.  The guess tests a
// candidate start against them before walking it: garbage starts (multi-KB values are mostly garbage starts) cost two
// compares instead of a walk of divergent lanes.  A hint only -- a wrong guess costs time, never correctness.
struct PwFixedHint {
  uint64_t full;      // vint(klen) vint(vlen), little endian in the low full_len bytes
  uint64_t rep;       // vint(vlen)
  uint32_t full_len, rep_len;   // 0 = no hint
  __device__ __forceinline__ static bool starts_with(uint64_t x, uint64_t pat, uint32_t len) {
    return len >= 8 ? x == pat : ((x ^ pat) & ((1ull << (8 * len)) - 1ull)) == 0;
  }
  // x = the 8 bytes at the candidate start; state 1 = the previous record was a repeat
  __device__ __forceinline__ bool plausible(uint64_t x, uint32_t state) const {
    if (full_len == 0) return true;
    const uint32_t b0 = (uint32_t)(x & 0xFF);
    if (state == 0)   // key length + value length, or RLE_MARKER (0xFE = vint -2) + value length
      return starts_with(x, full, full_len) || (b0 == 0xFEu && starts_with(x >> 8, rep, rep_len));
    // repeat state: value length, or V_END_MARKER (0xFD = vint -3) + key length + value length
    return starts_with(x, rep, rep_len) || (b0 == 0xFDu && starts_with(x >> 8, full, full_len));
  }
};

// Guess of a window's exit without knowing its entry (k_parse_guess, one WARP per window): candidate starts ws, ws+1,
// ... in both reader states are walked to the window's end, 32 candidates at a time (lane l: offset l/2, state l&1).
// Almost every wrong start dies within a few records (a byte decoded as a negative or absurd length); one that
// survives usually fell into step with the true chain (two walks are identical from the first (position, state) they
// share) and so reports the true exit.  The exceptions are flukes that decode a large length and "survive" by jumping
// out of the window, and walks in the "previous record was a repeat" state, which read every byte they land on as a
// value length and hop on for a long time (on word-count data, taking the first survivor guesses wrong for a few
// percent of the windows).  Hence:
//   * EOF markers count only where a well-formed body has them (its last two bytes);
//   * an exit beyond the NEXT window is only the fallback (records longer than a window are rare; when they exist every
//     walk on the true chain reports the same far exit and the fallback is right);
//   * exits are ranked by evidence (agreement of two candidates, reader state, records covered; see the kernel).
//     CPU emulation of these rules, wrong guesses per windows tested: word-count text 0/60, long run-length encoded
//     runs of small records 0/60, 80-byte binary records 0/60, 4 KB values of one hot key (encoded run) 0/36, Zipf-like
//     mix of encoded 4 KB records 0/22, unique 4 KB random-byte values 3/36.
// Exactness never rests on any of this (k_parse_chase) -- only the number of windows walked a second time does.
__global__ void __launch_bounds__(PW_GUESS_THREADS)
    k_parse_guess(const uint8_t *__restrict__ data, const PwSeg *__restrict__ segs, uint32_t nseg, uint32_t nwin_total,
                  uint64_t *__restrict__ entry_out, PwFixedHint hint) {
  const uint32_t w = (blockIdx.x * PW_GUESS_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= nwin_total) return;
  const uint32_t s = pw_seg_of(segs, nseg, w);
  const PwSeg sd = segs[s];
  const uint8_t *__restrict__ seg = data + sd.off;
  const uint32_t k = w - sd.win0;
  const uint64_t ws = sd.body0 + (uint64_t)k * PW_WINDOW;
  const uint64_t wend = min(sd.body_end, ws + PW_WINDOW);
  const bool last_win = (k + 1 == sd.nwin);
  ParseArrays none{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  if (k == 0 && lane == 0) entry_out[w] = sd.body0 << 1;
  if (last_win) return;                       // nobody to hand an exit to
  if (k == 0) {                               // the first window's entry is known: its exit is exact
    if (lane == 0) entry_out[w + 1] = pw_walk<false>(seg, sd, s, wend, false, sd.body0 << 1, 0, ~0ull, 0, none).exit_v;
    return;
  }
  uint64_t far = PW_BAD, seen0 = PW_BAD, seen1 = PW_BAD, seen2 = PW_BAD, result = PW_BAD, alt = PW_BAD, weak = PW_BAD;
  uint32_t round = 0, alt_round = 0, alt_n = 0, weak_n = 0;
  bool done = false;
  // Phase A: candidates in the window's last PW_TAIL bytes -- a walk that falls into step with the true chain there
  // reaches the window's end after a few dozen records instead of a thousand; only walks of >= PW_TAIL_MIN_RECS records
  // count (a start inside the last records "survives" by a single hop).  Phase B (when A found nothing: records of a
  // hundred bytes and more, long encoded runs): candidates from the window's start, as far as PW_MAX_TRIES.
  const uint64_t tail0 = wend - ws > PW_TAIL ? wend - PW_TAIL : ws;
  const uint32_t tries_a = tail0 > ws ? PW_TAIL_TRIES : 0u;
  for (uint32_t t = 0; t < tries_a + PW_MAX_TRIES && !done; t += 16, round++) {
    const bool phase_a = t < tries_a;
    const uint64_t base = phase_a ? tail0 + t : ws + (t - tries_a);
    if (base >= wend) {
      if (!phase_a) break;
      t = tries_a - 16;          // the tail is exhausted: on to phase B
      continue;
    }
    const uint64_t start = base + (lane >> 1);
    uint64_t x = PW_BAD;
    uint32_t nrec = 0;
    if (start < wend && hint.plausible(pw_load8(seg, start, sd.len), lane & 1u)) {
      const PwWalk r = pw_walk<false>(seg, sd, s, wend, false, (start << 1) | (uint64_t)(lane & 1u), 0, ~0ull, 0, none);
      nrec = r.n;
      x = (r.early_eof || r.n < (phase_a ? PW_TAIL_MIN_RECS : 2u)) ? PW_BAD : r.exit_v;
      if (x == PW_EOF) x = PW_BAD;            // EOF inside a window that is not the last one
    }
    __syncwarp();
    const bool is_far = x != PW_BAD && (x >> 1) >= wend + PW_WINDOW;
    const bool near = x != PW_BAD && !is_far;
    const uint32_t fm = __ballot_sync(0xffffffffu, is_far);
    if (far == PW_BAD && fm) far = __shfl_sync(0xffffffffu, x, __ffs((int)fm) - 1);
    const uint32_t nm = __ballot_sync(0xffffffffu, near);
    if (nm) {
      bool agreed = false;
      if (near) agreed = __popc(__match_any_sync(nm, x)) + ((x == seen0 || x == seen1 || x == seen2) ? 1 : 0) >= 2;
      // The evidence for an exit: how many candidates report it, in which reader state, and how many records the walk
      // covered (in random bytes a wrong walk of k records has probability ~0.3^k; in text every byte is a plausible
      // length, but there the true chain is found at once).
      //   strong (>= PW_STRONG records) + agreed + plain state        -> taken at once
      //   strong otherwise (agreed in the repeat state, or alone)    -> best of them taken PW_ALT_WAIT rounds later
      //   weak agreed                                                -> only if nothing strong turns up at all
      const bool strong = near && nrec >= PW_STRONG;
      const uint32_t am0 = __ballot_sync(0xffffffffu, strong && agreed && (x & 1ull) == 0);
      if (am0) {
        result = __shfl_sync(0xffffffffu, x, __ffs((int)am0) - 1);
        done = true;
      } else {
        const uint32_t ks = __reduce_max_sync(0xffffffffu, strong ? ((min(nrec, 0x3FFFFFFu) << 5) | (31u - lane)) : 0u);
        if (ks && (ks >> 5) > alt_n) {
          if (alt == PW_BAD) alt_round = round;
          alt = __shfl_sync(0xffffffffu, x, 31 - (int)(ks & 31u));
          alt_n = ks >> 5;
        }
        const uint32_t kw = __reduce_max_sync(0xffffffffu, (near && agreed && !strong) ? ((nrec << 5) | (31u - lane)) : 0u);
        if (kw && (kw >> 5) > weak_n) {
          weak = __shfl_sync(0xffffffffu, x, 31 - (int)(kw & 31u));
          weak_n = kw >> 5;
        }
        for (uint32_t m = nm; m && seen2 == PW_BAD; m &= m - 1) {   // remember up to three lone survivors
          const uint64_t v = __shfl_sync(0xffffffffu, x, __ffs((int)m) - 1);
          if (v == seen0 || v == seen1) continue;
          if (seen0 == PW_BAD) seen0 = v;
          else if (seen1 == PW_BAD) seen1 = v;
          else seen2 = v;
        }
      }
    }
    if (!done && alt != PW_BAD && round >= alt_round + PW_ALT_WAIT) {
      result = alt;
      done = true;
    }
  }
  if (!done) result = alt != PW_BAD ? alt : (weak != PW_BAD ? weak : (seen0 != PW_BAD ? seen0 : far));
  if (lane == 0) entry_out[w + 1] = result;
}

//   MODE 1  evaluate (one thread per window): walks from the presumed entry; stores the exit, the record count and the
//           last full key.
//   MODE 2  emit (PW_EMIT_GROUP lanes per window, see pw_walk): entries are final (k_parse_chase); writes the per-record
//           metadata at rec_base[w]...
template <int MODE>
__global__ void __launch_bounds__(PW_THREADS)
    k_parse_windows(const uint8_t *__restrict__ data, const PwSeg *__restrict__ segs, uint32_t nseg,
                    uint32_t nwin_total, const uint64_t *__restrict__ entry_in, uint64_t *__restrict__ entry_out,
                    uint32_t *__restrict__ wcount, uint64_t *__restrict__ wlastkey /*[2*nwin]: off, len*/,
                    unsigned long long *__restrict__ kv_total, int *__restrict__ flags /*[0] changed, [1] bad*/,
                    const uint64_t *__restrict__ rec_base, const uint64_t *__restrict__ carry /*[2*nwin]*/, ParseArrays out) {
  constexpr bool EMIT = MODE == 2;
  const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t w = EMIT ? gt / PW_EMIT_GROUP : gt, lane = threadIdx.x & (PW_EMIT_GROUP - 1u);
  uint64_t my_bytes = 0;
  if (w < nwin_total) {
    const uint32_t s = pw_seg_of(segs, nseg, w);
    const PwSeg sd = segs[s];
    const uint8_t *__restrict__ seg = data + sd.off;
    const uint32_t k = w - sd.win0;
    const uint64_t ws = sd.body0 + (uint64_t)k * PW_WINDOW;
    const uint64_t wend = min(sd.body_end, ws + PW_WINDOW);
    const bool last_win = (k + 1 == sd.nwin);
    const uint64_t e = (k == 0) ? (sd.body0 << 1) : entry_in[w];
    const PwWalk r = pw_walk<EMIT>(seg, sd, s, wend, last_win, e, EMIT ? rec_base[w] : 0, EMIT ? carry[2 * (uint64_t)w] : ~0ull,
                                   EMIT ? carry[2 * (uint64_t)w + 1] : 0, out, lane);
    if (MODE == 1) {
      wcount[w] = r.n;
      wlastkey[2 * (uint64_t)w] = r.lk_off;
      wlastkey[2 * (uint64_t)w + 1] = r.lk_len;
      // a walk that met a malformed record, or EOF markers anywhere but at the end of the last window, is recorded as
      // dead: if its entry turns out to be the true one the chase reports the segment, otherwise it is walked again
      const bool dead = r.exit_v == PW_BAD || r.early_eof || (last_win ? r.exit_v != PW_EOF : r.exit_v == PW_EOF);
      entry_out[w] = dead ? PW_BAD : r.exit_v;   // MODE 1: entry_out = exit of every window
    } else {
      if (r.exit_v == PW_BAD) atomicMax(flags + 1, (int)s + 1);
      my_bytes = r.bytes;
    }
  }
  if (EMIT) {
    // key + value bytes of the merged stream: warp-reduce, one atomic per warp
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) my_bytes += __shfl_xor_sync(0xffffffffu, my_bytes, o);
    if ((threadIdx.x & 31) == 0 && my_bytes) atomicAdd(kv_total, (unsigned long long)my_bytes);
  }
}

// Follows the true chain of every segment through the evaluated windows (one warp per segment).
//   entry[w]  in: presumed entry of window w (guess), out: true entry
//   wexit[w]  exit of the walk from entry[w]; wcount / wlastkey likewise -- rewritten for hand-walked windows
//   flags[1]  segment + 1 of a segment the sequential reader would reject (or that ends early): caller falls back
//   flags[2]  number of windows walked by hand (diagnostics)
__global__ void __launch_bounds__(32 * PW_CHASE_WARPS)
    k_parse_chase(const uint8_t *__restrict__ data, const PwSeg *__restrict__ segs, uint32_t nseg, uint64_t *__restrict__ entry,
                  uint64_t *__restrict__ wexit, uint32_t *__restrict__ wcount, uint64_t *__restrict__ wlastkey, int *__restrict__ flags) {
  const uint32_t s = blockIdx.x * PW_CHASE_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (s >= nseg) return;
  const PwSeg sd = segs[s];
  const uint8_t *__restrict__ seg = data + sd.off;
  ParseArrays none{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  uint64_t e = sd.body0 << 1;   // true entry of window k
  uint32_t k = 0, by_hand = 0;
  bool bad = false;
  while (k < sd.nwin && !bad) {
    const uint32_t w = sd.win0 + k + lane;
    const bool in = k + lane < sd.nwin;
    const uint64_t eg = in ? entry[w] : PW_BAD;
    const uint64_t x = in ? wexit[w] : PW_BAD;
    // lane i: window k+i hands its exit to window k+i+1 unchanged (the last window has nobody to hand to)
    uint64_t eg_next = __shfl_down_sync(0xffffffffu, eg, 1);
    if (lane == 31) eg_next = (k + 32 < sd.nwin) ? entry[w + 1] : PW_BAD;
    const bool is_last = in && (k + lane + 1 == sd.nwin);
    const bool alive = in && x != PW_BAD;
    const bool hands_on = alive && !is_last && x == eg_next;
    const uint64_t eg0 = __shfl_sync(0xffffffffu, eg, 0);
    if (e == eg0) {
      // the stored evaluations are the reader's for windows k .. k+i, i = first lane that does not hand on
      const uint32_t stop = __ballot_sync(0xffffffffu, !hands_on);
      if (stop == 0) {                          // all 32 windows hand on: the chain enters window k+32 as guessed
        e = __shfl_sync(0xffffffffu, x, 31);
        k += 32;
        continue;
      }
      const int i = __ffs((int)stop) - 1;
      const bool alive_i = __shfl_sync(0xffffffffu, (int)alive, i) != 0;
      const bool last_i = __shfl_sync(0xffffffffu, (int)is_last, i) != 0;
      const uint64_t x_i = __shfl_sync(0xffffffffu, x, i);
      if (!alive_i) { bad = true; break; }      // the reader itself meets the malformed record / misplaced EOF
      if (last_i) { k = sd.nwin; break; }       // reached the end of the body (exit == EOF, checked when evaluated)
      e = x_i;
      k += (uint32_t)i + 1;
    } else {
      // wrong guess: lane 0 walks window k from the true entry
      uint64_t xe = PW_BAD;
      if (lane == 0) {
        const uint64_t ws = sd.body0 + (uint64_t)k * PW_WINDOW;
        const uint64_t wend = min(sd.body_end, ws + PW_WINDOW);
        const bool last_win = (k + 1 == sd.nwin);
        const PwWalk r = pw_walk<false>(seg, sd, s, wend, last_win, e, 0, ~0ull, 0, none);
        const bool dead = r.exit_v == PW_BAD || r.early_eof || (last_win ? r.exit_v != PW_EOF : r.exit_v == PW_EOF);
        const uint32_t w0 = sd.win0 + k;
        entry[w0] = e;
        wexit[w0] = dead ? PW_BAD : r.exit_v;
        wcount[w0] = r.n;
        wlastkey[2 * (uint64_t)w0] = r.lk_off;
        wlastkey[2 * (uint64_t)w0 + 1] = r.lk_len;
        xe = dead ? PW_BAD : r.exit_v;
      }
      xe = __shfl_sync(0xffffffffu, xe, 0);
      by_hand++;
      if (xe == PW_BAD) { bad = true; break; }
      e = xe;
      k++;
    }
  }
  if (lane == 0) {
    if (bad) atomicMax(flags + 1, (int)s + 1);
    if (by_hand) atomicAdd(flags + 2, (int)by_hand);
  }
}

// the last full key before every window (a repeat at a window's start refers to it): that of the nearest earlier
// window of the same segment that saw one
__global__ void k_parse_carry(const PwSeg *__restrict__ segs, uint32_t nseg, uint32_t nwin_total,
                              const uint64_t *__restrict__ entry, const uint64_t *__restrict__ wlastkey, uint64_t *__restrict__ carry) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nwin_total) return;
  uint64_t off = ~0ull, len = 0;
  const uint64_t e = entry[w];
  if (e != PW_EOF && e != PW_BAD) {
    const uint32_t w0 = segs[pw_seg_of(segs, nseg, w)].win0;
    for (uint32_t v = w; v > w0;) {
      v--;
      if (wlastkey[2 * (uint64_t)v] != ~0ull) { off = wlastkey[2 * (uint64_t)v]; len = wlastkey[2 * (uint64_t)v + 1]; break; }
    }
  }
  carry[2 * (uint64_t)w] = off;
  carry[2 * (uint64_t)w + 1] = len;
}

}  // namespace tezgpu

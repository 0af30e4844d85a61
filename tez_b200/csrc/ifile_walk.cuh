// ifile_walk.cuh -- IFile record framing on the device (IFile.Reader.positionToNextRecord, SORT/IFile.java:877-1000),
// shared by the three walkers of IFile bodies: the window parser (pw_walk, parse_windows.cuh), the sequential walker
// (k_parse_segments, merger.cuh) and the bounded merge's window scan and cut (k_step_walk, merge_steps.cuh).
//
// A record header is vint(key length) vint(value length); key length -2 (RLE_MARKER) repeats the last full key.  After
// a repeat comes a value length alone, or V_END_MARKER (-3) followed by both lengths; -1 -1 are the EOF markers.  Any
// other negative length, or one above 2^31-1, is malformed.
#pragma once
#include "common.cuh"

namespace tezgpu {

// ------------------------------------------------------------------------------------------------ vlong readers
// 8 bytes of the segment at offset pos (little endian); bytes past the segment read as zero.  fast: two aligned loads
__device__ __forceinline__ uint64_t pw_load8(const uint8_t *__restrict__ seg, uint64_t pos, uint64_t seg_len) {
  if (pos + 16 <= seg_len) {
    const uintptr_t a = (uintptr_t)(seg + pos);
    const uint32_t sh = (uint32_t)(a & 7u);
    const uint64_t *q = reinterpret_cast<const uint64_t *>(a - sh);
    const uint64_t x = __ldg(q);
    if (sh == 0) return x;
    const uint64_t y = __ldg(q + 1);
    return (x >> (8u * sh)) | (y << (64u - 8u * sh));
  }
  uint64_t v = 0;
  for (uint32_t b = 0; b < 8; b++)
    if (pos + b < seg_len) v |= (uint64_t)seg[pos + b] << (8u * b);
  return v;
}

// hadoop WritableUtils.readVLong at pos from global memory (bounded by end); false = runs past `end`
__device__ __forceinline__ bool pw_vlong(const uint8_t *__restrict__ seg, uint64_t seg_len, uint64_t &pos, uint64_t end,
                                         int64_t &out) {
  if (pos >= end) return false;
  const uint64_t x = pw_load8(seg, pos, seg_len);
  const int8_t first = (int8_t)(x & 0xFF);
  if (first >= -112) { out = first; pos += 1; return true; }
  const int len = vint_decode_size((uint8_t)first);
  if (pos + (uint64_t)len > end) return false;
  uint64_t v = 0;
  if (len <= 8) {
    for (int i = 1; i < len; i++) v = (v << 8) | ((x >> (8 * i)) & 0xFF);
  } else {  // 9-byte vlong: the last byte lies outside the 8-byte window
    for (int i = 1; i < 8; i++) v = (v << 8) | ((x >> (8 * i)) & 0xFF);
    v = (v << 8) | seg[pos + 8];
  }
  const bool neg = first < -120;   // (first >= -112 handled above)
  out = neg ? (int64_t)~v : (int64_t)v;
  pos += (uint64_t)len;
  return true;
}

// pw_vlong as a decode_header reader
struct GlobalVlong {
  const uint8_t *__restrict__ seg;
  uint64_t seg_len, end;
  __device__ __forceinline__ int operator()(uint64_t &pos, int64_t &out) const { return pw_vlong(seg, seg_len, pos, end, out) ? 0 : 2; }
};

// One WARP walks one source: the 32 lanes stage a PARSE_WIN window of it in shared memory with coalesced loads, lane 0
// decodes the record headers out of it (key / value bytes are skipped, never read), so a walk step costs tens of cycles
// instead of a DRAM round trip.
constexpr int PARSE_WARPS = 8;
constexpr uint32_t PARSE_WIN = 4096;

struct ParseWin {
  const uint8_t *seg;   // source base in global memory
  uint8_t *win;         // this warp's shared window
  uint64_t wbase;       // source offset of win[0]
  uint64_t end;         // body end
};
// readVLong from the shared window: 0 = ok, 1 = need reload at pos, 2 = runs past the body end
__device__ __forceinline__ int win_vlong(const ParseWin &w, uint64_t &pos, int64_t &out) {
  if (pos >= w.end) return 2;
  if (pos < w.wbase || pos >= w.wbase + PARSE_WIN) return 1;
  const uint8_t first = w.win[pos - w.wbase];
  const int len = vint_decode_size(first);
  if (pos + (uint64_t)len > w.end) return 2;
  if (pos + (uint64_t)len > w.wbase + PARSE_WIN) return 1;
  if (len == 1) { out = (int8_t)first; pos += 1; return 0; }
  uint64_t v = 0;
  for (int i = 1; i < len; i++) v = (v << 8) | w.win[pos + i - w.wbase];
  const int8_t f = (int8_t)first;
  const bool neg = f < -120 || (f >= -112 && f < 0);
  out = neg ? (int64_t)~v : (int64_t)v;
  pos += len;
  return 0;
}

// ------------------------------------------------------------------------------------------------ record header
// outcomes of decode_header, and the first statuses of a walk
constexpr int REC_OK = 0;         // a record header
constexpr int REC_EOF = 1;        // the EOF markers
constexpr int REC_BAD = 2;        // malformed lengths
constexpr int REC_PAST_END = 3;   // a vint runs past the body end
constexpr int REC_RELOAD = -1;    // the shared window must be staged again at the record start

struct RecHdr {
  int64_t kl, vl;   // kl = -2: the record repeats the last full key
  uint64_t pos;     // first byte after the header
  bool marker;      // a V_END_MARKER was consumed (the record's own bytes start one byte later)
};

// Decodes the header of the record at pos; after_repeat: the previous record was a repeat.  read(pos, out) is a vlong
// reader returning 0 ok, 1 reload, 2 past the end.  Nothing is committed before the whole header is decoded, so a
// reload restarts the record.
template <typename Read>
__device__ __forceinline__ int decode_header(Read read, bool after_repeat, uint64_t pos, RecHdr &h) {
  int64_t kl = 0, vl = 0;
  bool marker = false;
  int rc;
  if (after_repeat) {  // a value length, or V_END_MARKER followed by both lengths
    rc = read(pos, vl);
    kl = -2;
    if (rc == 0 && vl == -3) { marker = true; rc = read(pos, kl); if (rc == 0) rc = read(pos, vl); }
  } else {
    rc = read(pos, kl);
    if (rc == 0) rc = read(pos, vl);
  }
  h.kl = kl; h.vl = vl; h.pos = pos; h.marker = marker;
  if (rc != 0) return rc == 1 ? REC_RELOAD : REC_PAST_END;
  if (kl == -1 && vl == -1) return REC_EOF;
  if ((kl != -2 && kl < 0) || vl < 0 || kl > 0x7fffffffll || vl > 0x7fffffffll) return REC_BAD;
  return REC_OK;
}

// ------------------------------------------------------------------------------------------------ warp-window walk
struct WalkEnd {
  int status;       // REC_EOF, REC_BAD, REC_PAST_END, or the nonzero status on_record stopped with (all lanes)
  uint64_t stop;    // lane 0: start of the record the walk stopped at, after its V_END_MARKER
};

// Walks src[pos, end) with one warp (src holds len readable bytes; bytes past them stage as zero).  Lane 0 calls
// on_record(h) for every well-formed header: 0 takes the record and the walk moves past its key and value, any other
// value stops the walk with that status.
template <typename OnRecord>
__device__ __forceinline__ WalkEnd warp_window_walk(const uint8_t *__restrict__ src, uint64_t len, uint64_t pos,
                                                    uint64_t end, uint8_t *win, OnRecord on_record) {
  const int lane = threadIdx.x & 31;
  ParseWin w{src, win, pos, end};
  bool after_repeat = false;
  int status = 0;
  while (true) {
    for (uint32_t o = lane * 4; o < PARSE_WIN; o += 128) {
      const uint64_t p = w.wbase + o;
      uint32_t v = 0;
      if (p + 4 <= len && (((uintptr_t)(src + p)) & 3u) == 0) v = *reinterpret_cast<const uint32_t *>(src + p);
      else for (int b = 0; b < 4; b++) if (p + b < len) v |= (uint32_t)src[p + b] << (8 * b);
      *reinterpret_cast<uint32_t *>(win + o) = v;
    }
    __syncwarp();
    if (lane == 0) {
      while (status == 0) {
        RecHdr h;
        const int d = decode_header([&](uint64_t &p, int64_t &out) { return win_vlong(w, p, out); }, after_repeat, pos, h);
        if (d == REC_RELOAD) { w.wbase = pos & ~(uint64_t)15; break; }
        status = d == REC_OK ? on_record(h) : d;
        if (status != 0) { pos += h.marker ? 1 : 0; break; }
        pos = h.pos + (h.kl != -2 ? (uint64_t)h.kl : 0) + (uint64_t)h.vl;
        after_repeat = h.kl == -2;
      }
    }
    status = __shfl_sync(0xffffffffu, status, 0);
    w.wbase = __shfl_sync(0xffffffffu, w.wbase, 0);
    if (status != 0) return WalkEnd{status, pos};
    __syncwarp();
  }
}

}  // namespace tezgpu

// peer_fetch.cuh -- the shuffle transfer on an NVLink/NVSwitch box: the consumer pulls byte ranges of the producers'
// file.out straight out of their HBM (CUDA IPC peer mappings) with every SM, instead of the HTTP round trip of
// ShuffleHandler + FetcherOrderedGrouped.copyMapOutput (OG/FetcherOrderedGrouped.java:437-632).
// One launch moves any number of (source, destination, length) ranges; ranges whose two addresses agree modulo 16
// move as 128-bit words (the caller picks destinations that way), anything else falls back to bytes.
#pragma once
#include "common.cuh"
#include "crc32.cuh"
#include "emit_fast.cuh"

namespace tezgpu {

struct FetchRange {
  const uint8_t *src;
  uint8_t *dst;
  uint64_t len;
  uint64_t chunk0;  // index of this range's first chunk in the launch (prefix sum, filled by the host)
};

constexpr uint32_t FETCH_THREADS = 512;
constexpr uint32_t FETCH_UNROLL = 8;
constexpr uint64_t FETCH_CHUNK = (uint64_t)FETCH_THREADS * FETCH_UNROLL * 16 * 2;  // 128 KiB of 16-byte words per chunk

// the producer rewrites its buffer every step: never serve a peer byte from a local cache line (ld.cv)
__device__ __forceinline__ uint4 ld_peer_16(const uint4 *p) { return __ldcv(p); }
__device__ __forceinline__ uint8_t ld_peer_8(const uint8_t *p) { return __ldcv(p); }  // head / tail / misaligned bytes: same rule

__device__ __forceinline__ void fetch_ranges_body(const FetchRange *__restrict__ ranges, uint32_t nranges, uint64_t nchunks) {
  for (uint64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
    uint32_t lo = 0, hi = nranges;  // last range with chunk0 <= c
    while (hi - lo > 1) {
      uint32_t mid = (lo + hi) >> 1;
      if (ranges[mid].chunk0 <= c) lo = mid; else hi = mid;
    }
    const FetchRange r = ranges[lo];
    const uint64_t k = c - r.chunk0;
    const uint32_t mis = (uint32_t)((uintptr_t)r.src & 15u);
    if (mis != (uint32_t)((uintptr_t)r.dst & 15u)) {  // incompatible alignment: bytes
      const uint64_t a = k * FETCH_CHUNK, b = min(r.len, a + FETCH_CHUNK);
      for (uint64_t i = a + threadIdx.x; i < b; i += FETCH_THREADS) r.dst[i] = ld_peer_8(r.src + i);
      continue;
    }
    // body: the 16-byte words between the first and the last aligned address of the range
    const uint64_t head = min(r.len, (uint64_t)((16u - mis) & 15u));
    const uint64_t words = (r.len - head) >> 4;
    const uint4 *s16 = reinterpret_cast<const uint4 *>(r.src + head);
    uint4 *d16 = reinterpret_cast<uint4 *>(r.dst + head);
    const uint64_t w0 = k * (FETCH_CHUNK / 16), w1 = min(words, w0 + FETCH_CHUNK / 16);
    uint64_t i = w0 + threadIdx.x;
    for (; i + (uint64_t)(FETCH_UNROLL - 1) * FETCH_THREADS < w1; i += (uint64_t)FETCH_UNROLL * FETCH_THREADS) {
      uint4 v[FETCH_UNROLL];
#pragma unroll
      for (uint32_t u = 0; u < FETCH_UNROLL; u++) v[u] = ld_peer_16(s16 + i + (uint64_t)u * FETCH_THREADS);
#pragma unroll
      for (uint32_t u = 0; u < FETCH_UNROLL; u++) d16[i + (uint64_t)u * FETCH_THREADS] = v[u];
    }
    for (; i < w1; i += FETCH_THREADS) d16[i] = ld_peer_16(s16 + i);
    if (k == 0) {  // the unaligned head and tail bytes of the range travel with its first chunk
      const uint64_t tail0 = head + (words << 4);
      if (threadIdx.x < head) r.dst[threadIdx.x] = ld_peer_8(r.src + threadIdx.x);
      if (threadIdx.x >= 32 && tail0 + (threadIdx.x - 32) < r.len && threadIdx.x - 32 < 16)
        r.dst[tail0 + (threadIdx.x - 32)] = ld_peer_8(r.src + tail0 + (threadIdx.x - 32));
    }
  }
}

__global__ void __launch_bounds__(FETCH_THREADS)
    k_fetch_ranges(const FetchRange *__restrict__ ranges, uint32_t nranges, uint64_t nchunks) {
  fetch_ranges_body(ranges, nranges, nchunks);
}

// the usual case -- one range per peer GPU -- needs no device-side table: the ranges ride in the parameter space
constexpr uint32_t FETCH_INLINE_RANGES = 16;
struct FetchRangeList { FetchRange r[FETCH_INLINE_RANGES]; };
__global__ void __launch_bounds__(FETCH_THREADS)
    k_fetch_ranges_inline(const __grid_constant__ FetchRangeList lst, uint32_t nranges, uint64_t nchunks) {
  fetch_ranges_body(lst.r, nranges, nchunks);
}

// ---------------------------------------------------------------------------------------------- fetch + verify
// The same pull with the IFile checksum of every segment verified on the bytes as they pass through the registers --
// what the reference does when it fetches a map output to memory (IFile.Reader.readToMemory reads through an
// IFileInputStream that checks the CRC32 trailer, SORT/IFile.java:764-809; OG/FetcherOrderedGrouped.java:519-533), after
// which InMemoryReader never looks at a checksum again.  Work item = one 64 KiB piece of one segment body: the CTA
// moves the piece's 16-byte words (8 peer loads in flight per thread) and folds them with the chunk-interleaved
// scheme of k_crc_pieces (thread t owns the words at distance == T-1-t (mod T) from the piece's end; 3 x "next word" +
// one "skip to my next word" per 16 bytes, both as warp-resident SHFL digit tables); k_crc_combine / k_fetch_crc_check
// fold the pieces per segment and compare with the big-endian trailer.  The fold costs LSU/SHFL issue slots the
// NVLink-bound copy leaves idle, and saves the separate 1-byte-per-byte HBM read k_crc_pieces would need afterwards.
struct FetchSeg {
  const uint8_t *src;   // first byte of the segment (its 'TIF' header when has_header) in the peer's buffer
  uint8_t *dst;         // where it lands locally; (dst - src) is a multiple of 16
  uint64_t len;         // header + body + 4 checksum bytes
  uint32_t has_header;
  uint32_t pad;
};

constexpr uint32_t FV_THREADS = 256;
constexpr uint32_t FV_UNROLL = 8;
constexpr uint32_t FV_PIECE = 64 * 1024;

__global__ void __launch_bounds__(FV_THREADS)
    k_fetch_verify(const FetchSeg *__restrict__ segs, const uint32_t *__restrict__ piece_start, uint32_t nseg, uint32_t npieces,
                   const CrcTables *__restrict__ t, TileCrc *__restrict__ out) {
  static_assert(FV_THREADS == 256, "advc is built for the 256-thread chunk interleave (EMIT_CRC_STRIDE_WORDS)");
  __shared__ uint32_t s_tab[256], s_adv128[4 * 256], s_part[FV_THREADS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  s_tab[tid] = t->slice[0][tid];
  for (int i = tid; i < 4 * 256; i += FV_THREADS) s_adv128[i] = (&t->adv128[0][0])[i];
  CrcChunkFoldT<true> cf;
  cf.init(t, lane);
  const uint32_t lane_pow = cf.lane_pow;
  __syncthreads();
  for (uint32_t piece = blockIdx.x; piece < npieces; piece += gridDim.x) {
    uint32_t lo = 0, hi = nseg;  // last segment with piece_start[s] <= piece
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (piece_start[mid] <= piece) lo = mid; else hi = mid;
    }
    const FetchSeg sd = segs[lo];
    const uint64_t body0 = sd.has_header ? 4 : 0, body_bytes = sd.len - 4 - body0;
    const uint32_t k = piece - piece_start[lo];
    const uint64_t a = (uint64_t)k * FV_PIECE, b = min(body_bytes, a + FV_PIECE);
    const bool last_piece = b == body_bytes;
    const uint8_t *pa = sd.src + body0 + a, *pb = sd.src + body0 + b;
    const int64_t delta = sd.dst - sd.src;                      // same for every byte of the segment
    const uint32_t mis = (uint32_t)((uintptr_t)pa & 15u);
    const uint8_t *c0 = pa - mis;                               // aligned-down start of the piece's first word
    const uint32_t Cn = (uint32_t)((pb - c0) >> 4);             // whole words
    // the first word of the first piece may start before the segment (its leading bytes belong to whatever precedes
    // the segment): that word is moved byte by byte from the segment start on, never touching memory outside it
    const bool ragged_first = k == 0 && c0 < sd.src;
    uint32_t c = 0;
    if (Cn) {
      const uint32_t iters = (Cn + FV_THREADS - 1) / FV_THREADS;
      int32_t i = (int32_t)Cn + tid - (int32_t)(iters * FV_THREADS);
      for (uint32_t it0 = 0; it0 < iters; it0 += FV_UNROLL) {
        uint4 v[FV_UNROLL];
#pragma unroll
        for (uint32_t u = 0; u < FV_UNROLL; u++) {
          const int32_t iu = i + (int32_t)(u * FV_THREADS);
          v[u] = make_uint4(0, 0, 0, 0);
          if (it0 + u < iters && iu >= 0) {
            if (iu == 0 && ragged_first) {
              uint32_t w[4] = {0, 0, 0, 0};
              for (const uint8_t *q = sd.src; q < c0 + 16; q++) {
                const uint32_t byte = ld_peer_8(q);
                const_cast<uint8_t *>(q)[delta] = (uint8_t)byte;
                const uint32_t o = (uint32_t)(q - c0);
                w[o >> 2] |= byte << (8u * (o & 3u));
              }
              v[u] = make_uint4(w[0], w[1], w[2], w[3]);
            } else {
              v[u] = ld_peer_16(reinterpret_cast<const uint4 *>(c0) + iu);
            }
          }
        }
#pragma unroll
        for (uint32_t u = 0; u < FV_UNROLL; u++) {
          if (it0 + u >= iters) break;   // uniform
          const int32_t iu = i + (int32_t)(u * FV_THREADS);
          uint4 w = v[u];
          if (iu >= 0) {
            if (!(iu == 0 && ragged_first)) *reinterpret_cast<uint4 *>(const_cast<uint8_t *>(c0) + delta + 16ll * iu) = w;
            if (iu == 0 && mis) {  // bytes before the piece fold as zero (a remainder with zero initial value ignores them)
              uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
              for (uint32_t q = 0; q < 4; q++) {
                if (mis >= 4 * q + 4) ww[q] = 0;
                else if (mis > 4 * q) ww[q] &= 0xFFFFFFFFu << (8u * (mis - 4 * q));
              }
              w = make_uint4(ww[0], ww[1], ww[2], ww[3]);
            }
          }
          c = cf.fold(c, w, it0 + u + 1 == iters);
        }
        i += (int32_t)(FV_UNROLL * FV_THREADS);
      }
    }
    s_part[tid] = c;
    __syncthreads();
    if (warp == 0) {
      uint32_t q = 0;
#pragma unroll
      for (int kk = 0; kk < (int)FV_THREADS / 32; kk++) {
        q = s_adv128[q & 0xFF] ^ s_adv128[256 + ((q >> 8) & 0xFF)] ^ s_adv128[512 + ((q >> 16) & 0xFF)] ^ s_adv128[768 + (q >> 24)];
        q ^= s_part[lane + 32 * kk];
      }
      q = crc_multmodp(q, lane_pow);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q ^= __shfl_xor_sync(0xffffffffu, q, o);
      if (lane == 0) {
        // bytes after the last whole word: the rest of the piece (folded), and behind the last piece the 4 checksum
        // bytes (moved only).  A piece without a whole word is handled here entirely, segment header included.
        uint32_t raw = q;
        if (Cn && k == 0 && c0 > sd.src)   // header bytes that sit in the word before the first whole one
          for (const uint8_t *h = sd.src; h < c0; h++) const_cast<uint8_t *>(h)[delta] = ld_peer_8(h);
        const uint8_t *x = Cn ? c0 + 16ull * Cn : (k == 0 ? sd.src : pa);
        for (; x < pa; x++) const_cast<uint8_t *>(x)[delta] = ld_peer_8(x);   // only when Cn == 0: header bytes
        for (; x < pb; x++) {
          const uint32_t byte = ld_peer_8(x);
          const_cast<uint8_t *>(x)[delta] = (uint8_t)byte;
          raw = s_tab[(raw ^ byte) & 0xFF] ^ (raw >> 8);
        }
        if (last_piece) for (; x < pb + 4; x++) const_cast<uint8_t *>(x)[delta] = ld_peer_8(x);
        TileCrc tc;
        tc.raw = raw;
        tc.p = lo;
        tc.after = body_bytes - b;
        out[piece] = tc;
      }
    }
    __syncthreads();
  }
}

// compares every segment's folded remainder with the big-endian trailer that was just copied
__global__ void k_fetch_crc_check(const FetchSeg *__restrict__ segs, uint32_t nseg, const uint32_t *__restrict__ seg_crc,
                                  const CrcTables *__restrict__ t, int *__restrict__ bad) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const FetchSeg sd = segs[s];
  const uint64_t body = sd.len - 4 - (sd.has_header ? 4 : 0);
  if (crc_from_raw(t, seg_crc[s], body) != load_be32(sd.dst + sd.len - 4)) atomicExch(bad, (int)s + 1);
}

// number of chunks a range of `len` bytes starting at `src` occupies (at least one, so head/tail bytes always move)
static inline uint64_t fetch_chunks(const void *src, const void *dst, uint64_t len) {
  const uint32_t mis = (uint32_t)((uintptr_t)src & 15u);
  if (mis != (uint32_t)((uintptr_t)dst & 15u)) return len ? div_up(len, FETCH_CHUNK) : 0;
  if (!len) return 0;
  const uint64_t head = std::min<uint64_t>(len, (16u - mis) & 15u);
  const uint64_t words = (len - head) >> 4;
  return std::max<uint64_t>(1, div_up(words * 16, FETCH_CHUNK));
}

}  // namespace tezgpu

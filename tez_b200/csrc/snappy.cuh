// snappy.cuh -- SnappyCodec on the device: the writer's block compressor and the reader's chunk decoder.
//
// A compressed segment (SORT/IFile.java:351-420) is 'T' 'I' 'F' 0x01, the SnappyCodec stream of the uncompressed body
// and a big-endian CRC-32 over the stream.  SnappyCodec writes through Hadoop's BlockCompressorStream with the framing
// of Lz4Codec: blocks of a big-endian int32 raw length and one or more chunks, each a big-endian int32 compressed
// length and one raw Snappy block (no framing format).  A raw Snappy block is its uncompressed length as a
// little-endian base-128 varint (the preamble, at most 5 bytes), then elements whose tag's low 2 bits give the type:
// 00 literal (length - 1 in the top 6 bits below 60; tags 60-63: 1-4 little-endian length bytes follow), 01 copy of
// 4-11 bytes at an 11-bit offset, 10 copy of 1-64 bytes at a 16-bit offset, 11 copy of 1-64 bytes at a 32-bit offset.
// Java's reader decodes each chunk with snappy-java (libsnappy) into a buffer of io.compression.codec.snappy.buffersize
// bytes (262,144 by default), so a chunk decodes on its own to at most that many bytes.
//
// Writer: the body is cut into SN_BLOCK-byte blocks of one chunk each.  One CTA of SN_LANES threads compresses a
// block.  Lane l parses slice [l * SN_SLICE, (l + 1) * SN_SLICE) greedily with a hash table private to the lane
// (seeded with the SN_SLICE bytes before the slice; matches end inside the slice) and steps further on misses the way
// libsnappy does (+1 every 32 misses), so the output does not depend on thread timing.  Pass 1 sizes each lane's
// elements; thread 0 joins the literal runs that cross lanes and places the lanes; pass 2 writes.  Copies are encoded
// as libsnappy encodes them (copy-1 for 4-11 bytes below offset 2,048, copy-2 otherwise, long copies split 64 at a
// time while 68 or more remain, then 60 if more than 64 remain).  A chunk that is not smaller than the all-literal
// form is written all-literal, so no chunk exceeds TEZGPU_SNAPPY_CHUNK_BOUND.  The compressor is __host__ __device__:
// tezgpu_debug_snappy_compress_emulate runs it on the host and yields the bytes the device writes.  The parse is kept
// apart from lz4.cuh's: Snappy has no end-of-block rules, a different skip rule and byte-aligned elements.
//
// Reader: strict.  Every chunk states its raw length up front, so one thread per segment walks the block and chunk
// headers and every chunk's preamble (k_snwalk) and each chunk becomes a decode unit, also the chunks of multi-chunk
// blocks.  A block's raw length is > 0, its chunks' preambles add up to exactly that length, the blocks add up to
// rawLength - 4 and the stream ends right after the last block.  One warp per chunk decodes (k_snchunks): the input
// is consumed exactly and the output ends exactly at the preamble length.  An error is keyed by the position of its
// chunk in the segment, so the segment reports the first one in stream order: the reason the serial emulation gives.
#pragma once
#include "lz4.cuh"

namespace tezgpu {

// Raw bytes per written block: the LZ4 block size, for the same reasons (one 64 KiB slot and checksum piece per
// framed chunk, offsets below 65,536, the block and the lanes' hash tables in one SM's shared memory).
constexpr uint32_t SN_BLOCK = TEZGPU_SNAPPY_BLOCK_BYTES;   // 65,024
constexpr uint32_t SN_LANES = 32;                         // threads per block (one warp)
constexpr uint32_t SN_SLICE = SN_BLOCK / SN_LANES;        // bytes parsed by one lane: 2,032
constexpr uint32_t SN_HBITS = 11;                         // lane hash table: 2^SN_HBITS u16 positions
constexpr uint32_t SN_HSIZE = 1u << SN_HBITS;
constexpr uint32_t SN_SLOT = 65536;                       // device bytes per block: 8 header bytes + the chunk
constexpr uint32_t SN_CHUNK_CAP = 262144;                 // Java's SnappyDecompressor buffer: a chunk is at most this
constexpr uint32_t SN_SKIP_SHIFT = 5;                     // libsnappy: the probe step grows by one every 32 misses
constexpr uint32_t SN_MIN_UNIT_BYTES = 5;                 // the smallest chunk the walk takes: 4 length bytes, 1 preamble byte
static_assert(8 + TEZGPU_SNAPPY_CHUNK_BOUND <= SN_SLOT && SN_SLOT <= 64 * 1024, "a framed chunk must fit one slot and one CRC piece");
static_assert(SN_BLOCK % SN_LANES == 0 && SN_BLOCK < 65536 && SN_BLOCK < (1u << 21), "slices, offsets and a 3-byte preamble");

// error reasons (tezgpu_debug_snappy_decompress_emulate returns them; the merger reports them as TEZGPU_E_FORMAT)
enum SnErr : int32_t {
  SN_OK = 0,
  SN_ERR_HEADER = 1,      // the stream ends inside a block or chunk length
  SN_ERR_BLOCK = 2,       // a block's raw length is not in 1 .. the body bytes still expected
  SN_ERR_CHUNK = 3,       // a chunk's compressed length is over 262,144 or runs past the end of the stream
  SN_ERR_PREAMBLE = 4,    // the preamble runs past the chunk, is over 5 bytes or 32 bits, is 0 or is over 262,144
  SN_ERR_OVERRUN = 5,     // a preamble takes the block's chunks past the block's raw length
  SN_ERR_LITERAL = 6,     // a literal's length bytes or its bytes run past the chunk
  SN_ERR_COPY = 7,        // a copy's offset bytes run past the chunk
  SN_ERR_OFFSET = 8,      // copy offset 0 or before the start of the chunk
  SN_ERR_LONG = 9,        // an element writes past the preamble length
  SN_ERR_SHORT = 10,      // the chunk ends before the preamble length is written
  SN_ERR_TRAILING = 11,   // bytes after the last block
  SN_ERR_LENGTH = 12,     // the blocks add up to less than rawLength - 4
};

static inline const char *sn_err_name(int32_t e) {
  switch (e) {
    case SN_ERR_HEADER: return "truncated block header";
    case SN_ERR_BLOCK: return "block raw length outside the remaining rawLength - 4";
    case SN_ERR_CHUNK: return "chunk length over 262144 or past the end of the stream";
    case SN_ERR_PREAMBLE: return "invalid chunk preamble";
    case SN_ERR_OVERRUN: return "chunks decode past their block's raw length";
    case SN_ERR_LITERAL: return "literal past the end of the chunk";
    case SN_ERR_COPY: return "copy past the end of the chunk";
    case SN_ERR_OFFSET: return "invalid copy offset";
    case SN_ERR_LONG: return "chunk decodes past its preamble length";
    case SN_ERR_SHORT: return "chunk decodes short of its preamble length";
    case SN_ERR_TRAILING: return "bytes after the last block";
    case SN_ERR_LENGTH: return "decompressed length differs from rawLength - 4";
    default: return "ok";
  }
}

// bytes of the varint of v
Z_HD uint32_t sn_varint_size(uint32_t v) {
  uint32_t k = 1;
  for (; v >= 128; v >>= 7) k++;
  return k;
}
Z_HD uint32_t sn_put_varint(uint8_t *o, uint32_t v) {
  uint32_t k = 0;
  for (; v >= 128; v >>= 7) o[k++] = (uint8_t)(v | 128);
  o[k++] = (uint8_t)v;
  return k;
}
// tag and length bytes of a literal of n >= 1 bytes
Z_HD uint32_t sn_lit_head(uint32_t n) {
  const uint32_t m = n - 1;
  return m < 60 ? 1 : m < 256 ? 2 : m < 65536 ? 3 : m < (1u << 24) ? 4 : 5;
}
// the whole literal element of n bytes (0: none)
Z_HD uint32_t sn_lit_bytes(uint32_t n) { return n ? sn_lit_head(n) + n : 0; }
Z_HD uint32_t sn_put_lit_head(uint8_t *o, uint32_t n) {
  const uint32_t m = n - 1, k = sn_lit_head(n);
  if (k == 1) { o[0] = (uint8_t)(m << 2); return 1; }
  o[0] = (uint8_t)((58 + k) << 2);
  for (uint32_t b = 0; b + 1 < k; b++) o[1 + b] = (uint8_t)(m >> (8 * b));
  return k;
}
// one copy element of 1..64 bytes at offset off < 65,536 (W: write it to o); returns its bytes
template <bool W>
Z_HD uint32_t sn_copy64(uint8_t *o, uint32_t off, uint32_t len) {
  if (len < 12 && off < 2048) {
    if (W) { o[0] = (uint8_t)(1 | ((len - 4) << 2) | ((off >> 8) << 5)); o[1] = (uint8_t)off; }
    return 2;
  }
  if (W) { o[0] = (uint8_t)(2 | ((len - 1) << 2)); o[1] = (uint8_t)off; o[2] = (uint8_t)(off >> 8); }
  return 3;
}
// a match of len >= 4 bytes, split as libsnappy's EmitCopy splits it
template <bool W>
Z_HD uint32_t sn_emit_copy(uint8_t *o, uint32_t off, uint32_t len) {
  uint32_t k = 0;
  for (; len >= 68; len -= 64) k += sn_copy64<W>(o + k, off, 64);
  if (len > 64) { k += sn_copy64<W>(o + k, off, 60); len -= 60; }
  return k + sn_copy64<W>(o + k, off, len);
}

// ------------------------------------------------------------------------------------------------ writer
struct SnShared {
  uint8_t data[SN_BLOCK];
  uint16_t htab[SN_LANES][SN_HSIZE];
  uint32_t lhead[SN_LANES];    // literals from the slice start to the lane's first match
  uint32_t ltail[SN_LANES];    // literals from the lane's last match to the slice end
  uint32_t lnm[SN_LANES];      // matches of the lane
  uint32_t lbytes[SN_LANES];   // bytes of the lane's elements, less its first literal run
  uint32_t lcarry[SN_LANES];   // literals of earlier lanes that open the lane's first literal run
  uint32_t lout[SN_LANES];     // chunk offset of the lane's first element
  uint32_t run_dst[SN_LANES + 1], run_src[SN_LANES + 1], run_len[SN_LANES + 1];   // literal runs copied by every thread
  uint32_t fin_out, fin_len, bytes, clen, literal;
};

Z_HD uint32_t sn_hash4(const uint8_t *d) {
  const uint32_t v = (uint32_t)d[0] | ((uint32_t)d[1] << 8) | ((uint32_t)d[2] << 16) | ((uint32_t)d[3] << 24);
  return (v * 0x1e35a7bdu) >> (32 - SN_HBITS);
}

// Greedy parse of the lane's slice.  PASS 1: sizes; PASS 2: the elements into out (the chunk), except the bytes of
// the lane's first literal run, which go to run_* for all threads to copy.  An all-literal chunk skips pass 2.
template <int PASS>
Z_HD void sn_lane(SnShared &sh, uint32_t lane, uint8_t *out) {
  const uint32_t clen = sh.clen;
  const uint32_t s0 = lane * SN_SLICE;
  if (PASS == 1) { sh.lnm[lane] = 0; sh.lhead[lane] = 0; sh.ltail[lane] = 0; sh.lbytes[lane] = 0; }
  if (s0 >= clen || (PASS == 2 && sh.literal)) return;
  const uint32_t s1 = l4_min(clen, s0 + SN_SLICE);
  const uint8_t *d = sh.data;
  uint16_t *ht = sh.htab[lane];
  for (uint32_t i = 0; i < SN_HSIZE; i++) ht[i] = ZEMPTY;
  for (uint32_t q = s0 >= SN_SLICE ? s0 - SN_SLICE : 0; q < s0 && q + 4 <= clen; q++) ht[sn_hash4(d + q)] = (uint16_t)q;
  uint32_t p = s0, anchor = s0, nm = 0, bytes = 0, misses = 0;
  uint32_t o = PASS == 2 ? sh.lout[lane] : 0;
  while (p + 4 <= s1) {
    const uint32_t h = sn_hash4(d + p);
    uint32_t cand = ht[h];
    ht[h] = (uint16_t)p;
    if (cand != ZEMPTY && d[cand] == d[p] && d[cand + 1] == d[p + 1] && d[cand + 2] == d[p + 2] && d[cand + 3] == d[p + 3]) {
      uint32_t m = 4;
      while (p + m < s1 && d[cand + m] == d[p + m]) m++;
      while (p > anchor && cand > 0 && d[p - 1] == d[cand - 1]) { p--; cand--; m++; }
      const uint32_t off = p - cand;
      if (nm == 0) {
        if (PASS == 1) {
          sh.lhead[lane] = p - s0;
        } else {
          const uint32_t L = sh.lcarry[lane] + (p - s0);
          if (L) o += sn_put_lit_head(out + o, L);
          sh.run_dst[lane] = o; sh.run_src[lane] = p - L; sh.run_len[lane] = L;
          o += L;
        }
      } else {
        const uint32_t L = p - anchor;
        if (PASS == 1) {
          bytes += sn_lit_bytes(L);
        } else if (L) {
          o += sn_put_lit_head(out + o, L);
          for (uint32_t k = 0; k < L; k++) out[o + k] = d[anchor + k];
          o += L;
        }
      }
      if (PASS == 1) bytes += sn_emit_copy<false>(nullptr, off, m);
      else o += sn_emit_copy<true>(out + o, off, m);
      nm++;
      p += m;
      anchor = p;
      misses = 0;
      if (p - 2 + 4 <= clen) ht[sn_hash4(d + p - 2)] = (uint16_t)(p - 2);
    } else {
      p += 1 + (misses++ >> SN_SKIP_SHIFT);
    }
  }
  if (PASS == 1) {
    sh.lnm[lane] = nm;
    sh.ltail[lane] = s1 - anchor;
    sh.lbytes[lane] = bytes;
  }
}

// Thread 0, after pass 1: the literal runs that cross lanes, each lane's output offset, the last literals, the size;
// the all-literal form where the parse does not beat it.
Z_HD void sn_plan(SnShared &sh) {
  const uint32_t clen = sh.clen, pre = sn_varint_size(clen);
  uint32_t pos = pre, carry = 0;
  for (uint32_t l = 0; l < SN_LANES; l++) {
    sh.run_len[l] = 0;
    const uint32_t s0 = l * SN_SLICE;
    if (s0 >= clen) continue;
    if (!sh.lnm[l]) { carry += l4_min(clen, s0 + SN_SLICE) - s0; continue; }
    const uint32_t L = carry + sh.lhead[l];
    sh.lcarry[l] = carry;
    sh.lout[l] = pos;
    pos += sn_lit_bytes(L) + sh.lbytes[l];
    carry = sh.ltail[l];
  }
  sh.fin_out = pos;
  pos += sn_lit_bytes(carry);
  sh.literal = pos >= pre + sn_lit_bytes(clen) ? 1 : 0;
  if (sh.literal) {
    for (uint32_t l = 0; l < SN_LANES; l++) sh.run_len[l] = 0;
    sh.fin_out = pre;
    carry = clen;
    pos = pre + sn_lit_bytes(clen);
  }
  sh.fin_len = carry;
  sh.run_dst[SN_LANES] = sh.fin_out + (carry ? sn_lit_head(carry) : 0);
  sh.run_src[SN_LANES] = clen - carry;
  sh.run_len[SN_LANES] = carry;
  sh.bytes = pos;
}

// Thread 0, after the plan: the block and chunk lengths, the preamble and the last literal's tag
Z_HD void sn_write_frame(const SnShared &sh, uint8_t *slot) {
  store_be32(slot, sh.clen);
  store_be32(slot + 4, sh.bytes);
  uint8_t *out = slot + 8;
  sn_put_varint(out, sh.clen);
  if (sh.fin_len) sn_put_lit_head(out + sh.fin_out, sh.fin_len);
}

// the literal runs of the lanes' first elements and the last literals, threads i0, i0 + step, ...
Z_HD void sn_copy_runs(const SnShared &sh, uint8_t *out, uint32_t i0, uint32_t step) {
  for (uint32_t r = 0; r <= SN_LANES; r++) {
    const uint32_t n = sh.run_len[r], dst = sh.run_dst[r], src = sh.run_src[r];
    for (uint32_t k = i0; k < n; k += step) out[dst + k] = sh.data[src + k];
  }
}

// Host run of the device block compressor (lanes one after the other): slot receives 8 + sh.bytes bytes.
static inline void sn_compress_block_host(SnShared &sh, const uint8_t *block, uint32_t clen, uint8_t *slot) {
  memcpy(sh.data, block, clen);
  sh.clen = clen;
  for (uint32_t l = 0; l < SN_LANES; l++) sn_lane<1>(sh, l, nullptr);
  sn_plan(sh);
  for (uint32_t l = 0; l < SN_LANES; l++) sn_lane<2>(sh, l, slot + 8);
  sn_write_frame(sh, slot);
  sn_copy_runs(sh, slot + 8, 0, 1);
}

// one CTA per block; segs / chunk numbering: ZSeg, z_chunk_part (common.cuh), with SN_BLOCK-byte chunks
__global__ void __launch_bounds__(SN_LANES)
    k_sncompress(const uint8_t *__restrict__ img, const ZSeg *__restrict__ segs, uint32_t P, uint8_t *__restrict__ slots,
                 uint32_t *__restrict__ csize) {
  extern __shared__ __align__(16) uint8_t sn_smem[];
  SnShared &sh = *reinterpret_cast<SnShared *>(sn_smem);
  const uint32_t c = blockIdx.x, tid = threadIdx.x;
  const ZSeg sg = segs[z_chunk_part(segs, P, c)];
  const uint64_t a = (uint64_t)(c - sg.chunk0) * SN_BLOCK;
  const uint32_t clen = (uint32_t)z_min64(SN_BLOCK, sg.body_len - a);
  const uint8_t *src = img + sg.body_off + a;
  for (uint32_t i = tid; i < clen; i += SN_LANES) sh.data[i] = src[i];
  if (tid == 0) sh.clen = clen;
  __syncthreads();
  sn_lane<1>(sh, tid, nullptr);
  __syncthreads();
  if (tid == 0) sn_plan(sh);
  __syncthreads();
  uint8_t *slot = slots + (uint64_t)c * SN_SLOT;
  sn_lane<2>(sh, tid, slot + 8);
  if (tid == 0) sn_write_frame(sh, slot);
  __syncthreads();
  sn_copy_runs(sh, slot + 8, tid, SN_LANES);
  if (tid == 0) csize[c] = 8 + sh.bytes;
}

// ------------------------------------------------------------------------------------------------ reader
// The preamble of the chunk src[0..n): *len its value, *nb its bytes.  As libsnappy reads it: at most 5 bytes, the
// fifth below 16; then it must be 1 .. SN_CHUNK_CAP.
Z_HD int32_t sn_preamble(const uint8_t *src, uint32_t n, uint32_t *len, uint32_t *nb) {
  uint32_t v = 0;
  for (uint32_t k = 0; k < 5 && k < n; k++) {
    const uint32_t c = src[k];
    if (k == 4 && c > 15) break;
    v |= (c & 127) << (7 * k);
    if (c < 128) {
      *len = v;
      *nb = k + 1;
      return v == 0 || v > SN_CHUNK_CAP ? SN_ERR_PREAMBLE : SN_OK;
    }
  }
  return SN_ERR_PREAMBLE;
}

// One chunk src[0..n) into dst, on `nl` lanes of a warp in lockstep (host: one lane): every lane reads the same tags
// and takes the same branches; the lanes share each literal copy, and a copy moves in rounds of min(offset, nl) bytes
// (l4_copy_match).  Writes exactly the preamble's length, or fails.
Z_HD int32_t sn_decode_chunk(const uint8_t *src, uint32_t n, uint8_t *dst, uint32_t lane, uint32_t nl) {
  uint32_t raw = 0, ip = 0;
  const int32_t rc = sn_preamble(src, n, &raw, &ip);
  if (rc) return rc;
  uint32_t op = 0;
  while (ip < n) {
    const uint32_t tag = src[ip++], type = tag & 3;
    if (type == 0) {
      uint64_t L = tag >> 2;
      if (L >= 60) {
        const uint32_t b = (uint32_t)L - 59;
        if (b > n - ip) return SN_ERR_LITERAL;
        L = 0;
        for (uint32_t k = 0; k < b; k++) L |= (uint64_t)src[ip + k] << (8 * k);
        ip += b;
      }
      L += 1;
      if (L > n - ip) return SN_ERR_LITERAL;
      if (L > raw - op) return SN_ERR_LONG;
      for (uint32_t k = lane; k < L; k += nl) dst[op + k] = src[ip + k];
      ip += (uint32_t)L;
      op += (uint32_t)L;
      continue;
    }
    const uint32_t eb = type == 1 ? 1 : type == 2 ? 2 : 4;
    if (eb > n - ip) return SN_ERR_COPY;
    uint32_t len, off;
    if (type == 1) {
      len = ((tag >> 2) & 7) + 4;
      off = ((tag >> 5) << 8) | src[ip];
    } else {
      len = (tag >> 2) + 1;
      off = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8);
      if (type == 3) off |= ((uint32_t)src[ip + 2] << 16) | ((uint32_t)src[ip + 3] << 24);
    }
    ip += eb;
    if (off == 0 || off > op) return SN_ERR_OFFSET;
    if (len > raw - op) return SN_ERR_LONG;
    l4_copy_match(dst, op, off, len, lane, nl);
    op += len;
  }
  z_sync();
  return op == raw ? SN_OK : SN_ERR_SHORT;
}

// The block and chunk headers of a segment's stream in[0..n) that must decode to `expect` bytes, and every chunk's
// preamble.  sink(chunk, clen, out_off) is called for each chunk in stream order (out_off: where its raw bytes go);
// a nonzero return stops the walk with that status.  The walk and the chunk decoder give every framing error.
template <typename Sink>
Z_HD int32_t sn_walk(const uint8_t *in, uint64_t n, uint64_t expect, Sink &sink) {
  uint64_t ip = 0, op = 0;
  while (op < expect) {
    if (ip + 4 > n) return ip == n ? SN_ERR_LENGTH : SN_ERR_HEADER;
    const uint32_t raw = load_be32(in + ip);
    ip += 4;
    if (raw == 0 || raw > 0x7FFFFFFFu || raw > expect - op) return SN_ERR_BLOCK;
    uint32_t got = 0;
    while (got < raw) {
      if (ip + 4 > n) return SN_ERR_HEADER;
      const uint32_t c = load_be32(in + ip);
      ip += 4;
      if (c > SN_CHUNK_CAP || c > n - ip) return SN_ERR_CHUNK;
      uint32_t pre = 0, pn = 0;
      int32_t rc = sn_preamble(in + ip, c, &pre, &pn);
      if (rc) return rc;
      if (pre > raw - got) return SN_ERR_OVERRUN;
      rc = sink(in + ip, c, op + got);
      if (rc) return rc;
      got += pre;
      ip += c;
    }
    op += raw;
  }
  return ip != n ? SN_ERR_TRAILING : SN_OK;
}

// the host emulation's sink: decode each chunk at once, on one lane
struct SnDecodeSink {
  uint8_t *out;
  Z_HD int32_t operator()(const uint8_t *src, uint32_t c, uint64_t at) { return sn_decode_chunk(src, c, out + at, 0, 1); }
};

// A segment's stream in[0..n) into exactly `expect` bytes of out: the host emulation of the device reader.
static inline int32_t sn_decompress(const uint8_t *in, uint64_t n, uint8_t *out, uint64_t expect, uint64_t *out_len) {
  SnDecodeSink sink{out};
  const int32_t rc = sn_walk(in, n, expect, sink);
  *out_len = rc ? 0 : expect;
  return rc;
}

// a segment's error word: the status of its first failing chunk in stream order (k: the chunk's index in the
// segment; a walk error after k chunks has key k), largest word first; 0: no error
Z_HD unsigned long long sn_err_key(uint32_t k, int32_t rc) { return ((unsigned long long)(0xFFFFFFFFu - k) << 8) | (uint32_t)rc; }

// the device walk's sink: counts the chunks (FILL 0) or writes their units from `units` on (FILL 1)
template <int FILL>
struct SnUnitSink {
  ZUnit *units;
  uint8_t *dst;
  uint32_t seg, k;
  Z_HD int32_t operator()(const uint8_t *src, uint32_t c, uint64_t at) {
    if (FILL) {
      ZUnit u;
      u.src = src; u.dst = dst + at; u.clen = c; u.raw = 0; u.seg = seg; u.pad = k;
      units[k] = u;
    }
    k++;
    return SN_OK;
  }
};

// One thread per segment walks it.  FILL 0: the chunk count into nunit[s] and a walk error into err[s]; FILL 1: the
// units (ZUnit: the chunk, where its raw bytes go, pad = its index in the segment) from base[s] on.
template <int FILL>
__global__ void k_snwalk(const ZInSeg *__restrict__ segs, uint32_t nseg, uint32_t *__restrict__ nunit, const uint32_t *__restrict__ base,
                         ZUnit *__restrict__ units, unsigned long long *__restrict__ err) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const ZInSeg z = segs[s];
  if (FILL && !nunit[s]) return;
  SnUnitSink<FILL> sink{FILL ? units + base[s] : nullptr, z.dst + 4, s, 0};
  const int32_t rc = sn_walk(z.src + 4, z.len - 8, z.body, sink);
  if (!FILL) {
    nunit[s] = sink.k;
    err[s] = rc ? sn_err_key(sink.k, rc) : 0;
  }
}

// one warp per chunk; a failing chunk offers its key to its segment's error word
constexpr int SNDEC_WARPS = 4;
__global__ void __launch_bounds__(SNDEC_WARPS * 32) k_snchunks(const ZUnit *__restrict__ units, uint32_t n, unsigned long long *__restrict__ err) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t b = blockIdx.x * SNDEC_WARPS + (threadIdx.x >> 5);
  if (b >= n) return;
  const ZUnit u = units[b];
  const int32_t rc = sn_decode_chunk(u.src, (uint32_t)u.clen, u.dst, lane, 32);
  if (lane == 0 && rc != SN_OK) atomicMax(err + u.seg, sn_err_key(u.pad, rc));
}

// one thread per segment: the image frame (TIF\x00, 4 zero bytes after the body) and the status from the error word
__global__ void k_snfinish(const ZInSeg *__restrict__ segs, uint32_t n, const unsigned long long *__restrict__ err, int32_t *__restrict__ status) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const unsigned long long e = err[s];
  z_image_frame(segs[s], 0, e ? (int32_t)(e & 0xFF) : SN_OK, status + s);
}

}  // namespace tezgpu

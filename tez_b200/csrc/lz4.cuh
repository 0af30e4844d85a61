// lz4.cuh -- Lz4Codec on the device: the writer's block compressor and the reader's chunk decoder.
//
// A compressed segment (SORT/IFile.java:351-420) is 'T' 'I' 'F' 0x01, the Lz4Codec stream of the uncompressed body and
// a big-endian CRC-32 over the stream.  Lz4Codec writes through Hadoop's BlockCompressorStream: the stream is a sequence
// of blocks, each a big-endian int32 raw length and one or more chunks, each a big-endian int32 compressed length and
// one raw LZ4 block (no frame format).  The chunks of a block decode to its raw length in total.  Java's reader decodes
// every chunk with LZ4_decompress_safe into a buffer of io.compression.codec.lz4.buffersize (262,144 bytes by default),
// so each chunk decodes on its own (no match reaches into an earlier chunk) to at most that many bytes.
//
// Writer: the body is cut into L4_BLOCK-byte blocks of one chunk each.  One CTA of L4_LANES threads compresses a
// block.  Lane l parses slice [l * L4_SLICE, (l + 1) * L4_SLICE) greedily with a hash table private to the lane
// (seeded with the L4_SLICE bytes before the slice) and skips ahead on misses the way LZ4's fast mode does, so the
// output does not depend on thread timing and incompressible data is cheap.  Pass 1 sizes each lane's sequences;
// thread 0 resolves the literal runs that cross lanes and places the lanes; pass 2 writes.  LZ4's end-of-block rules
// hold: the last 5 bytes are literals and no match starts within the last 12 bytes.  The compressor is
// __host__ __device__: tezgpu_debug_lz4_compress_emulate runs it on the host and yields the bytes the device writes.
//
// Reader: strict.  Every block's raw length is > 0, its chunks decode to exactly that length, and the blocks' raw
// lengths add up to rawLength - 4 with the stream ending right after the last block; anything else is an error.  A
// chunk follows LZ4_decompress_safe(src, dst, n, 262144) of liblz4, including its end-of-chunk conditions, except
// that a match offset of 0 is refused (liblz4 1.9 accepts it on one code path, with undefined output bytes).
#pragma once
#include "inflate.cuh"

namespace tezgpu {

// Raw bytes per written block.  A block's worst-case chunk (all literals: 1 + 255 + L4_BLOCK bytes) plus its 8 header
// bytes fits one 64 KiB checksum piece (k_crc_pieces) and one L4_SLOT, every offset is below 65,536 without a check,
// the block and the lanes' hash tables fit one SM's shared memory, and a segment has many blocks to spread over the
// SMs on both sides.  LZ4's window is 64 KiB, so larger blocks would gain little ratio.
constexpr uint32_t L4_BLOCK = TEZGPU_LZ4_BLOCK_BYTES;   // 65,024
constexpr uint32_t L4_LANES = 32;                      // threads per block (one warp)
constexpr uint32_t L4_SLICE = L4_BLOCK / L4_LANES;     // bytes parsed by one lane
constexpr uint32_t L4_HBITS = 11;                      // lane hash table: 2^L4_HBITS u16 positions
constexpr uint32_t L4_HSIZE = 1u << L4_HBITS;
constexpr uint32_t L4_SLOT = 65536;                    // device bytes per block: 8 header bytes + the chunk
constexpr uint32_t L4_CHUNK_CAP = 262144;              // Java's Lz4Decompressor buffer: a chunk decodes to at most this
constexpr uint32_t L4_MINMATCH = 4, L4_LASTLIT = 5, L4_MFLIMIT = 12;
constexpr uint32_t L4_SKIP_TRIGGER = 6;                // LZ4's skipTrigger: the step grows by one every 2^6 misses
static_assert(8 + 1 + 255 + L4_BLOCK <= L4_SLOT && L4_SLOT <= 64 * 1024, "a framed chunk must fit one slot and one CRC piece");
static_assert(L4_BLOCK % L4_LANES == 0 && L4_BLOCK < 65536, "slices and offsets");

// error reasons (tezgpu_debug_lz4_decompress_emulate returns them; the merger reports them as TEZGPU_E_FORMAT)
enum L4Err : int32_t {
  L4_OK = 0,
  L4_ERR_HEADER = 1,      // the stream ends inside a block or chunk length
  L4_ERR_BLOCK = 2,       // a block's raw length is not in 1 .. the body bytes still expected
  L4_ERR_CHUNK = 3,       // a chunk's compressed length is over 262,144 or runs past the end of the stream
  L4_ERR_LITERALS = 4,    // a literal run runs past the chunk, or the chunk does not end with its last literals
  L4_ERR_OFFSET = 5,      // match offset 0 or before the start of the chunk
  L4_ERR_MATCH = 6,       // match length past the chunk, or a match ending within 5 bytes of 262,144
  L4_ERR_OVERRUN = 7,     // the chunks decode past their block's raw length
  L4_ERR_TRAILING = 8,    // bytes after the last block
  L4_ERR_LENGTH = 9,      // the blocks add up to less than rawLength - 4
};

static inline const char *l4_err_name(int32_t e) {
  switch (e) {
    case L4_ERR_HEADER: return "truncated block header";
    case L4_ERR_BLOCK: return "block raw length outside the remaining rawLength - 4";
    case L4_ERR_CHUNK: return "chunk length over 262144 or past the end of the stream";
    case L4_ERR_LITERALS: return "literal run past the end of the chunk";
    case L4_ERR_OFFSET: return "invalid match offset";
    case L4_ERR_MATCH: return "invalid match length";
    case L4_ERR_OVERRUN: return "chunks decode past their block's raw length";
    case L4_ERR_TRAILING: return "bytes after the last block";
    case L4_ERR_LENGTH: return "decompressed length differs from rawLength - 4";
    default: return "ok";
  }
}

Z_HD uint32_t l4_min(uint32_t a, uint32_t b) { return a < b ? a : b; }
// bytes after the token that a literal / match length n (its nibble part included) takes: 0 below 15
Z_HD uint32_t l4_ext_bytes(uint32_t n) { return n >= 15 ? (n - 15) / 255 + 1 : 0; }
Z_HD uint32_t l4_put_ext(uint8_t *o, uint32_t n) {
  if (n < 15) return 0;
  uint32_t r = n - 15, k = 0;
  for (; r >= 255; r -= 255) o[k++] = 255;
  o[k++] = (uint8_t)r;
  return k;
}

// ------------------------------------------------------------------------------------------------ writer
struct L4Shared {
  uint8_t data[L4_BLOCK];
  uint16_t htab[L4_LANES][L4_HSIZE];
  uint32_t lhead[L4_LANES];    // literals from the slice start to the lane's first match
  uint32_t ltail[L4_LANES];    // literals from the lane's last match to the slice end
  uint32_t lnm[L4_LANES];      // matches of the lane
  uint32_t lbytes[L4_LANES];   // bytes of the lane's sequences, less the first one's token, literal length and literals
  uint32_t lcarry[L4_LANES];   // literals of earlier lanes that open the lane's first sequence
  uint32_t lout[L4_LANES];     // chunk offset of the lane's first token
  uint32_t run_dst[L4_LANES + 1], run_src[L4_LANES + 1], run_len[L4_LANES + 1];   // literal runs copied by every thread
  uint32_t fin_out, fin_len, bytes, clen;
};

Z_HD uint32_t l4_hash4(const uint8_t *d) {
  const uint32_t v = (uint32_t)d[0] | ((uint32_t)d[1] << 8) | ((uint32_t)d[2] << 16) | ((uint32_t)d[3] << 24);
  return (v * 2654435761u) >> (32 - L4_HBITS);
}

// Greedy parse of the lane's slice.  PASS 1: sizes; PASS 2: the sequences into out (the chunk), except the literals of
// the lane's first sequence, which go to run_* for all threads to copy.
template <int PASS>
Z_HD void l4_lane(L4Shared &sh, uint32_t lane, uint8_t *out) {
  const uint32_t clen = sh.clen;
  const uint32_t s0 = lane * L4_SLICE;
  if (PASS == 1) { sh.lnm[lane] = 0; sh.lhead[lane] = 0; sh.ltail[lane] = 0; sh.lbytes[lane] = 0; }
  if (s0 >= clen) return;
  const uint32_t s1 = l4_min(clen, s0 + L4_SLICE);
  const uint8_t *d = sh.data;
  uint16_t *ht = sh.htab[lane];
  for (uint32_t i = 0; i < L4_HSIZE; i++) ht[i] = ZEMPTY;
  for (uint32_t q = s0 >= L4_SLICE ? s0 - L4_SLICE : 0; q < s0 && q + 4 <= clen; q++) ht[l4_hash4(d + q)] = (uint16_t)q;
  // a match starts at most 12 bytes before the end of the block and ends at least 5 bytes before it
  const uint32_t start_lim = clen >= L4_MFLIMIT ? l4_min(s1, clen - L4_MFLIMIT + 1) : 0;
  const uint32_t end_lim = clen >= L4_LASTLIT ? l4_min(s1, clen - L4_LASTLIT) : 0;
  uint32_t p = s0, anchor = s0, nm = 0, bytes = 0, misses = 0;
  uint32_t o = PASS == 2 ? sh.lout[lane] : 0;
  while (p < start_lim) {
    const uint32_t h = l4_hash4(d + p);
    uint32_t cand = ht[h];
    ht[h] = (uint16_t)p;
    if (cand != ZEMPTY && p + L4_MINMATCH <= end_lim && d[cand] == d[p] && d[cand + 1] == d[p + 1] && d[cand + 2] == d[p + 2] &&
        d[cand + 3] == d[p + 3]) {
      uint32_t m = L4_MINMATCH;
      while (p + m < end_lim && d[cand + m] == d[p + m]) m++;
      while (p > anchor && cand > 0 && d[p - 1] == d[cand - 1]) { p--; cand--; m++; }
      const uint32_t off = p - cand, mt = m - L4_MINMATCH;
      if (nm == 0) {
        if (PASS == 1) {
          sh.lhead[lane] = p - s0;
          bytes += 2 + l4_ext_bytes(mt);
        } else {
          const uint32_t L = sh.lcarry[lane] + (p - s0);
          out[o++] = (uint8_t)((l4_min(L, 15) << 4) | l4_min(mt, 15));
          o += l4_put_ext(out + o, L);
          sh.run_dst[lane] = o; sh.run_src[lane] = p - L; sh.run_len[lane] = L;
          o += L;
        }
      } else {
        const uint32_t L = p - anchor;
        if (PASS == 1) {
          bytes += 1 + l4_ext_bytes(L) + L + 2 + l4_ext_bytes(mt);
        } else {
          out[o++] = (uint8_t)((l4_min(L, 15) << 4) | l4_min(mt, 15));
          o += l4_put_ext(out + o, L);
          for (uint32_t k = 0; k < L; k++) out[o + k] = d[anchor + k];
          o += L;
        }
      }
      if (PASS == 2) {
        out[o++] = (uint8_t)off;
        out[o++] = (uint8_t)(off >> 8);
        o += l4_put_ext(out + o, mt);
      }
      nm++;
      p += m;
      anchor = p;
      misses = 0;
      if (p - 2 + 4 <= clen) ht[l4_hash4(d + p - 2)] = (uint16_t)(p - 2);
    } else {
      p += 1 + (misses++ >> L4_SKIP_TRIGGER);
    }
  }
  if (PASS == 1) {
    sh.lnm[lane] = nm;
    sh.ltail[lane] = s1 - anchor;
    sh.lbytes[lane] = bytes;
  }
}

// Thread 0, after pass 1: the literal runs that cross lanes, each lane's output offset, the last literals, the size.
Z_HD void l4_plan(L4Shared &sh) {
  const uint32_t clen = sh.clen;
  uint32_t pos = 0, carry = 0;
  for (uint32_t l = 0; l < L4_LANES; l++) {
    sh.run_len[l] = 0;
    const uint32_t s0 = l * L4_SLICE;
    if (s0 >= clen) continue;
    if (!sh.lnm[l]) { carry += l4_min(clen, s0 + L4_SLICE) - s0; continue; }
    const uint32_t L = carry + sh.lhead[l];
    sh.lcarry[l] = carry;
    sh.lout[l] = pos;
    pos += 1 + l4_ext_bytes(L) + L + sh.lbytes[l];
    carry = sh.ltail[l];
  }
  sh.fin_out = pos;
  sh.fin_len = carry;
  pos += 1 + l4_ext_bytes(carry);
  sh.run_dst[L4_LANES] = pos;
  sh.run_src[L4_LANES] = clen - carry;
  sh.run_len[L4_LANES] = carry;
  sh.bytes = pos + carry;
}

// Thread 0, after the plan: the last sequence's token and literal length, the block and chunk lengths before the chunk
Z_HD void l4_write_frame(const L4Shared &sh, uint8_t *slot) {
  store_be32(slot, sh.clen);
  store_be32(slot + 4, sh.bytes);
  uint8_t *out = slot + 8;
  out[sh.fin_out] = (uint8_t)(l4_min(sh.fin_len, 15) << 4);
  l4_put_ext(out + sh.fin_out + 1, sh.fin_len);
}

// the literal runs of the lanes' first sequences and the last literals, threads i0, i0 + step, ...
Z_HD void l4_copy_runs(const L4Shared &sh, uint8_t *out, uint32_t i0, uint32_t step) {
  for (uint32_t r = 0; r <= L4_LANES; r++) {
    const uint32_t n = sh.run_len[r], dst = sh.run_dst[r], src = sh.run_src[r];
    for (uint32_t k = i0; k < n; k += step) out[dst + k] = sh.data[src + k];
  }
}

// Host run of the device block compressor (lanes one after the other): slot receives 8 + sh.bytes bytes.
static inline void l4_compress_block_host(L4Shared &sh, const uint8_t *block, uint32_t clen, uint8_t *slot) {
  memcpy(sh.data, block, clen);
  sh.clen = clen;
  for (uint32_t l = 0; l < L4_LANES; l++) l4_lane<1>(sh, l, nullptr);
  l4_plan(sh);
  for (uint32_t l = 0; l < L4_LANES; l++) l4_lane<2>(sh, l, slot + 8);
  l4_write_frame(sh, slot);
  l4_copy_runs(sh, slot + 8, 0, 1);
}

// one CTA per block; segs / chunk numbering: ZSeg, z_chunk_part (common.cuh), with L4_BLOCK-byte chunks
__global__ void __launch_bounds__(L4_LANES)
    k_l4compress(const uint8_t *__restrict__ img, const ZSeg *__restrict__ segs, uint32_t P, uint8_t *__restrict__ slots,
                 uint32_t *__restrict__ csize) {
  extern __shared__ __align__(16) uint8_t l4_smem[];
  L4Shared &sh = *reinterpret_cast<L4Shared *>(l4_smem);
  const uint32_t c = blockIdx.x, tid = threadIdx.x;
  const ZSeg sg = segs[z_chunk_part(segs, P, c)];
  const uint64_t a = (uint64_t)(c - sg.chunk0) * L4_BLOCK;
  const uint32_t clen = (uint32_t)z_min64(L4_BLOCK, sg.body_len - a);
  const uint8_t *src = img + sg.body_off + a;
  for (uint32_t i = tid; i < clen; i += L4_LANES) sh.data[i] = src[i];
  if (tid == 0) sh.clen = clen;
  __syncthreads();
  l4_lane<1>(sh, tid, nullptr);
  __syncthreads();
  if (tid == 0) l4_plan(sh);
  __syncthreads();
  uint8_t *slot = slots + (uint64_t)c * L4_SLOT;
  l4_lane<2>(sh, tid, slot + 8);
  if (tid == 0) l4_write_frame(sh, slot);
  __syncthreads();
  l4_copy_runs(sh, slot + 8, tid, L4_LANES);
  if (tid == 0) csize[c] = 8 + sh.bytes;
}

// ------------------------------------------------------------------------------------------------ reader
// The decoder runs on `nl` lanes of a warp in lockstep (host: one lane): every lane reads the same bytes and takes the
// same branches; the lanes share the literal and match copies.
Z_HD void l4_copy_match(uint8_t *out, uint32_t op, uint32_t off, uint32_t len, uint32_t lane, uint32_t nl) {
  z_sync();
  const uint32_t step = off < nl ? off : nl;
  for (uint32_t base = 0; base < len; base += step) {
    const uint32_t k = base + lane;
    if (lane < step && k < len) out[op + k] = out[op + k - off];
    if (nl > 1) z_sync();
  }
}

// One chunk src[0..n) into dst, as LZ4_decompress_safe(src, dst, n, L4_CHUNK_CAP) but writing at most `limit` bytes
// (more is L4_ERR_OVERRUN).  *produced: the decoded bytes.
Z_HD int32_t l4_decode_chunk(const uint8_t *src, uint32_t n, uint8_t *dst, uint32_t limit, uint32_t *produced, uint32_t lane,
                             uint32_t nl) {
  const uint64_t C = L4_CHUNK_CAP;
  uint64_t ip = 0, op = 0;
  while (true) {
    if (ip >= n) return L4_ERR_LITERALS;
    const uint32_t tok = src[ip++];
    uint64_t L = tok >> 4;
    if (L == 15) {
      uint32_t s;
      do {
        if (ip >= n) return L4_ERR_LITERALS;
        s = src[ip++];
        L += s;
      } while (s == 255);
    }
    if (op + L + L4_MFLIMIT > C || ip + L + 8 > n) {   // the last literals: they must end the chunk
      if (ip + L != n || op + L > C) return L4_ERR_LITERALS;
      if (op + L > limit) return L4_ERR_OVERRUN;
      for (uint64_t k = lane; k < L; k += nl) dst[op + k] = src[ip + k];
      z_sync();
      *produced = (uint32_t)(op + L);
      return L4_OK;
    }
    if (op + L > limit) return L4_ERR_OVERRUN;
    for (uint64_t k = lane; k < L; k += nl) dst[op + k] = src[ip + k];
    ip += L;
    op += L;
    const uint32_t off = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8);
    ip += 2;
    if (off == 0 || off > op) return L4_ERR_OFFSET;
    uint64_t M = tok & 15;
    if (M == 15) {
      uint32_t s;
      do {
        s = src[ip++];
        if (ip + L4_LASTLIT > n) return L4_ERR_MATCH;
        M += s;
      } while (s == 255);
    }
    M += L4_MINMATCH;
    if (op + M + L4_LASTLIT > C) return L4_ERR_MATCH;
    if (op + M > limit) return L4_ERR_OVERRUN;
    l4_copy_match(dst, (uint32_t)op, off, (uint32_t)M, lane, nl);
    op += M;
  }
}

// A segment's compressed body in[0..n) walked block by block, chunk by chunk (any number of chunks per block), into
// exactly `expect` bytes of out.  The serial path of the device reader and the host emulation.
Z_HD int32_t l4_decompress(const uint8_t *in, uint64_t n, uint8_t *out, uint64_t expect, uint64_t *out_len, uint32_t lane = 0,
                           uint32_t nl = 1) {
  uint64_t ip = 0, op = 0;
  int32_t rc = L4_OK;
  while (op < expect) {
    if (ip + 4 > n) { rc = ip == n ? L4_ERR_LENGTH : L4_ERR_HEADER; break; }
    const uint32_t raw = load_be32(in + ip);
    ip += 4;
    if (raw == 0 || raw > 0x7FFFFFFFu || raw > expect - op) { rc = L4_ERR_BLOCK; break; }
    uint32_t got = 0;
    while (got < raw) {
      if (ip + 4 > n) { rc = L4_ERR_HEADER; break; }
      const uint32_t c = load_be32(in + ip);
      ip += 4;
      if (c > L4_CHUNK_CAP || c > n - ip) { rc = L4_ERR_CHUNK; break; }
      uint32_t r = 0;
      rc = l4_decode_chunk(in + ip, c, out + op + got, raw - got, &r, lane, nl);
      if (rc) break;
      got += r;
      ip += c;
    }
    if (rc) break;
    op += raw;
  }
  if (!rc && ip != n) rc = L4_ERR_TRAILING;
  z_sync();
  *out_len = op;
  return rc;
}

// One thread per segment walks the block headers on the assumption of one chunk per block.  FILL 0: counts the
// blocks into nblk[s] (0 = the assumption or the framing fails: the serial path decodes the segment); FILL 1: writes
// the blocks (ZUnit: the chunk and where its raw bytes go) from blk_base[s] on.
template <int FILL>
__global__ void k_l4walk(const ZInSeg *__restrict__ segs, uint32_t nseg, uint32_t *__restrict__ nblk, const uint32_t *__restrict__ blk_base,
                         ZUnit *__restrict__ blks) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const ZInSeg z = segs[s];
  if (FILL && !nblk[s]) return;
  const uint8_t *in = z.src + 4;
  const uint64_t n = z.len - 8;
  uint64_t ip = 0, op = 0;
  uint32_t k = 0;
  bool ok = true;
  while (ip < n) {
    if (ip + 8 > n) { ok = false; break; }
    const uint32_t raw = load_be32(in + ip), c = load_be32(in + ip + 4);
    ip += 8;
    if (raw == 0 || raw > L4_CHUNK_CAP || raw > z.body - op || c > L4_CHUNK_CAP || c > n - ip) { ok = false; break; }
    if (FILL) {
      ZUnit b;
      b.src = in + ip; b.dst = z.dst + 4 + op; b.clen = c; b.raw = raw; b.seg = s; b.pad = 0;
      blks[blk_base[s] + k] = b;
    }
    k++;
    ip += c;
    op += raw;
  }
  if (!FILL) nblk[s] = (ok && op == z.body && k) ? k : 0;
}

// one warp per block: a block that does not decode to exactly its raw length from exactly its chunk sends its segment
// to the serial path (slow[seg] = 1)
constexpr int L4DEC_WARPS = 4;
__global__ void __launch_bounds__(L4DEC_WARPS * 32) k_l4blocks(const ZUnit *__restrict__ blks, uint32_t n, int32_t *__restrict__ slow) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t b = blockIdx.x * L4DEC_WARPS + (threadIdx.x >> 5);
  if (b >= n) return;
  const ZUnit k = blks[b];
  uint32_t got = 0;   // the walk put clen and raw within L4_CHUNK_CAP
  const int32_t rc = l4_decode_chunk(k.src, (uint32_t)k.clen, k.dst, (uint32_t)k.raw, &got, lane, 32);
  if (lane == 0 && (rc != L4_OK || got != k.raw)) slow[k.seg] = 1;
}

// one warp per segment: the image frame (TIF\x00, 4 zero bytes after the body); segments marked slow (or never walked)
// are decoded again by the warp walking them serially, which is exact for multi-chunk blocks and names the errors
__global__ void __launch_bounds__(L4DEC_WARPS * 32) k_l4serial(const ZInSeg *__restrict__ segs, uint32_t n, const uint32_t *__restrict__ nblk,
                                                               const int32_t *__restrict__ slow, int32_t *__restrict__ status) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t s = blockIdx.x * L4DEC_WARPS + (threadIdx.x >> 5);
  if (s >= n) return;
  const ZInSeg z = segs[s];
  int32_t rc = L4_OK;
  if (!nblk[s] || slow[s]) {
    uint64_t got = 0;
    rc = l4_decompress(z.src + 4, z.len - 8, z.dst + 4, z.body, &got, lane, 32);
  }
  z_image_frame(z, lane, rc, status + s);
}

}  // namespace tezgpu

// inflate.cuh -- DefaultCodec reader: decodes the zlib body of a compressed IFile segment (SORT/IFile.java:764-809,
// readToMemory) on the device.  Accepts what Hadoop's DecompressorStream over zlib accepts: any valid zlib stream
// (stored / fixed / dynamic blocks, any window up to 32 KiB, flush points) and several complete streams back to back.
// The decoder is __host__ __device__: tezgpu_debug_inflate_emulate runs the same code on the host.
//
// Every read is bounded by the compressed length and every write by the expected body length (rawLength - 4), so a
// malformed stream yields an error code, never an out-of-bounds access.  Code-set rules follow zlib's inflate: an
// over-subscribed code is rejected; an incomplete one only when it is the code-length code or has a code longer than one
// bit; the literal/length code must give end-of-block a length.
#pragma once
#include "deflate.cuh"

namespace tezgpu {

// error reasons (tezgpu_debug_inflate_emulate returns them; the merger reports them as TEZGPU_E_FORMAT)
enum ZErr : int32_t {
  Z_OK = 0,
  Z_ERR_HEADER = 1,        // bad zlib header (method, window, check bits) or FDICT set
  Z_ERR_BTYPE = 2,         // block type 3
  Z_ERR_STORED_LEN = 3,    // stored block LEN / NLEN disagree
  Z_ERR_CODES = 4,         // over-subscribed or incomplete Huffman code, too many symbols, bad repeat
  Z_ERR_SYMBOL = 5,        // a code no symbol has, length symbol 286/287 or distance symbol 30/31
  Z_ERR_DIST = 6,          // distance before the start of the member
  Z_ERR_TRUNCATED = 7,     // input ends inside a member
  Z_ERR_ADLER = 8,         // Adler-32 mismatch
  Z_ERR_LENGTH = 9,        // output longer or shorter than expected
};

static inline const char *z_err_name(int32_t e) {
  switch (e) {
    case Z_ERR_HEADER: return "bad zlib header";
    case Z_ERR_BTYPE: return "invalid block type";
    case Z_ERR_STORED_LEN: return "stored block length mismatch";
    case Z_ERR_CODES: return "invalid Huffman code set";
    case Z_ERR_SYMBOL: return "invalid code";
    case Z_ERR_DIST: return "distance too far back";
    case Z_ERR_TRUNCATED: return "truncated stream";
    case Z_ERR_ADLER: return "incorrect data check";
    case Z_ERR_LENGTH: return "decompressed length differs from rawLength - 4";
    default: return "ok";
  }
}

constexpr uint32_t ZFBITS = 10;   // first-level decode table: codes of up to ZFBITS bits in one look-up

struct ZDec {
  uint16_t count[16];
  uint16_t sym[288];
  uint16_t fast[1 << ZFBITS];    // (code length << 9 | symbol) by the next ZFBITS input bits; 0 = longer or no code
};
struct ZInflateWork {
  ZDec lit, dist;
  uint8_t lens[352];   // code-length code at 0, a dynamic block's lengths at 32; fixed lengths at 0 (288) and 288 (32)
};

// The decoder runs on `nl` lanes of a warp in lockstep (host: one lane).  Every lane keeps the same bit-reader state
// and takes the same branches; lane 0 alone writes the code tables and literals, the lanes share long match copies,
// stored blocks and the Adler-32.  Shared state is published with z_sync().
Z_HD void z_sync() {
#ifdef __CUDA_ARCH__
  __syncwarp();
#endif
}
Z_HD int32_t z_bcast(int32_t v) {
#ifdef __CUDA_ARCH__
  return __shfl_sync(0xffffffffu, v, 0);
#else
  return v;
#endif
}

struct ZBitR {
  const uint8_t *p;
  uint64_t pos, end;
  uint64_t buf;
  uint32_t cnt;
  Z_HD bool need(uint32_t n) {
    while (cnt < n) {
      if (pos >= end) return false;
      buf |= (uint64_t)p[pos++] << cnt;
      cnt += 8;
    }
    return true;
  }
  // as many whole bytes as fit (at least up to 56 bits), without failing at the end of the input
  Z_HD void fill() {
    while (cnt <= 48 && pos < end) {
      buf |= (uint64_t)p[pos++] << cnt;
      cnt += 8;
    }
  }
  Z_HD uint32_t take(uint32_t n) {
    const uint32_t v = (uint32_t)(buf & ((1ull << n) - 1));
    buf >>= n;
    cnt -= n;
    return v;
  }
};

// type: 0 = code-length code, 1 = literal/length, 2 = distance (zlib's CODES / LENS / DISTS)
Z_HD int32_t z_dec_build(ZDec &h, const uint8_t *len, uint32_t n, int type) {
  for (uint32_t i = 0; i < (1u << ZFBITS); i++) h.fast[i] = 0;
  for (int l = 0; l < 16; l++) h.count[l] = 0;
  for (uint32_t i = 0; i < n; i++) h.count[len[i]]++;
  uint32_t max = 15;
  while (max >= 1 && h.count[max] == 0) max--;
  h.count[0] = 0;
  if (max == 0) return Z_OK;   // no codes: any decode through this table fails
  int32_t left = 1;
  for (int l = 1; l < 16; l++) {
    left <<= 1;
    left -= h.count[l];
    if (left < 0) return Z_ERR_CODES;
  }
  if (left > 0 && (type == 0 || max != 1)) return Z_ERR_CODES;
  uint16_t offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + h.count[l];
  for (uint32_t i = 0; i < n; i++)
    if (len[i]) h.sym[offs[len[i]]++] = (uint16_t)i;
  // first-level table: every canonical code of up to ZFBITS bits, bit-reversed, repeated over the unused high bits
  uint32_t code = 0, idx = 0;
  for (uint32_t l = 1; l <= ZFBITS; l++) {
    for (uint32_t c = 0; c < h.count[l]; c++, code++) {
      uint32_t r = 0, v = code;
      for (uint32_t b = 0; b < l; b++) { r = (r << 1) | (v & 1); v >>= 1; }
      const uint16_t e = (uint16_t)((l << 9) | h.sym[idx++]);
      for (uint32_t k = r; k < (1u << ZFBITS); k += 1u << l) h.fast[k] = e;
    }
    code <<= 1;
  }
  return Z_OK;
}

// lane 0 builds, every lane gets the verdict
Z_HD int32_t z_dec_build_w(ZDec &h, const uint8_t *len, uint32_t n, int type, uint32_t lane) {
  int32_t rc = Z_OK;
  z_sync();
  if (lane == 0) rc = z_dec_build(h, len, n, type);
  z_sync();
  return z_bcast(rc);
}

// one symbol: a first-level look-up, else the canonical walk one bit at a time; -1 = no such code, -2 = input ends
Z_HD int32_t z_decode(ZBitR &br, const ZDec &h) {
  br.fill();
  const uint32_t e = h.fast[br.buf & ((1u << ZFBITS) - 1)];
  const uint32_t l = e >> 9;
  if (l && l <= br.cnt) {
    br.take(l);
    return (int32_t)(e & 511);
  }
  int32_t code = 0, first = 0, index = 0;
  for (int len = 1; len < 16; len++) {
    if (!br.need(1)) return -2;
    code |= (int32_t)br.take(1);
    const int32_t c = h.count[len];
    if (code - c < first) return h.sym[index + (code - first)];
    index += c;
    first += c;
    first <<= 1;
    code <<= 1;
  }
  return -1;
}

// Adler-32 of p[0..n) over nl lanes (each a contiguous part, combined in order)
Z_HD uint32_t z_adler_lanes(const uint8_t *p, uint64_t n, uint32_t lane, uint32_t nl) {
  const uint64_t a = n * lane / nl, b = n * (lane + 1) / nl;
  uint32_t mine = z_adler_update(1, p + a, b - a);
#ifdef __CUDA_ARCH__
  uint32_t acc = 1;
  for (uint32_t j = 0; j < nl; j++) {
    const uint32_t aj = __shfl_sync(0xffffffffu, mine, (int)j);
    acc = z_adler_combine(acc, aj, n * (j + 1) / nl - n * j / nl);
  }
  return acc;
#else
  (void)nl;
  return mine;
#endif
}

// a back-reference of len bytes at distance dist: lane 0 alone for short ones, the lanes in rounds of min(dist, nl)
// bytes for long ones (a round only reads bytes written by earlier rounds)
Z_HD void z_copy_match(uint8_t *out, uint64_t op, uint32_t dist, uint32_t len, uint32_t lane, uint32_t nl) {
  if (nl == 1 || len < 32) {
    if (lane == 0)
      for (uint32_t k = 0; k < len; k++) out[op + k] = out[op + k - dist];
    return;
  }
  z_sync();
  const uint32_t step = dist < nl ? dist : nl;
  for (uint32_t base = 0; base < len; base += step) {
    const uint32_t k = base + lane;
    if (lane < step && k < len) out[op + k] = out[op + k - dist];
    z_sync();
  }
}

// one zlib member at br (byte aligned); output appended at out[*o], at most cap bytes in all
Z_HD int32_t z_inflate_member(ZBitR &br, uint8_t *out, uint64_t cap, uint64_t *o, ZInflateWork &w, uint32_t lane, uint32_t nl) {
  if (!br.need(16)) return Z_ERR_TRUNCATED;
  const uint32_t cmf = br.take(8), flg = br.take(8);
  if (((cmf << 8) | flg) % 31 != 0 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 0x20)) return Z_ERR_HEADER;
  const uint64_t m0 = *o;
  uint64_t op = m0;
  uint32_t bfinal;
  do {
    if (!br.need(3)) return Z_ERR_TRUNCATED;
    bfinal = br.take(1);
    const uint32_t type = br.take(2);
    if (type == 0) {
      br.take(br.cnt & 7);
      if (!br.need(32)) return Z_ERR_TRUNCATED;
      uint32_t len = br.take(16);
      const uint32_t nlen = br.take(16);
      if (len != (~nlen & 0xFFFF)) return Z_ERR_STORED_LEN;
      for (; len && br.cnt >= 8; len--) {           // bytes already in the bit buffer
        if (op >= cap) return Z_ERR_LENGTH;
        const uint8_t v = (uint8_t)br.take(8);
        if (lane == 0) out[op] = v;
        op++;
      }
      if (op + len > cap) return Z_ERR_LENGTH;
      if (br.pos + len > br.end) return Z_ERR_TRUNCATED;
      z_sync();
      for (uint32_t k = lane; k < len; k += nl) out[op + k] = br.p[br.pos + k];
      z_sync();
      op += len;
      br.pos += len;
      continue;
    }
    if (type == 3) return Z_ERR_BTYPE;
    if (type == 1) {
      z_sync();
      if (lane == 0) {
        for (uint32_t s = 0; s < 288; s++) w.lens[s] = (uint8_t)z_fixed_lit_len(s);
        for (uint32_t s = 288; s < 320; s++) w.lens[s] = 5;
      }
      z_dec_build_w(w.lit, w.lens, 288, 1, lane);
      z_dec_build_w(w.dist, w.lens + 288, 32, 2, lane);
    } else {
      if (!br.need(14)) return Z_ERR_TRUNCATED;
      const uint32_t nlen = br.take(5) + 257, ndist = br.take(5) + 1, ncode = br.take(4) + 4;
      if (nlen > 286 || ndist > 30) return Z_ERR_CODES;
      z_sync();
      if (lane == 0)
        for (int i = 0; i < 19; i++) w.lens[i] = 0;
      for (uint32_t i = 0; i < ncode; i++) {
        if (!br.need(3)) return Z_ERR_TRUNCATED;
        const uint8_t v = (uint8_t)br.take(3);
        if (lane == 0) w.lens[z_cl_order(i)] = v;
      }
      // the code-length code lives in the distance table until the lengths are read
      if (z_dec_build_w(w.dist, w.lens, 19, 0, lane)) return Z_ERR_CODES;
      uint32_t i = 0, prev = 0;
      while (i < nlen + ndist) {
        const int32_t s = z_decode(br, w.dist);
        if (s == -2) return Z_ERR_TRUNCATED;
        if (s < 0) return Z_ERR_CODES;
        if (s < 16) {
          if (lane == 0) w.lens[32 + i] = (uint8_t)s;
          prev = (uint32_t)s;
          i++;
          continue;
        }
        uint32_t v = 0, rep;
        if (s == 16) {
          if (i == 0) return Z_ERR_CODES;
          v = prev;
          if (!br.need(2)) return Z_ERR_TRUNCATED;
          rep = 3 + br.take(2);
        } else if (s == 17) {
          if (!br.need(3)) return Z_ERR_TRUNCATED;
          rep = 3 + br.take(3);
        } else {
          if (!br.need(7)) return Z_ERR_TRUNCATED;
          rep = 11 + br.take(7);
        }
        if (i + rep > nlen + ndist) return Z_ERR_CODES;
        if (lane == 0)
          for (uint32_t k = 0; k < rep; k++) w.lens[32 + i + k] = (uint8_t)v;
        prev = v;
        i += rep;
      }
      z_sync();
      const uint8_t eob = w.lens[32 + 256];
      if (eob == 0) return Z_ERR_CODES;
      if (z_dec_build_w(w.lit, w.lens + 32, nlen, 1, lane)) return Z_ERR_CODES;
      if (z_dec_build_w(w.dist, w.lens + 32 + nlen, ndist, 2, lane)) return Z_ERR_CODES;
    }
    while (true) {
      int32_t s = z_decode(br, w.lit);
      if (s == -2) return Z_ERR_TRUNCATED;
      if (s < 0) return Z_ERR_SYMBOL;
      if (s < 256) {
        if (op >= cap) return Z_ERR_LENGTH;
        if (lane == 0) out[op] = (uint8_t)s;
        op++;
        continue;
      }
      if (s == 256) break;
      if (s > 285) return Z_ERR_SYMBOL;
      uint32_t len, eb;
      z_len_base((uint32_t)s, len, eb);
      if (eb) {
        if (!br.need(eb)) return Z_ERR_TRUNCATED;
        len += br.take(eb);
      }
      s = z_decode(br, w.dist);
      if (s == -2) return Z_ERR_TRUNCATED;
      if (s < 0 || s > 29) return Z_ERR_SYMBOL;
      uint32_t dist;
      z_dist_base((uint32_t)s, dist, eb);
      if (eb) {
        if (!br.need(eb)) return Z_ERR_TRUNCATED;
        dist += br.take(eb);
      }
      if (dist > op - m0) return Z_ERR_DIST;
      if (op + len > cap) return Z_ERR_LENGTH;
      z_copy_match(out, op, dist, len, lane, nl);
      op += len;
    }
  } while (!bfinal);
  br.take(br.cnt & 7);
  if (!br.need(32)) return Z_ERR_TRUNCATED;
  uint32_t want = 0;
  for (int b = 0; b < 4; b++) want = (want << 8) | br.take(8);
  z_sync();
  if (z_adler_lanes(out + m0, op - m0, lane, nl) != want) return Z_ERR_ADLER;
  *o = op;
  return Z_OK;
}

// A segment's compressed body: one or more complete zlib members, decoding to exactly `expect` bytes.
Z_HD int32_t z_inflate(const uint8_t *in, uint64_t in_len, uint8_t *out, uint64_t expect, uint64_t *out_len, ZInflateWork &w,
                       uint32_t lane = 0, uint32_t nl = 1) {
  ZBitR br;
  br.p = in; br.pos = 0; br.end = in_len; br.buf = 0; br.cnt = 0;
  uint64_t o = 0;
  int32_t rc = Z_OK;
  do {
    rc = z_inflate_member(br, out, expect, &o, w, lane, nl);
    if (rc) break;
    // the trailer leaves the reader byte aligned: whole bytes still buffered belong to the next member
  } while (br.cnt || br.pos < br.end);
  z_sync();
  *out_len = o;
  if (rc) return rc;
  return o == expect ? Z_OK : Z_ERR_LENGTH;
}

// ------------------------------------------------------------------------------------------------ device reader
// one compressed segment to inflate: source bytes (TIF\x01 + zlib + CRC), destination image (TIF\x00 + body + 4)
struct ZInSeg {
  const uint8_t *src;
  uint64_t len;
  uint8_t *dst;
  uint64_t body;       // expected body bytes: rawLength - 4
};

// lane 0 of the warp that decoded segment z: the image frame around the body (TIF\x00, 4 zero bytes after it) and the
// decode status
__device__ __forceinline__ void z_image_frame(const ZInSeg &z, uint32_t lane, int32_t rc, int32_t *status) {
  if (lane == 0) {
    z.dst[0] = 'T'; z.dst[1] = 'I'; z.dst[2] = 'F'; z.dst[3] = 0;
    for (int b = 0; b < 4; b++) z.dst[4 + z.body + b] = 0;
    *status = rc;
  }
}

// the unit of the LZ4 and zstd block-parallel readers (one LZ4 block assumed to be one chunk, or one zstd frame with
// Frame_Content_Size): src[0..clen) decodes to exactly raw bytes at dst, or segment seg goes to the serial path
struct ZUnit {
  const uint8_t *src;
  uint8_t *dst;
  uint64_t clen, raw;
  uint32_t seg;         // index into the ZInSeg array
  uint32_t pad;
};

// one warp per segment (a Java-written segment is one serial zlib stream: parallelism comes from the segments); the
// decode tables of the warp's segment are in shared memory
constexpr int ZINF_WARPS = 4;
__global__ void __launch_bounds__(ZINF_WARPS * 32) k_zinflate(const ZInSeg *__restrict__ segs, uint32_t n, int32_t *__restrict__ status) {
  __shared__ ZInflateWork s_work[ZINF_WARPS];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t s = blockIdx.x * ZINF_WARPS + wid;
  if (s >= n) return;
  const ZInSeg z = segs[s];
  uint64_t got = 0;
  const int32_t rc = z_inflate(z.src + 4, z.len - 8, z.dst + 4, z.body, &got, s_work[wid], lane, 32);
  z_image_frame(z, lane, rc, status + s);
}

}  // namespace tezgpu

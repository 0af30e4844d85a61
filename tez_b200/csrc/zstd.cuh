// zstd.cuh -- ZStandardCodec on the device: the writer's frame compressor and the reader's frame decoder.
//
// A compressed segment (SORT/IFile.java:351-420) is 'T' 'I' 'F' 0x01, one or more Zstandard frames (RFC 8878) holding
// the uncompressed body, and a big-endian CRC-32 over the frame bytes.  ZStandardCodec (hadoop-common 3.4) writes
// through CompressorStream over ZStandardCompressor (libzstd's streaming compressor at io.compression.codec.zstd.level)
// and reads through DecompressorStream over ZStandardDecompressor (libzstd's streaming decoder, default parameters),
// which continues across concatenated frames.  A Java-written segment is normally one frame of many blocks without
// Frame_Content_Size.
//
// Writer: the body is cut into ZS_BLOCK-byte pieces and each becomes one independent frame: Single_Segment with
// Frame_Content_Size, no checksum, no dictionary, one block (compressed when smaller, raw otherwise).  One CTA of
// ZS_LANES threads compresses a piece: lane l parses slice [l * ZS_SLICE, (l + 1) * ZS_SLICE) greedily with a hash
// table private to the lane (the scheme of lz4.cuh), matches never use repeat offsets, sequences are coded with the
// predefined FSE distributions and literals with a Huffman code in direct 4-bit weights when every literal is below
// 128 and that is smaller, raw otherwise.  The output depends on the body alone; tezgpu_debug_zstd_compress_emulate
// runs the same __host__ __device__ code on the host.
//
// Reader: strict, what libzstd's default streaming decoder accepts (raw / RLE / compressed blocks, every literal and
// sequence mode, skippable frames, Content_Checksum) less dictionaries, and every malformed input is one of the ZsErr
// reasons.  Every read is bounded by the segment and every write by rawLength - 4.  The decoded literals of a block
// are placed at the end of the block's output range and consumed from there (a literal is never needed after the
// output reaches its position), so no scratch buffer is needed; matches read earlier output of the frame in place.
#pragma once
#include "lz4.cuh"

namespace tezgpu {

constexpr uint32_t ZS_BLOCK = TEZGPU_ZSTD_BLOCK_BYTES;   // 65,024 raw bytes per written frame
constexpr uint32_t ZS_LANES = 32;                       // threads per written frame (one warp)
constexpr uint32_t ZS_SLICE = ZS_BLOCK / ZS_LANES;      // bytes parsed by one lane
constexpr uint32_t ZS_HBITS = 10;                       // lane hash table: 2^ZS_HBITS u16 positions
constexpr uint32_t ZS_HSIZE = 1u << ZS_HBITS;
constexpr uint32_t ZS_MINMATCH = 4;
constexpr uint32_t ZS_LSEQ = ZS_SLICE / ZS_MINMATCH + 1;   // sequences one lane can find
constexpr uint32_t ZS_SLOT = 65536;                     // device bytes per written frame
constexpr uint32_t ZS_HUF_MIN = 64;                     // fewer literals stay raw
constexpr uint32_t ZS_BLOCK_MAX = 128 * 1024;           // Block_Maximum_Size cap
constexpr uint64_t ZS_WINDOW_MAX = (1ull << 27) + 1;    // libzstd's default window limit (ZSTD_WINDOWLOG_LIMIT_DEFAULT)
constexpr uint32_t ZS_MAGIC = 0xFD2FB528u;
static_assert(TEZGPU_ZSTD_FRAME_BOUND == ZS_BLOCK + 10 && TEZGPU_ZSTD_FRAME_BOUND <= ZS_SLOT && ZS_SLOT <= 64 * 1024,
              "a raw frame (4 magic + 1 descriptor + 2 content size + 3 block header + the piece) fits one slot and CRC piece");
static_assert(ZS_BLOCK % ZS_LANES == 0 && ZS_BLOCK < 65536, "slices and offsets");

// error reasons (tezgpu_debug_zstd_decompress_emulate returns them; the merger reports them as TEZGPU_E_FORMAT)
enum ZsErr : int32_t {
  ZS_OK = 0,
  ZS_ERR_MAGIC = 1,        // a frame does not start with the Zstandard or a skippable magic number
  ZS_ERR_RESERVED = 2,     // a reserved bit is set (frame header descriptor, sequence modes)
  ZS_ERR_DICT = 3,         // nonzero Dictionary_ID
  ZS_ERR_WINDOW = 4,       // Window_Size over libzstd's default limit (2^27 + 1)
  ZS_ERR_BLOCK_TYPE = 5,   // block type 3
  ZS_ERR_BLOCK_SIZE = 6,   // a block over Block_Maximum_Size (compressed or decoded)
  ZS_ERR_LITERALS = 7,     // malformed literals header or Huffman table, or a treeless block with no table
  ZS_ERR_SEQUENCES = 8,    // malformed sequences header or FSE table, or a sequence needing literals that are not there
  ZS_ERR_BITSTREAM = 9,    // a Huffman or sequence bitstream that is empty, unterminated or not consumed exactly
  ZS_ERR_OFFSET = 10,      // offset 0, before the frame start or beyond the window
  ZS_ERR_CONTENT_SIZE = 11,  // decoded bytes differ from Frame_Content_Size
  ZS_ERR_CHECKSUM = 12,    // Content_Checksum mismatch
  ZS_ERR_LENGTH = 13,      // the frames add up to more or less than rawLength - 4
  ZS_ERR_TRAILING = 14,    // bytes after the last frame
  ZS_ERR_TRUNCATED = 15,   // the stream ends inside a frame
};

static inline const char *zs_err_name(int32_t e) {
  switch (e) {
    case ZS_ERR_MAGIC: return "bad frame magic";
    case ZS_ERR_RESERVED: return "reserved bit set";
    case ZS_ERR_DICT: return "dictionary id set";
    case ZS_ERR_WINDOW: return "window size over 2^27";
    case ZS_ERR_BLOCK_TYPE: return "reserved block type";
    case ZS_ERR_BLOCK_SIZE: return "block over Block_Maximum_Size";
    case ZS_ERR_LITERALS: return "malformed literals section";
    case ZS_ERR_SEQUENCES: return "malformed sequences section";
    case ZS_ERR_BITSTREAM: return "bitstream not consumed exactly";
    case ZS_ERR_OFFSET: return "invalid match offset";
    case ZS_ERR_CONTENT_SIZE: return "decoded size differs from Frame_Content_Size";
    case ZS_ERR_CHECKSUM: return "content checksum mismatch";
    case ZS_ERR_LENGTH: return "decompressed length differs from rawLength - 4";
    case ZS_ERR_TRAILING: return "bytes after the last frame";
    case ZS_ERR_TRUNCATED: return "truncated frame";
    default: return "ok";
  }
}

// ------------------------------------------------------------------------------------------------ code tables (RFC 8878 3.1.1.3.2)
// one copy for the device (constant bank) and one for the host emulation
#ifdef __CUDA_ARCH__
#define ZS_TAB(name) name##_d
#else
#define ZS_TAB(name) name##_h
#endif
#define ZS_DEF_TABLE(type, name, ...)                    \
  static constexpr type name##_h[] = {__VA_ARGS__};      \
  __constant__ const type name##_d[] = {__VA_ARGS__};

ZS_DEF_TABLE(uint32_t, zs_ll_base, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64,
             128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536)
ZS_DEF_TABLE(uint8_t, zs_ll_bits, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12,
             13, 14, 15, 16)
ZS_DEF_TABLE(uint32_t, zs_ml_base, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28,
             29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387,
             32771, 65539)
ZS_DEF_TABLE(uint8_t, zs_ml_bits, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1,
             1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16)
// predefined distributions (accuracy logs 6, 5, 6)
ZS_DEF_TABLE(int16_t, zs_ll_norm, 4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1,
             -1, -1, -1)
ZS_DEF_TABLE(int16_t, zs_of_norm, 1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1)
ZS_DEF_TABLE(int16_t, zs_ml_norm, 1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
             1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1)

// table index: literal lengths, offsets, match lengths (the order of the sequence section's descriptions)
enum : uint32_t { ZS_LL = 0, ZS_OF = 1, ZS_ML = 2 };
Z_HD uint32_t zs_max_sym(uint32_t t) { return t == ZS_LL ? 35 : t == ZS_OF ? 31 : 52; }
Z_HD uint32_t zs_max_log(uint32_t t) { return t == ZS_OF ? 8 : 9; }
Z_HD const int16_t *zs_def_norm(uint32_t t, uint32_t *nsym, uint32_t *log) {
  if (t == ZS_LL) { *nsym = 36; *log = 6; return ZS_TAB(zs_ll_norm); }
  if (t == ZS_OF) { *nsym = 29; *log = 5; return ZS_TAB(zs_of_norm); }
  *nsym = 53; *log = 6;
  return ZS_TAB(zs_ml_norm);
}

Z_HD uint32_t zs_le16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
Z_HD uint32_t zs_le24(const uint8_t *p) { return zs_le16(p) | ((uint32_t)p[2] << 16); }
Z_HD uint32_t zs_le32(const uint8_t *p) { return zs_le24(p) | ((uint32_t)p[3] << 24); }
Z_HD uint64_t zs_le(const uint8_t *p, uint32_t n) {
  uint64_t v = 0;
  for (uint32_t i = 0; i < n; i++) v |= (uint64_t)p[i] << (8 * i);
  return v;
}
Z_HD uint64_t zs_min(uint64_t a, uint64_t b) { return a < b ? a : b; }

// ------------------------------------------------------------------------------------------------ XXH64 (Content_Checksum)
constexpr uint64_t XXP1 = 11400714785074694791ull, XXP2 = 14029467366897019727ull, XXP3 = 1609587929392839161ull,
                   XXP4 = 9650029242287828579ull, XXP5 = 2870177450012600261ull;
Z_HD uint64_t xx_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
Z_HD uint64_t xx_round(uint64_t acc, uint64_t in) { return xx_rotl(acc + in * XXP2, 31) * XXP1; }
Z_HD uint64_t xx_merge(uint64_t h, uint64_t v) { return (h ^ xx_round(0, v)) * XXP1 + XXP4; }
Z_HD uint64_t xxh64(const uint8_t *p, uint64_t n) {
  uint64_t h, i = 0;
  if (n >= 32) {
    uint64_t v1 = XXP1 + XXP2, v2 = XXP2, v3 = 0, v4 = 0 - XXP1;
    for (; i + 32 <= n; i += 32) {
      v1 = xx_round(v1, zs_le(p + i, 8));
      v2 = xx_round(v2, zs_le(p + i + 8, 8));
      v3 = xx_round(v3, zs_le(p + i + 16, 8));
      v4 = xx_round(v4, zs_le(p + i + 24, 8));
    }
    h = xx_rotl(v1, 1) + xx_rotl(v2, 7) + xx_rotl(v3, 12) + xx_rotl(v4, 18);
    h = xx_merge(h, v1); h = xx_merge(h, v2); h = xx_merge(h, v3); h = xx_merge(h, v4);
  } else {
    h = XXP5;
  }
  h += n;
  for (; i + 8 <= n; i += 8) h = xx_rotl(h ^ xx_round(0, zs_le(p + i, 8)), 27) * XXP1 + XXP4;
  if (i + 4 <= n) { h = xx_rotl(h ^ (zs_le(p + i, 4) * XXP1), 23) * XXP2 + XXP3; i += 4; }
  for (; i < n; i++) h = xx_rotl(h ^ (p[i] * XXP5), 11) * XXP1;
  h ^= h >> 33; h *= XXP2; h ^= h >> 29; h *= XXP3; h ^= h >> 32;
  return h;
}

// ------------------------------------------------------------------------------------------------ bit readers
// backward bitstream (Huffman streams, FSE streams): read from the last byte towards the first, the highest set bit of
// the last byte marks the start; bits past the first byte read as 0 and drive rem negative
struct ZsBitB {
  const uint8_t *p;
  int64_t pos, rem;    // bytes not yet loaded; bits not yet consumed (< 0: over-read)
  uint64_t c;
  uint32_t n;          // valid bits in the low end of c
  Z_HD bool init(const uint8_t *src, uint64_t size) {
    if (!size || !src[size - 1]) return false;
    p = src; pos = (int64_t)size; c = 0; n = 0;
    const uint32_t pad = 8 - z_log2(src[size - 1]);
    rem = (int64_t)size * 8 - pad;
    refill();
    n -= pad;
    return true;
  }
  Z_HD void refill() {
    while (n <= 56 && pos > 0) { c = (c << 8) | p[--pos]; n += 8; }
  }
  Z_HD uint32_t peek(uint32_t k) {
    if (n < k) {
      refill();
      if (n < k) { c <<= (k - n); n = k; }
    }
    return k ? (uint32_t)((c >> (n - k)) & ((1ull << k) - 1)) : 0;
  }
  Z_HD void skip(uint32_t k) { n -= k; rem -= k; }
  Z_HD uint32_t read(uint32_t k) { const uint32_t v = peek(k); skip(k); return v; }
};

// forward LSB-first reader of a table description: bits past n read as 0
Z_HD uint32_t zs_fwd_peek(const uint8_t *p, uint64_t n, uint64_t bit, uint32_t k) {
  const uint64_t b = bit >> 3;
  uint64_t v = 0;
  for (uint32_t i = 0; i < 8; i++)
    if (b + i < n) v |= (uint64_t)p[b + i] << (8 * i);
  return (uint32_t)((v >> (bit & 7)) & ((1ull << k) - 1));
}

// ------------------------------------------------------------------------------------------------ FSE tables
// An FSE table description (RFC 8878 4.1.1) as libzstd's FSE_readNCount reads it: norm[0..*nsym), the accuracy log;
// returns the bytes it takes, or -1.
Z_HD int32_t zs_ncount(const uint8_t *p, uint64_t n, uint32_t maxsv, uint32_t maxlog, int16_t *norm, uint32_t *log_out,
                       uint32_t *nsym) {
  for (uint32_t s = 0; s <= maxsv; s++) norm[s] = 0;
  uint64_t bit = 0;
  const uint32_t log = zs_fwd_peek(p, n, bit, 4) + 5;
  bit += 4;
  if (log > maxlog) return -1;
  int32_t remaining = (1 << log) + 1, threshold = 1 << log;
  uint32_t nbits = log + 1, ch = 0;
  bool prev0 = false;
  for (;;) {
    if (prev0) {
      uint32_t r;
      while ((r = zs_fwd_peek(p, n, bit, 2)) == 3 && bit < 8 * n + 64) { ch += 3; bit += 2; }
      ch += r;
      bit += 2;
      if (ch >= maxsv + 1) break;
    }
    const int32_t max = (2 * threshold - 1) - remaining;
    int32_t count;
    const uint32_t low = zs_fwd_peek(p, n, bit, nbits - 1);
    if ((int32_t)low < max) {
      count = (int32_t)low;
      bit += nbits - 1;
    } else {
      count = (int32_t)(zs_fwd_peek(p, n, bit, nbits) & (2 * threshold - 1));
      if (count >= threshold) count -= max;
      bit += nbits;
    }
    count--;
    remaining -= count >= 0 ? count : -count;
    norm[ch++] = (int16_t)count;
    prev0 = count == 0;
    if (remaining < threshold) {
      if (remaining <= 1) break;
      nbits = z_log2((uint32_t)remaining) + 1;
      threshold = 1 << (nbits - 1);
    }
    if (ch >= maxsv + 1) break;
  }
  if (remaining != 1 || ch > maxsv + 1) return -1;
  const uint64_t used = (bit + 7) >> 3;
  if (used > n) return -1;
  *log_out = log;
  *nsym = ch;
  return (int32_t)used;
}

// decoding table: entry = symbol | nbBits << 8 | baseline << 16
Z_HD void zs_fse_build(uint32_t *tab, const int16_t *norm, uint32_t nsym, uint32_t log, uint16_t *next) {
  const uint32_t size = 1u << log;
  uint32_t high = size - 1;
  for (uint32_t s = 0; s < nsym; s++) {
    if (norm[s] == -1) { tab[high--] = s; next[s] = 1; }
    else next[s] = (uint16_t)(norm[s] > 0 ? norm[s] : 0);
  }
  const uint32_t step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  uint32_t pos = 0;
  for (uint32_t s = 0; s < nsym; s++)
    for (int32_t i = 0; i < norm[s]; i++) {
      tab[pos] = s;
      do { pos = (pos + step) & mask; } while (pos > high);
    }
  for (uint32_t u = 0; u < size; u++) {
    const uint32_t s = tab[u] & 0xFF;
    const uint32_t ns = next[s]++;
    const uint32_t nb = log - z_log2(ns);
    tab[u] = s | (nb << 8) | (((ns << nb) - size) << 16);
  }
}

// ------------------------------------------------------------------------------------------------ reader
constexpr uint32_t ZS_HUF_LOG_MAX = 12;   // libzstd's HUF_TABLELOG_MAX (the RFC's encoders stay at 11)

// per-warp decoder state (shared memory on the device): the tables persist across the blocks of a frame (treeless
// literals, repeat-mode sequence tables); lane 0 parses headers and builds tables and publishes its results here
struct ZsDec {
  uint16_t huf[1u << ZS_HUF_LOG_MAX];   // symbol | nbBits << 8
  uint32_t fse[3][512];                 // LL, OF, ML decoding tables
  uint32_t hw[64];                      // the Huffman weights' FSE table
  int16_t norm[256];
  uint16_t next[256];
  uint8_t w[256];
  uint32_t huf_log, flog[3];
  int32_t have_huf, have_fse;
  // lane 0's literals-section results
  int32_t lrc, lt, herr[4];
  uint32_t lsz, lhs, lend, ns, soff[4], ssz[4];
  // lane 0's sequences-section results
  int32_t src_;
  uint32_t nseq, sbs;
  int32_t ck;
};

// Huffman weights in FSE form (libzstd's FSE_decompress with two interleaved states, at most 255 weights)
Z_HD int32_t zs_huf_weights_fse(const uint8_t *p, uint32_t isz, ZsDec &d) {
  uint32_t log, nsym;
  const int32_t c = zs_ncount(p, isz, 255, 6, d.norm, &log, &nsym);
  if (c < 0) return -1;
  zs_fse_build(d.hw, d.norm, nsym, log, d.next);
  ZsBitB br;
  if (!br.init(p + c, isz - (uint32_t)c)) return -1;
  uint32_t s1 = br.read(log), s2 = br.read(log), cnt = 0;
  for (;;) {
    if (cnt > 253) return -1;
    uint32_t e = d.hw[s1];
    d.w[cnt++] = (uint8_t)e;
    s1 = (e >> 16) + br.read((e >> 8) & 0xFF);
    if (br.rem < 0) { d.w[cnt++] = (uint8_t)d.hw[s2]; break; }
    if (cnt > 253) return -1;
    e = d.hw[s2];
    d.w[cnt++] = (uint8_t)e;
    s2 = (e >> 16) + br.read((e >> 8) & 0xFF);
    if (br.rem < 0) { d.w[cnt++] = (uint8_t)d.hw[s1]; break; }
  }
  return (int32_t)cnt;
}

// a Huffman tree description (RFC 8878 4.2.1) into d.huf; returns the bytes it takes, or -1
Z_HD int32_t zs_huf_table(const uint8_t *p, uint32_t m, ZsDec &d) {
  if (m < 1) return -1;
  const uint32_t hb = p[0];
  uint32_t isz, nw;
  if (hb >= 128) {
    nw = hb - 127;
    isz = (nw + 1) / 2;
    if (isz + 1 > m) return -1;
    for (uint32_t i = 0; i < nw; i++) d.w[i] = (i & 1) ? (p[1 + i / 2] & 15) : (p[1 + i / 2] >> 4);
  } else {
    isz = hb;
    if (isz + 1 > m) return -1;
    const int32_t r = zs_huf_weights_fse(p + 1, isz, d);
    if (r < 0) return -1;
    nw = (uint32_t)r;
  }
  uint32_t rank[ZS_HUF_LOG_MAX + 1] = {}, total = 0;
  for (uint32_t i = 0; i < nw; i++) {
    if (d.w[i] > ZS_HUF_LOG_MAX) return -1;
    rank[d.w[i]]++;
    total += (1u << d.w[i]) >> 1;
  }
  if (!total) return -1;
  const uint32_t log = z_log2(total) + 1;
  if (log > ZS_HUF_LOG_MAX) return -1;
  const uint32_t rest = (1u << log) - total, lw = z_log2(rest) + 1;
  if ((1u << (lw - 1)) != rest) return -1;
  d.w[nw] = (uint8_t)lw;
  rank[lw]++;
  if (rank[1] < 2 || (rank[1] & 1)) return -1;
  uint32_t start[ZS_HUF_LOG_MAX + 2], cur = 0;
  for (uint32_t w = 1; w <= log; w++) { start[w] = cur; cur += rank[w] << (w - 1); }
  for (uint32_t s = 0; s <= nw; s++) {
    const uint32_t w = d.w[s];
    if (!w) continue;
    const uint32_t len = 1u << (w - 1), e = s | ((log + 1 - w) << 8);
    for (uint32_t k = 0; k < len; k++) d.huf[start[w] + k] = (uint16_t)e;
    start[w] += len;
  }
  d.huf_log = log;
  return (int32_t)(isz + 1);
}

// Lane 0: the literals section header (and Huffman table) of a compressed block b[0..bn); room = output bytes the block
// may still produce, over = the error when the literals alone exceed it.
Z_HD int32_t zs_lit_header(const uint8_t *b, uint32_t bn, ZsDec &d, uint64_t room, int32_t over) {
  if (bn < 1) return ZS_ERR_LITERALS;
  const uint32_t b0 = b[0], lt = b0 & 3, sf = (b0 >> 2) & 3;
  d.lt = (int32_t)lt;
  d.ns = 0;
  if (lt < 2) {
    const uint32_t hs = sf == 1 ? 2 : sf == 3 ? 3 : 1;
    if (bn < hs) return ZS_ERR_LITERALS;
    const uint32_t size = hs == 1 ? b0 >> 3 : hs == 2 ? (b0 >> 4) | ((uint32_t)b[1] << 4)
                                                      : (b0 >> 4) | ((uint32_t)b[1] << 4) | ((uint32_t)b[2] << 12);
    if (size > ZS_BLOCK_MAX) return ZS_ERR_LITERALS;
    if (size > room) return over;
    const uint32_t body = lt == 0 ? size : 1;
    if (body > bn - hs) return ZS_ERR_LITERALS;
    d.lsz = size; d.lhs = hs; d.lend = hs + body;
    return ZS_OK;
  }
  const uint32_t hs = sf < 2 ? 3 : sf == 2 ? 4 : 5, ns = sf == 0 ? 1 : 4, bits = sf < 2 ? 10 : sf == 2 ? 14 : 18;
  if (bn < hs) return ZS_ERR_LITERALS;
  const uint64_t h = zs_le(b, hs);
  const uint32_t regen = (uint32_t)((h >> 4) & ((1u << bits) - 1)), comp = (uint32_t)((h >> (4 + bits)) & ((1u << bits) - 1));
  if (regen > ZS_BLOCK_MAX || (ns == 4 && regen < 6)) return ZS_ERR_LITERALS;
  if (regen > room) return over;
  if (comp > bn - hs) return ZS_ERR_LITERALS;
  uint32_t q = hs, m = comp;
  if (lt == 2) {
    const int32_t t = zs_huf_table(b + q, m, d);
    if (t < 0) return ZS_ERR_LITERALS;
    q += (uint32_t)t; m -= (uint32_t)t;
    d.have_huf = 1;
  } else if (!d.have_huf) {
    return ZS_ERR_LITERALS;
  }
  if (ns == 1) {
    d.soff[0] = q; d.ssz[0] = m;
  } else {
    if (m < 10) return ZS_ERR_LITERALS;
    const uint32_t s1 = zs_le16(b + q), s2 = zs_le16(b + q + 2), s3 = zs_le16(b + q + 4);
    if ((uint64_t)s1 + s2 + s3 + 6 > m) return ZS_ERR_LITERALS;
    d.soff[0] = q + 6; d.ssz[0] = s1;
    d.soff[1] = d.soff[0] + s1; d.ssz[1] = s2;
    d.soff[2] = d.soff[1] + s2; d.ssz[2] = s3;
    d.soff[3] = d.soff[2] + s3; d.ssz[3] = m - 6 - s1 - s2 - s3;
  }
  d.ns = ns; d.lsz = regen; d.lhs = hs; d.lend = hs + comp;
  return ZS_OK;
}

// one Huffman stream into dst[0..cnt); 0 or ZS_ERR_BITSTREAM
Z_HD int32_t zs_huf_stream(const uint8_t *p, uint32_t n, uint8_t *dst, uint32_t cnt, const ZsDec &d) {
  ZsBitB br;
  if (!br.init(p, n)) return ZS_ERR_BITSTREAM;
  const uint32_t log = d.huf_log;
  for (uint32_t i = 0; i < cnt; i++) {
    const uint32_t e = d.huf[br.peek(log)];
    dst[i] = (uint8_t)e;
    br.skip(e >> 8);
  }
  return br.rem == 0 ? ZS_OK : ZS_ERR_BITSTREAM;
}

// Lane 0: the sequences section header and tables of s[0..sn)
Z_HD int32_t zs_seq_header(const uint8_t *s, uint32_t sn, ZsDec &d) {
  if (sn < 1) return ZS_ERR_SEQUENCES;
  uint32_t ip = 0, nb = s[ip++];
  if (nb > 0x7F) {
    if (nb == 0xFF) {
      if (ip + 2 > sn) return ZS_ERR_SEQUENCES;
      nb = zs_le16(s + ip) + 0x7F00;
      ip += 2;
    } else {
      if (ip >= sn) return ZS_ERR_SEQUENCES;
      nb = ((nb - 0x80) << 8) + s[ip++];
    }
  }
  d.nseq = nb;
  if (nb == 0) {
    d.sbs = ip;
    return ip == sn ? ZS_OK : ZS_ERR_SEQUENCES;
  }
  if (ip + 1 > sn) return ZS_ERR_SEQUENCES;
  const uint32_t modes = s[ip++];
  if (modes & 3) return ZS_ERR_RESERVED;
  for (uint32_t t = 0; t < 3; t++) {
    const uint32_t mode = (modes >> (6 - 2 * t)) & 3;
    if (mode == 0) {
      uint32_t nsym, log;
      const int16_t *norm = zs_def_norm(t, &nsym, &log);
      zs_fse_build(d.fse[t], norm, nsym, log, d.next);
      d.flog[t] = log;
    } else if (mode == 1) {
      if (ip >= sn || s[ip] > zs_max_sym(t)) return ZS_ERR_SEQUENCES;
      d.fse[t][0] = s[ip++];
      d.flog[t] = 0;
    } else if (mode == 2) {
      uint32_t log, nsym;
      const int32_t c = zs_ncount(s + ip, sn - ip, zs_max_sym(t), zs_max_log(t), d.norm, &log, &nsym);
      if (c < 0) return ZS_ERR_SEQUENCES;
      zs_fse_build(d.fse[t], d.norm, nsym, log, d.next);
      d.flog[t] = log;
      ip += (uint32_t)c;
    } else if (!d.have_fse) {
      return ZS_ERR_SEQUENCES;
    }
  }
  d.have_fse = 1;
  d.sbs = ip;
  return ZS_OK;
}

// forward copy of len bytes from src to dst where src is another buffer or at or after dst in the same one
Z_HD void zs_move(uint8_t *dst, const uint8_t *src, uint32_t len, uint32_t lane, uint32_t nl) {
  if (!len || src == dst) return;
  const uint64_t gap = src > dst ? (uint64_t)(src - dst) : ~0ull;
  if (gap >= len) {
    for (uint32_t k = lane; k < len; k += nl) dst[k] = src[k];
  } else {
    const uint32_t step = gap < nl ? (uint32_t)gap : nl;
    for (uint32_t base = 0; base < len; base += step) {
      const uint32_t k = base + lane;
      if (lane < step && k < len) dst[k] = src[k];
      z_sync();
    }
  }
  z_sync();
}

// One compressed block b[0..bn) decoded at out[op0..); fstart: the frame's first output byte; E: the end of the bytes
// the block may write (over: the error past it); rep: the frame's repeat offsets.  *op_out: the end of its output.
Z_HD int32_t zs_block(const uint8_t *b, uint32_t bn, uint8_t *out, uint64_t op0, uint64_t fstart, uint64_t E, int32_t over,
                      uint64_t window, uint32_t *rep, ZsDec &d, uint32_t lane, uint32_t nl, uint64_t *op_out) {
  if (lane == 0) d.lrc = zs_lit_header(b, bn, d, E - op0, over);
  z_sync();
  int32_t rc = d.lrc;
  if (rc) { z_sync(); return rc; }
  const uint32_t lt = (uint32_t)d.lt, lsz = d.lsz, lend = d.lend;
  const uint64_t L0 = E - lsz;   // the decoded literals go to the end of the block's room
  const uint8_t *lp = out + L0;
  if (lt == 0) {
    lp = b + d.lhs;
  } else if (lt == 1) {
    const uint8_t v = b[d.lhs];
    for (uint32_t k = lane; k < lsz; k += nl) out[L0 + k] = v;
  } else {
    const uint32_t ns = d.ns, seg = ns == 1 ? lsz : (lsz + 3) / 4;
    for (uint32_t k = lane; k < ns; k += nl) {
      const uint32_t a = k * seg, cnt = k + 1 == ns ? lsz - a : seg;
      d.herr[k] = zs_huf_stream(b + d.soff[k], d.ssz[k], out + L0 + a, cnt, d);
    }
    z_sync();
    for (uint32_t k = 0; k < ns; k++) rc |= d.herr[k];
    if (rc) { z_sync(); return ZS_ERR_BITSTREAM; }
  }
  if (lane == 0) d.src_ = zs_seq_header(b + lend, bn - lend, d);
  z_sync();
  rc = d.src_;
  if (rc) { z_sync(); return rc; }
  const uint32_t nseq = d.nseq;
  uint64_t op = op0;
  uint32_t litrem = lsz;
  if (nseq) {
    ZsBitB br;
    if (!br.init(b + lend + d.sbs, bn - lend - d.sbs)) { z_sync(); return ZS_ERR_BITSTREAM; }
    const uint32_t *tl = d.fse[ZS_LL], *to = d.fse[ZS_OF], *tm = d.fse[ZS_ML];
    uint32_t sl = br.read(d.flog[ZS_LL]), so = br.read(d.flog[ZS_OF]), sm = br.read(d.flog[ZS_ML]);
    for (uint32_t i = 0; i < nseq; i++) {
      const uint32_t el = tl[sl], eo = to[so], em = tm[sm];
      const uint32_t oc = eo & 0xFF, mc = em & 0xFF, lc = el & 0xFF;
      const uint32_t ov = (1u << oc) + br.read(oc);
      const uint32_t ml = ZS_TAB(zs_ml_base)[mc] + br.read(ZS_TAB(zs_ml_bits)[mc]);
      const uint32_t ll = ZS_TAB(zs_ll_base)[lc] + br.read(ZS_TAB(zs_ll_bits)[lc]);
      uint32_t off;
      if (oc > 1) {
        off = ov - 3;
        rep[2] = rep[1]; rep[1] = rep[0]; rep[0] = off;
      } else {
        const uint32_t idx = ov - 1 + (ll == 0);
        if (idx == 0) {
          off = rep[0];
        } else {
          off = idx == 3 ? rep[0] - 1 : rep[idx];
          if (idx != 1) rep[2] = rep[1];
          rep[1] = rep[0];
          rep[0] = off;
        }
      }
      if (ll > litrem) { rc = ZS_ERR_SEQUENCES; break; }
      if (op + ml + litrem > E) { rc = over; break; }
      const uint64_t mp = op + ll;
      if (off == 0 || off > mp - fstart || off > window) { rc = ZS_ERR_OFFSET; break; }
      zs_move(out + op, lp, ll, lane, nl);
      lp += ll;
      litrem -= ll;
      z_copy_match(out, mp, off, ml, lane, nl);
      z_sync();
      op = mp + ml;
      if (i + 1 < nseq) {
        sl = (el >> 16) + br.read((el >> 8) & 0xFF);
        sm = (em >> 16) + br.read((em >> 8) & 0xFF);
        so = (eo >> 16) + br.read((eo >> 8) & 0xFF);
      }
    }
    if (!rc && br.rem != 0) rc = ZS_ERR_BITSTREAM;
    if (rc) { z_sync(); return rc; }
  }
  zs_move(out + op, lp, litrem, lane, nl);
  *op_out = op + litrem;
  return ZS_OK;
}

// the frame header at in[0..n): magic, descriptor, window, dictionary id, content size
struct ZsHdr {
  uint64_t window, fcs, bmax, skip;   // skip: a skippable frame's total length (0: a Zstandard frame)
  uint32_t hs;
  bool has_fcs, cksum;
};
Z_HD int32_t zs_header(const uint8_t *in, uint64_t n, ZsHdr &h) {
  if (n < 4) return ZS_ERR_TRUNCATED;
  const uint32_t magic = zs_le32(in);
  h.skip = 0;
  if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {
    if (n < 8) return ZS_ERR_TRUNCATED;
    const uint64_t sz = zs_le32(in + 4);
    if (sz > n - 8) return ZS_ERR_TRUNCATED;
    h.skip = 8 + sz;
    return ZS_OK;
  }
  if (magic != ZS_MAGIC) return ZS_ERR_MAGIC;
  if (n < 5) return ZS_ERR_TRUNCATED;
  const uint32_t fhd = in[4];
  if (fhd & 0x08) return ZS_ERR_RESERVED;
  const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, did_flag = fhd & 3;
  const uint32_t did_size = did_flag == 3 ? 4 : did_flag, fcs_size = fcs_flag == 0 ? single : 1u << fcs_flag;
  h.hs = 5 + !single + did_size + fcs_size;
  h.cksum = (fhd >> 2) & 1;
  if (n < h.hs) return ZS_ERR_TRUNCATED;
  uint32_t ip = 5;
  uint64_t window = 0;
  if (!single) {
    const uint32_t wd = in[ip++];
    const uint64_t base = 1ull << (10 + (wd >> 3));
    window = base + (base >> 3) * (wd & 7);
  }
  const uint64_t did = zs_le(in + ip, did_size);
  ip += did_size;
  uint64_t fcs = zs_le(in + ip, fcs_size);
  if (fcs_size == 2) fcs += 256;
  h.has_fcs = fcs_size > 0;
  h.fcs = fcs;
  if (single) window = fcs;
  h.bmax = zs_min(window, ZS_BLOCK_MAX);
  h.window = window < 1024 ? 1024 : window;
  if (did) return ZS_ERR_DICT;
  if (h.window > ZS_WINDOW_MAX) return ZS_ERR_WINDOW;
  return ZS_OK;
}

// One frame (or skippable frame) at in[0..n) decoded at out[op0..), at most up to out[cap]; *used: its length,
// *op_out: the end of its output.
Z_HD int32_t zs_frame(const uint8_t *in, uint64_t n, uint64_t *used, uint8_t *out, uint64_t op0, uint64_t cap, uint64_t *op_out,
                      ZsDec &d, uint32_t lane, uint32_t nl) {
  ZsHdr h;
  int32_t rc = zs_header(in, n, h);
  if (rc) return rc;
  if (h.skip) { *used = h.skip; *op_out = op0; return ZS_OK; }
  uint64_t lim = cap;
  int32_t over = ZS_ERR_LENGTH;
  if (h.has_fcs) {
    if (h.fcs > cap - op0) return ZS_ERR_LENGTH;
    lim = op0 + h.fcs;
    over = ZS_ERR_CONTENT_SIZE;
  }
  if (lane == 0) { d.have_huf = 0; d.have_fse = 0; }
  z_sync();
  uint32_t rep[3] = {1, 4, 8};
  uint64_t ip = h.hs, op = op0;
  bool last = false;
  while (!last) {
    if (n - ip < 3) return ZS_ERR_TRUNCATED;
    const uint32_t bh = zs_le24(in + ip), bt = (bh >> 1) & 3, bs = bh >> 3;
    last = bh & 1;
    ip += 3;
    if (bt == 3) return ZS_ERR_BLOCK_TYPE;
    if (bs > h.bmax) return ZS_ERR_BLOCK_SIZE;
    if (bs == 0 && bt != 1) continue;   // an empty raw or compressed block: libzstd's streaming decoder skips it
    if (bt == 0) {
      if (bs > n - ip) return ZS_ERR_TRUNCATED;
      if (bs > lim - op) return over;
      zs_move(out + op, in + ip, bs, lane, nl);
      ip += bs;
      op += bs;
    } else if (bt == 1) {
      if (n - ip < 1) return ZS_ERR_TRUNCATED;
      if (bs > lim - op) return over;
      const uint8_t v = in[ip];
      for (uint32_t k = lane; k < bs; k += nl) out[op + k] = v;
      z_sync();
      ip += 1;
      op += bs;
    } else {
      if (bs > n - ip) return ZS_ERR_TRUNCATED;
      if (bs >= ZS_BLOCK_MAX) return ZS_ERR_BLOCK_SIZE;
      const bool by_block = op + h.bmax <= lim;
      const uint64_t E = by_block ? op + h.bmax : lim;
      rc = zs_block(in + ip, bs, out, op, op0, E, by_block ? ZS_ERR_BLOCK_SIZE : over, h.window, rep, d, lane, nl, &op);
      if (rc) return rc;
      ip += bs;
    }
  }
  if (h.cksum) {
    if (n - ip < 4) return ZS_ERR_TRUNCATED;
    z_sync();
    if (lane == 0) d.ck = (uint32_t)xxh64(out + op0, op - op0) == zs_le32(in + ip);
    z_sync();
    const int32_t ok = d.ck;
    z_sync();
    if (!ok) return ZS_ERR_CHECKSUM;
    ip += 4;
  }
  if (h.has_fcs && op - op0 != h.fcs) return ZS_ERR_CONTENT_SIZE;
  *used = ip;
  *op_out = op;
  return ZS_OK;
}

// A segment's stream in[0..n): frames decoding to exactly `expect` bytes of out, nothing after the last one.  The serial
// path of the device reader and the host emulation.
Z_HD int32_t zs_decompress(const uint8_t *in, uint64_t n, uint8_t *out, uint64_t expect, uint64_t *out_len, ZsDec &d,
                           uint32_t lane = 0, uint32_t nl = 1) {
  uint64_t ip = 0, op = 0;
  int32_t rc = ZS_OK;
  while (ip < n) {
    if (op == expect) {
      const uint32_t magic = n - ip >= 4 ? zs_le32(in + ip) : 0;
      if (magic != ZS_MAGIC && (magic & 0xFFFFFFF0u) != 0x184D2A50u) { rc = ZS_ERR_TRAILING; break; }
    }
    uint64_t used = 0;
    rc = zs_frame(in + ip, n - ip, &used, out, op, expect, &op, d, lane, nl);
    if (rc) break;
    ip += used;
  }
  z_sync();
  if (!rc && op != expect) rc = ZS_ERR_LENGTH;
  *out_len = op;
  return rc;
}

// One thread per segment walks the frame and block headers.  FILL 0: counts the frames into nfr[s] (0 = a frame
// without Frame_Content_Size, or a framing error: the serial path decodes the segment); FILL 1: writes the frames
// (ZUnit: the frame, where its content goes, its Frame_Content_Size as raw) from fr_base[s] on.  Skippable frames are
// passed over.
template <int FILL>
__global__ void k_zswalk(const ZInSeg *__restrict__ segs, uint32_t nseg, uint32_t *__restrict__ nfr, const uint32_t *__restrict__ fr_base,
                         ZUnit *__restrict__ frs) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const ZInSeg z = segs[s];
  if (FILL && !nfr[s]) return;
  const uint8_t *in = z.src + 4;
  const uint64_t n = z.len - 8;
  uint64_t ip = 0, op = 0;
  uint32_t k = 0;
  bool ok = true;
  while (ip < n && ok) {
    ZsHdr h;
    if (zs_header(in + ip, n - ip, h)) { ok = false; break; }
    if (h.skip) { ip += h.skip; continue; }
    if (!h.has_fcs || h.fcs > z.body - op) { ok = false; break; }
    uint64_t q = ip + h.hs;
    bool last = false;
    while (!last) {
      if (n - q < 3) { ok = false; break; }
      const uint32_t bh = zs_le24(in + q), bt = (bh >> 1) & 3, bs = bh >> 3;
      last = bh & 1;
      q += 3 + (bt == 1 ? 1 : bs);
      if (bt == 3 || q > n) { ok = false; break; }
    }
    if (!ok) break;
    q += h.cksum ? 4 : 0;
    if (q > n) { ok = false; break; }
    if (FILL) {
      ZUnit f;
      f.src = in + ip; f.dst = z.dst + 4 + op; f.clen = q - ip; f.raw = h.fcs; f.seg = s; f.pad = 0;
      frs[fr_base[s] + k] = f;
    }
    k++;
    op += h.fcs;
    ip = q;
  }
  if (!FILL) nfr[s] = (ok && op == z.body && k) ? k : 0;
}

// one warp per frame: a frame that does not decode to exactly its content size from exactly its bytes sends its
// segment to the serial path (slow[seg] = 1)
constexpr int ZSD_WARPS = 2;
__global__ void __launch_bounds__(ZSD_WARPS * 32) k_zsframes(const ZUnit *__restrict__ frs, uint32_t n, int32_t *__restrict__ slow) {
  __shared__ ZsDec s_dec[ZSD_WARPS];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t f = blockIdx.x * ZSD_WARPS + wid;
  if (f >= n) return;
  const ZUnit fr = frs[f];
  uint64_t used = 0, got = 0;
  const int32_t rc = zs_frame(fr.src, fr.clen, &used, fr.dst, 0, fr.raw, &got, s_dec[wid], lane, 32);
  if (lane == 0 && (rc != ZS_OK || used != fr.clen || got != fr.raw)) slow[fr.seg] = 1;
}

// one warp per segment: the image frame (TIF\x00, 4 zero bytes after the body); segments marked slow (or never walked)
// are decoded by the warp walking them serially, which names the errors
__global__ void __launch_bounds__(ZSD_WARPS * 32) k_zsserial(const ZInSeg *__restrict__ segs, uint32_t n, const uint32_t *__restrict__ nfr,
                                                             const int32_t *__restrict__ slow, int32_t *__restrict__ status) {
  __shared__ ZsDec s_dec[ZSD_WARPS];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t s = blockIdx.x * ZSD_WARPS + wid;
  if (s >= n) return;
  const ZInSeg z = segs[s];
  int32_t rc = ZS_OK;
  if (!nfr[s] || slow[s]) {
    uint64_t got = 0;
    rc = zs_decompress(z.src + 4, z.len - 8, z.dst + 4, z.body, &got, s_dec[wid], lane, 32);
  }
  z_image_frame(z, lane, rc, status + s);
}

// ------------------------------------------------------------------------------------------------ writer
// FSE encoding table of a predefined distribution (libzstd's FSE_buildCTable)
struct ZsCTable {
  uint16_t state[64];
  int32_t dfs[53];      // deltaFindState
  uint32_t dnb[53];     // deltaNbBits
  uint32_t log;
};
struct ZsEncWork {
  ZBuildScratch scratch;
  ZsCTable ct[3];
  uint16_t hcode[128];
  uint8_t hlen[128], hw[128];
};
struct ZsShared {
  union {
    uint8_t data[ZS_BLOCK];   // the piece (parse, literal gather)
    ZsEncWork ew;             // then the entropy coders' tables
  };
  union {
    uint16_t htab[ZS_LANES][ZS_HSIZE];   // lane hash tables (parse)
    uint8_t lits[ZS_BLOCK];              // then the literals in order
  };
  uint16_t sll[ZS_LANES][ZS_LSEQ], sml[ZS_LANES][ZS_LSEQ], sof[ZS_LANES][ZS_LSEQ];   // each lane's sequences
  uint32_t freq[256];
  uint32_t lnm[ZS_LANES];      // sequences of the lane
  uint32_t llit[ZS_LANES];     // literal bytes of the lane's slice
  uint32_t lcarry[ZS_LANES];   // literals of earlier lanes that open the lane's first sequence
  uint32_t litbase[ZS_LANES];  // where the lane's literals go in lits
  uint32_t hbits[4];           // bits of the four Huffman streams
  uint32_t soff[4];            // their offsets in the slot
  uint32_t clen, nseq, nlit, huf, hlog, hmax, seq_at, bytes;
};
static_assert(sizeof(ZsEncWork) <= ZS_BLOCK, "the coders' tables fit in the piece's buffer");
static_assert(sizeof(ZsShared) <= 227 * 1024, "one CTA's shared memory on sm_90");

Z_HD uint32_t zs_hash4(const uint8_t *d) {
  const uint32_t v = (uint32_t)d[0] | ((uint32_t)d[1] << 8) | ((uint32_t)d[2] << 16) | ((uint32_t)d[3] << 24);
  return (v * 2654435761u) >> (32 - ZS_HBITS);
}

// greedy parse of the lane's slice into its sequences (literal run, match length, offset); matches end in the slice
Z_HD void zs_lane(ZsShared &sh, uint32_t lane) {
  const uint32_t clen = sh.clen, s0 = lane * ZS_SLICE;
  sh.lnm[lane] = 0;
  sh.llit[lane] = 0;
  if (s0 >= clen) return;
  const uint32_t s1 = l4_min(clen, s0 + ZS_SLICE);
  const uint8_t *d = sh.data;
  uint16_t *ht = sh.htab[lane];
  for (uint32_t i = 0; i < ZS_HSIZE; i++) ht[i] = ZEMPTY;
  for (uint32_t q = s0 >= ZS_SLICE ? s0 - ZS_SLICE : 0; q < s0 && q + 4 <= clen; q++) ht[zs_hash4(d + q)] = (uint16_t)q;
  uint32_t p = s0, anchor = s0, nm = 0, matched = 0, misses = 0;
  while (p + ZS_MINMATCH <= s1) {
    const uint32_t h = zs_hash4(d + p);
    uint32_t cand = ht[h];
    ht[h] = (uint16_t)p;
    if (cand != ZEMPTY && d[cand] == d[p] && d[cand + 1] == d[p + 1] && d[cand + 2] == d[p + 2] && d[cand + 3] == d[p + 3]) {
      uint32_t m = ZS_MINMATCH;
      while (p + m < s1 && d[cand + m] == d[p + m]) m++;
      while (p > anchor && cand > 0 && d[p - 1] == d[cand - 1]) { p--; cand--; m++; }
      sh.sll[lane][nm] = (uint16_t)(p - anchor);
      sh.sml[lane][nm] = (uint16_t)m;
      sh.sof[lane][nm] = (uint16_t)(p - cand);
      nm++;
      matched += m;
      p += m;
      anchor = p;
      misses = 0;
      if (p - 2 + 4 <= clen) ht[zs_hash4(d + p - 2)] = (uint16_t)(p - 2);
    } else {
      p += 1 + (misses++ >> L4_SKIP_TRIGGER);
    }
  }
  sh.lnm[lane] = nm;
  sh.llit[lane] = (s1 - s0) - matched;
}

// thread 0 after the parse: the literals that open each lane's first sequence, where each lane's literals go
Z_HD void zs_plan(ZsShared &sh) {
  uint32_t carry = 0, nseq = 0, lit = 0;
  for (uint32_t l = 0; l < ZS_LANES; l++) {
    const uint32_t s0 = l * ZS_SLICE;
    sh.lcarry[l] = carry;
    sh.litbase[l] = lit;
    if (s0 >= sh.clen) continue;
    lit += sh.llit[l];
    nseq += sh.lnm[l];
    if (!sh.lnm[l]) {
      carry += l4_min(sh.clen, s0 + ZS_SLICE) - s0;
    } else {
      uint32_t used = 0;   // the lane's tail: its slice after the last match
      for (uint32_t i = 0; i < sh.lnm[l]; i++) used += sh.sll[l][i] + sh.sml[l][i];
      carry = l4_min(sh.clen, s0 + ZS_SLICE) - s0 - used;
    }
  }
  sh.nseq = nseq;
  sh.nlit = lit;
}

// each lane: its literal bytes into lits (in order) and their histogram
Z_HD void zs_gather(ZsShared &sh, uint32_t lane) {
  const uint32_t s0 = lane * ZS_SLICE;
  if (s0 >= sh.clen) return;
  const uint32_t s1 = l4_min(sh.clen, s0 + ZS_SLICE);
  uint32_t o = sh.litbase[lane], p = s0;
  for (uint32_t i = 0; i <= sh.lnm[lane]; i++) {
    const uint32_t L = i < sh.lnm[lane] ? sh.sll[lane][i] : s1 - p;
    for (uint32_t k = 0; k < L; k++) {
      const uint8_t c = sh.data[p + k];
      sh.lits[o + k] = c;
#ifdef __CUDA_ARCH__
      atomicAdd(&sh.freq[c], 1u);
#else
      sh.freq[c]++;
#endif
    }
    o += L;
    p += L + (i < sh.lnm[lane] ? sh.sml[lane][i] : 0);
  }
}

// libzstd's FSE_buildCTable for a normalized distribution
Z_HD void zs_ctable(ZsCTable &ct, const int16_t *norm, uint32_t nsym, uint32_t log) {
  const uint32_t size = 1u << log, step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  uint8_t sym[64];
  uint32_t cumul[54], high = size - 1;
  cumul[0] = 0;
  for (uint32_t u = 1; u <= nsym; u++) {
    if (norm[u - 1] == -1) { cumul[u] = cumul[u - 1] + 1; sym[high--] = (uint8_t)(u - 1); }
    else cumul[u] = cumul[u - 1] + (uint32_t)norm[u - 1];
  }
  uint32_t pos = 0;
  for (uint32_t s = 0; s < nsym; s++)
    for (int32_t i = 0; i < norm[s]; i++) {
      sym[pos] = (uint8_t)s;
      do { pos = (pos + step) & mask; } while (pos > high);
    }
  for (uint32_t u = 0; u < size; u++) ct.state[cumul[sym[u]]++] = (uint16_t)(size + u);
  int32_t total = 0;
  for (uint32_t s = 0; s < nsym; s++) {
    const int32_t n = norm[s];
    if (n == -1 || n == 1) {
      ct.dnb[s] = (log << 16) - size;
      ct.dfs[s] = total - 1;
      total++;
    } else if (n > 1) {
      const uint32_t mbo = log - z_log2((uint32_t)n - 1), msp = (uint32_t)n << mbo;
      ct.dnb[s] = (mbo << 16) - msp;
      ct.dfs[s] = total - n;
      total += n;
    }
  }
  ct.log = log;
}

// LSB-first writer of a bitstream into out[0..cap); past cap it only counts
struct ZsBitW {
  uint8_t *o;
  uint32_t pos, cap, n;
  uint64_t acc;
  Z_HD void init(uint8_t *out, uint32_t capacity) { o = out; pos = 0; cap = capacity; n = 0; acc = 0; }
  Z_HD void put(uint32_t v, uint32_t nb) {
    acc |= (uint64_t)v << n;
    n += nb;
    while (n >= 8) {
      if (pos < cap) o[pos] = (uint8_t)acc;
      pos++;
      acc >>= 8;
      n -= 8;
    }
  }
  // the end mark and the last partial byte; returns the stream's bytes
  Z_HD uint32_t close() {
    put(1, 1);
    if (n) { if (pos < cap) o[pos] = (uint8_t)acc; pos++; }
    return pos;
  }
};

Z_HD void zs_enc_init(const ZsCTable &ct, uint32_t &st, uint32_t s) {
  const uint32_t nb = (ct.dnb[s] + (1u << 15)) >> 16;
  const uint32_t v = (nb << 16) - ct.dnb[s];
  st = ct.state[(int32_t)(v >> nb) + ct.dfs[s]];
}
Z_HD void zs_enc(ZsBitW &w, const ZsCTable &ct, uint32_t &st, uint32_t s) {
  const uint32_t nb = (st + ct.dnb[s]) >> 16;
  w.put(st & ((1u << nb) - 1), nb);
  st = ct.state[(int32_t)(st >> nb) + ct.dfs[s]];
}

Z_HD uint32_t zs_ll_code(uint32_t ll) {
  if (ll < 16) return ll;
  if (ll >= 64) return z_log2(ll) + 19;
  uint32_t c = 16;
  while (c < 24 && ZS_TAB(zs_ll_base)[c + 1] <= ll) c++;
  return c;
}
Z_HD uint32_t zs_ml_code(uint32_t ml) {
  const uint32_t mb = ml - 3;
  if (mb < 32) return mb;
  if (mb >= 128) return z_log2(mb) + 36;
  uint32_t c = 32;
  while (c < 42 && ZS_TAB(zs_ml_base)[c + 1] <= ml) c++;
  return c;
}

// sequence k of the block in order: literal run, match length, offset
Z_HD void zs_seq_at(const ZsShared &sh, uint32_t l, uint32_t i, uint32_t &ll, uint32_t &ml, uint32_t &off) {
  ll = sh.sll[l][i] + (i == 0 ? sh.lcarry[l] : 0);
  ml = sh.sml[l][i];
  off = sh.sof[l][i];
}

// thread 0: the Huffman code of the literals when they may take one (every literal below 128, enough of them)
Z_HD void zs_huf_plan(ZsShared &sh) {
  ZsEncWork &ew = sh.ew;
  int32_t maxlit = -1;
  for (int32_t c = 255; c >= 0; c--)
    if (sh.freq[c]) { maxlit = c; break; }
  sh.huf = sh.nlit >= ZS_HUF_MIN && maxlit < 128;
  for (uint32_t k = 0; k < 4; k++) sh.hbits[k] = 0;
  if (!sh.huf) return;
  const uint32_t n = maxlit + 1 < 2 ? 2 : (uint32_t)maxlit + 1;
  z_build_lengths(sh.freq, n, 11, ew.hlen, ew.scratch);
  uint32_t hmax = 0, log = 0, rank[13] = {};
  for (uint32_t s = 0; s < n; s++)
    if (ew.hlen[s]) { hmax = s; log = ew.hlen[s] > log ? ew.hlen[s] : log; }
  for (uint32_t s = 0; s < n; s++) {
    ew.hw[s] = ew.hlen[s] ? (uint8_t)(log + 1 - ew.hlen[s]) : 0;
    rank[ew.hw[s]]++;
  }
  // the decoder's table order: weights ascending, symbols ascending within a weight
  uint32_t start[13], cur = 0;
  for (uint32_t w = 1; w <= log; w++) { start[w] = cur; cur += rank[w] << (w - 1); }
  for (uint32_t s = 0; s < n; s++) {
    const uint32_t w = ew.hw[s];
    if (!w) continue;
    ew.hcode[s] = (uint16_t)(start[w] >> (w - 1));
    start[w] += 1u << (w - 1);
  }
  sh.hlog = log;
  sh.hmax = hmax;
}

// each lane: the bits of the Huffman streams (four segments of the literals)
Z_HD void zs_huf_count(ZsShared &sh, uint32_t lane, uint32_t nl) {
  if (!sh.huf) return;
  const uint32_t seg = (sh.nlit + 3) / 4;
  uint32_t b[4] = {0, 0, 0, 0};
  for (uint32_t i = lane; i < sh.nlit; i += nl) b[i / seg] += sh.ew.hlen[sh.lits[i]];
  for (uint32_t k = 0; k < 4; k++) {
#ifdef __CUDA_ARCH__
    atomicAdd(&sh.hbits[k], b[k]);
#else
    sh.hbits[k] += b[k];
#endif
  }
}

Z_HD uint32_t zs_fh_bytes(uint32_t clen) { return 4 + 1 + (clen < 256 ? 1 : 2); }

// thread 0: the literals section's layout and header; raw literals or Huffman (tree description, jump table) go to
// out = the block content in the slot; sets seq_at (where the sequences section starts) and soff
Z_HD void zs_lit_write(ZsShared &sh, uint8_t *out) {
  const uint32_t nlit = sh.nlit;
  const uint32_t raw_hs = nlit < 32 ? 1 : nlit < 4096 ? 2 : 3;
  if (sh.huf) {
    const uint32_t hmax = sh.hmax, tree = 1 + (hmax + 1) / 2;
    uint32_t streams = 0, sz[4];
    for (uint32_t k = 0; k < 4; k++) { sz[k] = (sh.hbits[k] + 1 + 7) / 8; streams += sz[k]; }
    const uint32_t comp = tree + 6 + streams, big = comp > nlit ? comp : nlit;
    const uint32_t hs = big < 1024 ? 3 : big < 16384 ? 4 : 5;
    if (hs + comp < raw_hs + nlit) {
      const uint32_t sf = hs - 2, bits = hs == 3 ? 10 : hs == 4 ? 14 : 18;
      const uint64_t h = 2u | (sf << 2) | ((uint64_t)nlit << 4) | ((uint64_t)comp << (4 + bits));
      for (uint32_t i = 0; i < hs; i++) out[i] = (uint8_t)(h >> (8 * i));
      uint32_t q = hs;
      out[q++] = (uint8_t)(127 + hmax);
      for (uint32_t i = 0; i < hmax; i += 2)
        out[q++] = (uint8_t)((sh.ew.hw[i] << 4) | (i + 1 < hmax ? sh.ew.hw[i + 1] : 0));
      for (uint32_t k = 0; k < 3; k++) { out[q++] = (uint8_t)sz[k]; out[q++] = (uint8_t)(sz[k] >> 8); }
      for (uint32_t k = 0; k < 4; k++) { sh.soff[k] = q; q += sz[k]; }
      sh.seq_at = q;
      return;
    }
    sh.huf = 0;
  }
  if (raw_hs == 1) out[0] = (uint8_t)(nlit << 3);
  else if (raw_hs == 2) { out[0] = (uint8_t)(4 | (nlit << 4)); out[1] = (uint8_t)(nlit >> 4); }
  else { out[0] = (uint8_t)(12 | (nlit << 4)); out[1] = (uint8_t)(nlit >> 4); out[2] = (uint8_t)(nlit >> 12); }
  sh.soff[0] = raw_hs;
  sh.seq_at = raw_hs + nlit;
}

// lanes: Huffman stream k on lane k (encoded last literal first), or the raw literals on every lane
Z_HD void zs_lit_streams(const ZsShared &sh, uint8_t *out, uint32_t lane, uint32_t nl) {
  const uint32_t nlit = sh.nlit;
  if (!sh.huf) {
    for (uint32_t k = lane; k < nlit; k += nl) out[sh.soff[0] + k] = sh.lits[k];
    return;
  }
  const uint32_t seg = (nlit + 3) / 4;
  for (uint32_t k = lane; k < 4; k += nl) {
    const uint32_t a = k * seg, e = k == 3 ? nlit : a + seg;
    ZsBitW w;
    w.init(out + sh.soff[k], ZS_SLOT);
    for (uint32_t i = e; i > a; i--) {
      const uint32_t c = sh.lits[i - 1];
      w.put(sh.ew.hcode[c], sh.ew.hlen[c]);
    }
    w.close();
  }
}

// thread 0: the sequences section (predefined tables) at out[seq_at..cap), the block and frame headers in front of the
// content at slot[fh + 3..); the frame's total length in sh.bytes, or 0 when a raw block is shorter
Z_HD void zs_seq_write(ZsShared &sh, uint8_t *slot) {
  const uint32_t clen = sh.clen, fh = zs_fh_bytes(clen), c0 = fh + 3, cap = ZS_SLOT - c0;
  uint8_t *out = slot + c0;
  const uint32_t nseq = sh.nseq;
  uint32_t q = sh.seq_at;
  uint32_t size = 0;
  if (q + 4 <= cap) {
    if (nseq < 128) out[q++] = (uint8_t)nseq;
    else if (nseq < 0x7F00) { out[q++] = (uint8_t)((nseq >> 8) + 0x80); out[q++] = (uint8_t)nseq; }
    else { out[q++] = 0xFF; out[q++] = (uint8_t)(nseq - 0x7F00); out[q++] = (uint8_t)((nseq - 0x7F00) >> 8); }
    if (nseq) {
      out[q++] = 0;   // predefined LL, OF, ML
      ZsEncWork &ew = sh.ew;
      for (uint32_t t = 0; t < 3; t++) {
        uint32_t ns, log;
        const int16_t *norm = zs_def_norm(t, &ns, &log);
        zs_ctable(ew.ct[t], norm, ns, log);
      }
      const ZsCTable &cl = ew.ct[ZS_LL], &co = ew.ct[ZS_OF], &cm = ew.ct[ZS_ML];
      ZsBitW w;
      w.init(out + q, cap - q);
      // sequences last to first: lanes from the last, each lane's sequences from its last
      uint32_t sl = 0, so = 0, sm = 0;
      bool first = true;
      for (int32_t l = ZS_LANES - 1; l >= 0; l--)
        for (int32_t i = (int32_t)sh.lnm[l] - 1; i >= 0; i--) {
          uint32_t ll, ml, off;
          zs_seq_at(sh, (uint32_t)l, (uint32_t)i, ll, ml, off);
          const uint32_t lc = zs_ll_code(ll), mc = zs_ml_code(ml), ov = off + 3, oc = z_log2(ov);
          if (first) {
            zs_enc_init(cm, sm, mc);
            zs_enc_init(co, so, oc);
            zs_enc_init(cl, sl, lc);
            first = false;
          } else {
            zs_enc(w, co, so, oc);
            zs_enc(w, cm, sm, mc);
            zs_enc(w, cl, sl, lc);
          }
          w.put(ll - ZS_TAB(zs_ll_base)[lc], ZS_TAB(zs_ll_bits)[lc]);
          w.put(ml - ZS_TAB(zs_ml_base)[mc], ZS_TAB(zs_ml_bits)[mc]);
          w.put(ov - (1u << oc), oc);
        }
      w.put(sm & ((1u << cm.log) - 1), cm.log);
      w.put(so & ((1u << co.log) - 1), co.log);
      w.put(sl & ((1u << cl.log) - 1), cl.log);
      q += w.close();
    }
    size = q;
  }
  const bool comp = size && size <= cap && size < clen;
  const uint32_t bs = comp ? size : clen;
  // frame header: magic, Single_Segment with Frame_Content_Size (1 byte below 256, else 2 bytes - 256)
  slot[0] = 0x28; slot[1] = 0xB5; slot[2] = 0x2F; slot[3] = 0xFD;
  if (clen < 256) { slot[4] = 0x20; slot[5] = (uint8_t)clen; }
  else { slot[4] = 0x60; slot[5] = (uint8_t)(clen - 256); slot[6] = (uint8_t)((clen - 256) >> 8); }
  const uint32_t bh = 1u | ((comp ? 2u : 0u) << 1) | (bs << 3);
  slot[fh] = (uint8_t)bh; slot[fh + 1] = (uint8_t)(bh >> 8); slot[fh + 2] = (uint8_t)(bh >> 16);
  sh.huf = comp;   // reused: 1 = compressed block, 0 = the raw piece is to be copied
  sh.bytes = c0 + bs;
}

// Host run of the device frame compressor (lanes one after the other): slot receives sh.bytes bytes.
static inline void zs_compress_block_host(ZsShared &sh, const uint8_t *block, uint32_t clen, uint8_t *slot) {
  memcpy(sh.data, block, clen);
  sh.clen = clen;
  for (uint32_t c = 0; c < 256; c++) sh.freq[c] = 0;
  for (uint32_t l = 0; l < ZS_LANES; l++) zs_lane(sh, l);
  zs_plan(sh);
  for (uint32_t l = 0; l < ZS_LANES; l++) zs_gather(sh, l);
  zs_huf_plan(sh);
  zs_huf_count(sh, 0, 1);
  uint8_t *out = slot + zs_fh_bytes(clen) + 3;
  zs_lit_write(sh, out);
  zs_lit_streams(sh, out, 0, 1);
  zs_seq_write(sh, slot);
  if (!sh.huf) memcpy(slot + zs_fh_bytes(clen) + 3, block, clen);
}

// one CTA per piece; segs / chunk numbering: ZSeg, z_chunk_part (common.cuh), with ZS_BLOCK-byte chunks
__global__ void __launch_bounds__(ZS_LANES)
    k_zscompress(const uint8_t *__restrict__ img, const ZSeg *__restrict__ segs, uint32_t P, uint8_t *__restrict__ slots,
                 uint32_t *__restrict__ csize) {
  extern __shared__ __align__(16) uint8_t zs_smem[];
  ZsShared &sh = *reinterpret_cast<ZsShared *>(zs_smem);
  const uint32_t c = blockIdx.x, tid = threadIdx.x;
  const ZSeg sg = segs[z_chunk_part(segs, P, c)];
  const uint64_t a = (uint64_t)(c - sg.chunk0) * ZS_BLOCK;
  const uint32_t clen = (uint32_t)z_min64(ZS_BLOCK, sg.body_len - a);
  const uint8_t *src = img + sg.body_off + a;
  for (uint32_t i = tid; i < clen; i += ZS_LANES) sh.data[i] = src[i];
  for (uint32_t i = tid; i < 256; i += ZS_LANES) sh.freq[i] = 0;
  if (tid == 0) sh.clen = clen;
  __syncthreads();
  zs_lane(sh, tid);
  __syncthreads();
  if (tid == 0) zs_plan(sh);
  __syncthreads();
  zs_gather(sh, tid);
  __syncthreads();
  if (tid == 0) zs_huf_plan(sh);
  __syncthreads();
  zs_huf_count(sh, tid, ZS_LANES);
  __syncthreads();
  uint8_t *slot = slots + (uint64_t)c * ZS_SLOT;
  uint8_t *out = slot + zs_fh_bytes(clen) + 3;
  if (tid == 0) zs_lit_write(sh, out);
  __syncthreads();
  zs_lit_streams(sh, out, tid, ZS_LANES);
  __syncthreads();
  if (tid == 0) zs_seq_write(sh, slot);
  __syncthreads();
  if (!sh.huf)
    for (uint32_t i = tid; i < clen; i += ZS_LANES) out[i] = src[i];
  if (tid == 0) csize[c] = sh.bytes;
}

}  // namespace tezgpu

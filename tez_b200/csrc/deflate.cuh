// deflate.cuh -- DefaultCodec writer: IFile segments as zlib streams (RFC 1950 / 1951), compressed on the device.
//
// A compressed segment (SORT/IFile.java:351-420) is 'T' 'I' 'F' 0x01, one zlib stream of the uncompressed body (records,
// RLE markers, the ff ff EOF marker) and a big-endian CRC-32 over the compressed bytes.  The stream written here:
//   - zlib header 78 01;
//   - the body cut into ZCHUNK-byte chunks, no back-reference crossing a chunk start, every chunk but the last ending
//     byte-aligned (an empty stored block, as zlib's Z_SYNC_FLUSH writes), so chunks compress independently and
//     concatenate at byte granularity;
//   - each chunk the smallest of a stored, a fixed-Huffman and a dynamic-Huffman block of one LZ77 parse;
//   - the Adler-32 of the body, combined from per-chunk values.
// The output is a deterministic function of the body: the chunk compressor below is __host__ __device__ and
// tezgpu_debug_deflate_emulate runs it on the host, lane by lane, to produce the same bytes the device writes.
//
// One chunk = one CTA of ZLANES threads.  Lane l parses slice [l * ZSLICE, (l + 1) * ZSLICE) of the chunk greedily with
// a single-candidate hash table private to the lane (seeded with the ZSLICE bytes before the slice), so the parse does
// not depend on thread timing.  Pass 1 counts symbols per lane; thread 0 builds the codes and picks the block type;
// pass 2 re-parses and every lane writes its bits at its scanned bit offset (atomicOr into a zeroed slot).
#pragma once
#include "crc32.cuh"

namespace tezgpu {

#define Z_HD __host__ __device__ __forceinline__

constexpr uint32_t ZCHUNK = 32768;                 // body bytes per chunk (= the deflate window)
constexpr uint32_t ZLANES = 16;                    // threads per chunk
constexpr uint32_t ZSLICE = ZCHUNK / ZLANES;       // bytes parsed by one lane
constexpr uint32_t ZHBITS = 10;                    // lane hash table: 2^ZHBITS u16 positions
constexpr uint32_t ZHSIZE = 1u << ZHBITS;
constexpr uint32_t ZSLOT = ZCHUNK + 16;            // device bytes reserved per compressed chunk (stored block worst case)
constexpr uint32_t ZNLIT = 286, ZNDIST = 30, ZNSYM = ZNLIT + ZNDIST;
constexpr uint32_t ZDOFF = 288;                    // code / len arrays: literal/length 0..287 (fixed code), distance at 288
constexpr uint16_t ZEMPTY = 0xFFFF;
constexpr uint32_t ADLER_BASE = 65521;

// ------------------------------------------------------------------------------------------------ symbol arithmetic
Z_HD uint32_t z_log2(uint32_t x) {
#ifdef __CUDA_ARCH__
  return 31 - __clz(x);
#else
  return 31 - __builtin_clz(x);
#endif
}
Z_HD uint64_t z_min64(uint64_t a, uint64_t b) { return a < b ? a : b; }

// length 3..258 -> symbol 257..285, extra bits, extra value
Z_HD void z_len_sym(uint32_t l, uint32_t &sym, uint32_t &ebits, uint32_t &eval) {
  if (l == 258) { sym = 285; ebits = 0; eval = 0; return; }
  const uint32_t x = l - 3;
  if (x < 8) { sym = 257 + x; ebits = 0; eval = 0; return; }
  const uint32_t e = z_log2(x) - 2;
  sym = 257 + 4 * e + (x >> e);
  ebits = e;
  eval = x & ((1u << e) - 1);
}
// symbol 257..285 -> base length, extra bits
Z_HD void z_len_base(uint32_t sym, uint32_t &base, uint32_t &ebits) {
  if (sym == 285) { base = 258; ebits = 0; return; }
  if (sym < 265) { base = sym - 254; ebits = 0; return; }
  ebits = (sym - 261) >> 2;
  base = 3 + ((4 + ((sym - 265) & 3)) << ebits);
}
// distance 1..32768 -> symbol 0..29, extra bits, extra value
Z_HD void z_dist_sym(uint32_t d, uint32_t &sym, uint32_t &ebits, uint32_t &eval) {
  const uint32_t x = d - 1;
  if (x < 4) { sym = x; ebits = 0; eval = 0; return; }
  const uint32_t e = z_log2(x) - 1;
  sym = 2 * e + 2 + ((x >> e) & 1);
  ebits = e;
  eval = x & ((1u << e) - 1);
}
Z_HD void z_dist_base(uint32_t sym, uint32_t &base, uint32_t &ebits) {
  if (sym < 4) { base = sym + 1; ebits = 0; return; }
  ebits = (sym >> 1) - 1;
  base = 1 + ((2 | (sym & 1)) << ebits);
}
// symbol index (literal/length 0..285, distance 286..315) -> index into the code / len arrays
Z_HD uint32_t z_code_index(uint32_t s) { return s < ZNLIT ? s : s - ZNLIT + ZDOFF; }
Z_HD uint32_t z_fixed_lit_len(uint32_t s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }
// the order code-length code lengths are sent in (RFC 1951 3.2.7)
Z_HD uint32_t z_cl_order(uint32_t i) {
  switch (i) {
    case 0: return 16; case 1: return 17; case 2: return 18; case 3: return 0; case 4: return 8; case 5: return 7;
    case 6: return 9; case 7: return 6; case 8: return 10; case 9: return 5; case 10: return 11; case 11: return 4;
    case 12: return 12; case 13: return 3; case 14: return 13; case 15: return 2; case 16: return 14; case 17: return 1;
    default: return 15;
  }
}

// ------------------------------------------------------------------------------------------------ Adler-32
Z_HD uint32_t z_adler_update(uint32_t adler, const uint8_t *p, uint64_t n) {
  uint32_t a = adler & 0xFFFF, b = adler >> 16;
  while (n) {
    const uint32_t k = n < 5552 ? (uint32_t)n : 5552u;   // largest run without u32 overflow
    for (uint32_t i = 0; i < k; i++) { a += p[i]; b += a; }
    a %= ADLER_BASE;
    b %= ADLER_BASE;
    p += k;
    n -= k;
  }
  return a | (b << 16);
}
// adler(A || B) from adler(A), adler(B) and |B|
Z_HD uint32_t z_adler_combine(uint32_t a1, uint32_t a2, uint64_t len2) {
  const uint32_t rem = (uint32_t)(len2 % ADLER_BASE);
  uint32_t s1 = a1 & 0xFFFF;
  uint32_t s2 = (uint32_t)(((uint64_t)rem * s1) % ADLER_BASE);
  s1 += (a2 & 0xFFFF) + ADLER_BASE - 1;
  s2 += (a1 >> 16) + (a2 >> 16) + ADLER_BASE - rem;
  if (s1 >= ADLER_BASE) s1 -= ADLER_BASE;
  if (s1 >= ADLER_BASE) s1 -= ADLER_BASE;
  if (s2 >= 2 * ADLER_BASE) s2 -= 2 * ADLER_BASE;
  if (s2 >= ADLER_BASE) s2 -= ADLER_BASE;
  return s1 | (s2 << 16);
}

// ------------------------------------------------------------------------------------------------ Huffman codes
struct ZBuildScratch {
  uint16_t sym[288];
  uint32_t w[288];
  uint32_t iw[288];
  uint16_t par_leaf[288];
  uint16_t par_int[288];
  uint16_t depth[288];
  uint32_t cnt[16];
};

// Code lengths for freq[0..n), limited to maxbits, always a complete code over at least two symbols (unused symbols
// 0, 1, ... are added with weight 0 when fewer than two are used).  Deterministic: leaves are ordered by (weight,
// symbol), the two-queue Huffman construction prefers leaves on ties, an over-long code is repaired on the length
// counts (move the deepest codes up, split the deepest shorter code), and lengths go to symbols in weight order.
Z_HD void z_build_lengths(const uint32_t *freq, uint32_t n, uint32_t maxbits, uint8_t *len, ZBuildScratch &s) {
  uint32_t m = 0;
  for (uint32_t i = 0; i < n; i++) {
    len[i] = 0;
    if (freq[i]) { s.sym[m] = (uint16_t)i; s.w[m] = freq[i]; m++; }
  }
  for (uint32_t i = 0; m < 2 && i < n; i++)
    if (!freq[i]) { s.sym[m] = (uint16_t)i; s.w[m] = 0; m++; }
  // insertion sort by (weight, symbol)
  for (uint32_t i = 1; i < m; i++) {
    const uint16_t ks = s.sym[i];
    const uint32_t kw = s.w[i];
    uint32_t j = i;
    while (j > 0 && (s.w[j - 1] > kw || (s.w[j - 1] == kw && s.sym[j - 1] > ks))) { s.sym[j] = s.sym[j - 1]; s.w[j] = s.w[j - 1]; j--; }
    s.sym[j] = ks;
    s.w[j] = kw;
  }
  // two queues: leaves (sorted) and internal nodes (created in non-decreasing weight order)
  uint32_t li = 0, ii = 0;
  for (uint32_t k = 0; k + 1 < m; k++) {
    uint32_t sum = 0;
    for (int t = 0; t < 2; t++) {
      if (li < m && (ii >= k || s.w[li] <= s.iw[ii])) { s.par_leaf[li] = (uint16_t)k; sum += s.w[li]; li++; }
      else { s.par_int[ii] = (uint16_t)k; sum += s.iw[ii]; ii++; }
    }
    s.iw[k] = sum;
  }
  s.depth[m - 2] = 0;
  for (int k = (int)m - 3; k >= 0; k--) s.depth[k] = s.depth[s.par_int[k]] + 1;
  for (uint32_t l = 0; l < 16; l++) s.cnt[l] = 0;
  for (uint32_t i = 0; i < m; i++) {
    uint32_t d = s.depth[s.par_leaf[i]] + 1u;
    s.cnt[d > maxbits ? maxbits : d]++;
  }
  uint32_t total = 0;
  for (uint32_t l = 1; l <= maxbits; l++) total += s.cnt[l] << (maxbits - l);
  while (total > (1u << maxbits)) {
    s.cnt[maxbits]--;
    for (uint32_t l = maxbits - 1; l > 0; l--)
      if (s.cnt[l]) { s.cnt[l]--; s.cnt[l + 1] += 2; break; }
    total--;
  }
  uint32_t idx = 0;
  for (uint32_t l = maxbits; l >= 1; l--)
    for (uint32_t c = 0; c < s.cnt[l]; c++) len[s.sym[idx++]] = (uint8_t)l;
}

// canonical codes, bit-reversed for LSB-first output
Z_HD void z_build_codes(const uint8_t *len, uint32_t n, uint16_t *code) {
  uint32_t cnt[16], next[16];
  for (int l = 0; l < 16; l++) cnt[l] = 0;
  for (uint32_t i = 0; i < n; i++) cnt[len[i]]++;
  cnt[0] = 0;
  uint32_t c = 0;
  for (int l = 1; l < 16; l++) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t l = len[i];
    if (!l) { code[i] = 0; continue; }
    uint32_t v = next[l]++, r = 0;
    for (uint32_t b = 0; b < l; b++) { r = (r << 1) | (v & 1); v >>= 1; }
    code[i] = (uint16_t)r;
  }
}

// ------------------------------------------------------------------------------------------------ chunk state
enum : uint32_t { ZB_STORED = 0, ZB_FIXED = 1, ZB_DYN = 2 };

struct ZShared {
  uint8_t data[ZCHUNK];
  uint16_t htab[ZLANES][ZHSIZE];
  uint16_t lhist[ZLANES][ZNSYM];   // symbol counts per lane (literal/length 0..285, distance 286..315)
  uint32_t lextra[ZLANES];         // extra bits per lane
  uint32_t ladler[ZLANES];         // Adler-32 of the lane's slice
  uint32_t lbit0[ZLANES];          // bit offset of the lane's first symbol in the chunk
  uint32_t freq[ZNSYM];
  uint32_t clfreq[19];
  uint16_t code[ZDOFF + ZNDIST];
  uint8_t len[ZDOFF + ZNDIST];
  uint8_t cllen[19];
  uint16_t clcode[19];
  uint16_t tok[ZNSYM];             // run-length coded code lengths: symbol | extra value << 5
  uint32_t ntok, hlit, hdist, hclen;
  uint32_t btype, hdr_bits, eob_bit, bytes, adler, last, clen;
  ZBuildScratch scratch;
};

// LSB-first bit writer into zeroed u32 words; flushes OR whole words (atomicOr on the device: neighbouring lanes share
// the words at their boundaries)
struct ZBitW {
  uint32_t *w;
  uint64_t acc;
  uint32_t n, wi;
  Z_HD void init(uint32_t *words, uint32_t bitpos) { w = words; wi = bitpos >> 5; n = bitpos & 31; acc = 0; }
  Z_HD void flush_word(uint32_t v) {
#ifdef __CUDA_ARCH__
    if (v) atomicOr(&w[wi], v);
#else
    w[wi] |= v;
#endif
    wi++;
  }
  Z_HD void put(uint32_t v, uint32_t nb) {
    acc |= (uint64_t)v << n;
    n += nb;
    while (n >= 32) { flush_word((uint32_t)acc); acc >>= 32; n -= 32; }
  }
  Z_HD void align_byte() { n = (n + 7) & ~7u; if (n == 32) { flush_word((uint32_t)acc); acc = 0; n = 0; } }
  Z_HD void done() { if (n) flush_word((uint32_t)acc); }
};

Z_HD uint32_t z_hash3(const uint8_t *d) {
  const uint32_t v = (uint32_t)d[0] | ((uint32_t)d[1] << 8) | ((uint32_t)d[2] << 16);
  return (v * 2654435761u) >> (32 - ZHBITS);
}

// Greedy parse of the lane's slice.  PASS 1: symbol counts, extra bits and the slice's Adler-32; PASS 2: the bits.
template <int PASS>
Z_HD void z_lane(ZShared &sh, uint32_t lane, uint32_t *slot) {
  const uint32_t clen = sh.clen;
  const uint32_t s0 = lane * ZSLICE;
  if (PASS == 1) {
    for (uint32_t i = 0; i < ZNSYM; i++) sh.lhist[lane][i] = 0;
    sh.lextra[lane] = 0;
    sh.ladler[lane] = 1;
  }
  if (s0 >= clen) return;
  const uint32_t s1 = clen < s0 + ZSLICE ? clen : s0 + ZSLICE;
  const uint8_t *d = sh.data;
  uint16_t *ht = sh.htab[lane];
  for (uint32_t i = 0; i < ZHSIZE; i++) ht[i] = ZEMPTY;
  for (uint32_t q = s0 >= ZSLICE ? s0 - ZSLICE : 0; q < s0 && q + 3 <= clen; q++) ht[z_hash3(d + q)] = (uint16_t)q;
  uint16_t *hist = sh.lhist[lane];
  uint32_t extra = 0;
  ZBitW bw;
  if (PASS == 2) bw.init(slot, sh.lbit0[lane]);
  uint32_t p = s0;
  while (p < s1) {
    uint32_t mlen = 0, dist = 0;
    if (p + 3 <= s1) {
      const uint32_t h = z_hash3(d + p);
      const uint32_t cand = ht[h];
      ht[h] = (uint16_t)p;
      if (cand != ZEMPTY && d[cand] == d[p] && d[cand + 1] == d[p + 1] && d[cand + 2] == d[p + 2]) {
        const uint32_t maxl = (s1 - p) < 258u ? (s1 - p) : 258u;
        mlen = 3;
        while (mlen < maxl && d[cand + mlen] == d[p + mlen]) mlen++;
        dist = p - cand;
      }
    }
    if (mlen) {
      uint32_t ls, le, lv, ds, de, dv;
      z_len_sym(mlen, ls, le, lv);
      z_dist_sym(dist, ds, de, dv);
      if (PASS == 1) {
        hist[ls]++;
        hist[ZNLIT + ds]++;
        extra += le + de;
      } else {
        bw.put(sh.code[ls], sh.len[ls]);
        if (le) bw.put(lv, le);
        bw.put(sh.code[ZDOFF + ds], sh.len[ZDOFF + ds]);
        if (de) bw.put(dv, de);
      }
      for (uint32_t q = p + 1; q < p + mlen; q++)
        if (q + 3 <= clen) ht[z_hash3(d + q)] = (uint16_t)q;
      p += mlen;
    } else {
      if (PASS == 1) hist[d[p]]++;
      else bw.put(sh.code[d[p]], sh.len[d[p]]);
      p++;
    }
  }
  if (PASS == 1) {
    sh.lextra[lane] = extra;
    sh.ladler[lane] = z_adler_update(1, d + s0, s1 - s0);
  } else {
    bw.done();
  }
}

// Thread 0, after pass 1 and the frequency sum: codes, block type, bit offsets, byte size, Adler-32 of the chunk.
Z_HD void z_plan(ZShared &sh) {
  const uint32_t clen = sh.clen, last = sh.last;
  sh.freq[256] = 1;
  uint64_t extra = 0;
  for (uint32_t l = 0; l < ZLANES; l++) extra += sh.lextra[l];
  // fixed-Huffman size
  uint64_t fixed_bits = 3 + extra;
  for (uint32_t s = 0; s < ZNLIT; s++) fixed_bits += (uint64_t)sh.freq[s] * z_fixed_lit_len(s);
  for (uint32_t s = 0; s < ZNDIST; s++) fixed_bits += (uint64_t)sh.freq[ZNLIT + s] * 5;
  // dynamic code
  z_build_lengths(sh.freq, ZNLIT, 15, sh.len, sh.scratch);
  z_build_lengths(sh.freq + ZNLIT, ZNDIST, 15, sh.len + ZDOFF, sh.scratch);
  sh.len[286] = sh.len[287] = 0;
  uint32_t hlit = ZNLIT, hdist = ZNDIST;
  while (hlit > 257 && sh.len[hlit - 1] == 0) hlit--;
  while (hdist > 1 && sh.len[ZDOFF + hdist - 1] == 0) hdist--;
  // run-length code of the hlit + hdist code lengths
  uint32_t ntok = 0;
  for (uint32_t i = 0; i < 19; i++) sh.clfreq[i] = 0;
  const uint32_t total = hlit + hdist;
  auto lenat = [&](uint32_t i) -> uint32_t { return i < hlit ? sh.len[i] : sh.len[ZDOFF + i - hlit]; };
  uint32_t i = 0;
  while (i < total) {
    const uint32_t l = lenat(i);
    uint32_t run = 1;
    while (i + run < total && lenat(i + run) == l) run++;
    if (l == 0) {
      while (run >= 11) { const uint32_t r = run < 138 ? run : 138; sh.tok[ntok++] = (uint16_t)(18 | ((r - 11) << 5)); sh.clfreq[18]++; run -= r; i += r; }
      if (run >= 3) { sh.tok[ntok++] = (uint16_t)(17 | ((run - 3) << 5)); sh.clfreq[17]++; i += run; run = 0; }
      while (run) { sh.tok[ntok++] = 0; sh.clfreq[0]++; run--; i++; }
    } else {
      sh.tok[ntok++] = (uint16_t)l; sh.clfreq[l]++; run--; i++;
      while (run >= 3) { const uint32_t r = run < 6 ? run : 6; sh.tok[ntok++] = (uint16_t)(16 | ((r - 3) << 5)); sh.clfreq[16]++; run -= r; i += r; }
      while (run) { sh.tok[ntok++] = (uint16_t)l; sh.clfreq[l]++; run--; i++; }
    }
  }
  z_build_lengths(sh.clfreq, 19, 7, sh.cllen, sh.scratch);
  uint32_t hclen = 19;
  while (hclen > 4 && sh.cllen[z_cl_order(hclen - 1)] == 0) hclen--;
  uint64_t hdr = 3 + 5 + 5 + 4 + 3ull * hclen;
  for (uint32_t t = 0; t < ntok; t++) {
    const uint32_t s = sh.tok[t] & 31;
    hdr += sh.cllen[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
  }
  uint64_t dyn_bits = hdr + extra;
  for (uint32_t s = 0; s < ZNSYM; s++) dyn_bits += (uint64_t)sh.freq[s] * sh.len[z_code_index(s)];
  auto block_bytes = [&](uint64_t bits) -> uint64_t { return last ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4; };
  const uint64_t stored = 5 + (uint64_t)clen, fixed = block_bytes(fixed_bits), dyn = block_bytes(dyn_bits);
  uint32_t bt = ZB_STORED;
  uint64_t best = stored;
  if (fixed < best) { bt = ZB_FIXED; best = fixed; }
  if (dyn < best) { bt = ZB_DYN; best = dyn; }
  sh.btype = bt;
  sh.bytes = (uint32_t)best;
  sh.ntok = ntok; sh.hlit = hlit; sh.hdist = hdist; sh.hclen = hclen;
  if (bt == ZB_FIXED) {
    for (uint32_t s = 0; s < ZDOFF; s++) sh.len[s] = (uint8_t)z_fixed_lit_len(s);
    for (uint32_t s = 0; s < ZNDIST; s++) sh.len[ZDOFF + s] = 5;
    sh.hdr_bits = 3;
  } else {
    sh.hdr_bits = (uint32_t)hdr;
  }
  if (bt != ZB_STORED) {
    z_build_codes(sh.len, ZDOFF, sh.code);
    z_build_codes(sh.len + ZDOFF, ZNDIST, sh.code + ZDOFF);
    z_build_codes(sh.cllen, 19, sh.clcode);
    uint32_t bit = sh.hdr_bits;
    for (uint32_t l = 0; l < ZLANES; l++) {
      sh.lbit0[l] = bit;
      uint32_t b = sh.lextra[l];
      for (uint32_t s = 0; s < ZNSYM; s++) b += (uint32_t)sh.lhist[l][s] * sh.len[z_code_index(s)];
      bit += b;
    }
    sh.eob_bit = bit;
  }
  uint32_t adler = 1;
  for (uint32_t l = 0; l < ZLANES; l++) {
    const uint32_t a = l * ZSLICE;
    if (a >= clen) break;
    const uint32_t b = clen < a + ZSLICE ? clen : a + ZSLICE;
    adler = z_adler_combine(adler, sh.ladler[l], b - a);
  }
  sh.adler = adler;
}

// Thread 0: block header (before the lanes' bits) and EOB + sync-flush trailer (after them)
Z_HD void z_write_header(const ZShared &sh, uint32_t *slot) {
  ZBitW bw;
  bw.init(slot, 0);
  bw.put(sh.last, 1);
  if (sh.btype == ZB_FIXED) {
    bw.put(1, 2);
  } else {
    bw.put(2, 2);
    bw.put(sh.hlit - 257, 5);
    bw.put(sh.hdist - 1, 5);
    bw.put(sh.hclen - 4, 4);
    for (uint32_t i = 0; i < sh.hclen; i++) bw.put(sh.cllen[z_cl_order(i)], 3);
    for (uint32_t t = 0; t < sh.ntok; t++) {
      const uint32_t s = sh.tok[t] & 31, v = sh.tok[t] >> 5;
      bw.put(sh.clcode[s], sh.cllen[s]);
      if (s == 16) bw.put(v, 2);
      else if (s == 17) bw.put(v, 3);
      else if (s == 18) bw.put(v, 7);
    }
  }
  bw.done();
  bw.init(slot, sh.eob_bit);
  bw.put(sh.code[256], sh.len[256]);
  if (!sh.last) {
    bw.put(0, 3);          // empty stored block: BFINAL 0, BTYPE 00, then LEN 0000 NLEN ffff on a byte boundary
    bw.align_byte();
    bw.put(0, 16);
    bw.put(0xFFFF, 16);
  }
  bw.done();
}

Z_HD void z_write_stored(const ZShared &sh, uint8_t *out, uint32_t i0, uint32_t step) {
  if (i0 == 0) {
    out[0] = (uint8_t)sh.last;
    out[1] = (uint8_t)sh.clen; out[2] = (uint8_t)(sh.clen >> 8);
    out[3] = (uint8_t)~sh.clen; out[4] = (uint8_t)(~sh.clen >> 8);
  }
  for (uint32_t i = i0; i < sh.clen; i += step) out[5 + i] = sh.data[i];
}

// Host run of the device chunk compressor (lanes one after the other): out receives sh.bytes bytes (cap >= ZSLOT).
static inline void z_deflate_chunk_host(ZShared &sh, const uint8_t *chunk, uint32_t clen, bool last, uint8_t *out) {
  memcpy(sh.data, chunk, clen);
  sh.clen = clen;
  sh.last = last ? 1 : 0;
  for (uint32_t l = 0; l < ZLANES; l++) z_lane<1>(sh, l, nullptr);
  for (uint32_t s = 0; s < ZNSYM; s++) {
    uint32_t f = 0;
    for (uint32_t l = 0; l < ZLANES; l++) f += sh.lhist[l][s];
    sh.freq[s] = f;
  }
  z_plan(sh);
  memset(out, 0, ZSLOT);
  if (sh.btype == ZB_STORED) {
    z_write_stored(sh, out, 0, 1);
    return;
  }
  uint32_t *w = reinterpret_cast<uint32_t *>(out);
  z_write_header(sh, w);
  for (uint32_t l = 0; l < ZLANES; l++) z_lane<2>(sh, l, w);
}

// ------------------------------------------------------------------------------------------------ device writer
// one CTA per chunk; segs / chunk numbering: ZSeg, z_chunk_part (common.cuh)
__global__ void __launch_bounds__(ZLANES)
    k_zdeflate(const uint8_t *__restrict__ img, const ZSeg *__restrict__ segs, uint32_t P, uint8_t *__restrict__ slots,
               uint32_t *__restrict__ csize, uint32_t *__restrict__ cadler) {
  extern __shared__ __align__(16) uint8_t z_smem[];
  ZShared &sh = *reinterpret_cast<ZShared *>(z_smem);
  const uint32_t c = blockIdx.x, tid = threadIdx.x;
  const uint32_t p = z_chunk_part(segs, P, c);
  const ZSeg sg = segs[p];
  const uint32_t k = c - sg.chunk0;
  const uint64_t a = (uint64_t)k * ZCHUNK;
  const uint32_t clen = (uint32_t)z_min64(ZCHUNK, sg.body_len - a);
  const uint8_t *src = img + sg.body_off + a;
  for (uint32_t i = tid; i < clen; i += ZLANES) sh.data[i] = src[i];
  if (tid == 0) { sh.clen = clen; sh.last = (k + 1 == sg.nchunks && !sg.open) ? 1 : 0; }
  __syncthreads();
  z_lane<1>(sh, tid, nullptr);
  __syncthreads();
  for (uint32_t s = tid; s < ZNSYM; s += ZLANES) {
    uint32_t f = 0;
    for (uint32_t l = 0; l < ZLANES; l++) f += sh.lhist[l][s];
    sh.freq[s] = f;
  }
  __syncthreads();
  if (tid == 0) z_plan(sh);
  __syncthreads();
  uint8_t *out = slots + (uint64_t)c * ZSLOT;
  uint32_t *w = reinterpret_cast<uint32_t *>(out);
  if (sh.btype == ZB_STORED) {
    z_write_stored(sh, out, tid, ZLANES);
  } else {
    for (uint32_t i = tid; i < (sh.bytes + 3) / 4; i += ZLANES) w[i] = 0;
    __syncthreads();
    if (tid == 0) z_write_header(sh, w);
    z_lane<2>(sh, tid, w);
  }
  if (tid == 0) { csize[c] = sh.bytes; cadler[c] = sh.adler; }
}

// per segment: TIF\x01, zlib header, Adler-32 (combined over the chunks), CRC-32 of the compressed bytes
__global__ void k_zfinish(const ZSeg *__restrict__ segs, uint32_t P, const uint32_t *__restrict__ cadler,
                          const uint32_t *__restrict__ csize, const uint32_t *__restrict__ seg_crc,
                          const CrcTables *__restrict__ t, uint8_t *__restrict__ out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const ZSeg s = segs[p];
  if (!s.nchunks) return;
  uint8_t *o = out + s.zstart;
  o[0] = 'T'; o[1] = 'I'; o[2] = 'F'; o[3] = 1; o[4] = 0x78; o[5] = 0x01;
  uint32_t adler = 1;
  for (uint32_t k = 0; k < s.nchunks; k++) {
    const uint64_t a = (uint64_t)k * ZCHUNK;
    adler = z_adler_combine(adler, cadler[s.chunk0 + k], z_min64(ZCHUNK, s.body_len - a));
  }
  uint8_t *tr = o + s.zlen - 8;
  store_be32(tr, adler);
  // checksummed bytes = 78 01 | chunks | adler: the chunks' raw remainders are in seg_crc (shifted past the adler)
  const uint64_t region = s.zlen - 8;
  uint32_t hraw = 0;
  hraw = t->slice[0][(hraw ^ 0x78) & 0xFF] ^ (hraw >> 8);
  hraw = t->slice[0][(hraw ^ 0x01) & 0xFF] ^ (hraw >> 8);
  uint32_t araw = 0;
  for (int b = 0; b < 4; b++) araw = t->slice[0][(araw ^ tr[b]) & 0xFF] ^ (araw >> 8);
  uint32_t raw = seg_crc[p] ^ crc_shift_bytes(t, hraw, region - 2) ^ araw;
  store_be32(tr + 4, crc_from_raw(t, raw, region));
}

}  // namespace tezgpu

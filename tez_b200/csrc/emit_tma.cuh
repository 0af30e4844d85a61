// emit_tma.cuh -- the source-oriented emit for packed, 16-byte aligned fixed-width records with the gather done by the
// bulk-copy engine (TMA): one cp.async.bulk.shared::cluster.global per record lands the record in a 16-byte aligned slot
// of a shared-memory ring and completes on the stage's mbarrier; no register staging, no LSU work, no scoreboard stalls
// for the random gather.  Warp-specialised persistent CTAs:
//   * ET_PW producer warps: sorted order -> record index -> one bulk copy per record into stage s (the issue of a bulk
//     copy is a warp-uniform instruction -- SASS UBLKCP -- so per-lane addresses serialise at ~8 instructions per copy;
//     several producer warps share a tile to keep ET_STAGES tiles in flight);
//   * ET_CW = 8 consumer warps (the 256-thread chunk interleave of the checksum): wait on the stage's mbarrier, ASSEMBLE
//     every aligned 16-byte chunk of the output byte image directly from the staged records (two LDS.128 + a funnel
//     shift for a chunk inside one record's bytes, a short composition for the chunks that straddle the 2-byte framing
//     of the next record), fold it into the tile's CRC32 and stream it to HBM -- the image of emit_pipe.cuh (five STS per
//     16 bytes + one LDS.128) is never materialised.
// Same tiles and byte-exact output as k_emit_fast4 (emit_pipe.cuh); the per-tile checksum is the chunk-interleaved
// fold of k_emit_fast4u (emit_pipe_u.cuh), not k_emit_fast4's per-thread runs.
#pragma once
#include "emit_pipe_u.cuh"

#ifndef TEZGPU_EMIT_TMA_MIN_CTAS
#define TEZGPU_EMIT_TMA_MIN_CTAS 2
#endif

namespace tezgpu {

constexpr int ET_PW = 4;                         // producer warps
constexpr int ET_CW = FE_THREADS / 32;           // consumer warps (8)
constexpr int ET_THREADS = 32 * (ET_PW + ET_CW);
constexpr int ET_STAGES = 4;
constexpr int ET_BATCH = ET_CW;                  // parked tiles per deferred second-level fold (one per consumer warp)

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t lds_b8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}

// ------------------------------------------------------------------------------------------------ 128-bit byte helpers
// (host + device: tezgpu_debug_assemble_emulate runs the same chunk assembly on the CPU, tests/test_abi_cpu.py)
__host__ __device__ __forceinline__ uint4 or4(uint4 a, uint4 b) { return make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w); }
// the low n bytes of v (n in [0, 16])
__host__ __device__ __forceinline__ uint4 low_bytes(uint4 v, uint32_t n) {
  uint32_t w[4] = {v.x, v.y, v.z, v.w};
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (uint32_t k = 0; k < 4; k++) {
    if (n <= 4 * k) w[k] = 0;
    else if (n < 4 * k + 4) w[k] &= 0xFFFFFFFFu >> (8u * (4 * k + 4 - n));
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
// v moved up by t bytes (t in [0, 15]): byte q of the result is byte q - t of v
__host__ __device__ __forceinline__ uint4 shl_bytes(uint4 v, uint32_t t) {
  uint32_t a = v.x, b = v.y, c = v.z, d = v.w, z = 0;
  // whole words first
  if (t & 8u) { d = b; c = a; b = z; a = z; }
  if (t & 4u) { d = c; c = b; b = a; a = z; }
  const uint32_t s = (t & 3u) * 8u;
  return make_uint4(a << s, fsl32(a, b, s), fsl32(b, c, s), fsl32(c, d, s));
}
// v moved down by t bytes (t in [0, 15])
__host__ __device__ __forceinline__ uint4 shr_bytes(uint4 v, uint32_t t) {
  uint32_t a = v.x, b = v.y, c = v.z, d = v.w, z = 0;
  if (t & 8u) { a = c; b = d; c = z; d = z; }
  if (t & 4u) { a = b; b = c; c = d; d = z; }
  const uint32_t s = (t & 3u) * 8u;
  return make_uint4(fsr32(a, b, s), fsr32(b, c, s), fsr32(c, d, s), d >> s);
}

// shared-memory accessors: the device one issues LDS, the host one reads a byte array (unit test)
struct DevSmem {
  __device__ __forceinline__ uint4 ld16(uint32_t a) const { return lds_v4(a); }
  __device__ __forceinline__ uint32_t ld8(uint32_t a) const { return lds_b8(a); }
};
struct HostSmem {
  const uint8_t *base;
  __host__ __device__ uint4 ld16(uint32_t a) const {
    uint4 v;
    memcpy(&v, base + a, 16);
    return v;
  }
  __host__ __device__ uint32_t ld8(uint32_t a) const { return base[a]; }
};

// 16 bytes at an arbitrary shared-memory byte address (reads the two aligned words around it)
template <class S>
__host__ __device__ __forceinline__ uint4 lds16_any(const S &sm, uint32_t a) {
  const uint32_t sh = a & 15u, a0 = a - sh;
  const uint4 lo = sm.ld16(a0);
  if (sh == 0) return lo;
  return window16(lo, sm.ld16(a0 + 16), sh);
}

struct TmaTileGeom {
  uint32_t stg;        // shared address of the stage holding the tile's records (slot j at stg + j * stride)
  uint32_t rec0;       // image offset of the first record's framing bytes
  uint32_t nr;
  uint32_t body;       // nr * rec_size
  bool first, last;
};

struct TmaEmitConst {
  uint32_t rec_size, hdr_len, stride, magic;  // magic = floor(2^32 / rec_size) + 1
  uint4 hdr;                                  // framing bytes in the low hdr_len bytes
};

__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

// one byte of the tile's output image at offset rel from the first record (edges of a tile only)
template <class S>
__host__ __device__ __forceinline__ uint32_t tma_image_byte(const S &sm, const TmaEmitConst &k, const TmaTileGeom &g, int32_t rel) {
  if (rel < 0) {
    if (!g.first || rel < -4) return 0u;
    return rel == -4 ? (uint32_t)'T' : (rel == -3 ? (uint32_t)'I' : (rel == -2 ? (uint32_t)'F' : 0u));
  }
  if ((uint32_t)rel >= g.body) return (g.last && (uint32_t)rel < g.body + 2u) ? 0xFFu : 0u;
  const uint32_t j = mulhi32((uint32_t)rel, k.magic), w = (uint32_t)rel - j * k.rec_size;
  if (w < k.hdr_len) {
    const uint32_t hw[4] = {k.hdr.x, k.hdr.y, k.hdr.z, k.hdr.w};
    return (hw[w >> 2] >> (8u * (w & 3u))) & 0xFFu;
  }
  return sm.ld8(g.stg + j * k.stride + (w - k.hdr_len));
}

// the aligned 16-byte chunk of the tile's output image that starts at image offset X
template <class S>
__host__ __device__ __forceinline__ uint4 tma_assemble(const S &sm, const TmaEmitConst &k, const TmaTileGeom &g, uint32_t X) {
  const int32_t rel = (int32_t)X - (int32_t)g.rec0;
  if (rel >= 0 && (uint32_t)rel + 16u <= g.body) {
    uint32_t j = mulhi32((uint32_t)rel, k.magic), w = (uint32_t)rel - j * k.rec_size;
    if (w >= k.hdr_len && w + 16u <= k.rec_size)      // inside one record's key||value bytes: the common case
      return lds16_any(sm, g.stg + j * k.stride + (w - k.hdr_len));
    // the chunk straddles framing bytes: [rest of record j] [framing of j+1] [start of j+1's bytes]
    uint4 acc = make_uint4(0, 0, 0, 0);
    uint32_t t = 0;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int q = 0; q < 2 && t < 16u; q++, j++, w = 0) {
      if (w < k.hdr_len) {
        const uint32_t n = (k.hdr_len - w) < (16u - t) ? (k.hdr_len - w) : (16u - t);
        acc = or4(acc, shl_bytes(low_bytes(shr_bytes(k.hdr, w), n), t));
        t += n;
        w += n;
      }
      if (t < 16u) {
        const uint32_t d = w - k.hdr_len, n = (k.stride - d) < (16u - t) ? (k.stride - d) : (16u - t);
        acc = or4(acc, shl_bytes(low_bytes(lds16_any(sm, g.stg + j * k.stride + d), n), t));
        t += n;
      }
    }
    return acc;
  }
  // tile edges (segment header, EOF markers, the neighbours' bytes): byte by byte
  uint32_t w4[4] = {0, 0, 0, 0};
  for (uint32_t b = 0; b < 16u; b++) w4[b >> 2] |= tma_image_byte(sm, k, g, rel + (int32_t)b) << (8u * (b & 3u));
  return make_uint4(w4[0], w4[1], w4[2], w4[3]);
}

struct EmitTmaLayout {
  // shared memory: [mbarriers 256 B][classic table 1 KB][adv128 4 KB][stages][partials 2 x BATCH x 256 x 4][fold meta 2 x BATCH]
  static constexpr size_t BARS = 256;
  static constexpr size_t TABS = 256 * 4 + 4 * 256 * 4;
  static size_t stage_bytes(uint32_t recs_per_tile, uint32_t stride) { return align_up((uint64_t)recs_per_tile * stride + 32, 128); }
  static size_t total(uint32_t recs_per_tile, uint32_t stride) {
    return BARS + TABS + ET_STAGES * stage_bytes(recs_per_tile, stride) + 2 * (size_t)ET_BATCH * FE_THREADS * 4 +
           2 * (size_t)ET_BATCH * sizeof(FoldMeta);
  }
};

__global__ void __launch_bounds__(ET_THREADS, TEZGPU_EMIT_TMA_MIN_CTAS) k_emit_tma(FastEmitParams fp, uint32_t stage_bytes) {
  extern __shared__ __align__(128) uint8_t smem_t[];
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem_t);                                  // [STAGES] full, [STAGES] empty
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem_t + EmitTmaLayout::BARS);           // classic byte table (trailing bytes)
  uint32_t *s_adv128 = s_tab + 256;                                                       // * x^(32*128): second-level fold
  uint8_t *s_ring = smem_t + EmitTmaLayout::BARS + EmitTmaLayout::TABS;
  uint32_t(*s_part)[FE_THREADS] = reinterpret_cast<uint32_t(*)[FE_THREADS]>(s_ring + (size_t)ET_STAGES * stage_bytes);
  FoldMeta *s_meta = reinterpret_cast<FoldMeta *>(reinterpret_cast<uint8_t *>(s_part) + 2 * (size_t)ET_BATCH * FE_THREADS * 4);

  const EmitParams &e = fp.e;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t G = gridDim.x, ntiles = fp.ntiles;
  const uint32_t full0 = (uint32_t)__cvta_generic_to_shared(bars), empty0 = full0 + 8 * ET_STAGES;
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(s_ring);
  if (threadIdx.x == 0) {
    for (int s = 0; s < ET_STAGES; s++) {
      mbar_init(full0 + 8 * s, ET_PW);
      mbar_init(empty0 + 8 * s, ET_CW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < 256; i += ET_THREADS) s_tab[i] = e.crc->slice[0][i];
  for (int i = threadIdx.x; i < 4 * 256; i += ET_THREADS) s_adv128[i] = (&e.crc->adv128[0][0])[i];
  __syncthreads();
  if (blockIdx.x >= ntiles) return;
  const TileDesc *__restrict__ tiles = fp.tiles;
  const uint32_t stride = fp.stride;

  if (warp < ET_PW) {
    // ================================================================ producers
    const uint8_t *__restrict__ kv = e.rec.kv;
    const uint32_t full_nr = e.recs_per_tile;
    const uint32_t rpw = (full_nr + ET_PW - 1) / ET_PW;        // records of a tile per producer warp
    const uint32_t rpl = (rpw + 31) / 32;                      // ... per lane (consecutive slots)
    const uint32_t j0 = (uint32_t)warp * rpw + (uint32_t)lane * rpl;
    uint32_t it = 0;
    // indices of the first tile
    uint32_t r0n = tiles[blockIdx.x].r0, nrn = tiles[blockIdx.x].nr;
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += G, it++) {
      const uint32_t s = it % ET_STAGES, ph = (it / ET_STAGES) & 1u;
      const uint32_t r0 = r0n, nr = nrn;
      if (tile + G < ntiles) { r0n = tiles[tile + G].r0; nrn = tiles[tile + G].nr; }
      const uint32_t wend = min(nr, ((uint32_t)warp + 1u) * rpw);   // this warp moves slots [warp * rpw, wend)
      const uint32_t wcnt = wend > (uint32_t)warp * rpw ? wend - (uint32_t)warp * rpw : 0u;
      const uint32_t jend = min(wend, j0 + rpl);
      // record indices first (their latency overlaps the wait for the stage)
      uint32_t idx[8];
#pragma unroll
      for (uint32_t q = 0; q < 8; q++) idx[q] = (q < rpl && j0 + q < jend) ? __ldg(e.order + r0 + j0 + q) : 0u;
      if (it >= ET_STAGES) mbar_wait(empty0 + 8 * s, ph ^ 1u);
      const uint32_t bar = full0 + 8 * s;
      if (lane == 0) mbar_arrive_expect_tx(bar, wcnt * stride);
      __syncwarp();
      const uint32_t dst = ring0 + s * stage_bytes + j0 * stride;
#pragma unroll
      for (uint32_t q = 0; q < 8; q++)
        if (q < rpl && j0 + q < jend) bulk_copy_g2s(dst + q * stride, kv + (uint64_t)idx[q] * stride, stride, bar);
    }
    return;
  }

  // ================================================================== consumers (256 threads)
  const int tid = threadIdx.x - 32 * ET_PW, cwarp = tid >> 5;
  TmaEmitConst kc;
  kc.rec_size = e.rec_size;
  kc.hdr_len = e.fixed_hdr_len;
  kc.stride = stride;
  kc.magic = (uint32_t)((1ull << 32) / e.rec_size) + 1u;
  {
    uint32_t hw[4] = {0, 0, 0, 0};
    for (uint32_t b = 0; b < e.fixed_hdr_len; b++) hw[b >> 2] |= (uint32_t)e.fixed_hdr[b] << (8u * (b & 3u));
    kc.hdr = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  }
  CrcChunkFoldT<false> cf;  // the chunk fold's linear maps as warp-resident digit tables (crc32.cuh)
  cf.init(e.crc, lane);
  const uint32_t lane_pow = cf.lane_pow;
  auto consumer_sync = [&]() { asm volatile("bar.sync 1, %0;" ::"n"(FE_THREADS) : "memory"); };

  uint32_t it = 0, slot = 0, batch = 0;
  TileDesc tdn = tiles[blockIdx.x];
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += G, it++) {
    const uint32_t s = it % ET_STAGES, ph = (it / ET_STAGES) & 1u;
    const TileDesc td = tdn;
    const bool has1 = tile + G < ntiles;
    if (has1) tdn = tiles[tile + G];
    TmaTileGeom g;
    g.stg = ring0 + s * stage_bytes;
    g.nr = td.nr;
    g.first = td.flags & 1u;
    g.last = td.flags & 2u;
    const uint32_t lead = (uint32_t)(td.abs0 & 15u);
    g.rec0 = lead + (g.first ? 4u : 0u);
    g.body = td.nr * kc.rec_size;
    const uint32_t body_end = g.rec0 + g.body + (g.last ? 2u : 0u);
    const uint32_t cb0 = g.rec0, cb1 = body_end;
    const uint32_t ca = cb0 >> 4, cz = cb1 >> 4;
    uint8_t *dstg = e.out + (td.abs0 - lead);

    mbar_wait(full0 + 8 * s, ph);   // the tile's records have landed

    // ---- fused assemble + CRC + write-out: thread t owns the chunks at distance == T-1-t (mod T) from the end
    uint32_t c = 0;
    if (cz > ca) {
      const uint32_t Cn = cz - ca;
      const uint32_t iters = (Cn + FE_THREADS - 1) / FE_THREADS;
      int32_t i = (int32_t)Cn + tid - (int32_t)(iters * FE_THREADS);
      uint8_t *gp = dstg + 16ll * ((int64_t)ca + i);
      for (uint32_t itc = 0; itc < iters; itc++, i += FE_THREADS, gp += 16 * FE_THREADS) {
        if (i + (31 - lane) < 0) continue;  // no lane of this warp owns a chunk yet (first, ragged round only)
        uint4 w = make_uint4(0, 0, 0, 0);
        if (i >= 0) {
          w = tma_assemble(DevSmem(), kc, g, 16u * (ca + (uint32_t)i));
          if (i == 0) {
            const uint32_t b0 = 16u * ca;
            if (b0 >= lead) stg_stream_v4(gp, w);
            else {  // ragged first chunk of the tile: the bytes before `lead` belong to the previous tile
              const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
              for (uint32_t x = lead; x < b0 + 16u; x++) dstg[x] = (uint8_t)(ww[(x - b0) >> 2] >> (8u * ((x - b0) & 3u)));
            }
            const uint32_t skip = cb0 & 15u;  // bytes before the body (segment header / previous tile) fold as zero
            if (skip) {
              uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
              for (uint32_t q = 0; q < 4; q++) {
                if (skip >= 4 * q + 4) ww[q] = 0;
                else if (skip > 4 * q) ww[q] &= 0xFFFFFFFFu << (8u * (skip - 4 * q));
              }
              w = make_uint4(ww[0], ww[1], ww[2], ww[3]);
            }
          } else {
            stg_stream_v4(gp, w);
          }
        }
        c = cf.fold(c, w, itc + 1 == iters);
      }
    }
    const uint32_t row = (batch & 1u) * ET_BATCH + slot;
    s_part[row][tid] = c;
    if (tid == 0) {
      // bytes outside the whole chunks: trailing partial chunk, and a leading header-only chunk
      const uint4 tail = tma_assemble(DevSmem(), kc, g, 16u * cz);   // cz == ca when there is no whole chunk
      const uint32_t tw[4] = {tail.x, tail.y, tail.z, tail.w};
      for (uint32_t x = max(lead, 16u * cz); x < body_end; x++) dstg[x] = (uint8_t)(tw[(x & 15u) >> 2] >> (8u * (x & 3u)));
      if (ca > (lead >> 4))
        for (uint32_t x = lead; x < 16u * ca; x++) dstg[x] = (uint8_t)tma_image_byte(DevSmem(), kc, g, (int32_t)x - (int32_t)g.rec0);
      FoldMeta m;
      m.tail = tail;
      m.tile = tile;
      m.tiny = cz > ca ? 0u : 1u;
      m.start = cz > ca ? 0u : (cb0 & 15u);
      m.end = cb1 & 15u;
      s_meta[row] = m;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * s);   // this warp is done reading the stage
    slot++;

    if (slot == (uint32_t)ET_BATCH || !has1) {
      // ---- deferred second level: consumer warp w folds parked tile w of this batch.  Rows alternate between two
      // banks per batch: a row of this bank is rewritten two batches later, i.e. after the next batch's barrier, which
      // every folding warp reaches only after its fold.
      consumer_sync();
      if ((uint32_t)cwarp < slot) {
        const uint32_t r2 = (batch & 1u) * ET_BATCH + (uint32_t)cwarp;
        uint32_t q = 0;
#pragma unroll
        for (int kk = 0; kk < FE_THREADS / 32; kk++) {
          q = s_adv128[q & 0xFF] ^ s_adv128[256 + ((q >> 8) & 0xFF)] ^ s_adv128[512 + ((q >> 16) & 0xFF)] ^ s_adv128[768 + (q >> 24)];
          q ^= s_part[r2][lane + 32 * kk];
        }
        q = crc_multmodp(q, lane_pow);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) q ^= __shfl_xor_sync(0xffffffffu, q, o);
        if (lane == 0) {
          const FoldMeta m = s_meta[r2];
          const uint32_t tw[4] = {m.tail.x, m.tail.y, m.tail.z, m.tail.w};
          uint32_t raw = m.tiny ? 0u : q;
          for (uint32_t b = m.start; b < m.end; b++) {
            const uint32_t byte = (tw[b >> 2] >> (8u * (b & 3u))) & 0xFFu;
            raw = s_tab[(raw ^ byte) & 0xFF] ^ (raw >> 8);
          }
          const TileDesc t2 = tiles[m.tile];
          TileCrc tc;
          tc.raw = raw;
          tc.p = t2.p;
          tc.after = t2.after;
          fp.tile_crc[m.tile] = tc;
        }
      }
      slot = 0;
      batch++;
    }
  }
}

// can the TMA kernel serve this layout?  (slots per lane, shared memory)
static inline bool emit_tma_fits(uint32_t recs_per_tile, uint32_t stride) {
  const uint32_t rpw = (recs_per_tile + ET_PW - 1) / ET_PW, rpl = (rpw + 31) / 32;
  return stride % 16 == 0 && stride >= 16 && rpl <= 8 && EmitTmaLayout::total(recs_per_tile, stride) <= 110 * 1024;
}

}  // namespace tezgpu

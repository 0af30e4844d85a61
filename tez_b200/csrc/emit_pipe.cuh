// emit_pipe.cuh -- software-pipelined variant of the source-oriented emit kernel (emit_fast.cuh) for packed,
// 16-byte aligned fixed-width records.
//
// k_emit_fast saturates no pipe: its warps wait on the gather's global loads and at barriers (behind warp 0 folding
// the tile's partial checksums while seven warps idle).  This kernel keeps the same byte-exact output but reorders the
// work of a persistent CTA:
//   * the 128-bit gather loads of tile N+1 are issued into registers BEFORE the checksum / write-out of tile N and
//     stored to the image after it (record indices are fetched two tiles ahead, tile descriptors three), so the DRAM
//     latency of the random gather hides behind the checksum work;
//   * the per-tile second-level checksum fold is deferred: partials of FE4_PARKED tiles are parked in shared memory
//     and folded together, one tile per warp, so no warp waits for another's serial fold;
//   * two barriers per tile instead of three.
// Checksum organisation (CRC32 in parallel, see DESIGN.md): a tile image holds at most FE_THREADS * FE4_RUN 16-byte
// chunks; thread t folds the FE4_RUN whole chunks at distance [FE4_RUN*(255-t), FE4_RUN*(256-t)) from the end of the
// tile body with the textbook chain c = W(c ^ word) ("next word" map W = * x^32 only), so its alignment multiplier
// x^(8*80*(255-t)) does not depend on the tile's length.  W runs on lane-private digit tables in shared memory.
#pragma once
#include "emit_fast.cuh"

#ifndef TEZGPU_EMIT4_MIN_CTAS
#define TEZGPU_EMIT4_MIN_CTAS 3  // CTAs per SM of k_emit_fast4u (emit_pipe_u.cuh)
#endif

namespace tezgpu {

constexpr int FE4_BATCH = FE_THREADS / 32;  // one parked tile per warp (k_emit_fast4u)
constexpr int FE4_UNROLL = 5;               // gather rounds held in registers
constexpr int FE4_RUN = 5;                  // 16-byte chunks per thread-run of the checksum
constexpr uint32_t FE4_RUN_BYTES = 16u * FE4_RUN;
constexpr int FE4_IMG_BYTES = FE_THREADS * FE4_RUN * 16;  // 20480: the tile image is exactly FE4_RUN rounds of chunks
// Shared-memory footprint decides this kernel on H100 (DESIGN.md §7): the CTA's total picks the carveout, and what the
// carveout leaves as L1 bounds the random gather's loads in flight.  Two groups, four parked tiles and 7-bit digits
// come to 125 KB (the 132 KB carveout).  8-bit digits (4 tables, 16 LDS per chunk instead of 20) take 128 KB of
// tables alone and were 1.8 ms slower than 7-bit ones at the same layout; 6-bit digits with three groups fit the
// 132 KB carveout too and were 0.07 ms slower.
// independent 256-thread groups per CTA (one CTA per SM); they share the checksum tables
constexpr int FE4_GROUPS = 2;
// tiles whose partials a group parks before folding them (one warp each)
constexpr int FE4_PARKED = 4;
// digit width of the lane-private tables of W: 7 bits -> tables of 128, 128, 128, 128 and 16 entries (66 KB, 20 LDS
// per chunk)
constexpr int FE4_WBITS = 7;
constexpr int FE4_WDIGITS = (32 + FE4_WBITS - 1) / FE4_WBITS;
constexpr int FE4_WENTRIES = ((FE4_WDIGITS - 1) << FE4_WBITS) + (1 << (32 - FE4_WBITS * (FE4_WDIGITS - 1)));

// records of `rec_size` bytes a tile image holds in the worst case (lead <= 15, segment header 4, EOF marker 2)
static inline uint32_t emit4_max_recs(uint32_t rec_size) {
  return std::min<uint32_t>(FE_MAX_RECS, (FE4_IMG_BYTES - 15 - 4 - 2) / rec_size);
}

// pieces per record the kernel serves: the packed piece map of full tiles (k_emit_fast4) keeps a piece's byte offset
// in its record, 16c, in 7 bits
constexpr uint32_t FE4_MAX_CPR = 8;

// can a tile of `recs` records of `rec_size` bytes with `cpr` pieces each be gathered in FE4_UNROLL rounds and fit the
// image?
static inline bool emit4_fits(uint32_t recs, uint32_t cpr, uint32_t rec_size) {
  if (cpr > FE4_MAX_CPR || recs > emit4_max_recs(rec_size)) return false;
  return (uint64_t)recs * cpr <= (uint64_t)FE4_UNROLL * FE_THREADS;
}

// W = "* x^32" on a word whose digit k (FE4_WBITS wide, the top one narrower) is e: the value of entry e of digit
// table k (host and device: the host emulation in tezgpu_api.cu builds the same tables)
__host__ __device__ __forceinline__ uint32_t emit4_wtab_value(const CrcTables *__restrict__ t, uint32_t k, uint32_t e) {
  const uint32_t v = e << (FE4_WBITS * k);
  return t->slice[3][v & 0xFF] ^ t->slice[2][(v >> 8) & 0xFF] ^ t->slice[1][(v >> 16) & 0xFF] ^ t->slice[0][v >> 24];
}

// W (* x^32) of x through the lane-private digit tables (layout: Emit4Smem); `wt` is this lane's word of entry 0 of
// table 0.  Entry e of a table is e * 128 bytes from its start: digit k is shifted straight to that position and
// masked (shift, and, add, load per digit).  Host and device: the host emulation in tezgpu_api.cu runs this code on a
// table laid out like the kernel's.
__host__ __device__ __forceinline__ uint32_t emit4_next_word(const uint8_t *wt, uint32_t x) {
  uint32_t r = 0;
#pragma unroll
  for (int k = 0; k < FE4_WDIGITS; k++) {
    constexpr int E = 7;  // log2(32 lanes * 4 bytes)
    const int sh = FE4_WBITS * k - E;
    const uint32_t m = (k + 1 < FE4_WDIGITS ? (1u << FE4_WBITS) - 1 : (1u << (32 - FE4_WBITS * k)) - 1) << E;
    const uint32_t off = (sh >= 0 ? x >> sh : x << -sh) & m;
    r ^= *reinterpret_cast<const uint32_t *>(wt + off + ((size_t)k << (FE4_WBITS + E)));
  }
  return r;
}

struct FoldMeta {
  uint4 tail;       // the 16-byte chunk holding the bytes the chunk loop did not fold
  uint32_t tile;
  uint32_t start;   // byte range [start, end) of `tail` to fold bytewise
  uint32_t end;
  uint32_t tiny;    // 1: the whole body lies inside `tail` (no whole chunk): start from a zero remainder
};

__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}

// Shared memory: the lane-private digit tables of W (entry e of table k for lane l at word (k << FE4_WBITS + e) * 32
// + l, always bank l: conflict-free whatever the digits), the classic byte table (trailing bytes) and the byte tables
// of the second-level Horner step; then per group the tile image, three tiles' record indices and the parked tiles.
struct Emit4Smem {
  static constexpr size_t WTAB = (size_t)FE4_WENTRIES * 32 * 4;
  static constexpr size_t SHARED = WTAB + 256 * 4 + 4 * 256 * 4;
  static constexpr size_t GROUP = FE4_IMG_BYTES + 3 * FE_MAX_RECS * 4 + (size_t)FE4_PARKED * FE_THREADS * 4 + (size_t)FE4_PARKED * sizeof(FoldMeta);
  static constexpr size_t TOTAL = SHARED + FE4_GROUPS * GROUP;
};

template <int UNROLL>
__global__ void __launch_bounds__(FE_THREADS * FE4_GROUPS, 1) k_emit_fast4(FastEmitParams fp) {
  using L = Emit4Smem;
  constexpr int BATCH = FE4_PARKED;
  extern __shared__ __align__(16) uint8_t smem4[];
  uint32_t *s_wtab = reinterpret_cast<uint32_t *>(smem4);              // [FE4_WENTRIES][32] lane-private
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem4 + L::WTAB);     // classic byte table (trailing bytes)
  uint32_t *s_hor = s_tab + 256;                                       // * x^(8*80*32): second-level Horner step
  const int sub = threadIdx.x / FE_THREADS, tid = threadIdx.x % FE_THREADS, lane = tid & 31, warp = tid >> 5;
  uint8_t *gbase = smem4 + L::SHARED + (size_t)sub * L::GROUP;
  uint8_t *s_img = gbase;
  uint32_t(*s_idx)[FE_MAX_RECS] = reinterpret_cast<uint32_t(*)[FE_MAX_RECS]>(gbase + FE4_IMG_BYTES);  // tiles N, N+1, N+2
  uint32_t(*s_part)[FE_THREADS] = reinterpret_cast<uint32_t(*)[FE_THREADS]>(gbase + FE4_IMG_BYTES + 3 * FE_MAX_RECS * 4);
  FoldMeta *s_meta = reinterpret_cast<FoldMeta *>(gbase + FE4_IMG_BYTES + 3 * FE_MAX_RECS * 4 + (size_t)BATCH * FE_THREADS * 4);
  auto group_sync = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(sub + 1), "r"(FE_THREADS) : "memory"); };

  const EmitParams &e = fp.e;
  const uint32_t G = gridDim.x * FE4_GROUPS, ntiles = fp.ntiles;
  uint32_t tile = blockIdx.x * FE4_GROUPS + sub;
  for (int i = threadIdx.x; i < FE4_WENTRIES * 32; i += FE_THREADS * FE4_GROUPS)
    s_wtab[i] = emit4_wtab_value(e.crc, (uint32_t)(i >> 5) >> FE4_WBITS, (uint32_t)(i >> 5) & ((1u << FE4_WBITS) - 1));
  for (int i = threadIdx.x; i < 256; i += FE_THREADS * FE4_GROUPS) s_tab[i] = e.crc->slice[0][i];
  {
    const uint32_t x_hor = e.crc->pow0[FE4_RUN_BYTES * 32];
    for (int i = threadIdx.x; i < 4 * 256; i += FE_THREADS * FE4_GROUPS) s_hor[i] = crc_multmodp((uint32_t)(i & 255) << (8 * (i >> 8)), x_hor);
  }
  __syncthreads();
  if (tile >= ntiles) return;
  const uint32_t lane_pow = e.crc->pow0[FE4_RUN_BYTES * (31 - lane)];  // x^(8*80*(31-lane))
  const uint8_t *wt = reinterpret_cast<const uint8_t *>(s_wtab + lane);  // this lane's bank
  auto next_word = [&](uint32_t x) -> uint32_t { return emit4_next_word(wt, x); };
  const uint32_t img_base = (uint32_t)__cvta_generic_to_shared(s_img);
  const uint8_t *__restrict__ kv = e.rec.kv;
  const uint32_t rec_size = e.rec_size, hdr_len = e.fixed_hdr_len, stride = fp.stride, cpr = fp.cpr;
  const TileDesc *__restrict__ tiles = fp.tiles;

  // piece slot of a tile <-> (record j, 16-byte piece c): consecutive lanes take consecutive pieces.
  // Even records first, then odd ones (emit_fast.cuh): keeps a warp on one unaligned-store path.
  auto piece = [&](int u, uint32_t nr, uint32_t &j, uint32_t &c) -> bool {
    const uint32_t q = tid + u * FE_THREADS;
    const uint32_t jp = cpr == 1 ? q : __umulhi(q, fp.cpr_magic);
    c = q - jp * cpr;
    const uint32_t half_up = (nr + 1) >> 1;
    j = jp < half_up ? 2u * jp : 2u * (jp - half_up) + 1u;
    return q < nr * cpr;
  };
  // Full tiles (all but the last of a partition) share one piece map: packed once per thread as
  // j | 16c << 8 | (j * rec_size + hdr_len + 16c) << 15 (j < 256, 16c < 128: cpr <= FE4_MAX_CPR, checked by
  // emit4_fits), so a piece costs an index look-up and one multiply-add instead of the divide / permute arithmetic
  // (which was ~25 % of the kernel's instructions).
  const uint32_t full_nr = e.recs_per_tile;
  uint32_t pk[UNROLL], onmask = 0;
#pragma unroll
  for (int u = 0; u < UNROLL; u++) {
    uint32_t j, c;
    const bool on = piece(u, full_nr, j, c);
    pk[u] = on ? (j | (16u * c) << 8 | (j * rec_size + hdr_len + 16u * c) << 15) : 0u;
    onmask |= on ? 1u << u : 0u;
  }
  uint4 v[UNROLL];
  // all addresses first, then the loads back to back (keeps ptxas from reusing the destination registers of later
  // rounds as temporaries between the loads)
  auto issue_gather = [&](uint32_t nr, const uint32_t *idx) {
    const uint8_t *src[UNROLL];
    bool on[UNROLL];
    if (nr == full_nr) {
#pragma unroll
      for (int u = 0; u < UNROLL; u++) {
        on[u] = (onmask >> u) & 1u;
        src[u] = kv + (uint64_t)idx[pk[u] & 0xFFu] * stride + ((pk[u] >> 8) & 0x7Fu);
      }
    } else {
#pragma unroll
      for (int u = 0; u < UNROLL; u++) {
        uint32_t j, c;
        on[u] = piece(u, nr, j, c);
        src[u] = kv + (uint64_t)idx[on[u] ? j : 0u] * stride + 16u * c;
      }
    }
    if (UNROLL == 5) asm volatile("" : "+l"(src[0]), "+l"(src[1]), "+l"(src[2]), "+l"(src[3]), "+l"(src[UNROLL - 1]));
#pragma unroll
    for (int u = 0; u < UNROLL; u++)
      if (on[u]) v[u] = ldg_stream_v4(src[u]);
  };
  // vint(klen) vint(vlen) of the fixed framing as one 16-bit store when it is two bytes at an even address
  const uint32_t hdr16 = (uint32_t)e.fixed_hdr[0] | (uint32_t)e.fixed_hdr[1] << 8;

  // ---- prologue: descriptors of tiles 0..2 of this CTA, indices of tiles 0 and 1, gather of tile 0 in flight
  uint32_t nr0, fl0, nr1 = 0, fl1 = 0, r0_2 = 0, nr2 = 0;
  uint64_t abs0, abs1 = 0;
  {
    const TileDesc t0 = tiles[tile];
    nr0 = t0.nr; fl0 = t0.flags; abs0 = t0.abs0;
    if ((uint32_t)tid < nr0) s_idx[0][tid] = e.order[t0.r0 + tid];
    if (tile + G < ntiles) {
      const TileDesc t1 = tiles[tile + G];
      nr1 = t1.nr; fl1 = t1.flags; abs1 = t1.abs0;
      if ((uint32_t)tid < nr1) s_idx[1][tid] = e.order[t1.r0 + tid];
    }
    if (tile + 2 * (uint64_t)G < ntiles) { r0_2 = tiles[tile + 2 * G].r0; nr2 = tiles[tile + 2 * G].nr; }
  }
  group_sync();
  issue_gather(nr0, s_idx[0]);

  uint32_t n_it = 0, slot = 0;
  for (;; tile += G, n_it++) {
    const bool has1 = tile + G < ntiles, has2 = tile + 2 * (uint64_t)G < ntiles, has3 = tile + 3 * (uint64_t)G < ntiles;
    const uint32_t nr = nr0;
    const bool first_tile = fl0 & 1u, last_tile = fl0 & 2u;
    const uint32_t lead = (uint32_t)(abs0 & 15u);
    const uint32_t rec0 = lead + (first_tile ? 4u : 0u);
    const uint32_t body_end = rec0 + nr * rec_size + (last_tile ? 2u : 0u);

    // ---- prefetches that are consumed at the end of this iteration / in the next one
    uint32_t r_idx = 0, r0_3 = 0, nr3 = 0, nr2n = 0, fl2n = 0;
    uint64_t abs2n = 0;
    if (has2) {
      if ((uint32_t)tid < nr2) r_idx = e.order[r0_2 + tid];
      const TileDesc *t2 = tiles + tile + 2 * (uint64_t)G;
      nr2n = t2->nr; fl2n = t2->flags; abs2n = t2->abs0;
    }
    if (has3) { const TileDesc *t3 = tiles + tile + 3 * (uint64_t)G; r0_3 = t3->r0; nr3 = t3->nr; }

    // ---- this tile's pieces (loaded during the previous iteration) -> image; framing
    if (nr == full_nr) {
#pragma unroll
      for (int u = 0; u < UNROLL; u++)
        if ((onmask >> u) & 1u) sts16_unaligned(img_base + rec0 + (pk[u] >> 15), v[u]);
    } else {
#pragma unroll
      for (int u = 0; u < UNROLL; u++) {
        uint32_t j, c;
        if (piece(u, nr, j, c)) sts16_unaligned(img_base + rec0 + j * rec_size + hdr_len + 16u * c, v[u]);
      }
    }
    if ((uint32_t)tid < nr) {
      const uint32_t a = img_base + rec0 + tid * rec_size;
      if (hdr_len == 2 && !(a & 1u)) sts_b16(a, hdr16);
      else for (uint32_t b = 0; b < hdr_len; b++) sts_b8(a + b, e.fixed_hdr[b]);
    }
    if (tid == 0) {
      if (first_tile) { s_img[lead] = 'T'; s_img[lead + 1] = 'I'; s_img[lead + 2] = 'F'; s_img[lead + 3] = 0; }
      if (last_tile) { s_img[body_end - 2] = 0xFF; s_img[body_end - 1] = 0xFF; }
    }
    group_sync();  // (B) image complete

    // ---- gather of the next tile goes out now; it lands while this tile is checksummed and written
    if (has1) issue_gather(nr1, s_idx[(n_it + 1) % 3]);

    // ---- write-out (lane-consecutive chunks, coalesced), then the checksum of this thread's run
    const uint32_t cb0 = rec0, cb1 = body_end;
    const uint32_t ca = cb0 >> 4, cz = cb1 >> 4;
    uint8_t *dstg = e.out + (abs0 - lead);
    uint32_t c = 0;
    if (cz > ca) {
      const int32_t Cn = (int32_t)(cz - ca);
      for (int32_t i = tid; i < Cn; i += FE_THREADS) {
        const uint4 w = lds_v4(img_base + 16u * (ca + (uint32_t)i));
        if (i > 0 || 16u * ca >= lead) stg_stream_v4(dstg + 16u * (ca + (uint32_t)i), w);
        else for (uint32_t x = lead; x < 16u * ca + 16u; x++) dstg[x] = s_img[x];  // ragged first chunk of the tile
      }
      // thread t: chunks [Cn - FE4_RUN*(256-t), Cn - FE4_RUN*(255-t)); those before the body are zeros, which leave a
      // zero remainder unchanged
      const int32_t i0 = Cn - FE4_RUN * (FE_THREADS - tid);
#pragma unroll
      for (int k = 0; k < FE4_RUN; k++) {
        const int32_t i = i0 + k;
        if (i < 0) continue;
        uint4 w = lds_v4(img_base + 16u * (ca + (uint32_t)i));  // 80-byte lane stride: conflict-free quarter-warps
        if (i == 0) {
          const uint32_t skip = cb0 & 15u;  // bytes before the body (segment header / previous tile) fold as zero
          uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
          for (uint32_t q = 0; q < 4; q++) {
            if (skip >= 4 * q + 4) ww[q] = 0;
            else if (skip > 4 * q) ww[q] &= 0xFFFFFFFFu << (8u * (skip - 4 * q));
          }
          w = make_uint4(ww[0], ww[1], ww[2], ww[3]);
        }
        c = next_word(c ^ w.x);
        c = next_word(c ^ w.y);
        c = next_word(c ^ w.z);
        c = next_word(c ^ w.w);
      }
    }
    s_part[slot][tid] = c;
    if (tid == 0) {
      // bytes outside the whole chunks: trailing partial chunk, and a leading header-only chunk
      for (uint32_t x = max(lead, 16u * cz); x < body_end; x++) dstg[x] = s_img[x];
      if (ca > (lead >> 4)) for (uint32_t x = lead; x < 16u * ca; x++) dstg[x] = s_img[x];
      FoldMeta m;
      m.tail = *reinterpret_cast<const uint4 *>(s_img + 16u * cz);  // cz == ca when there is no whole chunk
      m.tile = tile;
      m.tiny = cz > ca ? 0u : 1u;
      m.start = cz > ca ? 0u : (cb0 & 15u);
      m.end = cb1 & 15u;
      s_meta[slot] = m;
    }
    if (has2) s_idx[(n_it + 2) % 3][tid] = r_idx;
    slot++;
    group_sync();  // (C) image free, partials / indices visible

    if (slot == (uint32_t)BATCH || !has1) {
      // ---- deferred second level: warp w folds parked tile w.  lane l folds partials l, l+32, ... (Horner with
      // x^(8*80*32)), aligns by x^(8*80*(31-l)), xor-reduce; lane 0 appends the trailing bytes
      if ((uint32_t)warp < slot) {
        uint32_t q = 0;
#pragma unroll
        for (int k = 0; k < FE_THREADS / 32; k++) {
          q = s_hor[q & 0xFF] ^ s_hor[256 + ((q >> 8) & 0xFF)] ^ s_hor[512 + ((q >> 16) & 0xFF)] ^ s_hor[768 + (q >> 24)];
          q ^= s_part[warp][lane + 32 * k];
        }
        q = crc_multmodp(q, lane_pow);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) q ^= __shfl_xor_sync(0xffffffffu, q, o);
        if (lane == 0) {
          const FoldMeta m = s_meta[warp];
          const uint32_t tw[4] = {m.tail.x, m.tail.y, m.tail.z, m.tail.w};
          uint32_t raw = m.tiny ? 0u : q;
          for (uint32_t b = m.start; b < m.end; b++) {
            const uint32_t byte = (tw[b >> 2] >> (8u * (b & 3u))) & 0xFFu;
            raw = s_tab[(raw ^ byte) & 0xFF] ^ (raw >> 8);
          }
          const TileDesc td = tiles[m.tile];
          TileCrc tc;
          tc.raw = raw;
          tc.p = td.p;
          tc.after = td.after;
          fp.tile_crc[m.tile] = tc;
        }
      }
      slot = 0;
      // the parked rows are rewritten only after barrier (B) of the next iteration, which every folding warp joins
    }
    if (!has1) break;
    // the descriptor prefetches are consumed HERE: without this the compiler renames them straight into the next
    // iteration, where their scoreboard is shared with the freshly issued gather loads and the first use stalls on
    // those (the first use of a prefetched descriptor then waits for the whole gather)
    asm volatile("" : "+r"(nr2n), "+r"(fl2n), "+l"(abs2n), "+r"(r0_3), "+r"(nr3));
    nr0 = nr1; fl0 = fl1; abs0 = abs1;
    nr1 = nr2n; fl1 = fl2n; abs1 = abs2n;
    r0_2 = r0_3; nr2 = nr3;
  }
}

}  // namespace tezgpu

// emit_pipe_u.cuh -- the software-pipelined emit kernel (emit_pipe.cuh) for fixed-width records at ARBITRARY byte
// offsets: parsed IFile segments on the reduce side, where a record's key||value bytes start wherever the producer's
// framing put them.  Same tile algorithm and byte-exact output as k_emit_fast<.,false>; differences:
//   * gather by aligned 128-bit words: a record of cpr 16-byte pieces spans at most cpr+1 aligned words; a warp takes
//     32/(cpr+1) whole records per round, lane k of a record loads word k once (k_emit_fast<.,false> loads two words per
//     piece) and gets word k+1 from its neighbour lane by SHFL when the piece is assembled (funnel shift by the
//     record's misalignment);
//   * the loads of tile N+1 are issued before the checksum loop of tile N; source offsets (two dependent global loads:
//     sorted order -> record index -> byte offset) are fetched three / two tiles ahead;
//   * batched second-level checksum folds, two barriers per tile (as emit_pipe.cuh).
// Records of more than 31 pieces do not fit a warp's round and take k_emit_fast<5,false> (plan_fixed_emit, sorter.cuh).
//
// The checksum / write-out loop and the batched fold are NOT those of k_emit_fast4 any more: that kernel folds
// per-thread runs of five chunks on lane-private tables (one CTA of two groups per SM), this one still folds the
// 256-thread chunk interleave with SHFL digit tables (CrcChunkFoldT<false>) at three CTAs per SM.  Porting the run fold
// here is a separate, measured change.
#pragma once
#include "emit_pipe.cuh"

namespace tezgpu {

struct Emit4uSmem {
  static constexpr size_t SHARED = 256 * 4 + 4 * 256 * 4;
  static constexpr size_t TOTAL = SHARED + FE_IMG_BYTES + 3 * FE_MAX_RECS * 8 + (size_t)FE4_BATCH * FE_THREADS * 4 + (size_t)FE4_BATCH * sizeof(FoldMeta);
};

// records a tile may hold so that FE4U_UNROLL gather rounds cover it: 8 warps x 32/(cpr+1) records per round
constexpr int FE4U_UNROLL = 5;
static inline uint32_t emit4u_max_recs(uint32_t cpr) {
  const uint32_t w = cpr + 1;
  return w > 32 ? 0u : (uint32_t)FE4U_UNROLL * (FE_THREADS / 32) * (32u / w);
}

// bytes [sh, sh + 16) of the 32-byte window lo || hi
__device__ __forceinline__ uint4 window16(uint4 lo, uint4 hi, uint32_t sh) {
  uint32_t w0 = lo.x, w1 = lo.y, w2 = lo.z, w3 = lo.w, w4 = hi.x, w5 = hi.y, w6 = hi.z, w7 = hi.w;
  if (sh & 4u) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7; }
  if (sh & 8u) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; }
  const uint32_t bsh = (sh & 3u) * 8u;
  return make_uint4(__funnelshift_r(w0, w1, bsh), __funnelshift_r(w1, w2, bsh), __funnelshift_r(w2, w3, bsh), __funnelshift_r(w3, w4, bsh));
}

template <int UNROLL>
__global__ void __launch_bounds__(FE_THREADS, TEZGPU_EMIT4_MIN_CTAS) k_emit_fast4u(FastEmitParams fp) {
  constexpr int BATCH = FE4_BATCH;
  extern __shared__ __align__(16) uint8_t smem4u[];
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem4u);   // classic byte table (trailing bytes)
  uint32_t *s_adv128 = s_tab + 256;                         // * x^(32*128): second-level fold
  uint8_t *s_img = smem4u + Emit4uSmem::SHARED;
  uint64_t(*s_off)[FE_MAX_RECS] = reinterpret_cast<uint64_t(*)[FE_MAX_RECS]>(s_img + FE_IMG_BYTES);  // tiles N, N+1, N+2
  uint32_t(*s_part)[FE_THREADS] = reinterpret_cast<uint32_t(*)[FE_THREADS]>(s_img + FE_IMG_BYTES + 3 * FE_MAX_RECS * 8);
  FoldMeta *s_meta = reinterpret_cast<FoldMeta *>(s_img + FE_IMG_BYTES + 3 * FE_MAX_RECS * 8 + (size_t)BATCH * FE_THREADS * 4);

  const EmitParams &e = fp.e;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t G = gridDim.x, ntiles = fp.ntiles;
  uint32_t tile = blockIdx.x;
  if (tile >= ntiles) return;
  s_tab[tid] = e.crc->slice[0][tid];
  for (int i = tid; i < 4 * 256; i += FE_THREADS) s_adv128[i] = (&e.crc->adv128[0][0])[i];
  CrcChunkFoldT<false> cf;  // the chunk fold's linear maps as warp-resident digit tables (crc32.cuh)
  cf.init(e.crc, lane);
  const uint32_t lane_pow = cf.lane_pow;
  const uint32_t img_base = (uint32_t)__cvta_generic_to_shared(s_img);
  const uint8_t *__restrict__ kv = e.rec.kv;
  const uint8_t *kv_end = kv + e.rec.kv_bytes;
  const uint64_t *__restrict__ key_off = e.rec.key_off;
  const uint32_t rec_size = e.rec_size, hdr_len = e.fixed_hdr_len, stride = fp.stride, cpr = fp.cpr;
  const TileDesc *__restrict__ tiles = fp.tiles;
  const bool use_runs = e.rec.use_runs;
  auto source_offset = [&](uint32_t ri, uint32_t p) -> uint64_t {
    // fixed-framing runs read in place: offset = f(segment table, index) -- the record lies in one of the few runs of
    // the tile's partition p -- no per-record array
    if (use_runs) return run_record_off_p(e.rec.runs, p, ri) + e.rec.runs.hdr_len;
    return key_off ? key_off[ri] : (uint64_t)ri * stride;
  };

  // lane <-> (record slot of the warp, aligned word k of that record); leftover lanes idle
  const uint32_t wpr = cpr + 1, rpw = 32u / wpr;                 // words per record, records per warp and round
  const uint32_t rl = (uint32_t)lane / wpr, wk = (uint32_t)lane - rl * wpr;
  const bool lane_used = rl < rpw, has_piece = lane_used && wk < cpr;
  // even records first, then odd ones (emit_fast.cuh): keeps a warp on one unaligned-store path
  auto slot_record = [&](int u, uint32_t nr, uint32_t &j) -> bool {
    const uint32_t jp = ((uint32_t)u * (FE_THREADS / 32) + (uint32_t)warp) * rpw + rl;
    const uint32_t half_up = (nr + 1) >> 1;
    j = jp < half_up ? 2u * jp : 2u * (jp - half_up) + 1u;
    return lane_used && jp < nr;
  };
  // full tiles share one map: j | (j * rec_size + hdr_len + 16 * wk) << 8, valid bits in onmask
  const uint32_t full_nr = e.recs_per_tile;
  uint32_t pk[UNROLL], onmask = 0;
#pragma unroll
  for (int u = 0; u < UNROLL; u++) {
    uint32_t j;
    const bool on = slot_record(u, full_nr, j);
    pk[u] = on ? (j | (j * rec_size + hdr_len + 16u * wk) << 8) : 0u;
    onmask |= on ? 1u << u : 0u;
  }
  uint4 v[UNROLL];
  // all addresses first, then the loads back to back (emit_pipe.cuh)
  auto issue_gather = [&](uint32_t nr, const uint64_t *offs) {
    const uint8_t *src[UNROLL];
    bool on[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; u++) {
      uint32_t j;
      bool valid;
      if (nr == full_nr) { valid = (onmask >> u) & 1u; j = pk[u] & 0xFFu; }
      else valid = slot_record(u, nr, j);
      const uint8_t *first = kv + offs[valid ? j : 0u];
      const uint32_t sh = (uint32_t)((uintptr_t)first & 15u);
      src[u] = first - sh + 16u * wk;
      on[u] = valid && !(wk == cpr && sh == 0u);   // an aligned record needs no extra word
    }
    if (UNROLL == 5) asm volatile("" : "+l"(src[0]), "+l"(src[1]), "+l"(src[2]), "+l"(src[3]), "+l"(src[UNROLL - 1]));
#pragma unroll
    for (int u = 0; u < UNROLL; u++) {
      v[u] = make_uint4(0, 0, 0, 0);
      if (on[u]) {
        if (src[u] >= kv && src[u] + 16 <= kv_end) v[u] = ldg_stream_v4(src[u]);
        else v[u] = load16_clamped(src[u], kv, kv_end);   // first / last word of the buffer
      }
    }
  };
  const uint32_t hdr16 = (uint32_t)e.fixed_hdr[0] | (uint32_t)e.fixed_hdr[1] << 8;

  // ---- prologue: offsets of tiles 0 and 1 (order -> index -> offset, exposed once), record indices of tile 2,
  //      descriptors up to tile 3, gather of tile 0 in flight
  uint32_t nr0, fl0, nr1 = 0, fl1 = 0, nr2 = 0, ri2 = 0, r0_3 = 0, nr3 = 0;
  uint32_t p2 = 0, p3 = 0;   // partitions of tiles N+2 / N+3 (run-table offsets)
  uint64_t abs0, abs1 = 0;
  {
    const TileDesc t0 = tiles[tile];
    nr0 = t0.nr; fl0 = t0.flags; abs0 = t0.abs0;
    if ((uint32_t)tid < nr0) s_off[0][tid] = source_offset(e.order[t0.r0 + tid], t0.p);
    if (tile + G < ntiles) {
      const TileDesc t1 = tiles[tile + G];
      nr1 = t1.nr; fl1 = t1.flags; abs1 = t1.abs0;
      if ((uint32_t)tid < nr1) s_off[1][tid] = source_offset(e.order[t1.r0 + tid], t1.p);
    }
    if (tile + 2 * (uint64_t)G < ntiles) {
      const TileDesc t2 = tiles[tile + 2 * (uint64_t)G];
      nr2 = t2.nr;
      p2 = t2.p;
      if ((uint32_t)tid < nr2) ri2 = e.order[t2.r0 + tid];
    }
    if (tile + 3 * (uint64_t)G < ntiles) { r0_3 = tiles[tile + 3 * (uint64_t)G].r0; nr3 = tiles[tile + 3 * (uint64_t)G].nr; p3 = tiles[tile + 3 * (uint64_t)G].p; }
  }
  __syncthreads();
  issue_gather(nr0, s_off[0]);

  uint32_t n_it = 0, slot = 0;
  for (;; tile += G, n_it++) {
    const bool has1 = tile + G < ntiles, has2 = tile + 2 * (uint64_t)G < ntiles, has3 = tile + 3 * (uint64_t)G < ntiles,
               has4 = tile + 4 * (uint64_t)G < ntiles;
    const uint32_t nr = nr0;
    const bool first_tile = fl0 & 1u, last_tile = fl0 & 2u;
    const uint32_t lead = (uint32_t)(abs0 & 15u);
    const uint32_t rec0 = lead + (first_tile ? 4u : 0u);
    const uint32_t body_end = rec0 + nr * rec_size + (last_tile ? 2u : 0u);
    const uint64_t *cur_off = s_off[n_it % 3];

    // ---- prefetches consumed at the end of this iteration: offsets of tile N+2, indices of tile N+3, descriptors
    uint64_t off2 = 0, abs2n = 0;
    uint32_t ri3 = 0, r0_4 = 0, nr4 = 0, nr2n = 0, fl2n = 0, p4 = 0;
    if (has2) {
      if ((uint32_t)tid < nr2) off2 = source_offset(ri2, p2);
      const TileDesc *t2 = tiles + tile + 2 * (uint64_t)G;
      nr2n = t2->nr; fl2n = t2->flags; abs2n = t2->abs0;
    }
    if (has3 && (uint32_t)tid < nr3) ri3 = e.order[r0_3 + tid];
    if (has4) { const TileDesc *t4 = tiles + tile + 4 * (uint64_t)G; r0_4 = t4->r0; nr4 = t4->nr; p4 = t4->p; }

    // ---- this tile's words (loaded during the previous iteration) -> pieces -> image; framing
#pragma unroll
    for (int u = 0; u < UNROLL; u++) {
      uint32_t j, dst;
      bool valid;
      if (nr == full_nr) { valid = (onmask >> u) & 1u; j = pk[u] & 0xFFu; dst = pk[u] >> 8; }
      else { valid = slot_record(u, nr, j); dst = j * rec_size + hdr_len + 16u * wk; }
      const uint4 w = v[u];
      uint4 h;  // the record's next aligned word lives in the neighbour lane
      h.x = __shfl_down_sync(0xffffffffu, w.x, 1);
      h.y = __shfl_down_sync(0xffffffffu, w.y, 1);
      h.z = __shfl_down_sync(0xffffffffu, w.z, 1);
      h.w = __shfl_down_sync(0xffffffffu, w.w, 1);
      if (valid && has_piece) {
        const uint32_t sh = (uint32_t)((uintptr_t)(kv + cur_off[j]) & 15u);
        sts16_unaligned(img_base + rec0 + dst, window16(w, h, sh));
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
    __syncthreads();  // (B) image complete

    // ---- gather of the next tile goes out now; it lands while this tile is checksummed and written
    if (has1) issue_gather(nr1, s_off[(n_it + 1) % 3]);

    // ---- fused CRC + write-out (emit_fast.cuh): thread t owns the chunks at distance == T-1-t (mod T) from the end
    const uint32_t cb0 = rec0, cb1 = body_end;
    const uint32_t ca = cb0 >> 4, cz = cb1 >> 4;
    uint8_t *dstg = e.out + (abs0 - lead);
    uint32_t c = 0;
    if (cz > ca) {
      const uint32_t Cn = cz - ca;
      const uint32_t iters = (Cn + FE_THREADS - 1) / FE_THREADS;
      int32_t i = (int32_t)Cn + tid - (int32_t)(iters * FE_THREADS);
      uint32_t sa = img_base + 16u * (uint32_t)((int32_t)ca + i);
      uint8_t *gp = dstg + 16ll * ((int64_t)ca + i);
      for (uint32_t it = 0; it < iters; it++, i += FE_THREADS, sa += 16u * FE_THREADS, gp += 16 * FE_THREADS) {
        if (i + (31 - lane) < 0) continue;  // no lane of this warp owns a chunk yet (first, ragged round only)
        uint4 w = make_uint4(0, 0, 0, 0);
        if (i >= 0) {
          w = lds_v4(sa);
          if (i == 0) {
            const uint32_t b0 = 16u * ca;
            if (b0 >= lead) stg_stream_v4(gp, w);
            else for (uint32_t x = lead; x < b0 + 16u; x++) dstg[x] = s_img[x];  // ragged first chunk of the tile
            const uint32_t skip = cb0 & 15u;  // bytes before the body (segment header / previous tile) fold as zero
            if (skip) {
              uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
              for (uint32_t k = 0; k < 4; k++) {
                if (skip >= 4 * k + 4) ww[k] = 0;
                else if (skip > 4 * k) ww[k] &= 0xFFFFFFFFu << (8u * (skip - 4 * k));
              }
              w = make_uint4(ww[0], ww[1], ww[2], ww[3]);
            }
          } else {
            stg_stream_v4(gp, w);
          }
        }
        c = cf.fold(c, w, it + 1 == iters);
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
    if (has2 && (uint32_t)tid < nr2) s_off[(n_it + 2) % 3][tid] = off2;
    slot++;
    __syncthreads();  // (C) image free, partials / offsets visible

    if (slot == (uint32_t)BATCH || !has1) {
      // ---- deferred second level: warp w folds parked tile w (emit_pipe.cuh)
      if ((uint32_t)warp < slot) {
        uint32_t q = 0;
#pragma unroll
        for (int k = 0; k < FE_THREADS / 32; k++) {
          q = s_adv128[q & 0xFF] ^ s_adv128[256 + ((q >> 8) & 0xFF)] ^ s_adv128[512 + ((q >> 16) & 0xFF)] ^ s_adv128[768 + (q >> 24)];
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
    }
    if (!has1) break;
    // the prefetches are consumed HERE (emit_pipe.cuh)
    asm volatile("" : "+r"(nr2n), "+r"(fl2n), "+l"(abs2n), "+r"(ri3), "+r"(r0_4), "+r"(nr4));
    nr0 = nr1; fl0 = fl1; abs0 = abs1;
    nr1 = nr2n; fl1 = fl2n; abs1 = abs2n;
    nr2 = nr3; ri2 = ri3; p2 = p3;
    r0_3 = r0_4; nr3 = nr4; p3 = p4;
  }
}

}  // namespace tezgpu

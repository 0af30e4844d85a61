// radix_sort.cuh -- hand-written LSD radix sort for sm_90a ("onesweep": one read + one write of the data per
// 8-bit digit, chained-scan with decoupled look-back across tiles, warp-match ranking, shared-memory reorder so the
// scatter leaves the SM as contiguous per-digit runs).
//
// Shape of the 32-bit pass: 384 threads x 16 keys, two CTAs per SM (80 registers, no spill; 75,840 bytes of shared
// memory per CTA).  Swept on an H100 80GB HBM3 at a 400 W power limit with tools/bench_radix.cu, 1e8 keys, four passes,
// medians (DESIGN.md section 7): 384x16 2.98 ms, 512x12 2.98, 512x10 3.10, 384x12 3.19, 256x16 at three CTAs 3.31,
// 512x16 3.33 (spills 84 bytes at the 64-register cap), 256x16 at four CTAs 3.90 (spills); look-back depth 4 / 8 / 16
// at 384x16: 2.96 / 2.98 / 3.02 ms.  The previous kernel (separate key and index arrays, 512x16, per-item validity
// branches, volatile tile states) took 3.90 ms.
//
// Tried and reverted: a second instantiation of the tile body without the per-item validity predicates (every tile but
// the last is full) -- fewer SASS instructions in that path, but twice the code for the instruction cache of a kernel
// that is issue-bound, and the pass got slower.  The predicates are gone from the one body instead: padding items rank
// into digit 255 behind the real ones (see the load loop).
//
// Used by the sorter for the (partition|key-prefix, record-index) pairs of the hot path -- the device counterpart of
// PipelinedSorter's per-span QuickSort + SpanMerger (SORT/PipelinedSorter.java:965-1023,1116-1503) -- and by the
// tie-refinement / merge stages.  Integer work only; HBM-bound.
#pragma once
#include "common.cuh"

#ifndef TEZGPU_RADIX_THREADS32
#define TEZGPU_RADIX_THREADS32 384
#endif
#ifndef TEZGPU_RADIX_IPT32
#define TEZGPU_RADIX_IPT32 16
#endif
#ifndef TEZGPU_RADIX_MINB32
#define TEZGPU_RADIX_MINB32 (1024 / TEZGPU_RADIX_THREADS32)
#endif
#ifndef TEZGPU_RADIX_LOOKBACK
#define TEZGPU_RADIX_LOOKBACK 4
#endif
#ifndef TEZGPU_RANK_MODE
#define TEZGPU_RANK_MODE 2
#endif

namespace tezgpu {

constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;
constexpr uint32_t STATE_FLAG_LOCAL = 1u << 30;
constexpr uint32_t STATE_FLAG_INCL = 2u << 30;
constexpr uint32_t STATE_VALUE_MASK = (1u << 30) - 1;
constexpr uint32_t RADIX_MAX_N = (1u << 30) - 1;

template <typename KeyT>
__device__ __forceinline__ uint32_t radix_digit(KeyT k, int shift) {
  return (uint32_t)(k >> shift) & (RADIX - 1);
}

// ------------------------------------------------------------------------------------------------ histograms
// One pass over the keys builds the digit histograms of every radix pass at once.
template <typename KeyT, int NPASS>
__global__ void __launch_bounds__(512) k_radix_hist(const KeyT *__restrict__ keys, uint32_t n, int begin_bit,
                                                    uint32_t *__restrict__ hist /*[NPASS][RADIX]*/) {
  __shared__ uint32_t s_hist[NPASS * RADIX];
  for (int i = threadIdx.x; i < NPASS * RADIX; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    KeyT k = keys[i];
#pragma unroll
    for (int p = 0; p < NPASS; p++) atomicAdd(&s_hist[p * RADIX + radix_digit(k, begin_bit + p * RADIX_BITS)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NPASS * RADIX; i += blockDim.x) {
    uint32_t c = s_hist[i];
    if (c) atomicAdd(&hist[i], c);
  }
}

// exclusive scan of each pass's 256 bins (in place); trivial[p] = 1 when a single bin holds every key
__global__ void __launch_bounds__(RADIX) k_radix_scan_hist(uint32_t *__restrict__ hist, int npass, uint32_t n,
                                                          uint32_t *__restrict__ trivial) {
  __shared__ uint32_t s_warp[RADIX / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int p = 0; p < npass; p++) {
    uint32_t c = hist[p * RADIX + tid];
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t base = 0;
    for (int w = 0; w < warp; w++) base += s_warp[w];
    hist[p * RADIX + tid] = base + incl - c;
    uint32_t any = __syncthreads_or(c == n && n > 0);
    if (tid == 0 && trivial) trivial[p] = any ? 1u : 0u;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ onesweep pass
// Where a pass reads its (key, index) items and where it writes them.  32-bit keys travel between passes as one 8-byte
// {key, index} pair (one load, one shared-memory store and load, one store and one address per item): the first
// executed pass reads the separate key array with the iota index, middle passes read and write pairs, and the last
// executed pass writes separate key and index arrays.  64-bit keys (tie refinement) keep separate arrays.
enum RadixIO : int { IO_SEP = 0, IO_SEP_IOTA = 1, IO_PAIR = 2 };

template <typename KeyT, int THREADS, int IPT>
struct OnesweepCfg {
  static constexpr int NWARPS = THREADS / 32;
  static constexpr int TILE = THREADS * IPT;
  static constexpr size_t SMEM = (size_t)TILE * (sizeof(KeyT) + sizeof(uint32_t)) + (size_t)NWARPS * RADIX * 4 +
                                 2 * RADIX * 4 + 64 + (TEZGPU_RANK_MODE == 2 ? (size_t)NWARPS * RADIX * 4 : 0);
};

// IO_PAIR: keys_in / keys_out point to uint2 {key, index} arrays and the vals pointers are unused.
template <typename KeyT, int THREADS, int IPT, int MINB, int IN, int OUT>
__global__ void __launch_bounds__(THREADS, MINB)
    k_onesweep_pass(const KeyT *__restrict__ keys_in, KeyT *__restrict__ keys_out, const uint32_t *__restrict__ vals_in,
                    uint32_t *__restrict__ vals_out, uint32_t n, int shift, const uint32_t *__restrict__ hist_base,
                    uint32_t *tile_state, uint32_t *tile_counter) {
  using Cfg = OnesweepCfg<KeyT, THREADS, IPT>;
  constexpr int NWARPS = Cfg::NWARPS;
  constexpr int TILE = Cfg::TILE;
  constexpr bool PAIRS = sizeof(KeyT) == 4;  // the shared-memory reorder buffer holds {key, index} pairs
  static_assert(THREADS >= RADIX, "one thread per digit for the look-back");
  static_assert(PAIRS || (IN != IO_PAIR && OUT != IO_PAIR), "pairs carry 32-bit keys");
  static_assert(OUT != IO_SEP_IOTA, "iota is an input layout");

  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint2 *s_pair = reinterpret_cast<uint2 *>(smem_raw);
  KeyT *s_keys = reinterpret_cast<KeyT *>(smem_raw);
  uint32_t *s_vals = reinterpret_cast<uint32_t *>(smem_raw + (size_t)TILE * sizeof(KeyT));
  uint32_t *s_wcnt = s_vals + TILE;           // [NWARPS][RADIX]
  uint32_t *s_dstart = s_wcnt + NWARPS * RADIX;  // [RADIX] tile-local start of each digit
  uint32_t *s_goff = s_dstart + RADIX;        // [RADIX] global offset - local start
  uint32_t *s_misc = s_goff + RADIX;          // [0]=tile id, [1..8] warp scan scratch
#if TEZGPU_RANK_MODE == 2
  uint32_t *s_wmask = s_misc + 16;            // [NWARPS][RADIX] warp-private peer bit tables
#endif

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // Tile id = block index: blocks of a 1-D grid are dispatched in index order, which is what the look-back's forward
  // progress needs (same assumption as CUB's decoupled look-back scan).  A global ticket counter costs one same-address
  // atomic per tile, serialised on one address across all tiles of a pass.
#ifdef TEZGPU_TICKET_ATOMIC
  if (tid == 0) s_misc[0] = atomicAdd(tile_counter, 1u);
#else
  if (tid == 0) s_misc[0] = blockIdx.x;
#endif
  for (int i = tid; i < NWARPS * RADIX; i += THREADS) s_wcnt[i] = 0;
#if TEZGPU_RANK_MODE == 2
  for (int i = tid; i < NWARPS * RADIX; i += THREADS) s_wmask[i] = 0;
#endif
  __syncthreads();
  const uint32_t tile = s_misc[0];
  const uint32_t tile_base = tile * (uint32_t)TILE;
  const uint32_t tile_n = min((uint32_t)TILE, n - tile_base);
  const uint32_t warp_base = (uint32_t)warp * 32u * IPT;

  // ---- load the items (warp-striped => coalesced) with their index, so nothing is loaded after the rank barrier.
  // Items past the end of the last tile get the all-ones key: they rank into digit 255 behind every real item, that is
  // into the slots [tile_n, TILE) the write-out skips, so ranking and reorder need no per-item validity test.  Only the
  // last tile's own count of digit 255 includes them, and no tile looks back at the last one.
  KeyT key[IPT];
  uint32_t val[IN == IO_SEP_IOTA ? 1 : IPT];
  uint32_t rnk[IPT];
#pragma unroll
  for (int j = 0; j < IPT; j++) {
    const uint32_t li = warp_base + j * 32 + lane;
    const bool valid = li < tile_n;
    if constexpr (IN == IO_PAIR) {
      uint2 p = make_uint2(~0u, 0u);
      if (valid) p = reinterpret_cast<const uint2 *>(keys_in)[tile_base + li];
      key[j] = p.x;
      val[j] = p.y;
    } else {
      key[j] = valid ? keys_in[tile_base + li] : ~(KeyT)0;
      if constexpr (IN == IO_SEP) val[j] = valid ? vals_in[tile_base + li] : 0u;
    }
  }
  uint32_t *wc = s_wcnt + warp * RADIX;
  const uint32_t lt = lanemask_lt();
  // warp-private digit counters: the first lane of every group of equal digits claims the group's slots with one
  // shared-memory atomic (no warp barriers; the atomics of successive items pipeline)
#pragma unroll
  for (int j = 0; j < IPT; j++) {
    const uint32_t d = radix_digit(key[j], shift);
    uint32_t peers;
#if TEZGPU_RANK_MODE == 0
    peers = __match_any_sync(0xffffffffu, d);
#elif TEZGPU_RANK_MODE == 2
    // peer mask through a warp-private shared-memory bit table: every lane ORs its bit into the entry of its digit,
    // reads the entry back, then removes its own bit again (atomics, so the next row may already be setting bits)
    {
      uint32_t *wm = s_wmask + warp * RADIX;
      atomicOr(&wm[d], 1u << lane);
      __syncwarp();
      peers = wm[d];
      __syncwarp();
      atomicAnd(&wm[d], ~(1u << lane));
    }
#else
    // MATCH.ANY runs on the (slow) ADU pipe; eight ballots + logic ops build the same peer mask on the ALU path
    peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < RADIX_BITS; b++) {
      const bool bit = (d >> b) & 1u;
      const uint32_t bm = __ballot_sync(0xffffffffu, bit);
      peers &= bit ? bm : ~bm;
    }
#endif
    uint32_t pre = 0;
    if ((peers & lt) == 0) pre = atomicAdd(&wc[d], (uint32_t)__popc(peers));
    pre = __shfl_sync(0xffffffffu, pre, __ffs(peers) - 1);
    rnk[j] = pre + __popc(peers & lt);
  }
  __syncthreads();

  // ---- per-digit: exclusive scan over warps, tile count, publish, block scan over digits
  uint32_t count = 0;
  if (tid < RADIX) {
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < NWARPS; w++) {
      uint32_t c = s_wcnt[w * RADIX + tid];
      s_wcnt[w * RADIX + tid] = run;
      run += c;
    }
    count = run;
    // publish the tile aggregate as early as possible (tile 0 publishes its inclusive prefix directly)
    st_relaxed_gpu_u32(&tile_state[(size_t)tile * RADIX + tid], (tile == 0 ? STATE_FLAG_INCL : STATE_FLAG_LOCAL) | count);
    uint32_t incl = count;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_misc[1 + warp] = incl;
    s_dstart[tid] = incl - count;  // completed after the barrier below
  }
  __syncthreads();
  if (tid < RADIX) {
    uint32_t base = 0;
    for (int w = 0; w < warp; w++) base += s_misc[1 + w];
    s_dstart[tid] += base;
  }
  __syncthreads();

  // ---- reorder through shared memory: slot = digit start + warp offset + rank in warp
#pragma unroll
  for (int j = 0; j < IPT; j++) {
    const uint32_t d = radix_digit(key[j], shift);
    const uint32_t slot = s_dstart[d] + wc[d] + rnk[j];
    uint32_t v;
    if constexpr (IN == IO_SEP_IOTA) v = tile_base + warp_base + j * 32 + lane;
    else v = val[j];
    if constexpr (PAIRS) {
      s_pair[slot] = make_uint2((uint32_t)key[j], v);
    } else {
      s_keys[slot] = key[j];
      s_vals[slot] = v;
    }
  }

  // ---- decoupled look-back (thread d resolves digit d) overlapped with the shared-memory scatter above
  if (tid < RADIX) {
    uint32_t excl = 0;
    if (tile > 0) {
      // look back over the predecessors' published counts, LOOKBACK states per round trip (independent loads)
      constexpr int LOOKBACK = TEZGPU_RADIX_LOOKBACK;
      int64_t t = (int64_t)tile - 1;
      bool done = false;
      while (!done) {
        uint32_t st[LOOKBACK];
#ifdef TEZGPU_RADIX_DEBUG
        if (tid == 0) atomicAdd(tile_counter + 7, 1u);
#endif
#pragma unroll
        for (int b = 0; b < LOOKBACK; b++)
          st[b] = (t - b >= 0) ? ld_relaxed_gpu_u32(&tile_state[(size_t)(t - b) * RADIX + tid]) : STATE_FLAG_INCL;
#pragma unroll
        for (int b = 0; b < LOOKBACK; b++) {
          if (done) break;
          uint32_t flag = st[b] & ~STATE_VALUE_MASK;
          if (flag == 0) break;  // not published yet: retry from here
          excl += st[b] & STATE_VALUE_MASK;
          t--;
          if (flag == STATE_FLAG_INCL) done = true;
        }
      }
      st_relaxed_gpu_u32(&tile_state[(size_t)tile * RADIX + tid], STATE_FLAG_INCL | (excl + count));
    }
    s_goff[tid] = hist_base[tid] + excl - s_dstart[tid];
  }
  __syncthreads();

  // ---- coalesced write-out: consecutive slots of one digit are consecutive in global memory
#pragma unroll
  for (int k = 0; k < IPT; k++) {
    const uint32_t slot = (uint32_t)tid + k * THREADS;
    if (slot < tile_n) {
      KeyT kk;
      uint32_t v;
      if constexpr (PAIRS) {
        const uint2 p = s_pair[slot];
        kk = p.x;
        v = p.y;
      } else {
        kk = s_keys[slot];
        v = s_vals[slot];
      }
      const uint32_t dest = s_goff[radix_digit(kk, shift)] + slot;
      if constexpr (OUT == IO_PAIR) {
        reinterpret_cast<uint2 *>(keys_out)[dest] = make_uint2((uint32_t)kk, v);
      } else {
        keys_out[dest] = kk;
        vals_out[dest] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host driver
struct RadixWorkspace {
  uint32_t *hist = nullptr;        // [8][RADIX]
  uint32_t *trivial = nullptr;     // [8]
  uint32_t *tile_state = nullptr;  // [npass][ntiles][RADIX]
  uint32_t *tile_counter = nullptr;  // [8]
  size_t tile_state_words = 0;
  int device = 0;                  // the current device
};

// MINB: CTAs per SM that __launch_bounds__ asks for, which caps the registers at 64K / (MINB * THREADS).
template <typename KeyT>
struct RadixTuning {
  static constexpr int THREADS = sizeof(KeyT) == 4 ? TEZGPU_RADIX_THREADS32 : 512;
  static constexpr int IPT = sizeof(KeyT) == 4 ? TEZGPU_RADIX_IPT32 : 10;
  static constexpr int MINB = sizeof(KeyT) == 4 ? TEZGPU_RADIX_MINB32 : 2;
};

template <typename KeyT>
static inline uint32_t radix_num_tiles(uint32_t n) {
  using T = RadixTuning<KeyT>;
  return (uint32_t)div_up(n, (uint64_t)T::THREADS * T::IPT);
}
template <typename KeyT>
static inline size_t radix_tile_state_words(uint32_t n, int npass) {
  return (size_t)radix_num_tiles<KeyT>(n) * RADIX * (size_t)npass;
}

// launches pass p of a sort that starts at begin_bit; its digit offsets, look-back state and tile counter come from ws
template <typename KeyT, int IN, int OUT>
static void radix_launch_pass(cudaStream_t st, const RadixWorkspace &ws, uint32_t ntiles, int begin_bit, int p, const KeyT *kin,
                              KeyT *kout, const uint32_t *vin, uint32_t *vout, uint32_t n) {
  using T = RadixTuning<KeyT>;
  using Cfg = OnesweepCfg<KeyT, T::THREADS, T::IPT>;
  constexpr auto kern = k_onesweep_pass<KeyT, T::THREADS, T::IPT, T::MINB, IN, OUT>;
  set_smem_limit<kern>(ws.device, Cfg::SMEM);
  kern<<<ntiles, T::THREADS, Cfg::SMEM, st>>>(kin, kout, vin, vout, n, begin_bit + p * RADIX_BITS, ws.hist + p * RADIX,
                                               ws.tile_state + (size_t)p * ntiles * RADIX, ws.tile_counter + p);
  TG_CUDA(cudaGetLastError());
}

// clears the look-back state of npass passes over n keys; returns the tiles per pass
template <typename KeyT>
static uint32_t radix_prepare(cudaStream_t st, const RadixWorkspace &ws, uint32_t n, int npass) {
  const uint32_t ntiles = radix_num_tiles<KeyT>(n);
  TG_CHECK((size_t)ntiles * RADIX * (size_t)npass <= ws.tile_state_words, -1, "radix workspace too small");
  TG_CUDA(cudaMemsetAsync(ws.tile_state, 0, (size_t)ntiles * RADIX * (size_t)npass * 4, st));
  TG_CUDA(cudaMemsetAsync(ws.tile_counter, 0, 8 * 4, st));
  return ntiles;
}

// Both drivers launch the passes for bits [begin_bit, begin_bit + 8*npass).  `hist` must already hold the
// exclusive-scanned per-pass digit offsets (k_radix_hist / a fused producer + k_radix_scan_hist).  pass_mask bit p =
// run pass p.  They return the number of passes executed.

// 32-bit keys, with the record index as payload.  blk_a and blk_b are blocks of 2n words; the keys come in at
// blk_a[0, n) and the index is the iota.  Between passes the items are {key, index} pairs (uint2) filling a block.  The
// last executed pass writes the sorted keys to words [0, n) and the indices to words [n, 2n) of its output block, which
// is blk_b when the number of executed passes is odd and blk_a when it is even.  At least one pass must run.
static int radix_sort_pairs(cudaStream_t st, const RadixWorkspace &ws, uint32_t *blk_a, uint32_t *blk_b, uint32_t n,
                            int begin_bit, int npass, uint32_t pass_mask, int *launches) {
  const int total = __builtin_popcount(pass_mask & ((1u << npass) - 1));
  TG_CHECK(total >= 1, -1, "radix sort without a pass");
  const uint32_t ntiles = radix_prepare<uint32_t>(st, ws, n, npass);
  int done = 0;
  for (int p = 0; p < npass; p++) {
    if (!((pass_mask >> p) & 1u)) continue;
    uint32_t *in = (done & 1) ? blk_b : blk_a, *out = (done & 1) ? blk_a : blk_b;
    const bool first = done == 0, last = done + 1 == total;
    if (first && last)
      radix_launch_pass<uint32_t, IO_SEP_IOTA, IO_SEP>(st, ws, ntiles, begin_bit, p, in, out, nullptr, out + n, n);
    else if (first)
      radix_launch_pass<uint32_t, IO_SEP_IOTA, IO_PAIR>(st, ws, ntiles, begin_bit, p, in, out, nullptr, nullptr, n);
    else if (last)
      radix_launch_pass<uint32_t, IO_PAIR, IO_SEP>(st, ws, ntiles, begin_bit, p, in, out, nullptr, out + n, n);
    else
      radix_launch_pass<uint32_t, IO_PAIR, IO_PAIR>(st, ws, ntiles, begin_bit, p, in, out, nullptr, nullptr, n);
    if (launches) (*launches)++;
    done++;
  }
  return done;
}

// 64-bit keys (tie refinement) with a u32 payload, in separate arrays; the result is in (keys_b, vals_b) when the
// number of executed passes is odd.
template <typename KeyT>
static int radix_sort_passes(cudaStream_t st, const RadixWorkspace &ws, KeyT *keys_a, KeyT *keys_b, uint32_t *vals_a,
                             uint32_t *vals_b, uint32_t n, int begin_bit, int npass, uint32_t pass_mask, int *launches) {
  static_assert(sizeof(KeyT) == 8, "32-bit keys are sorted as pairs (radix_sort_pairs)");
  const uint32_t ntiles = radix_prepare<KeyT>(st, ws, n, npass);
  int done = 0;
  for (int p = 0; p < npass; p++) {
    if (!((pass_mask >> p) & 1u)) continue;
    KeyT *kin = (done & 1) ? keys_b : keys_a, *kout = (done & 1) ? keys_a : keys_b;
    uint32_t *vin = (done & 1) ? vals_b : vals_a, *vout = (done & 1) ? vals_a : vals_b;
    radix_launch_pass<KeyT, IO_SEP, IO_SEP>(st, ws, ntiles, begin_bit, p, kin, kout, vin, vout, n);
    if (launches) (*launches)++;
    done++;
  }
  return done;
}

}  // namespace tezgpu

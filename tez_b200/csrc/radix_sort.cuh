// radix_sort.cuh -- hand-written LSD radix sort for sm_90a ("onesweep": one read + one write of the data per
// 8-bit digit, chained-scan with decoupled look-back across tiles, warp-match ranking, shared-memory reorder so the
// scatter leaves the SM as contiguous per-digit runs).
//
// Tried and reverted: a second instantiation of the tile body without the per-item validity predicates (every tile but
// the last is full) -- fewer SASS instructions in that path, but twice the code for the instruction cache of a kernel
// that is issue-bound, and the pass got slower.
//
// Used by the sorter for the (partition|key-prefix, record-index) pairs of the hot path -- the device counterpart of
// PipelinedSorter's per-span QuickSort + SpanMerger (SORT/PipelinedSorter.java:965-1023,1116-1503) -- and by the
// tie-refinement / merge stages.  Integer work only; HBM-bound.
#pragma once
#include "common.cuh"

#ifndef TEZGPU_RADIX_THREADS32
#define TEZGPU_RADIX_THREADS32 512
#endif
#ifndef TEZGPU_RADIX_IPT32
#define TEZGPU_RADIX_IPT32 16
#endif
#ifndef TEZGPU_RADIX_LOOKBACK
#define TEZGPU_RADIX_LOOKBACK 8
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
template <typename KeyT, int THREADS, int IPT>
struct OnesweepCfg {
  static constexpr int NWARPS = THREADS / 32;
  static constexpr int TILE = THREADS * IPT;
  static constexpr size_t SMEM = (size_t)TILE * (sizeof(KeyT) + sizeof(uint32_t)) + (size_t)NWARPS * RADIX * 4 +
                                 2 * RADIX * 4 + 64 + (TEZGPU_RANK_MODE == 2 ? (size_t)NWARPS * RADIX * 4 : 0);
};

template <typename KeyT, int THREADS, int IPT, bool VALS_IOTA>
__global__ void __launch_bounds__(THREADS, 1024 / THREADS)
    k_onesweep_pass(const KeyT *__restrict__ keys_in, KeyT *__restrict__ keys_out, const uint32_t *__restrict__ vals_in,
                    uint32_t *__restrict__ vals_out, uint32_t n, int shift, const uint32_t *__restrict__ hist_base,
                    uint32_t *tile_state, uint32_t *tile_counter) {
  using Cfg = OnesweepCfg<KeyT, THREADS, IPT>;
  constexpr int NWARPS = Cfg::NWARPS;
  constexpr int TILE = Cfg::TILE;
  static_assert(THREADS >= RADIX, "one thread per digit for the look-back");

  extern __shared__ __align__(16) uint8_t smem_raw[];
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

  // ---- load keys (warp-striped => coalesced) and rank them inside the warp
  KeyT key[IPT];
  uint32_t rnk[IPT];
#pragma unroll
  for (int j = 0; j < IPT; j++) {
    uint32_t li = warp_base + j * 32 + lane;
    key[j] = (li < tile_n) ? keys_in[tile_base + li] : (KeyT)0;
  }
  uint32_t *wc = s_wcnt + warp * RADIX;
  const uint32_t lt = lanemask_lt();
  // warp-private digit counters: the first lane of every group of equal digits claims the group's slots with one
  // shared-memory atomic (no warp barriers; the atomics of successive items pipeline)
#pragma unroll
  for (int j = 0; j < IPT; j++) {
    uint32_t li = warp_base + j * 32 + lane;
    bool valid = li < tile_n;
    uint32_t d = radix_digit(key[j], shift);
    uint32_t peers;
#if TEZGPU_RANK_MODE == 0
    peers = __match_any_sync(0xffffffffu, valid ? d : (uint32_t)RADIX);
#elif TEZGPU_RANK_MODE == 2
    // peer mask through a warp-private shared-memory bit table: every lane ORs its bit into the entry of its digit,
    // reads the entry back, then removes its own bit again (atomics, so the next row may already be setting bits)
    {
      uint32_t *wm = s_wmask + warp * RADIX;
      if (valid) atomicOr(&wm[d], 1u << lane);
      __syncwarp();
      peers = valid ? wm[d] : 0u;
      __syncwarp();
      if (valid) atomicAnd(&wm[d], ~(1u << lane));
    }
#else
    // MATCH.ANY runs on the (slow) ADU pipe; eight ballots + logic ops build the same peer mask on the ALU path
    peers = __ballot_sync(0xffffffffu, valid);
    if (!valid) peers = ~peers;
#pragma unroll
    for (int b = 0; b < RADIX_BITS; b++) {
      const bool bit = (d >> b) & 1u;
      const uint32_t bm = __ballot_sync(0xffffffffu, bit);
      peers &= bit ? bm : ~bm;
    }
#endif
    uint32_t pre = 0;
    if (valid && (peers & lt) == 0) pre = atomicAdd(&wc[d], (uint32_t)__popc(peers));
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
    st_volatile_u32(&tile_state[(size_t)tile * RADIX + tid], (tile == 0 ? STATE_FLAG_INCL : STATE_FLAG_LOCAL) | count);
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
    uint32_t li = warp_base + j * 32 + lane;
    if (li < tile_n) {
      uint32_t d = radix_digit(key[j], shift);
      uint32_t slot = s_dstart[d] + wc[d] + rnk[j];
      s_keys[slot] = key[j];
      uint32_t v;
      if (VALS_IOTA) v = tile_base + li;
      else v = vals_in[tile_base + li];
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
          st[b] = (t - b >= 0) ? ld_volatile_u32(&tile_state[(size_t)(t - b) * RADIX + tid]) : STATE_FLAG_INCL;
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
      st_volatile_u32(&tile_state[(size_t)tile * RADIX + tid], STATE_FLAG_INCL | (excl + count));
    }
    s_goff[tid] = hist_base[tid] + excl - s_dstart[tid];
  }
  __syncthreads();

  // ---- coalesced write-out: consecutive slots of one digit are consecutive in global memory
#pragma unroll
  for (int k = 0; k < IPT; k++) {
    uint32_t slot = (uint32_t)tid + k * THREADS;
    if (slot < tile_n) {
      KeyT kk = s_keys[slot];
      uint32_t dest = s_goff[radix_digit(kk, shift)] + slot;
      keys_out[dest] = kk;
      vals_out[dest] = s_vals[slot];
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
};

template <typename KeyT>
struct RadixTuning {
  static constexpr int THREADS = sizeof(KeyT) == 4 ? TEZGPU_RADIX_THREADS32 : 512;
  static constexpr int IPT = sizeof(KeyT) == 4 ? TEZGPU_RADIX_IPT32 : 10;
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

// Launches the passes for bits [begin_bit, begin_bit + 8*npass).  `hist` must already hold the exclusive-scanned
// per-pass digit offsets (k_radix_hist / a fused producer + k_radix_scan_hist).  pass_mask bit p = run pass p.
// Returns the number of passes executed; result is in (keys_b, vals_b) when that number is odd.
template <typename KeyT>
static int radix_sort_passes(cudaStream_t st, const RadixWorkspace &ws, KeyT *keys_a, KeyT *keys_b, uint32_t *vals_a,
                             uint32_t *vals_b, uint32_t n, int begin_bit, int npass, uint32_t pass_mask,
                             bool first_vals_iota, int *launches) {
  using T = RadixTuning<KeyT>;
  using Cfg = OnesweepCfg<KeyT, T::THREADS, T::IPT>;
  static bool attr_set = false;
  if (!attr_set) {
    TG_CUDA(cudaFuncSetAttribute(k_onesweep_pass<KeyT, T::THREADS, T::IPT, false>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM));
    TG_CUDA(cudaFuncSetAttribute(k_onesweep_pass<KeyT, T::THREADS, T::IPT, true>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM));
    attr_set = true;
  }
  uint32_t ntiles = radix_num_tiles<KeyT>(n);
  TG_CHECK((size_t)ntiles * RADIX * (size_t)npass <= ws.tile_state_words, -1, "radix workspace too small");
  TG_CUDA(cudaMemsetAsync(ws.tile_state, 0, (size_t)ntiles * RADIX * (size_t)npass * 4, st));
  TG_CUDA(cudaMemsetAsync(ws.tile_counter, 0, 8 * 4, st));
  int done = 0;
  bool iota = first_vals_iota;
  for (int p = 0; p < npass; p++) {
    if (!((pass_mask >> p) & 1u)) continue;
    KeyT *kin = (done & 1) ? keys_b : keys_a, *kout = (done & 1) ? keys_a : keys_b;
    uint32_t *vin = (done & 1) ? vals_b : vals_a, *vout = (done & 1) ? vals_a : vals_b;
    uint32_t *state = ws.tile_state + (size_t)p * ntiles * RADIX;
    if (iota)
      k_onesweep_pass<KeyT, T::THREADS, T::IPT, true><<<ntiles, T::THREADS, Cfg::SMEM, st>>>(
          kin, kout, vin, vout, n, begin_bit + p * RADIX_BITS, ws.hist + p * RADIX, state, ws.tile_counter + p);
    else
      k_onesweep_pass<KeyT, T::THREADS, T::IPT, false><<<ntiles, T::THREADS, Cfg::SMEM, st>>>(
          kin, kout, vin, vout, n, begin_bit + p * RADIX_BITS, ws.hist + p * RADIX, state, ws.tile_counter + p);
    TG_CUDA(cudaGetLastError());
    if (launches) (*launches)++;
    iota = false;
    done++;
  }
  return done;
}

}  // namespace tezgpu

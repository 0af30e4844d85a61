// sample.cuh -- InputSampler.RandomSampler and InputSampler.writePartitionFile on the device (SURVEY A.2): a seeded
// sample of device-resident keys (tezgpu_sample_keys) and the split points TotalOrderPartitioner takes, picked from the
// sorted sample by writePartitionFile's rule (tezgpu_select_split_points).
//
// Record i of a sample call has the global number gid = gid_base + i and the hash h = splitmix64(seed ^ gid).  It is a
// candidate when h < ceil(freq * 2^64) (every record when freq = 1); of more than max_samples candidates the
// max_samples smallest (h, gid) are kept.  The sample is a function of (seed, gid) alone, so the records can be split
// between calls (ranks) in any way and the union, capped again, is the same.
#pragma once
#include <stdint.h>

#include "record_table.cuh"
#include "scan.cuh"

namespace tezgpu {

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// Which records a pass keeps.  Candidates: all, or h < thr.  Kept: the candidates with h < cut, and of those with
// h == cut the first need_eq in record order (= gid order).  Before the cap cut = thr and need_eq = 0 (or, with every
// record a candidate, cut = need_eq = 2^64 - 1), so the kept records are the candidates.
struct SampleCut {
  uint64_t seed, gid_base, mask;   // mask: ~0, or fewer hash bits (tezgpu_debug_set_sample_hash_mask: forced ties)
  uint64_t thr, cut, need_eq;
  int all;
};
__device__ __forceinline__ uint64_t sample_hash(const SampleCut &c, uint64_t i) { return splitmix64(c.seed ^ (c.gid_base + i)) & c.mask; }
// (h < cut) << 32 | (h == cut) of one candidate; 0 for a record that is not one.  The per-tile sums of these words carry
// no bits between the halves while a call holds fewer than 2^32 records.
__device__ __forceinline__ uint64_t sample_class(const SampleCut &c, uint64_t h) {
  if (!c.all && h >= c.thr) return 0;
  return h < c.cut ? (1ull << 32) : (h == c.cut ? 1ull : 0ull);
}

// Candidate pass, the only kernel that reads every record: with CHECK, record_bounds_check on every record (the lowest
// bad one, with its reason, into first_bad as k_record_table reports it); the class words of the tile summed into
// blk[tile].  SCAN_TILE records per CTA, read strided so that the loads coalesce.
template <bool CHECK>
__global__ void __launch_bounds__(SCAN_THREADS)
    k_sample_count(const uint64_t *__restrict__ key_off, const uint64_t *__restrict__ val_off, const uint32_t *__restrict__ val_len,
                   uint64_t kv_bytes, uint32_t n, SampleCut c, uint64_t *__restrict__ blk, unsigned long long *__restrict__ first_bad) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE;
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    const uint32_t i = base + k * SCAN_THREADS + threadIdx.x;
    if (i >= n) break;
    if constexpr (CHECK) {
      const uint32_t why = record_bounds_check(key_off[i], val_off[i], val_len[i], kv_bytes);
      if (why) atomicMin(first_bad, ((unsigned long long)i << RECTAB_REASON_BITS) | why);
    }
    s += sample_class(c, sample_hash(c, i));
  }
  uint64_t tot;
  block_exclusive_scan_u64(s, s_warp, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
}

// Histogram of hash digit (h >> shift) & 255 over the candidates whose digits above it equal prefix's (the cap's radix
// select, one pass per digit, most significant first).  Hashes are recomputed, no record is read.
__global__ void __launch_bounds__(256) k_sample_digit_hist(uint32_t n, SampleCut c, uint64_t prefix, int shift,
                                                           uint32_t *__restrict__ hist) {
  __shared__ uint32_t s_hist[256];
  s_hist[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t hi_mask = shift >= 56 ? 0ull : ~0ull << (shift + 8);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t h = sample_hash(c, i);
    if ((c.all || h < c.thr) && (h & hi_mask) == (prefix & hi_mask)) atomicAdd(&s_hist[(h >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (s_hist[threadIdx.x]) atomicAdd(&hist[threadIdx.x], s_hist[threadIdx.x]);
}

// Compaction of the kept records, in record order: blk holds the exclusive scan of k_sample_count's tile sums (same cut).
// Each thread owns SCAN_IPT consecutive records; kept record -> slot (h < cut before it) + min(h == cut before it, need_eq).
__global__ void __launch_bounds__(SCAN_THREADS)
    k_sample_compact(uint32_t n, SampleCut c, const uint64_t *__restrict__ blk, uint32_t *__restrict__ sel_idx,
                     uint64_t *__restrict__ sel_h) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_IPT;
  uint64_t cls[SCAN_IPT], hs[SCAN_IPT], s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    hs[k] = sample_hash(c, base + k);
    cls[k] = base + k < n ? sample_class(c, hs[k]) : 0;
    s += cls[k];
  }
  const uint64_t ex = block_exclusive_scan_u64(s, s_warp, nullptr) + blk[blockIdx.x];
  uint64_t lt = ex >> 32, eq = ex & 0xFFFFFFFFull;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    if (cls[k] >> 32) {
      const uint64_t slot = lt + (eq < c.need_eq ? eq : c.need_eq);
      sel_idx[slot] = base + k;
      sel_h[slot] = hs[k];
      lt++;
    } else if (cls[k]) {
      if (eq < c.need_eq) {
        sel_idx[lt + eq] = base + k;
        sel_h[lt + eq] = hs[k];
      }
      eq++;
    }
  }
}

// The sampled records' key lengths (for the scan of their offsets) and global numbers
__global__ void k_sample_key_meta(const uint64_t *__restrict__ key_off, const uint64_t *__restrict__ val_off,
                                  const uint32_t *__restrict__ sel_idx, uint32_t m, uint64_t gid_base, uint32_t *__restrict__ len,
                                  uint64_t *__restrict__ gid) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint32_t i = sel_idx[j];
  len[j] = (uint32_t)(val_off[i] - key_off[i]);
  gid[j] = gid_base + i;
}

// The sampled keys packed back to back at out_off (the scan of their lengths): one warp per key
__global__ void k_sample_gather(const uint8_t *__restrict__ kv, const uint64_t *__restrict__ key_off, const uint32_t *__restrict__ sel_idx,
                                const uint32_t *__restrict__ len, const uint64_t *__restrict__ out_off, uint32_t m,
                                uint8_t *__restrict__ out) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= m) return;
  const uint8_t *src = kv + key_off[sel_idx[w]];
  uint8_t *dst = out + out_off[w];
  const uint32_t l = len[w];
  for (uint32_t b = lane; b < l; b += 32) dst[b] = src[b];
}

// ---- split selection over the sorted sample
// run heads of the sorted sample as 0/1 words: position r starts a run of equal keys unless same[r]
__global__ void k_split_heads(const uint8_t *__restrict__ same, uint32_t n, uint32_t *__restrict__ head) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) head[r] = (r == 0 || !same[r]) ? 1u : 0u;
}

// Math.round(float) (Java 7 on): the nearest integer, halves toward +inf, with no rounding in between (x - floor(x) is
// exact in float, where x + 0.5f is not)
__host__ __device__ __forceinline__ int64_t java_round_float(float x) {
  const float f = floorf(x);
  return (int64_t)f + ((x - f) >= 0.5f ? 1 : 0);
}

// InputSampler.writePartitionFile's loop over the sorted sample of n keys:
//   float stepSize = n / (float) P;  int last = -1;
//   for i in 1 .. P-1: k = Math.round(stepSize * i); while (last >= k && cmp(samples[last], samples[k]) == 0) ++k;
//                      emit samples[k]; last = k;
// Two keys compare equal iff they lie in one run of equal keys: run_ex[r + 1] (inclusive count of run heads) names the
// run of position r.  As k <= last and the keys are sorted, the while loop ends at last + 1 when k shares last's run and
// at k otherwise, so every step is O(1).  Each step depends on the one before, so one thread walks them; P - 1 steps of
// a few loads are not a hot path and are not parallelised.  chosen[i - 1] = k, rec[i - 1] = order[k]; a k past the end
// of the sample (Java: ArrayIndexOutOfBoundsException) stops the walk with *bad = (i << 32) | k (k saturated).
__global__ void k_split_pick(const uint64_t *__restrict__ run_ex, const uint32_t *__restrict__ order, uint32_t n, uint32_t P,
                             uint64_t *__restrict__ chosen, uint32_t *__restrict__ rec, unsigned long long *__restrict__ bad) {
  if (blockIdx.x || threadIdx.x) return;
  const float step = __fdiv_rn(__uint2float_rn(n), __uint2float_rn(P));
  int64_t last = -1;
  for (uint32_t i = 1; i < P; i++) {
    int64_t k = java_round_float(__fmul_rn(step, __uint2float_rn(i)));
    if (last >= k && run_ex[last + 1] == run_ex[k + 1]) k = last + 1;
    if (k >= (int64_t)n) {
      *bad = ((unsigned long long)i << 32) | (unsigned long long)(k < 0xFFFFFFFFll ? k : 0xFFFFFFFFll);
      return;
    }
    chosen[i - 1] = (uint64_t)k;
    rec[i - 1] = order[k];
    last = k;
  }
}

}  // namespace tezgpu

// combine.cuh -- device combiner between the sort and the emit: MRCombiner running IntSumReducer / LongSumReducer
// (tez-mapreduce combine/MRCombiner.java; SORT/PipelinedSorter.java:601-609,815-820, SORT/dflt/DefaultSorter.java:915-945).
//
// Semantics (DESIGN.md §6):
//   - a group is a maximal run of adjacent records in sorted order, inside one partition, whose keys compare equal under
//     the job's comparator (ReduceContextImpl / RL/common/ValuesIterator.java:178-197).  sort_phase leaves exactly that
//     in same[]: same[r] = 1 iff the key at r equals the key at r-1 under the RawComparator (k_tie_fix, the large-group
//     head comparison, the refinement rounds and the merger's run-table mode all set it only from a full comparison of
//     two keys whose sort words are equal, and the sort word holds the partition).  For the device comparators and
//     canonically serialised keys comparator equality is byte equality of the raw key.
//   - one record per group: the key bytes of the group's first record, then the big-endian sum of the values.
//     SUM_INT: 4-byte IntWritable values, Java int arithmetic (wraps mod 2^32); SUM_LONG: 8-byte LongWritable values
//     (wraps mod 2^64).  The sums do not depend on the order inside a group, so the combined output does not depend on
//     the tie order among equal keys.
//   - a value of any other width fails the flush / write with TEZGPU_E_INVALID naming the record.
//   - keys are unique per partition afterwards: the emit never writes a repeat, whatever the RLE decision was.
//   - a group of one record re-encodes to exactly its input bytes.
#pragma once
#include "sorter_kernels.cuh"

namespace tezgpu {

constexpr int CMB_THREADS = 256;
constexpr int CMB_ROWS = 8;   // a warp folds CMB_ROWS rows of 32 consecutive sorted positions

static inline uint32_t combine_width(int combiner) {
  return combiner == TEZGPU_COMBINE_SUM_INT ? 4u : (combiner == TEZGPU_COMBINE_SUM_LONG ? 8u : 0u);
}

// the emit's value-address rule (k_emit: val_off only for parsed variable-width records)
__device__ __forceinline__ uint64_t combine_val_off(const Records &r, uint32_t i, uint64_t koff, uint32_t klen) {
  return (r.val_off && !r.fixed) ? r.val_off[i] : koff + klen;
}

// nothing to combine (no two adjacent keys are equal): only the value widths are checked; *bad = lowest bad record
__global__ void __launch_bounds__(256) k_combine_check_width(Records r, uint32_t width, uint32_t *__restrict__ bad) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += stride) {
    uint64_t koff;
    uint32_t klen, vlen;
    record_lookup(r, i, koff, klen, vlen);
    if (vlen != width) atomicMin(bad, i);
  }
}

// group heads as 0/1 words for the scan: head[r] = r == 0 || !same[r]
__global__ void __launch_bounds__(256) k_combine_heads(const uint8_t *__restrict__ same, uint32_t n, uint32_t *__restrict__ head) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) head[r] = (r == 0 || !same[r]) ? 1u : 0u;
}

// Segmented sum.  gid = exclusive scan of the heads (n + 1 entries): record r belongs to group gid[r + 1] - 1 and heads
// it when gid[r + 1] != gid[r].  Each warp walks CMB_ROWS rows of 32 consecutive positions; inside a row a segmented
// shuffle reduction folds every group fragment into its first lane, and the fragment that reaches the end of the row is
// carried into the next row.  So a group costs at most one atomic per warp (CMB_ROWS * 32 records): one hot key over
// millions of records does not serialise on its sum.  Heads also record their position and compact the sort word.
template <int W>
__global__ void __launch_bounds__(CMB_THREADS)
    k_combine_sum(Records rec, const uint32_t *__restrict__ order, const uint32_t *__restrict__ K, const uint64_t *__restrict__ gid,
                  uint32_t n, unsigned long long *__restrict__ sums, uint32_t *__restrict__ head_pos, uint32_t *__restrict__ K_out,
                  uint32_t *__restrict__ bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t base = warp * 32 * CMB_ROWS;
  const uint64_t NONE = ~0ull;
  uint64_t carry_g = NONE;
  unsigned long long carry = 0;
  for (int k = 0; k < CMB_ROWS; k++) {
    const uint64_t r = base + (uint64_t)k * 32 + lane;
    const bool valid = r < n;
    uint64_t g = NONE;
    unsigned long long v = 0;
    if (valid) {
      const uint64_t g0 = gid[r], g1 = gid[r + 1];
      g = g1 - 1;
      if (g1 != g0) {
        head_pos[g] = (uint32_t)r;
        K_out[g] = K[r];
      }
      const uint32_t i = order[r];
      uint64_t koff;
      uint32_t klen, vlen;
      record_lookup(rec, i, koff, klen, vlen);
      if (vlen != (uint32_t)W) {
        atomicMin(bad, i);
      } else {
        const uint8_t *p = rec.kv + combine_val_off(rec, i, koff, klen);
#pragma unroll
        for (int b = 0; b < W; b++) v = (v << 8) | p[b];
      }
    }
    // the carried fragment continues in lane 0 or is finished
    if (lane == 0 && carry_g != NONE) {
      if (g == carry_g) v += carry;
      else atomicAdd(&sums[carry_g], carry);
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long ov = __shfl_down_sync(0xffffffffu, v, o);
      const uint64_t og = __shfl_down_sync(0xffffffffu, g, o);
      if (lane + o < 32 && og == g) v += ov;
    }
    const uint64_t gp = __shfl_up_sync(0xffffffffu, g, 1);
    const uint64_t g31 = __shfl_sync(0xffffffffu, g, 31);
    const bool first = valid && (lane == 0 || gp != g);
    const bool carried = g31 != NONE && k + 1 < CMB_ROWS;   // the row's last fragment goes on into the next row
    if (first && !(carried && g == g31)) atomicAdd(&sums[g], v);
    const uint32_t tail = __ballot_sync(0xffffffffu, first && g == g31);
    carry_g = NONE;
    if (carried && tail) {
      carry = __shfl_sync(0xffffffffu, v, __ffs(tail) - 1);
      carry_g = g31;
    }
  }
}

// var mode: bytes of every combined record (key + sum), scanned into its offset
__global__ void __launch_bounds__(256)
    k_combine_sizes(Records rec, const uint32_t *__restrict__ order, const uint32_t *__restrict__ head_pos, uint32_t m,
                    uint32_t width, uint32_t *__restrict__ sizes) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m) return;
  uint64_t koff;
  uint32_t klen, vlen;
  record_lookup(rec, order[head_pos[g]], koff, klen, vlen);
  sizes[g] = klen + width;
}

// Compaction: LANES threads per combined record copy the head's key bytes and write the big-endian sum behind them.
// Fixed width: record g at g * (klen + W); variable width: at off[g], with its key offset / lengths.  order becomes the
// identity over the combined records.
template <int W, int LANES>
__global__ void __launch_bounds__(256)
    k_combine_write(Records rec, const uint32_t *__restrict__ order, const uint32_t *__restrict__ head_pos,
                    const unsigned long long *__restrict__ sums, uint32_t m, const uint64_t *__restrict__ off, uint8_t *__restrict__ out,
                    uint32_t *__restrict__ order_out, uint64_t *__restrict__ koff_out, uint32_t *__restrict__ klen_out,
                    uint32_t *__restrict__ vlen_out) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t g = (uint32_t)(t / LANES), lane = (uint32_t)(t % LANES);
  if (g >= m) return;
  uint64_t koff;
  uint32_t klen, vlen;
  record_lookup(rec, order[head_pos[g]], koff, klen, vlen);
  const uint64_t dst = off ? off[g] : (uint64_t)g * (klen + W);
  const uint8_t *src = rec.kv + koff;
  for (uint32_t b = lane; b < klen; b += LANES) out[dst + b] = src[b];
  if (lane == 0) {
    const unsigned long long s = sums[g];
#pragma unroll
    for (int b = 0; b < W; b++) out[dst + klen + b] = (uint8_t)(s >> (8 * (W - 1 - b)));
    order_out[g] = g;
    if (off) {
      koff_out[g] = dst;
      klen_out[g] = klen;
      vlen_out[g] = W;
    }
  }
}

}  // namespace tezgpu

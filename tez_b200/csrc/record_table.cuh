// record_table.cuh -- the record table of a sort whose variable-length records are already in device memory
// (tezgpu_sorter_sort_device): the caller's 64-bit (key_off, val_off, val_len) triples checked and turned into the
// pipeline's (key_off, key_len, val_len) arrays, before any key byte is read.
#pragma once
#include <stdint.h>

#include <string>

namespace tezgpu {

// why a record is refused: the low RECTAB_REASON_BITS of RecordTableVerdict::first_bad, above them the record index
constexpr int RECTAB_REASON_BITS = 3;
constexpr uint32_t RECTAB_KEY_AFTER_VALUE = 1, RECTAB_KEY_TOO_LONG = 2, RECTAB_PAST_END = 3, RECTAB_PARTITION = 4;
constexpr int RECTAB_THREADS = 256;

static inline std::string record_table_reason(uint32_t r) {
  switch (r) {
    case RECTAB_KEY_AFTER_VALUE: return "key offset after value offset";
    case RECTAB_KEY_TOO_LONG: return "key of 4 GiB or more";
    case RECTAB_PAST_END: return "value ends past kv_bytes";
    default: return "Illegal partition (outside [0, numPartitions))";
  }
}

// Why a record (key at ko, value at vo, vl value bytes) does not lie in a buffer of kv_bytes, 0 when it does: the
// record checks every device-resident record table goes through (k_record_table, the sampler's k_sample_count)
__host__ __device__ __forceinline__ uint32_t record_bounds_check(uint64_t ko, uint64_t vo, uint32_t vl, uint64_t kv_bytes) {
  if (vo < ko) return RECTAB_KEY_AFTER_VALUE;
  if (vo - ko > 0xFFFFFFFFull) return RECTAB_KEY_TOO_LONG;
  if (vo > kv_bytes || vl > kv_bytes - vo) return RECTAB_PAST_END;
  return 0;
}

// One pass over the caller's arrays (64-bit sibling of k_rebase_offsets).  A record is valid when key_off <= val_off,
// val_off - key_off < 2^32, val_off + val_len <= kv_bytes and, with partition ids, 0 <= partition < P.  first_bad
// (initialised to ~0) receives min((i << RECTAB_REASON_BITS) | reason) over the invalid records i, so the host names the
// lowest one; payload the sum of key + value bytes (one atomic per CTA).  The pipeline then reads the table written
// here, never the caller's arrays again: what it sorts is what was checked.
__global__ void __launch_bounds__(RECTAB_THREADS)
    k_record_table(const uint64_t *__restrict__ key_off, const uint64_t *__restrict__ val_off, const uint32_t *__restrict__ val_len,
                   const int32_t *__restrict__ partition, uint32_t n, uint64_t kv_bytes, int32_t P, uint64_t *__restrict__ koff,
                   uint32_t *__restrict__ klen, uint32_t *__restrict__ vlen, unsigned long long *__restrict__ first_bad,
                   unsigned long long *__restrict__ payload) {
  __shared__ unsigned long long s_sum[RECTAB_THREADS / 32];
  unsigned long long sum = 0;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t ko = key_off[i], vo = val_off[i];
    const uint32_t vl = val_len[i];
    uint32_t why = record_bounds_check(ko, vo, vl, kv_bytes);
    if (!why && partition) {
      const int32_t p = partition[i];
      if (p < 0 || p >= P) why = RECTAB_PARTITION;
    }
    if (why) {
      atomicMin(first_bad, ((unsigned long long)i << RECTAB_REASON_BITS) | why);
      continue;
    }
    koff[i] = ko;
    klen[i] = (uint32_t)(vo - ko);
    vlen[i] = vl;
    sum += (vo - ko) + vl;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < RECTAB_THREADS / 32; w++) t += s_sum[w];
    if (t) atomicAdd(payload, t);
  }
}

}  // namespace tezgpu

// scan.cuh -- small device-wide scan / compaction building blocks (reduce-then-scan, 2048 elements per block).
#pragma once
#include "device_util.h"

namespace tezgpu {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_IPT = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_IPT;

// block-wide exclusive scan of one u64 per thread (SCAN_THREADS threads); returns exclusive prefix, *total = block sum
__device__ __forceinline__ uint64_t block_exclusive_scan_u64(uint64_t v, uint64_t *s_warp /*[SCAN_THREADS/32]*/,
                                                             uint64_t *total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint64_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < SCAN_THREADS / 32; w++) {
    uint64_t x = s_warp[w];
    if (w < warp) base += x;
    tot += x;
  }
  __syncthreads();
  if (total) *total = tot;
  return base + incl - v;
}

// single-block exclusive scan of u64 block sums; total written to blk[nblk]
__global__ void __launch_bounds__(1024) k_scan_block_sums(uint64_t *blk, uint32_t nblk) {
  __shared__ uint64_t s_warp[32];
  __shared__ uint64_t s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nblk; base += 1024) {
    uint32_t i = base + threadIdx.x;
    uint64_t v = i < nblk ? blk[i] : 0, incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint64_t wbase = 0, tot = 0;
    for (int w = 0; w < 32; w++) {
      uint64_t x = s_warp[w];
      if (w < warp) wbase += x;
      tot += x;
    }
    uint64_t carry = s_carry;
    if (i < nblk) blk[i] = carry + wbase + incl - v;
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) blk[nblk] = s_carry;
}

// ---- u32 sizes -> u64 exclusive offsets (out has n+1 entries)
__global__ void __launch_bounds__(SCAN_THREADS) k_sum_u32_blocks(const uint32_t *__restrict__ in, uint32_t n,
                                                                 uint64_t *__restrict__ blk) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  uint32_t base = blockIdx.x * SCAN_TILE;
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t i = base + k * SCAN_THREADS + threadIdx.x;
    if (i < n) s += in[i];
  }
  uint64_t tot;
  block_exclusive_scan_u64(s, s_warp, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_u32_apply(const uint32_t *__restrict__ in, uint32_t n,
                                                                 const uint64_t *__restrict__ blk,
                                                                 uint64_t *__restrict__ out) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_IPT;  // blocked arrangement: thread owns 8 consecutive
  uint32_t v[SCAN_IPT];
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t i = base + k;
    v[k] = i < n ? in[i] : 0;
    s += v[k];
  }
  uint64_t ex = block_exclusive_scan_u64(s, s_warp, nullptr) + blk[blockIdx.x];
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t i = base + k;
    if (i < n) out[i] = ex;
    ex += v[k];
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == SCAN_THREADS - 1) out[n] = blk[gridDim.x];
}

// u32 sizes -> u64 exclusive offsets: out[i] = in[0] + ... + in[i-1] for i < n, out[n] = the total (n > 0).  blk holds the
// block sums.  Returns the launches.
inline int scan_u32_exclusive(cudaStream_t st, DeviceBuffer &blk, const uint32_t *in, uint32_t n, uint64_t *out) {
  const uint32_t nblk = (uint32_t)div_up(n, SCAN_TILE);
  blk.ensure(((size_t)nblk + 2) * 8);
  k_sum_u32_blocks<<<nblk, SCAN_THREADS, 0, st>>>(in, n, blk.as<uint64_t>());
  k_scan_block_sums<<<1, 1024, 0, st>>>(blk.as<uint64_t>(), nblk);
  k_scan_u32_apply<<<nblk, SCAN_THREADS, 0, st>>>(in, n, blk.as<uint64_t>(), out);
  return 3;
}

}  // namespace tezgpu

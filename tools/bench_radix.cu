// tools/bench_radix.cu -- micro-benchmark of the onesweep radix pass (tuning aid; not part of the product path).
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -DTEZGPU_RADIX_THREADS32=.. -DTEZGPU_RADIX_IPT32=.. tools/bench_radix.cu
//
// bench_radix [n] [pass_mask] [key_bits]
//   n          keys (default 1e8, the config-2 flush)
//   pass_mask  hex, which of the four 8-bit passes run (default f; 8 = the unordered writer's single top pass at P=64)
//   key_bits   distinct bits per key (default 32; fewer means more equal keys, which exercises stability)
// Like the sorter, the first executed pass takes the iota index.  The timed sort is then checked over the whole array:
// keys sorted on the bits the executed passes cover, the index array a permutation that maps back to the input keys,
// and equal keys in index order (stability).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../tez_b200/csrc/radix_sort.cuh"

using namespace tezgpu;

__global__ void k_fill(uint32_t *k, uint32_t n, int key_bits) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    uint64_t x = i * 0x9E3779B97F4A7C15ull + 12345;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    uint32_t v = (uint32_t)(x ^ (x >> 31));
    k[i] = key_bits >= 32 ? v : v >> (32 - key_bits);
  }
}

int main(int argc, char **argv) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const uint32_t n = argc > 1 ? (uint32_t)atoll(argv[1]) : 100000000u;
  const uint32_t mask = argc > 2 ? (uint32_t)strtoul(argv[2], nullptr, 16) & 0xFu : 0xFu;
  const int key_bits = argc > 3 ? atoi(argv[3]) : 32;
  if (n == 0 || n > RADIX_MAX_N || mask == 0 || key_bits < 1 || key_bits > 32) {
    fprintf(stderr, "usage: bench_radix [n <= 2^30-1] [pass_mask 1..f] [key_bits 1..32]\n");
    return 2;
  }
  uint32_t *blk_a, *blk_b, *small;
  cudaMalloc(&blk_a, n * 8ull); cudaMalloc(&blk_b, n * 8ull);
  cudaMalloc(&small, 16384);
  cudaStream_t st;
  cudaStreamCreate(&st);
  RadixWorkspace ws;
  ws.hist = small; ws.trivial = small + 2048; ws.tile_counter = small + 2056;
  ws.tile_state_words = radix_tile_state_words<uint32_t>(n, 4);
  cudaMalloc(&ws.tile_state, ws.tile_state_words * 4);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int runs = 7;
  std::vector<float> ms(runs);
  int done = 0;
  for (int it = 0; it < runs; it++) {
    k_fill<<<(n + 255) / 256, 256, 0, st>>>(blk_a, n, key_bits);
    cudaMemsetAsync(small, 0, 16384, st);
    k_radix_hist<uint32_t, 4><<<sms * 8, 512, 0, st>>>(blk_a, n, 0, ws.hist);
    k_radix_scan_hist<<<1, RADIX, 0, st>>>(ws.hist, 4, n, ws.trivial);
    cudaEventRecord(e0, st);
    int launches = 0;
    done = radix_sort_pairs(st, ws, blk_a, blk_b, n, 0, 4, mask, &launches);
    cudaEventRecord(e1, st);
    cudaStreamSynchronize(st);
    cudaEventElapsedTime(&ms[it], e0, e1);
  }
  // check the last sort over the whole array against the input keys
  std::vector<uint32_t> in(n), K(n), order(n);
  const uint32_t *res = (done & 1) ? blk_b : blk_a;
  uint32_t *scratch = (done & 1) ? blk_a : blk_b;  // the input keys again, in the block that does not hold the result
  k_fill<<<(n + 255) / 256, 256, 0, st>>>(scratch, n, key_bits);
  cudaMemcpy(in.data(), scratch, n * 4ull, cudaMemcpyDeviceToHost);
  cudaMemcpy(K.data(), res, n * 4ull, cudaMemcpyDeviceToHost);
  cudaMemcpy(order.data(), res + n, n * 4ull, cudaMemcpyDeviceToHost);
  uint32_t bits = 0;
  for (int p = 0; p < 4; p++)
    if ((mask >> p) & 1u) bits |= 0xFFu << (8 * p);
  std::vector<uint8_t> seen(n, 0);
  uint64_t bad_perm = 0, bad_key = 0, bad_sort = 0, bad_stable = 0, ties = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t o = order[i];
    if (o >= n || seen[o]) { bad_perm++; continue; }
    seen[o] = 1;
    if (K[i] != in[o]) bad_key++;
    if (i) {
      const uint32_t a = K[i - 1] & bits, b = K[i] & bits;
      if (a > b) bad_sort++;
      if (a == b) {
        ties++;
        if (order[i - 1] > o) bad_stable++;
      }
    }
  }
  const bool ok = !bad_perm && !bad_key && !bad_sort && !bad_stable;
#ifdef TEZGPU_RADIX_DEBUG
  uint32_t rounds = 0;
  cudaMemcpy(&rounds, ws.tile_counter + 7, 4, cudaMemcpyDeviceToHost);
  printf("look-back round trips of digit 0: %u (tiles/pass %u) => %.1f per tile and pass\n", rounds, radix_num_tiles<uint32_t>(n),
         rounds / (double)done / radix_num_tiles<uint32_t>(n));
#endif
  cudaError_t err = cudaGetLastError();
  std::vector<float> sorted_ms(ms.begin() + 1, ms.end());  // run 0 loads the modules
  std::sort(sorted_ms.begin(), sorted_ms.end());
  const float med = sorted_ms[sorted_ms.size() / 2];
  // bytes: the first pass reads 4 B keys (iota index), writes 8 B; later passes read and write 8 B
  const double bytes = (double)n * (12.0 + 16.0 * (done - 1));
  printf("threads=%d ipt=%d minb=%d lookback=%d n=%u mask=%x key_bits=%d passes=%d median=%.3f ms min=%.3f max=%.3f "
         "(%.3f ms/pass, %.2f TB/s) checked=%s ties=%llu bad(perm,key,sort,stable)=%llu,%llu,%llu,%llu err=%s\n",
         TEZGPU_RADIX_THREADS32, TEZGPU_RADIX_IPT32, TEZGPU_RADIX_MINB32, TEZGPU_RADIX_LOOKBACK, n, mask, key_bits, done, med,
         sorted_ms.front(), sorted_ms.back(), med / done, bytes / (med * 1e-3) / 1e12, ok ? "ok" : "FAILED",
         (unsigned long long)ties, (unsigned long long)bad_perm, (unsigned long long)bad_key, (unsigned long long)bad_sort,
         (unsigned long long)bad_stable, cudaGetErrorString(err));
  return ok && err == cudaSuccess ? 0 : 1;
}

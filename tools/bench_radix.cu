// tools/bench_radix.cu -- micro-benchmark of the onesweep radix pass (tuning aid; not part of the product path).
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -DTEZGPU_RADIX_THREADS32=.. -DTEZGPU_RADIX_IPT32=.. tools/bench_radix.cu
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../tez_b200/csrc/radix_sort.cuh"

using namespace tezgpu;

__global__ void k_fill(uint32_t *k, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    uint64_t x = i * 0x9E3779B97F4A7C15ull + 12345;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    k[i] = (uint32_t)(x ^ (x >> 31));
  }
}

int main(int argc, char **argv) {
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  uint32_t n = argc > 1 ? (uint32_t)atoll(argv[1]) : 100000000u;
  uint32_t *ka, *kb, *va, *vb, *small;
  cudaMalloc(&ka, n * 4ull); cudaMalloc(&kb, n * 4ull); cudaMalloc(&va, n * 4ull); cudaMalloc(&vb, n * 4ull);
  cudaMalloc(&small, 16384);
  cudaStream_t st;
  cudaStreamCreate(&st);
  RadixWorkspace ws;
  ws.hist = small; ws.trivial = small + 2048; ws.tile_counter = small + 2056;
  ws.tile_state_words = radix_tile_state_words<uint32_t>(n, 4);
  cudaMalloc(&ws.tile_state, ws.tile_state_words * 4);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9;
  for (int it = 0; it < 6; it++) {
    k_fill<<<(n + 255) / 256, 256, 0, st>>>(ka, n);
    cudaMemsetAsync(small, 0, 16384, st);
    k_radix_hist<uint32_t, 4><<<sms * 8, 512, 0, st>>>(ka, n, 0, ws.hist);
    k_radix_scan_hist<<<1, RADIX, 0, st>>>(ws.hist, 4, n, ws.trivial);
    cudaEventRecord(e0, st);
    int launches = 0;
    radix_sort_passes<uint32_t>(st, ws, ka, kb, va, vb, n, 0, 4, 0xF, true, &launches);
    cudaEventRecord(e1, st);
    cudaStreamSynchronize(st);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    best = std::min(best, ms);
  }
  // verify sortedness on a sample
  std::vector<uint32_t> h(1 << 20);
  cudaMemcpy(h.data(), ka + (n > (1u << 20) ? n / 2 : 0), std::min<size_t>(n, 1 << 20) * 4, cudaMemcpyDeviceToHost);
  bool ok = true;
  for (size_t i = 1; i < std::min<size_t>(n, 1 << 20); i++) ok &= h[i - 1] <= h[i];
#ifdef TEZGPU_RADIX_DEBUG
  uint32_t rounds = 0;
  cudaMemcpy(&rounds, ws.tile_counter + 7, 4, cudaMemcpyDeviceToHost);
  printf("look-back round trips of digit 0 over 4 passes: %u (tiles/pass %u) => %.1f per tile\n", rounds, radix_num_tiles<uint32_t>(n),
         rounds / 4.0 / radix_num_tiles<uint32_t>(n));
#endif
  cudaError_t err = cudaGetLastError();
  printf("threads=%d ipt=%d n=%u 4 passes best=%.3f ms (%.3f ms/pass) sorted=%d err=%s\n", TEZGPU_RADIX_THREADS32,
         TEZGPU_RADIX_IPT32, n, best, best / 4, (int)ok, cudaGetErrorString(err));
  return 0;
}

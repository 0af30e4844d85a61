// common.cuh -- shared device/host helpers for libtezgpu (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <stdexcept>
#include <string>

namespace tezgpu {

struct Error : public std::runtime_error {
  int code;
  Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

#define TG_CUDA(expr)                                                                                   \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess) {                                                                            \
      throw ::tezgpu::Error(_e == cudaErrorMemoryAllocation ? -3 : -2,                                  \
                            std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" + \
                                std::to_string(__LINE__) + ")");                                        \
    }                                                                                                   \
  } while (0)

#define TG_CHECK(cond, code, msg)                      \
  do {                                                 \
    if (!(cond)) throw ::tezgpu::Error((code), (msg)); \
  } while (0)

static inline uint64_t div_up(uint64_t a, uint64_t b) { return (a + b - 1) / b; }
static inline uint64_t align_up(uint64_t a, uint64_t b) { return div_up(a, b) * b; }

// 4-byte big-endian words at any alignment (IFile checksum trailers, LZ4 block headers)
__host__ __device__ __forceinline__ uint32_t load_be32(const uint8_t *p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
__host__ __device__ __forceinline__ void store_be32(uint8_t *p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

// Lets kernel Kern take `bytes` of dynamic shared memory on `device`, the current device.  The limit is an attribute
// per device: it is set once per kernel and device (racing first calls set the same value); later calls load one flag.
template <auto Kern>
inline void set_smem_limit(int device, size_t bytes) {
  static std::atomic<bool> done[64];
  if ((unsigned)device < 64 && done[device].load(std::memory_order_acquire)) return;
  TG_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  if ((unsigned)device < 64) done[device].store(true, std::memory_order_release);
}

// comparator ids (include/tezgpu.h)
enum { CMP_BYTES = 0, CMP_TEXT = 1, CMP_BYTESWRITABLE = 2, CMP_INT = 3, CMP_LONG = 4 };

// -------------------------------------------------------------------------------------------- device helpers
// (the key helpers are __host__ __device__: tezgpu_debug_sort_words_emulate runs the sort word build on the host)
// hadoop WritableUtils.decodeVIntSize on the first byte
__host__ __device__ __forceinline__ int vint_decode_size(uint8_t first) {
  int v = (int)(int8_t)first;
  if (v >= -112) return 1;
  if (v < -120) return -119 - v;
  return -111 - v;
}
// WritableUtils.getVIntSize for non-negative lengths
__host__ __device__ __forceinline__ int vint_size_u32(uint32_t v) {
  if (v <= 127) return 1;
  if (v < (1u << 8)) return 2;
  if (v < (1u << 16)) return 3;
  if (v < (1u << 24)) return 4;
  return 5;
}
// byte `b` (0-based) of the vint encoding of non-negative v
__host__ __device__ __forceinline__ uint8_t vint_byte_u32(uint32_t v, int b) {
  int sz = vint_size_u32(v);
  if (sz == 1) return (uint8_t)v;
  if (b == 0) return (uint8_t)(-112 - (sz - 1));  // -113..-116
  int shift = (sz - 1 - b) * 8;
  return (uint8_t)(v >> shift);
}

// bytes of key content to skip before comparing / hashing (Text: vint prefix, BytesWritable: 4-byte length)
__host__ __device__ __forceinline__ uint32_t key_content_skip(int cmp, const uint8_t *key, uint32_t klen) {
  if (klen == 0) return 0;
  if (cmp == CMP_TEXT) {
    uint32_t s = (uint32_t)vint_decode_size(key[0]);
    return s < klen ? s : klen;
  }
  if (cmp == CMP_BYTESWRITABLE) return klen < 4 ? klen : 4;
  return 0;
}

// normalised content byte i: unsigned lexicographic order over these bytes == comparator order
// (IntWritable / LongWritable: two's complement big-endian => flip the sign bit of byte 0)
__host__ __device__ __forceinline__ uint32_t norm_byte(int cmp, const uint8_t *content, uint32_t i) {
  uint32_t b = content[i];
  if (i == 0 && (cmp == CMP_INT || cmp == CMP_LONG)) b ^= 0x80u;
  return b;
}

// WritableComparator.hashBytes
__host__ __device__ __forceinline__ int32_t hash_bytes_dev(const uint8_t *p, uint32_t n) {
  uint32_t h = 1;
  for (uint32_t i = 0; i < n; i++) h = 31u * h + (uint32_t)(int32_t)(int8_t)p[i];
  return (int32_t)h;
}

// key.hashCode() for the supported key classes
__host__ __device__ __forceinline__ int32_t key_hash_dev(int cmp, const uint8_t *key, uint32_t klen) {
  if (cmp == CMP_INT && klen >= 4)
    return (int32_t)(((uint32_t)key[0] << 24) | ((uint32_t)key[1] << 16) | ((uint32_t)key[2] << 8) | key[3]);
  if (cmp == CMP_LONG && klen >= 8) {
    uint64_t v = 0;
    for (int i = 0; i < 8; i++) v = (v << 8) | key[i];
    return (int32_t)(uint32_t)(v ^ (v >> 32));
  }
  uint32_t s = key_content_skip(cmp, key, klen);
  return hash_bytes_dev(key + s, klen - s);
}

__device__ __forceinline__ uint32_t lanemask_lt() {
  uint32_t m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// Coherent at GPU scope (L2), without the system-scope cost of `volatile`: for flags that only other CTAs of the same
// device read, where the flag and its value share one word.
__device__ __forceinline__ uint32_t ld_relaxed_gpu_u32(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u32(uint32_t *p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ uint64_t ld_volatile_u64(const uint64_t *p) {
  uint64_t v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_volatile_u64(uint64_t *p, uint64_t v) {
  asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// -------------------------------------------------------------------------------------------- compressed segments
// The codec writers' segment table (codec.cuh): per output partition, where its uncompressed segment lies in the
// emit's image and where its chunks are.  Every codec's chunk kernel finds its chunk's segment through it.
struct ZSeg {
  uint64_t body_off;   // image offset of the first body byte (after TIF\x00)
  uint64_t body_len;   // body bytes (records + EOF marker)
  uint32_t chunk0, nchunks;
  uint64_t rank;       // segments before this partition
  uint64_t zstart;     // out: file offset of the compressed segment
  uint64_t zlen;       // out: its length (0: no segment)
  uint32_t open;       // the body continues after these chunks (a bounded merge's open partition): zlib ends the
                       // last chunk with the sync-flush block instead of marking it final
  uint32_t pad;
};

// chunk c -> its partition: the last p with chunk0 <= c (partitions without a segment own no chunk)
__device__ __forceinline__ uint32_t z_chunk_part(const ZSeg *__restrict__ segs, uint32_t P, uint32_t c) {
  uint32_t lo = 0, hi = P;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (segs[mid].chunk0 <= c) lo = mid; else hi = mid;
  }
  return lo;
}

}  // namespace tezgpu

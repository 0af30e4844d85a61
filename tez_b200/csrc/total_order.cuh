// total_order.cuh -- Hadoop's TotalOrderPartitioner on the device: the partition of a key is the number of split points
// that are <= the key in the search order (BinarySearchNode: Arrays.binarySearch + 1, then pos < 0 ? -pos : pos; the
// byte trie's leaves run the same search over a sub-range).  k_stage calls split_partition per record instead of the
// hash; the host emulation tezgpu_debug_total_order_emulate runs the same code.
#pragma once
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"

namespace tezgpu {

// Split points prepared for the search (device or host memory).  Each split's content -- the key bytes after the
// comparator's length prefix, byte 0 normalised (norm_byte) -- lies in `blob`; `prefix` holds its first 8 content bytes
// big-endian, zero padded, so that unsigned order of prefix words is order of the content's first 8 bytes.
struct SplitTable {
  const uint64_t *prefix;  // [n]
  const uint32_t *len;     // [n] content bytes
  const uint64_t *off;     // [n] offset of the content in blob
  const uint8_t *blob;
  uint32_t n;              // P - 1 split points; 0 = no table (the partition comes from the hash or the caller)
  int order;               // CMP_* of the search
};

// k_stage copies the prefix words to shared memory when there are at most this many: 4096 x 8 B = 32 KB next to the
// stage's 4 KB of histograms keeps the kernel under the 48 KB a launch may take without an opt-in, and at P = 1024
// (8 KB) six CTAs of 256 threads still fit an SM.  Larger tables are searched in global memory (L2 / L1 resident).
constexpr uint32_t SPLIT_SMEM_MAX = 4096;

// 8 normalised content bytes of a key, big-endian, zero after its end
__host__ __device__ __forceinline__ uint64_t split_prefix_word(int order, const uint8_t *content, uint32_t clen) {
  uint64_t w = 0;
#pragma unroll
  for (uint32_t b = 0; b < 8; b++) w = (w << 8) | (b < clen ? norm_byte(order, content, b) : 0u);
  return w;
}

// Upper bound of the key among the splits: the number of splits <= key.  kp is the key's prefix word, `pw` the table's
// prefix words (shared or global memory).  Equal prefix words compare the content from byte 8 on and then the length,
// so a key and a split that differ only in trailing zero bytes ("ab" / "ab\0") stay distinct.
__host__ __device__ __forceinline__ uint32_t split_upper_bound(const SplitTable &t, const uint64_t *pw, uint64_t kp,
                                                               const uint8_t *content, uint32_t clen) {
  uint32_t lo = 0, hi = t.n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const uint64_t sp = pw[mid];
    bool split_le_key;
    if (sp != kp) {
      split_le_key = sp < kp;
    } else {
      const uint32_t sl = t.len[mid];
      const uint8_t *s = t.blob + t.off[mid];
      const uint32_t m = clen < sl ? clen : sl;
      int c = 0;
      for (uint32_t i = 8; i < m && c == 0; i++) c = (int)content[i] - (int)s[i];   // bytes past 0 need no normalising
      if (c == 0) c = clen < sl ? -1 : (clen == sl ? 0 : 1);
      split_le_key = c >= 0;
    }
    if (split_le_key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// partition of one serialized key
__host__ __device__ __forceinline__ int32_t split_partition(const SplitTable &t, const uint64_t *pw, const uint8_t *key,
                                                            uint32_t klen) {
  const uint32_t skip = key_content_skip(t.order, key, klen);
  const uint8_t *content = key + skip;
  const uint32_t clen = klen - skip;
  return (int32_t)split_upper_bound(t, pw, split_prefix_word(t.order, content, clen), content, clen);
}

// full comparator order of two serialized keys (the split point check)
static inline int compare_serialized(int cmp, const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb) {
  const uint32_t sa = key_content_skip(cmp, a, la), sb = key_content_skip(cmp, b, lb);
  a += sa; b += sb; la -= sa; lb -= sb;
  const uint32_t m = la < lb ? la : lb;
  for (uint32_t i = 0; i < m; i++) {
    const uint32_t x = norm_byte(cmp, a, i), y = norm_byte(cmp, b, i);
    if (x != y) return x < y ? -1 : 1;
  }
  return la < lb ? -1 : (la == lb ? 0 : 1);
}

// The table in host memory, built from the serialized split keys after TotalOrderPartitioner.setConf's checks: P - 1
// keys ("Wrong number of partitions in keyset"), strictly increasing under the sort comparator ("Split points are out
// of order").  Throws TEZGPU_E_INVALID with Hadoop's messages, and for a search order that is neither the sort
// comparator nor a natural order the comparator allows.
struct HostSplitTable {
  std::vector<uint64_t> prefix, off;
  std::vector<uint32_t> len;
  std::vector<uint8_t> blob;
  int order = 0;
  SplitTable view() const {
    return SplitTable{prefix.data(), len.data(), off.data(), blob.data(), (uint32_t)prefix.size(), order};
  }
};
// the search order of split points: the handle's own order, or the natural (content) order of Text / BytesWritable keys
// sorted by raw bytes
static inline void check_split_order(int sort_cmp, int order) {
  TG_CHECK(order == sort_cmp || (sort_cmp == CMP_BYTES && (order == CMP_TEXT || order == CMP_BYTESWRITABLE)), TEZGPU_E_INVALID,
           "search order " + std::to_string(order) + " does not fit comparator " + std::to_string(sort_cmp) +
               " (the comparator itself, or TEXT / BYTESWRITABLE under BYTES)");
}
static inline void build_split_table(int sort_cmp, int order, int P, const uint8_t *keys, const uint64_t *key_off,
                                     const uint32_t *key_len, uint32_t n, HostSplitTable &t) {
  check_split_order(sort_cmp, order);
  TG_CHECK((int64_t)n == (int64_t)P - 1, TEZGPU_E_INVALID, "Wrong number of partitions in keyset");
  TG_CHECK((keys && key_off && key_len) || n == 0, TEZGPU_E_INVALID, "null argument");
  for (uint32_t i = 1; i < n; i++)
    TG_CHECK(compare_serialized(sort_cmp, keys + key_off[i - 1], key_len[i - 1], keys + key_off[i], key_len[i]) < 0,
             TEZGPU_E_INVALID, "Split points are out of order");
  t.order = order;
  t.prefix.resize(n);
  t.off.resize(n);
  t.len.resize(n);
  t.blob.clear();
  for (uint32_t i = 0; i < n; i++) {
    const uint8_t *key = keys + key_off[i];
    const uint32_t skip = key_content_skip(order, key, key_len[i]);
    const uint32_t clen = key_len[i] - skip;
    t.prefix[i] = split_prefix_word(order, key + skip, clen);
    t.off[i] = t.blob.size();
    t.len[i] = clen;
    for (uint32_t b = 0; b < clen; b++) t.blob.push_back((uint8_t)norm_byte(order, key + skip, b));
  }
}

}  // namespace tezgpu

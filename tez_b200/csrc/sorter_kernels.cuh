// sorter_kernels.cuh -- map-output side of the hot path on sm_90a:
//   stage (key -> partition, sort word)  ->  onesweep radix sort  ->  tie refinement on key suffixes
//   ->  partition bounds / layout  ->  gather + IFile emit (vint framing, RLE markers, per-segment CRC32).
// Device counterpart of PipelinedSorter.collect/sort/spill + IFile.Writer
// (SORT/PipelinedSorter.java:398-466,558-647,965-1023; SORT/IFile.java:262-634).  Integer/byte work, HBM-bound.
#pragma once
#include "common.cuh"
#include "crc32.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "total_order.cuh"

namespace tezgpu {

// Fixed-framing IFile runs read in place (reduce side of the device shuffle): record i of the merge lives in segment
// s = last segment with rec_base[s] <= i, at body offset (i - rec_base[s]) * rec_size -- pure arithmetic, so no
// per-record metadata arrays exist at all (they were 32 B per record of extra HBM traffic each way).
struct RunTable {
  const uint64_t *seg_off;    // [nseg] offset in kv of the first record (its framing bytes) of every segment
  const uint32_t *rec_base;   // [nseg + 1] first merge record index of every segment
  const uint32_t *seg_part;   // [nseg] output partition of every segment
  const uint32_t *part_seg0;  // [P + 1] segments are listed partition-major: partition p owns [part_seg0[p], part_seg0[p+1])
  uint32_t nseg;
  uint32_t rec_size;          // framing + key + value bytes
  uint32_t hdr_len;           // framing bytes: vint(klen) vint(vlen)
  uint64_t hdr_bytes[2];      // the framing bytes (up to 10), little-endian packed: bytes 0-7, 8-9 (checked by k_stage)
};

// last segment s with rec_base[s] <= i (rec_base is small and hot in L1)
__device__ __forceinline__ uint32_t run_of(const RunTable &t, uint32_t i) {
  uint32_t lo = 0, hi = t.nseg;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(t.rec_base + mid) <= i) lo = mid; else hi = mid;
  }
  return lo;
}
// the same when the record's partition is known: its segment is one of the few runs of that partition
__device__ __forceinline__ uint32_t run_of_in_partition(const RunTable &t, uint32_t p, uint32_t i) {
  uint32_t seg = __ldg(t.part_seg0 + p);
  const uint32_t end = __ldg(t.part_seg0 + p + 1);
  while (seg + 1 < end && i >= __ldg(t.rec_base + seg + 1)) seg++;
  return seg;
}
// byte offset in kv of record i's framing bytes
__device__ __forceinline__ uint64_t run_record_off(const RunTable &t, uint32_t i, uint32_t &seg) {
  seg = run_of(t, i);
  return __ldg(t.seg_off + seg) + (uint64_t)(i - __ldg(t.rec_base + seg)) * t.rec_size;
}
__device__ __forceinline__ uint64_t run_record_off_p(const RunTable &t, uint32_t p, uint32_t i) {
  const uint32_t seg = run_of_in_partition(t, p, i);
  return __ldg(t.seg_off + seg) + (uint64_t)(i - __ldg(t.rec_base + seg)) * t.rec_size;
}

// Alphabet-compressed sort word for variable-length keys.  The 32-bit sort word normally holds the first
// (32 - pbits) / 8 normalised content bytes; keys over a small alphabet (text: 26 letters) waste most of those bits,
// everything ties on the prefix and the whole order is left to the key-suffix refinement.  Instead, a pass over the keys
// records WHICH byte values occur at each of the first SYM_MAX_POS content positions; position q then needs only
// ceil(log2(#values + 1)) bits (rank 0 = "key ended before q", so a proper prefix still sorts first), and as many
// positions as fit are packed, most significant first.  Order-preserving by construction (ranks follow byte order per
// position), exact for any input; lower-case words get 6 characters into 30 bits instead of 3-4.  A position where all
// 256 byte values occur needs ranks 1..256, i.e. 9 bits and a rank wider than a byte.
constexpr int SYM_MAX_POS = 16;
struct SymTable {
  uint16_t rank[SYM_MAX_POS][256];  // 1 + number of occurring byte values below b (0 for values that never occur)
  uint8_t shift[SYM_MAX_POS];       // left shift of position q's rank inside the (32 - pbits)-bit field
  uint32_t npos;                    // positions packed; equal sort words <=> equal first npos content bytes (or both ended)
};

// Host: the table from k_symbols' occurrence sets (sets[q * 8 + (b >> 5)] bit (b & 31) = byte value b occurs at content
// position q).  Packs positions while their ranks fit the (32 - pbits)-bit field and returns how many it packed; the sort
// uses the table only when that is more than the (32 - pbits) / 8 positions the raw prefix holds.
static inline uint32_t sym_table_build(const uint32_t *sets, int pbits, SymTable *t) {
  memset(t, 0, sizeof(*t));
  const uint32_t avail = 32u - (uint32_t)pbits;
  uint32_t used = 0, np = 0;
  for (; np < (uint32_t)SYM_MAX_POS; np++) {
    uint32_t cnt = 0;
    for (int w = 0; w < 8; w++) cnt += (uint32_t)__builtin_popcount(sets[np * 8 + w]);
    if (cnt == 0) break;                       // no key is this long
    uint32_t bits = 0;
    while ((1u << bits) < cnt + 1) bits++;     // ranks 1..cnt, 0 = the key ended
    if (used + bits > avail) break;
    used += bits;
    t->shift[np] = (uint8_t)(avail - used);
    uint32_t rk = 0;
    for (uint32_t b = 0; b < 256; b++)
      if ((sets[np * 8 + (b >> 5)] >> (b & 31u)) & 1u) t->rank[np][b] = (uint16_t)(++rk);
  }
  t->npos = np;
  return np;
}
static inline bool sym_table_pays(uint32_t npos, int pbits) { return npos > (32u - (uint32_t)pbits) / 8u; }

// Collected records as they sit in HBM (the analogue of PipelinedSorter's kvbuffer + kvmeta, :957-959)
struct Records {
  const uint8_t *kv;        // serialized bytes, key immediately followed by value
  uint64_t kv_bytes;        // valid bytes in kv (multiple of 16 allocated)
  const uint64_t *key_off;  // var mode
  const uint64_t *val_off;  // optional: value bytes not adjacent to the key (parsed IFile segments with repeats)
  const uint32_t *key_len;
  const uint32_t *val_len;
  const int32_t *partition;  // optional
  const uint32_t *tag;       // merge only: (segment id << 1) | record was run-length encoded in its input segment
  uint32_t n;
  uint32_t klen, vlen;  // fixed mode
  int fixed;
  int cmp;
  int hash_partition;
  int num_partitions;
  int pbits;  // bits of the sort word that hold the partition
  int use_runs;   // fixed mode: records are addressed through `runs` instead of index * stride / key_off
  RunTable runs;
  const SymTable *sym;  // optional alphabet-compressed sort word (variable-length keys)
  int unordered;        // UnorderedPartitionedKVWriter: no key order; the sort word is the partition alone and record i is
                        // staged at position n-1-i, so the stable sort leaves every partition newest record first
};

__device__ __forceinline__ void record_lookup(const Records &r, uint32_t i, uint64_t &koff, uint32_t &klen,
                                              uint32_t &vlen) {
  if (r.fixed) {
    // fixed framing; key_off present = records live at explicit offsets (parsed fixed-width IFile segments);
    // use_runs = offsets are arithmetic over the segment table
    if (r.use_runs) {
      uint32_t seg;
      koff = run_record_off(r.runs, i, seg) + r.runs.hdr_len;
    } else {
      koff = r.key_off ? r.key_off[i] : (uint64_t)i * (r.klen + r.vlen);
    }
    klen = r.klen;
    vlen = r.vlen;
  } else {
    koff = r.key_off[i];
    klen = r.key_len[i];
    vlen = r.val_len[i];
  }
}

// merge only: (segment id << 1) | record was run-length encoded in its input segment
__device__ __forceinline__ uint32_t record_tag(const Records &r, uint32_t i) {
  return (r.fixed && r.use_runs) ? run_of(r.runs, i) << 1 : r.tag[i];
}

// ------------------------------------------------------------------------------------------------ stage
// K = partition << (32 - pbits) | prefix >> pbits.  bad: the partition lies outside [0, num_partitions) (it is replaced
// by 0).  Unordered: the word is the partition alone.
__host__ __device__ __forceinline__ uint32_t compose_sort_word(const Records &r, int32_t p, uint32_t prefix, bool &bad) {
  bad = p < 0 || p >= r.num_partitions;
  if (bad) p = 0;
  if (r.unordered) prefix = 0;
  return r.pbits ? (((uint32_t)p << (32 - r.pbits)) | (prefix >> r.pbits)) : prefix;
}

// Sort word of one record with its key at `key` (every path of k_stage but the 16-byte fast one; the host emulation
// tezgpu_debug_sort_words_emulate runs the same code): partition id (TOTAL_ORDER: the search among the split points of
// `sp`, whose prefix words are read from `split_pw`; else HashPartitioner, else `given`) and prefix = the first
// normalised content bytes or the packed SymTable ranks.
template <bool TOTAL_ORDER = false>
__host__ __device__ __forceinline__ uint32_t stage_sort_word(const Records &r, const uint8_t *key, uint32_t klen,
                                                             int32_t given, bool &bad, const SplitTable *sp = nullptr,
                                                             const uint64_t *split_pw = nullptr) {
  const uint32_t skip = key_content_skip(r.cmp, key, klen);
  const uint8_t *content = key + skip;
  const uint32_t clen = klen - skip;
  uint32_t prefix = 0;
  if (r.sym) {   // packed ranks: already a (32 - pbits)-bit value, shifted up so that the common `>> pbits` below fits
    const SymTable *__restrict__ st = r.sym;
    const uint32_t np = st->npos;
    for (uint32_t q = 0; q < np && q < clen; q++) prefix |= (uint32_t)st->rank[q][norm_byte(r.cmp, content, q)] << st->shift[q];
    prefix <<= r.pbits;
  } else {
#pragma unroll
    for (uint32_t b = 0; b < 4; b++) prefix = (prefix << 8) | (b < clen ? norm_byte(r.cmp, content, b) : 0u);
  }
  int32_t p;
  if constexpr (TOTAL_ORDER) p = split_partition(*sp, split_pw, key, klen);
  else p = r.hash_partition ? (int32_t)((uint32_t)(key_hash_dev(r.cmp, key, klen) & 0x7fffffff) % (uint32_t)r.num_partitions)
                            : given;
  return compose_sort_word(r, p, prefix, bad);
}

constexpr int STAGE_ERR_PARTITION = 1;  // k_stage's error bits: "Illegal partition" (PipelinedSorter.java:410-413),
constexpr int STAGE_ERR_FRAMING = 2;    // and in run-table mode, a record position that lacks the fixed framing bytes

// One thread per record: its sort word (stage_sort_word, or inline for 16-byte fixed keys) and the digit histograms of
// all four radix passes (so the sort never re-reads the keys for counting).  TOTAL_ORDER: the partition is the search
// among the split points `sp` (TotalOrderPartitioner; unused otherwise -- it is the last parameter, so the other
// instantiations keep their parameter layout); the launch passes sp.n * 8 bytes of dynamic shared memory when
// sp.n <= SPLIT_SMEM_MAX (the prefix words are staged there), else 0 and the search reads the table in global memory.
template <bool FAST16, bool TOTAL_ORDER = false>
__global__ void __launch_bounds__(256) k_stage(Records r, uint32_t *__restrict__ keys_out, uint32_t *__restrict__ hist,
                                               int *__restrict__ error_flag, SplitTable sp) {
  __shared__ uint32_t s_hist[4 * RADIX];
  const uint64_t *split_pw = nullptr;
  if constexpr (TOTAL_ORDER) {
    extern __shared__ uint64_t s_split_pw[];
    split_pw = sp.prefix;
    if (sp.n <= SPLIT_SMEM_MAX) {
      for (uint32_t i = threadIdx.x; i < sp.n; i += blockDim.x) s_split_pw[i] = sp.prefix[i];
      split_pw = s_split_pw;
    }
  }
  for (int i = threadIdx.x; i < 4 * RADIX; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += stride) {
    uint32_t K;
    bool bad;
    if (FAST16) {
      // fixed 16-byte keys on a 16-byte aligned stride (config C2): one 128-bit load per record
      const uint4 kq = *reinterpret_cast<const uint4 *>(r.kv + (uint64_t)i * (r.klen + r.vlen));
      const uint32_t prefix = __byte_perm(kq.x, 0, 0x0123);
      int32_t p;
      if constexpr (TOTAL_ORDER) {
        const uint8_t *key = r.kv + (uint64_t)i * (r.klen + r.vlen);
        p = sp.order == CMP_BYTES
                ? (int32_t)split_upper_bound(sp, split_pw, ((uint64_t)prefix << 32) | __byte_perm(kq.y, 0, 0x0123), key, 16)
                : split_partition(sp, split_pw, key, 16);
      } else if (r.hash_partition) {
        uint32_t h = 1;
        const uint32_t w[4] = {kq.x, kq.y, kq.z, kq.w};
#pragma unroll
        for (int k = 0; k < 16; k++) h = 31u * h + (uint32_t)(int32_t)(int8_t)((w[k >> 2] >> (8 * (k & 3))) & 0xFF);
        p = (int32_t)((h & 0x7fffffffu) % (uint32_t)r.num_partitions);
      } else {
        p = r.partition ? r.partition[i] : 0;
      }
      K = compose_sort_word(r, p, prefix, bad);
    } else {
      uint64_t koff;
      uint32_t klen, vlen;
      int32_t run_part = 0;
      if (r.fixed && r.use_runs) {
        // consecutive records of a warp sit in the same run or the next few: one binary search per warp, lanes walk on
        const unsigned am = __activemask();
        const int leader = __ffs(am) - 1;
        uint32_t seg = (int)(threadIdx.x & 31) == leader ? run_of(r.runs, i) : 0u;
        seg = __shfl_sync(am, seg, leader);
        while (seg + 1 < r.runs.nseg && i >= __ldg(r.runs.rec_base + seg + 1)) seg++;
        const uint64_t roff = __ldg(r.runs.seg_off + seg) + (uint64_t)(i - __ldg(r.runs.rec_base + seg)) * r.runs.rec_size;
        koff = roff + r.runs.hdr_len;
        klen = r.klen;
        vlen = r.vlen;
        run_part = (int32_t)__ldg(r.runs.seg_part + seg);
        // the sequential IFile.Reader walk visits exactly these positions iff every one of them carries the fixed
        // framing bytes (same sector as the key: free); a mismatch sends the merge to the general parser
        bool ok = true;
        for (uint32_t b = 0; b < r.runs.hdr_len; b++) ok &= r.kv[roff + b] == (uint8_t)(r.runs.hdr_bytes[b >> 3] >> (8 * (b & 7)));
        if (!ok) atomicOr(error_flag, STAGE_ERR_FRAMING);
      } else {
        record_lookup(r, i, koff, klen, vlen);
      }
      const int32_t given = r.hash_partition ? 0 : ((r.fixed && r.use_runs) ? run_part : (r.partition ? r.partition[i] : 0));
      K = stage_sort_word<TOTAL_ORDER>(r, r.kv + koff, klen, given, bad, &sp, split_pw);
    }
    if (bad) atomicOr(error_flag, STAGE_ERR_PARTITION);
    keys_out[r.unordered ? r.n - 1u - i : i] = K;
#pragma unroll
    for (int q = 0; q < 4; q++) atomicAdd(&s_hist[q * RADIX + ((K >> (8 * q)) & 0xFF)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * RADIX; i += blockDim.x) {
    uint32_t c = s_hist[i];
    if (c) atomicAdd(&hist[i], c);
  }
}

// which byte values occur at each of the first SYM_MAX_POS normalised content positions: sets[q][b >> 5] bit (b & 31)
__global__ void __launch_bounds__(256) k_symbols(Records r, uint32_t *__restrict__ sets /*[SYM_MAX_POS][8]*/) {
  __shared__ uint32_t s_set[SYM_MAX_POS * 8];
  for (int i = threadIdx.x; i < SYM_MAX_POS * 8; i += blockDim.x) s_set[i] = 0;
  __syncthreads();
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < r.n; i += stride) {
    uint64_t koff;
    uint32_t klen, vlen;
    record_lookup(r, i, koff, klen, vlen);
    const uint8_t *key = r.kv + koff;
    const uint32_t skip = key_content_skip(r.cmp, key, klen);
    const uint8_t *content = key + skip;
    const uint32_t clen = klen - skip;
    for (uint32_t q = 0; q < (uint32_t)SYM_MAX_POS && q < clen; q++) {
      const uint32_t b = norm_byte(r.cmp, content, q);
      const uint32_t bit = 1u << (b & 31u);
      if (!(s_set[q * 8 + (b >> 5)] & bit)) atomicOr(&s_set[q * 8 + (b >> 5)], bit);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SYM_MAX_POS * 8; i += blockDim.x)
    if (s_set[i]) atomicOr(&sets[i], s_set[i]);
}

// ------------------------------------------------------------------------------------------------ tie detection
// After the prefix sort, records whose sort words collide form contiguous groups that still need ordering by the
// rest of the key (the RawComparator's job in SortSpan.compareKeys, :996-1010).
__device__ __forceinline__ void tie_flags(const uint32_t *__restrict__ K, uint32_t n, uint32_t i, bool &tied, bool &head) {
  uint32_t k = K[i];
  bool eq_prev = i > 0 && K[i - 1] == k;
  bool eq_next = i + 1 < n && K[i + 1] == k;
  tied = eq_prev || eq_next;
  head = tied && !eq_prev;
}

// Ordered block-level ranking of two flag sets over a tile processed in striped rows (row k holds elements
// k*THREADS + tid): returns, for this thread's element of row k, the number of flagged elements that precede it in
// index order, for both flag sets packed as (tied | heads << 32).  s_cnt: [SCAN_IPT][SCAN_THREADS/32] u64.
struct TileFlags {
  bool t[SCAN_IPT], h[SCAN_IPT];
};

__device__ __forceinline__ void tile_load_flags(const uint32_t *__restrict__ K, uint32_t n, uint32_t *s_k, TileFlags &f,
                                                uint32_t tile) {
  const uint32_t base = tile * SCAN_TILE;
  for (uint32_t i = threadIdx.x; i < SCAN_TILE + 2; i += SCAN_THREADS) {
    int64_t gi = (int64_t)base + i - 1;
    s_k[i] = (gi >= 0 && gi < (int64_t)n) ? K[gi] : 0u;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t li = k * SCAN_THREADS + threadIdx.x, i = base + li;
    f.t[k] = f.h[k] = false;
    if (i < n) {
      uint32_t v = s_k[li + 1];
      bool eq_prev = i > 0 && s_k[li] == v;
      bool eq_next = i + 1 < n && s_k[li + 2] == v;
      f.t[k] = eq_prev || eq_next;
      f.h[k] = f.t[k] && !eq_prev;
    }
  }
}

__global__ void __launch_bounds__(SCAN_THREADS) k_tie_count(const uint32_t *__restrict__ K, uint32_t n,
                                                            uint64_t *__restrict__ blk) {
  __shared__ uint32_t s_k[SCAN_TILE + 2];
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  TileFlags f;
  tile_load_flags(K, n, s_k, f, blockIdx.x);
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) s += (uint64_t)f.t[k] | ((uint64_t)f.h[k] << 32);
  uint64_t tot;
  block_exclusive_scan_u64(s, s_warp, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
}

// writes, for every tied position (ascending): its position, dense group id and record index
__global__ void __launch_bounds__(SCAN_THREADS)
    k_tie_compact(const uint32_t *__restrict__ K, const uint32_t *__restrict__ order, uint32_t n,
                  const uint64_t *__restrict__ blk, uint32_t *__restrict__ pos, uint32_t *__restrict__ gid,
                  uint32_t *__restrict__ lidx) {
  __shared__ uint32_t s_k[SCAN_TILE + 2];
  __shared__ uint32_t s_ct[SCAN_IPT][SCAN_THREADS / 32], s_ch[SCAN_IPT][SCAN_THREADS / 32];
  TileFlags f;
  tile_load_flags(K, n, s_k, f, blockIdx.x);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = lanemask_lt();
  uint32_t bt[SCAN_IPT], bh[SCAN_IPT];
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    bt[k] = __ballot_sync(0xffffffffu, f.t[k]);
    bh[k] = __ballot_sync(0xffffffffu, f.h[k]);
    if (lane == 0) { s_ct[k][warp] = __popc(bt[k]); s_ch[k][warp] = __popc(bh[k]); }
  }
  __syncthreads();
  // exclusive prefix over (row, warp) in index order; rows are few, so every thread walks the small table
  const uint64_t b0 = blk[blockIdx.x];
  uint32_t run_t = (uint32_t)b0, run_h = (uint32_t)(b0 >> 32);
  const uint32_t base = blockIdx.x * SCAN_TILE;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t pre_t = run_t, pre_h = run_h;
#pragma unroll
    for (int w = 0; w < SCAN_THREADS / 32; w++) {
      uint32_t ct = s_ct[k][w], ch = s_ch[k][w];
      if (w < warp) { pre_t += ct; pre_h += ch; }
      run_t += ct; run_h += ch;
    }
    if (f.t[k]) {
      uint32_t at = pre_t + __popc(bt[k] & lt);
      uint32_t heads = pre_h + __popc(bh[k] & lt) + (f.h[k] ? 1u : 0u);  // heads up to and including this element
      uint32_t i = base + k * SCAN_THREADS + threadIdx.x;
      pos[at] = i;
      gid[at] = heads - 1;
      lidx[at] = order[i];
    }
  }
}

// ------------------------------------------------------------------------------------------------ equal-key groups
// Large tie groups are usually large because the SAME key occurs many times (a reduce-side merge of word counts, a
// 2^24-word key space spread over 256 runs): such a group needs no ordering at all -- the radix sort is stable, so its
// members already stand in (run, position) order -- only its same[] flags.  These kernels test every group larger than
// TIE_SMALL_MAX for "all members equal to the first" and settle those; only groups that really contain different keys
// go on to the key-suffix refinement rounds.  Input: the compacted tied list (pos, gid, lidx) of k_tie_compact.
__global__ void __launch_bounds__(256) k_group_heads(const uint32_t *__restrict__ gid, uint32_t m, uint32_t *__restrict__ ghead) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint32_t g = gid[j];
  if (j == 0 || gid[j - 1] != g) ghead[g] = j;
  if (j + 1 == m) ghead[g + 1] = m;
}

__device__ __forceinline__ int compare_keys_from(const Records &r, uint32_t ra, uint32_t rb, uint32_t depth);

__global__ void __launch_bounds__(256)
    k_group_equal(Records r, const uint32_t *__restrict__ gid, const uint32_t *__restrict__ lidx, const uint32_t *__restrict__ ghead,
                  uint32_t m, uint32_t depth, uint32_t small_max, uint8_t *__restrict__ gneq) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint32_t g = gid[j], h = ghead[g];
  if (ghead[g + 1] - h <= small_max || j == h) return;     // small groups were ordered in place by k_tie_fix
  if (compare_keys_from(r, lidx[h], lidx[j], depth) != 0) gneq[g] = 1;
}

// settles the all-equal large groups (flags + duplicate count) and counts what still needs refinement:
// blk[b] = survivors | heads of surviving groups << 32
__global__ void __launch_bounds__(SCAN_THREADS)
    k_group_mark(const uint32_t *__restrict__ pos, const uint32_t *__restrict__ gid, const uint32_t *__restrict__ ghead,
                 const uint8_t *__restrict__ gneq, uint32_t m, uint32_t small_max, uint8_t *__restrict__ same,
                 unsigned long long *__restrict__ dup_count, uint64_t *__restrict__ blk) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_IPT;
  uint64_t sv = 0;
  uint32_t dups = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    const uint32_t j = base + k;
    if (j < m) {
      const uint32_t g = gid[j], h = ghead[g];
      if (ghead[g + 1] - h > small_max) {
        if (gneq[g]) sv += 1ull | ((uint64_t)(j == h) << 32);
        else if (j != h) { same[pos[j]] = 1; dups++; }
      }
    }
  }
  uint64_t tot;
  block_exclusive_scan_u64(sv, s_warp, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dups += __shfl_xor_sync(0xffffffffu, dups, o);
  if ((threadIdx.x & 31) == 0 && dups) atomicAdd(dup_count, (unsigned long long)dups);
}

__global__ void __launch_bounds__(SCAN_THREADS)
    k_group_compact(const uint32_t *__restrict__ pos, const uint32_t *__restrict__ gid, const uint32_t *__restrict__ lidx,
                    const uint32_t *__restrict__ ghead, const uint8_t *__restrict__ gneq, uint32_t m, uint32_t small_max,
                    const uint64_t *__restrict__ blk, uint32_t *__restrict__ pos_out, uint32_t *__restrict__ gid_out,
                    uint32_t *__restrict__ lidx_out) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_IPT;
  bool keep[SCAN_IPT], head[SCAN_IPT];
  uint64_t sv = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    const uint32_t j = base + k;
    keep[k] = head[k] = false;
    if (j < m) {
      const uint32_t g = gid[j], h = ghead[g];
      keep[k] = (ghead[g + 1] - h > small_max) && gneq[g];
      head[k] = keep[k] && j == h;
    }
    sv += (uint64_t)keep[k] | ((uint64_t)head[k] << 32);
  }
  const uint64_t ex = block_exclusive_scan_u64(sv, s_warp, nullptr) + blk[blockIdx.x];
  uint32_t at = (uint32_t)ex, heads = (uint32_t)(ex >> 32);
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    if (keep[k]) {
      if (head[k]) heads++;
      const uint32_t j = base + k;
      pos_out[at] = pos[j];
      gid_out[at] = heads - 1;
      lidx_out[at] = lidx[j];
      at++;
    }
  }
}

// ------------------------------------------------------------------------------------------------ key comparison
// full RawComparator order of two records' keys from normalised content byte `depth` on (bytes before it are equal)
__device__ __forceinline__ int compare_keys_from(const Records &r, uint32_t ra, uint32_t rb, uint32_t depth) {
  uint64_t ka, kb;
  uint32_t la, lb, va, vb;
  record_lookup(r, ra, ka, la, va);
  record_lookup(r, rb, kb, lb, vb);
  const uint8_t *a = r.kv + ka, *b = r.kv + kb;
  uint32_t sa = key_content_skip(r.cmp, a, la), sb = key_content_skip(r.cmp, b, lb);
  a += sa; b += sb; la -= sa; lb -= sb;
  uint32_t nmin = la < lb ? la : lb;
  uint32_t i = depth;
  if (i == 0 && nmin > 0) {   // byte 0 is the only one a comparator normalises (sign bit of IntWritable / LongWritable)
    uint32_t x = norm_byte(r.cmp, a, 0), y = norm_byte(r.cmp, b, 0);
    if (x != y) return x < y ? -1 : 1;
    i = 1;
  }
  // eight bytes per step: sixteen independent byte loads (any alignment, never past the keys) instead of a chain of
  // load-compare-branch per byte -- equal keys (the common case when merging word counts) are compared to their end
  for (; i + 8 <= nmin; i += 8) {
    uint64_t x = 0, y = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) {
      x = (x << 8) | a[i + q];
      y = (y << 8) | b[i + q];
    }
    if (x != y) return x < y ? -1 : 1;
  }
  for (; i < nmin; i++) {
    uint32_t x = a[i], y = b[i];
    if (x != y) return x < y ? -1 : 1;
  }
  return la < lb ? -1 : (la == lb ? 0 : 1);
}

constexpr uint32_t TIE_SMALL_MAX = 16;

// ------------------------------------------------------------------------------------------------ in-place tie fix
// One streaming pass over the sorted sort words finds the head of every group of colliding records; groups of at most
// TIE_SMALL_MAX records (with uniformly distributed keys: essentially all of them, 2-3 members each) are ordered on the
// spot by ONE thread with a stable insertion sort under the full RawComparator.  No compaction, no scan, no host round
// trip.  Larger groups are only counted (-> general refinement path).
constexpr int TIEFIX_THREADS = 256;
constexpr int TIEFIX_IPT = 8;
constexpr int TIEFIX_TILE = TIEFIX_THREADS * TIEFIX_IPT;

constexpr int TIEFIX_FLUSH = 4 * TIEFIX_THREADS;               // process the collected heads once this many are queued
constexpr int TIEFIX_CAP = TIEFIX_FLUSH + TIEFIX_TILE / 2 + 8;  // a tile adds at most TILE/2 heads

__device__ __forceinline__ void tie_fix_group(const Records &r, const uint32_t *__restrict__ K, uint32_t *__restrict__ order,
                                              uint32_t n, uint32_t i, uint32_t depth, uint8_t *__restrict__ same,
                                              uint32_t &my_dups, uint32_t &my_ties, uint32_t *__restrict__ large_groups) {
  const uint32_t k = K[i];
  uint32_t e = i + 2;
  while (e < n && e - i <= TIE_SMALL_MAX && K[e] == k) e++;
  const uint32_t sz = e - i;
  if (sz > TIE_SMALL_MAX) { atomicAdd(large_groups, 1u); return; }
  my_ties += sz;
  uint32_t idx[TIE_SMALL_MAX];
  for (uint32_t j = 0; j < sz; j++) idx[j] = order[i + j];
  // stable insertion sort (equal keys keep their original relative order).  eq bit j = "idx[j] equals idx[j-1]" is kept
  // up to date from the comparisons the sort makes anyway (a merge of word counts is mostly duplicates: one comparison
  // per record instead of two): the element an insertion stops at compares <= v, everything shifted right compares > v,
  // and whatever is later inserted between two equal neighbours equals both.
  uint32_t eq = 0;
  for (uint32_t a = 1; a < sz; a++) {
    const uint32_t v = idx[a];
    uint32_t b = a;
    int c = 1;
    while (b > 0) {
      c = compare_keys_from(r, idx[b - 1], v, depth);
      if (c <= 0) break;
      idx[b] = idx[b - 1];
      b--;
    }
    idx[b] = v;
    // bits b+1 .. a-1 (pairs that moved together) shift up by one, bit b+1 (v < its new successor) and bit b are rewritten
    const uint32_t low = eq & ((1u << b) - 1u);
    const uint32_t high = b < a ? ((eq >> (b + 1)) << (b + 2)) : 0u;
    eq = low | high | ((b > 0 && c == 0) ? (1u << b) : 0u);
  }
  order[i] = idx[0];
  for (uint32_t j = 1; j < sz; j++) {
    order[i + j] = idx[j];
    if ((eq >> j) & 1u) same[i + j] = 1;
  }
  my_dups += (uint32_t)__popc(eq);
}

// The streaming part (all warps) queues group heads in shared memory; once a few hundred are queued every thread takes
// one, so the latency-bound comparator work runs with the whole CTA instead of one warp.
__global__ void __launch_bounds__(TIEFIX_THREADS)
    k_tie_fix(Records r, const uint32_t *__restrict__ K, uint32_t *__restrict__ order, uint32_t n, uint32_t depth,
              uint8_t *__restrict__ same, unsigned long long *__restrict__ dup_count, uint32_t *__restrict__ large_groups,
              unsigned long long *__restrict__ tie_records) {
  __shared__ uint32_t s_heads[TIEFIX_CAP];
  __shared__ uint32_t s_nheads;
  const uint32_t ntiles = (n + TIEFIX_TILE - 1) / TIEFIX_TILE;
  if (threadIdx.x == 0) s_nheads = 0;
  __syncthreads();
  uint32_t my_dups = 0, my_ties = 0;
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const uint32_t base = tile * TIEFIX_TILE;
    uint32_t kk[TIEFIX_IPT], kp[TIEFIX_IPT], kn[TIEFIX_IPT];
#pragma unroll
    for (int q = 0; q < TIEFIX_IPT; q++) {
      const uint32_t i = base + q * TIEFIX_THREADS + threadIdx.x;
      kk[q] = i < n ? __ldg(K + i) : 0u;
      kp[q] = (i > 0 && i < n) ? __ldg(K + i - 1) : ~kk[q];
      kn[q] = (i + 1 < n) ? __ldg(K + i + 1) : ~kk[q];
    }
#pragma unroll
    for (int q = 0; q < TIEFIX_IPT; q++) {
      const uint32_t i = base + q * TIEFIX_THREADS + threadIdx.x;
      if (i < n && kp[q] != kk[q] && kn[q] == kk[q]) s_heads[atomicAdd(&s_nheads, 1u)] = i;
    }
    __syncthreads();
    const uint32_t nh = s_nheads;
    const bool last = tile + gridDim.x >= ntiles;
    // every thread has read nh before any thread of the next iteration bumps s_nheads again (the flush decision must be
    // CTA-uniform: the branches below contain barriers)
    __syncthreads();
    if (nh >= (uint32_t)TIEFIX_FLUSH || last) {
      for (uint32_t hidx = threadIdx.x; hidx < nh; hidx += TIEFIX_THREADS)
        tie_fix_group(r, K, order, n, s_heads[hidx], depth, same, my_dups, my_ties, large_groups);
      __syncthreads();
      if (threadIdx.x == 0) s_nheads = 0;
      __syncthreads();
    }
  }
  if (my_dups) atomicAdd(dup_count, (unsigned long long)my_dups);
  if (my_ties) atomicAdd(tie_records, (unsigned long long)my_ties);
}

// ------------------------------------------------------------------------------------------------ refinement rounds
// sub-key for the next 3 normalised content bytes at `depth`:
//   len >  depth : chunk24 << 8 | (128 + min(3, len - depth))
//   len <= depth : min(len, 127)                (a proper prefix of every longer key in the group => sorts first)
// a tag of 131 means "may still differ further on"; anything smaller is final.
__device__ __forceinline__ uint32_t ref_subkey(const Records &r, uint32_t rec, uint32_t depth) {
  uint64_t koff;
  uint32_t klen, vlen;
  record_lookup(r, rec, koff, klen, vlen);
  const uint8_t *key = r.kv + koff;
  uint32_t skip = key_content_skip(r.cmp, key, klen);
  const uint8_t *content = key + skip;
  uint32_t clen = klen - skip;
  if (clen <= depth) return clen < 127u ? clen : 127u;
  uint32_t chunk = 0;
#pragma unroll
  for (uint32_t b = 0; b < 3; b++) chunk = (chunk << 8) | (depth + b < clen ? norm_byte(r.cmp, content, depth + b) : 0u);
  uint32_t rem = clen - depth;
  return (chunk << 8) | (128u + (rem < 3u ? rem : 3u));
}

__global__ void __launch_bounds__(256) k_ref_build_keys(Records r, const uint32_t *__restrict__ gid,
                                                        const uint32_t *__restrict__ lidx, uint32_t m, uint32_t depth,
                                                        uint64_t *__restrict__ key64) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < m) key64[j] = ((uint64_t)gid[j] << 32) | ref_subkey(r, lidx[j], depth);
}

__device__ __forceinline__ void ref_flags(const uint64_t *__restrict__ K, uint32_t m, uint32_t j, bool &tied, bool &head,
                                          bool &open) {
  uint64_t k = K[j];
  bool eq_prev = j > 0 && K[j - 1] == k;
  bool eq_next = j + 1 < m && K[j + 1] == k;
  tied = eq_prev || eq_next;
  head = tied && !eq_prev;
  open = ((uint32_t)k & 0xFF) == 131u;  // more key bytes may follow
}

// applies the round's order, records finished duplicates, counts what is still unresolved
__global__ void __launch_bounds__(SCAN_THREADS)
    k_ref_apply_count(const uint64_t *__restrict__ K, const uint32_t *__restrict__ lidx_sorted,
                      const uint32_t *__restrict__ pos, uint32_t m, uint32_t *__restrict__ order,
                      uint8_t *__restrict__ same, unsigned long long *__restrict__ dup_count,
                      uint64_t *__restrict__ blk) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_IPT;
  uint64_t s = 0;
  uint32_t dups = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t j = base + k;
    if (j < m) {
      bool t, h, open;
      ref_flags(K, m, j, t, h, open);
      uint32_t p = pos[j];
      order[p] = lidx_sorted[j];
      if (t && open) s += 1ull | ((uint64_t)h << 32);
      if (t && !open && !h) {
        same[p] = 1;  // byte-identical to the key at sorted position p-1
        dups++;
      }
    }
  }
  uint64_t tot;
  block_exclusive_scan_u64(s, s_warp, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dups += __shfl_xor_sync(0xffffffffu, dups, o);
  if ((threadIdx.x & 31) == 0 && dups) atomicAdd(dup_count, (unsigned long long)dups);
}

__global__ void __launch_bounds__(SCAN_THREADS)
    k_ref_compact(const uint64_t *__restrict__ K, const uint32_t *__restrict__ lidx_sorted,
                  const uint32_t *__restrict__ pos, uint32_t m, const uint64_t *__restrict__ blk,
                  uint32_t *__restrict__ pos_out, uint32_t *__restrict__ gid_out, uint32_t *__restrict__ lidx_out) {
  __shared__ uint64_t s_warp[SCAN_THREADS / 32];
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_IPT;
  bool u[SCAN_IPT], h[SCAN_IPT];
  uint64_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    uint32_t j = base + k;
    u[k] = h[k] = false;
    if (j < m) {
      bool t, hh, open;
      ref_flags(K, m, j, t, hh, open);
      u[k] = t && open;
      h[k] = u[k] && hh;
    }
    s += (uint64_t)u[k] | ((uint64_t)h[k] << 32);
  }
  uint64_t ex = block_exclusive_scan_u64(s, s_warp, nullptr) + blk[blockIdx.x];
  uint32_t at = (uint32_t)ex, heads = (uint32_t)(ex >> 32);
#pragma unroll
  for (int k = 0; k < SCAN_IPT; k++) {
    if (u[k]) {
      if (h[k]) heads++;
      uint32_t j = base + k;
      pos_out[at] = pos[j];
      gid_out[at] = heads - 1;
      lidx_out[at] = lidx_sorted[j];
      at++;
    }
  }
}

// unordered mode: the sort ran over positions n-1-i; turn them back into record indices
__global__ void k_flip_order(uint32_t *__restrict__ order, uint32_t n) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) order[r] = n - 1u - order[r];
}

// ------------------------------------------------------------------------------------------------ layout
// part_start[p] = first sorted position of partition p (p in [0, P]); lower_bound over the sorted sort words
__global__ void k_part_bounds(const uint32_t *__restrict__ K, uint32_t n, int P, int pbits,
                              uint32_t *__restrict__ part_start) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > P) return;
  if (p == P) { part_start[p] = n; return; }
  if (pbits == 0) { part_start[p] = 0; return; }
  uint64_t target = (uint64_t)p << (32 - pbits);
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    uint32_t mid = lo + ((hi - lo) >> 1);
    if ((uint64_t)K[mid] < target) lo = mid + 1;
    else hi = mid;
  }
  part_start[p] = lo;
}

struct EmitParams {
  Records rec;
  const uint32_t *order;       // sorted position -> record index
  const uint8_t *same;         // same[r]: key at r equals key at r-1 (only meaningful when rle)
  const uint64_t *rec_off;     // var mode: exclusive scan of emitted record sizes (n+1 entries); null in fixed mode
  const uint32_t *part_start;  // [P+1]
  const uint64_t *seg_start;   // [P+1] byte offset of every segment in file.out
  const uint32_t *tile_start;  // [P+1] first emit tile of every partition
  uint8_t *out;                // file.out bytes (16-byte aligned)
  uint32_t *seg_crc;           // [P] xor-accumulated CRC contributions
  const CrcTables *crc;
  uint32_t recs_per_tile;
  uint32_t rec_size;           // fixed mode: emitted bytes per record
  uint8_t fixed_hdr[12];       // fixed mode: vint(klen) vint(vlen)
  uint32_t fixed_hdr_len;
  int rle;
  int merge_mode;      // TezMerger.writeFile semantics: isSameKey() records go through IFile.REPEAT_KEY
  int check_same;      // merge_mode: MergeQueue.checkForSameKeys (SORT/TezMerger.java:563-573,597-652)
  int send_empty;
  int unordered;       // UnorderedPartitionedKVWriter.mergeAll: partitions without records get an all-zero index entry
  int P;
  const uint8_t *rep;  // optional, [n]: emit_is_repeat() of every sorted position, computed once (k_emit_repeat_flags)
};

// Is the record at sorted position r written as a repeat of the previous key ([RLE_MARKER] vint(vlen) value)?
//  sorter: IFile.Writer(rle) compares the raw key bytes with the previous key and never fires for empty keys
//          (SORT/IFile.java:541-544);
//  merger: TezMerger.writeFile passes IFile.REPEAT_KEY when MergeQueue.isSameKey() -- the record was read as SAME_KEY
//          from its own segment, or the top segment changed and the comparator reports equality
//          (SORT/TezMerger.java:215-245,597-652) -- and the writer's own test applies on top when it was built with rle.
__device__ __forceinline__ bool emit_is_repeat(const EmitParams &e, uint32_t r, uint32_t ps) {
  if (e.rep) return e.rep[r] != 0;   // k_emit_sizes and k_emit ask twice per record each: one gather pass instead of four
  if (r == ps || !e.same[r]) return false;
  const Records &rec = e.rec;
  const uint32_t i = e.order[r];
  uint64_t koff;
  uint32_t klen, vlen;
  record_lookup(rec, i, koff, klen, vlen);
  const bool writer = e.rle && klen > 0;
  if (!e.merge_mode) return writer;
  // read as SAME_KEY from its own segment; with checkForSameKeys also "the top segment changed and its key equals the
  // previous key" (compareKeyWithNextTopKey, :640-652)
  const uint32_t tag = record_tag(rec, i);
  if (writer || (tag & 1u)) return true;
  return e.check_same && ((tag >> 1) != (record_tag(rec, e.order[r - 1]) >> 1));
}

// emit_is_repeat() of every sorted position, once: the rule gathers the record's lengths and the tags of two records,
// and both k_emit_sizes and k_emit need it for r and r-1 (merging word counts: 6e8 records, ~6 random sector reads per
// evaluation)
__global__ void __launch_bounds__(256) k_emit_repeat_flags(EmitParams e, const uint32_t *__restrict__ K, uint8_t *__restrict__ flags) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= e.rec.n) return;
  const int sh = 32 - e.rec.pbits;
  const uint32_t p = e.rec.pbits ? (K[r] >> sh) : 0;
  flags[r] = emit_is_repeat(e, r, e.part_start[p]) ? 1 : 0;    // e.rep is null here: the rule itself
}

// var mode: emitted size of the record at sorted position r (IFile.Writer.writeKVPair / writeValue / markers,
// SORT/IFile.java:559-614): a repeated key costs [RLE_MARKER once] vint(vlen) val, the first new key after a run
// is preceded by V_END_MARKER, and a run that ends the segment is closed by V_END_MARKER before EOF.
__global__ void __launch_bounds__(256) k_emit_sizes(EmitParams e, const uint32_t *__restrict__ K, uint32_t *__restrict__ sizes) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  const Records &rec = e.rec;
  if (r >= rec.n) return;
  uint64_t koff;
  uint32_t klen, vlen;
  record_lookup(rec, e.order[r], koff, klen, vlen);
  const int sh = 32 - rec.pbits;
  const uint32_t p = rec.pbits ? (K[r] >> sh) : 0;
  const uint32_t ps = e.part_start[p], pe = e.part_start[p + 1];
  const bool last = (r + 1 == pe);
  const bool same_r = emit_is_repeat(e, r, ps);
  const bool same_prev = (r > ps) && emit_is_repeat(e, r - 1, ps);
  uint32_t sz;
  if (same_r) sz = (same_prev ? 0u : 1u) + vint_size_u32(vlen) + vlen;
  else sz = (same_prev ? 1u : 0u) + vint_size_u32(klen) + vint_size_u32(vlen) + klen + vlen;
  if (last && same_r) sz += 1;
  sizes[r] = sz;
}

// per-partition segment layout; single block.  index triples follow TezIndexRecord (start, rawLength, partLength).
__global__ void __launch_bounds__(1024)
    k_layout(EmitParams e, uint64_t *__restrict__ seg_start, uint32_t *__restrict__ tile_start,
             int64_t *__restrict__ index, uint64_t *__restrict__ totals /*[0]=file bytes,[1]=tiles*/) {
  __shared__ uint64_t s_warp[32];
  __shared__ uint64_t s_carry_b;
  __shared__ uint64_t s_carry_t;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_carry_b = 0; s_carry_t = 0; }
  __syncthreads();
  for (int base = 0; base < e.P; base += 1024) {
    int p = base + threadIdx.x;
    uint64_t seglen = 0, tiles = 0, body = 0;
    uint32_t cnt = 0;
    if (p < e.P) {
      uint32_t a = e.part_start[p], b = e.part_start[p + 1];
      cnt = b - a;
      if (cnt) {
        body = e.rec_off ? (e.rec_off[b] - e.rec_off[a]) : (uint64_t)cnt * e.rec_size;
        seglen = 4 + body + 2 + 4;
        tiles = (cnt + e.recs_per_tile - 1) / e.recs_per_tile;
      } else if (!e.send_empty && !e.unordered) {
        seglen = 10;
      }
    }
    // two independent scans packed sequentially (bytes can exceed 32 bits, so no packing tricks)
    uint64_t vb = seglen, ib = vb;
    uint64_t vt = tiles, it = vt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t tb = __shfl_up_sync(0xffffffffu, ib, o);
      uint64_t tt = __shfl_up_sync(0xffffffffu, it, o);
      if (lane >= o) { ib += tb; it += tt; }
    }
    if (lane == 31) s_warp[warp] = ib;
    __syncthreads();
    uint64_t wb = 0, totb = 0;
    for (int w = 0; w < 32; w++) { uint64_t x = s_warp[w]; if (w < warp) wb += x; totb += x; }
    __syncthreads();
    if (lane == 31) s_warp[warp] = it;
    __syncthreads();
    uint64_t wt = 0, tott = 0;
    for (int w = 0; w < 32; w++) { uint64_t x = s_warp[w]; if (w < warp) wt += x; tott += x; }
    uint64_t cb = s_carry_b, ct = s_carry_t;
    if (p < e.P) {
      uint64_t start = cb + wb + ib - vb;
      seg_start[p] = start;
      tile_start[p] = (uint32_t)(ct + wt + it - vt);
      index[3 * p + 0] = (e.unordered && !seglen) ? 0 : (int64_t)start;
      index[3 * p + 1] = seglen ? (int64_t)(seglen - 4) : 0;  // rawLength = header + body + EOF, no checksum
      index[3 * p + 2] = (int64_t)seglen;                     // partLength (uncompressed) = rawLength + 4
    }
    __syncthreads();
    if (threadIdx.x == 0) { s_carry_b = cb + totb; s_carry_t = ct + tott; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    seg_start[e.P] = s_carry_b;
    tile_start[e.P] = (uint32_t)s_carry_t;
    totals[0] = s_carry_b;
    totals[1] = s_carry_t;
  }
}

// ------------------------------------------------------------------------------------------------ emit
constexpr int EMIT_THREADS = 256;
constexpr int EMIT_MAX_RECS = 256;         // records per tile
constexpr int EMIT_IMG_BYTES = 24 * 1024;  // shared-memory image of the output bytes (one "piece")
constexpr int EMIT_CRC_STRIDE_WORDS = EMIT_THREADS;

struct EmitEntry {      // one record (or the header / EOF pseudo record) of a tile
  uint64_t src;         // offset in kv of the source bytes that follow the framing bytes
  uint64_t src2;        // second source range (value bytes when they are not adjacent to the key)
  uint32_t src_len;
  uint32_t src2_len;
  uint8_t hdr[12];      // framing bytes: [V_END] [RLE] vint(klen) vint(vlen)   or 'TIF\0' / EOF markers
  uint8_t hdr_len;
  uint8_t tail_fd;      // V_END_MARKER closing a run that ends the segment
};

// 16 aligned bytes at p; bytes outside [lo, hi) read as zero (never touches memory outside the buffer)
__device__ __forceinline__ uint4 load16_clamped(const uint8_t *p, const uint8_t *__restrict__ lo, const uint8_t *__restrict__ hi) {
  if (p >= lo && p + 16 <= hi) return *reinterpret_cast<const uint4 *>(p);
  uint32_t w[4] = {0, 0, 0, 0};
  for (int b = 0; b < 16; b++) {
    const uint8_t *q = p + b;
    if (q >= lo && q < hi) w[b >> 2] |= (uint32_t)(*q) << (8 * (b & 3));
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// merges `len` source bytes starting at global address src into bytes [o, o+len) of the 16-byte accumulator
__device__ __forceinline__ void merge_bytes(uint32_t acc[4], const uint8_t *__restrict__ src, uint32_t o, uint32_t len,
                                            const uint8_t *__restrict__ lo, const uint8_t *__restrict__ hi) {
  // window: 32 aligned source bytes such that accumulator byte q comes from window byte sh + q
  const uint8_t *first = src - o;  // address that would land on accumulator byte 0 (may precede the buffer)
  uint32_t sh = (uint32_t)((uintptr_t)first & 15u);
  const uint8_t *wb = first - sh;
  uint4 v0 = make_uint4(0, 0, 0, 0), v1 = make_uint4(0, 0, 0, 0);
  if (sh + o < 16u) v0 = load16_clamped(wb, lo, hi);
  if (sh + o + len > 16u) v1 = load16_clamped(wb + 16, lo, hi);
  const uint32_t bsh = (sh & 3u) * 8u;
  uint32_t r0, r1, r2, r3;
  switch (sh >> 2) {
    case 0:
      r0 = __funnelshift_r(v0.x, v0.y, bsh); r1 = __funnelshift_r(v0.y, v0.z, bsh);
      r2 = __funnelshift_r(v0.z, v0.w, bsh); r3 = __funnelshift_r(v0.w, v1.x, bsh);
      break;
    case 1:
      r0 = __funnelshift_r(v0.y, v0.z, bsh); r1 = __funnelshift_r(v0.z, v0.w, bsh);
      r2 = __funnelshift_r(v0.w, v1.x, bsh); r3 = __funnelshift_r(v1.x, v1.y, bsh);
      break;
    case 2:
      r0 = __funnelshift_r(v0.z, v0.w, bsh); r1 = __funnelshift_r(v0.w, v1.x, bsh);
      r2 = __funnelshift_r(v1.x, v1.y, bsh); r3 = __funnelshift_r(v1.y, v1.z, bsh);
      break;
    default:
      r0 = __funnelshift_r(v0.w, v1.x, bsh); r1 = __funnelshift_r(v1.x, v1.y, bsh);
      r2 = __funnelshift_r(v1.y, v1.z, bsh); r3 = __funnelshift_r(v1.z, v1.w, bsh);
      break;
  }
  const uint32_t rr[4] = {r0, r1, r2, r3};
  const uint32_t end = o + len;
#pragma unroll
  for (uint32_t w = 0; w < 4; w++) {
    uint32_t a = o > 4 * w ? o - 4 * w : 0u;
    uint32_t b = end < 4 * w + 4 ? (end > 4 * w ? end - 4 * w : 0u) : 4u;
    if (b > a) {
      uint32_t m = (0xFFFFFFFFu >> (8u * (4u - b))) & (0xFFFFFFFFu << (8u * a));
      acc[w] = (acc[w] & ~m) | (rr[w] & m);
    }
  }
}

__device__ __forceinline__ void put_byte(uint32_t acc[4], uint32_t q, uint32_t v) {
  uint32_t w = q >> 2, s = (q & 3u) * 8u;
#pragma unroll
  for (uint32_t k = 0; k < 4; k++)
    if (k == w) acc[k] = (acc[k] & ~(0xFFu << s)) | (v << s);
}

// One CTA per tile = up to EMIT_MAX_RECS consecutive sorted records of ONE partition.  The CTA builds the exact
// file.out byte image of those records in shared memory ("destination oriented": every lane assembles one aligned
// 16-byte output vector from the framing bytes and at most two 128-bit gathers per source record), folds the image
// into the segment CRC, and streams it out with coalesced 128-bit stores.
template <bool FIXED>
__global__ void __launch_bounds__(EMIT_THREADS) k_emit(EmitParams e) {
  __shared__ __align__(16) uint8_t s_img[EMIT_IMG_BYTES];
  __shared__ uint64_t s_loc[EMIT_MAX_RECS + 3];  // tile-relative start of every entry (header, records, EOF) + total
  __shared__ EmitEntry s_ent[EMIT_MAX_RECS + 2];
  __shared__ uint32_t s_tab[4 * 256];    // slice-by-4 tables
  __shared__ uint32_t s_adv[4 * 256];    // advance-by-stride tables
  __shared__ uint32_t s_red[EMIT_THREADS / 32];
  __shared__ uint32_t s_info[8];

  const int tid = threadIdx.x;
  for (int i = tid; i < 4 * 256; i += EMIT_THREADS) {
    s_tab[i] = (&e.crc->slice[0][0])[i];
    s_adv[i] = (&e.crc->adv[0][0])[i];
  }
  const uint32_t ntiles = e.tile_start[e.P];
  // persistent CTAs: with small records a tile is a few KB of output and there are millions of them -- the checksum
  // tables are loaded once per CTA, not once per tile
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
  __syncthreads();  // the previous tile's shared state is dead (and, first time round, the tables are in place)

  // ---- locate the tile: partition p, records [r0, r0 + nr)
  if (tid == 0) {
    int lo = 0, hi = e.P;  // last p with tile_start[p] <= tile
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (e.tile_start[mid] <= tile) lo = mid; else hi = mid;
    }
    // skip empty partitions that share the same tile_start
    while (lo + 1 < e.P && e.tile_start[lo + 1] <= tile) lo++;
    s_info[0] = (uint32_t)lo;
  }
  __syncthreads();
  const uint32_t p = s_info[0];
  const uint32_t ps = e.part_start[p], pe = e.part_start[p + 1];
  const uint32_t k = tile - e.tile_start[p];
  const uint32_t r0 = ps + k * e.recs_per_tile;
  const uint32_t nr = min(e.recs_per_tile, pe - r0);
  const bool first_tile = (k == 0), last_tile = (r0 + nr == pe);
  const Records &rec = e.rec;

  // ---- entries: [0] segment header, [1..nr] records, [nr+1] EOF markers
  const uint64_t body0 = FIXED ? (uint64_t)(r0 - ps) * e.rec_size : (e.rec_off[r0] - e.rec_off[ps]);
  for (uint32_t j = tid; j < nr + 2; j += EMIT_THREADS) {
    EmitEntry en;
    en.src = 0; en.src_len = 0; en.src2 = 0; en.src2_len = 0; en.hdr_len = 0; en.tail_fd = 0;
    uint64_t loc;
    if (j == 0) {
      loc = 0;
      if (first_tile) { en.hdr[0] = 'T'; en.hdr[1] = 'I'; en.hdr[2] = 'F'; en.hdr[3] = 0; en.hdr_len = 4; }
    } else if (j == nr + 1) {
      uint64_t body_end = FIXED ? (uint64_t)(r0 - ps + nr) * e.rec_size : (e.rec_off[r0 + nr] - e.rec_off[ps]);
      loc = (first_tile ? 4 : 0) + (body_end - body0);
      if (last_tile) { en.hdr[0] = 0xFF; en.hdr[1] = 0xFF; en.hdr_len = 2; }
    } else {
      const uint32_t r = r0 + j - 1;
      uint64_t koff;
      uint32_t klen, vlen;
      record_lookup(rec, e.order[r], koff, klen, vlen);
      if (FIXED) {
        loc = (first_tile ? 4 : 0) + (uint64_t)(j - 1) * e.rec_size;
        for (uint32_t b = 0; b < e.fixed_hdr_len; b++) en.hdr[b] = e.fixed_hdr[b];
        en.hdr_len = (uint8_t)e.fixed_hdr_len;
        en.src = koff;
        en.src_len = klen + vlen;
      } else {
        loc = (first_tile ? 4 : 0) + (e.rec_off[r] - e.rec_off[ps]) - body0;
        const bool last = (r + 1 == pe);
        const bool same_r = emit_is_repeat(e, r, ps);
        const bool same_prev = (r > ps) && emit_is_repeat(e, r - 1, ps);
        uint32_t h = 0;
        if (same_r) {
          if (!same_prev) en.hdr[h++] = 0xFE;  // RLE_MARKER
          int s = vint_size_u32(vlen);
          for (int b = 0; b < s; b++) en.hdr[h++] = vint_byte_u32(vlen, b);
          en.src = (rec.val_off && !rec.fixed) ? rec.val_off[e.order[r]] : koff + klen;
          en.src_len = vlen;
          en.tail_fd = last ? 1 : 0;
        } else {
          if (same_prev) en.hdr[h++] = 0xFD;   // V_END_MARKER
          int s = vint_size_u32(klen);
          for (int b = 0; b < s; b++) en.hdr[h++] = vint_byte_u32(klen, b);
          s = vint_size_u32(vlen);
          for (int b = 0; b < s; b++) en.hdr[h++] = vint_byte_u32(vlen, b);
          en.src = koff;
          if (rec.val_off && !rec.fixed) { en.src_len = klen; en.src2 = rec.val_off[e.order[r]]; en.src2_len = vlen; }
          else en.src_len = klen + vlen;
        }
        en.hdr_len = (uint8_t)h;
      }
    }
    s_ent[j] = en;
    s_loc[j] = loc;
    if (j == nr + 1) s_loc[nr + 2] = loc + en.hdr_len;
  }
  __syncthreads();

  const uint32_t nent = nr + 2;
  const uint64_t tile_bytes = s_loc[nent];
  const uint64_t abs0 = e.seg_start[p] + (first_tile ? 0 : 4 + body0);  // file offset of the tile's first byte
  const uint64_t seg_body_end = e.seg_start[p + 1] - 4;                  // file offset just past the EOF markers
  const uint8_t *kv_lo = rec.kv, *kv_hi = rec.kv + rec.kv_bytes;

  // ---- pieces of at most EMIT_IMG_BYTES (a single piece unless records are large)
  uint64_t done = 0;
  while (done < tile_bytes) {
    const uint64_t abs_piece = abs0 + done;
    const uint32_t lead = (uint32_t)(abs_piece & 15u);
    const uint32_t plen = (uint32_t)min((uint64_t)(EMIT_IMG_BYTES - lead), tile_bytes - done);
    const uint32_t nchunks = (lead + plen + 15u) >> 4;

    for (uint32_t c = tid; c < nchunks; c += EMIT_THREADS) {
      uint32_t acc[4] = {0, 0, 0, 0};
      // tile-relative byte range covered by this 16-byte vector
      uint64_t x0 = done + (c == 0 ? 0u : 16u * c - lead);
      const uint64_t x1 = min(done + (uint64_t)plen, done + (uint64_t)(16u * (c + 1) - lead));
      uint32_t q = (c == 0) ? lead : 0u;  // accumulator byte that receives x0
      // entry containing x0
      uint32_t j;
      if (FIXED) {
        uint64_t hdr = first_tile ? 4 : 0;
        j = x0 < hdr ? 0u : (uint32_t)min((uint64_t)nr, (x0 - hdr) / e.rec_size) + 1u;
        while (j + 1 < nent && s_loc[j + 1] <= x0) j++;
      } else {
        uint32_t lo = 0, hi = nent;  // last j with s_loc[j] <= x0
        while (hi - lo > 1) {
          uint32_t mid = (lo + hi) >> 1;
          if (s_loc[mid] <= x0) lo = mid; else hi = mid;
        }
        j = lo;
      }
      while (x0 < x1 && j < nent) {
        const uint64_t e_end = s_loc[j + 1];
        if (e_end <= x0) { j++; continue; }
        const uint64_t stop = min(x1, e_end);
        const EmitEntry &en = s_ent[j];
        uint32_t y = (uint32_t)(x0 - s_loc[j]);        // offset inside the entry
        uint32_t left = (uint32_t)(stop - x0);
        // framing bytes
        while (left && y < en.hdr_len) { put_byte(acc, q, en.hdr[y]); y++; q++; left--; }
        // source bytes
        if (left && y < en.hdr_len + en.src_len) {
          uint32_t take = min(left, en.hdr_len + en.src_len - y);
          merge_bytes(acc, kv_lo + en.src + (y - en.hdr_len), q, take, kv_lo, kv_hi);
          y += take; q += take; left -= take;
        }
        if (left && y < en.hdr_len + en.src_len + en.src2_len) {
          uint32_t take = min(left, en.hdr_len + en.src_len + en.src2_len - y);
          merge_bytes(acc, kv_lo + en.src2 + (y - en.hdr_len - en.src_len), q, take, kv_lo, kv_hi);
          y += take; q += take; left -= take;
        }
        if (left) { put_byte(acc, q, 0xFDu); q++; left--; }  // closing V_END_MARKER
        x0 = stop;
        j++;
      }
      *reinterpret_cast<uint4 *>(s_img + 16u * c) = make_uint4(acc[0], acc[1], acc[2], acc[3]);
    }
    __syncthreads();

    // ---- CRC of the body bytes of this piece (everything except the 4-byte segment header)
    uint32_t cb0 = lead, cb1 = lead + plen;  // image byte range that belongs to the checksummed body
    if (first_tile && done < 4) cb0 = min(cb1, lead + (uint32_t)(4 - done));
    {
      // words [wa, wb) are processed interleaved (thread t: wa+t, wa+t+T, ...); edge bytes by thread 0
      const uint32_t wa = (cb0 + 3u) >> 2, wb = cb1 >> 2;
      uint32_t c_thread = 0;
      uint32_t c_head = 0, n_tailbytes = 0;
      const uint32_t *img32 = reinterpret_cast<const uint32_t *>(s_img);
      if (wb > wa) {
        const uint32_t W = wb - wa;
        if ((uint32_t)tid < W) {
          uint32_t i = wa + tid;
          uint32_t c = 0;
          // all but the last word of this thread: c = (c ^ w) * x^(32*T)
          for (; i + EMIT_CRC_STRIDE_WORDS < wb; i += EMIT_CRC_STRIDE_WORDS) {
            uint32_t v = c ^ img32[i];
            c = s_adv[v & 0xFF] ^ s_adv[256 + ((v >> 8) & 0xFF)] ^ s_adv[512 + ((v >> 16) & 0xFF)] ^ s_adv[768 + (v >> 24)];
          }
          // last word: c = (c ^ w) * x^32, then align to the end of the word range
          uint32_t v = c ^ img32[i];
          c = s_tab[768 + (v & 0xFF)] ^ s_tab[512 + ((v >> 8) & 0xFF)] ^ s_tab[256 + ((v >> 16) & 0xFF)] ^ s_tab[v >> 24];
          uint32_t d = wb - 1 - i;  // whole words after this thread's last word (< T)
          if (d) c = crc_multmodp(c, e.crc->pow_word[d]);
          c_thread = c;
        }
        if (tid == 0) {
          // leading bytes [cb0, 4*wa): raw remainder with the standard pre-conditioning folded in below
          n_tailbytes = cb1 - 4 * wb;
        }
      }
      // block xor-reduce
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) c_thread ^= __shfl_xor_sync(0xffffffffu, c_thread, o);
      if ((tid & 31) == 0) s_red[tid >> 5] = c_thread;
      __syncthreads();
      if (tid == 0) {
        uint32_t words_crc = 0;
        for (int w = 0; w < EMIT_THREADS / 32; w++) words_crc ^= s_red[w];
        // raw (init 0, no final xor) remainder of [cb0, cb1): head bytes, words, tail bytes
        uint32_t raw = 0;
        uint32_t head_end = (wb > wa) ? 4 * wa : cb1;
        for (uint32_t b = cb0; b < head_end; b++) raw = s_tab[(raw ^ s_img[b]) & 0xFF] ^ (raw >> 8);
        if (wb > wa) {
          raw = crc_shift_bytes(e.crc, raw, 4ull * (wb - wa)) ^ words_crc;
          for (uint32_t b = 4 * wb; b < cb1; b++) raw = s_tab[(raw ^ s_img[b]) & 0xFF] ^ (raw >> 8);
        }
        (void)c_head; (void)n_tailbytes;
        // contribution to the segment's raw remainder: shift by the body bytes that follow this piece
        const uint32_t nbody = cb1 - cb0;
        if (nbody) {
          const uint64_t after = seg_body_end - (abs_piece + plen);
          uint32_t contrib = crc_shift_bytes(e.crc, raw, after);
          atomicXor(&e.seg_crc[p], contrib);
        }
      }
    }

    // ---- stream the image out: aligned 16-byte stores, byte stores on the ragged edges
    uint8_t *dst = e.out + (abs_piece - lead);
    for (uint32_t c = tid; c < nchunks; c += EMIT_THREADS) {
      uint32_t b0 = 16u * c, b1 = b0 + 16u;
      if (b0 >= lead && b1 <= lead + plen) {
        *reinterpret_cast<uint4 *>(dst + b0) = *reinterpret_cast<const uint4 *>(s_img + b0);
      } else {
        uint32_t a = max(b0, lead), b = min(b1, lead + plen);
        for (uint32_t x = a; x < b; x++) dst[x] = s_img[x];
      }
    }
    __syncthreads();
    done += plen;
  }
  }  // tiles
}

// writes the 4-byte big-endian checksum of every segment (and the constant 10-byte empty segments)
__global__ void k_finalize_segments(EmitParams e) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= e.P) return;
  uint64_t s0 = e.seg_start[p], s1 = e.seg_start[p + 1];
  if (s1 == s0) return;
  uint32_t cnt = e.part_start[p + 1] - e.part_start[p];
  uint8_t *o = e.out + s0;
  uint32_t crc;
  if (cnt == 0) {
    o[0] = 'T'; o[1] = 'I'; o[2] = 'F'; o[3] = 0; o[4] = 0xFF; o[5] = 0xFF;
    crc = 0xFFFF0000u;  // crc32(FF FF)
    o += 6;
  } else {
    crc = crc_from_raw(e.crc, e.seg_crc[p], s1 - s0 - 8);
    o += s1 - s0 - 4;
  }
  store_be32(o, crc);
}

}  // namespace tezgpu

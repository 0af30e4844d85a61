// merger.cuh -- reduce side of the hot path on sm_90a: k-way merge of sorted IFile segments.
// Device counterpart of TezMerger.MergeQueue (SORT/TezMerger.java:465-1065): segments are checksum-verified and
// parsed on the device, the union of their records is ordered with the same radix-sort + key-refinement machinery
// as the map side (a stable sort of already sorted runs IS their k-way merge: equal keys keep (segment, position)
// order), and the merged stream is either iterated (TezRawKeyValueIterator) or written as one IFile segment
// (TezMerger.writeFile, :215-245) with REPEAT_KEY run-length encoding of equal adjacent keys.
#pragma once
#include <algorithm>
#include <tuple>
#include <vector>

#include "sorter.cuh"
#include "parse_windows.cuh"

namespace tezgpu {

struct SegDesc {
  uint64_t off;       // offset of the segment in the staging buffer (16-byte aligned)
  uint64_t len;       // total bytes
  uint64_t body0;     // offset of the first body byte inside the segment (4 with header, 0 in-memory)
  uint64_t body_end;  // offset just past the EOF markers' possible position: len - 4 (checksum / slack excluded)
  uint32_t has_header;  // bit 0: 'TIF' header present; bit 1: checksum already verified by the transport (skip);
                        // bit 2: decoded image of a compressed segment (its trailer is not the body's checksum)
  uint32_t partition;
};
// tezgpu_segment.flags bit the codec path sets on the decoded images it hands to open() (never part of the ABI)
constexpr uint32_t SEG_DECODED = 1u << 31;

// ------------------------------------------------------------------------------------------------ checksum
// raw CRC remainder of 64 KiB pieces of the segment bodies, combined per segment by k_crc_combine
constexpr uint32_t CRC_PIECE = 64 * 1024;
constexpr int CRCV_THREADS = 256;

__global__ void __launch_bounds__(CRCV_THREADS)
    k_crc_pieces(const uint8_t *__restrict__ data, const SegDesc *__restrict__ segs, const uint32_t *__restrict__ piece_start,
                 uint32_t nseg, const CrcTables *__restrict__ t, TileCrc *__restrict__ out) {
  static_assert(CRCV_THREADS == EMIT_CRC_STRIDE_WORDS, "advc is built for this chunk interleave");
  __shared__ uint32_t s_tab[256], s_adv128[4 * 256], s_part[CRCV_THREADS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  s_tab[tid] = t->slice[0][tid];
  for (int i = tid; i < 4 * 256; i += CRCV_THREADS) s_adv128[i] = (&t->adv128[0][0])[i];
  // the two maps of the 16-byte-chunk interleave as warp-resident digit tables (crc32.cuh)
  CrcChunkFoldT<true> cf;
  cf.init(t, lane);
  const uint32_t piece = blockIdx.x;
  uint32_t lo = 0, hi = nseg;  // last segment with piece_start[s] <= piece
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (piece_start[mid] <= piece) lo = mid; else hi = mid;
  }
  const SegDesc sd = segs[lo];
  const uint64_t body_bytes = sd.body_end - sd.body0;
  const uint64_t a = (uint64_t)(piece - piece_start[lo]) * CRC_PIECE;
  const uint64_t b = min(body_bytes, a + CRC_PIECE);
  // piece = body bytes [a, b) seen as 16-byte chunks from the aligned-down address: bytes of the first chunk that
  // precede the piece are masked to zero (a remainder with zero initial value ignores leading zeros), the trailing
  // partial chunk is folded bytewise by lane 0.  Thread t owns the chunks whose distance from the last whole chunk is
  // == T-1-t (mod T): 3 x "next word" and one "skip to my next chunk" per chunk, partials aligned by a constant.
  const uint8_t *base = data + sd.off + sd.body0;
  const uint8_t *pa = base + a, *pb = base + b;
  const uint32_t mis = (uint32_t)((uintptr_t)pa & 15u);
  const uint4 *c16 = reinterpret_cast<const uint4 *>(pa - mis);
  const uint32_t Cn = (uint32_t)((pb - (pa - mis)) >> 4);  // whole chunks
  uint32_t c = 0;
  if (Cn) {
    const uint32_t iters = (Cn + CRCV_THREADS - 1) / CRCV_THREADS;
    const int32_t last_i = (int32_t)Cn - CRCV_THREADS + tid;
    int32_t i = last_i - (int32_t)(iters - 1) * CRCV_THREADS;
    for (uint32_t it = 0; it < iters; it++, i += CRCV_THREADS) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (i >= 0) {
        v = c16[i];
        if (i == 0 && mis) {
          uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (uint32_t k = 0; k < 4; k++) {
            if (mis >= 4 * k + 4) w[k] = 0;
            else if (mis > 4 * k) w[k] &= 0xFFFFFFFFu << (8u * (mis - 4 * k));
          }
          v = make_uint4(w[0], w[1], w[2], w[3]);
        }
      }
      c = cf.fold(c, v, it + 1 == iters);
    }
  }
  s_part[tid] = c;
  __syncthreads();
  if (warp == 0) {
    // lane l folds partials l, l+32, ... (Horner with x^(128*32)), aligns by x^(128*(31-l)), xor-reduce
    uint32_t q = 0;
#pragma unroll
    for (int k = 0; k < CRCV_THREADS / 32; k++) {
      q = s_adv128[q & 0xFF] ^ s_adv128[256 + ((q >> 8) & 0xFF)] ^ s_adv128[512 + ((q >> 16) & 0xFF)] ^ s_adv128[768 + (q >> 24)];
      q ^= s_part[lane + 32 * k];
    }
    q = crc_multmodp(q, cf.lane_pow);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q ^= __shfl_xor_sync(0xffffffffu, q, o);
    if (lane == 0) {
      uint32_t raw = q;
      const uint8_t *tail = Cn ? (pa - mis) + 16ull * Cn : pa;  // no whole chunk: everything bytewise
      for (const uint8_t *x = tail; x < pb; x++) raw = s_tab[(raw ^ *x) & 0xFF] ^ (raw >> 8);
      TileCrc tc;
      tc.raw = raw;
      tc.p = lo;
      tc.after = body_bytes - b;
      out[piece] = tc;
    }
  }
}

// verifyHeaderMagic + compressed flag (SORT/IFile.java:1004-1016): 1 = bad magic, 2 = compressed segment
__global__ void k_check_headers(const uint8_t *__restrict__ data, const SegDesc *__restrict__ segs, uint32_t nseg,
                                int *__restrict__ bad_magic, int *__restrict__ compressed) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const SegDesc sd = segs[s];
  if (!(sd.has_header & 1u)) return;
  const uint8_t *h = data + sd.off;
  if (!(h[0] == 'T' && h[1] == 'I' && h[2] == 'F')) atomicExch(bad_magic, (int)s + 1);
  else if (h[3] != 0) atomicExch(compressed, (int)s + 1);
}

// compares the folded remainder with the big-endian trailer (SORT/IFileInputStream.java:235-289)
__global__ void k_crc_check(const uint8_t *__restrict__ data, const SegDesc *__restrict__ segs, uint32_t nseg,
                            const uint32_t *__restrict__ seg_crc, const CrcTables *__restrict__ t, int *__restrict__ bad) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const SegDesc sd = segs[s];
  // in-memory segments carry no checksum stream (OG/InMemoryReader.java:142-254); segments the transport verified
  // while copying them (IFile.Reader.readToMemory, SORT/IFile.java:764-809) are not verified twice
  if (sd.has_header != 1u) return;
  if (crc_from_raw(t, seg_crc[s], sd.body_end - sd.body0) != load_be32(data + sd.off + sd.body_end)) atomicExch(bad, (int)s + 1);
}

// ------------------------------------------------------------------------------------------------ parse
// Walks the segments with IFile.Reader semantics, one warp per segment (warp_window_walk).  EMIT=false counts records,
// EMIT=true writes their metadata at rec_base[s]...
template <bool EMIT>
__global__ void __launch_bounds__(PARSE_WARPS * 32)
    k_parse_segments(const uint8_t *__restrict__ data, const SegDesc *__restrict__ segs, uint32_t nseg,
                     uint64_t *__restrict__ counts /*[nseg] records*/, uint64_t *__restrict__ kvbytes /*[nseg]*/,
                     const uint64_t *__restrict__ rec_base, ParseArrays out, int *__restrict__ bad) {
  __shared__ __align__(16) uint8_t s_win[PARSE_WARPS][PARSE_WIN];
  const int warp = threadIdx.x >> 5;
  const uint32_t s = blockIdx.x * PARSE_WARPS + warp;
  if (s >= nseg) return;
  const SegDesc sd = segs[s];
  uint64_t orig_koff = 0, orig_klen = 0, n = 0, bytes = 0;
  const uint64_t base = EMIT ? rec_base[s] : 0;
  const WalkEnd e = warp_window_walk(data + sd.off, sd.len, sd.body0, sd.body_end, s_win[warp], [&](const RecHdr &h) {
    uint64_t q = h.pos;
    if (h.kl != -2) {
      if (q + (uint64_t)h.kl > sd.body_end) return REC_BAD;
      orig_koff = q;
      orig_klen = (uint64_t)h.kl;
      q += (uint64_t)h.kl;
    } else if (n == 0) return REC_BAD;  // a repeat needs a previous key
    if (q + (uint64_t)h.vl > sd.body_end) return REC_BAD;
    if (EMIT) {
      // a repeated key points at the bytes of the last full key; its value bytes are not adjacent to it
      out.key_off[base + n] = sd.off + orig_koff;
      out.val_off[base + n] = sd.off + q;
      out.key_len[base + n] = (uint32_t)orig_klen;
      out.val_len[base + n] = (uint32_t)h.vl;
      out.tag[base + n] = (s << 1) | (h.kl == -2 ? 1u : 0u);
      out.partition[base + n] = (int32_t)sd.partition;
    }
    n++;
    bytes += orig_klen + (uint64_t)h.vl;
    return REC_OK;
  });
  if ((threadIdx.x & 31) == 0) {
    if (e.status != REC_EOF) atomicExch(bad, (int)s + 1);
    if (!EMIT) { counts[s] = n; kvbytes[s] = bytes; }
  }
}

// run-table mode -> explicit arrays (only when the record iterator or the run-length encoding emit needs them):
// every body is exactly n records of a known framing (checked by k_stage), so the metadata is pure arithmetic
__global__ void k_fill_fixed_arrays(const SegDesc *__restrict__ segs, uint32_t nseg, const uint64_t *__restrict__ rec_base,
                                    uint32_t klen, uint32_t vlen, uint32_t hdr_len, ParseArrays out) {
  const uint64_t total = rec_base[nseg];
  const uint32_t rs = hdr_len + klen + vlen;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = nseg;  // segment of record i
    while (hi - lo > 1) {
      uint32_t mid = (lo + hi) >> 1;
      if (rec_base[mid] <= i) lo = mid; else hi = mid;
    }
    const SegDesc sd = segs[lo];
    const uint64_t pos = sd.off + sd.body0 + (i - rec_base[lo]) * rs;
    out.key_off[i] = pos + hdr_len;
    out.val_off[i] = pos + hdr_len + klen;
    out.key_len[i] = klen;
    out.val_len[i] = vlen;
    out.tag[i] = lo << 1;
    out.partition[i] = (int32_t)sd.partition;
  }
}

// ------------------------------------------------------------------------------------------------ iterator batches
// kv_off[r] = sum of (klen + vlen) of the merged records before sorted position r
__global__ void __launch_bounds__(256) k_kv_sizes(Records rec, const uint32_t *__restrict__ order, uint32_t *__restrict__ sizes) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rec.n) return;
  uint32_t i = order[r];
  sizes[r] = rec.key_len[i] + rec.val_len[i];
}

// largest count <= max_records starting at `cursor` whose key+value bytes fit in cap
__global__ void k_find_batch(const uint64_t *__restrict__ kv_off, uint32_t n, uint32_t cursor, uint32_t max_records,
                             uint64_t cap, uint32_t *__restrict__ out_count) {
  uint32_t lo = 0, hi = min(max_records, n - cursor);
  const uint64_t base = kv_off[cursor];
  while (lo < hi) {
    uint32_t mid = lo + (hi - lo + 1) / 2;
    if (kv_off[cursor + mid] - base <= cap) lo = mid; else hi = mid - 1;
  }
  *out_count = lo;
}

// The record table of a batch, in the layout its consumer reads.  put() writes record w: its bytes start at o in the
// batch, key then value.
// tezgpu_merge_next_batch: 32-bit array of structs, copied to the caller's tezgpu_kv_index
struct KvIndexDev { uint32_t key_off, key_len, val_off, val_len, same_key; };
struct BatchIndexAos {
  KvIndexDev *idx;
  __device__ __forceinline__ void put(uint32_t w, uint64_t o, uint32_t kl, uint32_t vl, bool sk) const {
    KvIndexDev &e = idx[w];
    e.key_off = (uint32_t)o; e.key_len = kl; e.val_off = (uint32_t)(o + kl); e.val_len = vl; e.same_key = sk ? 1u : 0u;
  }
};
// tezgpu_merge_next_batch_device: struct of arrays with 64-bit offsets, the input triple of tezgpu_sorter_sort_device
struct BatchIndexSoa {
  uint64_t *key_off, *val_off;
  uint32_t *val_len;
  uint8_t *same_key;   // may be null
  __device__ __forceinline__ void put(uint32_t w, uint64_t o, uint32_t kl, uint32_t vl, bool sk) const {
    key_off[w] = o;
    val_off[w] = o + kl;
    val_len[w] = vl;
    if (same_key) same_key[w] = sk ? 1 : 0;
  }
};

constexpr int GATHER_THREADS = 256;

// the 16 bytes at p, any alignment, from the aligned 16-byte words that hold them (both hold bytes of [p, p + 16), so
// nothing is read from a word without a wanted byte)
__device__ __forceinline__ uint4 load16_any(const uint8_t *p) {
  const uintptr_t a = (uintptr_t)p & ~(uintptr_t)15;
  const uint32_t m = (uint32_t)((uintptr_t)p & 15u);
  const uint4 lo = *reinterpret_cast<const uint4 *>(a);
  if (m == 0) return lo;
  const uint4 hi = *reinterpret_cast<const uint4 *>(a + 16);
  const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  const uint32_t k = m >> 2, sh = 8 * (m & 3u);
  uint32_t s[5];
#pragma unroll
  for (int j = 0; j < 5; j++) s[j] = k == 0 ? w[j] : k == 1 ? w[j + 1] : k == 2 ? w[j + 2] : w[j + 3];
  return make_uint4(__funnelshift_r(s[0], s[1], sh), __funnelshift_r(s[1], s[2], sh), __funnelshift_r(s[2], s[3], sh),
                    __funnelshift_r(s[3], s[4], sh));
}

// len bytes src -> dst by the g lanes of a group (lane = rank in the group): the 16-byte words of dst that lie wholly
// inside the span as 16-byte stores, the bytes before and after them one by one.  Neighbouring records share the
// edge words, so no lane stores a byte outside its span.
__device__ __forceinline__ void gather_span(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, uint32_t len,
                                            uint32_t lane, uint32_t g) {
  const uint32_t head = min(len, (uint32_t)(-(uintptr_t)dst & 15u));
  const uint32_t words = (len - head) >> 4, tail = head + (words << 4);
  for (uint32_t b = lane; b < head; b += g) dst[b] = src[b];
  for (uint32_t b = tail + lane; b < len; b += g) dst[b] = src[b];
  uint4 *d16 = reinterpret_cast<uint4 *>(dst + head);
  const uint8_t *s = src + head;
  for (uint32_t q = lane; q < words; q += g) d16[q] = load16_any(s + 16ull * q);
}

// One batch of the record iterator: the record table, one thread per record, and the key then value bytes of every
// record packed back to back from out[0], 2^lanes_log2 lanes per record (the host sizes the group to the batch's mean
// record length, so short records do not leave most of a warp idle).  out must be 16-byte aligned.
template <typename Index>
__global__ void __launch_bounds__(GATHER_THREADS)
    k_gather_batch(Records rec, const uint32_t *__restrict__ order, const uint8_t *__restrict__ same,
                   const uint64_t *__restrict__ kv_off, uint32_t cursor, uint32_t count, uint8_t *__restrict__ out,
                   Index index, int check_same, uint32_t lanes_log2) {
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t base = kv_off[cursor];
  for (uint64_t w = tid; w < count; w += nthreads) {
    const uint32_t r = cursor + (uint32_t)w, i = order[r];
    // MergeQueue.isSameKey(): read as SAME_KEY from its segment, or (checkForSameKeys) equal to the previous key of
    // another segment
    bool sk = false;
    if (r > 0 && same[r]) {
      const uint32_t tag = rec.tag[i], tagp = rec.tag[order[r - 1]];
      sk = (tag & 1u) || (check_same && ((tag >> 1) != (tagp >> 1)));
    }
    index.put((uint32_t)w, kv_off[r] - base, rec.key_len[i], rec.val_len[i], sk);
  }
  const uint32_t g = 1u << lanes_log2, lane = (uint32_t)tid & (g - 1);
  for (uint64_t w = tid >> lanes_log2; w < count; w += nthreads >> lanes_log2) {
    const uint32_t r = cursor + (uint32_t)w, i = order[r];
    const uint64_t o = kv_off[r] - base;
    const uint32_t kl = rec.key_len[i], vl = rec.val_len[i];
    const uint8_t *k = rec.kv + rec.key_off[i];
    const uint8_t *v = rec.kv + (rec.val_off ? rec.val_off[i] : rec.key_off[i] + kl);
    gather_span(out + o, k, kl, lane, g);
    gather_span(out + o + kl, v, vl, lane, g);
  }
}

// ------------------------------------------------------------------------------------------------ host orchestration
// where a batch of the record iterator goes: host memory with the 32-bit index (idx set), or the caller's device
// buffers with the 64-bit table (idx null; same_key may be null); kv_bytes (may be null) receives the batch's bytes
struct BatchDest {
  uint8_t *kv;
  tezgpu_kv_index *idx;
  uint64_t *key_off, *val_off;
  uint32_t *val_len;
  uint8_t *same_key;
  uint64_t *kv_bytes;
};

class Merger {
 public:
  SortPipeline pipe;
  DeviceBuffer d_data, d_segs, d_piece_start, d_piece_crc, d_seg_crc, d_counts, d_rec_base;
  DeviceBuffer d_koff, d_voff, d_klen, d_vlen, d_tag, d_part, d_sizes, d_kvoff, d_batch, d_batch_idx, d_out;
  PinnedBuffer h_stage, h_out;
  std::vector<SegDesc> segs;
  uint64_t n = 0, kv_bytes = 0, seg_bytes = 0, cursor = 0;
  bool have_kvoff = false;
  int launches = 0;
  const uint8_t *data = nullptr;  // base of the segment bytes on the device

  static tezgpu_conf pipe_conf(tezgpu_conf c) {
    if (c.num_partitions < 1) c.num_partitions = 1;
    c.partitioner = TEZGPU_PART_GIVEN;
    if (c.num_partitions == 1) c.send_empty_partition_details = 0;  // a merge always writes its (possibly empty) segment
    c.fixed_key_len = c.fixed_val_len = 0;
    return c;
  }
  uint32_t fixed_klen = 0, fixed_vlen = 0;
  uint32_t data_slack = 32;

  explicit Merger(const tezgpu_conf &c) : pipe(pipe_conf(c)), fixed_klen(c.fixed_key_len), fixed_vlen(c.fixed_val_len) {}

  DeviceBuffer d_run_off, d_run_base, d_run_part, d_run_pseg, d_flags;
  std::vector<uint32_t> seg_orig;   // position in the partition-major list -> index in the caller's segment array
  bool arrays_ready = false;   // the per-record metadata arrays (d_koff ...) are filled (never in run-table mode unless asked)
  std::vector<uint64_t> h_counts, h_rec_base;

  // the host checks of a caller's segment, before any of its bytes is read
  void check_segment(const tezgpu_segment &sg) const {
    TG_CHECK(sg.data || sg.len == 0, TEZGPU_E_INVALID, "null segment");
    TG_CHECK(sg.len >= ((sg.flags & TEZGPU_SEG_HAS_HEADER) ? 10u : 6u), TEZGPU_E_FORMAT, "IFile segment shorter than an empty segment");
    TG_CHECK((int)sg.partition < pipe.conf.num_partitions, TEZGPU_E_INVALID, "segment partition out of range");
  }

  // ---- intake: builds the segment table (segs, d_segs) and launches the header and checksum checks, whose verdicts
  //      check_verdicts() reads.  Segments already on this device are used in place (no copy; kernels handle any byte
  //      alignment); host segments are staged contiguously with 16-byte aligned starts.
  void intake(const tezgpu_segment *in, uint32_t nseg) {
    cudaStream_t st = pipe.stream;
    arrays_ready = false;
    segs.resize(nseg);
    bool all_device = nseg > 0;
    for (uint32_t s = 0; s < nseg; s++) all_device &= (in[s].flags & TEZGPU_SEG_DEVICE) != 0;
    uint64_t off = 0;
    uintptr_t lo_addr = ~(uintptr_t)0, hi_addr = 0;
    if (all_device)
      for (uint32_t s = 0; s < nseg; s++) {
        lo_addr = std::min(lo_addr, (uintptr_t)in[s].data);
        hi_addr = std::max(hi_addr, (uintptr_t)in[s].data + in[s].len);
      }
    lo_addr &= ~(uintptr_t)15;
    bool any_header = false;
    // Segments are kept partition-major (stable: the caller's order inside a partition is the merge's tie order): the
    // records of one output partition then live in a handful of consecutive runs, which makes the run-table lookups of
    // the stage / emit kernels a scan over <= G entries instead of a binary search over all segments.
    seg_orig.resize(nseg);
    for (uint32_t s = 0; s < nseg; s++) seg_orig[s] = s;
    if (pipe.conf.num_partitions > 1)
      std::stable_sort(seg_orig.begin(), seg_orig.end(), [&](uint32_t a, uint32_t b) { return in[a].partition < in[b].partition; });
    for (uint32_t s = 0; s < nseg; s++) {
      const tezgpu_segment &sg = in[seg_orig[s]];
      check_segment(sg);
      const bool hdr = sg.flags & TEZGPU_SEG_HAS_HEADER;
      any_header |= hdr;
      segs[s].off = all_device ? (uint64_t)((uintptr_t)sg.data - lo_addr) : off;
      segs[s].len = sg.len;
      segs[s].body0 = hdr ? 4 : 0;
      segs[s].body_end = sg.len - 4;
      segs[s].has_header = (hdr ? 1u : 0u) | ((hdr && (sg.flags & TEZGPU_SEG_VERIFIED)) ? 2u : 0u) |
                           ((hdr && (sg.flags & SEG_DECODED)) ? 4u : 0u);
      segs[s].partition = sg.partition;
      off = align_up(off + sg.len, 16);
    }
    if (all_device) {
      data = reinterpret_cast<const uint8_t *>(lo_addr);
      seg_bytes = (uint64_t)(hi_addr - lo_addr);
      data_slack = 0;  // caller's buffer: never read past its end
    } else {
      seg_bytes = off;
      d_data.ensure(off + 64);
      for (uint32_t s = 0; s < nseg; s++) {
        const tezgpu_segment &sg = in[seg_orig[s]];
        if (!sg.len) continue;
        const bool dev = sg.flags & TEZGPU_SEG_DEVICE;
        TG_CUDA(cudaMemcpyAsync(d_data.as<uint8_t>() + segs[s].off, sg.data, sg.len,
                                dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
      }
      data = d_data.as<uint8_t>();
      data_slack = 32;
    }
    d_segs.ensure((size_t)(nseg ? nseg : 1) * sizeof(SegDesc));
    if (nseg) TG_CUDA(cudaMemcpyAsync(d_segs.p, segs.data(), (size_t)nseg * sizeof(SegDesc), cudaMemcpyHostToDevice, st));
    // verdict words of the header / checksum checks: [0] bad magic, [1] compressed, [2] checksum mismatch (segment + 1).
    // They live outside the sorter's scratch so the whole fixed-framing path needs no host round trip before the sort.
    d_flags.ensure(64);
    TG_CUDA(cudaMemsetAsync(d_flags.p, 0, 64, st));
    int *d_vflags = d_flags.as<int>();
    if (nseg) {
      if (any_header) {
        k_check_headers<<<(uint32_t)div_up(nseg, 128), 128, 0, st>>>(data, d_segs.as<SegDesc>(), nseg, d_vflags, d_vflags + 1);
        launches++;
      }
      // ---- checksums of the segments nobody verified yet; a concatenation also needs the body remainder of every
      //      segment whose trailer is no checksum it can trust (in-memory segments, decoded images)
      std::vector<uint32_t> piece_start;
      launches += check_checksums(data, segs, d_segs.as<SegDesc>(), [&](const SegDesc &sd) {
        return sd.has_header == 1u || (concat && (!(sd.has_header & 2u) || (sd.has_header & 4u)));
      }, piece_start, true, d_vflags + 2);
    }
  }

  // waits for the verdict words and throws the first one set
  void check_verdicts() {
    cudaStream_t st = pipe.stream;
    int f[4] = {0, 0, 0, 0};
    TG_CUDA(cudaMemcpyAsync(f, d_flags.p, 16, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    TG_CHECK(f[0] == 0, TEZGPU_E_FORMAT, "Not a valid ifile header (segment " + std::to_string(f[0] ? seg_orig[f[0] - 1] : 0) + ")");
    TG_CHECK(f[1] == 0, TEZGPU_E_UNSUPPORTED, "compressed IFile segments are not supported on the device path");
    TG_CHECK(f[2] == 0, TEZGPU_E_FORMAT, "IFile checksum mismatch in segment " + std::to_string(f[2] ? seg_orig[f[2] - 1] : 0));
    TG_CHECK(f[3] == 0, TEZGPU_E_FORMAT, "IFile segment " + std::to_string(f[3] ? seg_orig[f[3] - 1] : 0) + " does not end in the EOF marker");
  }

  void open(const tezgpu_segment *in, uint32_t nseg) {
    intake(in, nseg);
    if (concat) {
      // tezgpu_concat_open: nothing is parsed or sorted here (concat.cuh)
      concat_inputs(nseg, d_flags.as<int>() + 3);
      check_verdicts();
      return;
    }
    // ---- merge = stable sort of the union of the runs by the RawComparator
    bool sorted = false;
    if (count_fixed_records(nseg, FRAMING_MAX_LEN)) {
      // ---- run-table mode: offsets are arithmetic, the stage kernel checks the framing bytes it passes over anyway.
      //      No per-record arrays, no host round trip before the sort's own.
      pipe.merge_inputs_plain = true;
      try {
        pipe.sort_phase(run_table_records(nseg));
        sorted = true;
      } catch (const FramingMismatch &) {
        // not the fixed framing after all (e.g. run-length encoded input): take the general walk
      }
    }
    check_verdicts();  // also: the caller's host buffers may go away after open()
    if (sorted) {
      parse_mode = 0;
      parse_rounds = 0;
    } else {
      find_records_general(nseg);
      pipe.merge_inputs_plain = false;
      pipe.sort_phase(array_records());
    }
    launches += pipe.state.launches;
    cursor = 0;
    have_kvoff = false;
  }

  // Checksums of the segments `need` selects (open() and open_codec()): segment_remainders, then the trailers are
  // compared; a mismatch writes segment + 1 to *d_bad.  Returns the launches.
  template <typename Need>
  int check_checksums(const uint8_t *bytes, const std::vector<SegDesc> &sd, const SegDesc *d_sd, Need need,
                      std::vector<uint32_t> &piece_start, bool sync_copy, int *d_bad) {
    const int launches = segment_remainders(bytes, sd, d_sd, need, piece_start, sync_copy);
    if (!launches) return 0;
    const uint32_t nseg = (uint32_t)sd.size();
    k_crc_check<<<(uint32_t)div_up(nseg, 128), 128, 0, pipe.stream>>>(bytes, d_sd, nseg, d_seg_crc.as<uint32_t>(),
                                                                      DeviceConstants::get(pipe.conf.device).d_crc, d_bad);
    TG_CUDA(cudaGetLastError());
    return launches + 1;
  }

  // Raw CRC remainders of the bodies of the segments `need` selects, from 64 KiB pieces, folded per segment into
  // d_seg_crc (0 for the others).  piece_start receives the host piece table, which must live until the stream has
  // copied it: sync_copy waits for the copy here, otherwise the caller keeps the table until its next synchronise.
  // Returns the launches (none when no segment is selected: d_seg_crc is then left alone).
  template <typename Need>
  int segment_remainders(const uint8_t *bytes, const std::vector<SegDesc> &sd, const SegDesc *d_sd, Need need,
                         std::vector<uint32_t> &piece_start, bool sync_copy) {
    cudaStream_t st = pipe.stream;
    const uint32_t nseg = (uint32_t)sd.size();
    piece_start.resize(nseg + 1);
    uint32_t np = 0;
    for (uint32_t s = 0; s < nseg; s++) {
      piece_start[s] = np;
      if (need(sd[s])) np += (uint32_t)div_up(sd[s].body_end - sd[s].body0, CRC_PIECE);
    }
    piece_start[nseg] = np;
    if (!np) return 0;
    const CrcTables *d_crc = DeviceConstants::get(pipe.conf.device).d_crc;
    d_piece_start.ensure((size_t)(nseg + 1) * 4);
    TG_CUDA(cudaMemcpyAsync(d_piece_start.p, piece_start.data(), (size_t)(nseg + 1) * 4, cudaMemcpyHostToDevice, st));
    if (sync_copy) TG_CUDA(cudaStreamSynchronize(st));
    d_piece_crc.ensure((size_t)np * sizeof(TileCrc));
    d_seg_crc.ensure((size_t)nseg * 4);
    TG_CUDA(cudaMemsetAsync(d_seg_crc.p, 0, (size_t)nseg * 4, st));
    k_crc_pieces<<<np, CRCV_THREADS, 0, st>>>(bytes, d_sd, d_piece_start.as<uint32_t>(), nseg, d_crc, d_piece_crc.as<TileCrc>());
    k_crc_combine<<<(uint32_t)div_up(np, 256), 256, 0, st>>>(d_piece_crc.as<TileCrc>(), np, d_crc, d_seg_crc.as<uint32_t>());
    TG_CUDA(cudaGetLastError());
    return 2;
  }

  // ---- record finding, shared by open() and concat_parse().  Run-table candidate: every body is exactly k records of
  //      the fixed framing (at most max_len bytes) + EOF markers.  Fills h_counts / h_rec_base, n and kv_bytes when it
  //      holds and returns whether it does.
  bool count_fixed_records(uint32_t nseg, uint32_t max_len) {
    h_counts.assign(2 * (size_t)nseg + 2, 0);
    h_rec_base.assign(nseg + 1, 0);
    n = kv_bytes = 0;
    const FixedFraming f = fixed_framing(fixed_klen, fixed_vlen);
    if (!nseg || fixed_klen + fixed_vlen == 0 || f.len > max_len) return false;
    for (uint32_t s = 0; s < nseg; s++) {
      const uint64_t body = segs[s].body_end - segs[s].body0;
      if (body < 2 || (body - 2) % f.rec_size) return false;
      h_counts[s] = (body - 2) / f.rec_size;
      h_counts[nseg + s] = h_counts[s] * (fixed_klen + fixed_vlen);
    }
    set_record_bases(nseg);
    return true;
  }

  // h_counts = the records of every segment, then their key + value bytes -> h_rec_base, n and kv_bytes (the window
  // parser sums the key + value bytes on the device and sets kv_bytes afterwards)
  void set_record_bases(uint32_t nseg) {
    n = kv_bytes = 0;
    for (uint32_t s = 0; s < nseg; s++) { h_rec_base[s] = n; n += h_counts[s]; kv_bytes += h_counts[nseg + s]; }
    h_rec_base[nseg] = n;
    TG_CHECK(n <= RADIX_MAX_N, TEZGPU_E_INVALID, "more than 2^30-1 records in one merge");
  }

  // general path: walk the segments (IFile.Reader semantics), materialise the per-record metadata
  void find_records_general(uint32_t nseg) {
    TG_CUDA(cudaMemsetAsync(pipe.small.p, 0, SORT_SCRATCH_BYTES, pipe.stream));
    d_counts.ensure((size_t)(nseg + 1) * 16);
    d_rec_base.ensure((size_t)(nseg + 2) * 8);
    n = 0;
    kv_bytes = 0;
    if (nseg) open_general_reparse(nseg);
    else record_arrays(0);
    TG_CUDA(cudaGetLastError());
    arrays_ready = true;
  }

  // the per-record metadata arrays, sized for nrec records
  ParseArrays record_arrays(uint64_t nrec) {
    const size_t m = (size_t)(nrec ? nrec : 1);
    d_koff.ensure(m * 8); d_voff.ensure(m * 8);
    d_klen.ensure(m * 4); d_vlen.ensure(m * 4); d_tag.ensure(m * 4); d_part.ensure(m * 4);
    return {d_koff.as<uint64_t>(), d_voff.as<uint64_t>(), d_klen.as<uint32_t>(), d_vlen.as<uint32_t>(), d_tag.as<uint32_t>(), d_part.as<int32_t>()};
  }

  // Records over the materialised per-record arrays
  Records array_records() {
    Records r;
    memset(&r, 0, sizeof(r));
    r.kv = data;
    r.kv_bytes = data_slack ? align_up(seg_bytes, 16) + data_slack : seg_bytes;
    r.key_off = d_koff.as<uint64_t>();
    r.val_off = d_voff.as<uint64_t>();
    r.key_len = d_klen.as<uint32_t>();
    r.val_len = d_vlen.as<uint32_t>();
    r.tag = d_tag.as<uint32_t>();
    r.partition = pipe.conf.num_partitions > 1 ? d_part.as<int32_t>() : nullptr;
    r.n = (uint32_t)n;
    r.fixed = 0;
    return r;
  }

  // Records over the run table of the fixed framing (uploaded here): no per-record arrays
  Records run_table_records(uint32_t nseg) {
    cudaStream_t st = pipe.stream;
    std::vector<uint64_t> roff(nseg);
    std::vector<uint32_t> rbase(nseg + 1), rpart(nseg);
    for (uint32_t s = 0; s < nseg; s++) { roff[s] = segs[s].off + segs[s].body0; rbase[s] = (uint32_t)h_rec_base[s]; rpart[s] = segs[s].partition; }
    rbase[nseg] = (uint32_t)n;
    const int P = pipe.conf.num_partitions;
    std::vector<uint32_t> pseg((size_t)P + 1, 0);
    for (uint32_t s = 0; s < nseg; s++) pseg[segs[s].partition + 1]++;
    for (int p = 0; p < P; p++) pseg[p + 1] += pseg[p];
    d_run_pseg.ensure(((size_t)P + 1) * 4);
    TG_CUDA(cudaMemcpyAsync(d_run_pseg.p, pseg.data(), ((size_t)P + 1) * 4, cudaMemcpyHostToDevice, st));
    d_run_off.ensure((size_t)nseg * 8); d_run_base.ensure((size_t)(nseg + 1) * 4); d_run_part.ensure((size_t)nseg * 4);
    TG_CUDA(cudaMemcpyAsync(d_run_off.p, roff.data(), (size_t)nseg * 8, cudaMemcpyHostToDevice, st));
    TG_CUDA(cudaMemcpyAsync(d_run_base.p, rbase.data(), (size_t)(nseg + 1) * 4, cudaMemcpyHostToDevice, st));
    TG_CUDA(cudaMemcpyAsync(d_run_part.p, rpart.data(), (size_t)nseg * 4, cudaMemcpyHostToDevice, st));
    TG_CUDA(cudaStreamSynchronize(st));  // stack-lifetime staging vectors (and: the caller's host segments may go away)
    const FixedFraming f = fixed_framing(fixed_klen, fixed_vlen);
    Records r;
    memset(&r, 0, sizeof(r));
    r.kv = data;
    r.kv_bytes = data_slack ? align_up(seg_bytes, 16) + data_slack : seg_bytes;
    r.n = (uint32_t)n;
    r.fixed = 1;
    r.klen = fixed_klen;
    r.vlen = fixed_vlen;
    r.use_runs = 1;
    r.runs.seg_off = d_run_off.as<uint64_t>();
    r.runs.rec_base = d_run_base.as<uint32_t>();
    r.runs.seg_part = d_run_part.as<uint32_t>();
    r.runs.part_seg0 = d_run_pseg.as<uint32_t>();
    r.runs.nseg = nseg;
    r.runs.rec_size = f.rec_size;
    r.runs.hdr_len = f.len;
    r.runs.hdr_bytes[0] = f.packed(0);
    r.runs.hdr_bytes[1] = f.packed(1);
    return r;
  }

  // blocks of the grid-stride kernels over the records
  uint32_t record_grid() const { return (uint32_t)std::min<uint64_t>(div_up(n, 256), (uint64_t)pipe.num_sms * 16); }

  // the per-record arrays of the fixed framing, in the run table's record numbering (h_rec_base).  Returns the launches.
  int fill_fixed_arrays() {
    const uint32_t nseg = (uint32_t)segs.size();
    d_rec_base.ensure((size_t)(nseg + 2) * 8);
    TG_CUDA(cudaMemcpyAsync(d_rec_base.p, h_rec_base.data(), (size_t)(nseg + 1) * 8, cudaMemcpyHostToDevice, pipe.stream));
    const ParseArrays pa = record_arrays(n);
    if (!n) return 0;
    k_fill_fixed_arrays<<<record_grid(), 256, 0, pipe.stream>>>(d_segs.as<SegDesc>(), nseg, d_rec_base.as<uint64_t>(), fixed_klen,
                                                                fixed_vlen, fixed_framing(fixed_klen, fixed_vlen).len, pa);
    TG_CUDA(cudaGetLastError());
    return 1;
  }

  // run-table mode keeps no per-record arrays; the record iterator and the general (run-length encoding) emit need
  // them: fill them now (same record numbering, so the sorted order stays valid) and switch the sorter's view over
  void ensure_arrays() {
    if (arrays_ready) return;
    launches += fill_fixed_arrays();
    Records r = array_records();
    r.fixed = 1;
    r.klen = fixed_klen;
    r.vlen = fixed_vlen;
    const Records &sorted = pipe.state.rec;   // the comparator and partitioning the sort ran with
    std::tie(r.cmp, r.hash_partition, r.num_partitions, r.pbits) = std::tie(sorted.cmp, sorted.hash_partition, sorted.num_partitions, sorted.pbits);
    pipe.state.rec = r;
    // the record view changed (explicit offsets instead of the run table): the emit must lay its tiles out again --
    // tile sizes depend on the kernel that serves the view (set_fixed_layout)
    pipe.state.spec_layout = false;
    arrays_ready = true;
  }

  // ---- parallel parser (parse_windows.cuh): every window of every segment walks at once, entries iterate to the fixed
  // point.  Returns false when the rounds cap is hit (adversarial bytes): the caller falls back to the sequential walker.
  DeviceBuffer d_pwseg, d_entry[2], d_wcount, d_wbase, d_wlast, d_carry, d_pwflags;
  int parse_rounds = 0;
  int parse_mode = 0;   // how the last open() found the records: 0 fixed framing (run table), 1 window parser, 2 sequential walker
  bool parse_parallel(uint32_t nseg) {
    cudaStream_t st = pipe.stream;
    std::vector<PwSeg> ps(nseg);
    uint64_t nw = 0;
    for (uint32_t s = 0; s < nseg; s++) {
      ps[s].off = segs[s].off; ps[s].len = segs[s].len; ps[s].body0 = segs[s].body0; ps[s].body_end = segs[s].body_end;
      ps[s].win0 = (uint32_t)nw;
      ps[s].nwin = (uint32_t)std::max<uint64_t>(1, div_up(segs[s].body_end - segs[s].body0, PW_WINDOW));
      ps[s].partition = segs[s].partition;
      ps[s].pad = 0;
      nw += ps[s].nwin;
    }
    TG_CHECK(nw < (1ull << 31), TEZGPU_E_INVALID, "segments too large for one merge");
    const uint32_t nwin = (uint32_t)nw;
    d_pwseg.ensure((size_t)nseg * sizeof(PwSeg));
    for (int b = 0; b < 2; b++) d_entry[b].ensure((size_t)nwin * 8);
    d_wcount.ensure((size_t)nwin * 4);
    d_wbase.ensure(((size_t)nwin + 2) * 8);
    d_wlast.ensure((size_t)nwin * 16);
    d_pwflags.ensure(64);
    TG_CUDA(cudaMemcpyAsync(d_pwseg.p, ps.data(), (size_t)nseg * sizeof(PwSeg), cudaMemcpyHostToDevice, st));
    const uint32_t grid = (uint32_t)div_up(nwin, PW_THREADS);
    ParseArrays none{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    // guess -> evaluate from the guessed entries -> chase the true chain (parse_windows.cuh); one host round trip
    TG_CUDA(cudaMemsetAsync(d_pwflags.p, 0, 64, st));
    PwFixedHint hint{0, 0, 0, 0};
    const FixedFraming f = fixed_framing(fixed_klen, fixed_vlen);
    if (fixed_klen + fixed_vlen > 0 && f.len <= 7) {
      const uint32_t vl = (uint32_t)vint_size_u32(fixed_vlen);   // the framing ends in vint(vlen)
      hint = PwFixedHint{f.packed(), f.packed() >> (8 * (f.len - vl)), f.len, vl};
    }
    k_parse_guess<<<(uint32_t)div_up((uint64_t)nwin * 32, PW_GUESS_THREADS), PW_GUESS_THREADS, 0, st>>>(data, d_pwseg.as<PwSeg>(), nseg, nwin,
                                                                                                        d_entry[0].as<uint64_t>(), hint);
    k_parse_windows<1><<<grid, PW_THREADS, 0, st>>>(data, d_pwseg.as<PwSeg>(), nseg, nwin, d_entry[0].as<uint64_t>(),
                                                    d_entry[1].as<uint64_t>(), d_wcount.as<uint32_t>(), d_wlast.as<uint64_t>(),
                                                    nullptr, d_pwflags.as<int>(), nullptr, nullptr, none);
    k_parse_chase<<<(uint32_t)div_up(nseg, PW_CHASE_WARPS), 32 * PW_CHASE_WARPS, 0, st>>>(
        data, d_pwseg.as<PwSeg>(), nseg, d_entry[0].as<uint64_t>(), d_entry[1].as<uint64_t>(), d_wcount.as<uint32_t>(),
        d_wlast.as<uint64_t>(), d_pwflags.as<int>());
    launches += 3;
    TG_CUDA(cudaGetLastError());
    int flags[4] = {0, 0, 0, 0};
    TG_CUDA(cudaMemcpyAsync(flags, d_pwflags.p, 16, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    parse_rounds = flags[2];   // windows the chase had to walk by hand
    // the sequential reader would reject a segment (or it ends early): the sequential walker reports it
    if (flags[1]) return false;
    const int cur = 0;         // d_entry[0] now holds the true entries
    // ---- record offsets of every window, totals
    launches += scan_u32_exclusive(st, pipe.blk, d_wcount.as<uint32_t>(), nwin, d_wbase.as<uint64_t>());
    d_counts.ensure((size_t)(nseg + 1) * 16);
    k_parse_seg_counts<<<(uint32_t)div_up(nseg, 128), 128, 0, st>>>(d_pwseg.as<PwSeg>(), nseg, d_wbase.as<uint64_t>(), d_counts.as<uint64_t>());
    launches++;
    TG_CUDA(cudaMemcpyAsync(h_counts.data(), d_counts.p, (size_t)nseg * 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    set_record_bases(nseg);
    const ParseArrays pa = record_arrays(n);
    d_carry.ensure((size_t)nwin * 16);
    k_parse_carry<<<grid, PW_THREADS, 0, st>>>(d_pwseg.as<PwSeg>(), nseg, nwin, d_entry[cur].as<uint64_t>(), d_wlast.as<uint64_t>(), d_carry.as<uint64_t>());
    const uint64_t *carry = d_carry.as<uint64_t>();
    launches++;
    TG_CUDA(cudaMemsetAsync(d_pwflags.p, 0, 64, st));
    unsigned long long *d_kv_total = reinterpret_cast<unsigned long long *>(d_pwflags.as<int>() + 8);
    k_parse_windows<2><<<(uint32_t)div_up((uint64_t)nwin * PW_EMIT_GROUP, PW_THREADS), PW_THREADS, 0, st>>>(data, d_pwseg.as<PwSeg>(), nseg, nwin, d_entry[cur].as<uint64_t>(), nullptr, nullptr, nullptr,
                                                       d_kv_total, d_pwflags.as<int>(), d_wbase.as<uint64_t>(), carry, pa);
    launches++;
    TG_CUDA(cudaGetLastError());
    unsigned long long kvb = 0;
    TG_CUDA(cudaMemcpyAsync(flags, d_pwflags.p, 16, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaMemcpyAsync(&kvb, d_kv_total, 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    TG_CHECK(flags[1] == 0, TEZGPU_E_FORMAT, "malformed IFile segment " + std::to_string(flags[1] ? seg_orig[flags[1] - 1] : 0));
    kv_bytes = kvb;
    return true;
  }

  void open_general_reparse(uint32_t nseg) {
    cudaStream_t st = pipe.stream;
    static const bool serial_only = getenv("TEZGPU_PARSE_SERIAL") && atoi(getenv("TEZGPU_PARSE_SERIAL")) != 0;
    parse_mode = 1;
    if (!serial_only && parse_parallel(nseg)) return;
    parse_mode = 2;
    int *d_bad = &pipe.d_scratch()->verdict.error;
    ParseArrays pa{nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    k_parse_segments<false><<<(uint32_t)div_up(nseg, PARSE_WARPS), PARSE_WARPS * 32, 0, st>>>(data, d_segs.as<SegDesc>(), nseg, d_counts.as<uint64_t>(),
                                                                     d_counts.as<uint64_t>() + nseg, nullptr, pa, d_bad);
    int bad = 0;
    TG_CUDA(cudaMemcpyAsync(h_counts.data(), d_counts.p, (size_t)nseg * 16, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    TG_CHECK(bad == 0, TEZGPU_E_FORMAT, "malformed IFile segment " + std::to_string(bad ? seg_orig[bad - 1] : 0));
    set_record_bases(nseg);
    TG_CUDA(cudaMemcpyAsync(d_rec_base.p, h_rec_base.data(), (size_t)(nseg + 1) * 8, cudaMemcpyHostToDevice, st));
    pa = record_arrays(n);
    if (n) k_parse_segments<true><<<(uint32_t)div_up(nseg, PARSE_WARPS), PARSE_WARPS * 32, 0, st>>>(data, d_segs.as<SegDesc>(), nseg, nullptr, nullptr,
                                                                            d_rec_base.as<uint64_t>(), pa, d_bad);
    launches += 2;
  }

  // ---- concatenation (tezgpu_concat_open, concat.cuh): records leave in (segment, position) order.  The write copies
  // the record bytes of every input as they are; next_batch parses them on its first call.
  bool concat = false, concat_parsed = false;
  uint64_t concat_bytes = 0;              // sum of the input bodies (records + EOF markers)
  std::vector<uint64_t> cat_rec;          // record bytes of every segment (partition-major, as segs)
  DeviceBuffer d_cat_tc, d_cat_units, d_cat_parts, d_order;
  void concat_inputs(uint32_t nseg, int *d_bad_eof);
  void concat_write(uint8_t *d_out_buf, uint64_t cap, int writer_rle, uint64_t *out_len, int64_t *index, tezgpu_stats *stats);
  void concat_parse();

  uint64_t raw_output_bound() const {
    if (concat) return concat_bytes + 10ull * pipe.conf.num_partitions + 64;
    return SortPipeline::output_bound(n, kv_bytes, pipe.conf.num_partitions) + 16;
  }
  uint64_t output_bound() const {
    return pipe.codec ? SortPipeline::codec_bound(pipe.codec, raw_output_bound(), pipe.conf.num_partitions) : raw_output_bound();
  }

  // ---- codec (codec.cuh): compressed segments are checked, decompressed into z_img and merged as ordinary segments
  DeviceBuffer z_in, z_img, z_insegs, z_status, z_descs, z_flag;
  DeviceBuffer z_nblk, z_base, z_blks, z_slow;   // LZ4 / zstd: blocks (frames) per segment, their first index, the units, serial-path flags
  std::vector<uint64_t> z_img_off;                // image of the i-th decoded segment: z_img + z_img_off[i]
  void open_codec(const tezgpu_segment *in, const int64_t *raw_len, uint32_t nseg);
  void decode_compressed(const tezgpu_segment *in, const int64_t *raw_len, const std::vector<uint32_t> &zs);
  void decode_to_host(const tezgpu_segment *in, const int64_t *raw_len, uint32_t nseg, uint64_t base, uint64_t budget,
                      uint8_t *const *out);

  // the writer behind every write_*: TezMerger.writeFile semantics per partition, or -- with a combiner -- the combined
  // records, which carry no segment tags and unique keys (merge mode and the plain writer then write the same bytes)
  void write_device(uint8_t *d_out_buf, uint64_t cap, int writer_rle, uint64_t *out_len, int64_t *index, tezgpu_stats *stats) {
    tezgpu_stats st;
    if (concat) {
      concat_write(d_out_buf, cap, writer_rle, out_len, index, &st);
    } else {
      pipe.emit_out(writer_rle ? 1 : 0, true, raw_output_bound(), d_out_buf, cap, out_len, index, &st);
      st.output_bytes = (int64_t)kv_bytes;
      st.kernel_launches += launches - pipe.state.launches;
    }
    if (stats) *stats = st;
  }

  // where a write into host memory lands: the caller's buffer, which must hold len bytes, or h_out
  uint8_t *host_out(uint8_t *out, uint64_t cap, uint64_t len) {
    if (!out) {
      h_out.ensure(len + 16);
      return h_out.as<uint8_t>();
    }
    TG_CHECK(len <= cap, TEZGPU_E_NOMEM, "output buffer too small for the merged segment");
    return out;
  }

  // write_device into d_out, then one copy into host memory (host_out); returns where the *len bytes are
  const uint8_t *write_host(int writer_rle, uint8_t *out, uint64_t cap, uint64_t *len, int64_t *index, tezgpu_stats *stats) {
    d_out.ensure(output_bound());
    write_device(d_out.as<uint8_t>(), d_out.cap, writer_rle, len, index, stats);
    uint8_t *host = host_out(out, cap, *len);
    if (*len) {
      TG_CUDA(cudaMemcpyAsync(host, d_out.p, *len, cudaMemcpyDeviceToHost, pipe.stream));
      TG_CUDA(cudaStreamSynchronize(pipe.stream));
    }
    return host;
  }

  void ensure_kvoff() {
    if (have_kvoff) return;
    ensure_arrays();
    cudaStream_t st = pipe.stream;
    const uint32_t nn = (uint32_t)n;
    d_sizes.ensure((size_t)(nn ? nn : 1) * 4);
    d_kvoff.ensure(((size_t)nn + 2) * 8);
    if (nn) {
      k_kv_sizes<<<(uint32_t)div_up(nn, 256), 256, 0, st>>>(pipe.state.rec, pipe.state.order, d_sizes.as<uint32_t>());
      scan_u32_exclusive(st, pipe.blk, d_sizes.as<uint32_t>(), nn, d_kvoff.as<uint64_t>());
      TG_CUDA(cudaGetLastError());
    } else {
      TG_CUDA(cudaMemsetAsync(d_kvoff.p, 0, 16, st));
    }
    have_kvoff = true;
  }

  // next()/getKey()/getValue()/isSameKey() in batches, into host memory (idx != null: tezgpu_merge_next_batch) or into
  // the caller's device buffers (dev: tezgpu_merge_next_batch_device, whose *kv_bytes receives the batch's bytes)
  void next_batch(const BatchDest &d, uint64_t cap, uint32_t idx_cap, uint32_t *count) {
    cudaStream_t st = pipe.stream;
    *count = 0;
    if (d.kv_bytes) *d.kv_bytes = 0;
    TG_CHECK(!pipe.combiner, TEZGPU_E_STATE, "a merger with a combiner has no record iterator: use tezgpu_merge_write_*");
    if (concat) concat_parse();
    if (cursor >= n || idx_cap == 0) return;
    ensure_kvoff();
    if (d.idx) cap = std::min<uint64_t>(cap, 0xFFFFFFFFull);   // tezgpu_kv_index offsets are 32-bit
    uint32_t *d_cnt = &pipe.d_scratch()->verdict.batch_count;
    k_find_batch<<<1, 1, 0, st>>>(d_kvoff.as<uint64_t>(), (uint32_t)n, (uint32_t)cursor, idx_cap, cap, d_cnt);
    uint32_t cnt = 0;
    TG_CUDA(cudaMemcpyAsync(&cnt, d_cnt, 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    if (cnt == 0) {
      // the next record alone exceeds cap: report its lengths in idx[0] so that the caller can grow its buffer and
      // call again; the cursor stays where it is
      const Records &rec = pipe.state.rec;
      uint32_t i = 0, kl = 0, vl = 0;
      TG_CUDA(cudaMemcpyAsync(&i, pipe.state.order + cursor, 4, cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaStreamSynchronize(st));
      TG_CUDA(cudaMemcpyAsync(&kl, rec.key_len + i, 4, cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaMemcpyAsync(&vl, rec.val_len + i, 4, cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaStreamSynchronize(st));
      if (d.idx) d.idx[0] = tezgpu_kv_index{0, kl, kl, vl, 0};
      if (d.kv_bytes) *d.kv_bytes = (uint64_t)kl + vl;
      throw Error(TEZGPU_E_NOMEM, "batch buffer smaller than one record: the next record needs " +
                                      std::to_string((uint64_t)kl + vl) + " bytes");
    }
    uint64_t ends[2];
    TG_CUDA(cudaMemcpyAsync(&ends[0], d_kvoff.as<uint64_t>() + cursor, 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaMemcpyAsync(&ends[1], d_kvoff.as<uint64_t>() + cursor + cnt, 8, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    const uint64_t bytes = ends[1] - ends[0];
    if (d.idx) {
      d_batch.ensure(bytes + 16);
      d_batch_idx.ensure((size_t)cnt * sizeof(KvIndexDev));
      gather(cnt, bytes, d_batch.as<uint8_t>(), BatchIndexAos{d_batch_idx.as<KvIndexDev>()});
      if (bytes) TG_CUDA(cudaMemcpyAsync(d.kv, d_batch.p, bytes, cudaMemcpyDeviceToHost, st));
      static_assert(sizeof(KvIndexDev) == sizeof(tezgpu_kv_index), "index layout");
      TG_CUDA(cudaMemcpyAsync(d.idx, d_batch_idx.p, (size_t)cnt * sizeof(KvIndexDev), cudaMemcpyDeviceToHost, st));
    } else {
      gather(cnt, bytes, d.kv, BatchIndexSoa{d.key_off, d.val_off, d.val_len, d.same_key});
    }
    TG_CUDA(cudaStreamSynchronize(st));
    cursor += cnt;
    *count = cnt;
    if (d.kv_bytes) *d.kv_bytes = bytes;
  }

  // k_gather_batch of the cnt records at the cursor (bytes of key + value) into out
  template <typename Index>
  void gather(uint32_t cnt, uint64_t bytes, uint8_t *out, Index index) {
    // lanes per record: the power of two nearest above a 32nd of the mean record length, at most a warp
    uint32_t lanes_log2 = 0;
    while (lanes_log2 < 5 && (32ull << lanes_log2) * cnt < bytes) lanes_log2++;
    const uint64_t threads = std::max<uint64_t>(cnt, (uint64_t)cnt << lanes_log2);
    const uint32_t grid = (uint32_t)std::min<uint64_t>(div_up(threads, GATHER_THREADS), (uint64_t)pipe.num_sms * 16);
    k_gather_batch<<<grid, GATHER_THREADS, 0, pipe.stream>>>(pipe.state.rec, pipe.state.order, pipe.same.as<uint8_t>(),
                                                              d_kvoff.as<uint64_t>(), (uint32_t)cursor, cnt, out, index,
                                                              pipe.merge_check_same, lanes_log2);
    TG_CUDA(cudaGetLastError());
  }
};

}  // namespace tezgpu

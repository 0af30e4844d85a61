// sorter.cuh -- host orchestration of the device sort pipeline (one "spill" covering everything collected:
// HBM is the sort buffer, so this is always the numSpills==1 branch of PipelinedSorter.flush, :730-756).
#pragma once
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <mutex>
#include <vector>

#include "../../include/tezgpu.h"
#include "device_util.h"
#include "combine.cuh"
#include "emit_pipe_u.cuh"
#include "sorter_kernels.cuh"

namespace tezgpu {

// Small device -> host results (flags, counters, the spill index) are WRITTEN BY A KERNEL into mapped pinned memory
// instead of going through cudaMemcpyAsync: a tiny copy is queued on a copy engine, and when another task slot's
// multi-GB upload occupies that engine the sort's one host round trip waits for all of it (tools/e2e_probe.py shows
// the timeline of two task slots).
__global__ void k_store_to_host(uint32_t *__restrict__ dst0, const uint32_t *__restrict__ src0, uint32_t n0, uint32_t *__restrict__ dst1,
                                const uint32_t *__restrict__ src1, uint32_t n1, uint32_t *__restrict__ dst2,
                                const uint32_t *__restrict__ src2, uint32_t n2) {
  for (uint32_t i = threadIdx.x; i < n0; i += blockDim.x) dst0[i] = src0[i];
  for (uint32_t i = threadIdx.x; i < n1; i += blockDim.x) dst1[i] = src1[i];
  for (uint32_t i = threadIdx.x; i < n2; i += blockDim.x) dst2[i] = src2[i];
  __threadfence_system();
}
// up to three word-aligned ranges; dst = cudaHostAlloc memory (device-accessible under unified addressing)
static inline void store_to_host(cudaStream_t st, void *d0, const void *s0, size_t b0, void *d1 = nullptr, const void *s1 = nullptr,
                                 size_t b1 = 0, void *d2 = nullptr, const void *s2 = nullptr, size_t b2 = 0) {
  k_store_to_host<<<1, 256, 0, st>>>((uint32_t *)d0, (const uint32_t *)s0, (uint32_t)(b0 / 4), (uint32_t *)d1, (const uint32_t *)s1,
                                     (uint32_t)(b1 / 4), (uint32_t *)d2, (const uint32_t *)s2, (uint32_t)(b2 / 4));
}


static inline int partition_bits(int P) {
  int b = 0;
  while ((1ll << b) < (long long)P) b++;
  return b;
}

// per-device constant tables (CRC), created once per device on the current one (the caller's DeviceScope on `device`)
struct DeviceConstants {
  CrcTables *d_crc = nullptr;
  static const DeviceConstants &get(int device) {
    static DeviceConstants inst[64];
    static std::once_flag built[64];
    DeviceConstants &d = inst[device & 63];
    std::call_once(built[device & 63], [&d] {
      std::unique_ptr<CrcTables> h(new CrcTables());
      crc_build_tables(*h, EMIT_CRC_STRIDE_WORDS);
      CrcTables *p = nullptr;
      TG_CUDA(cudaMalloc((void **)&p, sizeof(CrcTables)));
      cudaError_t e = cudaMemcpy(p, h.get(), sizeof(CrcTables), cudaMemcpyHostToDevice);
      if (e == cudaSuccess) e = cudaStreamSynchronize(0);   // a copy from pageable memory can return before it lands
      if (e != cudaSuccess) cudaFree(p);   // the next call tries again
      TG_CUDA(e);
      d.d_crc = p;
    });
    return d;
  }
};

// The framing vint(klen) vint(vlen) in front of every fixed-width record written without repeats
constexpr uint32_t FRAMING_MAX_LEN = 10;   // two vints of at most 5 bytes
struct FixedFraming {
  uint8_t bytes[FRAMING_MAX_LEN];
  uint32_t len;        // framing bytes
  uint32_t rec_size;   // len + klen + vlen
  // framing bytes [8 * word, 8 * word + 8), little-endian packed
  uint64_t packed(uint32_t word = 0) const {
    uint64_t x = 0;
    for (uint32_t b = 8 * word; b < len && b < 8 * word + 8; b++) x |= (uint64_t)bytes[b] << (8 * (b - 8 * word));
    return x;
  }
};
static inline FixedFraming fixed_framing(uint32_t klen, uint32_t vlen) {
  FixedFraming f{};
  for (int b = 0; b < vint_size_u32(klen); b++) f.bytes[f.len++] = vint_byte_u32(klen, b);
  for (int b = 0; b < vint_size_u32(vlen); b++) f.bytes[f.len++] = vint_byte_u32(vlen, b);
  f.rec_size = f.len + klen + vlen;
  return f;
}

// thrown by sort_phase in run-table mode (Records::use_runs): the merger then re-parses the segments with the walker
struct FramingMismatch {};

// The sort's device scratch (SortPipeline::small), cleared before every sort
struct SortVerdict {          // what the sort's one host round trip reads, in one piece
  int error;                  // STAGE_ERR_* bits; the handle's other steps borrow it as their error word
  union { uint32_t large_groups; uint32_t batch_count; };  // tie groups > TIE_SMALL_MAX (k_tie_fix); the merger's batch size
  unsigned long long dups;    // adjacent equal keys
  uint64_t totals[2];         // k_layout: file bytes, tiles
};
struct SortScratch {
  uint32_t hist[8 * RADIX];   // digit offsets of up to eight radix passes
  uint32_t trivial[8];        // per pass: one digit holds every key
  uint32_t tile_counter[8];
  SortVerdict verdict;
  uint32_t unused[2];
  unsigned long long ties;    // tied records (k_tie_fix)
};
constexpr size_t SORT_SCRATCH_BYTES = 16 * 1024;
struct SortHostScratch {           // its pinned mirror (SortPipeline::h_small): what the host reads, then the spill index
  SortVerdict verdict;             // sort_phase's round trip; emit_phase's totals when it lays the records out itself
  uint32_t ties;                   // the low word of SortScratch::ties
  uint64_t total;                  // refine_large_groups: a scan total, then the duplicate count
  uint32_t trivial[8];             // SortScratch::trivial of a refinement round
  static constexpr size_t INDEX_OFFSET = 4096;  // P (start, rawLength, partLength) triples
  int64_t *index() { return reinterpret_cast<int64_t *>(reinterpret_cast<uint8_t *>(this) + INDEX_OFFSET); }
};
static_assert(offsetof(SortScratch, trivial) == 2048 * 4 && offsetof(SortScratch, tile_counter) == 2056 * 4 &&
                  offsetof(SortScratch, verdict) == 2064 * 4 && sizeof(SortVerdict) == 32 && offsetof(SortScratch, ties) == 2074 * 4 &&
                  sizeof(SortScratch) <= SORT_SCRATCH_BYTES && offsetof(SortHostScratch, ties) == 32 &&
                  sizeof(SortHostScratch) <= SortHostScratch::INDEX_OFFSET, "sort scratch layout");

// The emit kernels for fixed-width records written without repeats (records with repeats take k_emit<false>).
enum class FixedEmitKernel {
  Pipe,           // k_emit_fast4: packed, 16-byte aligned records, stride a multiple of 16, at most FE4_MAX_CPR pieces
  Fast,           // k_emit_fast<5, true>: the same, wider records
  PipeUnaligned,  // k_emit_fast4u: records at arbitrary offsets, stride a multiple of 16, at most 31 pieces
  FastUnaligned,  // k_emit_fast<5, false>: the same, wider records
  General,        // k_emit<true>: strides that are not a multiple of 16
};
struct FixedEmitPlan {
  FixedEmitKernel kernel;
  uint32_t recs_per_tile;
};

// Kernel and tile size of a fixed-width emit, from the record view alone.  sort_phase lays the tiles out with it
// speculatively and emit_phase launches the kernel it names, so the tile size always suits the kernel.
static inline FixedEmitPlan plan_fixed_emit(const Records &rec, uint32_t rec_size) {
  const uint32_t stride = rec.klen + rec.vlen, cpr = stride / 16;
  // the tile image must fit the image buffer of the source-oriented emit kernels (FE_IMG_BYTES)
  const uint32_t cap = std::max<uint32_t>(1, std::min<uint32_t>(EMIT_MAX_RECS, (FE_IMG_BYTES - 32) / rec_size));
  // Those kernels build a whole tile in that buffer without cutting it: a record that does not fit it with the worst-case
  // lead, the segment header and the EOF marker takes k_emit<true>, which writes a tile in pieces of any size.
  // (k_emit_fast4's smaller image is bounded by emit4_max_recs below.)
  if (stride < 16 || stride % 16 || (uint64_t)rec_size + 15 + 4 + 2 > FE_IMG_BYTES) return {FixedEmitKernel::General, cap};
  if (!rec.key_off && !rec.use_runs && ((uintptr_t)rec.kv & 15u) == 0) {
    // k_emit_fast4's image holds exactly FE4_RUN checksum rounds, so a tile takes as many records as fit it in the
    // worst case (249 of 82 bytes: 1278 chunks, 1280 slots)
    const uint32_t m = emit4_max_recs(rec_size);
    if (emit4_fits(m, cpr, rec_size)) return {FixedEmitKernel::Pipe, std::min(cap, m)};
    return {FixedEmitKernel::Fast, cap};
  }
  // k_emit_fast4u holds a tile's words in FE4U_UNROLL gather rounds (at least 40 records when a record fits a warp)
  const uint32_t m = emit4u_max_recs(cpr);
  if (m == 0) return {FixedEmitKernel::FastUnaligned, cap};
  // Round filling: its checksum / write-out loop walks a tile in rounds of FE_THREADS 16-byte chunks.  Among the tile
  // sizes within 10 % of the cap, take the one with the most records per executed round.
  const uint32_t top = std::min(cap, m);
  uint32_t best = top;
  double best_eff = 0;
  for (uint32_t r = top; r >= top - top / 10; r--) {
    const uint64_t chunks = ((uint64_t)r * rec_size + 15 + 4 + 2 + 15) / 16;  // worst-case lead, header, EOF
    const uint64_t rounds = (chunks + FE_THREADS - 1) / FE_THREADS;
    const double eff = (double)r / (double)rounds;
    if (eff > best_eff) { best_eff = eff; best = r; }
  }
  return {FixedEmitKernel::PipeUnaligned, best};
}

// persistent CTAs of a one-group emit kernel over `tiles` tiles: as many as fit the device at once
template <typename Kern>
static inline uint32_t persistent_ctas(Kern kern, int threads, size_t smem, int num_sms, uint64_t tiles) {
  int per_sm = 0;
  TG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
  return (uint32_t)std::min<uint64_t>(tiles, (uint64_t)num_sms * (per_sm > 0 ? per_sm : 1));
}

// Launch shape of a fixed-width emit kernel over `tiles` tiles: `ctas` CTAs of `groups` independent tile groups; group
// g of CTA b takes tile b * groups + g, then every (ctas * groups)-th.  Sets the kernel's shared-memory limit on
// `device` first where it needs one, so the shape is the one the launch gets.
struct EmitGrid {
  uint32_t ctas, groups;
};
static inline EmitGrid fixed_emit_grid(int device, int num_sms, FixedEmitKernel kernel, uint64_t tiles) {
  switch (kernel) {
    case FixedEmitKernel::Pipe:
      // One CTA per SM, FE4_GROUPS independent 256-thread groups sharing the lane-private checksum tables (66 KB)
      // next to their images, indices and parked partials (54 KB): 125 KB keeps the CTA in the 132 KB
      // shared-memory carveout, which leaves the random gather enough L1 for its loads in flight (larger
      // footprints measured slower, DESIGN.md §7).
      set_smem_limit<k_emit_fast4<FE4_UNROLL>>(device, Emit4Smem::TOTAL);
      return {(uint32_t)std::min<uint64_t>(div_up(tiles, FE4_GROUPS), (uint64_t)num_sms), (uint32_t)FE4_GROUPS};
    case FixedEmitKernel::Fast:
      return {persistent_ctas(k_emit_fast<5, true>, FE_THREADS, 0, num_sms, tiles), 1};
    case FixedEmitKernel::PipeUnaligned:
      set_smem_limit<k_emit_fast4u<FE4U_UNROLL>>(device, Emit4uSmem::TOTAL);
      return {persistent_ctas(k_emit_fast4u<FE4U_UNROLL>, FE_THREADS, Emit4uSmem::TOTAL, num_sms, tiles), 1};
    case FixedEmitKernel::FastUnaligned:
      return {persistent_ctas(k_emit_fast<5, false>, FE_THREADS, 0, num_sms, tiles), 1};
    case FixedEmitKernel::General:
      break;
  }
  return {persistent_ctas(k_emit<true>, EMIT_THREADS, 0, num_sms, tiles), 1};
}

class SortPipeline {
 public:
  tezgpu_conf conf;
  int pbits;
  cudaStream_t stream = nullptr;
  EventTimer timer;
  int num_sms = 132;

  // workspace (grow-only, reused across flushes)
  // sortA / sortB: the radix sort's two 8n-byte blocks (radix_sort_pairs).  The stage writes the sort words to the
  // first half of sortA; the sorted words and the index array end up in the two halves of one block.
  DeviceBuffer sortA, sortB, same, blk, small, tile_state, sizes, rec_off;
  DeviceBuffer t_pos[2], t_gid[2], t_lidx[2], t_key64[2], t_val[2], t_state, t_ghead, t_gneq, sym_sets, sym_tab, rep_flags;
  DeviceBuffer seg_start, tile_start, part_start, d_index, seg_crc, tile_desc, tile_crc, tie_state;
  PinnedBuffer h_small;

  // run by the caller before it opens the constructor's DeviceScope: a bad configuration is reported before a bad device
  static void check_conf(const tezgpu_conf &c) {
    TG_CHECK(c.num_partitions >= 1, TEZGPU_E_INVALID, "num_partitions must be >= 1");
    TG_CHECK(c.comparator >= TEZGPU_CMP_BYTES && c.comparator <= TEZGPU_CMP_LONG, TEZGPU_E_UNSUPPORTED,
             "comparator outside the device-supported set (BYTES, TEXT, BYTESWRITABLE, INT, LONG)");
    TG_CHECK(c.partitioner == TEZGPU_PART_GIVEN || c.partitioner == TEZGPU_PART_HASH || c.partitioner == TEZGPU_PART_TOTAL_ORDER,
             TEZGPU_E_UNSUPPORTED, "partitioner outside the device-supported set (GIVEN, HASH, TOTAL_ORDER)");
  }

  explicit SortPipeline(const tezgpu_conf &c) : conf(c) {
    TG_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    TG_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, c.device));
    // The path is dominated by sparse reads (16-byte keys out of 80-byte records, 80-byte record gathers): ask L2 to
    // fetch 32-byte sectors instead of wider granules (k_stage reads 16 of every 80 bytes).  TEZGPU_L2_FETCH=0 leaves
    // the device limit untouched, any other value overrides.
    {
      const char *g = getenv("TEZGPU_L2_FETCH");
      int gran = g ? atoi(g) : 32;
      if (gran > 0 && cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)gran) != cudaSuccess) cudaGetLastError();
    }
    pbits = partition_bits(c.num_partitions);
    TG_CHECK(pbits <= 31, TEZGPU_E_INVALID, "too many partitions");
    h_small.ensure(SortHostScratch::INDEX_OFFSET);
    small.ensure(SORT_SCRATCH_BYTES);
    DeviceConstants::get(c.device);
  }
  ~SortPipeline() {
    if (stream) cudaStreamDestroy(stream);
  }

  static uint64_t output_bound(uint64_t n, uint64_t kv_bytes, int P) { return kv_bytes + 12 * n + 10ull * P + 64; }

  SortScratch *d_scratch() const { return small.as<SortScratch>(); }
  SortHostScratch *h_scratch() const { return h_small.as<SortHostScratch>(); }

  // state left behind by sort_phase for emit_phase / the merger's record iterator
  struct SortState {
    Records rec;
    uint32_t *K = nullptr;      // sorted sort words
    uint32_t *order = nullptr;  // sorted position -> record index
    uint64_t dup_count = 0, tie_records = 0;
    int launches = 0;
    bool have_bounds = false, spec_layout = false;  // partition bounds / fixed-width layout (totals, index: h_scratch()) on the device
    const uint8_t *same = nullptr;  // the combined records' same[] (all zero); nullptr = the sort's own `same`
  } state;
  // merge mode only (the Merger sets them): MergeQueue.checkForSameKeys, and "no input record was run-length encoded"
  // (every segment had the plain fixed framing), which together decide whether any record can be written as a repeat
  int merge_check_same = 1;
  bool merge_inputs_plain = false;
  int combiner = TEZGPU_COMBINE_NONE;  // TEZGPU_COMBINE_*: combine_phase runs between the sort and the emit
  // TOTAL_ORDER: the split table (total_order.cuh) in device memory, grow-only; splits.n = 0 until set_split_points
  DeviceBuffer sp_prefix, sp_len, sp_off, sp_blob;
  SplitTable splits{};
  bool have_splits = false;
  // uploads a table build_split_table made; the stream is idle between flushes, so the old table is no longer read
  void set_split_points(const HostSplitTable &t) {
    const size_t n = t.prefix.size();
    sp_prefix.ensure(std::max<size_t>(n, 1) * 8);
    sp_len.ensure(std::max<size_t>(n, 1) * 4);
    sp_off.ensure(std::max<size_t>(n, 1) * 8);
    sp_blob.ensure(std::max<size_t>(t.blob.size(), 16));
    if (n) {
      TG_CUDA(cudaMemcpyAsync(sp_prefix.p, t.prefix.data(), n * 8, cudaMemcpyHostToDevice, stream));
      TG_CUDA(cudaMemcpyAsync(sp_len.p, t.len.data(), n * 4, cudaMemcpyHostToDevice, stream));
      TG_CUDA(cudaMemcpyAsync(sp_off.p, t.off.data(), n * 8, cudaMemcpyHostToDevice, stream));
    }
    if (!t.blob.empty()) TG_CUDA(cudaMemcpyAsync(sp_blob.p, t.blob.data(), t.blob.size(), cudaMemcpyHostToDevice, stream));
    TG_CUDA(cudaStreamSynchronize(stream));
    splits = SplitTable{sp_prefix.as<uint64_t>(), sp_len.as<uint32_t>(), sp_off.as<uint64_t>(), sp_blob.as<uint8_t>(), (uint32_t)n, t.order};
    have_splits = true;
  }
  // the split points k_stage searches: none unless the handle is TOTAL_ORDER (the merger's pipeline never is)
  SplitTable stage_splits() const { return conf.partitioner == TEZGPU_PART_TOTAL_ORDER ? splits : SplitTable{}; }
  // combine workspace (grow-only): head flags / group ids, sums, head positions, and the combined records' sort words,
  // order, same[], bytes and (variable width) metadata
  DeviceBuffer c_head, c_gid, c_sums, c_hpos, c_K, c_order, c_same, c_kv, c_koff, c_klen, c_vlen, c_bad;
  PinnedBuffer c_host;
  EventTimer c_timer;

  EmitParams make_emit_params(const Records &rec, const uint32_t *order, int rle, bool merge_mode, uint8_t *d_out) {
    EmitParams e;
    memset(&e, 0, sizeof(e));
    e.rec = rec;
    e.order = order;
    e.same = state.same ? state.same : same.as<uint8_t>();
    e.part_start = part_start.as<uint32_t>();
    e.seg_start = seg_start.as<uint64_t>();
    e.tile_start = tile_start.as<uint32_t>();
    e.out = d_out;
    e.seg_crc = seg_crc.as<uint32_t>();
    e.crc = DeviceConstants::get(conf.device).d_crc;
    e.rle = rle;
    e.send_empty = conf.send_empty_partition_details;
    e.unordered = conf.sorter_impl == TEZGPU_SORTER_UNORDERED;
    e.merge_mode = merge_mode ? 1 : 0;
    e.check_same = merge_check_same;
    e.P = conf.num_partitions;
    return e;
  }
  // fixed framing (vint klen, vint vlen) and the tile size of the emit kernel the plan picks, which it returns
  FixedEmitKernel set_fixed_layout(EmitParams &e, const Records &rec) {
    const FixedFraming f = fixed_framing(rec.klen, rec.vlen);
    memcpy(e.fixed_hdr, f.bytes, f.len);
    e.fixed_hdr_len = f.len;
    e.rec_size = f.rec_size;
    const FixedEmitPlan plan = plan_fixed_emit(rec, e.rec_size);
    e.recs_per_tile = plan.recs_per_tile;
    e.rec_off = nullptr;
    return plan.kernel;
  }

  void run(Records rec, uint8_t *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index, tezgpu_stats *stats) {
    const uint64_t raw_bound = output_bound(rec.n, rec.fixed ? (uint64_t)rec.n * (rec.klen + rec.vlen) : rec.kv_bytes, conf.num_partitions);
    sort_phase(rec);
    int rle;
    if (conf.rle_policy == TEZGPU_RLE_ON) rle = 1;
    else if (conf.rle_policy == TEZGPU_RLE_OFF) rle = 0;
    else rle = (conf.sorter_impl == 1) ? 0 : ((double)state.dup_count > 0.1 * (double)rec.n);
    if (conf.sorter_impl == TEZGPU_SORTER_UNORDERED) rle = 0;   // Writer(..., codec, null, null): no run-length encoding (:1092)
    emit_out(rle, false, raw_bound, d_out, out_cap, out_len, index, stats);
  }

  // ---- codec (deflate.cuh, lz4.cuh, zstd.cuh, codec.cuh): with a codec the emit writes the uncompressed file into z_img
  // and compress_image turns every segment into a compressed one (zlib, LZ4 or zstd) in d_out
  int codec = TEZGPU_CODEC_NONE;
  DeviceBuffer z_img, z_slots, z_csize, z_cadler, z_coff, z_segs, z_descs, z_pstart, z_tc, z_crc;
  PinnedBuffer z_host;
  EventTimer z_timer;
  // worst case of the compressed file given the uncompressed file's bound (codec.cuh)
  static uint64_t codec_bound(int codec, uint64_t raw_bound, int P);
  void compress_image(const int64_t *raw_index, uint8_t *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index, tezgpu_stats *stats);
  uint64_t compress_chunks(int32_t zc, const uint8_t *img, ZSeg *hs, uint32_t nseg, uint32_t nchunks, uint32_t frame, uint32_t tail, int *launches);

  // the emit of the sorted (merged) records: combined or not, compressed or not.  raw_bound bounds the uncompressed file.
  void emit_out(int rle, bool merge_mode, uint64_t raw_bound, uint8_t *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index,
                tezgpu_stats *stats) {
    if (!codec) {
      if (combiner) emit_combined(rle, d_out, out_cap, out_len, index, stats);
      else emit_phase(rle, merge_mode, d_out, out_cap, out_len, index, stats);
      return;
    }
    const int P = conf.num_partitions;
    z_img.ensure(raw_bound + 64);
    std::vector<int64_t> raw_index((size_t)P * 3, 0);
    uint64_t raw_len = 0;
    tezgpu_stats st;
    memset(&st, 0, sizeof(st));
    if (combiner) emit_combined(rle, z_img.as<uint8_t>(), z_img.cap, &raw_len, raw_index.data(), &st);
    else emit_phase(rle, merge_mode, z_img.as<uint8_t>(), z_img.cap, &raw_len, raw_index.data(), &st);
    compress_image(raw_index.data(), d_out, out_cap, out_len, index, &st);
    if (stats) *stats = st;
  }

  // partition + sort: stage, radix sort of (sort word, index), tie refinement.  Leaves K / order / same / counts.
  void sort_phase(Records rec) {
    const uint32_t n = rec.n;
    const int P = conf.num_partitions;
    TG_CHECK(n <= RADIX_MAX_N, TEZGPU_E_INVALID, "more than 2^30-1 records in one sort");
    rec.cmp = conf.comparator;
    rec.hash_partition = conf.partitioner == TEZGPU_PART_HASH;
    rec.num_partitions = P;
    rec.pbits = pbits;
    rec.unordered = conf.sorter_impl == TEZGPU_SORTER_UNORDERED ? 1 : 0;
    TG_CHECK(rec.hash_partition || rec.partition || rec.use_runs || stage_splits().n || n == 0 || P == 1, TEZGPU_E_INVALID,
             "partition ids required (partitioner=GIVEN)");
    state.have_bounds = state.spec_layout = false;
    state.same = nullptr;
    timer.reset();
    timer.mark(stream);

    const size_t n4 = (size_t)(n ? n : 1) * 4;
    sortA.ensure(2 * n4); sortB.ensure(2 * n4);
    same.ensure(n ? n : 1);
    blk.ensure((div_up(n ? n : 1, SCAN_TILE) + 2) * 8);
    part_start.ensure(((size_t)P + 1) * 4);
    seg_start.ensure(((size_t)P + 1) * 8);
    tile_start.ensure(((size_t)P + 1) * 4);
    d_index.ensure((size_t)P * 24);
    seg_crc.ensure((size_t)P * 4);
    h_small.ensure(SortHostScratch::INDEX_OFFSET + (size_t)P * 24);

    TG_CUDA(cudaMemsetAsync(small.p, 0, SORT_SCRATCH_BYTES, stream));
    TG_CUDA(cudaMemsetAsync(seg_crc.p, 0, (size_t)P * 4, stream));

    state.K = sortA.as<uint32_t>();
    state.order = sortA.as<uint32_t>() + n;
    state.dup_count = state.tie_records = 0;
    int launches = 0;
    if (n) {
      uint32_t depth0;
      launches += alphabet_table(rec, &depth0);
      launches += stage_and_sort(rec);
      launches += fix_ties(rec, depth0);
      if (h_scratch()->verdict.large_groups) launches += refine_large_groups(rec, depth0);
    }
    timer.mark(stream);
    state.rec = rec;
    state.launches = launches;
  }

  // The alphabet-compressed sort word (SymTable, sorter_kernels.cuh): the byte values at the first content positions ->
  // ranks, packed while they fit the key field.  *depth = normalised content bytes the sort word fully covers.
  int alphabet_table(Records &rec, uint32_t *depth) {
    *depth = (uint32_t)((32 - pbits) / 8);
    if (rec.fixed || rec.unordered || (getenv("TEZGPU_NO_SYM") && atoi(getenv("TEZGPU_NO_SYM")))) return 0;
    sym_sets.ensure(SYM_MAX_POS * 8 * 4);
    sym_tab.ensure(sizeof(SymTable));
    TG_CUDA(cudaMemsetAsync(sym_sets.p, 0, SYM_MAX_POS * 8 * 4, stream));
    k_symbols<<<(int)std::min<uint64_t>(div_up(rec.n, 256), (uint64_t)num_sms * 8), 256, 0, stream>>>(rec, sym_sets.as<uint32_t>());
    uint32_t hs[SYM_MAX_POS * 8];
    TG_CUDA(cudaMemcpyAsync(hs, sym_sets.p, sizeof(hs), cudaMemcpyDeviceToHost, stream));
    TG_CUDA(cudaStreamSynchronize(stream));
    SymTable *t = new SymTable();
    const uint32_t np = sym_table_build(hs, pbits, t);
    if (sym_table_pays(np, pbits)) {
      TG_CUDA(cudaMemcpyAsync(sym_tab.p, t, sizeof(SymTable), cudaMemcpyHostToDevice, stream));
      TG_CUDA(cudaStreamSynchronize(stream));
      rec.sym = sym_tab.as<SymTable>();
      *depth = np;
    }
    delete t;
    return 1;
  }

  // The stage (sort words, and the digit histograms of every pass) and the radix sort of (sort word, record index)
  int stage_and_sort(const Records &rec) {
    const uint32_t n = rec.n;
    SortScratch *d = d_scratch();
    TG_CUDA(cudaMemsetAsync(same.p, 0, n, stream));
    const bool fast16 = rec.fixed && !rec.key_off && !rec.use_runs && rec.klen == 16 && ((rec.klen + rec.vlen) % 16 == 0) && rec.cmp == CMP_BYTES &&
                        (((uintptr_t)rec.kv & 15u) == 0);
    int sgrid = (int)std::min<uint64_t>(div_up(n, 256), (uint64_t)num_sms * 16);
    const SplitTable sp = stage_splits();
    if (sp.n) {
      const size_t smem = sp.n <= SPLIT_SMEM_MAX ? (size_t)sp.n * 8 : 0;
      if (fast16) k_stage<true, true><<<sgrid, 256, smem, stream>>>(rec, state.K, d->hist, &d->verdict.error, sp);
      else k_stage<false, true><<<sgrid, 256, smem, stream>>>(rec, state.K, d->hist, &d->verdict.error, sp);
    } else if (fast16) {
      k_stage<true><<<sgrid, 256, 0, stream>>>(rec, state.K, d->hist, &d->verdict.error, sp);
    } else {
      k_stage<false><<<sgrid, 256, 0, stream>>>(rec, state.K, d->hist, &d->verdict.error, sp);
    }
    TG_CUDA(cudaGetLastError());
    k_radix_scan_hist<<<1, RADIX, 0, stream>>>(d->hist, 4, n, d->trivial);
    TG_CUDA(cudaGetLastError());
    int launches = 2;
    timer.mark(stream);

    const size_t words = radix_tile_state_words<uint32_t>(n, 4);
    tile_state.ensure(words * 4);
    const RadixWorkspace ws{d->hist, d->trivial, tile_state.as<uint32_t>(), d->tile_counter, words, conf.device};
    // unordered: only the passes that cover the partition bits (the top pbits of the word); none when P == 1 -- the
    // first pass is still needed then, to produce the identity index array
    uint32_t pass_mask = 0xF;
    if (rec.unordered) {
      pass_mask = 0;
      for (int q = 0; q < 4; q++) if (8 * q + 8 > 32 - pbits) pass_mask |= 1u << q;
      if (!pass_mask) pass_mask = 1;
    }
    const int done = radix_sort_pairs(stream, ws, sortA.as<uint32_t>(), sortB.as<uint32_t>(), n, 0, 4, pass_mask, &launches);
    if (done & 1) { state.K = sortB.as<uint32_t>(); state.order = sortB.as<uint32_t>() + n; }
    if (rec.unordered) {
      k_flip_order<<<(uint32_t)div_up(n, 256), 256, 0, stream>>>(state.order, n);
      launches++;
    }
    timer.mark(stream);
    return launches;
  }

  // Ties: records whose sort words collide are ordered by the rest of the key.  One streaming kernel finds the groups
  // and orders the (common) small ones in place; the partition bounds and -- for fixed-width records -- the segment
  // layout are computed speculatively, so that the whole common path needs this one host round trip (its verdict).
  int fix_ties(const Records &rec, uint32_t depth0) {
    const uint32_t n = rec.n;
    const int P = conf.num_partitions;
    SortScratch *d = d_scratch();
    SortHostScratch *h = h_scratch();
    int per_sm_tf = 0;
    TG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_tf, k_tie_fix, TIEFIX_THREADS, 0));
    if (!rec.unordered)   // no comparator on an unordered edge: records of a partition keep their (reversed arrival) order
      k_tie_fix<<<(uint32_t)std::min<uint64_t>(div_up(n, TIEFIX_TILE), (uint64_t)num_sms * std::max(per_sm_tf, 1)), TIEFIX_THREADS, 0, stream>>>(
          rec, state.K, state.order, n, depth0, same.as<uint8_t>(), &d->verdict.dups, &d->verdict.large_groups, &d->ties);
    k_part_bounds<<<(uint32_t)div_up((uint64_t)P + 1, 256), 256, 0, stream>>>(state.K, n, P, pbits, part_start.as<uint32_t>());
    int launches = 2;   // k_tie_fix is counted on unordered edges too
    state.have_bounds = true;
    if (rec.fixed) {
      EmitParams e = make_emit_params(rec, state.order, 0, false, nullptr);
      set_fixed_layout(e, rec);
      k_layout<<<1, 1024, 0, stream>>>(e, seg_start.as<uint64_t>(), tile_start.as<uint32_t>(), d_index.as<int64_t>(), d->verdict.totals);
      launches++;
      state.spec_layout = true;
    }
    TG_CUDA(cudaGetLastError());
    store_to_host(stream, &h->verdict, &d->verdict, sizeof(SortVerdict), &h->ties, &d->ties, 4, h->index(), d_index.p,
                  state.spec_layout ? (size_t)P * 24 : 0);
    TG_CUDA(cudaGetLastError());
    TG_CUDA(cudaStreamSynchronize(stream));
    TG_CHECK(!(h->verdict.error & STAGE_ERR_PARTITION), TEZGPU_E_INVALID, "Illegal partition (outside [0, numPartitions))");
    if (h->verdict.error & STAGE_ERR_FRAMING) throw FramingMismatch();
    state.tie_records = h->ties;
    state.dup_count = h->verdict.dups;
    return launches;
  }

  // Some tie group is larger than TIE_SMALL_MAX: radix refinement rounds over all tied records.  Groups whose members
  // all carry the same key need no ordering (the radix sort is stable) and are settled first; only groups with really
  // different keys go through the rounds.  Small groups keep the order, flags and duplicate count k_tie_fix gave them.
  int refine_large_groups(const Records &rec, uint32_t depth0) {
    const uint32_t n = rec.n, nblk = (uint32_t)div_up(n, SCAN_TILE);
    SortScratch *d = d_scratch();
    SortHostScratch *h = h_scratch();
    int launches = 0;
    auto scan_total = [&](uint32_t nb) {
      k_scan_block_sums<<<1, 1024, 0, stream>>>(blk.as<uint64_t>(), nb);
      launches++;
      TG_CUDA(cudaGetLastError());
      TG_CUDA(cudaMemcpyAsync(&h->total, blk.as<uint64_t>() + nb, 8, cudaMemcpyDeviceToHost, stream));
      TG_CUDA(cudaStreamSynchronize(stream));
      return h->total;
    };
    k_tie_count<<<nblk, SCAN_THREADS, 0, stream>>>(state.K, n, blk.as<uint64_t>());
    const uint64_t tied = scan_total(nblk);
    uint32_t m = (uint32_t)tied;
    const uint32_t ngroups = (uint32_t)(tied >> 32);
    state.tie_records = m;
    for (int s2 = 0; s2 < 2; s2++) { t_pos[s2].ensure((size_t)m * 4); t_gid[s2].ensure((size_t)m * 4); t_lidx[s2].ensure((size_t)m * 4); }
    k_tie_compact<<<nblk, SCAN_THREADS, 0, stream>>>(state.K, state.order, n, blk.as<uint64_t>(), t_pos[0].as<uint32_t>(),
                                                     t_gid[0].as<uint32_t>(), t_lidx[0].as<uint32_t>());
    launches += 2;
    t_ghead.ensure(((size_t)ngroups + 2) * 4);
    t_gneq.ensure((size_t)ngroups + 1);
    TG_CUDA(cudaMemsetAsync(t_gneq.p, 0, (size_t)ngroups + 1, stream));
    const uint32_t mgrid = (uint32_t)div_up(m, 256), mblk0 = (uint32_t)div_up(m, SCAN_TILE);
    k_group_heads<<<mgrid, 256, 0, stream>>>(t_gid[0].as<uint32_t>(), m, t_ghead.as<uint32_t>());
    k_group_equal<<<mgrid, 256, 0, stream>>>(rec, t_gid[0].as<uint32_t>(), t_lidx[0].as<uint32_t>(), t_ghead.as<uint32_t>(), m, depth0,
                                           TIE_SMALL_MAX, t_gneq.as<uint8_t>());
    blk.ensure(((size_t)std::max(mblk0, nblk) + 2) * 8);
    k_group_mark<<<mblk0, SCAN_THREADS, 0, stream>>>(t_pos[0].as<uint32_t>(), t_gid[0].as<uint32_t>(), t_ghead.as<uint32_t>(),
                                                    t_gneq.as<uint8_t>(), m, TIE_SMALL_MAX, same.as<uint8_t>(), &d->verdict.dups, blk.as<uint64_t>());
    launches += 3;
    uint32_t left = (uint32_t)scan_total(mblk0);   // records of the groups whose keys differ
    if (left) {
      k_group_compact<<<mblk0, SCAN_THREADS, 0, stream>>>(t_pos[0].as<uint32_t>(), t_gid[0].as<uint32_t>(), t_lidx[0].as<uint32_t>(),
                                                         t_ghead.as<uint32_t>(), t_gneq.as<uint8_t>(), m, TIE_SMALL_MAX, blk.as<uint64_t>(),
                                                         t_pos[1].as<uint32_t>(), t_gid[1].as<uint32_t>(), t_lidx[1].as<uint32_t>());
      launches++;
      TG_CUDA(cudaGetLastError());
    }
    for (uint32_t depth = depth0, cur = 1; left; depth += 3, cur ^= 1) {
      m = left;
      t_key64[0].ensure((size_t)m * 8); t_key64[1].ensure((size_t)m * 8); t_val[0].ensure((size_t)m * 4);
      const uint32_t mblk = (uint32_t)div_up(m, SCAN_TILE);
      k_ref_build_keys<<<(uint32_t)div_up(m, 256), 256, 0, stream>>>(rec, t_gid[cur].as<uint32_t>(), t_lidx[cur].as<uint32_t>(), m,
                                                                depth, t_key64[0].as<uint64_t>());
      TG_CUDA(cudaMemsetAsync(d->hist, 0, sizeof(d->hist), stream));
      k_radix_hist<uint64_t, 8><<<(int)std::min<uint64_t>(div_up(m, 512 * 8), (uint64_t)num_sms * 4), 512, 0, stream>>>(t_key64[0].as<uint64_t>(), m, 0, d->hist);
      k_radix_scan_hist<<<1, RADIX, 0, stream>>>(d->hist, 8, m, d->trivial);
      launches += 3;
      TG_CUDA(cudaGetLastError());
      TG_CUDA(cudaMemcpyAsync(h->trivial, d->trivial, sizeof(h->trivial), cudaMemcpyDeviceToHost, stream));
      TG_CUDA(cudaStreamSynchronize(stream));
      uint32_t mask = 0;
      for (int q = 0; q < 8; q++) if (!h->trivial[q]) mask |= 1u << q;
      const size_t words = radix_tile_state_words<uint64_t>(m, 8);
      t_state.ensure(words * 4);
      const RadixWorkspace ws{d->hist, d->trivial, t_state.as<uint32_t>(), d->tile_counter, words, conf.device};
      const int passes = radix_sort_passes<uint64_t>(stream, ws, t_key64[0].as<uint64_t>(), t_key64[1].as<uint64_t>(), t_lidx[cur].as<uint32_t>(),
                                                     t_val[0].as<uint32_t>(), m, 0, 8, mask, &launches);
      const uint64_t *Ks = (passes & 1) ? t_key64[1].as<uint64_t>() : t_key64[0].as<uint64_t>();
      const uint32_t *Ls = (passes & 1) ? t_val[0].as<uint32_t>() : t_lidx[cur].as<uint32_t>();
      k_ref_apply_count<<<mblk, SCAN_THREADS, 0, stream>>>(Ks, Ls, t_pos[cur].as<uint32_t>(), m, state.order, same.as<uint8_t>(), &d->verdict.dups,
                                                          blk.as<uint64_t>());
      launches++;
      left = (uint32_t)scan_total(mblk);
      if (left) {
        k_ref_compact<<<mblk, SCAN_THREADS, 0, stream>>>(Ks, Ls, t_pos[cur].as<uint32_t>(), m, blk.as<uint64_t>(),
                                                        t_pos[cur ^ 1].as<uint32_t>(), t_gid[cur ^ 1].as<uint32_t>(),
                                                        t_lidx[cur ^ 1].as<uint32_t>());
        launches++;
        TG_CUDA(cudaGetLastError());
      }
    }
    TG_CUDA(cudaMemcpyAsync(&h->total, &d->verdict.dups, 8, cudaMemcpyDeviceToHost, stream));
    TG_CUDA(cudaStreamSynchronize(stream));
    state.dup_count = h->total;
    return launches;
  }

  // layout + emit of the sorted records as IFile segments.  merge_mode: REPEAT_KEY semantics of TezMerger.writeFile
  // (empty keys may be run-length encoded too, SORT/TezMerger.java:215-245).
  void emit_phase(int rle, bool merge_mode, uint8_t *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index,
                  tezgpu_stats *stats) {
    TG_CHECK(((uintptr_t)d_out & 15u) == 0, TEZGPU_E_INVALID, "output buffer must be 16-byte aligned");
    const Records rec = state.rec;
    const uint32_t n = rec.n;
    const int P = conf.num_partitions;
    uint32_t *K = state.K, *order = state.order;
    const uint64_t dup_count = state.dup_count, tie_records = state.tie_records;
    int launches = state.launches;
    const CrcTables *d_crc = DeviceConstants::get(conf.device).d_crc;
    const size_t n4 = (size_t)(n ? n : 1) * 4;
    TG_CUDA(cudaMemsetAsync(seg_crc.p, 0, (size_t)P * 4, stream));
    if (timer.n > (n ? 4 : 2)) timer.n = n ? 4 : 2;  // re-emit: drop the marks of a previous emit

    // ---------------- layout + emit
    EmitParams e = make_emit_params(rec, order, rle, merge_mode, d_out);
    if (!state.have_bounds) {
      k_part_bounds<<<(uint32_t)div_up((uint64_t)P + 1, 256), 256, 0, stream>>>(K, n, P, pbits, part_start.as<uint32_t>());
      launches++;
    }
    // constant-size framing is only valid when no record is written as a repeat (merge mode flags repeats on its own)
    // (a merge writes repeats for isSameKey() records: none exist when checkForSameKeys is off and no input was encoded)
    const bool no_repeats = !rle && (!merge_mode || (!merge_check_same && merge_inputs_plain));
    const bool fixed_emit = rec.fixed && (dup_count == 0 || no_repeats);
    uint64_t bound = output_bound(n, rec.fixed ? (uint64_t)n * (rec.klen + rec.vlen) : rec.kv_bytes, P);
    const FixedEmitKernel kernel = fixed_emit ? set_fixed_layout(e, rec) : FixedEmitKernel::General;
    // layout, totals and index triples produced during the sort phase (same plan) need no round trip here
    if (!fixed_emit || !state.spec_layout) {
      if (!fixed_emit) {
        uint64_t avg = n ? (rec.fixed ? (uint64_t)(rec.klen + rec.vlen) : rec.kv_bytes / n) + 4 : 16;
        e.recs_per_tile = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(EMIT_MAX_RECS, (EMIT_IMG_BYTES - 32) / avg));
        sizes.ensure(n4);
        rec_off.ensure(((size_t)n + 2) * 8);
        if (n) {
          rep_flags.ensure(n);
          k_emit_repeat_flags<<<(uint32_t)div_up(n, 256), 256, 0, stream>>>(e, K, rep_flags.as<uint8_t>());
          launches++;
          e.rep = rep_flags.as<uint8_t>();
          k_emit_sizes<<<(uint32_t)div_up(n, 256), 256, 0, stream>>>(e, K, sizes.as<uint32_t>());
          launches += 1 + scan_u32_exclusive(stream, blk, sizes.as<uint32_t>(), n, rec_off.as<uint64_t>());
          TG_CUDA(cudaGetLastError());
        } else {
          TG_CUDA(cudaMemsetAsync(rec_off.p, 0, 16, stream));
        }
        e.rec_off = rec_off.as<uint64_t>();
      }
      k_layout<<<1, 1024, 0, stream>>>(e, seg_start.as<uint64_t>(), tile_start.as<uint32_t>(), d_index.as<int64_t>(), d_scratch()->verdict.totals);
      launches++;
      TG_CUDA(cudaGetLastError());
      store_to_host(stream, h_scratch()->verdict.totals, d_scratch()->verdict.totals, 16, h_scratch()->index(), d_index.p, (size_t)P * 24);
      TG_CUDA(cudaGetLastError());
      TG_CUDA(cudaStreamSynchronize(stream));
      state.spec_layout = false;  // the device layout now belongs to this emit
    }
    const uint64_t file_bytes = h_scratch()->verdict.totals[0];
    const uint64_t tiles = h_scratch()->verdict.totals[1];
    TG_CHECK(file_bytes <= bound, TEZGPU_E_INVALID, "internal: output exceeds bound");
    TG_CHECK(file_bytes <= out_cap, TEZGPU_E_NOMEM, "output buffer too small for file.out");
    // the source-oriented kernels (emit_fast.cuh, emit_pipe*.cuh) gather 16-byte pieces of the records tile by tile
    // and leave one checksum per tile
    const bool source_oriented = fixed_emit && kernel != FixedEmitKernel::General;
    const uint32_t stride = rec.klen + rec.vlen;
    FastEmitParams fp;
    if (tiles && source_oriented) {
      tile_desc.ensure((size_t)tiles * sizeof(TileDesc));
      k_build_tiles<<<(uint32_t)div_up(tiles, 256), 256, 0, stream>>>(e, tile_desc.as<TileDesc>());
      launches++;
      fp.e = e;
      tile_crc.ensure((size_t)tiles * sizeof(TileCrc));
      fp.tile_crc = tile_crc.as<TileCrc>();
      fp.tiles = tile_desc.as<TileDesc>();
      fp.ntiles = (uint32_t)tiles;
      fp.cpr = stride / 16;
      fp.cpr_magic = fp.cpr == 1 ? 0u : (uint32_t)((1ull << 32) / fp.cpr) + 1u;
      fp.stride = stride;
    }
    timer.mark(stream);
    if (tiles) {
      if (!fixed_emit) {
        k_emit<false><<<persistent_ctas(k_emit<false>, EMIT_THREADS, 0, num_sms, tiles), EMIT_THREADS, 0, stream>>>(e);
      } else {
        const uint32_t grid = fixed_emit_grid(conf.device, num_sms, kernel, tiles).ctas;
        switch (kernel) {
          case FixedEmitKernel::Pipe:
            k_emit_fast4<FE4_UNROLL><<<grid, FE_THREADS * FE4_GROUPS, Emit4Smem::TOTAL, stream>>>(fp);
            break;
          case FixedEmitKernel::Fast:
            k_emit_fast<5, true><<<grid, FE_THREADS, 0, stream>>>(fp);
            break;
          case FixedEmitKernel::PipeUnaligned:
            k_emit_fast4u<FE4U_UNROLL><<<grid, FE_THREADS, Emit4uSmem::TOTAL, stream>>>(fp);
            break;
          case FixedEmitKernel::FastUnaligned:
            k_emit_fast<5, false><<<grid, FE_THREADS, 0, stream>>>(fp);
            break;
          case FixedEmitKernel::General:
            k_emit<true><<<grid, EMIT_THREADS, 0, stream>>>(e);
            break;
        }
      }
      if (source_oriented) {
        k_crc_combine<<<(uint32_t)div_up(tiles, 256), 256, 0, stream>>>(fp.tile_crc, (uint32_t)tiles, d_crc, seg_crc.as<uint32_t>());
        launches++;
      }
      launches++;
      TG_CUDA(cudaGetLastError());
    }
    timer.mark(stream);
    k_finalize_segments<<<(uint32_t)div_up(P, 256), 256, 0, stream>>>(e);
    launches++;
    TG_CUDA(cudaGetLastError());
    timer.mark(stream);
    TG_CUDA(cudaStreamSynchronize(stream));

    if (out_len) *out_len = file_bytes;
    const int64_t *hidx = h_scratch()->index();
    if (index) memcpy(index, hidx, (size_t)P * 24);
    if (stats) {
      memset(stats, 0, sizeof(*stats));
      stats->output_records = n;
      int64_t raw = 0;
      for (int p = 0; p < P; p++) raw += hidx[3 * p + 1];
      stats->output_bytes_with_overhead = raw;
      stats->output_bytes_physical = (int64_t)file_bytes;
      stats->file_out_bytes = (int64_t)file_bytes;
      stats->spilled_records = n;
      stats->num_spills = 1;
      stats->rle_used = rle;
      stats->adjacent_equal_keys = (int64_t)dup_count;
      stats->tie_records = (int64_t)tie_records;
      // marks: n>0: start, stage, sort, ties, pre-emit-kernel, post-emit-kernel, end ; n==0: start, ties, pre, post, end
      const int b = n ? 3 : 1;
      stats->ms_stage = n ? timer.ms(0, 1) : 0;
      stats->ms_sort = n ? timer.ms(1, 2) : 0;
      stats->ms_ties = n ? timer.ms(2, 3) : 0;
      stats->ms_emit = timer.ms(b, b + 3);
      stats->ms_emit_kernel = timer.ms(b + 1, b + 2);
      stats->ms_total = timer.ms(0, b + 3);
      stats->kernel_launches = launches;
    }
  }

  // Combine (combine.cuh): replaces state.rec / K / order / same by one record per group of equal keys, in sorted order,
  // so that the unchanged emit_phase writes them.  Returns false when no two adjacent keys are equal: the records are then
  // their own combined form (a group of one re-encodes to its input bytes) and only the value widths are checked.
  // Throws TEZGPU_E_INVALID, naming the record (collection / merge order), on a value of the wrong width.
  bool combine_phase() {
    const Records rec = state.rec;
    const uint32_t n = rec.n, W = combine_width(combiner);
    TG_CHECK(W, TEZGPU_E_INVALID, "unknown combiner");
    const char *name = combiner == TEZGPU_COMBINE_SUM_INT ? "IntSumReducer needs 4-byte IntWritable values"
                                                          : "LongSumReducer needs 8-byte LongWritable values";
    if (n == 0) return false;
    c_bad.ensure(16);
    c_host.ensure(64);
    uint32_t *bad = c_bad.as<uint32_t>();
    TG_CUDA(cudaMemsetAsync(bad, 0xFF, 4, stream));
    int launches = 0;
    if (state.dup_count == 0) {
      if (rec.fixed) {
        TG_CHECK(rec.vlen == W, TEZGPU_E_INVALID, "combiner: record 0 has a " + std::to_string(rec.vlen) + "-byte value (" + name + ")");
        return false;
      }
      k_combine_check_width<<<(uint32_t)std::min<uint64_t>(div_up(n, 256), (uint64_t)num_sms * 16), 256, 0, stream>>>(rec, W, bad);
      TG_CUDA(cudaGetLastError());
      state.launches += 1;
      uint32_t *h = c_host.as<uint32_t>();
      TG_CUDA(cudaMemcpyAsync(h, bad, 4, cudaMemcpyDeviceToHost, stream));
      TG_CUDA(cudaStreamSynchronize(stream));
      TG_CHECK(h[0] == 0xFFFFFFFFu, TEZGPU_E_INVALID, "combiner: record " + std::to_string(h[0]) + " has a value of the wrong width (" + name + ")");
      return false;
    }
    // ---- group ids: exclusive scan of the heads
    c_head.ensure((size_t)n * 4);
    c_gid.ensure(((size_t)n + 1) * 8);
    k_combine_heads<<<(uint32_t)div_up(n, 256), 256, 0, stream>>>(same.as<uint8_t>(), n, c_head.as<uint32_t>());
    launches += 1 + scan_u32_exclusive(stream, blk, c_head.as<uint32_t>(), n, c_gid.as<uint64_t>());
    // ---- segmented sums (groups <= n: sized by n, no round trip first)
    c_sums.ensure((size_t)n * 8);
    c_hpos.ensure((size_t)n * 4);
    c_K.ensure((size_t)n * 4);
    TG_CUDA(cudaMemsetAsync(c_sums.p, 0, (size_t)n * 8, stream));
    const uint32_t sgrid = (uint32_t)div_up(div_up(n, 32 * CMB_ROWS) * 32, CMB_THREADS);
    if (W == 4)
      k_combine_sum<4><<<sgrid, CMB_THREADS, 0, stream>>>(rec, state.order, state.K, c_gid.as<uint64_t>(), n, c_sums.as<unsigned long long>(),
                                                          c_hpos.as<uint32_t>(), c_K.as<uint32_t>(), bad);
    else
      k_combine_sum<8><<<sgrid, CMB_THREADS, 0, stream>>>(rec, state.order, state.K, c_gid.as<uint64_t>(), n, c_sums.as<unsigned long long>(),
                                                          c_hpos.as<uint32_t>(), c_K.as<uint32_t>(), bad);
    launches++;
    TG_CUDA(cudaGetLastError());
    uint32_t *h = c_host.as<uint32_t>();
    TG_CUDA(cudaMemcpyAsync(h, bad, 4, cudaMemcpyDeviceToHost, stream));
    TG_CUDA(cudaMemcpyAsync(h + 2, c_gid.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, stream));
    TG_CUDA(cudaStreamSynchronize(stream));
    TG_CHECK(h[0] == 0xFFFFFFFFu, TEZGPU_E_INVALID, "combiner: record " + std::to_string(h[0]) + " has a value of the wrong width (" + name + ")");
    uint64_t m64;
    memcpy(&m64, h + 2, 8);
    const uint32_t m = (uint32_t)m64;
    // ---- compaction
    c_order.ensure((size_t)m * 4);
    c_same.ensure(m);
    TG_CUDA(cudaMemsetAsync(c_same.p, 0, m, stream));
    Records out;
    memset(&out, 0, sizeof(out));
    out.n = m;
    out.cmp = rec.cmp;
    out.hash_partition = rec.hash_partition;
    out.num_partitions = rec.num_partitions;
    out.pbits = rec.pbits;
    const uint64_t *off = nullptr;
    uint64_t bytes;
    if (rec.fixed) {
      bytes = (uint64_t)m * (rec.klen + W);
      out.fixed = 1;
      out.klen = rec.klen;
      out.vlen = W;
    } else {
      // key offsets: scan of (key length + width) over the groups; c_head / c_gid are free again
      k_combine_sizes<<<(uint32_t)div_up(m, 256), 256, 0, stream>>>(rec, state.order, c_hpos.as<uint32_t>(), m, W, c_head.as<uint32_t>());
      launches += 1 + scan_u32_exclusive(stream, blk, c_head.as<uint32_t>(), m, c_gid.as<uint64_t>());
      TG_CUDA(cudaGetLastError());
      TG_CUDA(cudaMemcpyAsync(h + 4, c_gid.as<uint64_t>() + m, 8, cudaMemcpyDeviceToHost, stream));
      TG_CUDA(cudaStreamSynchronize(stream));
      memcpy(&bytes, h + 4, 8);
      off = c_gid.as<uint64_t>();
      c_koff.ensure((size_t)m * 8);
      c_klen.ensure((size_t)m * 4);
      c_vlen.ensure((size_t)m * 4);
      out.key_off = c_koff.as<uint64_t>();
      out.key_len = c_klen.as<uint32_t>();
      out.val_len = c_vlen.as<uint32_t>();
    }
    c_kv.ensure(align_up(bytes, 16) + 32);
    out.kv = c_kv.as<uint8_t>();
    out.kv_bytes = rec.fixed ? bytes : align_up(bytes, 16);
    // one thread per record for short fixed keys, a warp per record otherwise (multi-KB BytesWritable keys)
    const bool narrow = rec.fixed && rec.klen <= 64;
    const uint32_t lanes = narrow ? 1 : 32;
    const uint32_t wgrid = (uint32_t)div_up((uint64_t)m * lanes, 256);
    auto write = [&](auto kern) {
      kern<<<wgrid, 256, 0, stream>>>(rec, state.order, c_hpos.as<uint32_t>(), c_sums.as<unsigned long long>(), m, off, c_kv.as<uint8_t>(),
                                      c_order.as<uint32_t>(), c_koff.as<uint64_t>(), c_klen.as<uint32_t>(), c_vlen.as<uint32_t>());
    };
    if (W == 4) narrow ? write(k_combine_write<4, 1>) : write(k_combine_write<4, 32>);
    else narrow ? write(k_combine_write<8, 1>) : write(k_combine_write<8, 32>);
    launches++;
    TG_CUDA(cudaGetLastError());
    state.rec = out;
    state.K = c_K.as<uint32_t>();
    state.order = c_order.as<uint32_t>();
    state.same = c_same.as<uint8_t>();
    state.dup_count = 0;
    state.have_bounds = state.spec_layout = false;   // emit_phase lays the combined records out again
    state.launches += launches;
    return true;
  }

  // combine + emit.  The stats keep the meaning they have without a combiner (rle_used / adjacent_equal_keys describe
  // the uncombined stream, ms_emit the emit alone) except output_records = records that entered the combine and
  // spilled_records = records written.  The sort's state is restored afterwards, so a merger can write again.
  void emit_combined(int rle, uint8_t *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index, tezgpu_stats *stats) {
    // emit_phase's precondition, checked before the combine launches anything
    TG_CHECK(((uintptr_t)d_out & 15u) == 0, TEZGPU_E_INVALID, "output buffer must be 16-byte aligned");
    const SortState saved = state;
    c_timer.reset();
    c_timer.mark(stream);
    bool replaced = false;
    try {
      replaced = combine_phase();
      c_timer.mark(stream);
      emit_phase(rle, false, d_out, out_cap, out_len, index, stats);
    } catch (...) {
      restore_after_combine(saved, replaced);
      throw;
    }
    const uint64_t written = state.rec.n;
    restore_after_combine(saved, replaced);
    if (stats) {
      const float ms_combine = c_timer.ms(0, 1);
      stats->output_records = (int64_t)saved.rec.n;
      stats->spilled_records = (int64_t)written;
      stats->adjacent_equal_keys = (int64_t)saved.dup_count;
      stats->ms_emit = std::max(0.f, stats->ms_emit - ms_combine);
    }
  }
  void restore_after_combine(const SortState &saved, bool replaced) {
    if (!replaced) return;   // the emit ran over the sort's own records
    const int launches = state.launches;
    state = saved;
    state.launches = launches;
    // the combined emit overwrote the partition bounds and the layout of the sorted records
    state.have_bounds = state.spec_layout = false;
  }
};

}  // namespace tezgpu

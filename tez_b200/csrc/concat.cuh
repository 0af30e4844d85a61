// concat.cuh -- the concatenating "merge" behind tezgpu_concat_open: UnorderedPartitionedKVWriter.mergeAll
// (RL/common/writers/UnorderedPartitionedKVWriter.java:1058-1144) and UnorderedKVReader
// (RL/common/readers/UnorderedKVReader.java:119-230).  Records leave in (segment, position) order, with no comparator.
//
// The writer behind mergeAll appends every record with rle = false (:1092), and Writer.append frames a record exactly as
// its input framed it, so an output body is the input bodies without their FF FF EOF markers, back to back, then one
// EOF.  The write is therefore a copy, not a parse: the headers, EOF markers and checksums of the inputs are checked at
// open, one batched kernel copies the record bytes, and the output checksum is derived from the input checksums
// without reading the bytes again.  No parse, stage, sort, tie or emit kernel runs.  next_batch parses on its first call
// (run table or window parser) and runs the merger's batch kernels over the identity order.
#pragma once
#include "codec.cuh"

namespace tezgpu {

// raw remainder of the record bytes R of a body R || FF FF, from the raw remainder of the whole body:
//   rem(R || FF FF) = rem(R) * x^16  xor  rem(FF FF),  and x^16 is invertible modulo the (primitive) polynomial
__host__ __device__ __forceinline__ uint32_t concat_records_raw(uint32_t body_raw, const CrcTables &t) {
  return crc_multmodp(body_raw ^ t.eof_raw, t.xinv16);
}

// One thread per input segment: checks the EOF marker and places the raw remainder of the segment's record bytes in
// its output body, tc[s] = (rem(R_s), partition, bytes that follow R_s there), for k_crc_combine's crc(A||B) rule.
// A segment whose trailer is its verified checksum contributes that trailer; every other one the remainder
// k_crc_pieces computed (for a checked segment the two are equal).
__global__ void k_concat_inputs(const uint8_t *__restrict__ data, const SegDesc *__restrict__ segs, uint32_t nseg,
                                const uint32_t *__restrict__ seg_crc, const uint64_t *__restrict__ after,
                                const CrcTables *__restrict__ t, TileCrc *__restrict__ tc, int *__restrict__ bad_eof) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const SegDesc sd = segs[s];
  const uint64_t body = sd.body_end - sd.body0;   // >= 2: open() refuses shorter segments
  const uint8_t *b = data + sd.off + sd.body0;
  if (b[body - 2] != 0xFF || b[body - 1] != 0xFF) atomicExch(bad_eof, (int)s + 1);
  const bool trusted = (sd.has_header & 2u) && !(sd.has_header & 4u);
  const uint32_t body_raw = trusted ? crc_to_raw(t, load_be32(data + sd.off + sd.body_end), body) : seg_crc[s];
  TileCrc c;
  c.raw = concat_records_raw(body_raw, *t);
  c.p = sd.partition;
  c.after = after[s];
  tc[s] = c;
}

// ------------------------------------------------------------------------------------------------ batched copy
// A unit is at most CAT_UNIT bytes of one input's records and their place in the output.  Each CTA copies a contiguous
// range of units, so many small segments cost no extra launches.  Source and destination have arbitrary relative
// alignment: the destination is written in aligned 16-byte stores, each built from two aligned 16-byte loads of the
// source with a funnel shift by the misalignment (the technique of k_emit_fast4u).
struct CatUnit {
  uint64_t src;   // offset in the merger's segment bytes
  uint64_t dst;   // offset in the output
  uint64_t len;
};
constexpr int CAT_THREADS = 256;
constexpr uint64_t CAT_UNIT = 128 * 1024;

// blocks i of the destination from source words starting Q words (+ r bits) into the aligned source block
template <int Q>
__device__ __forceinline__ void cat_shifted_blocks(const uint4 *__restrict__ sa, uint4 *__restrict__ o, uint64_t nblk, uint32_t r) {
#pragma unroll 4
  for (uint64_t i = threadIdx.x; i < nblk; i += CAT_THREADS) {
    const uint4 a = __ldg(sa + i), b = __ldg(sa + i + 1);   // b holds at least one wanted byte: never past the source
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    o[i] = make_uint4(__funnelshift_r(w[Q], w[Q + 1], r), __funnelshift_r(w[Q + 1], w[Q + 2], r),
                      __funnelshift_r(w[Q + 2], w[Q + 3], r), __funnelshift_r(w[Q + 3], w[Q + 4], r));
  }
}

__global__ void __launch_bounds__(CAT_THREADS)
    k_concat_copy(const uint8_t *__restrict__ data, const CatUnit *__restrict__ units, uint32_t nunits, uint8_t *__restrict__ out) {
  const uint32_t u0 = (uint32_t)((uint64_t)blockIdx.x * nunits / gridDim.x);
  const uint32_t u1 = (uint32_t)((uint64_t)(blockIdx.x + 1) * nunits / gridDim.x);
  for (uint32_t u = u0; u < u1; u++) {
    const CatUnit cu = units[u];
    const uint8_t *s = data + cu.src;
    uint8_t *o = out + cu.dst;
    const uint64_t lead = (16u - (uint32_t)((uintptr_t)o & 15u)) & 15u;
    const uint32_t head = (uint32_t)(cu.len < lead ? cu.len : lead);
    if (threadIdx.x < head) o[threadIdx.x] = s[threadIdx.x];
    const uint64_t nblk = (cu.len - head) >> 4;
    const uint8_t *s1 = s + head;
    uint4 *o1 = reinterpret_cast<uint4 *>(o + head);
    const uint32_t mis = (uint32_t)((uintptr_t)s1 & 15u), r = 8u * (mis & 3u);
    const uint4 *sa = reinterpret_cast<const uint4 *>(s1 - mis);
    switch (mis >> 2) {
      case 0:
        if (!mis) {
#pragma unroll 4
          for (uint64_t i = threadIdx.x; i < nblk; i += CAT_THREADS) o1[i] = __ldg(sa + i);
        } else {
          cat_shifted_blocks<0>(sa, o1, nblk, r);
        }
        break;
      case 1: cat_shifted_blocks<1>(sa, o1, nblk, r); break;
      case 2: cat_shifted_blocks<2>(sa, o1, nblk, r); break;
      default: cat_shifted_blocks<3>(sa, o1, nblk, r); break;
    }
    const uint64_t done = head + (nblk << 4);   // fewer than 16 bytes remain
    if (threadIdx.x < cu.len - done) o[done + threadIdx.x] = s[done + threadIdx.x];
  }
}

// one output segment per partition with records: TIF\0 | records (copied) | FF FF | CRC-32.  seg_crc[p] is the xor of
// rem(R_s) * x^(8 * bytes after R_s) over the partition's inputs, i.e. rem(records) * x^16.
struct CatPart {
  uint64_t start;   // segment offset in the output
  uint64_t rec;     // record bytes; 0 = no segment
};
__global__ void k_concat_finish(const CatPart *__restrict__ parts, uint32_t P, const uint32_t *__restrict__ seg_crc,
                                const CrcTables *__restrict__ t, uint8_t *__restrict__ out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const CatPart c = parts[p];
  if (!c.rec) return;
  uint8_t *o = out + c.start;
  o[0] = 'T'; o[1] = 'I'; o[2] = 'F'; o[3] = 0;
  o[4 + c.rec] = 0xFF;
  o[5 + c.rec] = 0xFF;
  const uint64_t body = c.rec + 2;
  const uint32_t crc = crc_from_raw(t, seg_crc[p] ^ t->eof_raw, body);
  store_be32(o + 4 + body, crc);
}

// ------------------------------------------------------------------------------------------------ record iterator
// run-table mode for declared fixed widths: every record's framing bytes must be the fixed header (an input written
// with REPEAT_KEY markers is not), else the window parser takes over
__global__ void k_concat_check_fixed(const uint8_t *__restrict__ data, const SegDesc *__restrict__ segs, uint32_t nseg,
                                     const uint64_t *__restrict__ rec_base, uint32_t rs, uint32_t hl, uint64_t hdr,
                                     int *__restrict__ bad) {
  const uint64_t total = rec_base[nseg];
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = nseg;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (rec_base[mid] <= i) lo = mid; else hi = mid;
    }
    const SegDesc sd = segs[lo];
    const uint8_t *rp = data + sd.off + sd.body0 + (i - rec_base[lo]) * rs;
    for (uint32_t b = 0; b < hl; b++)
      if (rp[b] != (uint8_t)(hdr >> (8 * b))) { atomicExch(bad, 1); return; }
  }
}

__global__ void k_iota(uint32_t *__restrict__ v, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v[i] = i;
}

// ------------------------------------------------------------------------------------------------ host side
// called by open() after the header and checksum kernels: record bytes per input and their remainders
inline void Merger::concat_inputs(uint32_t nseg, int *d_bad_eof) {
  cudaStream_t st = pipe.stream;
  concat_parsed = false;
  parse_mode = 3;
  parse_rounds = 0;
  n = kv_bytes = cursor = 0;
  have_kvoff = false;
  cat_rec.resize(nseg);
  concat_bytes = 0;
  for (uint32_t s = 0; s < nseg; s++) {
    cat_rec[s] = segs[s].body_end - segs[s].body0 - 2;
    concat_bytes += cat_rec[s] + 2;
  }
  if (!nseg) return;
  // bytes that follow each input's records in its partition's body (segs are partition-major), EOF markers included
  std::vector<uint64_t> after(nseg);
  uint64_t acc = 0;
  for (uint32_t s = nseg; s-- > 0;) {
    if (s + 1 == nseg || segs[s + 1].partition != segs[s].partition) acc = 2;
    after[s] = acc;
    acc += cat_rec[s];
  }
  d_cat_units.ensure((size_t)nseg * 8);   // holds `after` until the write lays its units out
  d_cat_tc.ensure((size_t)nseg * sizeof(TileCrc));
  d_seg_crc.ensure((size_t)nseg * 4);
  TG_CUDA(cudaMemcpyAsync(d_cat_units.p, after.data(), (size_t)nseg * 8, cudaMemcpyHostToDevice, st));
  k_concat_inputs<<<(uint32_t)div_up(nseg, 128), 128, 0, st>>>(data, d_segs.as<SegDesc>(), nseg, d_seg_crc.as<uint32_t>(),
                                                              d_cat_units.as<uint64_t>(), DeviceConstants::get(pipe.conf.device).d_crc,
                                                              d_cat_tc.as<TileCrc>(), d_bad_eof);
  launches++;
  TG_CUDA(cudaGetLastError());
  TG_CUDA(cudaStreamSynchronize(st));   // `after` is a stack-lifetime vector
}

inline void Merger::concat_write(uint8_t *d_out_buf, uint64_t cap, int writer_rle, uint64_t *out_len, int64_t *index,
                                 tezgpu_stats *stats) {
  TG_CHECK(writer_rle == 0, TEZGPU_E_INVALID,
           "rle " + std::to_string(writer_rle) + ": a concatenating merger writes without run-length encoding (rle must be 0)");
  cudaStream_t st = pipe.stream;
  const int P = pipe.conf.num_partitions;
  const uint32_t nseg = (uint32_t)segs.size();
  EventTimer &tm = pipe.timer;
  tm.reset();
  tm.mark(st);
  // layout: partition p's segment is TIF\0, its inputs' records in segs order, FF FF, CRC; no bytes and an all-zero
  // index entry for a partition without records (mergeAll :1087-1091)
  std::vector<CatPart> parts((size_t)P);
  for (uint32_t s = 0; s < nseg; s++) parts[segs[s].partition].rec += cat_rec[s];
  std::vector<int64_t> raw_index((size_t)P * 3, 0);
  uint64_t total = 0;
  int64_t raw_sum = 0;
  for (int p = 0; p < P; p++) {
    parts[p].start = total;
    if (!parts[p].rec) continue;
    const uint64_t seglen = parts[p].rec + 10;
    raw_index[3 * p] = (int64_t)total;
    raw_index[3 * p + 1] = (int64_t)seglen - 4;   // rawLength: header + body, no checksum
    raw_index[3 * p + 2] = (int64_t)seglen;
    raw_sum += (int64_t)seglen - 4;
    total += seglen;
  }
  const bool zc = pipe.codec != TEZGPU_CODEC_NONE;
  uint8_t *img = d_out_buf;
  if (zc) {
    pipe.z_img.ensure(total + 64);
    img = pipe.z_img.as<uint8_t>();
  } else {
    TG_CHECK(total <= cap, TEZGPU_E_NOMEM, "output buffer too small for the concatenated file.out");
  }
  std::vector<CatUnit> units;
  uint64_t dst = 0;
  for (uint32_t s = 0; s < nseg; s++) {
    if (s == 0 || segs[s].partition != segs[s - 1].partition) dst = parts[segs[s].partition].start + 4;
    for (uint64_t o = 0; o < cat_rec[s]; o += CAT_UNIT)
      units.push_back({segs[s].off + segs[s].body0 + o, dst + o, std::min<uint64_t>(CAT_UNIT, cat_rec[s] - o)});
    dst += cat_rec[s];
  }
  TG_CHECK(units.size() < (1ull << 32), TEZGPU_E_INVALID, "segments too large for one concatenation");
  int nl = 0;
  if (!units.empty()) {
    d_cat_units.ensure(units.size() * sizeof(CatUnit));
    TG_CUDA(cudaMemcpyAsync(d_cat_units.p, units.data(), units.size() * sizeof(CatUnit), cudaMemcpyHostToDevice, st));
    const uint32_t grid = (uint32_t)std::min<uint64_t>(units.size(), (uint64_t)pipe.num_sms * 8);
    k_concat_copy<<<grid, CAT_THREADS, 0, st>>>(data, d_cat_units.as<CatUnit>(), (uint32_t)units.size(), img);
    nl++;
  }
  if (total) {
    const CrcTables *d_crc = DeviceConstants::get(pipe.conf.device).d_crc;
    pipe.seg_crc.ensure((size_t)P * 4);
    d_cat_parts.ensure((size_t)P * sizeof(CatPart));
    TG_CUDA(cudaMemsetAsync(pipe.seg_crc.p, 0, (size_t)P * 4, st));
    TG_CUDA(cudaMemcpyAsync(d_cat_parts.p, parts.data(), (size_t)P * sizeof(CatPart), cudaMemcpyHostToDevice, st));
    k_crc_combine<<<(uint32_t)div_up(nseg, 256), 256, 0, st>>>(d_cat_tc.as<TileCrc>(), nseg, d_crc, pipe.seg_crc.as<uint32_t>());
    k_concat_finish<<<(uint32_t)div_up(P, 128), 128, 0, st>>>(d_cat_parts.as<CatPart>(), (uint32_t)P, pipe.seg_crc.as<uint32_t>(), d_crc, img);
    nl += 2;
  }
  TG_CUDA(cudaGetLastError());
  tm.mark(st);
  TG_CUDA(cudaStreamSynchronize(st));   // units / parts are stack-lifetime vectors
  tezgpu_stats s;
  memset(&s, 0, sizeof(s));
  if (zc) {
    pipe.compress_image(raw_index.data(), d_out_buf, cap, out_len, index, &s);
  } else {
    if (out_len) *out_len = total;
    if (index) memcpy(index, raw_index.data(), (size_t)P * 24);
    s.output_bytes_physical = s.file_out_bytes = (int64_t)total;
  }
  // records are not counted here: the write does not parse (tezgpu_merge_counts does)
  s.output_bytes_with_overhead = raw_sum;
  s.num_spills = 1;
  s.kernel_launches += launches + nl;
  s.ms_total += tm.ms(0, 1);
  if (stats) *stats = s;
}

// next_batch / counts: find the records (run table or window parser), then the identity order with no SAME_KEY
inline void Merger::concat_parse() {
  if (concat_parsed) return;
  cudaStream_t st = pipe.stream;
  const uint32_t nseg = (uint32_t)segs.size();
  bool fixed_ok = count_fixed_records(nseg, 8);
  if (fixed_ok) {
    const FixedFraming f = fixed_framing(fixed_klen, fixed_vlen);
    int *d_bad = &pipe.d_scratch()->verdict.error;
    TG_CUDA(cudaMemsetAsync(d_bad, 0, 4, st));
    int bad = 0;
    launches += fill_fixed_arrays();
    if (n) {
      k_concat_check_fixed<<<record_grid(), 256, 0, st>>>(data, d_segs.as<SegDesc>(), nseg, d_rec_base.as<uint64_t>(), f.rec_size,
                                                          f.len, f.packed(), d_bad);
      launches++;
      TG_CUDA(cudaGetLastError());
      TG_CUDA(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, st));
    }
    TG_CUDA(cudaStreamSynchronize(st));
    fixed_ok = bad == 0;
    parse_mode = 0;
    parse_rounds = 0;
  }
  if (!fixed_ok) {
    find_records_general(nseg);
    if (!nseg) parse_mode = 1;
  }
  arrays_ready = true;
  pipe.state.rec = array_records();
  d_order.ensure((size_t)(n ? n : 1) * 4);
  pipe.same.ensure(n ? n : 1);
  TG_CUDA(cudaMemsetAsync(pipe.same.p, 0, n ? n : 1, st));
  if (n) {
    k_iota<<<record_grid(), 256, 0, st>>>(d_order.as<uint32_t>(), (uint32_t)n);
    launches++;
  }
  TG_CUDA(cudaGetLastError());
  pipe.state.order = d_order.as<uint32_t>();
  cursor = 0;
  have_kvoff = false;
  concat_parsed = true;
}

}  // namespace tezgpu

// codec.cuh -- DefaultCodec, Lz4Codec, ZStandardCodec and SnappyCodec on both sides of the shuffle: the compress phase
// behind every emit (SortPipeline) and the decompress step in front of every merge open (Merger).  Formats, chunk
// kernels and decoders: deflate.cuh, inflate.cuh (DefaultCodec), lz4.cuh (Lz4Codec), zstd.cuh (ZStandardCodec),
// snappy.cuh (SnappyCodec).  What the codecs share is here: the segment layout and its kernels, the finish of LZ4, zstd
// and Snappy segments, the reader's staging and checksum check, its block-parallel sequence for LZ4 and zstd, and the
// writers' host runs.
#pragma once
#include <memory>
#include "inflate.cuh"
#include "lz4.cuh"
#include "zstd.cuh"
#include "snappy.cuh"
#include "merger.cuh"

namespace tezgpu {

// the codecs the device writes and reads (TEZGPU_CODEC_*)
inline void check_codec(int32_t codec) {
  TG_CHECK(codec == TEZGPU_CODEC_NONE || codec == TEZGPU_CODEC_DEFAULT || codec == TEZGPU_CODEC_LZ4 || codec == TEZGPU_CODEC_ZSTD ||
               codec == TEZGPU_CODEC_SNAPPY,
           TEZGPU_E_UNSUPPORTED, "codec " + std::to_string(codec) + " is not on the device (DefaultCodec, Lz4Codec, ZStandardCodec and SnappyCodec only)");
}

// How a codec's compressed segment is laid out around its chunks.  zlib: 32 KiB chunks, framed by
// TIF\x01 78 01 | chunks | Adler-32 CRC; LZ4 and Snappy: blocks of one chunk each (their 8 header bytes in the slot),
// framed by TIF\x01 | blocks | CRC; zstd: one frame per chunk, framed by TIF\x01 | frames | CRC.
struct CodecLayout {
  uint64_t chunk;   // body bytes per chunk
  uint32_t slot;    // device bytes reserved per compressed chunk
  uint32_t frame;   // segment bytes outside the chunks
  uint32_t head;    // segment bytes before the first chunk
  uint32_t tail;    // checksummed bytes after the last chunk
};
inline CodecLayout codec_layout(int32_t codec) {
  switch (codec) {
    case TEZGPU_CODEC_LZ4: return {L4_BLOCK, L4_SLOT, 8, 4, 0};
    case TEZGPU_CODEC_ZSTD: return {ZS_BLOCK, ZS_SLOT, 8, 4, 0};
    case TEZGPU_CODEC_SNAPPY: return {SN_BLOCK, SN_SLOT, 8, 4, 0};
    default: return {ZCHUNK, ZSLOT, 14, 6, 4};
  }
}

// ------------------------------------------------------------------------------------------------ writer kernels
// chunk descriptors for k_crc_pieces (one piece per chunk: a chunk is < CRC_PIECE bytes); slot: bytes per chunk slot
__global__ void k_zchunk_descs(const uint32_t *__restrict__ csize, uint32_t nchunks, uint32_t slot, SegDesc *__restrict__ descs,
                               uint32_t *__restrict__ piece_start) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > nchunks) return;
  piece_start[c] = c;
  if (c == nchunks) return;
  SegDesc d;
  d.off = (uint64_t)c * slot;
  d.len = csize[c] + 4;
  d.body0 = 0;
  d.body_end = csize[c];
  d.has_header = 1;
  d.partition = 0;
  descs[c] = d;
}

// per partition: file offset and length of its compressed segment; frame: bytes of a segment outside its chunks
__global__ void k_zseg_layout(ZSeg *__restrict__ segs, uint32_t P, const uint64_t *__restrict__ coff, uint32_t frame) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  ZSeg &s = segs[p];
  s.zstart = coff[s.chunk0] + frame * s.rank;
  s.zlen = s.nchunks ? coff[s.chunk0 + s.nchunks] - coff[s.chunk0] + frame : 0;
}

// chunk checksums -> positions in their segment's checksummed bytes (zlib: header, chunks, Adler-32; LZ4 and zstd: the
// chunks); tail: checksummed bytes after the last chunk
__global__ void k_zcrc_place(TileCrc *__restrict__ tc, uint32_t nchunks, const ZSeg *__restrict__ segs, uint32_t P,
                             const uint64_t *__restrict__ coff, uint32_t tail) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nchunks) return;
  const uint32_t p = z_chunk_part(segs, P, c);
  const ZSeg s = segs[p];
  tc[c].p = p;
  tc[c].after = coff[s.chunk0 + s.nchunks] - coff[c + 1] + tail;
}

// one CTA per chunk: the chunk's bytes into the file (slot: bytes per chunk slot; head: segment bytes before the chunks)
__global__ void k_zpack(const uint8_t *__restrict__ slots, const uint32_t *__restrict__ csize, const uint64_t *__restrict__ coff,
                        const ZSeg *__restrict__ segs, uint32_t P, uint32_t slot, uint32_t head, uint8_t *__restrict__ out) {
  const uint32_t c = blockIdx.x;
  const ZSeg s = segs[z_chunk_part(segs, P, c)];
  uint8_t *dst = out + s.zstart + head + (coff[c] - coff[s.chunk0]);
  const uint8_t *src = slots + (uint64_t)c * slot;
  const uint32_t n = csize[c];
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// per block-framed (LZ4, zstd, Snappy) segment: TIF\x01 and the CRC-32 of the stream (the chunks' raw remainders are in seg_crc)
__global__ void k_zfinish_blocks(const ZSeg *__restrict__ segs, uint32_t P, const uint32_t *__restrict__ seg_crc,
                                 const CrcTables *__restrict__ t, uint8_t *__restrict__ out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const ZSeg s = segs[p];
  if (!s.nchunks) return;
  uint8_t *o = out + s.zstart;
  o[0] = 'T'; o[1] = 'I'; o[2] = 'F'; o[3] = 1;
  const uint32_t crc = crc_from_raw(t, seg_crc[p], s.zlen - 8);
  store_be32(o + s.zlen - 4, crc);
}

// The chunks of the segments hs[0, nseg) in codec zc (host table: body_off into img, body_len, chunk0, nchunks, rank,
// open; nchunks chunks in all, at least one): each compressed into its slot of z_slots (sizes z_csize, zlib's Adler-32 values
// z_cadler), their file offsets z_coff, the segments' zstart / zlen (frame: segment bytes outside its chunks) back in
// hs and on the device in z_segs, and z_crc[s] = the raw CRC remainder of segment s's chunk bytes followed by `tail`
// zero bytes.  One host round trip (the layout).  Returns the chunk bytes; *launches counts the kernels.
inline uint64_t SortPipeline::compress_chunks(int32_t zc, const uint8_t *img, ZSeg *hs, uint32_t nseg, uint32_t nchunks,
                                              uint32_t frame, uint32_t tail, int *launches) {
  cudaStream_t st = stream;
  const CodecLayout L = codec_layout(zc);
  z_segs.ensure((size_t)nseg * sizeof(ZSeg));
  TG_CUDA(cudaMemcpyAsync(z_segs.p, hs, (size_t)nseg * sizeof(ZSeg), cudaMemcpyHostToDevice, st));
  z_slots.ensure((size_t)nchunks * L.slot);
  z_csize.ensure((size_t)nchunks * 4);
  z_coff.ensure(((size_t)nchunks + 2) * 8);
  switch (zc) {
    case TEZGPU_CODEC_LZ4:
      set_smem_limit<k_l4compress>(conf.device, sizeof(L4Shared));
      k_l4compress<<<nchunks, L4_LANES, sizeof(L4Shared), st>>>(img, z_segs.as<ZSeg>(), nseg, z_slots.as<uint8_t>(), z_csize.as<uint32_t>());
      break;
    case TEZGPU_CODEC_ZSTD:
      set_smem_limit<k_zscompress>(conf.device, sizeof(ZsShared));
      k_zscompress<<<nchunks, ZS_LANES, sizeof(ZsShared), st>>>(img, z_segs.as<ZSeg>(), nseg, z_slots.as<uint8_t>(), z_csize.as<uint32_t>());
      break;
    case TEZGPU_CODEC_SNAPPY:
      set_smem_limit<k_sncompress>(conf.device, sizeof(SnShared));
      k_sncompress<<<nchunks, SN_LANES, sizeof(SnShared), st>>>(img, z_segs.as<ZSeg>(), nseg, z_slots.as<uint8_t>(), z_csize.as<uint32_t>());
      break;
    default:
      set_smem_limit<k_zdeflate>(conf.device, sizeof(ZShared));
      z_cadler.ensure((size_t)nchunks * 4);
      k_zdeflate<<<nchunks, ZLANES, sizeof(ZShared), st>>>(img, z_segs.as<ZSeg>(), nseg, z_slots.as<uint8_t>(), z_csize.as<uint32_t>(),
                                                          z_cadler.as<uint32_t>());
  }
  *launches += 1 + scan_u32_exclusive(st, blk, z_csize.as<uint32_t>(), nchunks, z_coff.as<uint64_t>());
  k_zseg_layout<<<(uint32_t)div_up(nseg, 128), 128, 0, st>>>(z_segs.as<ZSeg>(), nseg, z_coff.as<uint64_t>(), frame);
  // checksums of the chunks (k_crc_pieces, one piece per chunk), placed in their segments and folded per segment
  const CrcTables *d_crc = DeviceConstants::get(conf.device).d_crc;
  z_descs.ensure((size_t)nchunks * sizeof(SegDesc));
  z_pstart.ensure(((size_t)nchunks + 1) * 4);
  z_tc.ensure((size_t)nchunks * sizeof(TileCrc));
  z_crc.ensure((size_t)nseg * 4);
  TG_CUDA(cudaMemsetAsync(z_crc.p, 0, (size_t)nseg * 4, st));
  k_zchunk_descs<<<(uint32_t)div_up((uint64_t)nchunks + 1, 256), 256, 0, st>>>(z_csize.as<uint32_t>(), nchunks, L.slot,
                                                                            z_descs.as<SegDesc>(), z_pstart.as<uint32_t>());
  k_crc_pieces<<<nchunks, CRCV_THREADS, 0, st>>>(z_slots.as<uint8_t>(), z_descs.as<SegDesc>(), z_pstart.as<uint32_t>(), nchunks, d_crc,
                                                 z_tc.as<TileCrc>());
  k_zcrc_place<<<(uint32_t)div_up(nchunks, 256), 256, 0, st>>>(z_tc.as<TileCrc>(), nchunks, z_segs.as<ZSeg>(), nseg,
                                                              z_coff.as<uint64_t>(), tail);
  k_crc_combine<<<(uint32_t)div_up(nchunks, 256), 256, 0, st>>>(z_tc.as<TileCrc>(), nchunks, d_crc, z_crc.as<uint32_t>());
  *launches += 5;
  TG_CUDA(cudaGetLastError());
  TG_CUDA(cudaMemcpyAsync(hs, z_segs.p, (size_t)nseg * sizeof(ZSeg), cudaMemcpyDeviceToHost, st));
  TG_CUDA(cudaMemcpyAsync(reinterpret_cast<uint8_t *>(hs) + (size_t)nseg * sizeof(ZSeg), z_coff.as<uint64_t>() + nchunks, 8,
                          cudaMemcpyDeviceToHost, st));
  TG_CUDA(cudaStreamSynchronize(st));
  uint64_t cbytes;
  memcpy(&cbytes, reinterpret_cast<uint8_t *>(hs) + (size_t)nseg * sizeof(ZSeg), 8);
  return cbytes;
}

// The uncompressed file is in z_img with its index raw_index (start, rawLength, partLength per partition).  Every
// partition that has a segment gets a compressed one: TIF\x01, the codec stream of the same body (zlib, or LZ4 blocks),
// CRC-32 of the stream.  index receives (start, the same rawLength, compressed length).  One host round trip (the
// compressed layout).
inline void SortPipeline::compress_image(const int64_t *raw_index, uint8_t *d_out, uint64_t out_cap, uint64_t *out_len,
                                         int64_t *index, tezgpu_stats *stats) {
  const int P = conf.num_partitions;
  cudaStream_t st = stream;
  const CodecLayout L = codec_layout(codec);
  z_timer.reset();
  z_timer.mark(st);
  z_host.ensure((size_t)P * sizeof(ZSeg) + 64);
  ZSeg *hs = z_host.as<ZSeg>();
  uint32_t nchunks = 0;
  uint64_t nsegs = 0;
  for (int p = 0; p < P; p++) {
    const int64_t start = raw_index[3 * p], part = raw_index[3 * p + 2];
    ZSeg &s = hs[p];
    memset(&s, 0, sizeof(s));
    s.chunk0 = nchunks;
    s.rank = nsegs;
    if (part > 0) {
      s.body_off = (uint64_t)start + 4;
      s.body_len = (uint64_t)part - 8;
      s.nchunks = (uint32_t)std::max<uint64_t>(1, div_up(s.body_len, L.chunk));
      nchunks += s.nchunks;
      nsegs++;
    }
  }
  int launches = 0;
  uint64_t total = 0;
  if (nchunks) {
    const uint64_t cbytes = compress_chunks(codec, z_img.as<uint8_t>(), hs, (uint32_t)P, nchunks, L.frame, L.tail, &launches);
    total = cbytes + L.frame * nsegs;
    TG_CHECK(total <= out_cap, TEZGPU_E_NOMEM, "output buffer too small for the compressed file.out");
    const CrcTables *d_crc = DeviceConstants::get(conf.device).d_crc;
    k_zpack<<<nchunks, 256, 0, st>>>(z_slots.as<uint8_t>(), z_csize.as<uint32_t>(), z_coff.as<uint64_t>(), z_segs.as<ZSeg>(), (uint32_t)P,
                                     L.slot, L.head, d_out);
    switch (codec) {
      case TEZGPU_CODEC_LZ4:
      case TEZGPU_CODEC_ZSTD:
      case TEZGPU_CODEC_SNAPPY:
        k_zfinish_blocks<<<(uint32_t)div_up(P, 128), 128, 0, st>>>(z_segs.as<ZSeg>(), (uint32_t)P, z_crc.as<uint32_t>(), d_crc, d_out);
        break;
      default:
        k_zfinish<<<(uint32_t)div_up(P, 128), 128, 0, st>>>(z_segs.as<ZSeg>(), (uint32_t)P, z_cadler.as<uint32_t>(), z_csize.as<uint32_t>(),
                                                           z_crc.as<uint32_t>(), d_crc, d_out);
    }
    launches += 2;
    TG_CUDA(cudaGetLastError());
  }
  z_timer.mark(st);
  TG_CUDA(cudaStreamSynchronize(st));
  if (out_len) *out_len = total;
  if (index) {
    for (int p = 0; p < P; p++) {
      const int64_t start = raw_index[3 * p], raw = raw_index[3 * p + 1], part = raw_index[3 * p + 2];
      const uint64_t zstart = nchunks ? hs[p].zstart : 0;
      index[3 * p] = part > 0 ? (int64_t)zstart : (start == 0 ? 0 : (int64_t)zstart);
      index[3 * p + 1] = raw;
      index[3 * p + 2] = part > 0 ? (int64_t)hs[p].zlen : 0;
    }
  }
  if (stats) {
    stats->output_bytes_physical = (int64_t)total;
    stats->file_out_bytes = (int64_t)total;
    stats->ms_total += z_timer.ms(0, 1);
    stats->kernel_launches += launches;
  }
}

// the name of status rc of a codec's reader (0: "ok")
static inline const char *codec_err_name(int32_t codec, int32_t rc) {
  switch (codec) {
    case TEZGPU_CODEC_LZ4: return l4_err_name(rc);
    case TEZGPU_CODEC_ZSTD: return zs_err_name(rc);
    case TEZGPU_CODEC_SNAPPY: return sn_err_name(rc);
    default: return z_err_name(rc);
  }
}

inline void check_raw_len(uint32_t s, int64_t raw) {
  TG_CHECK(raw >= 6 && raw < (1ll << 40), TEZGPU_E_INVALID,
           "segment " + std::to_string(s) + ": raw length " + std::to_string(raw) + " is not a valid IFile rawLength");
}

// The caller's indices of the compressed segments: header TIF and flag byte 1.  Headers of device segments are read
// through `st`.
inline std::vector<uint32_t> compressed_segments(const tezgpu_segment *in, uint32_t nseg, cudaStream_t st) {
  std::vector<uint8_t> hdr((size_t)nseg * 4, 0);
  bool on_device = false;
  for (uint32_t s = 0; s < nseg; s++) {
    if (!(in[s].flags & TEZGPU_SEG_HAS_HEADER) || in[s].len < 10 || !in[s].data) continue;
    if (in[s].flags & TEZGPU_SEG_DEVICE) {
      TG_CUDA(cudaMemcpyAsync(&hdr[4 * (size_t)s], in[s].data, 4, cudaMemcpyDeviceToHost, st));
      on_device = true;
    } else {
      memcpy(&hdr[4 * (size_t)s], in[s].data, 4);
    }
  }
  if (on_device) TG_CUDA(cudaStreamSynchronize(st));
  std::vector<uint32_t> zs;
  for (uint32_t s = 0; s < nseg; s++)
    if (hdr[4 * s] == 'T' && hdr[4 * s + 1] == 'I' && hdr[4 * s + 2] == 'F' && hdr[4 * s + 3] == 1) zs.push_back(s);
  return zs;
}

// Compressed segments go through decode_compressed, and their images TIF\x00 + body + 4 bytes are merged as verified
// ordinary segments.  Every other segment goes to open() unchanged, so errors keep naming the caller's segment index.
inline void Merger::open_codec(const tezgpu_segment *in, const int64_t *raw_len, uint32_t nseg) {
  if (!pipe.codec) { open(in, nseg); return; }
  const std::vector<uint32_t> zs = compressed_segments(in, nseg, pipe.stream);
  if (zs.empty()) { open(in, nseg); return; }
  decode_compressed(in, raw_len, zs);
  std::vector<tezgpu_segment> segs2(in, in + nseg);
  for (size_t i = 0; i < zs.size(); i++) {
    tezgpu_segment &sg = segs2[zs[i]];
    sg.data = z_img.as<uint8_t>() + z_img_off[i];
    sg.len = (uint64_t)raw_len[zs[i]] + 4;
    sg.flags = TEZGPU_SEG_HAS_HEADER | TEZGPU_SEG_DEVICE | TEZGPU_SEG_VERIFIED | SEG_DECODED;
  }
  open(segs2.data(), nseg);
}

// The segments zs of `in` (caller's indices, all compressed) are staged, their CRC checked (unless the transport
// verified it), and decompressed into images at z_img + z_img_off[i]: TIF\x00, the body, 4 zero bytes.  zlib: one warp
// per segment.  LZ4: one thread per segment walks the block headers (one host round trip for the block count), one warp
// per block decodes, and a segment the block pass could not take is decoded again serially by one warp.  zstd: the same
// shape with frames: a segment whose frames all carry Frame_Content_Size is decoded one warp per frame, any other one
// warp per segment.  Snappy: the walk makes every chunk a unit (each states its raw length), one warp per chunk
// decodes, and each segment reports its first error in stream order.  Returns once every image is complete; errors name the caller's segment index.
inline void Merger::decode_compressed(const tezgpu_segment *in, const int64_t *raw_len, const std::vector<uint32_t> &zs) {
  cudaStream_t st = pipe.stream;
  TG_CHECK(raw_len, TEZGPU_E_INVALID, "segment " + std::to_string(zs[0]) + " is compressed: its raw length is required");
  const uint32_t nz = (uint32_t)zs.size();
  uint64_t in_bytes = 0, img_bytes = 0;
  std::vector<uint64_t> in_off(nz), img_off(nz);
  // device segments the transport verified are inflated in place; the others are staged for the checksum kernels
  auto in_place = [&](const tezgpu_segment &sg) {
    return (sg.flags & TEZGPU_SEG_DEVICE) && (sg.flags & TEZGPU_SEG_VERIFIED);
  };
  for (uint32_t i = 0; i < nz; i++) {
    const uint32_t s = zs[i];
    check_raw_len(s, raw_len[s]);
    in_off[i] = in_bytes;
    if (!in_place(in[s])) in_bytes = align_up(in_bytes + in[s].len, 16);
    img_off[i] = img_bytes;
    img_bytes = align_up(img_bytes + (uint64_t)raw_len[s] + 4, 16);
  }
  z_in.ensure(in_bytes + 64);
  z_img.ensure(img_bytes + 64);
  std::vector<SegDesc> sd(nz);
  std::vector<ZInSeg> zi(nz);
  for (uint32_t i = 0; i < nz; i++) {
    const tezgpu_segment &sg = in[zs[i]];
    const bool inplace = in_place(sg);
    if (!inplace)
      TG_CUDA(cudaMemcpyAsync(z_in.as<uint8_t>() + in_off[i], sg.data, sg.len,
                              (sg.flags & TEZGPU_SEG_DEVICE) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    sd[i].off = in_off[i];
    sd[i].len = sg.len;
    sd[i].body0 = 4;
    sd[i].body_end = sg.len - 4;
    sd[i].has_header = 1u | ((sg.flags & TEZGPU_SEG_VERIFIED) ? 2u : 0u);
    sd[i].partition = 0;
    zi[i].src = inplace ? static_cast<const uint8_t *>(sg.data) : z_in.as<uint8_t>() + in_off[i];
    zi[i].len = sg.len;
    zi[i].dst = z_img.as<uint8_t>() + img_off[i];
    zi[i].body = (uint64_t)raw_len[zs[i]] - 4;
  }
  z_descs.ensure((size_t)nz * sizeof(SegDesc));
  z_insegs.ensure((size_t)nz * sizeof(ZInSeg));
  z_status.ensure((size_t)nz * 4 + 16);
  z_flag.ensure(16);
  TG_CUDA(cudaMemcpyAsync(z_descs.p, sd.data(), (size_t)nz * sizeof(SegDesc), cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemcpyAsync(z_insegs.p, zi.data(), (size_t)nz * sizeof(ZInSeg), cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemsetAsync(z_flag.p, 0, 16, st));
  // checksums of the compressed bytes: the open() machinery over the staged segments.  piece_start lives until the
  // verdict read below; open() reuses the checksum buffers only after it.
  std::vector<uint32_t> piece_start;
  launches += check_checksums(z_in.as<uint8_t>(), sd, z_descs.as<SegDesc>(), [](const SegDesc &d) { return d.has_header == 1u; },
                              piece_start, false, z_flag.as<int>());
  // LZ4 and zstd: the count walk, one host round trip for the unit counts, the base table, the fill walk, one warp per
  // unit (`warps` per CTA), and the serial kernel, which decodes the segments the units did not take
  using Walk = void (*)(const ZInSeg *, uint32_t, uint32_t *, const uint32_t *, ZUnit *);
  using Units = void (*)(const ZUnit *, uint32_t, int32_t *);
  using Serial = void (*)(const ZInSeg *, uint32_t, const uint32_t *, const int32_t *, int32_t *);
  auto decode_units = [&](Walk count, Walk fill, Units units, Serial serial, uint32_t warps, const char *too_many) {
    z_nblk.ensure((size_t)nz * 4);
    z_slow.ensure((size_t)nz * 4);
    TG_CUDA(cudaMemsetAsync(z_slow.p, 0, (size_t)nz * 4, st));
    count<<<(uint32_t)div_up(nz, 128), 128, 0, st>>>(z_insegs.as<ZInSeg>(), nz, z_nblk.as<uint32_t>(), nullptr, nullptr);
    launches++;
    TG_CUDA(cudaGetLastError());
    std::vector<uint32_t> nunit(nz), base(nz);
    TG_CUDA(cudaMemcpyAsync(nunit.data(), z_nblk.p, (size_t)nz * 4, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));
    uint64_t nu = 0;
    for (uint32_t i = 0; i < nz; i++) { base[i] = (uint32_t)nu; nu += nunit[i]; }
    TG_CHECK(nu < (1ull << 32), TEZGPU_E_INVALID, too_many);
    if (nu) {
      z_base.ensure((size_t)nz * 4);
      z_blks.ensure((size_t)nu * sizeof(ZUnit));
      TG_CUDA(cudaMemcpyAsync(z_base.p, base.data(), (size_t)nz * 4, cudaMemcpyHostToDevice, st));
      fill<<<(uint32_t)div_up(nz, 128), 128, 0, st>>>(z_insegs.as<ZInSeg>(), nz, z_nblk.as<uint32_t>(), z_base.as<uint32_t>(), z_blks.as<ZUnit>());
      units<<<(uint32_t)div_up(nu, warps), warps * 32, 0, st>>>(z_blks.as<ZUnit>(), (uint32_t)nu, z_slow.as<int32_t>());
      launches += 2;
    }
    serial<<<(uint32_t)div_up(nz, warps), warps * 32, 0, st>>>(z_insegs.as<ZInSeg>(), nz, z_nblk.as<uint32_t>(), z_slow.as<int32_t>(),
                                                               z_status.as<int32_t>());
  };
  switch (pipe.codec) {
    case TEZGPU_CODEC_LZ4:
      decode_units(k_l4walk<0>, k_l4walk<1>, k_l4blocks, k_l4serial, L4DEC_WARPS, "too many LZ4 blocks in one merge");
      break;
    case TEZGPU_CODEC_ZSTD:
      decode_units(k_zswalk<0>, k_zswalk<1>, k_zsframes, k_zsserial, ZSD_WARPS, "too many zstd frames in one merge");
      break;
    case TEZGPU_CODEC_SNAPPY: {
      // the count walk (and the walk errors), one host round trip for the chunk counts, the fill walk, one warp per
      // chunk, and the image frames with each segment's first error
      z_nblk.ensure((size_t)nz * 4);
      z_slow.ensure((size_t)nz * 8);
      unsigned long long *err = reinterpret_cast<unsigned long long *>(z_slow.p);
      k_snwalk<0><<<(uint32_t)div_up(nz, 128), 128, 0, st>>>(z_insegs.as<ZInSeg>(), nz, z_nblk.as<uint32_t>(), nullptr, nullptr, err);
      launches++;
      TG_CUDA(cudaGetLastError());
      std::vector<uint32_t> nunit(nz), base(nz);
      TG_CUDA(cudaMemcpyAsync(nunit.data(), z_nblk.p, (size_t)nz * 4, cudaMemcpyDeviceToHost, st));
      TG_CUDA(cudaStreamSynchronize(st));
      uint64_t nu = 0;
      for (uint32_t i = 0; i < nz; i++) { base[i] = (uint32_t)nu; nu += nunit[i]; }
      TG_CHECK(nu < (1ull << 32), TEZGPU_E_INVALID, "too many Snappy chunks in one merge");
      if (nu) {
        z_base.ensure((size_t)nz * 4);
        z_blks.ensure((size_t)nu * sizeof(ZUnit));
        TG_CUDA(cudaMemcpyAsync(z_base.p, base.data(), (size_t)nz * 4, cudaMemcpyHostToDevice, st));
        k_snwalk<1><<<(uint32_t)div_up(nz, 128), 128, 0, st>>>(z_insegs.as<ZInSeg>(), nz, z_nblk.as<uint32_t>(), z_base.as<uint32_t>(),
                                                               z_blks.as<ZUnit>(), err);
        k_snchunks<<<(uint32_t)div_up(nu, SNDEC_WARPS), SNDEC_WARPS * 32, 0, st>>>(z_blks.as<ZUnit>(), (uint32_t)nu, err);
        launches += 2;
      }
      k_snfinish<<<(uint32_t)div_up(nz, 128), 128, 0, st>>>(z_insegs.as<ZInSeg>(), nz, err, z_status.as<int32_t>());
      break;
    }
    default:
      k_zinflate<<<(uint32_t)div_up(nz, ZINF_WARPS), ZINF_WARPS * 32, 0, st>>>(z_insegs.as<ZInSeg>(), nz, z_status.as<int32_t>());
  }
  launches++;
  TG_CUDA(cudaGetLastError());
  std::vector<int32_t> status(nz);
  int bad_crc = 0;
  TG_CUDA(cudaMemcpyAsync(status.data(), z_status.p, (size_t)nz * 4, cudaMemcpyDeviceToHost, st));
  TG_CUDA(cudaMemcpyAsync(&bad_crc, z_flag.p, 4, cudaMemcpyDeviceToHost, st));
  TG_CUDA(cudaStreamSynchronize(st));
  TG_CHECK(bad_crc == 0, TEZGPU_E_FORMAT, "IFile checksum mismatch in segment " + std::to_string(bad_crc ? zs[bad_crc - 1] : 0));
  for (uint32_t i = 0; i < nz; i++)
    TG_CHECK(status[i] == Z_OK, TEZGPU_E_FORMAT,
             std::string("compressed segment ") + std::to_string(zs[i]) + ": " + codec_err_name(pipe.codec, status[i]));
  z_img_off = img_off;
}

// the CRC-32 trailer of every image after its body, from the body's raw remainder in seg_crc
__global__ void k_image_trailers(uint8_t *__restrict__ img, const SegDesc *__restrict__ sd, uint32_t n,
                                 const uint32_t *__restrict__ seg_crc, const CrcTables *__restrict__ t) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const SegDesc d = sd[s];
  store_be32(img + d.off + d.body_end, crc_from_raw(t, seg_crc[s], d.body_end - d.body0));
}

// ---- tezgpu_decode_segments: the compressed host segments decoded into uncompressed IFile segments in host memory,
//      in groups that hold at most `budget` device bytes.  A group holds its staged compressed bytes, its images and
//      the decoder's workspace, bounded by decode_group_bytes; the buffers are released between groups, so the device
//      holds the Merger's own (`base`, measured by the caller) plus one group at a time.
constexpr uint64_t DECODE_FIXED_BYTES = 16 << 10;     // the 256-byte rounding of the group's buffers, their slack
constexpr uint64_t DECODE_BYTES_PER_SEGMENT = 128;    // descriptors, statuses, unit counts, piece starts, CRCs
constexpr uint64_t DECODE_MIN_UNIT_BYTES = 8;         // the smallest LZ4 block or zstd frame: a decode unit per 8 bytes

inline uint64_t decode_group_bytes(int32_t codec, uint64_t len, uint64_t raw) {
  uint64_t units;
  switch (codec) {
    case TEZGPU_CODEC_DEFAULT: units = 0; break;
    case TEZGPU_CODEC_SNAPPY: units = len / SN_MIN_UNIT_BYTES + 1; break;   // and the 8-byte error words, within the 128
    default: units = len / DECODE_MIN_UNIT_BYTES + 1;
  }
  const uint64_t pieces = div_up(len, CRC_PIECE) + div_up(raw + 4, CRC_PIECE);
  return align_up(len, 16) + align_up(raw + 4, 16) + units * sizeof(ZUnit) + pieces * sizeof(TileCrc) + DECODE_BYTES_PER_SEGMENT;
}

inline void Merger::decode_to_host(const tezgpu_segment *in, const int64_t *raw_len, uint32_t nseg, uint64_t base,
                                   uint64_t budget, uint8_t *const *out) {
  cudaStream_t st = pipe.stream;
  const std::vector<uint32_t> zs = compressed_segments(in, nseg, st);
  auto decode_group = [&](const std::vector<uint32_t> &g) {
    decode_compressed(in, raw_len, g);
    // the trailers: the bodies' remainders (k_crc_pieces / k_crc_combine), then k_image_trailers
    const uint32_t n = (uint32_t)g.size();
    std::vector<SegDesc> sd(n);
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t raw = (uint64_t)raw_len[g[i]];
      sd[i] = SegDesc{z_img_off[i], raw + 4, 4, raw, 1u, 0};
    }
    TG_CUDA(cudaMemcpyAsync(z_descs.p, sd.data(), (size_t)n * sizeof(SegDesc), cudaMemcpyHostToDevice, st));
    std::vector<uint32_t> piece_start;
    launches += segment_remainders(z_img.as<uint8_t>(), sd, z_descs.as<SegDesc>(), [](const SegDesc &) { return true; },
                                   piece_start, false);
    k_image_trailers<<<(uint32_t)div_up(n, 128), 128, 0, st>>>(z_img.as<uint8_t>(), z_descs.as<SegDesc>(), n, d_seg_crc.as<uint32_t>(),
                                                               DeviceConstants::get(pipe.conf.device).d_crc);
    launches++;
    TG_CUDA(cudaGetLastError());
    for (uint32_t i = 0; i < n; i++)
      TG_CUDA(cudaMemcpyAsync(out[g[i]], z_img.as<uint8_t>() + z_img_off[i], sd[i].len, cudaMemcpyDeviceToHost, st));
    TG_CUDA(cudaStreamSynchronize(st));   // also: the host tables above live on this stack
    for (DeviceBuffer *b : {&z_in, &z_img, &z_insegs, &z_status, &z_descs, &z_flag, &z_nblk, &z_base, &z_blks, &z_slow,
                            &d_piece_start, &d_piece_crc, &d_seg_crc})
      b->release();
  };
  std::vector<uint32_t> group;
  uint64_t held = 0;
  for (const uint32_t s : zs) {
    const int64_t raw = raw_len[s];
    check_raw_len(s, raw);
    const uint64_t b = decode_group_bytes(pipe.codec, in[s].len, (uint64_t)raw);
    TG_CHECK(base + DECODE_FIXED_BYTES + b <= budget, TEZGPU_E_NOMEM,
             "segment " + std::to_string(s) + " (" + std::to_string(in[s].len) + " compressed bytes, " + std::to_string(raw) +
                 " raw bytes) does not fit the device budget of " + std::to_string(budget) + " bytes");
    if (base + DECODE_FIXED_BYTES + held + b > budget) {
      decode_group(group);
      group.clear();
      held = 0;
    }
    group.push_back(s);
    held += b;
  }
  if (!group.empty()) decode_group(group);
}

// host run of the device writer over one body: 78 01, the chunks, Adler-32 (tezgpu_debug_deflate_emulate)
static inline std::vector<uint8_t> z_deflate_host(const uint8_t *body, uint64_t len) {
  std::vector<uint8_t> out = {0x78, 0x01};
  ZShared *sh = new ZShared();
  std::vector<uint8_t> slot(ZSLOT);
  const uint64_t nch = std::max<uint64_t>(1, div_up(len, ZCHUNK));
  uint32_t adler = 1;
  for (uint64_t k = 0; k < nch; k++) {
    const uint32_t clen = (uint32_t)std::min<uint64_t>(ZCHUNK, len - k * ZCHUNK);
    z_deflate_chunk_host(*sh, body + k * ZCHUNK, clen, k + 1 == nch, slot.data());
    out.insert(out.end(), slot.begin(), slot.begin() + sh->bytes);
    adler = z_adler_combine(adler, sh->adler, clen);
  }
  delete sh;
  for (int b = 3; b >= 0; b--) out.push_back((uint8_t)(adler >> (8 * b)));
  return out;
}

// host run of a block-framed device writer over one body: run(sh, piece, clen, slot) compresses each `block`-byte piece
// into a slot of slot_bytes, which then holds head + sh.bytes bytes of the stream
template <typename Shared>
static inline std::vector<uint8_t> blocks_compress_host(const uint8_t *body, uint64_t len, uint32_t block, uint32_t slot_bytes,
                                                       uint32_t head, void (*run)(Shared &, const uint8_t *, uint32_t, uint8_t *)) {
  std::vector<uint8_t> out, slot(slot_bytes);
  std::unique_ptr<Shared> sh(new Shared());
  const uint64_t nb = div_up(len, block);
  for (uint64_t k = 0; k < nb; k++) {
    const uint32_t clen = (uint32_t)std::min<uint64_t>(block, len - k * block);
    run(*sh, body + k * block, clen, slot.data());
    out.insert(out.end(), slot.begin(), slot.begin() + head + sh->bytes);
  }
  return out;
}
// LZ4: the blocks, each its 8 header bytes and one chunk (tezgpu_debug_lz4_compress_emulate)
static inline std::vector<uint8_t> l4_compress_host(const uint8_t *body, uint64_t len) {
  return blocks_compress_host<L4Shared>(body, len, L4_BLOCK, L4_SLOT, 8, l4_compress_block_host);
}
// zstd: the frames (tezgpu_debug_zstd_compress_emulate)
static inline std::vector<uint8_t> zs_compress_host(const uint8_t *body, uint64_t len) {
  return blocks_compress_host<ZsShared>(body, len, ZS_BLOCK, ZS_SLOT, 0, zs_compress_block_host);
}
// Snappy: the blocks, each its 8 header bytes and one chunk (tezgpu_debug_snappy_compress_emulate)
static inline std::vector<uint8_t> sn_compress_host(const uint8_t *body, uint64_t len) {
  return blocks_compress_host<SnShared>(body, len, SN_BLOCK, SN_SLOT, 8, sn_compress_block_host);
}

// worst case of the compressed file given the uncompressed file's bound.  zlib: every chunk stored.  LZ4: every block
// all literals (one token, (n - 15) / 255 + 1 length bytes) plus its 8 header bytes.  zstd: every frame raw (10 bytes
// of frame and block header).  Snappy: every block all literals (3 preamble and 3 literal-tag bytes) plus its 8 header
// bytes.
inline uint64_t SortPipeline::codec_bound(int codec, uint64_t raw_bound, int P) {
  if (codec == TEZGPU_CODEC_SNAPPY) return raw_bound + 14 * (raw_bound / SN_BLOCK + (uint64_t)P + 1) + 64;
  if (codec == TEZGPU_CODEC_ZSTD) return raw_bound + 10 * (raw_bound / ZS_BLOCK + (uint64_t)P + 1) + 64;
  if (codec == TEZGPU_CODEC_LZ4) return raw_bound + raw_bound / 255 + 10 * (raw_bound / L4_BLOCK + (uint64_t)P + 1) + 64;
  return raw_bound + 5 * (raw_bound / ZCHUNK + (uint64_t)P + 1) + 11ull * P + 64;
}

}  // namespace tezgpu

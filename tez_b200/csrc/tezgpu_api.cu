// tezgpu_api.cu -- extern "C" boundary of libtezgpu.so (include/tezgpu.h).  No CPU fallback: every compute entry
// point needs a CUDA device and fails with TEZGPU_E_CUDA otherwise.
#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <memory>
#include <mutex>
#include <string>

#include "../../include/tezgpu.h"
#include "codec.cuh"
#include "concat.cuh"
#include "merger.cuh"
#include "merge_steps.cuh"
#include "sorter.cuh"
#include "peer_fetch.cuh"
#include "record_table.cuh"

using namespace tezgpu;

static thread_local std::string g_last_error;

#define TG_API_BEGIN try {
#define TG_API_END                                  \
  }                                                 \
  catch (const tezgpu::Error &e) {                  \
    g_last_error = e.what();                        \
    return e.code;                                  \
  }                                                 \
  catch (const std::bad_alloc &) {                  \
    g_last_error = "host allocation failed";        \
    return TEZGPU_E_NOMEM;                          \
  }                                                 \
  catch (const std::exception &e) {                 \
    g_last_error = e.what();                        \
    return TEZGPU_E_INVALID;                        \
  }                                                 \
  return TEZGPU_OK;

// TezSpillRecord.writeToFile layout (SORT/TezSpillRecord.java:111-146): P x 3 big-endian longs + CRC32 as a long
static void spill_record_bytes(const int64_t *idx, int P, std::vector<uint8_t> &out) {
  out.resize((size_t)P * 24 + 8);
  for (int i = 0; i < P * 3; i++)
    for (int b = 0; b < 8; b++) out[(size_t)i * 8 + b] = (uint8_t)((uint64_t)idx[i] >> (56 - 8 * b));
  CrcTables *t = new CrcTables();
  crc_build_tables(*t, 1);
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < (size_t)P * 24; i++) c = t->slice[0][(c ^ out[i]) & 0xFF] ^ (c >> 8);
  c = ~c;
  delete t;
  for (int b = 0; b < 8; b++) out[(size_t)P * 24 + b] = (uint8_t)((uint64_t)c >> (56 - 8 * b));
}

static void write_file_0640(const char *path, const void *data, size_t len) {
  // SPILL_FILE_PERMS = 0640 (SORT/TezSpillRecord.java:41,148-152)
  int fd = ::open(path, O_WRONLY | O_CREAT | O_TRUNC, 0640);
  TG_CHECK(fd >= 0, TEZGPU_E_IO, std::string("open ") + path + ": " + strerror(errno));
  const uint8_t *p = (const uint8_t *)data;
  size_t left = len;
  while (left) {
    ssize_t w = ::write(fd, p, left);
    if (w < 0) {
      if (errno == EINTR) continue;
      int e = errno;
      ::close(fd);
      throw Error(TEZGPU_E_IO, std::string("write ") + path + ": " + strerror(e));
    }
    p += w;
    left -= (size_t)w;
  }
  ::fchmod(fd, 0640);
  TG_CHECK(::close(fd) == 0, TEZGPU_E_IO, std::string("close ") + path + ": " + strerror(errno));
}

struct tezgpu_sorter {
  SortPipeline pipe;
  bool fixed;
  uint32_t klen, vlen;
  uint64_t n = 0, kv_bytes = 0, payload_bytes = 0;
  bool has_partition = false;
  bool flushed = false;
  DeviceBuffer d_kv, d_koff, d_klen, d_vlen, d_part, d_tmp, d_out;
  PinnedBuffer h_out;
  explicit tezgpu_sorter(const tezgpu_conf &c) : pipe(c) {
    fixed = c.fixed_key_len > 0 || c.fixed_val_len > 0;
    klen = c.fixed_key_len;
    vlen = c.fixed_val_len;
  }
  Records records() {
    Records r;
    memset(&r, 0, sizeof(r));
    r.kv = d_kv.as<uint8_t>();
    r.kv_bytes = align_up(kv_bytes, 16);
    r.key_off = d_koff.as<uint64_t>();
    r.key_len = d_klen.as<uint32_t>();
    r.val_len = d_vlen.as<uint32_t>();
    r.partition = has_partition ? d_part.as<int32_t>() : nullptr;
    r.n = (uint32_t)n;
    r.klen = klen;
    r.vlen = vlen;
    r.fixed = fixed;
    return r;
  }
};

// the partition source of a collect or flush: a TOTAL_ORDER handle takes no partition ids and needs its split points
static void check_partition_source(const tezgpu_sorter *h, bool given) {
  const tezgpu_conf &c = h->pipe.conf;
  if (c.partitioner == TEZGPU_PART_TOTAL_ORDER) {
    TG_CHECK(!given, TEZGPU_E_INVALID, "partition ids given to a TotalOrderPartitioner handle (the device computes them)");
    TG_CHECK(h->pipe.have_splits || c.num_partitions == 1, TEZGPU_E_STATE,
             "TotalOrderPartitioner: set the split points (tezgpu_sorter_set_split_points) first");
    return;
  }
  TG_CHECK(given || c.partitioner == TEZGPU_PART_HASH, TEZGPU_E_INVALID, "partition ids required (partitioner=GIVEN)");
}

__global__ void k_rebase_offsets(const uint32_t *__restrict__ key_off, const uint32_t *__restrict__ val_off,
                                 const uint32_t *__restrict__ val_len, uint32_t n, uint64_t base, uint64_t kv_bytes,
                                 uint64_t *__restrict__ koff64, uint32_t *__restrict__ klen, uint32_t *__restrict__ vlen,
                                 int *__restrict__ err) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t ko = key_off[i], vo = val_off[i], vl = val_len[i];
  if (vo < ko || (uint64_t)vo + vl > kv_bytes) { *err = 1; vo = ko; vl = 0; }
  koff64[i] = base + ko;
  klen[i] = vo - ko;
  vlen[i] = vl;
}

// the body of the tezgpu_debug_*_compress_emulate entry points: host_run is the codec's host run of the device writer
static int32_t compress_emulate(std::vector<uint8_t> (*host_run)(const uint8_t *, uint64_t), const uint8_t *body, uint64_t len,
                                uint8_t *out, uint64_t cap, uint64_t *out_len) {
  TG_API_BEGIN
  TG_CHECK((body || len == 0) && out && out_len, TEZGPU_E_INVALID, "null argument");
  const std::vector<uint8_t> z = host_run(body, len);
  *out_len = z.size();
  TG_CHECK(z.size() <= cap, TEZGPU_E_NOMEM, "output buffer too small");
  memcpy(out, z.data(), z.size());
  TG_API_END
}

// the body of the tezgpu_debug_*_decompress_emulate entry points: decode(&got) runs the codec's host decoder and returns
// its status
template <typename Decode>
static int32_t decompress_emulate(int32_t codec, const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                  uint64_t *out_len, Decode decode) {
  TG_API_BEGIN
  TG_CHECK((z || len == 0) && (out || body_len == 0) && out_len, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(body_len <= cap, TEZGPU_E_INVALID, "output buffer smaller than body_len");
  uint64_t got = 0;
  const int32_t rc = decode(&got);
  *out_len = got;
  TG_CHECK(rc == 0, TEZGPU_E_FORMAT, std::string("compressed segment 0: ") + codec_err_name(codec, rc));
  TG_API_END
}

extern "C" {

const char *tezgpu_last_error(void) { return g_last_error.c_str(); }
int32_t tezgpu_abi_version(void) { return TEZGPU_ABI_VERSION; }
int32_t tezgpu_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int32_t tezgpu_sorter_create(const tezgpu_conf *conf, tezgpu_sorter **out) {
  TG_API_BEGIN
  TG_CHECK(conf && out, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(conf->abi_version == TEZGPU_ABI_VERSION, TEZGPU_E_INVALID, "tezgpu_conf.abi_version mismatch");
  SortPipeline::check_conf(*conf);
  DeviceScope ds(conf->device);
  *out = new tezgpu_sorter(*conf);
  TG_API_END
}

int32_t tezgpu_sorter_destroy(tezgpu_sorter *h) {
  TG_API_BEGIN
  std::unique_ptr<tezgpu_sorter> own(h);   // deleted also when its device cannot be selected
  if (h) {
    DeviceScope ds(h->pipe.conf.device);
    own.reset();
  }
  TG_API_END
}

int32_t tezgpu_sorter_reset(tezgpu_sorter *h) {
  TG_API_BEGIN
  TG_CHECK(h, TEZGPU_E_INVALID, "null handle");
  h->n = h->kv_bytes = h->payload_bytes = 0;
  h->has_partition = false;
  h->flushed = false;
  TG_API_END
}

int32_t tezgpu_sorter_collect_batch(tezgpu_sorter *h, const uint8_t *kv, uint64_t kv_bytes, const uint32_t *key_off,
                                    const uint32_t *val_off, const uint32_t *val_len, const int32_t *partition,
                                    uint32_t n) {
  TG_API_BEGIN
  TG_CHECK(h, TEZGPU_E_INVALID, "null handle");
  TG_CHECK(!h->flushed, TEZGPU_E_STATE, "collect after flush");
  TG_CHECK(!h->fixed, TEZGPU_E_STATE, "handle is in fixed-width mode: use tezgpu_sorter_collect_fixed");
  if (n == 0) return TEZGPU_OK;
  TG_CHECK(kv && key_off && val_off && val_len, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(kv_bytes < (1ull << 32), TEZGPU_E_INVALID, "batch larger than 4 GiB");
  TG_CHECK(h->n + n <= RADIX_MAX_N, TEZGPU_E_INVALID, "more than 2^30-1 records collected");
  TG_CHECK((h->n == 0) || (h->has_partition == (partition != nullptr)), TEZGPU_E_INVALID,
           "partition ids must be given for all batches or none");
  check_partition_source(h, partition != nullptr);
  {
    // the sort memory granted to this output (ExternalSorter.getInitialMemoryRequirement, SORT/ExternalSorter.java:330-347;
    // PipelinedSorter spills when its kvbuffer is full, :415-444): past it the caller must spill -- flush + reset --
    // first.  A first batch larger than the whole budget is still taken (the reference writes such records through).
    uint64_t add = 0;
    for (uint32_t i = 0; i < n; i++) add += (uint64_t)(val_off[i] - key_off[i]) + val_len[i];
    const uint64_t budget = h->pipe.conf.mem_budget_bytes;
    TG_CHECK(budget == 0 || h->n == 0 || h->payload_bytes + add <= budget, TEZGPU_E_NOMEM,
             "sort memory budget exceeded (" + std::to_string(h->payload_bytes + add) + " > " + std::to_string(budget) +
                 " bytes): spill (flush + reset) before collecting more");
  }
  DeviceScope ds(h->pipe.conf.device);
  cudaStream_t st = h->pipe.stream;
  const uint64_t base = align_up(h->kv_bytes, 16);  // every batch starts 16-byte aligned
  h->d_kv.grow_preserve(base + kv_bytes + 32, h->kv_bytes, st);
  h->d_koff.grow_preserve((h->n + n) * 8, h->n * 8, st);
  h->d_klen.grow_preserve((h->n + n) * 4, h->n * 4, st);
  h->d_vlen.grow_preserve((h->n + n) * 4, h->n * 4, st);
  if (partition) h->d_part.grow_preserve((h->n + n) * 4, h->n * 4, st);
  h->d_tmp.ensure((size_t)n * 12);
  uint32_t *t = h->d_tmp.as<uint32_t>();
  TG_CUDA(cudaMemcpyAsync(h->d_kv.as<uint8_t>() + base, kv, kv_bytes, cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemcpyAsync(t, key_off, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemcpyAsync(t + n, val_off, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemcpyAsync(t + 2 * (size_t)n, val_len, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  if (partition)
    TG_CUDA(cudaMemcpyAsync(h->d_part.as<int32_t>() + h->n, partition, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemsetAsync(&h->pipe.d_scratch()->verdict.error, 0, 4, st));
  k_rebase_offsets<<<(uint32_t)div_up(n, 256), 256, 0, st>>>(t, t + n, t + 2 * (size_t)n, n, base, kv_bytes,
                                                           h->d_koff.as<uint64_t>() + h->n, h->d_klen.as<uint32_t>() + h->n,
                                                           h->d_vlen.as<uint32_t>() + h->n, &h->pipe.d_scratch()->verdict.error);
  TG_CUDA(cudaGetLastError());
  int err = 0;
  TG_CUDA(cudaMemcpyAsync(&err, &h->pipe.d_scratch()->verdict.error, 4, cudaMemcpyDeviceToHost, st));
  TG_CUDA(cudaStreamSynchronize(st));  // caller may reuse its buffers once we return
  TG_CHECK(err == 0, TEZGPU_E_INVALID, "record offsets outside the batch buffer");
  for (uint32_t i = 0; i < n; i++) h->payload_bytes += (uint64_t)(val_off[i] - key_off[i]) + val_len[i];
  h->has_partition = partition != nullptr;
  h->n += n;
  h->kv_bytes = base + kv_bytes;
  TG_API_END
}

int32_t tezgpu_sorter_collect_fixed(tezgpu_sorter *h, const uint8_t *kv, const int32_t *partition, uint64_t n) {
  TG_API_BEGIN
  TG_CHECK(h, TEZGPU_E_INVALID, "null handle");
  TG_CHECK(!h->flushed, TEZGPU_E_STATE, "collect after flush");
  TG_CHECK(h->fixed, TEZGPU_E_STATE, "handle is not in fixed-width mode");
  if (n == 0) return TEZGPU_OK;
  TG_CHECK(kv, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(h->n + n <= RADIX_MAX_N, TEZGPU_E_INVALID, "more than 2^30-1 records collected");
  TG_CHECK((h->n == 0) || (h->has_partition == (partition != nullptr)), TEZGPU_E_INVALID,
           "partition ids must be given for all batches or none");
  check_partition_source(h, partition != nullptr);
  const uint64_t stride = (uint64_t)h->klen + h->vlen;
  {
    const uint64_t budget = h->pipe.conf.mem_budget_bytes;
    TG_CHECK(budget == 0 || h->n == 0 || (h->n + n) * stride <= budget, TEZGPU_E_NOMEM,
             "sort memory budget exceeded (" + std::to_string((h->n + n) * stride) + " > " + std::to_string(budget) +
                 " bytes): spill (flush + reset) before collecting more");
  }
  DeviceScope ds(h->pipe.conf.device);
  cudaStream_t st = h->pipe.stream;
  h->d_kv.grow_preserve((h->n + n) * stride + 32, h->n * stride, st);
  if (partition) h->d_part.grow_preserve((h->n + n) * 4, h->n * 4, st);
  TG_CUDA(cudaMemcpyAsync(h->d_kv.as<uint8_t>() + h->n * stride, kv, n * stride, cudaMemcpyHostToDevice, st));
  if (partition)
    TG_CUDA(cudaMemcpyAsync(h->d_part.as<int32_t>() + h->n, partition, n * 4, cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaStreamSynchronize(st));
  h->has_partition = partition != nullptr;
  h->n += n;
  h->kv_bytes = h->n * stride;
  h->payload_bytes = h->kv_bytes;
  TG_API_END
}

static uint64_t sorter_raw_bound(const tezgpu_sorter *h) {
  if (h->fixed && h->pipe.conf.rle_policy == TEZGPU_RLE_OFF)  // exact: n * (vint(k) + vint(v) + k + v) + 10 bytes per segment
    return h->n * ((uint64_t)vint_size_u32(h->klen) + vint_size_u32(h->vlen) + h->klen + h->vlen) +
           10ull * h->pipe.conf.num_partitions + 64;
  return SortPipeline::output_bound(h->n, h->kv_bytes, h->pipe.conf.num_partitions);
}

// out_cap that always suffices for tezgpu_sorter_sort_device of n records in kv_bytes bytes: the uncompressed file's
// bound, and with a codec that file's worst case compressed
static uint64_t device_output_bound(int P, int codec, uint64_t n, uint64_t kv_bytes) {
  const uint64_t raw = SortPipeline::output_bound(n, kv_bytes, P);
  return codec ? SortPipeline::codec_bound(codec, raw, P) : raw;
}

uint64_t tezgpu_sorter_output_bound(const tezgpu_sorter *h) {
  if (!h) return 0;
  const uint64_t raw = sorter_raw_bound(h);
  return h->pipe.codec ? SortPipeline::codec_bound(h->pipe.codec, raw, h->pipe.conf.num_partitions) : raw;
}

static void sorter_run(tezgpu_sorter *h, uint8_t *host_out, uint64_t out_cap, uint64_t *out_len, int64_t *index,
                       tezgpu_stats *stats, std::vector<int64_t> &idx_store) {
  TG_CHECK(!h->flushed, TEZGPU_E_STATE, "flush called twice");
  if (h->pipe.conf.partitioner == TEZGPU_PART_TOTAL_ORDER) check_partition_source(h, false);
  const int P = h->pipe.conf.num_partitions;
  idx_store.assign((size_t)P * 3, 0);
  uint64_t bound = tezgpu_sorter_output_bound(h);
  h->d_out.ensure(bound);
  uint64_t len = 0;
  tezgpu_stats st;
  h->pipe.run(h->records(), h->d_out.as<uint8_t>(), h->d_out.cap, &len, idx_store.data(), &st);
  st.output_bytes = (int64_t)h->payload_bytes;
  TG_CHECK(len <= out_cap, TEZGPU_E_NOMEM, "output buffer too small for file.out");
  if (len) {
    // one copy, not pieces: 64 MB pieces of a download running next to another task slot's upload were slower than
    // one whole copy (tools/e2e_probe.py)
    TG_CUDA(cudaMemcpyAsync(host_out, h->d_out.p, len, cudaMemcpyDeviceToHost, h->pipe.stream));
    TG_CUDA(cudaStreamSynchronize(h->pipe.stream));
  }
  if (out_len) *out_len = len;
  if (index) memcpy(index, idx_store.data(), (size_t)P * 24);
  if (stats) *stats = st;
  h->flushed = true;
}

int32_t tezgpu_sorter_flush_to_memory(tezgpu_sorter *h, uint8_t *out, uint64_t out_cap, uint64_t *out_len,
                                      uint8_t *index_out, int64_t *index, tezgpu_stats *stats) {
  TG_API_BEGIN
  TG_CHECK(h && (out || out_cap == 0), TEZGPU_E_INVALID, "null argument");
  DeviceScope ds(h->pipe.conf.device);
  std::vector<int64_t> idx;
  sorter_run(h, out, out_cap, out_len, index, stats, idx);
  if (index_out) {
    std::vector<uint8_t> b;
    spill_record_bytes(idx.data(), h->pipe.conf.num_partitions, b);
    memcpy(index_out, b.data(), b.size());
  }
  TG_API_END
}

int32_t tezgpu_sorter_flush(tezgpu_sorter *h, const char *out_path, const char *index_path, int64_t *index,
                            tezgpu_stats *stats) {
  TG_API_BEGIN
  TG_CHECK(h && out_path && index_path, TEZGPU_E_INVALID, "null argument");
  DeviceScope ds(h->pipe.conf.device);
  uint64_t bound = tezgpu_sorter_output_bound(h);
  h->h_out.ensure(bound);
  std::vector<int64_t> idx;
  uint64_t len = 0;
  sorter_run(h, h->h_out.as<uint8_t>(), h->h_out.cap, &len, index, stats, idx);
  write_file_0640(out_path, h->h_out.p, len);
  std::vector<uint8_t> b;
  spill_record_bytes(idx.data(), h->pipe.conf.num_partitions, b);
  write_file_0640(index_path, b.data(), b.size());
  TG_API_END
}

int32_t tezgpu_sorter_sort_device_fixed(tezgpu_sorter *h, const void *d_kv, const void *d_partition, uint64_t n,
                                        void *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index,
                                        tezgpu_stats *stats) {
  TG_API_BEGIN
  TG_CHECK(h && (d_kv || n == 0) && d_out, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(h->fixed, TEZGPU_E_STATE, "handle is not in fixed-width mode");
  TG_CHECK(n <= RADIX_MAX_N, TEZGPU_E_INVALID, "more than 2^30-1 records in one sort");
  check_partition_source(h, d_partition != nullptr);
  Records r;
  memset(&r, 0, sizeof(r));
  r.kv = (const uint8_t *)d_kv;
  r.kv_bytes = n * ((uint64_t)h->klen + h->vlen);  // exact: boundary loads are clamped, nothing is read past the caller's buffer
  r.partition = (const int32_t *)d_partition;
  r.n = (uint32_t)n;
  r.klen = h->klen;
  r.vlen = h->vlen;
  r.fixed = 1;
  TG_CHECK(((uintptr_t)d_kv & 15u) == 0, TEZGPU_E_INVALID, "device-resident input must be 16-byte aligned");
  DeviceScope ds(h->pipe.conf.device);
  tezgpu_stats st;
  h->pipe.run(r, (uint8_t *)d_out, out_cap, out_len, index, &st);
  st.output_bytes = (int64_t)(n * ((uint64_t)h->klen + h->vlen));
  if (stats) *stats = st;
  TG_API_END
}

uint64_t tezgpu_sorter_device_output_bound(const tezgpu_sorter *h, uint64_t n, uint64_t kv_bytes) {
  return h ? device_output_bound(h->pipe.conf.num_partitions, h->pipe.codec, n, kv_bytes) : 0;
}

uint64_t tezgpu_debug_device_output_bound(int32_t num_partitions, int32_t codec, uint64_t n, uint64_t kv_bytes) {
  if (num_partitions < 1 || codec < TEZGPU_CODEC_NONE || codec > TEZGPU_CODEC_SNAPPY) return 0;
  return device_output_bound(num_partitions, codec, n, kv_bytes);
}

int32_t tezgpu_sorter_sort_device(tezgpu_sorter *h, const void *d_kv, uint64_t kv_bytes, const uint64_t *d_key_off,
                                  const uint64_t *d_val_off, const uint32_t *d_val_len, const int32_t *d_partition, uint64_t n,
                                  void *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index, tezgpu_stats *stats) {
  TG_API_BEGIN
  TG_CHECK(h && d_out, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(n == 0 || (d_kv && d_key_off && d_val_off && d_val_len), TEZGPU_E_INVALID, "null argument");
  TG_CHECK(!h->fixed, TEZGPU_E_STATE, "handle is in fixed-width mode: use tezgpu_sorter_sort_device_fixed");
  TG_CHECK(h->n == 0, TEZGPU_E_STATE, "records were collected on this handle: reset it first");
  TG_CHECK(n <= RADIX_MAX_N, TEZGPU_E_INVALID, "more than 2^30-1 records in one sort");
  check_partition_source(h, d_partition != nullptr);
  TG_CHECK(((uintptr_t)d_kv & 15u) == 0, TEZGPU_E_INVALID, "device-resident input must be 16-byte aligned");
  TG_CHECK(h->pipe.codec || ((uintptr_t)d_out & 15u) == 0, TEZGPU_E_INVALID, "output buffer must be 16-byte aligned");
  DeviceScope ds(h->pipe.conf.device);
  SortPipeline &pipe = h->pipe;
  cudaStream_t st = pipe.stream;
  uint64_t payload = 0;
  if (n) {
    // the record table goes into the handle's collect arrays (free: nothing is collected); the verdict borrows the
    // sort's scratch, which sort_phase clears before it sorts
    h->d_koff.ensure(n * 8);
    h->d_klen.ensure(n * 4);
    h->d_vlen.ensure(n * 4);
    SortVerdict *v = &pipe.d_scratch()->verdict;
    TG_CUDA(cudaMemsetAsync(&v->dups, 0xFF, sizeof(v->dups), st));
    TG_CUDA(cudaMemsetAsync(&v->totals[0], 0, sizeof(v->totals[0]), st));
    const uint32_t grid = (uint32_t)std::min<uint64_t>(div_up(n, RECTAB_THREADS), (uint64_t)pipe.num_sms * 8);
    k_record_table<<<grid, RECTAB_THREADS, 0, st>>>(d_key_off, d_val_off, d_val_len, d_partition, (uint32_t)n, kv_bytes,
                                                    pipe.conf.num_partitions, h->d_koff.as<uint64_t>(), h->d_klen.as<uint32_t>(),
                                                    h->d_vlen.as<uint32_t>(), &v->dups, (unsigned long long *)&v->totals[0]);
    TG_CUDA(cudaGetLastError());
    store_to_host(st, &pipe.h_scratch()->verdict, v, sizeof(SortVerdict));
    TG_CUDA(cudaGetLastError());
    TG_CUDA(cudaStreamSynchronize(st));
    const SortVerdict &hv = pipe.h_scratch()->verdict;
    TG_CHECK(hv.dups == ~0ull, TEZGPU_E_INVALID,
             "record " + std::to_string(hv.dups >> RECTAB_REASON_BITS) + ": " +
                 record_table_reason((uint32_t)(hv.dups & ((1u << RECTAB_REASON_BITS) - 1))));
    payload = hv.totals[0];
  }
  Records r;
  memset(&r, 0, sizeof(r));
  r.kv = (const uint8_t *)d_kv;
  r.kv_bytes = kv_bytes;  // exact: the emit's loads are clamped to it, every other kernel reads inside the records
  r.key_off = h->d_koff.as<uint64_t>();
  r.key_len = h->d_klen.as<uint32_t>();
  r.val_len = h->d_vlen.as<uint32_t>();
  r.partition = d_partition;
  r.n = (uint32_t)n;
  tezgpu_stats s;
  pipe.run(r, (uint8_t *)d_out, out_cap, out_len, index, &s);
  s.output_bytes = (int64_t)payload;
  if (stats) *stats = s;
  TG_API_END
}

void *tezgpu_sorter_stream(tezgpu_sorter *h) { return h ? (void *)h->pipe.stream : nullptr; }

int32_t tezgpu_sorter_set_combiner(tezgpu_sorter *h, int32_t combiner) {
  TG_API_BEGIN
  TG_CHECK(h, TEZGPU_E_INVALID, "null handle");
  TG_CHECK(combiner == TEZGPU_COMBINE_NONE || combine_width(combiner), TEZGPU_E_INVALID, "unknown combiner");
  TG_CHECK(!combiner || h->pipe.conf.sorter_impl != TEZGPU_SORTER_UNORDERED, TEZGPU_E_INVALID,
           "the unordered writer (UnorderedPartitionedKVWriter) runs no combiner");
  TG_CHECK(!combiner || !h->fixed || h->vlen == combine_width(combiner), TEZGPU_E_INVALID,
           "fixed_val_len " + std::to_string(h->vlen) + " is not the combiner's value width");
  TG_CHECK(h->n == 0 && !h->flushed, TEZGPU_E_STATE, "set the combiner before the first collect (or after a reset)");
  h->pipe.combiner = combiner;
  TG_API_END
}

int32_t tezgpu_sorter_set_codec(tezgpu_sorter *h, int32_t codec) {
  TG_API_BEGIN
  TG_CHECK(h, TEZGPU_E_INVALID, "null handle");
  check_codec(codec);
  TG_CHECK(h->n == 0 && !h->flushed, TEZGPU_E_STATE, "set the codec before the first collect (or after a reset)");
  h->pipe.codec = codec;
  TG_API_END
}

int32_t tezgpu_sorter_set_split_points(tezgpu_sorter *h, const uint8_t *keys, const uint64_t *key_off, const uint32_t *key_len,
                                       uint32_t n, int32_t order) {
  TG_API_BEGIN
  TG_CHECK(h, TEZGPU_E_INVALID, "null handle");
  const tezgpu_conf &c = h->pipe.conf;
  TG_CHECK(c.partitioner == TEZGPU_PART_TOTAL_ORDER, TEZGPU_E_INVALID, "split points on a handle whose partitioner is not TOTAL_ORDER");
  TG_CHECK(h->n == 0 && !h->flushed, TEZGPU_E_STATE, "set the split points before the first collect (or after a reset)");
  HostSplitTable t;
  build_split_table(c.comparator, order, c.num_partitions, keys, key_off, key_len, n, t);
  DeviceScope ds(c.device);
  h->pipe.set_split_points(t);
  TG_API_END
}

int32_t tezgpu_debug_total_order_emulate(const uint8_t *kv, const uint64_t *key_off, const uint32_t *key_len, uint32_t n,
                                         const uint8_t *splits, const uint64_t *split_off, const uint32_t *split_len,
                                         uint32_t nsplits, int32_t comparator, int32_t order, int32_t *partition) {
  TG_API_BEGIN
  TG_CHECK(((kv && key_off && key_len && partition) || n == 0), TEZGPU_E_INVALID, "null argument");
  TG_CHECK(comparator >= TEZGPU_CMP_BYTES && comparator <= TEZGPU_CMP_LONG, TEZGPU_E_UNSUPPORTED, "unknown comparator");
  TG_CHECK(nsplits < (1u << 31) - 1, TEZGPU_E_INVALID, "too many split points");
  HostSplitTable t;
  build_split_table(comparator, order, (int)nsplits + 1, splits, split_off, split_len, nsplits, t);
  const SplitTable v = t.view();
  for (uint32_t i = 0; i < n; i++) partition[i] = split_partition(v, v.prefix, kv + key_off[i], key_len[i]);
  TG_API_END
}

int32_t tezgpu_debug_deflate_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len) {
  return compress_emulate(z_deflate_host, body, len, out, cap, out_len);
}

int32_t tezgpu_debug_inflate_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                     uint64_t *out_len) {
  return decompress_emulate(TEZGPU_CODEC_DEFAULT, z, len, body_len, out, cap, out_len, [&](uint64_t *got) {
    std::unique_ptr<ZInflateWork> w(new ZInflateWork());
    return z_inflate(z, len, out, body_len, got, *w);
  });
}

int32_t tezgpu_debug_lz4_compress_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len) {
  return compress_emulate(l4_compress_host, body, len, out, cap, out_len);
}

int32_t tezgpu_debug_lz4_decompress_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                            uint64_t *out_len) {
  return decompress_emulate(TEZGPU_CODEC_LZ4, z, len, body_len, out, cap, out_len,
                            [&](uint64_t *got) { return l4_decompress(z, len, out, body_len, got); });
}

int32_t tezgpu_debug_zstd_compress_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len) {
  return compress_emulate(zs_compress_host, body, len, out, cap, out_len);
}

int32_t tezgpu_debug_zstd_decompress_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                             uint64_t *out_len) {
  return decompress_emulate(TEZGPU_CODEC_ZSTD, z, len, body_len, out, cap, out_len, [&](uint64_t *got) {
    std::unique_ptr<ZsDec> d(new ZsDec());
    return zs_decompress(z, len, out, body_len, got, *d);
  });
}

int32_t tezgpu_debug_snappy_compress_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len) {
  return compress_emulate(sn_compress_host, body, len, out, cap, out_len);
}

int32_t tezgpu_debug_stitched_compress_emulate(int32_t codec, const uint8_t *body, uint64_t len, const uint64_t *cuts, uint32_t ncuts,
                                               uint8_t *out, uint64_t cap, uint64_t *out_len) {
  TG_API_BEGIN
  TG_CHECK((body || len == 0) && (cuts || ncuts == 0) && out && out_len, TEZGPU_E_INVALID, "null argument");
  check_codec(codec);
  TG_CHECK(codec != TEZGPU_CODEC_NONE, TEZGPU_E_INVALID, "tezgpu_debug_stitched_compress_emulate: no codec");
  TG_CHECK(len > 0, TEZGPU_E_INVALID, "an IFile body holds at least its EOF markers");
  const std::vector<uint8_t> z = stitched_compress_host(codec, body, len, cuts, ncuts);
  *out_len = z.size();
  TG_CHECK(z.size() <= cap, TEZGPU_E_NOMEM, "output buffer too small");
  memcpy(out, z.data(), z.size());
  TG_API_END
}

int32_t tezgpu_debug_snappy_decompress_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                               uint64_t *out_len) {
  return decompress_emulate(TEZGPU_CODEC_SNAPPY, z, len, body_len, out, cap, out_len,
                            [&](uint64_t *got) { return sn_decompress(z, len, out, body_len, got); });
}

int32_t tezgpu_debug_crc_concat_emulate(const uint8_t *const *bodies, const uint64_t *lens, uint32_t n, uint32_t *crc) {
  TG_API_BEGIN
  TG_CHECK(((bodies && lens) || n == 0) && crc, TEZGPU_E_INVALID, "null argument");
  std::unique_ptr<CrcTables> t(new CrcTables());
  crc_build_tables(*t, EMIT_CRC_STRIDE_WORDS);
  // every input's IFile checksum, as its trailer carries it; from here on only the algebra of concat.cuh
  uint32_t acc = 0;   // raw remainder of the records so far
  uint64_t rec_total = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint8_t *b = bodies[i];
    const uint64_t len = lens[i];
    TG_CHECK(len >= 2 && b && b[len - 2] == 0xFF && b[len - 1] == 0xFF, TEZGPU_E_FORMAT,
             "body " + std::to_string(i) + " does not end in the EOF marker");
    uint32_t c = 0xFFFFFFFFu;
    for (uint64_t k = 0; k < len; k++) c = t->slice[0][(c ^ b[k]) & 0xFF] ^ (c >> 8);
    const uint32_t stored = ~c;
    const uint32_t body_raw = stored ^ 0xFFFFFFFFu ^ crc_multmodp(0xFFFFFFFFu, crc_host_xpow8(len));
    acc = crc_multmodp(acc, crc_host_xpow8(len - 2)) ^ concat_records_raw(body_raw, *t);   // crc(A||B)
    rec_total += len - 2;
  }
  const uint32_t raw = crc_multmodp(acc, crc_host_xpow8(2)) ^ t->eof_raw;
  *crc = raw ^ crc_multmodp(0xFFFFFFFFu, crc_host_xpow8(rec_total + 2)) ^ 0xFFFFFFFFu;
  TG_API_END
}

int32_t tezgpu_debug_sort_words_emulate(const uint8_t *kv, const uint64_t *key_off, const uint32_t *key_len, uint32_t n,
                                        int32_t comparator, int32_t num_partitions, const int32_t *partition,
                                        int32_t use_sym, uint32_t *words, uint32_t *npos, int32_t *sym_used) {
  TG_API_BEGIN
  TG_CHECK((kv || n == 0) && ((key_off && key_len) || n == 0) && (words || n == 0) && npos && sym_used, TEZGPU_E_INVALID,
           "null argument");
  TG_CHECK(comparator >= TEZGPU_CMP_BYTES && comparator <= TEZGPU_CMP_LONG, TEZGPU_E_UNSUPPORTED, "unknown comparator");
  const int pbits = partition_bits(num_partitions);
  TG_CHECK(num_partitions >= 1 && pbits <= 31, TEZGPU_E_INVALID, "num_partitions out of range");
  Records r;
  memset(&r, 0, sizeof(r));
  r.kv = kv;
  r.n = n;
  r.cmp = comparator;
  r.hash_partition = partition == nullptr;
  r.num_partitions = num_partitions;
  r.pbits = pbits;
  // k_symbols: which normalised byte values occur at each of the first SYM_MAX_POS content positions
  uint32_t sets[SYM_MAX_POS * 8] = {0};
  for (uint32_t i = 0; i < n; i++) {
    const uint8_t *key = kv + key_off[i];
    const uint32_t skip = key_content_skip(comparator, key, key_len[i]);
    for (uint32_t q = 0; q < (uint32_t)SYM_MAX_POS && q < key_len[i] - skip; q++) {
      const uint32_t b = norm_byte(comparator, key + skip, q);
      sets[q * 8 + (b >> 5)] |= 1u << (b & 31u);
    }
  }
  SymTable *t = new SymTable();
  *npos = n ? sym_table_build(sets, pbits, t) : 0;
  *sym_used = (n && use_sym && sym_table_pays(*npos, pbits)) ? 1 : 0;
  r.sym = *sym_used ? t : nullptr;
  bool bad = false;
  for (uint32_t i = 0; i < n && !bad; i++) words[i] = stage_sort_word(r, kv + key_off[i], key_len[i], partition ? partition[i] : 0, bad);
  delete t;
  TG_CHECK(!bad, TEZGPU_E_INVALID, "Illegal partition (outside [0, numPartitions))");
  TG_API_END
}

// ------------------------------------------------------------------------------------------------ NVLink peer fetch
int32_t tezgpu_peer_alloc(int32_t device, uint64_t bytes, void **dptr, uint8_t *handle_out) {
  TG_API_BEGIN
  TG_CHECK(dptr && handle_out && bytes, TEZGPU_E_INVALID, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == TEZGPU_PEER_HANDLE_BYTES, "export handle size");
  DeviceScope ds(device);
  void *p = nullptr;
  TG_CUDA(cudaMalloc(&p, bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    TG_CUDA(e);
  }
  memcpy(handle_out, &h, sizeof(h));
  *dptr = p;
  TG_API_END
}

int32_t tezgpu_peer_free(int32_t device, void *dptr) {
  TG_API_BEGIN
  DeviceScope ds(device);
  if (dptr) TG_CUDA(cudaFree(dptr));
  TG_API_END
}

int32_t tezgpu_peer_open(int32_t device, const uint8_t *handle, void **dptr) {
  TG_API_BEGIN
  TG_CHECK(handle && dptr, TEZGPU_E_INVALID, "null argument");
  DeviceScope ds(device);
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void *p = nullptr;
  TG_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *dptr = p;
  TG_API_END
}

int32_t tezgpu_peer_close(int32_t device, void *dptr) {
  TG_API_BEGIN
  DeviceScope ds(device);
  if (dptr) TG_CUDA(cudaIpcCloseMemHandle(dptr));
  TG_API_END
}

}  // extern "C"
// TEZGPU_FETCH_CTAS (read at every call): upper bound on the pull kernels' grid.  The pull is NVLink-bound; when it runs
// next to another stream's HBM-bound kernels (TEZ_SHUFFLE_OVERLAP: the sort of the next batch) a grid that fills every
// SM makes the two serialise, a grid of about one CTA per SM leaves room for the other kernels' CTAs.
static uint32_t fetch_grid_cap(uint32_t grid) {
  const char *e = getenv("TEZGPU_FETCH_CTAS");
  const long cap = e ? atol(e) : 0;
  return cap > 0 && (uint32_t)cap < grid ? (uint32_t)cap : grid;
}
extern "C" {
int32_t tezgpu_fetch_ranges(int32_t device, const tezgpu_copy_range *ranges, uint32_t n, void *stream, float *ms_kernel) {
  TG_API_BEGIN
  TG_CHECK(ranges || n == 0, TEZGPU_E_INVALID, "null argument");
  if (ms_kernel) *ms_kernel = 0;
  if (n == 0) return TEZGPU_OK;
  DeviceScope ds(device);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<FetchRange> fr(n);
  uint64_t chunks = 0;
  for (uint32_t i = 0; i < n; i++) {
    TG_CHECK((ranges[i].src && ranges[i].dst) || ranges[i].len == 0, TEZGPU_E_INVALID, "null range");
    fr[i].src = (const uint8_t *)ranges[i].src;
    fr[i].dst = (uint8_t *)ranges[i].dst;
    fr[i].len = ranges[i].len;
    fr[i].chunk0 = chunks;
    chunks += fetch_chunks(ranges[i].src, ranges[i].dst, ranges[i].len);
  }
  if (chunks == 0) return TEZGPU_OK;
  // ranges travel as a kernel parameter when they are few (one per peer GPU); larger lists through a device copy
  FetchRange *d_fr = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaError_t err = cudaSuccess;
  if (n > FETCH_INLINE_RANGES) {
    TG_CUDA(cudaMalloc(&d_fr, (size_t)n * sizeof(FetchRange)));
    err = cudaMemcpyAsync(d_fr, fr.data(), (size_t)n * sizeof(FetchRange), cudaMemcpyHostToDevice, st);
  }
  if (err == cudaSuccess && ms_kernel) {
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0, st);
  }
  if (err == cudaSuccess) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    uint32_t grid = (uint32_t)std::min<uint64_t>(chunks, (uint64_t)sms * 2);
    grid = fetch_grid_cap(grid);
    if (d_fr) {
      k_fetch_ranges<<<grid, FETCH_THREADS, 0, st>>>(d_fr, n, chunks);
    } else {
      FetchRangeList lst;
      for (uint32_t i = 0; i < n; i++) lst.r[i] = fr[i];
      k_fetch_ranges_inline<<<grid, FETCH_THREADS, 0, st>>>(lst, n, chunks);
    }
    err = cudaGetLastError();
  }
  if (err == cudaSuccess && ms_kernel) cudaEventRecord(e1, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);
  if (err == cudaSuccess && ms_kernel) cudaEventElapsedTime(ms_kernel, e0, e1);
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  if (d_fr) cudaFree(d_fr);
  TG_CUDA(err);
  TG_API_END
}

// per-device scratch of tezgpu_fetch_ranges_verified (grow-only; one fetch at a time per device)
struct FetchVerifyScratch {
  DeviceBuffer segs, piece_start, piece_crc, seg_crc, flag;
  std::mutex mu;
};
static FetchVerifyScratch &fetch_scratch(int device) {
  static FetchVerifyScratch inst[64];
  return inst[device & 63];
}

int32_t tezgpu_fetch_segments_verified(int32_t device, const tezgpu_fetch_segment *segs, uint32_t n, void *stream,
                                       float *ms_kernel) {
  TG_API_BEGIN
  TG_CHECK(segs || n == 0, TEZGPU_E_INVALID, "null argument");
  if (ms_kernel) *ms_kernel = 0;
  if (n == 0) return TEZGPU_OK;
  DeviceScope ds(device);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<FetchSeg> fs(n);
  std::vector<uint32_t> piece_start(n + 1);
  uint32_t np = 0;
  for (uint32_t i = 0; i < n; i++) {
    const bool hdr = segs[i].flags & TEZGPU_SEG_HAS_HEADER;
    TG_CHECK(segs[i].src && segs[i].dst, TEZGPU_E_INVALID, "null segment");
    TG_CHECK(segs[i].len >= (hdr ? 10u : 6u), TEZGPU_E_FORMAT, "IFile segment shorter than an empty segment");
    TG_CHECK((((uintptr_t)segs[i].src ^ (uintptr_t)segs[i].dst) & 15u) == 0, TEZGPU_E_INVALID,
             "source and destination of a verified fetch must agree modulo 16");
    fs[i].src = (const uint8_t *)segs[i].src;
    fs[i].dst = (uint8_t *)segs[i].dst;
    fs[i].len = segs[i].len;
    fs[i].has_header = hdr ? 1 : 0;
    fs[i].pad = 0;
    piece_start[i] = np;
    np += (uint32_t)div_up(segs[i].len - 4 - (hdr ? 4 : 0), FV_PIECE);
  }
  piece_start[n] = np;
  FetchVerifyScratch &sc = fetch_scratch(device);
  std::lock_guard<std::mutex> lock(sc.mu);
  sc.segs.ensure((size_t)n * sizeof(FetchSeg));
  sc.piece_start.ensure((size_t)(n + 1) * 4);
  sc.piece_crc.ensure((size_t)np * sizeof(TileCrc));
  sc.seg_crc.ensure((size_t)n * 4);
  sc.flag.ensure(16);
  const CrcTables *d_crc = DeviceConstants::get(device).d_crc;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  TG_CUDA(cudaMemcpyAsync(sc.segs.p, fs.data(), (size_t)n * sizeof(FetchSeg), cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemcpyAsync(sc.piece_start.p, piece_start.data(), (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, st));
  TG_CUDA(cudaMemsetAsync(sc.seg_crc.p, 0, (size_t)n * 4, st));
  TG_CUDA(cudaMemsetAsync(sc.flag.p, 0, 16, st));
  if (ms_kernel) {
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0, st);
  }
  int sms = 132, per_sm = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fetch_verify, FV_THREADS, 0);
  const uint32_t grid = fetch_grid_cap((uint32_t)std::min<uint64_t>(np, (uint64_t)sms * (per_sm > 0 ? per_sm : 1)));
  k_fetch_verify<<<grid, FV_THREADS, 0, st>>>(sc.segs.as<FetchSeg>(), sc.piece_start.as<uint32_t>(), n, np, d_crc, sc.piece_crc.as<TileCrc>());
  if (ms_kernel) cudaEventRecord(e1, st);
  k_crc_combine<<<(uint32_t)div_up(np, 256), 256, 0, st>>>(sc.piece_crc.as<TileCrc>(), np, d_crc, sc.seg_crc.as<uint32_t>());
  k_fetch_crc_check<<<(uint32_t)div_up(n, 128), 128, 0, st>>>(sc.segs.as<FetchSeg>(), n, sc.seg_crc.as<uint32_t>(), d_crc, sc.flag.as<int>());
  cudaError_t err = cudaGetLastError();
  int bad = 0;
  if (err == cudaSuccess) err = cudaMemcpyAsync(&bad, sc.flag.p, 4, cudaMemcpyDeviceToHost, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);
  if (err == cudaSuccess && ms_kernel) cudaEventElapsedTime(ms_kernel, e0, e1);
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  TG_CUDA(err);
  TG_CHECK(bad == 0, TEZGPU_E_FORMAT, "IFile checksum mismatch in fetched segment " + std::to_string(bad - 1));
  TG_API_END
}

#include "shuffle_wire.inl"

// Host emulation of the emit kernel's parallel CRC scheme (interleaved per-thread streams over the 4-byte words of a
// piece, power-table alignment, xor-fold of piece contributions into the segment remainder, final conditioning).
// Pure host arithmetic on the same tables the device uses; lets the CPU test-suite check the GF(2) algebra.
uint32_t tezgpu_debug_crc_emulate(const uint8_t *body, uint64_t len, uint32_t piece_bytes, uint32_t lead) {
  CrcTables *t = new CrcTables();
  const int T = EMIT_CRC_STRIDE_WORDS;
  crc_build_tables(*t, T);
  auto shift = [&](uint32_t crc, uint64_t nbytes) {
    uint32_t a0 = (uint32_t)(nbytes & 4095), a1 = (uint32_t)((nbytes >> 12) & 4095), a2 = (uint32_t)((nbytes >> 24) & 4095);
    if (a0) crc = crc_multmodp(crc, t->pow0[a0]);
    if (a1) crc = crc_multmodp(crc, t->pow1[a1]);
    if (a2) crc = crc_multmodp(crc, t->pow2[a2]);
    return crc;
  };
  uint32_t seg = 0;
  uint64_t done = 0;
  std::vector<uint8_t> img;
  while (done < len) {
    uint32_t ld = (uint32_t)((done + lead) & 15u);
    uint32_t plen = (uint32_t)std::min<uint64_t>(piece_bytes - ld, len - done);
    img.assign((size_t)ld + plen + 16, 0);
    memcpy(img.data() + ld, body + done, plen);
    uint32_t cb0 = ld, cb1 = ld + plen;
    uint32_t wa = (cb0 + 3u) >> 2, wb = cb1 >> 2;
    uint32_t words_crc = 0;
    const uint32_t *img32 = reinterpret_cast<const uint32_t *>(img.data());
    if (wb > wa) {
      uint32_t W = wb - wa;
      for (uint32_t tid = 0; tid < (uint32_t)T && tid < W; tid++) {
        uint32_t i = wa + tid, c = 0;
        for (; i + T < wb; i += T) {
          uint32_t v = c ^ img32[i];
          c = t->adv[0][v & 0xFF] ^ t->adv[1][(v >> 8) & 0xFF] ^ t->adv[2][(v >> 16) & 0xFF] ^ t->adv[3][v >> 24];
        }
        uint32_t v = c ^ img32[i];
        c = t->slice[3][v & 0xFF] ^ t->slice[2][(v >> 8) & 0xFF] ^ t->slice[1][(v >> 16) & 0xFF] ^ t->slice[0][v >> 24];
        uint32_t d = wb - 1 - i;
        if (d) c = crc_multmodp(c, t->pow_word[d]);
        words_crc ^= c;
      }
    }
    uint32_t raw = 0;
    uint32_t head_end = (wb > wa) ? 4 * wa : cb1;
    for (uint32_t b = cb0; b < head_end; b++) raw = t->slice[0][(raw ^ img[b]) & 0xFF] ^ (raw >> 8);
    if (wb > wa) {
      raw = shift(raw, 4ull * (wb - wa)) ^ words_crc;
      for (uint32_t b = 4 * wb; b < cb1; b++) raw = t->slice[0][(raw ^ img[b]) & 0xFF] ^ (raw >> 8);
    }
    seg ^= shift(raw, len - (done + plen));
    done += plen;
  }
  uint32_t crc = seg ^ shift(0xFFFFFFFFu, len) ^ 0xFFFFFFFFu;
  delete t;
  return crc;
}

// Host emulation of the chunk-interleaved checksum of the emit / verify kernels (crc32.cuh CrcChunkFold): 256 threads,
// thread t folds chunks i = Cn + t - iters*256 (+256 ...), partials are combined by the adv128 second-level fold, the
// per-lane alignment multiplier and an xor across lanes.  ilp = 1 runs the two-deep fold with the einv correction,
// ilp = 0 the textbook chain.  Returns the raw remainder (init 0, no final xor) of the nchunks * 16 bytes.
uint32_t tezgpu_debug_chunk_fold_emulate(const uint8_t *data, uint32_t nchunks, int32_t ilp) {
  CrcTables *t = new CrcTables();
  const int T = EMIT_CRC_STRIDE_WORDS;
  crc_build_tables(*t, T);
  auto tab = [](const uint32_t(*m)[256], uint32_t x) { return m[0][x & 0xFF] ^ m[1][(x >> 8) & 0xFF] ^ m[2][(x >> 16) & 0xFF] ^ m[3][x >> 24]; };
  auto W = [&](uint32_t x) { return t->slice[3][x & 0xFF] ^ t->slice[2][(x >> 8) & 0xFF] ^ t->slice[1][(x >> 16) & 0xFF] ^ t->slice[0][x >> 24]; };
  auto S = [&](uint32_t x) { return tab(t->advc, x); };
  auto SW2 = [&](uint32_t x) { return tab(t->advc2, x); };
  const uint32_t Cn = nchunks, iters = (Cn + T - 1) / T;
  std::vector<uint32_t> part(T, 0);
  for (int tid = 0; tid < T; tid++) {
    int64_t i = (int64_t)Cn + tid - (int64_t)iters * T;
    uint32_t c = 0;
    for (uint32_t it = 0; it < iters; it++, i += T) {
      uint32_t w[4] = {0, 0, 0, 0};
      if (i >= 0) memcpy(w, data + 16 * i, 16);
      if (ilp) {
        const uint32_t u = W(c ^ w[0]) ^ w[1], r = W(w[2]) ^ w[3];
        c = SW2(u) ^ S(r);
      } else {
        uint32_t x = W(c ^ w[0]) ^ w[1];
        x = W(x) ^ w[2];
        x = W(x) ^ w[3];
        c = (it + 1 == iters) ? W(x) : S(x);
      }
    }
    part[tid] = c;
  }
  uint32_t total = 0;
  for (int lane = 0; lane < 32; lane++) {
    uint32_t q = 0;
    for (int kk = 0; kk < T / 32; kk++) q = tab(t->adv128, q) ^ part[lane + 32 * kk];
    uint32_t lp = t->pow_word[4 * (31 - lane)];
    if (ilp) lp = crc_multmodp(lp, t->einv);
    total ^= crc_multmodp(q, lp);
  }
  // the identity the correction rests on: einv * x^(128*(T-1)) == 1
  if (crc_multmodp(t->einv, crc_host_xpow8((uint64_t)16 * (uint64_t)(T - 1))) != 0x80000000u) total = ~total;
  delete t;
  return total;
}

// Host emulation of the run checksum of k_emit_fast4 (emit_pipe.cuh): FE_THREADS threads, thread t folds the FE4_RUN
// chunks ending FE4_RUN*(255-t) chunks before the end (chunks before the data are zeros) through the lane-private digit
// tables of W, laid out and read with the kernel's code (emit4_wtab_value, emit4_next_word); lane l folds partials
// l, l+32, ... by Horner with x^(8*80*32), multiplies by x^(8*80*(31-l)), and the lanes xor.  nchunks <= FE_THREADS * FE4_RUN.  Returns the raw remainder (init 0, no final xor) of the nchunks * 16
// bytes.
uint32_t tezgpu_debug_run_fold_emulate(const uint8_t *data, uint32_t nchunks) {
  if (nchunks > (uint32_t)(FE_THREADS * FE4_RUN)) return 0;
  CrcTables *t = new CrcTables();
  crc_build_tables(*t, EMIT_CRC_STRIDE_WORDS);
  // the kernel's shared-memory layout: entry e of table k for lane l at word ((k << FE4_WBITS) + e) * 32 + l
  std::vector<uint32_t> wtab((size_t)FE4_WENTRIES * 32);
  for (uint32_t i = 0; i < (uint32_t)FE4_WENTRIES * 32; i++) wtab[i] = emit4_wtab_value(t, (i >> 5) >> FE4_WBITS, (i >> 5) & ((1u << FE4_WBITS) - 1));
  const uint32_t x_hor = t->pow0[FE4_RUN_BYTES * 32];
  auto H = [&](uint32_t x) { return crc_multmodp(x, x_hor); };
  const int32_t Cn = (int32_t)nchunks;
  std::vector<uint32_t> part(FE_THREADS, 0);
  for (int tid = 0; tid < FE_THREADS; tid++) {
    uint32_t c = 0;
    for (int k = 0; k < FE4_RUN; k++) {
      const int32_t i = Cn - FE4_RUN * (FE_THREADS - tid) + k;
      if (i < 0) continue;
      uint32_t w[4];
      memcpy(w, data + 16 * (size_t)i, 16);
      const uint8_t *wt = reinterpret_cast<const uint8_t *>(wtab.data() + (tid & 31));
      for (int q = 0; q < 4; q++) c = emit4_next_word(wt, c ^ w[q]);
    }
    part[tid] = c;
  }
  uint32_t total = 0;
  for (int lane = 0; lane < 32; lane++) {
    uint32_t q = 0;
    for (int kk = 0; kk < FE_THREADS / 32; kk++) q = H(q) ^ part[lane + 32 * kk];
    total ^= crc_multmodp(q, t->pow0[FE4_RUN_BYTES * (31 - lane)]);
  }
  delete t;
  return total;
}

int32_t tezgpu_debug_fixed_emit_plan(uint32_t klen, uint32_t vlen, int32_t layout, int32_t *kernel, uint32_t *recs_per_tile) {
  TG_API_BEGIN
  TG_CHECK(kernel && recs_per_tile, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(layout >= 0 && layout <= 2, TEZGPU_E_INVALID, "layout must be 0 (packed, aligned), 1 (explicit offsets) or 2 (run table)");
  TG_CHECK((uint64_t)klen + vlen > 0 && (uint64_t)klen + vlen + 10 < (1ull << 32), TEZGPU_E_INVALID, "record size out of range");
  // only the view's shape is read: which layout, and the alignment of kv
  static const uint64_t some_offsets[1] = {0};
  Records r;
  memset(&r, 0, sizeof(r));
  r.kv = reinterpret_cast<const uint8_t *>(uintptr_t(1) << 12);
  r.fixed = 1;
  r.klen = klen;
  r.vlen = vlen;
  if (layout == 1) r.key_off = some_offsets;
  if (layout == 2) r.use_runs = 1;
  const FixedEmitPlan plan = plan_fixed_emit(r, fixed_framing(klen, vlen).rec_size);
  *kernel = (int32_t)plan.kernel;
  *recs_per_tile = plan.recs_per_tile;
  TG_API_END
}

int32_t tezgpu_debug_emit_grid(int32_t device, int32_t kernel, uint64_t tiles, uint32_t *ctas, uint32_t *groups_per_cta) {
  TG_API_BEGIN
  TG_CHECK(ctas && groups_per_cta, TEZGPU_E_INVALID, "null argument");
  TG_CHECK(kernel >= 0 && kernel <= (int32_t)FixedEmitKernel::General, TEZGPU_E_INVALID, "kernel must be 0 to 4 (tezgpu_debug_fixed_emit_plan)");
  TG_CHECK(tiles < (1ull << 32), TEZGPU_E_INVALID, "more than 2^32-1 tiles");
  DeviceScope ds(device);
  int sms = 0;
  TG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const EmitGrid g = fixed_emit_grid(device, sms, (FixedEmitKernel)kernel, tiles);
  *ctas = g.ctas;
  *groups_per_cta = g.groups;
  TG_API_END
}

}  // extern "C"

#include "merger_api.inl"
#include "sample_api.inl"

// tez_runtime_library.cc -- host-side C++ mirror of OrderedPartitionedKVOutput / OrderedGroupedKVInput on top of the
// tezgpu_* C ABI (include/tezgpu.h).  See include/tez_runtime.h.  Host logic only: configuration, memory request,
// spill policy, file naming, counters, events, value grouping.  All sorting / merging / IFile bytes come from the
// device library -- there is no CPU implementation of the hot path in here.
//
// RL/  = /root/reference/tez-runtime-library/src/main/java/org/apache/tez/runtime/library/
// SORT/ = RL/common/sort/impl/   OG/ = RL/common/shuffle/orderedgrouped/
#include <errno.h>
#include <fcntl.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/tez_runtime.h"
#include "../../../include/tezgpu.h"

namespace tezrt {

struct Err : std::runtime_error {
  int code;
  Err(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};
static thread_local std::string g_err;
#define RT_CHECK(cond, code, msg) do { if (!(cond)) throw Err((code), (msg)); } while (0)
static void gpu_check(int32_t rc) { if (rc != 0) throw Err(rc, tezgpu_last_error()); }

// ---------------------------------------------------------------- configuration (keys: RL/api/TezRuntimeConfiguration.java)
struct Configuration {
  std::map<std::string, std::string> kv;
  explicit Configuration(const char *text) {
    std::string s = text ? text : "";
    size_t pos = 0;
    while (pos < s.size()) {
      size_t nl = s.find('\n', pos);
      if (nl == std::string::npos) nl = s.size();
      std::string line = s.substr(pos, nl - pos);
      size_t eq = line.find('=');
      if (eq != std::string::npos) kv[line.substr(0, eq)] = line.substr(eq + 1);
      pos = nl + 1;
    }
  }
  std::string get(const std::string &k, const std::string &d) const { auto it = kv.find(k); return it == kv.end() ? d : it->second; }
  long getInt(const std::string &k, long d) const { auto it = kv.find(k); return it == kv.end() ? d : atol(it->second.c_str()); }
  double getFloat(const std::string &k, double d) const { auto it = kv.find(k); return it == kv.end() ? d : atof(it->second.c_str()); }
  bool getBoolean(const std::string &k, bool d) const {
    auto it = kv.find(k);
    if (it == kv.end()) return d;
    return it->second == "true" || it->second == "TRUE" || it->second == "1";
  }
};

static const char *K_SORT_MB = "tez.runtime.io.sort.mb";                       // :115-116 default 100
static const char *K_SORTER_CLASS = "tez.runtime.sorter.class";                // :167-169 default PIPELINED
static const char *K_KEY_CLASS = "tez.runtime.key.class";
static const char *K_KEY_COMPARATOR = "tez.runtime.key.comparator.class";
static const char *K_PARTITIONER = "tez.runtime.partitioner.class";
static const char *K_EMPTY_PARTITIONS = "tez.runtime.empty.partitions.info-via-events.enabled";  // :506-509 default true
static const char *K_FINAL_MERGE = "tez.runtime.enable.final-merge.in.output";  // :555-557 default true
static const char *K_REPORT_STATS = "tez.runtime.report.partition.stats";       // :195-198 default memory_optimized
static const char *K_COMPRESS = "tez.runtime.compress";
static const char *K_COMPRESS_CODEC = "tez.runtime.compress.codec";
static const char *DEFAULT_CODEC = "org.apache.hadoop.io.compress.DefaultCodec";
static const char *LZ4_CODEC = "org.apache.hadoop.io.compress.Lz4Codec";
static const char *K_LZ4_BUFFERSIZE = "io.compression.codec.lz4.buffersize";   // CommonConfigurationKeys, default 256 KiB
static const char *ZSTD_CODEC = "org.apache.hadoop.io.compress.ZStandardCodec";
static const char *K_SERIALIZATIONS = "io.serializations";
static const char *K_VALUE_CLASS = "tez.runtime.value.class";
static const char *K_COMBINER_CLASS = "tez.runtime.combiner.class";
static const char *K_COMBINE_MIN_SPILLS = "tez.runtime.combine.min.spills";  // TezRuntimeConfiguration:128-130 default 3
static const char *K_UNORDERED_BUFFER_MB = "tez.runtime.unordered.output.buffer.size-mb";  // :204-206 default 100
static const char *K_PIPELINED_SHUFFLE = "tez.runtime.pipelined-shuffle.enabled";           // default false
static const char *K_MERGE_BUDGET_MB = "tez.runtime.gpu.merge.device.budget.mb";           // this project's; default 0

static bool ends_with(const std::string &s, const char *suf) {
  size_t n = strlen(suf);
  return s.size() >= n && s.compare(s.size() - n, n, suf) == 0;
}

// closed set of key classes the device can order (SURVEY 7 "hard parts"); anything else is rejected at start()
static int comparator_for(const Configuration &c) {
  std::string key = c.get(K_KEY_CLASS, ""), cmp = c.get(K_KEY_COMPARATOR, ""), ser = c.get(K_SERIALIZATIONS, "");
  if (ends_with(key, "io.Text")) return TEZGPU_CMP_TEXT;
  if (ends_with(key, "io.IntWritable")) return TEZGPU_CMP_INT;
  if (ends_with(key, "io.LongWritable")) return TEZGPU_CMP_LONG;
  if (ends_with(key, "io.BytesWritable")) {
    if (ends_with(cmp, "TezBytesComparator") || ser.find("TezBytesWritableSerialization") != std::string::npos) return TEZGPU_CMP_BYTES;
    return TEZGPU_CMP_BYTESWRITABLE;
  }
  throw Err(TEZGPU_E_UNSUPPORTED, "key class '" + key + "' has no device comparator (supported: Text, BytesWritable, IntWritable, LongWritable)");
}

// The combiners the device runs: MRCombiner (tez-mapreduce combine/MRCombiner.java) with a sum reducer over the value
// class it sums.  The reducer class is mapreduce.job.combine.class under the new API and mapred.combiner.class under
// the old one (ConfigUtils.useNewApi: mapred.mapper.new-api, default false).  Any other combiner is not run: MR
// semantics allow a combiner to run zero times.
static int combiner_for(const Configuration &c) {
  if (!ends_with(c.get(K_COMBINER_CLASS, ""), "combine.MRCombiner")) return TEZGPU_COMBINE_NONE;
  const bool new_api = c.getBoolean("mapred.mapper.new-api", false);
  const std::string red = c.get(new_api ? "mapreduce.job.combine.class" : "mapred.combiner.class", "");
  const std::string val = c.get(K_VALUE_CLASS, "");
  if ((red == "org.apache.hadoop.mapreduce.lib.reduce.IntSumReducer" || red == "org.apache.hadoop.examples.WordCount$IntSumReducer") &&
      val == "org.apache.hadoop.io.IntWritable")
    return TEZGPU_COMBINE_SUM_INT;
  if ((red == "org.apache.hadoop.mapreduce.lib.reduce.LongSumReducer" || red == "org.apache.hadoop.mapred.lib.LongSumReducer") &&
      val == "org.apache.hadoop.io.LongWritable")
    return TEZGPU_COMBINE_SUM_LONG;
  return TEZGPU_COMBINE_NONE;
}

// ---------------------------------------------------------------- TotalOrderPartitioner
static const char *TOTAL_ORDER_NEW = "org.apache.hadoop.mapreduce.lib.partition.TotalOrderPartitioner";
static const char *TOTAL_ORDER_OLD = "org.apache.hadoop.mapred.lib.TotalOrderPartitioner";
static const char *K_PARTITION_PATH = "mapreduce.totalorderpartitioner.path";           // default _partition.lst
static const char *K_NATURAL_ORDER = "mapreduce.totalorderpartitioner.naturalorder";    // default true
// (mapreduce.totalorderpartitioner.trie.maxdepth only shapes Java's index over the split points: nothing to do here)

// The output's partitioner is TotalOrderPartitioner: named directly, or wrapped by MRPartitioner (with more than one
// partition, where MRPartitioner instantiates it) as mapreduce.job.partitioner.class under the new API and
// mapred.partitioner.class under the old one (tez-mapreduce partition/MRPartitioner.java).
static bool total_order_partitioner(const Configuration &c, int P) {
  auto is_total = [](const std::string &cls) { return cls == TOTAL_ORDER_NEW || cls == TOTAL_ORDER_OLD; };
  const std::string pc = c.get(K_PARTITIONER, "");
  if (is_total(pc)) return true;
  if (pc != "org.apache.tez.mapreduce.partition.MRPartitioner" || P <= 1) return false;
  const bool new_api = c.getBoolean("mapred.mapper.new-api", false);
  return is_total(c.get(new_api ? "mapreduce.job.partitioner.class" : "mapred.partitioner.class", ""));
}

// The split keys of a partition file (what TotalOrderPartitioner.readPartitions reads with SequenceFile.Reader):
// SequenceFile version 6, uncompressed or record-compressed (only values are compressed there, and they are skipped).
// Keys come back serialized, exactly as stored.  Refusals name the file: TEZGPU_E_INVALID for an unreadable file, a
// key class other than `key_class`, or a malformed header or record; TEZGPU_E_UNSUPPORTED for block compression.
struct PartitionFile {
  std::vector<uint8_t> keys;
  std::vector<uint64_t> off;
  std::vector<uint32_t> len;
};
static PartitionFile read_partition_file(const std::string &path, const std::string &key_class) {
  std::vector<uint8_t> b;
  {
    int fd = ::open(path.c_str(), O_RDONLY);
    RT_CHECK(fd >= 0, TEZGPU_E_INVALID, "Can't read partitions file " + path + ": " + strerror(errno));
    uint8_t buf[1 << 16];
    ssize_t r;
    while ((r = ::read(fd, buf, sizeof(buf))) > 0) b.insert(b.end(), buf, buf + r);
    const int e = errno;
    ::close(fd);
    RT_CHECK(r == 0, TEZGPU_E_INVALID, "Can't read partitions file " + path + ": " + strerror(e));
  }
  size_t pos = 0;
  auto bad = [&](const std::string &why) { return Err(TEZGPU_E_INVALID, "partitions file " + path + ": " + why); };
  auto need = [&](size_t n, const char *what) { if (b.size() - pos < n) throw bad(std::string("truncated ") + what); };
  auto i32 = [&](const char *what) {
    need(4, what);
    const uint32_t v = ((uint32_t)b[pos] << 24) | ((uint32_t)b[pos + 1] << 16) | ((uint32_t)b[pos + 2] << 8) | b[pos + 3];
    pos += 4;
    return (int32_t)v;
  };
  auto vint = [&](const char *what) {   // WritableUtils.readVInt
    need(1, what);
    const int8_t first = (int8_t)b[pos++];
    if (first >= -112) return (int64_t)first;
    const bool neg = first < -120;
    const int n = neg ? -(first + 120) : -(first + 112);
    need((size_t)n, what);
    int64_t v = 0;
    for (int i = 0; i < n; i++) v = (v << 8) | b[pos++];
    return neg ? ~v : v;
  };
  auto text = [&](const char *what) {   // Text.readString
    const int64_t n = vint(what);
    if (n < 0) throw bad(std::string("negative length in ") + what);
    need((size_t)n, what);
    std::string t(b.begin() + pos, b.begin() + pos + n);
    pos += (size_t)n;
    return t;
  };
  need(4, "header");
  if (memcmp(b.data(), "SEQ", 3) != 0 || b[3] != 6) throw bad("not a SequenceFile of version 6");
  pos = 4;
  const std::string kc = text("key class");
  if (kc != key_class) throw bad("wrong key class: " + key_class + " is not " + kc);   // SequenceFile.Reader.next's order
  text("value class");
  need(2, "header");
  const bool compressed = b[pos++] != 0, block = b[pos++] != 0;
  if (block) throw Err(TEZGPU_E_UNSUPPORTED, "partitions file " + path + ": block-compressed SequenceFiles are not read");
  if (compressed) text("codec class");
  const int32_t meta = i32("metadata");
  if (meta < 0) throw bad("negative metadata count");
  for (int32_t i = 0; i < 2 * meta; i++) text("metadata");
  need(16, "sync marker");
  const size_t sync = pos;
  pos += 16;
  PartitionFile f;
  while (pos < b.size()) {
    const int32_t rec = i32("record");
    if (rec == -1) {
      need(16, "sync marker");
      if (memcmp(b.data() + pos, b.data() + sync, 16) != 0) throw bad("sync marker mismatch");
      pos += 16;
      continue;
    }
    const int32_t kl = i32("record");
    if (rec < 0 || kl < 0 || kl > rec) throw bad("malformed record");
    need((size_t)rec, "record");
    f.off.push_back(f.keys.size());
    f.len.push_back((uint32_t)kl);
    f.keys.insert(f.keys.end(), b.begin() + pos, b.begin() + pos + kl);
    pos += (size_t)rec;
  }
  f.keys.reserve(f.keys.size() + 1);   // a valid pointer even when every split key is empty
  return f;
}

// ---------------------------------------------------------------- small utilities
static void mkdirs(const std::string &path) {
  for (size_t i = 1; i <= path.size(); i++)
    if (i == path.size() || path[i] == '/') {
      std::string p = path.substr(0, i);
      if (::mkdir(p.c_str(), 0755) != 0 && errno != EEXIST) throw Err(TEZGPU_E_IO, "mkdir " + p + ": " + strerror(errno));
    }
}
static std::vector<uint8_t> read_file(const std::string &p, uint64_t off = 0, int64_t len = -1) {
  int fd = ::open(p.c_str(), O_RDONLY);
  RT_CHECK(fd >= 0, TEZGPU_E_IO, "open " + p + ": " + strerror(errno));
  struct stat st;
  fstat(fd, &st);
  uint64_t n = len < 0 ? (uint64_t)st.st_size - off : (uint64_t)len;
  std::vector<uint8_t> b(n);
  uint64_t got = 0;
  while (got < n) {
    ssize_t r = ::pread(fd, b.data() + got, n - got, (off_t)(off + got));
    if (r <= 0) { ::close(fd); throw Err(TEZGPU_E_IO, "short read of " + p); }
    got += (uint64_t)r;
  }
  ::close(fd);
  return b;
}
// TezCommonUtils.compressByteArrayToByteString with newBestCompressionDeflater(): raw deflate, level 9
static std::string deflate_raw(const std::vector<uint8_t> &in) {
  z_stream z;
  memset(&z, 0, sizeof(z));
  RT_CHECK(deflateInit2(&z, 9, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) == Z_OK, TEZGPU_E_INVALID, "deflateInit2");
  std::string out(deflateBound(&z, in.size()) + 16, '\0');
  z.next_in = const_cast<Bytef *>(in.data());
  z.avail_in = (uInt)in.size();
  z.next_out = (Bytef *)&out[0];
  z.avail_out = (uInt)out.size();
  int rc = deflate(&z, Z_FINISH);
  RT_CHECK(rc == Z_STREAM_END, TEZGPU_E_INVALID, "deflate");
  out.resize(z.total_out);
  deflateEnd(&z);
  return out;
}
// protobuf wire helpers (ShufflePayloads.proto)
static void pb_varint(std::string &o, uint64_t v) { while (v >= 0x80) { o.push_back((char)(v | 0x80)); v >>= 7; } o.push_back((char)v); }
static void pb_tag(std::string &o, int field, int wt) { pb_varint(o, (uint64_t)(field << 3 | wt)); }
static void pb_bytes(std::string &o, int field, const std::string &b) { pb_tag(o, field, 2); pb_varint(o, b.size()); o += b; }
static void pb_int(std::string &o, int field, int64_t v) { pb_tag(o, field, 0); pb_varint(o, (uint64_t)v); }

struct Event {
  int type;
  std::string payload;
  int source_index_start = 0, count = 0;
};

// RoaringBitmap portable serialization (no run containers) of a sorted value list -- the format
// RoaringBitmap.serialize(DataOutput) writes for ShuffleUtils.getPartitionStatsForPhysicalOutput (:486-500)
static std::vector<uint8_t> roaring_serialize(const std::vector<uint32_t> &vals) {
  std::vector<std::pair<uint16_t, std::vector<uint16_t>>> cont;
  for (uint32_t v : vals) {
    uint16_t hi = (uint16_t)(v >> 16), lo = (uint16_t)v;
    if (cont.empty() || cont.back().first != hi) cont.push_back({hi, {}});
    cont.back().second.push_back(lo);
  }
  std::vector<uint8_t> o;
  auto u16 = [&](uint32_t x) { o.push_back((uint8_t)x); o.push_back((uint8_t)(x >> 8)); };
  auto u32 = [&](uint32_t x) { u16(x & 0xFFFF); u16(x >> 16); };
  u32(12346);  // SERIAL_COOKIE_NO_RUNCONTAINER
  u32((uint32_t)cont.size());
  for (auto &c : cont) { u16(c.first); u16((uint32_t)c.second.size() - 1); }
  uint32_t off = 8 + 8 * (uint32_t)cont.size();
  for (auto &c : cont) { u32(off); off += c.second.size() > 4096 ? 8192u : 2u * (uint32_t)c.second.size(); }
  for (auto &c : cont) {
    if (c.second.size() > 4096) {
      std::vector<uint8_t> bm(8192, 0);
      for (uint16_t x : c.second) bm[x >> 3] |= (uint8_t)(1u << (x & 7));
      o.insert(o.end(), bm.begin(), bm.end());
    } else {
      for (uint16_t x : c.second) u16(x);
    }
  }
  return o;
}

// tez.runtime.compress / tez.runtime.compress.codec (IFile.Writer / Reader via CodecUtils.getCodec): DefaultCodec and
// Lz4Codec run on the device, any other class is refused by name.  Deviation from Tez: with compression on and no codec
// named, Tez uses DefaultCodec; here that configuration keeps being refused (DESIGN.md 9).  Lz4Codec: Java's
// Lz4Decompressor decodes each chunk into a buffer of io.compression.codec.lz4.buffersize bytes, so a buffer smaller
// than the device writer's worst-case chunk (TEZGPU_LZ4_CHUNK_BOUND) could not read the device's output, and Java
// writers with a buffer over 262,144 bytes write chunks the device reader refuses: both are refused by key name.
// ZStandardCodec: io.compression.codec.zstd.level is accepted and has no effect on the device writer, which has one
// parse; a Java reader reads its frames at any level (DESIGN.md 9).
static int codec_for(const Configuration &conf) {
  if (!conf.getBoolean(K_COMPRESS, false)) return TEZGPU_CODEC_NONE;
  const std::string codec = conf.get(K_COMPRESS_CODEC, "");
  RT_CHECK(!codec.empty(), TEZGPU_E_UNSUPPORTED, "tez.runtime.compress=true: IFile codecs are not supported on the device path yet");
  if (codec == LZ4_CODEC) {
    const long buf = conf.getInt(K_LZ4_BUFFERSIZE, 256 * 1024);
    RT_CHECK(buf >= TEZGPU_LZ4_CHUNK_BOUND && buf <= 256 * 1024, TEZGPU_E_UNSUPPORTED,
             std::string(K_LZ4_BUFFERSIZE) + "=" + std::to_string(buf) + ": the device path needs " +
                 std::to_string(TEZGPU_LZ4_CHUNK_BOUND) + " to 262144 bytes with " + LZ4_CODEC);
    return TEZGPU_CODEC_LZ4;
  }
  if (codec == ZSTD_CODEC) return TEZGPU_CODEC_ZSTD;
  RT_CHECK(codec == DEFAULT_CODEC, TEZGPU_E_UNSUPPORTED,
           std::string(K_COMPRESS_CODEC) + "=" + codec + ": only " + DEFAULT_CODEC + ", " + LZ4_CODEC + " and " + ZSTD_CODEC +
               " are supported on the device path");
  return TEZGPU_CODEC_DEFAULT;
}

// tez.runtime.gpu.merge.device.budget.mb: the device memory, in MiB, that the reduce-side merge and the output's final
// merge over several spills may hold (tezgpu_merge_open_bounded; compressed inputs are decoded first with
// tezgpu_decode_segments).  0 or unset: no budget, the one-step merge as before.  Checked at initialize(), before any
// device call.  Concatenations (the unordered edges) hold no merge workspace and ignore it.
static uint64_t merge_budget(const Configuration &c) {
  const long mb = c.getInt(K_MERGE_BUDGET_MB, 0);
  RT_CHECK(mb == 0 || mb >= (long)(TEZGPU_MERGE_BUDGET_MIN >> 20), TEZGPU_E_INVALID,
           std::string(K_MERGE_BUDGET_MB) + "=" + std::to_string(mb) + ": a device budget is at least " +
               std::to_string(TEZGPU_MERGE_BUDGET_MIN >> 20) + " MiB (0: none)");
  return (uint64_t)mb << 20;
}

// what a merge took: steps (0: no merge ran, 1: one step), the most device memory it held at once and the bytes it
// uploaded from the host (both 0 unless it ran under a budget; the larger of the decode's and the merge's peak)
struct MergeInfo {
  int32_t steps = 0;
  uint64_t peak = 0, h2d = 0;
};

// ================================================================================================ output side
// GpuSorter: the ExternalSorter seam (SORT/ExternalSorter.java:74-92,281-288) backed by tezgpu_sorter.  Records are
// batched on the host and handed to the device; when the collected bytes reach the granted sort memory the device
// content is spilled (sorted IFile + index), and flush() either renames the single spill or runs the final merge over
// the spills on the device (PipelinedSorter.flush :664-859).
struct GpuSorter {
  tezgpu_sorter *h = nullptr;
  tezgpu_conf gc;
  int P;
  int64_t available_memory;
  bool final_merge;
  std::string work_dir, uid;
  // host batch
  std::vector<uint8_t> kv;
  std::vector<uint32_t> koff, voff, vlen;
  std::vector<int32_t> part;
  bool given_partitions = false;
  uint64_t collected_bytes = 0;
  int num_spills = 0;
  std::vector<std::string> spill_files, spill_index_files;
  std::vector<std::vector<int64_t>> spill_index;
  std::string final_out, final_index;
  std::vector<int64_t> final_idx;
  std::vector<int64_t> partition_stats;  // partitionStats[p] += rawLength at every spill (SORT/PipelinedSorter.java:631-633)
  int last_spill_rle = 0;                // merger.needsRLE() of the most recent spill's SpanMerger (:599,805,814)
  int combiner = TEZGPU_COMBINE_NONE;    // runs on every spill, and on the final merge from min_spills spills on (:601-609,815-820)
  int min_spills = 3;
  int codec = TEZGPU_CODEC_NONE;         // every spill is compressed; the final merge reads and writes through it
  uint64_t budget = 0;                   // merge_budget: the final merge of an uncompressed ordered output holds at most this
  MergeInfo info;                        // of the final merge
  std::map<std::string, int64_t> &counters;

  GpuSorter(const tezgpu_conf &c, int64_t mem, bool fm, const std::string &wd, const std::string &u, std::map<std::string, int64_t> &ctr)
      : gc(c), P(c.num_partitions), available_memory(mem), final_merge(fm), work_dir(wd), uid(u), counters(ctr) {
    gpu_check(tezgpu_sorter_create(&gc, &h));
  }
  ~GpuSorter() { if (h) tezgpu_sorter_destroy(h); }
  void set_combiner(int c, int min_spills_for_combine) {
    gpu_check(tezgpu_sorter_set_combiner(h, c));
    combiner = c;
    min_spills = min_spills_for_combine;
  }
  void set_codec(int c) {
    gpu_check(tezgpu_sorter_set_codec(h, c));
    codec = c;
  }
  // MRCombiner's COMBINE_INPUT_RECORDS / COMBINE_OUTPUT_RECORDS of one combined write
  void count_combine(const tezgpu_stats &st) {
    counters["COMBINE_INPUT_RECORDS"] += st.output_records;
    counters["COMBINE_OUTPUT_RECORDS"] += st.spilled_records;
  }

  // TezTaskOutputFiles (RL/common/task/local/output/TezTaskOutputFiles.java:88-231)
  std::string spill_dir(int n) const { return work_dir + "/output/" + uid + "_" + std::to_string(n); }
  std::string final_dir() const { return work_dir + "/output/" + uid; }

  void push_batch() {
    if (koff.empty()) return;
    gpu_check(tezgpu_sorter_collect_batch(h, kv.data(), kv.size(), koff.data(), voff.data(), vlen.data(),
                                          given_partitions ? part.data() : nullptr, (uint32_t)koff.size()));
    kv.clear(); koff.clear(); voff.clear(); vlen.clear(); part.clear();
  }

  void write(const uint8_t *k, uint32_t kl, const uint8_t *v, uint32_t vl, int32_t partition) {
    if (partition >= 0) {
      RT_CHECK(partition < P, TEZGPU_E_INVALID, "Illegal partition for key (" + std::to_string(partition) + ")");  // PipelinedSorter.java:410-413
      RT_CHECK(given_partitions || (koff.empty() && collected_bytes == 0 && num_spills == 0), TEZGPU_E_INVALID, "mixing partitioner modes");
      given_partitions = true;
    } else {
      RT_CHECK(!given_partitions, TEZGPU_E_INVALID, "mixing partitioner modes");
    }
    uint64_t rec = (uint64_t)kl + vl;
    if (collected_bytes && collected_bytes + kv.size() + rec > (uint64_t)available_memory) { push_batch(); spill(); }
    koff.push_back((uint32_t)kv.size());
    kv.insert(kv.end(), k, k + kl);
    voff.push_back((uint32_t)kv.size());
    kv.insert(kv.end(), v, v + vl);
    vlen.push_back(vl);
    if (given_partitions) part.push_back(partition);
    counters["OUTPUT_RECORDS"]++;
    counters["OUTPUT_BYTES"] += (int64_t)rec;
    if (kv.size() >= (32u << 20) || kv.size() + 8 >= (uint64_t)available_memory) {
      collected_bytes += kv.size();
      push_batch();
    }
  }

  // last: the spill flush() forces, i.e. the unordered writer's current buffer, whose records
  // UnorderedPartitionedKVWriter does not count as spilled (finalSpill passes no counter, :985)
  void spill(bool last = false) {
    std::string dir = spill_dir(num_spills);
    mkdirs(dir);
    std::string f = dir + "/file.out", fi = f + ".index";
    std::vector<int64_t> idx((size_t)P * 3);
    tezgpu_stats st;
    gpu_check(tezgpu_sorter_flush(h, f.c_str(), fi.c_str(), idx.data(), &st));
    gpu_check(tezgpu_sorter_reset(h));
    // adjustSpillCounters (:468-482)
    if (!final_merge) counters["OUTPUT_BYTES_WITH_OVERHEAD"] += st.output_bytes_with_overhead;
    else if (num_spills > 0) { counters["ADDITIONAL_SPILLS_BYTES_WRITTEN"] += st.file_out_bytes; counters["OUTPUT_BYTES_WITH_OVERHEAD"] = 0; }
    else counters["OUTPUT_BYTES_WITH_OVERHEAD"] += st.output_bytes_with_overhead;
    if (!(last && gc.sorter_impl == TEZGPU_SORTER_UNORDERED)) counters["SPILLED_RECORDS"] += st.spilled_records;
    if (combiner) count_combine(st);
    last_spill_rle = st.rle_used;
    partition_stats.resize((size_t)P, 0);
    for (int p = 0; p < P; p++) partition_stats[p] += idx[3 * p + 1];
    spill_files.push_back(f);
    spill_index_files.push_back(fi);
    spill_index.push_back(idx);
    num_spills++;
    collected_bytes = 0;
  }

  void flush() {
    collected_bytes += kv.size();
    push_batch();
    spill(true);  // "force a spill in flush()" (:679-690)
    counters["ADDITIONAL_SPILL_COUNT"] += num_spills - 1;
    if (!final_merge) {
      counters["SHUFFLE_CHUNK_COUNT"] = num_spills;
      int64_t phys = 0;
      for (auto &f : spill_files) { struct stat st; if (stat(f.c_str(), &st) == 0) phys += st.st_size; }
      counters["OUTPUT_BYTES_PHYSICAL"] += phys;
      return;
    }
    mkdirs(final_dir());
    final_out = final_dir() + "/file.out";
    final_index = final_out + ".index";
    if (num_spills == 1) {
      // sameVolRename (:730-756)
      RT_CHECK(::rename(spill_files[0].c_str(), final_out.c_str()) == 0, TEZGPU_E_IO, "rename " + spill_files[0]);
      RT_CHECK(::rename(spill_index_files[0].c_str(), final_index.c_str()) == 0, TEZGPU_E_IO, "rename " + spill_index_files[0]);
      ::rmdir(spill_dir(0).c_str());
      final_idx = spill_index[0];
      counters["SHUFFLE_CHUNK_COUNT"] = 1;
      struct stat st;
      stat(final_out.c_str(), &st);
      counters["OUTPUT_BYTES_PHYSICAL"] += st.st_size;
      return;
    }
    // final merge across spills, every partition at once on the device (:774-836)
    std::vector<std::vector<uint8_t>> bytes(num_spills);
    std::vector<tezgpu_segment> segs;
    std::vector<int64_t> raws;   // rawLength of every segment (the compressed ones need it)
    std::vector<int> seg_spill;  // spill of every segment
    for (int s = 0; s < num_spills; s++) {
      bytes[s] = read_file(spill_files[s]);
      counters["ADDITIONAL_SPILLS_BYTES_READ"] += (int64_t)bytes[s].size();
      for (int p = 0; p < P; p++) {
        int64_t start = spill_index[s][3 * p], raw = spill_index[s][3 * p + 1], part_len = spill_index[s][3 * p + 2];
        if (raw > 6 || (!gc.send_empty_partition_details && part_len > 0)) {  // TezIndexRecord.hasData (:51-55)
          tezgpu_segment sg;
          sg.data = bytes[s].data() + start;
          sg.len = (uint64_t)part_len;
          sg.flags = TEZGPU_SEG_HAS_HEADER;
          sg.partition = (uint32_t)p;
          segs.push_back(sg);
          raws.push_back(raw);
          seg_spill.push_back(s);
        }
      }
    }
    tezgpu_conf mc = gc;
    mc.fixed_key_len = mc.fixed_val_len = 0;
    tezgpu_merger *m = nullptr;
    final_idx.assign((size_t)P * 3, 0);
    tezgpu_stats st;
    const bool combine = combiner && num_spills >= min_spills;
    int32_t rc;
    if (gc.sorter_impl == TEZGPU_SORTER_UNORDERED) {
      // UnorderedPartitionedKVWriter.mergeAll (:1058-1144): per partition the current buffer (the forced last spill),
      // then the spills in order, concatenated, written without run-length encoding
      std::vector<int64_t> at((size_t)num_spills * P, -1);   // segment of (spill, partition), if any
      for (size_t i = 0; i < segs.size(); i++) at[(size_t)seg_spill[i] * P + segs[i].partition] = (int64_t)i;
      std::vector<tezgpu_segment> cs;
      std::vector<int64_t> craws;
      for (int p = 0; p < P; p++)
        for (int k = 0; k < num_spills; k++) {
          const int64_t i = at[(size_t)(k == 0 ? num_spills - 1 : k - 1) * P + p];
          if (i >= 0) { cs.push_back(segs[(size_t)i]); craws.push_back(raws[(size_t)i]); }
        }
      gpu_check(tezgpu_concat_open(&mc, cs.data(), craws.data(), (uint32_t)cs.size(), codec, &m));
      rc = tezgpu_merge_write_partitions(m, final_out.c_str(), final_index.c_str(), /*rle=*/0, final_idx.data(), &st);
    } else {
      // under a budget the merge runs in key-range steps over the spills in host memory; a bounded merge writes no
      // compressed output, so a compressed final merge takes one step whatever the budget
      const bool bounded = budget && !codec;
      if (bounded) gpu_check(tezgpu_merge_open_bounded(&mc, segs.data(), raws.data(), (uint32_t)segs.size(), codec, budget, &m));
      else gpu_check(tezgpu_merge_open_codec(&mc, segs.data(), raws.data(), (uint32_t)segs.size(), codec, &m));
      // TezMerger.merge(..., checkForSameKeys = merger.needsRLE()) into Writer(..., rle = merger.needsRLE()), `merger`
      // being the SpanMerger of the last spill (SORT/PipelinedSorter.java:797-814)
      rc = tezgpu_merge_set_check_for_same_keys(m, last_spill_rle);
      if (rc == 0 && combine) rc = tezgpu_merge_set_combiner(m, combiner);
      if (rc == 0)
        rc = tezgpu_merge_write_partitions(m, final_out.c_str(), final_index.c_str(), /*rle=*/last_spill_rle, final_idx.data(), &st);
      if (rc == 0 && bounded) rc = tezgpu_merge_bounded_info(m, &info.steps, &info.peak, &info.h2d);
    }
    tezgpu_merge_close(m);
    if (!info.steps) info.steps = 1;
    gpu_check(rc);
    const uint64_t len = (uint64_t)st.file_out_bytes;
    counters["SPILLED_RECORDS"] += st.spilled_records;
    if (combine) count_combine(st);
    int64_t raw = 0;
    for (int p = 0; p < P; p++) raw += final_idx[3 * p + 1];
    counters["OUTPUT_BYTES_WITH_OVERHEAD"] += raw;
    counters["SHUFFLE_CHUNK_COUNT"] = 1;
    counters["OUTPUT_BYTES_PHYSICAL"] += (int64_t)len;
    for (int s = 0; s < num_spills; s++) {
      ::unlink(spill_files[s].c_str());
      ::unlink(spill_index_files[s].c_str());
      ::rmdir(spill_dir(s).c_str());
    }
  }
};

struct Output {
  Configuration conf;
  std::string work_dir, uid, dest_vertex, host;
  int port, P, device;
  int64_t task_memory, requested = 0, granted = -1;
  bool initialized = false, started = false, closed = false;
  bool send_empty = true, final_merge = true;
  bool unordered = false;   // UnorderedPartitionedKVOutput / UnorderedKVOutput: the writer in TEZGPU_SORTER_UNORDERED mode
  uint64_t budget = 0;      // merge_budget
  bool total_order;         // TotalOrderPartitioner: the device partitions by the split points of the partition file
  std::map<std::string, int64_t> counters;
  GpuSorter *sorter = nullptr;
  std::vector<Event> events;
  Output(const char *c, const char *wd, const char *u, const char *dv, const char *h, int pt, int64_t mem, int p, int dev)
      : conf(c), work_dir(wd ? wd : "."), uid(u ? u : "attempt"), dest_vertex(dv ? dv : ""), host(h ? h : "localhost"),
        port(pt), P(p), device(dev), task_memory(mem), total_order(total_order_partitioner(conf, p)) {}
  ~Output() { delete sorter; }

  void initialize() {
    budget = merge_budget(conf);
    if (unordered) {
      // UnorderedPartitionedKVWriter.getInitialMemoryRequirement (RL/common/writers/UnorderedPartitionedKVWriter.java:705-716)
      const long mb = conf.getInt(K_UNORDERED_BUFFER_MB, 100);
      RT_CHECK(mb > 0, TEZGPU_E_INVALID, std::string(K_UNORDERED_BUFFER_MB) + " should be larger than 0");
      requested = (int64_t)mb << 20;
      send_empty = true;   // the unordered writer always reports its empty partitions (generateDMEvent)
      final_merge = conf.getBoolean(K_FINAL_MERGE, true) && !conf.getBoolean(K_PIPELINED_SHUFFLE, false);
      initialized = true;
      return;
    }
    // ExternalSorter.getInitialMemoryRequirement (SORT/ExternalSorter.java:330-347)
    long mb = conf.getInt(K_SORT_MB, 100);
    int64_t req = (int64_t)mb << 20;
    RT_CHECK(mb > 0 && req < task_memory, TEZGPU_E_INVALID,
             std::string(K_SORT_MB) + " " + std::to_string(mb) + " should be larger than 0 and should be less than the available task memory (MB):" +
                 std::to_string(task_memory >> 20));
    requested = req;
    send_empty = conf.getBoolean(K_EMPTY_PARTITIONS, true);
    final_merge = conf.getBoolean(K_FINAL_MERGE, true);
    initialized = true;
  }
  void start() {
    RT_CHECK(initialized, TEZGPU_E_STATE, "start() before initialize()");
    if (started) return;
    RT_CHECK(granted >= 0, TEZGPU_E_STATE, "memory update not received (MemoryUpdateCallbackHandler.validateUpdateReceived)");
    std::string sc = conf.get(K_SORTER_CLASS, "PIPELINED");
    std::transform(sc.begin(), sc.end(), sc.begin(), ::toupper);
    RT_CHECK(unordered || sc == "PIPELINED" || sc == "LEGACY", TEZGPU_E_INVALID,
             "Invalid sorter class specified in config, propertyName=" + std::string(K_SORTER_CLASS) + ", value=" + sc + ", validValues=[LEGACY, PIPELINED]");
    const int codec = codec_for(conf);
    tezgpu_conf gc;
    memset(&gc, 0, sizeof(gc));
    gc.abi_version = TEZGPU_ABI_VERSION;
    gc.device = device;
    gc.num_partitions = P;
    std::string pc = conf.get(K_PARTITIONER, "org.apache.tez.runtime.library.partitioner.HashPartitioner");
    gc.partitioner = total_order ? TEZGPU_PART_TOTAL_ORDER : ends_with(pc, "HashPartitioner") ? TEZGPU_PART_HASH : TEZGPU_PART_GIVEN;
    // an unordered edge compares no keys: its key class only matters to the HashPartitioner's hashCode and to the
    // split points' order check
    gc.comparator = (!unordered || total_order || (gc.partitioner == TEZGPU_PART_HASH && P > 1)) ? comparator_for(conf) : TEZGPU_CMP_BYTES;
    // TotalOrderPartitioner.setConf: the partition file is read and checked here, before any device call
    PartitionFile splits;
    int32_t split_order = gc.comparator;
    if (total_order) {
      std::string path = conf.get(K_PARTITION_PATH, "_partition.lst");
      if (path.empty() || path[0] != '/') path = work_dir + "/" + path;
      const std::string kc = conf.get(K_KEY_CLASS, "");
      splits = read_partition_file(path, kc);
      if (conf.getBoolean(K_NATURAL_ORDER, true)) {
        if (ends_with(kc, "io.Text")) split_order = TEZGPU_CMP_TEXT;
        else if (ends_with(kc, "io.BytesWritable")) split_order = TEZGPU_CMP_BYTESWRITABLE;
      }
      // the count and order checks of tezgpu_sorter_set_split_points, on the host
      RT_CHECK((int64_t)splits.len.size() == (int64_t)P - 1, TEZGPU_E_INVALID, "Wrong number of partitions in keyset");
      gpu_check(tezgpu_debug_total_order_emulate(nullptr, nullptr, nullptr, 0, splits.keys.data(), splits.off.data(), splits.len.data(),
                                                 (uint32_t)splits.len.size(), gc.comparator, split_order, nullptr));
    }
    gc.rle_policy = TEZGPU_RLE_AUTO;
    gc.send_empty_partition_details = send_empty ? 1 : 0;
    gc.sorter_impl = unordered ? TEZGPU_SORTER_UNORDERED : sc == "LEGACY" ? 1 : 0;
    gc.mem_budget_bytes = (uint64_t)granted;
    sorter = new GpuSorter(gc, granted > 0 ? granted : requested, final_merge, work_dir, uid, counters);
    // UnorderedPartitionedKVWriter runs no combiner (and tezgpu_sorter_set_combiner refuses an unordered handle)
    if (const int c = unordered ? 0 : combiner_for(conf)) sorter->set_combiner(c, (int)conf.getInt(K_COMBINE_MIN_SPILLS, 3));
    if (codec) sorter->set_codec(codec);
    sorter->budget = budget;
    if (total_order)
      gpu_check(tezgpu_sorter_set_split_points(sorter->h, splits.keys.data(), splits.off.data(), splits.len.data(),
                                               (uint32_t)splits.len.size(), split_order));
    started = true;
  }
  void write(const uint8_t *k, uint32_t kl, const uint8_t *v, uint32_t vl, int32_t partition) {
    RT_CHECK(!(total_order && partition >= 0), TEZGPU_E_INVALID,
             "TotalOrderPartitioner output: the device computes the partition, write() takes none");
    RT_CHECK(started && !closed, TEZGPU_E_STATE, "write() outside start()..close()");
    RT_CHECK(partition >= 0 || sorter->gc.partitioner != TEZGPU_PART_GIVEN, TEZGPU_E_UNSUPPORTED,
             "custom partitioner: the caller must pass Partitioner.getPartition(key, value, numPartitions)");
    sorter->write(k, kl, v, vl, partition);
  }

  // ShuffleUtils.generateEventOnSpill / generateDMEPayload / generateVMEvent (RL/common/shuffle/ShuffleUtils.java:288-484)
  void generate_events(const std::vector<int64_t> &idx, const std::string &path_component, int spill_id, bool last) {
    // VertexManagerEvent
    if (final_merge || last) {
      std::string vm;
      pb_int(vm, 1, counters["OUTPUT_BYTES"]);
      std::string mode = conf.get(K_REPORT_STATS, "memory_optimized");
      std::vector<int64_t> sizes(P);
      // without the final merge the event of the last spill reports the sizes accumulated over every spill
      // (partitionStats, SORT/PipelinedSorter.java:631-633 -> ExternalSorter.getPartitionStats)
      for (int p = 0; p < P; p++)
        sizes[p] = (!final_merge && sorter && (int)sorter->partition_stats.size() == P) ? sorter->partition_stats[p] : idx[3 * p + 1];
      if (mode == "precise") {
        std::string d, packed;
        for (int p = 0; p < P; p++) pb_varint(packed, (uint64_t)((sizes[p] + (1 << 20) - 1) >> 20));
        pb_bytes(d, 1, packed);
        pb_bytes(vm, 3, d);
      } else if (mode != "none" && mode != "false") {
        // DATA_RANGE_IN_MB buckets THOUSAND,HUNDRED,TEN,ONE,ZERO -> RoaringBitmap (RL/utils/DATA_RANGE_IN_MB.java:22-47)
        static const int64_t lim[5] = {1000, 100, 10, 1, 0};
        std::vector<uint32_t> vals;
        for (int p = 0; p < P; p++) {
          int64_t mbs = (sizes[p] + (1 << 20) - 1) >> 20;
          int b = 4;
          for (int r = 0; r < 5; r++) if (mbs >= lim[r]) { b = r; break; }
          vals.push_back((uint32_t)(p * 5 + b));
        }
        std::vector<uint8_t> ser = roaring_serialize(vals);
        size_t cap = 32;  // DataOutputBuffer.getData(): the whole backing array goes through the deflater
        while (cap < ser.size()) cap <<= 1;
        ser.resize(cap, 0);
        pb_bytes(vm, 2, deflate_raw(ser));
      }
      pb_int(vm, 4, counters["OUTPUT_RECORDS"]);
      Event e;
      e.type = TEZRT_EVENT_VERTEX_MANAGER;
      e.payload = vm;
      events.push_back(e);
    }
    // CompositeDataMovementEvent(0, P, DataMovementEventPayloadProto)
    std::string dm;
    bool output_generated = true;
    if (send_empty) {
      int empty = 0, highest = -1;
      for (int p = 0; p < P; p++) if (!(idx[3 * p + 1] > 6)) { empty++; highest = p; }
      output_generated = empty != P;
      if (empty > 0) {
        std::vector<uint8_t> bits((size_t)(highest + 1 + 7) / 8, 0);  // TezUtilsInternal.toByteArray(BitSet) (big-endian byte order)
        for (int p = 0; p <= highest; p++) if (!(idx[3 * p + 1] > 6)) bits[bits.size() - (size_t)p / 8 - 1] |= (uint8_t)(1u << (p % 8));
        pb_bytes(dm, 1, deflate_raw(bits));
      }
    }
    if (!send_empty || output_generated) {
      pb_bytes(dm, 2, host);
      pb_int(dm, 3, port);
      pb_bytes(dm, 4, path_component);
    }
    pb_int(dm, 5, 0);  // run_duration
    if (!final_merge) { pb_int(dm, 8, last ? 1 : 0); pb_int(dm, 9, spill_id); }
    if (unordered && P == 1) pb_int(dm, 10, counters["OUTPUT_RECORDS"]);   // num_record (generateDMEvent)
    Event e;
    e.type = TEZRT_EVENT_COMPOSITE_DATA_MOVEMENT;
    e.payload = dm;
    e.source_index_start = 0;
    e.count = P;
    events.push_back(e);
  }

  void close() {
    RT_CHECK(started, TEZGPU_E_STATE, "close() before start()");
    if (closed) return;
    sorter->flush();
    if (final_merge) generate_events(sorter->final_idx, uid, -1, true);
    else
      for (int s = 0; s < sorter->num_spills; s++)
        generate_events(sorter->spill_index[s], uid + "_" + std::to_string(s), s, s == sorter->num_spills - 1);
    closed = true;
  }
};

// ================================================================================================ input side
struct Input {
  Configuration conf;
  std::string work_dir, uid;
  int N, device;
  int64_t task_memory, requested = 0;
  bool initialized = false, started = false, ready = false;
  std::map<std::string, int64_t> counters;
  std::vector<std::vector<uint8_t>> seg_bytes;
  std::vector<int64_t> seg_raw;   // rawLength of each fetched segment (index / ShuffleHeader)
  // per source: spill ids seen and the id carried by the event with last_event_flag (pipelined shuffle; the reference's
  // ShuffleScheduler tracks the same per input identifier: eventsProcessed / finalEventId, OG/ShuffleScheduler.java:540-600); spill id -1 = the single
  // event of a producer that ran its final merge
  struct SourceState { std::vector<int> spills; int last_id = -2; bool complete = false; };
  std::vector<SourceState> delivered;
  int num_delivered = 0;
  tezgpu_merger *merger = nullptr;
  int cmp = 0;
  int codec = TEZGPU_CODEC_NONE;
  uint64_t budget = 0;   // merge_budget
  MergeInfo info;        // one-step merges; a bounded one is asked when merge_info() is called, as it steps while read
  uint64_t decode_peak = 0;
  // iterator state (RL/common/ValuesIterator.java:91-201)
  std::vector<uint8_t> batch, next_batch_buf;
  std::vector<tezgpu_kv_index> idx;
  uint32_t bn = 0, bi = 0;
  std::vector<uint8_t> cur_key;
  bool have_rec = false, eos = false, in_group = false, first_of_group = false;

  Input(const char *c, const char *wd, const char *u, int64_t mem, int n, int dev)
      : conf(c), work_dir(wd ? wd : "."), uid(u ? u : "attempt"), N(n), device(dev), task_memory(mem), delivered(n) {}
  ~Input() { if (merger) tezgpu_merge_close(merger); }

  // UnorderedKVInput (RL/input/UnorderedKVInput.java): every delivered input read in turn, no merge
  // (UnorderedKVReader :119-230).  Order: delivery order, the spills of one source in spill-id order.
  bool unordered = false;
  std::vector<std::pair<int, int>> seg_order;   // (delivery rank of the source, spill id) of every fetched segment
  std::vector<int> src_rank;
  int next_rank = 0;

  void initialize() {
    // OrderedGroupedKVInput.initialize (:100-125): Shuffle memory = shuffle.fetch.buffer.percent of the task memory
    double pct = conf.getFloat("tez.runtime.shuffle.fetch.buffer.percent", 0.9);
    requested = (int64_t)(pct * (double)task_memory);
    cmp = unordered ? TEZGPU_CMP_BYTES : comparator_for(conf);
    codec = codec_for(conf);
    budget = merge_budget(conf);
    initialized = true;
  }
  void start() {
    RT_CHECK(initialized, TEZGPU_E_STATE, "start() before initialize()");
    started = true;
    if (N == 0) ready = true;
  }
  void add_local(int src, const char *file_out, const char *index_file, int partition, bool empty, int spill_id, bool last_event) {
    RT_CHECK(started, TEZGPU_E_STATE, "handleEvents() before start()");
    RT_CHECK(src >= 0 && src < N, TEZGPU_E_INVALID, "source index out of range");
    RT_CHECK(spill_id >= -1, TEZGPU_E_INVALID, "bad spill id");
    SourceState &ss = delivered[src];
    if (spill_id < 0) {
      if (ss.complete) return;  // duplicate event for an already fetched input
      RT_CHECK(ss.spills.empty(), TEZGPU_E_STATE, "final-merge event for a source that already delivered spill events");
      ss.complete = true;
    } else {
      RT_CHECK(!(ss.complete && ss.last_id == -2), TEZGPU_E_STATE, "spill event for a source that already delivered its final output");
      for (int id : ss.spills) if (id == spill_id) return;  // duplicate spill event
      RT_CHECK(ss.last_id == -2 || spill_id < ss.last_id, TEZGPU_E_INVALID, "spill id beyond the one flagged as last");
      ss.spills.push_back(spill_id);
      if (last_event) {
        for (int id : ss.spills) RT_CHECK(id <= spill_id, TEZGPU_E_INVALID, "spill id beyond the one flagged as last");
        ss.last_id = spill_id;
      }
      ss.complete = ss.last_id >= 0 && (int)ss.spills.size() == ss.last_id + 1;
    }
    if (ss.complete) num_delivered++;
    if (src_rank.empty()) src_rank.assign((size_t)N, -1);
    if (src_rank[src] < 0) src_rank[src] = next_rank++;   // a source's place: its first event, empty or not
    if (empty) { counters["NUM_SKIPPED_INPUTS"]++; return; }
    // TezSpillRecord(indexFile): P x 3 big-endian longs + checksum (SORT/TezSpillRecord.java:76-109)
    std::vector<uint8_t> ib = read_file(index_file);
    RT_CHECK(ib.size() >= 8 && (ib.size() - 8) % 24 == 0, TEZGPU_E_FORMAT, std::string("bad index file ") + index_file);
    int P = (int)((ib.size() - 8) / 24);
    RT_CHECK(partition >= 0 && partition < P, TEZGPU_E_INVALID, "partition outside the producer's index");
    uLong crc = crc32(0L, Z_NULL, 0);
    crc = crc32(crc, ib.data(), (uInt)(ib.size() - 8));
    uint64_t stored = 0;
    for (int b = 0; b < 8; b++) stored = (stored << 8) | ib[ib.size() - 8 + b];
    RT_CHECK(stored == (uint64_t)crc, TEZGPU_E_FORMAT, std::string("Checksum error reading spill index: ") + index_file);
    auto be64 = [&](size_t o) { uint64_t v = 0; for (int b = 0; b < 8; b++) v = (v << 8) | ib[o + b]; return (int64_t)v; };
    int64_t start = be64((size_t)partition * 24), raw = be64((size_t)partition * 24 + 8), part = be64((size_t)partition * 24 + 16);
    if (!(raw > 6)) { counters["NUM_SKIPPED_INPUTS"]++; return; }  // !hasData
    seg_bytes.push_back(read_file(file_out, (uint64_t)start, part));
    seg_raw.push_back(raw);
    seg_order.push_back({src_rank[src], spill_id});
    counters["NUM_SHUFFLED_INPUTS"]++;
    counters["SHUFFLE_BYTES"] += part;
    counters["SHUFFLE_BYTES_DECOMPRESSED"] += raw;
    counters["SHUFFLE_BYTES_DISK_DIRECT"] += part;
  }
  void wait_ready() {
    RT_CHECK(started, TEZGPU_E_STATE, "waitForInputReady() before start()");
    RT_CHECK(num_delivered == N, TEZGPU_E_STATE,
             "waitForInputReady(): " + std::to_string(N - num_delivered) + " physical inputs have not been delivered");
    if (ready) return;
    tezgpu_conf gc;
    memset(&gc, 0, sizeof(gc));
    gc.abi_version = TEZGPU_ABI_VERSION;
    gc.device = device;
    gc.num_partitions = 1;
    gc.comparator = cmp;
    gc.partitioner = TEZGPU_PART_GIVEN;
    std::vector<tezgpu_segment> segs(seg_bytes.size());
    for (size_t i = 0; i < seg_bytes.size(); i++) {
      segs[i].data = seg_bytes[i].data();
      segs[i].len = seg_bytes[i].size();
      segs[i].flags = TEZGPU_SEG_HAS_HEADER;
      segs[i].partition = 0;
    }
    if (unordered) {
      std::vector<size_t> ord(segs.size());
      for (size_t i = 0; i < ord.size(); i++) ord[i] = i;
      std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return seg_order[a] < seg_order[b]; });
      std::vector<tezgpu_segment> os(segs.size());
      std::vector<int64_t> oraw(segs.size());
      for (size_t i = 0; i < ord.size(); i++) { os[i] = segs[ord[i]]; oraw[i] = seg_raw[ord[i]]; }
      gpu_check(tezgpu_concat_open(&gc, os.data(), oraw.data(), (uint32_t)os.size(), codec, &merger));
    } else if (budget) {
      open_bounded(gc, segs);
      counters["MERGED_MAP_OUTPUTS"] += (int64_t)segs.size();
    } else {
      // MergeManager.finalMerge -> TezMerger.merge; compressed segments are inflated with their index rawLength
      gpu_check(tezgpu_merge_open_codec(&gc, segs.data(), seg_raw.data(), (uint32_t)segs.size(), codec, &merger));
      counters["MERGED_MAP_OUTPUTS"] += (int64_t)segs.size();
    }
    info.steps = 1;
    // a merge in several steps reads the fetched segments until it is closed
    if (!budget || unordered) seg_bytes.clear();
    seg_raw.clear();
    seg_order.clear();
    batch.resize(8u << 20);
    idx.resize(1u << 16);
    ready = true;
  }
  // MergeManager.finalMerge under the budget: the compressed segments are decoded on the device first (their images
  // replace their fetched bytes), then every segment is merged as an uncompressed host segment in key-range steps
  void open_bounded(const tezgpu_conf &gc, std::vector<tezgpu_segment> &segs) {
    std::vector<std::vector<uint8_t>> img(segs.size());
    std::vector<uint8_t *> out(segs.size(), nullptr);
    bool any = false;
    for (size_t i = 0; codec && i < segs.size(); i++)
      if (seg_bytes[i].size() >= 10 && memcmp(seg_bytes[i].data(), "TIF\x01", 4) == 0) {
        img[i].resize((size_t)seg_raw[i] + 4);
        out[i] = img[i].data();
        any = true;
      }
    if (any) {
      gpu_check(tezgpu_decode_segments(&gc, segs.data(), seg_raw.data(), (uint32_t)segs.size(), codec, budget, out.data(), &decode_peak));
      for (size_t i = 0; i < segs.size(); i++) {
        if (!out[i]) continue;
        seg_bytes[i].swap(img[i]);
        std::vector<uint8_t>().swap(img[i]);
        segs[i].data = seg_bytes[i].data();
        segs[i].len = seg_bytes[i].size();
        segs[i].flags |= TEZGPU_SEG_VERIFIED;   // the decode wrote the image's checksum from its bytes
      }
    }
    gpu_check(tezgpu_merge_open_bounded(&gc, segs.data(), nullptr, (uint32_t)segs.size(), TEZGPU_CODEC_NONE, budget, &merger));
  }
  MergeInfo merge_info() const {
    if (!merger || !budget || unordered) return info;
    MergeInfo mi;
    gpu_check(tezgpu_merge_bounded_info(merger, &mi.steps, &mi.peak, &mi.h2d));
    mi.peak = std::max(mi.peak, decode_peak);
    return mi;
  }
  bool fetch() {  // next record of the merged stream into (idx[bi])
    if (eos) return false;
    if (bi + 1 < bn) { bi++; return true; }
    uint32_t n = 0;
    int32_t rc = tezgpu_merge_next_batch(merger, batch.data(), batch.size(), idx.data(), (uint32_t)idx.size(), &n);
    if (rc == TEZGPU_E_NOMEM && n == 0 && (uint64_t)idx[0].key_len + idx[0].val_len > batch.size()) {
      // a record larger than the batch buffer: the stream has not moved, grow to fit it and ask again
      batch.resize((size_t)idx[0].key_len + idx[0].val_len);
      rc = tezgpu_merge_next_batch(merger, batch.data(), batch.size(), idx.data(), (uint32_t)idx.size(), &n);
    }
    gpu_check(rc);
    if (n == 0) { eos = true; return false; }
    bn = n;
    bi = 0;
    return true;
  }
  // KeyValuesReader.next(): ValuesIterator.moveToNext (:91-105) -- skip what is left of the current group
  bool next(const uint8_t **key, uint32_t *klen) {
    RT_CHECK(ready, TEZGPU_E_STATE, "getReader() before waitForInputReady()");
    if (!merger) return false;
    if (in_group) { const uint8_t *v; uint32_t vl; while (next_value(&v, &vl)) {} }
    if (!have_rec) { if (!fetch()) return false; have_rec = true; }
    const tezgpu_kv_index &e = idx[bi];
    cur_key.assign(batch.data() + e.key_off, batch.data() + e.key_off + e.key_len);
    in_group = true;
    first_of_group = true;
    counters["REDUCE_INPUT_GROUPS"]++;
    *key = cur_key.data();
    *klen = (uint32_t)cur_key.size();
    return true;
  }
  // KeyValueReader.next() of UnorderedKVInput: every record in turn; the first call opens the concatenation
  bool next_kv(const uint8_t **key, uint32_t *klen, const uint8_t **val, uint32_t *vlen) {
    RT_CHECK(unordered, TEZGPU_E_STATE, "next_kv() is the reader of an unordered input");
    wait_ready();
    if (!merger || !fetch()) return false;
    const tezgpu_kv_index &e = idx[bi];
    *key = batch.data() + e.key_off;
    *klen = e.key_len;
    *val = batch.data() + e.val_off;
    *vlen = e.val_len;
    counters["INPUT_RECORDS_PROCESSED"]++;
    return true;
  }
  bool next_value(const uint8_t **val, uint32_t *vlen) {
    if (!in_group) return false;
    if (!first_of_group) {
      // readNextKey (:177-201): same group when the merger says isSameKey(), else compare the raw key bytes
      // (equal keys of the supported classes have equal serialized bytes)
      if (!fetch()) { have_rec = false; in_group = false; return false; }
      const tezgpu_kv_index &e = idx[bi];
      bool same = e.same_key || (e.key_len == cur_key.size() && memcmp(batch.data() + e.key_off, cur_key.data(), e.key_len) == 0);
      if (!same) { in_group = false; have_rec = true; return false; }
    }
    first_of_group = false;
    const tezgpu_kv_index &e = idx[bi];
    *val = batch.data() + e.val_off;
    *vlen = e.val_len;
    counters["REDUCE_INPUT_RECORDS"]++;
    return true;
  }
};

}  // namespace tezrt

using namespace tezrt;

struct tezrt_output { Output o; tezrt_output(const char *c, const char *wd, const char *u, const char *dv, const char *h, int pt, int64_t mem, int p, int dev) : o(c, wd, u, dv, h, pt, mem, p, dev) {} };
struct tezrt_input { Input i; tezrt_input(const char *c, const char *wd, const char *u, int64_t mem, int n, int dev) : i(c, wd, u, mem, n, dev) {} };

#define RT_BEGIN try {
#define RT_END } catch (const Err &e) { g_err = e.what(); return e.code; } catch (const std::exception &e) { g_err = e.what(); return TEZGPU_E_INVALID; } return 0;

extern "C" {
const char *tezrt_last_error(void) { return g_err.c_str(); }

int32_t tezrt_output_create(const char *conf, const char *work_dir, const char *unique_id, const char *dest_vertex, const char *host,
                            int32_t port, int64_t task_memory, int32_t P, int32_t device, tezrt_output **out) {
  RT_BEGIN
  RT_CHECK(out && P >= 1, TEZGPU_E_INVALID, "bad arguments");
  *out = new tezrt_output(conf, work_dir, unique_id, dest_vertex, host, port, task_memory, P, device);
  RT_END
}
int32_t tezrt_output_create_unordered(const char *conf, const char *work_dir, const char *unique_id, const char *dest_vertex,
                                      const char *host, int32_t port, int64_t task_memory, int32_t P, int32_t partitioned,
                                      int32_t device, tezrt_output **out) {
  RT_BEGIN
  RT_CHECK(out && P >= 1, TEZGPU_E_INVALID, "bad arguments");
  // UnorderedKVOutput writes one partition whatever the number of physical outputs (RL/output/UnorderedKVOutput.java:107)
  *out = new tezrt_output(conf, work_dir, unique_id, dest_vertex, host, port, task_memory, partitioned ? P : 1, device);
  (*out)->o.unordered = true;
  if (!partitioned) (*out)->o.total_order = false;   // UnorderedKVOutput has no partitioner
  RT_END
}
int32_t tezrt_output_initialize(tezrt_output *o, int64_t *requested) { RT_BEGIN o->o.initialize(); if (requested) *requested = o->o.requested; RT_END }
int32_t tezrt_output_memory_assigned(tezrt_output *o, int64_t granted) { RT_BEGIN o->o.granted = granted; RT_END }
int32_t tezrt_output_start(tezrt_output *o) { RT_BEGIN o->o.start(); RT_END }
int32_t tezrt_output_write(tezrt_output *o, const uint8_t *k, uint32_t kl, const uint8_t *v, uint32_t vl, int32_t partition) {
  RT_BEGIN o->o.write(k, kl, v, vl, partition); RT_END
}
int32_t tezrt_output_close(tezrt_output *o, int32_t *n) { RT_BEGIN o->o.close(); if (n) *n = (int32_t)o->o.events.size(); RT_END }
int32_t tezrt_output_event(tezrt_output *o, int32_t i, int32_t *type, const uint8_t **payload, uint64_t *len, int32_t *start, int32_t *count) {
  RT_BEGIN
  RT_CHECK(i >= 0 && i < (int)o->o.events.size(), TEZGPU_E_INVALID, "event index");
  const Event &e = o->o.events[i];
  if (type) *type = e.type;
  if (payload) *payload = (const uint8_t *)e.payload.data();
  if (len) *len = e.payload.size();
  if (start) *start = e.source_index_start;
  if (count) *count = e.count;
  RT_END
}
int64_t tezrt_output_counter(tezrt_output *o, const char *name) { auto it = o->o.counters.find(name); return it == o->o.counters.end() ? 0 : it->second; }
int32_t tezrt_output_num_spills(tezrt_output *o) { return o->o.sorter ? o->o.sorter->num_spills : 0; }
static void merge_info(const MergeInfo &mi, int32_t *steps, uint64_t *peak, uint64_t *h2d) {
  if (steps) *steps = mi.steps;
  if (peak) *peak = mi.peak;
  if (h2d) *h2d = mi.h2d;
}
int32_t tezrt_output_merge_info(tezrt_output *o, int32_t *steps, uint64_t *peak_device_bytes, uint64_t *h2d_bytes) {
  RT_BEGIN
  RT_CHECK(o, TEZGPU_E_INVALID, "null handle");
  merge_info(o->o.sorter ? o->o.sorter->info : MergeInfo(), steps, peak_device_bytes, h2d_bytes);
  RT_END
}
const char *tezrt_output_file(tezrt_output *o) { return o->o.sorter ? o->o.sorter->final_out.c_str() : ""; }
const char *tezrt_output_index_file(tezrt_output *o) { return o->o.sorter ? o->o.sorter->final_index.c_str() : ""; }
int32_t tezrt_output_destroy(tezrt_output *o) { delete o; return 0; }

int32_t tezrt_input_create(const char *conf, const char *work_dir, const char *unique_id, int64_t task_memory, int32_t n, int32_t device,
                           tezrt_input **out) {
  RT_BEGIN
  RT_CHECK(out && n >= 0, TEZGPU_E_INVALID, "bad arguments");
  *out = new tezrt_input(conf, work_dir, unique_id, task_memory, n, device);
  RT_END
}
int32_t tezrt_input_create_unordered(const char *conf, const char *work_dir, const char *unique_id, int64_t task_memory, int32_t n,
                                     int32_t device, tezrt_input **out) {
  RT_BEGIN
  RT_CHECK(out && n >= 0, TEZGPU_E_INVALID, "bad arguments");
  *out = new tezrt_input(conf, work_dir, unique_id, task_memory, n, device);
  (*out)->i.unordered = true;
  RT_END
}
int32_t tezrt_input_next_kv(tezrt_input *in, const uint8_t **key, uint32_t *klen, const uint8_t **val, uint32_t *vlen) {
  try { return in->i.next_kv(key, klen, val, vlen) ? 1 : 0; } catch (const Err &e) { g_err = e.what(); return e.code; }
}
int32_t tezrt_input_initialize(tezrt_input *in, int64_t *requested) { RT_BEGIN in->i.initialize(); if (requested) *requested = in->i.requested; RT_END }
int32_t tezrt_input_start(tezrt_input *in) { RT_BEGIN in->i.start(); RT_END }
int32_t tezrt_input_add_local_output(tezrt_input *in, int32_t src, const char *file_out, const char *index_file, int32_t partition, int32_t empty) {
  RT_BEGIN in->i.add_local(src, file_out, index_file, partition, empty != 0, -1, true); RT_END
}
int32_t tezrt_input_add_local_spill(tezrt_input *in, int32_t src, const char *file_out, const char *index_file, int32_t partition, int32_t empty,
                                    int32_t spill_id, int32_t last_event) {
  RT_BEGIN in->i.add_local(src, file_out, index_file, partition, empty != 0, spill_id, last_event != 0); RT_END
}
int32_t tezrt_input_wait_ready(tezrt_input *in) { RT_BEGIN in->i.wait_ready(); RT_END }
int32_t tezrt_input_next(tezrt_input *in, const uint8_t **key, uint32_t *klen) {
  try { return in->i.next(key, klen) ? 1 : 0; } catch (const Err &e) { g_err = e.what(); return e.code; }
}
int32_t tezrt_input_next_value(tezrt_input *in, const uint8_t **val, uint32_t *vlen) {
  try { return in->i.next_value(val, vlen) ? 1 : 0; } catch (const Err &e) { g_err = e.what(); return e.code; }
}
int32_t tezrt_input_merge_info(tezrt_input *in, int32_t *steps, uint64_t *peak_device_bytes, uint64_t *h2d_bytes) {
  RT_BEGIN
  RT_CHECK(in, TEZGPU_E_INVALID, "null handle");
  merge_info(in->i.merge_info(), steps, peak_device_bytes, h2d_bytes);
  RT_END
}
int64_t tezrt_input_counter(tezrt_input *in, const char *name) { auto it = in->i.counters.find(name); return it == in->i.counters.end() ? 0 : it->second; }
int32_t tezrt_input_destroy(tezrt_input *in) { delete in; return 0; }
}

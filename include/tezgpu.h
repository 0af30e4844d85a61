/*
 * tezgpu.h -- C ABI of libtezgpu.so: H100-native (sm_90a) replacement of the Tez shuffle sort/merge hot path.
 *
 * This is the drop-in boundary (SURVEY.md 8b).  Plain pointers and sizes only -- no torch / C++ types.
 * Each entry point names the reference interface it replaces.  Paths are relative to
 * /root/reference/tez-runtime-library/src/main/java/org/apache/tez/runtime/library/ (RL/), SORT/ = RL/common/sort/impl/.
 *
 * Conventions
 *   - every function returns int32: 0 = ok, <0 = TEZGPU_E_*; tezgpu_last_error() gives the message of the last
 *     failure on the calling thread (the JNI stub turns it into java.io.IOException, like every failure of the
 *     reference path: SORT/PipelinedSorter.java:400-413).
 *   - no exceptions cross the boundary; handles are opaque; one producer thread per handle; handles independent.
 *   - the caller owns every buffer it passes, for the duration of the call only; the library owns device memory.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with TEZGPU_E_CUDA.
 *   - every call runs on its handle's conf.device (or its device argument) and returns with the calling thread's
 *     CUDA context as it found it; a thread that had none stays on the call's device (no context is created elsewhere).
 *   - a device ordinal outside [0, tezgpu_device_count()) fails with TEZGPU_E_INVALID ("bad device ordinal").
 */
#ifndef TEZGPU_H
#define TEZGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TEZGPU_ABI_VERSION 1

/* error codes */
#define TEZGPU_OK 0
#define TEZGPU_E_INVALID (-1)     /* bad argument / illegal partition ("Illegal partition for ...", PipelinedSorter.java:410-413) */
#define TEZGPU_E_CUDA (-2)        /* CUDA runtime failure (incl. no device) */
#define TEZGPU_E_NOMEM (-3)       /* device or host allocation failed -> task attempt fails, no CPU fallback */
#define TEZGPU_E_IO (-4)          /* file write failed */
#define TEZGPU_E_FORMAT (-5)      /* malformed IFile segment / checksum mismatch (IFileInputStream.java:235-289) */
#define TEZGPU_E_UNSUPPORTED (-6) /* comparator / partitioner / codec outside the device-supported closed set */
#define TEZGPU_E_STATE (-7)       /* call sequence violation (e.g. collect after flush) */

/* key comparator = RawComparator selected by ConfigUtils.getIntermediateOutputKeyComparator (RL/common/ConfigUtils.java:92-100) */
#define TEZGPU_CMP_BYTES 0          /* TezBytesComparator / raw bytes (RL/common/comparator/TezBytesComparator.java:37-41) */
#define TEZGPU_CMP_TEXT 1           /* hadoop Text.Comparator: skip the vint length prefix, then unsigned bytes */
#define TEZGPU_CMP_BYTESWRITABLE 2  /* hadoop BytesWritable.Comparator: skip the 4-byte length, then unsigned bytes */
#define TEZGPU_CMP_INT 3            /* IntWritable.Comparator: 4-byte big-endian signed */
#define TEZGPU_CMP_LONG 4           /* LongWritable.Comparator: 8-byte big-endian signed */

/* partitioner (RL/partitioner/HashPartitioner.java:33-35) */
#define TEZGPU_PART_GIVEN 0         /* caller computed Partitioner.getPartition in Java and passes the ids */
#define TEZGPU_PART_HASH 1          /* device computes (key.hashCode() & MAX_VALUE) % P for the comparator's key class */
#define TEZGPU_PART_TOTAL_ORDER 2   /* Hadoop TotalOrderPartitioner: the device computes the number of split points <= key
                                       (tezgpu_sorter_set_split_points) */

/* RLE policy of IFile.Writer (SORT/IFile.java:541-544; decision SORT/PipelinedSorter.java:1436-1438) */
#define TEZGPU_RLE_AUTO (-1)        /* on iff (#adjacent equal keys in sorted order) > 0.1 * records -- see DESIGN.md "RLE decision" */
#define TEZGPU_RLE_OFF 0
#define TEZGPU_RLE_ON 1

/* sorter_impl = 2: the writer behind UnorderedPartitionedKVOutput (RL/common/writers/UnorderedPartitionedKVWriter.java):
 * records are only partitioned; every partition's segment holds its records NEWEST FIRST (the per-partition chain of
 * :459-472 walked by writePartition :688-703 -- the order the reference writes when everything fits one buffer), IFile
 * without run-length encoding (:1092), no bytes and an all-zero index entry for a partition without records (mergeAll
 * :1058-1144).  The comparator is ignored.  With several buffers / spills the reference's order inside a partition
 * depends on buffer arithmetic and thread timing: parity is then the identical index + the per-partition multiset. */
#define TEZGPU_SORTER_UNORDERED 2

typedef struct tezgpu_conf {
  int32_t abi_version;                  /* TEZGPU_ABI_VERSION */
  int32_t device;                       /* CUDA ordinal */
  int32_t num_partitions;               /* numPhysicalOutputs (RL/output/OrderedPartitionedKVOutput.java:91-110) */
  int32_t comparator;                   /* TEZGPU_CMP_* */
  int32_t partitioner;                  /* TEZGPU_PART_* */
  int32_t rle_policy;                   /* TEZGPU_RLE_* */
  int32_t send_empty_partition_details; /* tez.runtime.empty.partitions.info-via-events.enabled (default 1) */
  int32_t sorter_impl;                  /* 0 = PipelinedSorter (default), 1 = DefaultSorter ("LEGACY"): only changes the AUTO RLE rule,
                                           2 = TEZGPU_SORTER_UNORDERED: UnorderedPartitionedKVWriter (partition only, no key order) */
  uint32_t fixed_key_len;               /* >0 with fixed_val_len: records are packed key||value of constant width */
  uint32_t fixed_val_len;
  uint64_t mem_budget_bytes;            /* granted by OutputContext.requestInitialMemory; 0 = no limit.  Enforced on the key+value
                                           bytes collected since the last reset: a collect that would pass it fails with
                                           TEZGPU_E_NOMEM and the caller spills (flush + reset), like PipelinedSorter when its
                                           kvbuffer is full (SORT/PipelinedSorter.java:415-444) */
} tezgpu_conf;

/* counters + per-partition results; mirrors TezSpillRecord / TezIndexRecord and the ExternalSorter counters
 * (SORT/TezSpillRecord.java:48-52, SORT/ExternalSorter.java:141-167) */
typedef struct tezgpu_stats {
  int64_t output_records;               /* OUTPUT_RECORDS */
  int64_t output_bytes;                 /* OUTPUT_BYTES: sum(keyLen+valLen) */
  int64_t output_bytes_with_overhead;   /* OUTPUT_BYTES_WITH_OVERHEAD: sum(rawLength) */
  int64_t output_bytes_physical;        /* OUTPUT_BYTES_PHYSICAL: file.out length */
  int64_t spilled_records;              /* SPILLED_RECORDS */
  int64_t file_out_bytes;               /* bytes produced for file.out */
  int32_t num_spills;                   /* always 1: HBM is the sort buffer (PipelinedSorter.flush numSpills==1 branch :730-756) */
  int32_t rle_used;
  int64_t adjacent_equal_keys;
  int64_t tie_records;                  /* records that needed key-suffix refinement after the prefix radix sort */
  float ms_stage, ms_sort, ms_ties, ms_emit, ms_total; /* device times of the last flush (CUDA events) */
  int32_t kernel_launches;              /* kernels launched by the last flush / merge */
  float ms_emit_kernel;                 /* device time of the gather+emit kernel alone (CUDA events around its launch) */
} tezgpu_stats;

typedef struct tezgpu_sorter tezgpu_sorter;
typedef struct tezgpu_merger tezgpu_merger;

/* Combiner: ExternalSorter.combiner = MRCombiner running one of the sum reducers below, applied on the device between
 * the sort and the IFile writer (SORT/PipelinedSorter.java:601-609,815-820; SORT/dflt/DefaultSorter.java:915-945).
 * A group is a maximal run of adjacent records of one partition whose keys compare equal (ValuesIterator); it is
 * written as one record: the key bytes, then the big-endian sum of the group's values (Java arithmetic: wraps).  Keys
 * are then unique per partition, so no REPEAT_KEY marker is written; stats.rle_used / adjacent_equal_keys still report
 * the decision made on the uncombined stream.  A value that is not 4 (INT) or 8 (LONG) bytes wide fails the flush /
 * write with TEZGPU_E_INVALID.  With a combiner, stats.output_records counts the records that entered the combine
 * (COMBINE_INPUT_RECORDS) and stats.spilled_records those written (COMBINE_OUTPUT_RECORDS); ms_total includes it. */
#define TEZGPU_COMBINE_NONE 0
#define TEZGPU_COMBINE_SUM_INT 1    /* IntSumReducer over IntWritable values */
#define TEZGPU_COMBINE_SUM_LONG 2   /* LongSumReducer over LongWritable values */

/* Codec of the IFile segments (tez.runtime.compress / tez.runtime.compress.codec, SORT/IFile.java:351-420): with
 * DEFAULT (org.apache.hadoop.io.compress.DefaultCodec, RL/common/ConfigUtils.java:44-66) a segment is 'T','I','F',1, one
 * zlib stream (RFC 1950) of the uncompressed body, and the CRC-32 of the compressed bytes; its index triple keeps the
 * uncompressed rawLength and has the compressed segment length as partLength.  With LZ4
 * (org.apache.hadoop.io.compress.Lz4Codec) the stream between header and CRC is Hadoop's BlockCompressorStream
 * framing: blocks of a big-endian int32 raw length and one or more chunks, each a big-endian int32 compressed length
 * and one raw LZ4 block.  The device writes blocks of TEZGPU_LZ4_BLOCK_BYTES raw bytes (the last one shorter), one
 * chunk each, no chunk longer than TEZGPU_LZ4_CHUNK_BOUND; a Java reader needs io.compression.codec.lz4.buffersize of
 * at least that.  The device reader takes chunks that decode to at most 262,144 bytes (the default buffersize).
 * With ZSTD (org.apache.hadoop.io.compress.ZStandardCodec) the stream is one or more Zstandard frames (RFC 8878).  The
 * device writes one frame per TEZGPU_ZSTD_BLOCK_BYTES raw bytes (the last one shorter): Single_Segment with
 * Frame_Content_Size, one block, no checksum, at most TEZGPU_ZSTD_FRAME_BOUND bytes.  The device reader takes what
 * libzstd's default streaming decoder takes (windows up to 2^27), except dictionaries.
 * With SNAPPY (org.apache.hadoop.io.compress.SnappyCodec) the stream has Lz4Codec's block framing with one raw Snappy
 * block per chunk (a varint preamble giving the chunk's raw length, then literal and copy elements).  The device writes
 * blocks of TEZGPU_SNAPPY_BLOCK_BYTES raw bytes (the last one shorter), one chunk each, no chunk longer than
 * TEZGPU_SNAPPY_CHUNK_BOUND; a Java reader needs io.compression.codec.snappy.buffersize of at least that (the default
 * is 262,144).  The device reader takes chunks of at most 262,144 bytes that decode to at most 262,144 bytes each.
 * Other codecs are not on the device. */
#define TEZGPU_CODEC_NONE 0
#define TEZGPU_CODEC_DEFAULT 1
#define TEZGPU_CODEC_LZ4 2
#define TEZGPU_LZ4_BLOCK_BYTES 65024
#define TEZGPU_LZ4_CHUNK_BOUND (TEZGPU_LZ4_BLOCK_BYTES + TEZGPU_LZ4_BLOCK_BYTES / 255 + 16) /* LZ4_compressBound */
#define TEZGPU_CODEC_ZSTD 3
#define TEZGPU_ZSTD_BLOCK_BYTES 65024
#define TEZGPU_ZSTD_FRAME_BOUND (TEZGPU_ZSTD_BLOCK_BYTES + 10) /* a raw frame: magic, descriptor, 2-byte size, block header */
#define TEZGPU_CODEC_SNAPPY 4
#define TEZGPU_SNAPPY_BLOCK_BYTES 65024
#define TEZGPU_SNAPPY_CHUNK_BOUND (3 + 3 + TEZGPU_SNAPPY_BLOCK_BYTES) /* all literal: 3 preamble, 3 literal-tag bytes */

const char *tezgpu_last_error(void);
int32_t tezgpu_abi_version(void);
/* number of visible CUDA devices (0 when none; never falls back to CPU) */
int32_t tezgpu_device_count(void);

/* ------------------------------------------------------------------------------------------------------------------
 * Sorter: replaces PipelinedSorter / DefaultSorter behind ExternalSorter (SORT/ExternalSorter.java:74-92,281-288)
 * ---------------------------------------------------------------------------------------------------------------- */

/* replaces `new PipelinedSorter(outputContext, conf, numOutputs, initialMemory)` (RL/output/OrderedPartitionedKVOutput.java:116-160) */
int32_t tezgpu_sorter_create(const tezgpu_conf *conf, tezgpu_sorter **out);

/* replaces PipelinedSorter.write/collect (SORT/PipelinedSorter.java:387-466), batched: one JNI crossing per n records.
 * kv holds the serialized records; record i's key is kv[key_off[i] .. val_off[i]) and its value kv[val_off[i] .. +val_len[i])
 * (the {KEYSTART, VALSTART, VALLEN} metadata triple of :459-462).  partition may be NULL when conf.partitioner==HASH.
 * Bytes are copied before the call returns (the caller reuses its buffers, WordCount.java:74-75,95-97). */
int32_t tezgpu_sorter_collect_batch(tezgpu_sorter *h, const uint8_t *kv, uint64_t kv_bytes, const uint32_t *key_off,
                                    const uint32_t *val_off, const uint32_t *val_len, const int32_t *partition,
                                    uint32_t n);

/* fixed-width fast path of the above: n records of (fixed_key_len + fixed_val_len) bytes packed back to back */
int32_t tezgpu_sorter_collect_fixed(tezgpu_sorter *h, const uint8_t *kv, const int32_t *partition, uint64_t n);

/* replaces PipelinedSorter.flush()+spill() (SORT/PipelinedSorter.java:558-647,664-859): sorts by (partition, key),
 * writes file.out (concatenated IFile segments, mode 0640) and file.out.index (TezSpillRecord), fills stats and
 * index[3*P] = (startOffset, rawLength, partLength) per partition.  index may be NULL. */
int32_t tezgpu_sorter_flush(tezgpu_sorter *h, const char *out_path, const char *index_path, int64_t *index,
                            tezgpu_stats *stats);

/* same, into caller memory instead of files (tests / in-process consumers). out_cap >= tezgpu_sorter_output_bound(h).
 * index_out (may be NULL) receives the P*24+8 bytes of file.out.index. */
int32_t tezgpu_sorter_flush_to_memory(tezgpu_sorter *h, uint8_t *out, uint64_t out_cap, uint64_t *out_len,
                                      uint8_t *index_out, int64_t *index, tezgpu_stats *stats);
uint64_t tezgpu_sorter_output_bound(const tezgpu_sorter *h);

/* replaces ExternalSorter.close() (SORT/ExternalSorter.java:281-288) */
int32_t tezgpu_sorter_destroy(tezgpu_sorter *h);
/* forgets the collected records but keeps every device / pinned allocation, so a container-reused task
 * (tez.am.container.reuse) can run its next output through the same handle */
int32_t tezgpu_sorter_reset(tezgpu_sorter *h);

/* Device-resident variant (records already in HBM; used by the multi-GPU shuffle and by bench.py's kernel-only
 * measurement).  d_kv: n packed fixed-width records on conf.device; d_partition may be 0.  d_out receives file.out
 * bytes (capacity out_cap); index (host, 3*P int64) and stats are filled after an internal stream sync.
 * Without a codec d_out must be 16-byte aligned (the emit stores 16-byte words); a misaligned d_out returns
 * TEZGPU_E_INVALID and writes nothing.
 * Runs on the handle's stream (tezgpu_sorter_stream). */
int32_t tezgpu_sorter_sort_device_fixed(tezgpu_sorter *h, const void *d_kv, const void *d_partition, uint64_t n,
                                        void *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index,
                                        tezgpu_stats *stats);
/* Device-resident variable-length records: replaces PipelinedSorter.write/collect (SORT/PipelinedSorter.java:387-466)
 * and flush()+spill() (:558-647,664-859) in one call, for records a GPU producer already holds in HBM -- nothing crosses
 * PCIe.  Record i's key is d_kv[d_key_off[i] .. d_val_off[i]) and its value d_kv[d_val_off[i] .. + d_val_len[i]), the
 * triple of collect_batch, but with 64-bit offsets (inputs past 4 GiB) and records in any order, with gaps between them.
 * Every array lives on conf.device; d_kv must be 16-byte aligned; d_partition may be 0 (HASH, TOTAL_ORDER).  Nothing is
 * read outside d_kv[0 .. kv_bytes).  A variable-length handle (not fixed), ordered or TEZGPU_SORTER_UNORDERED, with any
 * comparator, partitioner, combiner and codec; nothing may be collected on it (TEZGPU_E_STATE until reset), and the
 * call leaves nothing collected.  Before any key byte is read one kernel checks every record -- key_off <= val_off,
 * val_off - key_off < 2^32, val_off + val_len <= kv_bytes, 0 <= partition < num_partitions -- and fails with
 * TEZGPU_E_INVALID naming the lowest bad record ("record 1234: ..."); d_out is then untouched.  Output as
 * tezgpu_sorter_sort_device_fixed: d_out (16-byte aligned without a codec) receives file.out, index and stats are filled
 * after an internal stream sync; stats.output_bytes = key + value bytes.  out_cap >= tezgpu_sorter_device_output_bound
 * always suffices; a smaller out_cap that the file does not fit fails with TEZGPU_E_NOMEM and writes nothing. */
int32_t tezgpu_sorter_sort_device(tezgpu_sorter *h, const void *d_kv, uint64_t kv_bytes, const uint64_t *d_key_off,
                                  const uint64_t *d_val_off, const uint32_t *d_val_len, const int32_t *d_partition, uint64_t n,
                                  void *d_out, uint64_t out_cap, uint64_t *out_len, int64_t *index, tezgpu_stats *stats);
/* the out_cap tezgpu_sorter_sort_device always fits for n records in a buffer of kv_bytes (the bound of
 * tezgpu_sorter_output_bound for those records, with the handle's codec's worst case), known before the sort so that a
 * caller can size the exchange buffer it sorts into.  0 for a NULL handle. */
uint64_t tezgpu_sorter_device_output_bound(const tezgpu_sorter *h, uint64_t n, uint64_t kv_bytes);
/* cudaStream_t of the handle, as an opaque pointer (so callers can record events on it) */
void *tezgpu_sorter_stream(tezgpu_sorter *h);

/* runs the combiner (TEZGPU_COMBINE_*) on every flush of the handle.  Call before the first collect (or right after a
 * reset); survives reset.  Fails with TEZGPU_E_INVALID on an unordered handle (UnorderedPartitionedKVWriter has no
 * combiner) and on a fixed-width handle whose fixed_val_len is not the combiner's value width. */
int32_t tezgpu_sorter_set_combiner(tezgpu_sorter *h, int32_t combiner);

/* writes every segment through the codec (TEZGPU_CODEC_*) in flush, flush_to_memory and sort_device_fixed, after the
 * combiner when one is set; unordered handles too (UnorderedPartitionedKVWriter writes through the codec).  Call before
 * the first collect (or right after a reset); survives reset.  With a codec, tezgpu_sorter_output_bound includes the
 * worst case (every 32 KiB zlib chunk stored; every LZ4 block all literals; every zstd frame raw), stats.output_bytes_physical / file_out_bytes count compressed bytes,
 * output_bytes_with_overhead is still the sum of rawLength, and ms_total includes the compression (ms_emit does not).
 * TEZGPU_E_UNSUPPORTED for any other codec. */
int32_t tezgpu_sorter_set_codec(tezgpu_sorter *h, int32_t codec);

/* TotalOrderPartitioner (org.apache.hadoop.mapreduce.lib.partition / org.apache.hadoop.mapred.lib): the split points of a
 * TEZGPU_PART_TOTAL_ORDER handle.  Split i is keys[key_off[i] .. + key_len[i]), serialized like the handle's record keys
 * (Text: vint length + bytes; BytesWritable: 4-byte length + bytes; Int / Long: 4 / 8 bytes big-endian).  The partition
 * of a key is the number of split points <= key in the search order `order` (a TEZGPU_CMP_*): TEXT or BYTESWRITABLE for
 * mapreduce.totalorderpartitioner.naturalorder = true on Text / BytesWritable keys (unsigned bytes of the content, even
 * when the sort comparator is BYTES), else the handle's comparator; any other pairing fails with TEZGPU_E_INVALID.  So a
 * key equal to split i goes to partition i + 1.  Fails with TEZGPU_E_INVALID unless n == num_partitions - 1 ("Wrong number of partitions in keyset") and the splits are
 * strictly increasing under the handle's comparator ("Split points are out of order"), or on a handle that is not
 * TOTAL_ORDER; with TEZGPU_E_STATE unless called before the first collect (or right after a reset).  Survives reset.
 * On a TOTAL_ORDER handle with num_partitions > 1, collecting or flushing before the split points are set fails with
 * TEZGPU_E_STATE; a partition array passed to collect_batch, collect_fixed or sort_device_fixed fails with
 * TEZGPU_E_INVALID.  With num_partitions = 1 no split points are needed. */
int32_t tezgpu_sorter_set_split_points(tezgpu_sorter *h, const uint8_t *keys, const uint64_t *key_off, const uint32_t *key_len,
                                       uint32_t n, int32_t order);

/* InputSampler.RandomSampler on the device: a sample of the keys of device-resident records, given as the input triple of
 * tezgpu_sorter_sort_device (key i is d_kv[d_key_off[i] .. d_val_off[i]), the value d_val_len[i] bytes after it), so
 * that a producer passes the same arrays to both calls.  Record i has the global number gid = gid_base + i and the hash
 * h = splitmix64(seed ^ gid).  It is a candidate when h < ceil(freq * 2^64), computed exactly from the double freq in
 * [0, 1]; freq = 1 makes every record one.  Of more than max_samples candidates the max_samples with the smallest
 * (h, gid) are kept.  So the sample is a function of (seed, gid) alone: records divided between calls (ranks) with the
 * right gid_base give, capped again by tezgpu_select_split_points, the sample of the whole set.  This is RandomSampler's
 * contract (a uniform sample of at most numSamples keys at rate freq), not its java.util.Random stream.
 * Output, in gid order, to host buffers: *count <= max_samples keys back to back in keys (key_off[j], key_len[j]), and
 * h[j], gid[j]; key_off, key_len, h and gid hold max_samples entries.  When the keys need more than keys_cap bytes the
 * call fails with TEZGPU_E_NOMEM, *keys_bytes = the bytes they need, *count = 0 and nothing else written.
 * Before any key byte is read every record gets tezgpu_sorter_sort_device's checks (key_off <= val_off,
 * val_off - key_off < 2^32, val_off + val_len <= kv_bytes); a bad record fails the call with TEZGPU_E_INVALID naming the
 * lowest bad index ("record 1234: ...") and nothing written.  TEZGPU_E_INVALID also for a NULL argument, freq outside
 * [0, 1], n >= 2^32 or gid_base + n past 2^64.  Runs on a stream of the library's: work queued on the records must be
 * complete before the call; the call returns when its results are on the host. */
int32_t tezgpu_sample_keys(int32_t device, const void *d_kv, uint64_t kv_bytes, const uint64_t *d_key_off,
                           const uint64_t *d_val_off, const uint32_t *d_val_len, uint64_t n, uint64_t gid_base, uint64_t seed,
                           double freq, uint32_t max_samples, uint8_t *keys, uint64_t keys_cap, uint64_t *key_off,
                           uint32_t *key_len, uint64_t *h, uint64_t *gid, uint32_t *count, uint64_t *keys_bytes);

/* InputSampler.writePartitionFile on the device: the num_partitions - 1 split points of TotalOrderPartitioner from one or
 * more samples of tezgpu_sample_keys, given together as n host entries (keys, key_off, key_len, h, gid; for example the
 * union of every rank's sample).  First the global cap: the max_samples smallest (h, gid) of the union, so the result does
 * not depend on how the records were divided between sample calls.  The kept keys are sorted on the device under
 * `comparator` by the sort pipeline (ties in gid order), and the splits are picked by writePartitionFile's rule with
 * Java's float arithmetic:
 *   float stepSize = len / (float) P; last = -1;
 *   for i in 1 .. P-1: k = Math.round(stepSize * i); while (last >= k && cmp(samples[last], samples[k]) == 0) ++k;
 *                      split i-1 = samples[k]; last = k;
 * `order` is the search order of tezgpu_sorter_set_split_points, with the same pairing rule (TEZGPU_E_INVALID
 * otherwise); the splits do not depend on it.  Output in that call's layout: split i in split_keys[split_off[i] .. +
 * split_len[i]), *split_bytes = the bytes written; chosen (may be NULL) receives each split's index in the sorted sample.
 * Where Java's rule writes a split equal to or below the one before (a skewed sample), the split is returned as Java
 * writes it, and tezgpu_sorter_set_split_points then refuses it ("Split points are out of order").  Where Java would
 * fail the call fails with TEZGPU_E_INVALID: an empty sample with P > 1, or a k past the end of the sample
 * (ArrayIndexOutOfBoundsException); also for a gid that appears twice.  When the splits need more than split_cap bytes,
 * TEZGPU_E_NOMEM with *split_bytes = the bytes they need and nothing else written.  P = 1 returns no splits.
 * TEZGPU_E_UNSUPPORTED for an unknown comparator; TEZGPU_E_INVALID for a NULL argument, max_samples above 2^30 - 1 or
 * n >= 2^32. */
int32_t tezgpu_select_split_points(int32_t device, int32_t comparator, int32_t order, int32_t num_partitions, uint32_t max_samples,
                                   const uint8_t *keys, const uint64_t *key_off, const uint32_t *key_len, const uint64_t *h,
                                   const uint64_t *gid, uint64_t n, uint8_t *split_keys, uint64_t split_cap, uint64_t *split_off,
                                   uint32_t *split_len, uint64_t *split_bytes, uint64_t *chosen);

/* ------------------------------------------------------------------------------------------------------------------
 * Merger: replaces TezMerger.merge(...) -> TezRawKeyValueIterator (SORT/TezMerger.java:717-912,
 * SORT/TezRawKeyValueIterator.java:33-87) as called from OG/MergeManager.java:804-811,899-903,1035-1041,1197-1199
 * and PipelinedSorter.flush :774-836.
 * ---------------------------------------------------------------------------------------------------------------- */
#define TEZGPU_SEG_HAS_HEADER 1u   /* on-disk layout: 'T','I','F',flag + body + crc  (DiskSegment); else body + crc (InMemoryReader) */
#define TEZGPU_SEG_DEVICE 2u       /* data is a device pointer on conf.device */
#define TEZGPU_SEG_VERIFIED 4u     /* the transport already verified this segment's checksum while copying it (as
                                      IFile.Reader.readToMemory does for fetched MEMORY outputs, SORT/IFile.java:764-809,
                                      whose InMemoryReader then never re-checks): tezgpu_fetch_segments_verified */

typedef struct tezgpu_segment {
  const void *data;
  uint64_t len;
  uint32_t flags;
  uint32_t partition;              /* output partition this segment belongs to (0 for a single-partition merge) */
} tezgpu_segment;

/* one merged record: offsets into the batch buffer returned by tezgpu_merge_next_batch */
typedef struct tezgpu_kv_index {
  uint32_t key_off, key_len, val_off, val_len;
  uint32_t same_key;               /* TezRawKeyValueIterator.isSameKey() */
} tezgpu_kv_index;

/* opens the k-way merge over nseg sorted IFile segments: verifies checksums, parses, merges on device */
int32_t tezgpu_merge_open(const tezgpu_conf *conf, const tezgpu_segment *segs, uint32_t nseg, tezgpu_merger **out);
/* runs a new merge through an existing handle, keeping its device allocations (the per-step reduce side of the
 * multi-GPU shuffle; a container-reused task) */
int32_t tezgpu_merge_reopen(tezgpu_merger *m, const tezgpu_segment *segs, uint32_t nseg);
/* tezgpu_merge_open / reopen with a codec (TEZGPU_CODEC_*).  raw_len[i] is segment i's rawLength (spill index or
 * ShuffleHeader uncompressedLength): required for segments whose header flag is 1 (TEZGPU_E_INVALID without it), ignored
 * for the others; raw_len may be NULL when none is compressed.  Compressed and uncompressed segments may be mixed.  A
 * compressed segment's CRC is checked on the compressed bytes (unless TEZGPU_SEG_VERIFIED), its body must inflate to
 * exactly raw_len[i] - 4 bytes (DEFAULT: one or more complete zlib streams; LZ4: blocks of raw length > 0 whose chunks decode to
 * exactly that length, adding up to raw_len[i] - 4, nothing after the last block; ZSTD: frames and skippable frames whose
 * content adds up to raw_len[i] - 4, nothing after the last one), else TEZGPU_E_FORMAT naming the segment.  Every
 * tezgpu_merge_write_* of the handle writes through the same codec (PipelinedSorter's final merge, :774-836).
 * TEZGPU_CODEC_NONE behaves exactly like open / reopen. */
int32_t tezgpu_merge_open_codec(const tezgpu_conf *conf, const tezgpu_segment *segs, const int64_t *raw_len, uint32_t nseg,
                                int32_t codec, tezgpu_merger **out);
int32_t tezgpu_merge_reopen_codec(tezgpu_merger *m, const tezgpu_segment *segs, const int64_t *raw_len, uint32_t nseg);
/* UnorderedPartitionedKVWriter.mergeAll (RL/common/writers/UnorderedPartitionedKVWriter.java:1058-1144) and
 * UnorderedKVReader (RL/common/readers/UnorderedKVReader.java:119-230): records leave in (segment, position) order; no
 * key order, no comparator.  codec and raw_len as for tezgpu_merge_open_codec (compressed and plain segments may be
 * mixed).  Every segment's header and checksum are checked (the checksum unless TEZGPU_SEG_VERIFIED) and its body must
 * end in the FF FF EOF marker, else TEZGPU_E_FORMAT naming the segment.
 *   write_partitions* / write_ifile*: partition p's segment is the records of p's input segments, concatenated in the
 *     order of segs, written with rle = 0 (any other rle: TEZGPU_E_INVALID); a partition without records gets no bytes
 *     and an all-zero index triple (:1087-1091); with a codec the output is compressed like a merge's.  The write copies
 *     each input's record bytes as they are and derives the output checksum from the input checksums: nothing is parsed
 *     (tezgpu_merge_parse_info: mode 3).  It differs from mergeAll, which re-encodes every record, only for inputs that
 *     writer never produces: REPEAT_KEY markers are carried over (the output still reads back as the same records) and
 *     so are non-canonical vints.  stats.output_records / spilled_records / output_bytes stay 0: the write counts no
 *     records (tezgpu_merge_counts does).
 *   next_batch: the records in (segment, position) order, same_key = 0; the first call (or tezgpu_merge_counts) parses.
 *     With num_partitions > 1 the segments are taken partition by partition (stable: inside a partition in the order
 *     of segs), as the writes lay them out; segs listed partition-major keep exactly their order.
 *   tezgpu_merge_set_combiner and tezgpu_merge_set_check_for_same_keys fail with TEZGPU_E_STATE; reopen / reopen_codec
 *   keep the handle's mode. */
int32_t tezgpu_concat_open(const tezgpu_conf *conf, const tezgpu_segment *segs, const int64_t *raw_len, uint32_t nseg,
                           int32_t codec, tezgpu_merger **out);
/* MergeQueue's checkForSameKeys constructor argument (SORT/TezMerger.java:560-573; default true like the reference's
 * other constructors, :519).  When 0, isSameKey() -- and therefore REPEAT_KEY in tezgpu_merge_write_* -- is reported
 * only for records that were run-length encoded in their input segment, never across segment boundaries
 * (adjustPriorityQueue / compareKeyWithNextTopKey, :597-652).  PipelinedSorter's final merge passes
 * merger.needsRLE() here AND as the writer's rle (SORT/PipelinedSorter.java:797-814).  Call before next_batch / write. */
int32_t tezgpu_merge_set_check_for_same_keys(tezgpu_merger *m, int32_t check_for_same_keys);
/* runs the combiner (TEZGPU_COMBINE_*) in tezgpu_merge_write_*: PipelinedSorter's final merge when
 * numSpills >= tez.runtime.combine.min.spills (SORT/PipelinedSorter.java:815-820).  Call before write_*, like
 * set_check_for_same_keys.  A merger with a combiner has no record iterator: next_batch fails with TEZGPU_E_STATE. */
int32_t tezgpu_merge_set_combiner(tezgpu_merger *m, int32_t combiner);
/* total records / key+value bytes of the merged stream */
/* diagnostics: how the last open / reopen located the records -- mode 0: fixed framing, records addressed in place
 * (no parse); 1: parallel window parser (by_hand = windows whose guessed entry was wrong and that the chase walked
 * itself); 2: sequential walker (one lane per segment: taken when the window parser meets a malformed record);
 * 3: not parsed: concatenated (tezgpu_concat_open before its first next_batch / counts) */
int32_t tezgpu_merge_parse_info(tezgpu_merger *m, int32_t *mode, int32_t *by_hand);
int32_t tezgpu_merge_counts(tezgpu_merger *m, uint64_t *records, uint64_t *kv_bytes);
/* replaces the next()/getKey()/getValue()/isSameKey() loop: fills up to idx_cap records (key||value bytes appended to
 * out_kv, at most cap bytes; a cap above 2^32 - 1 counts as 2^32 - 1, the reach of the 32-bit offsets in idx); *n = 0
 * at end of stream.  When the next record alone needs more than cap bytes the call returns TEZGPU_E_NOMEM with *n = 0,
 * idx[0].key_len and idx[0].val_len set to that record's lengths and the stream where it was: a caller grows its buffer
 * to at least key_len + val_len bytes and calls again. */
int32_t tezgpu_merge_next_batch(tezgpu_merger *m, uint8_t *out_kv, uint64_t cap, tezgpu_kv_index *idx,
                                uint32_t idx_cap, uint32_t *n);
/* TezRawKeyValueIterator for a consumer on the device: the next records of the merged stream (the records, order and
 * same_key that tezgpu_merge_next_batch would return from the same position) written into device memory on conf.device.
 * Record i of the batch: key = d_kv[d_key_off[i] .. d_val_off[i]), value = d_kv[d_val_off[i] .. + d_val_len[i]), packed
 * back to back from d_kv[0]; d_same_key[i] = isSameKey() (d_same_key may be NULL).  64-bit offsets: a batch may pass 4 GiB.
 * The table is the input triple of tezgpu_sorter_sort_device, so a batch can be sorted again without leaving the device.
 *   A batch is the longest run from the cursor with at most idx_cap records whose bytes fit in kv_cap; *kv_bytes receives
 *   its bytes, and *n = 0 at the end of the stream.  When the next record alone needs more than kv_cap bytes the call
 *   fails with TEZGPU_E_NOMEM, *n = 0, *kv_bytes = the bytes that record needs, the cursor where it was and nothing
 *   written.  Nothing is written past d_kv[*kv_bytes) or past entry *n of the table.
 *   The cursor is the one of tezgpu_merge_next_batch: the two may be interleaved on one stream.  Every handle
 *   next_batch serves is served (merges, concatenations, codec and bounded handles; a bounded handle's batches never
 *   span two of its steps).  Runs on the handle's stream (tezgpu_merge_stream) and returns once the batch is written.
 *   Checked before anything is launched or written: TEZGPU_E_INVALID for a NULL argument (other than d_same_key) or a
 *   d_kv that is not 16-byte aligned; TEZGPU_E_STATE for a merger with a combiner, as next_batch. */
int32_t tezgpu_merge_next_batch_device(tezgpu_merger *m, void *d_kv, uint64_t kv_cap, uint64_t *d_key_off,
                                       uint64_t *d_val_off, uint32_t *d_val_len, uint8_t *d_same_key,
                                       uint32_t idx_cap, uint32_t *n, uint64_t *kv_bytes);
/* replaces TezMerger.writeFile(iter, new IFile.Writer(..., rle)) (SORT/TezMerger.java:215-245): one IFile segment.
 * path may be NULL when out != NULL.  raw_len / part_len as IFile.Writer.getRawLength / getCompressedLength. */
int32_t tezgpu_merge_write_ifile(tezgpu_merger *m, const char *path, uint8_t *out, uint64_t out_cap, int32_t rle,
                                 int64_t *raw_len, int64_t *part_len, tezgpu_stats *stats);
uint64_t tezgpu_merge_output_bound(const tezgpu_merger *m);
/* device-resident output of the merged IFile segment (multi-GPU reduce side, bench).  Unless the merger was opened
 * with a codec or as a concatenation, d_out must be 16-byte aligned (the emit stores 16-byte words); a misaligned
 * d_out returns TEZGPU_E_INVALID before anything is launched or written, and the handle can write again. */
int32_t tezgpu_merge_write_ifile_device(tezgpu_merger *m, void *d_out, uint64_t out_cap, int32_t rle, int64_t *raw_len,
                                        int64_t *part_len, tezgpu_stats *stats);
/* Batched reduce side (multi-GPU shuffle): the merger was opened with conf.num_partitions = P and every segment
 * names its partition; writes the P merged segments back to back like a file.out and fills index[3*P].  d_out: as
 * for tezgpu_merge_write_ifile_device, 16-byte aligned unless the merger has a codec or is a concatenation. */
int32_t tezgpu_merge_write_partitions_device(tezgpu_merger *m, void *d_out, uint64_t out_cap, int32_t rle,
                                             uint64_t *out_len, int64_t *index, tezgpu_stats *stats);
/* same, written to file.out + file.out.index (mode 0640): the final merge of PipelinedSorter.flush over several spills
 * (SORT/PipelinedSorter.java:774-836) */
int32_t tezgpu_merge_write_partitions(tezgpu_merger *m, const char *out_path, const char *index_path, int32_t rle,
                                      int64_t *index, tezgpu_stats *stats);
/* Bounded-memory merge (TezMerger merges any number of segments through one small buffer per segment,
 * SORT/TezMerger.java:717-912): the k-way merge of tezgpu_merge_open_codec over HOST segments, holding at most
 * budget_bytes of device memory.  budget_bytes = 0: the device's free memory at open; a budget below
 * TEZGPU_MERGE_BUDGET_MIN fails with TEZGPU_E_INVALID, a device segment (TEZGPU_SEG_DEVICE) too.  codec must be
 * TEZGPU_CODEC_NONE (else TEZGPU_E_UNSUPPORTED; compressed output: tezgpu_merge_open_bounded_write_codec); raw_len is
 * not read.
 *   When the inputs fit the budget with one record per input byte (the worst case of the workspace bound in DESIGN
 *   section 3, "Bounded-memory merge"), the handle takes one step: exactly tezgpu_merge_open.  Otherwise it merges in
 *   key-range steps over windows of the segments; when the first step's windows hold every segment whole and the
 *   bound on their scanned records fits, that step is the whole merge and the handle behaves as a one-step one.  With
 *   several steps the segments must stay valid and unchanged until close.  The stream, the written bytes and
 *   the counts are those of the one-step merge; a checksum mismatch fails with TEZGPU_E_FORMAT naming the segment
 *   before the stream ends or a write succeeds; a key group larger than the budget allows fails with TEZGPU_E_NOMEM.
 *   The handle takes set_check_for_same_keys, set_combiner, next_batch, write_ifile, write_partitions, parse_info
 *   (of the last step), counts and close.  With several steps: counts fails with TEZGPU_E_STATE until the stream has
 *   been read to its end or written, output_bound returns 0 until then, every write runs the steps again (a
 *   next_batch after it starts from the first record), and write_*_device and reopen* fail with TEZGPU_E_STATE. */
#define TEZGPU_MERGE_BUDGET_MIN (16ull << 20)
int32_t tezgpu_merge_open_bounded(const tezgpu_conf *conf, const tezgpu_segment *segs, const int64_t *raw_len, uint32_t nseg,
                                  int32_t codec, uint64_t budget_bytes, tezgpu_merger **out);
/* The bounded merge with compressed output: tezgpu_merge_open_bounded over the same uncompressed HOST segments, budget
 * and checks (same codes and messages), whose writes compress with write_codec (TEZGPU_CODEC_NONE, _DEFAULT, _LZ4,
 * _ZSTD or _SNAPPY; any other fails with TEZGPU_E_UNSUPPORTED before any device call).  NONE: exactly
 * tezgpu_merge_open_bounded.  A handle that takes one step is exactly tezgpu_merge_open_codec(conf, segs, NULL, nseg,
 * write_codec).  With several steps, write_ifile and write_partitions write the file and index that handle writes,
 * byte for byte (rawLength uncompressed, partLength compressed): every step compresses its pieces on the codec's chunk
 * grid of each partition, so the budget includes the compression workspace (DESIGN section 3).  stats are as the
 * codec writes give them (physical bytes compressed, ms_total with the compression), output_bound bounds the
 * compressed bytes once the counts are known; everything else is as for tezgpu_merge_open_bounded. */
int32_t tezgpu_merge_open_bounded_write_codec(const tezgpu_conf *conf, const tezgpu_segment *segs, uint32_t nseg,
                                              int32_t write_codec, uint64_t budget_bytes, tezgpu_merger **out);
/* steps the last pass over the inputs took (1 for a one-step handle), the most device memory the handle's buffers
 * held at once, and the bytes uploaded from the host segments by all passes.  TEZGPU_E_STATE on a handle that was
 * not opened bounded. */
int32_t tezgpu_merge_bounded_info(tezgpu_merger *m, int32_t *steps, uint64_t *peak_device_bytes, uint64_t *h2d_bytes);
/* Decodes compressed HOST segments on the device under a device budget, so that tezgpu_merge_open_bounded (which takes
 * uncompressed segments only) can merge them.  For every segment whose header flag byte is 1, out[i] receives its
 * uncompressed IFile segment of raw_len[i] + 4 bytes: TIF\0, the body, the CRC-32 of the body -- what an uncompressed
 * IFile.Writer writes for the same records.  Other segments are not read past their header and their out[i] may be NULL.
 * Checksums and streams are checked as tezgpu_merge_open_codec checks them (same codes and messages, naming the
 * caller's segment index); the decoders are that call's.  The segments are decoded whole, in groups whose staged
 * compressed bytes, images and decoder workspace stay within budget_bytes (DESIGN.md section 3); *peak_device_bytes
 * (may be NULL) receives the most device memory the call held at once.  A segment that does not fit the budget on its
 * own fails with TEZGPU_E_NOMEM naming it and its sizes.  TEZGPU_E_INVALID: a device segment, a budget below
 * TEZGPU_MERGE_BUDGET_MIN, raw_len NULL (with nseg > 0), out[i] NULL for a compressed segment.  TEZGPU_E_UNSUPPORTED:
 * a codec other than TEZGPU_CODEC_DEFAULT, _LZ4, _ZSTD and _SNAPPY.  Runs on conf->device; conf's other fields are checked as
 * for a merge. */
int32_t tezgpu_decode_segments(const tezgpu_conf *conf, const tezgpu_segment *segs, const int64_t *raw_len, uint32_t nseg,
                               int32_t codec, uint64_t budget_bytes, uint8_t *const *out, uint64_t *peak_device_bytes);
void *tezgpu_merge_stream(tezgpu_merger *m);
int32_t tezgpu_merge_close(tezgpu_merger *m);

/* ---------------------------------------------------------------------------------------------------------------
 * Shuffle transfer between the GPUs of one box (NVLink / NVSwitch).
 * Replaces the ShuffleHandler HTTP GET + FetcherOrderedGrouped.copyMapOutput round trip
 * (OG/FetcherOrderedGrouped.java:437-632, OG/ShuffleScheduler.java:1370-1470): the producer keeps file.out in an
 * exportable device buffer, the consumer maps it (CUDA IPC) and pulls the byte ranges of its partitions with one
 * kernel running on every SM.  Handles are 64 opaque bytes the host layer ships with the DataMovementEvent.
 * --------------------------------------------------------------------------------------------------------------- */
#define TEZGPU_PEER_HANDLE_BYTES 64
/* device buffer another process on the same box may map; *handle_out receives the 64-byte export handle */
int32_t tezgpu_peer_alloc(int32_t device, uint64_t bytes, void **dptr, uint8_t *handle_out);
int32_t tezgpu_peer_free(int32_t device, void *dptr);
/* maps a buffer exported by another process (any device of the box) into this process; enables peer access */
int32_t tezgpu_peer_open(int32_t device, const uint8_t *handle, void **dptr);
int32_t tezgpu_peer_close(int32_t device, void *dptr);
typedef struct tezgpu_copy_range {
  const void *src;                 /* device address (local, or a peer mapping from tezgpu_peer_open) */
  void *dst;                       /* device address on `device`; fastest when (dst - src) is a multiple of 16 */
  uint64_t len;
} tezgpu_copy_range;
/* copies n ranges with one launch on `stream` (a cudaStream_t, NULL = the legacy default stream) and returns once
 * the bytes have landed */
int32_t tezgpu_fetch_ranges(int32_t device, const tezgpu_copy_range *ranges, uint32_t n, void *stream,
                            float *ms_kernel);

/* The same pull with every segment's IFile checksum verified on the bytes as they pass through the copy kernel -- what
 * IFile.Reader.readToMemory does when FetcherOrderedGrouped fetches a map output to MEMORY (SORT/IFile.java:764-809,
 * OG/FetcherOrderedGrouped.java:519-533).  One entry per (non-empty) segment; src may be a peer mapping, dst is local,
 * (dst - src) must be a multiple of 16 and only the bytes of the listed segments move.  Fails with TEZGPU_E_FORMAT
 * ("IFile checksum mismatch in fetched segment i") like the reference's ChecksumException; segments that passed may be
 * handed to tezgpu_merge_open with TEZGPU_SEG_VERIFIED so the merge does not read them a second time to check. */
typedef struct tezgpu_fetch_segment {
  const void *src;
  void *dst;
  uint64_t len;                    /* whole segment: header + body + 4 checksum bytes */
  uint32_t flags;                  /* TEZGPU_SEG_HAS_HEADER */
  uint32_t reserved;
} tezgpu_fetch_segment;
int32_t tezgpu_fetch_segments_verified(int32_t device, const tezgpu_fetch_segment *segs, uint32_t n, void *stream,
                                       float *ms_kernel);

/* ---- SURVEY 8 f-2: the ShuffleHandler <-> FetcherOrderedGrouped wire format, for consumers outside the NVLink domain
 * (and unmodified fetchers).  Per map output and reducer: ShuffleHeader (OG/ShuffleHeader.java:101-106:
 * Text.writeString(mapId), vlong compressedLength = partLength, vlong uncompressedLength = rawLength, vint forReduce)
 * followed by partLength bytes of the partition's IFile segment (OG/FetcherOrderedGrouped.java:437-632 reads exactly
 * that).  Host-side framing; the segment bytes are copied out of the device-resident file.out. */
uint64_t tezgpu_shuffle_header_size(const char *map_id, int64_t part_len, int64_t raw_len, int32_t reduce);
int32_t tezgpu_shuffle_header_write(const char *map_id, int64_t part_len, int64_t raw_len, int32_t reduce, uint8_t *out,
                                    uint64_t cap, uint64_t *len);
/* ShuffleHeader.readFields (:82-87, map id at most 1000 bytes); consumed = header bytes */
int32_t tezgpu_shuffle_header_read(const uint8_t *in, uint64_t avail, char *map_id, uint64_t map_id_cap, int64_t *part_len,
                                   int64_t *raw_len, int32_t *reduce, uint64_t *consumed);
/* response body for reducers [reduce0, reduce0 + nreduce) of ONE map output whose file.out lives in device memory:
 * index = the 3 * P int64 triples (start, rawLength, partLength) of its spill record; out = host (ideally pinned) buffer
 * of at least tezgpu_shuffle_serve_bound bytes; returns after the copies completed */
uint64_t tezgpu_shuffle_serve_bound(const char *map_id, const int64_t *index, int32_t reduce0, int32_t nreduce);
int32_t tezgpu_shuffle_serve(int32_t device, const void *d_file_out, const int64_t *index, const char *map_id,
                             int32_t reduce0, int32_t nreduce, uint8_t *out, uint64_t cap, uint64_t *len, void *stream);
/* consumer side: splits a response body into its segments (what copyMapOutput does header by header); every segment is
 * in[offset .. offset + part_len) and can go to tezgpu_merge_open as a host segment with TEZGPU_SEG_HAS_HEADER */
typedef struct tezgpu_wire_segment {
  char map_id[1008];
  int64_t part_len;
  int64_t raw_len;
  uint64_t offset;
  int32_t reduce;
  int32_t reserved;
} tezgpu_wire_segment;
int32_t tezgpu_shuffle_receive(const uint8_t *in, uint64_t len, tezgpu_wire_segment *segs, uint32_t cap, uint32_t *n);

/* diagnostics: host-side emulation of the device's tiled CRC algebra (same tables, no GPU needed) */
uint32_t tezgpu_debug_crc_emulate(const uint8_t *body, uint64_t len, uint32_t piece_bytes, uint32_t lead);

/* diagnostics: host-side run of the chunk-interleaved CRC fold of the emit / verify kernels (ilp: two-deep form) */
uint32_t tezgpu_debug_chunk_fold_emulate(const uint8_t *data, uint32_t nchunks, int32_t ilp);

/* diagnostics: host-side run of the per-thread-run CRC fold of the packed fixed-width emit kernel (nchunks <= 1280) */
uint32_t tezgpu_debug_run_fold_emulate(const uint8_t *data, uint32_t nchunks);

/* diagnostics: the emit kernel and tile size the device picks for fixed-width records of klen + vlen bytes written
 * without repeats.  layout: 0 packed, 16-byte aligned records (the map side); 1 records at explicit offsets; 2 a run
 * table of fixed-framing segments (the reduce side).  *kernel: 0 k_emit_fast4 (20480-byte tile image), 1
 * k_emit_fast<5, true>, 2 k_emit_fast4u, 3 k_emit_fast<5, false> (22016-byte images), 4 k_emit<true> (tiles written
 * in pieces, any record size). */
int32_t tezgpu_debug_fixed_emit_plan(uint32_t klen, uint32_t vlen, int32_t layout, int32_t *kernel, uint32_t *recs_per_tile);

/* diagnostics: the launch shape of fixed-width emit kernel `kernel` (numbered as in tezgpu_debug_fixed_emit_plan) over
 * `tiles` tiles on `device`: *ctas CTAs of *groups_per_cta persistent tile groups each.  Group g of CTA b emits tile
 * b * groups_per_cta + g, then every (ctas * groups_per_cta)-th tile. */
int32_t tezgpu_debug_emit_grid(int32_t device, int32_t kernel, uint64_t tiles, uint32_t *ctas, uint32_t *groups_per_cta);

/* diagnostics: tezgpu_sorter_device_output_bound of a handle with num_partitions partitions and codec (TEZGPU_CODEC_*),
 * computed without a device; 0 for num_partitions < 1 or an unknown codec */
uint64_t tezgpu_debug_device_output_bound(int32_t num_partitions, int32_t codec, uint64_t n, uint64_t kv_bytes);

/* diagnostics: the checksum algebra of tezgpu_concat_open on the host: bodies[i] (lens[i] bytes, ending in FF FF) are
 * the input bodies; each one's CRC-32 becomes the remainder of its record bytes, those are folded with crc(A||B), and
 * the EOF marker is appended.  *crc = the CRC-32 of the concatenated record bytes followed by FF FF. */
int32_t tezgpu_debug_crc_concat_emulate(const uint8_t *const *bodies, const uint64_t *lens, uint32_t n, uint32_t *crc);

/* diagnostics: the device codec run on the host with the same code.  deflate: the zlib stream the device writes for one
 * segment body (a compressed segment is TIF\x01 + this + CRC-32).  inflate: decodes a compressed segment body (the bytes
 * between header and CRC) that must yield exactly body_len bytes; TEZGPU_E_FORMAT names the reason otherwise. */
int32_t tezgpu_debug_deflate_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len);
int32_t tezgpu_debug_inflate_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                     uint64_t *out_len);
/* the same for TEZGPU_CODEC_LZ4: lz4_compress gives the block stream the device writes for one body; lz4_decompress runs
 * the device reader's exact (serial) path over a stream that must yield exactly body_len bytes. */
int32_t tezgpu_debug_lz4_compress_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len);
int32_t tezgpu_debug_lz4_decompress_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                            uint64_t *out_len);
/* the same for TEZGPU_CODEC_ZSTD: zstd_compress gives the frames the device writes for one body; zstd_decompress runs
 * the device reader's exact (serial) path over a stream that must yield exactly body_len bytes. */
int32_t tezgpu_debug_zstd_compress_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len);
int32_t tezgpu_debug_zstd_decompress_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                             uint64_t *out_len);
/* the same for TEZGPU_CODEC_SNAPPY: snappy_compress gives the block stream the device writes for one body;
 * snappy_decompress runs the device reader's walk and chunk decoder on one lane and fails with the reason it gives */
int32_t tezgpu_debug_snappy_compress_emulate(const uint8_t *body, uint64_t len, uint8_t *out, uint64_t cap, uint64_t *out_len);
int32_t tezgpu_debug_snappy_decompress_emulate(const uint8_t *z, uint64_t len, uint64_t body_len, uint8_t *out, uint64_t cap,
                                               uint64_t *out_len);
/* the compressed write of a bounded merge that takes several steps, on the host: the body (len >= 1 bytes) of one
 * partition cut into pieces at the ncuts non-decreasing offsets cuts[], each piece compressed as a step compresses it
 * (the chunk grid from the body's start, the carry of the bytes after the last whole chunk, zlib's open chunks and
 * Adler-32 fold, the CRC-32 fold, checked against the stream).  out receives the codec stream, which is
 * tezgpu_debug_{deflate,lz4_compress,zstd_compress,snappy_compress}_emulate of the uncut body.  codec: _DEFAULT, _LZ4,
 * _ZSTD or _SNAPPY. */
int32_t tezgpu_debug_stitched_compress_emulate(int32_t codec, const uint8_t *body, uint64_t len, const uint64_t *cuts, uint32_t ncuts,
                                               uint8_t *out, uint64_t cap, uint64_t *out_len);

/* diagnostics: the 32-bit sort words the variable-width map side gives n keys (key i = kv[key_off[i] ..
 * key_off[i] + key_len[i])), computed on the host with the device's code: the alphabet table built from the byte values
 * that occur, then every key's word.  partition: given partition ids, or NULL for the HashPartitioner.  use_sym = 0
 * forces the raw 4-byte prefix (TEZGPU_NO_SYM=1).  npos: content positions the alphabet table packs; sym_used: 1 when
 * the words are packed ranks (the table packs more positions than the raw prefix holds), 0 for the raw prefix. */
int32_t tezgpu_debug_sort_words_emulate(const uint8_t *kv, const uint64_t *key_off, const uint32_t *key_len, uint32_t n,
                                        int32_t comparator, int32_t num_partitions, const int32_t *partition,
                                        int32_t use_sym, uint32_t *words, uint32_t *npos, int32_t *sym_used);

/* diagnostics: tezgpu_sorter_set_split_points' checks and the device's split search, on the host with the same code.
 * Key i = kv[key_off[i] .. + key_len[i]), split j = splits[split_off[j] .. + split_len[j]]; comparator is the sort
 * comparator the checks use, order the search order.  partition[i] receives key i's partition (P = nsplits + 1). */
int32_t tezgpu_debug_total_order_emulate(const uint8_t *kv, const uint64_t *key_off, const uint32_t *key_len, uint32_t n,
                                         const uint8_t *splits, const uint64_t *split_off, const uint32_t *split_len,
                                         uint32_t nsplits, int32_t comparator, int32_t order, int32_t *partition);

/* diagnostics: keeps only the bits of `mask` of every hash tezgpu_sample_keys computes (h = splitmix64(seed ^ gid) & mask)
 * and returns the mask it replaces; ~0 (the default) keeps them all.  splitmix64 is a bijection, so records of one seed
 * never tie in h: a narrow mask makes them tie, for tests of the cap's order (h, gid).  Process-wide. */
uint64_t tezgpu_debug_set_sample_hash_mask(uint64_t mask);

#ifdef __cplusplus
}
#endif
#endif /* TEZGPU_H */

/*
 * GpuSorter -- the ExternalSorter seam of OrderedPartitionedKVOutput backed by libtezgpu.so (include/tezgpu.h).
 *
 * Drop-in position: add `GPU` to OrderedPartitionedKVOutput.SorterImpl and construct this class where start() builds
 * PipelinedSorter / DefaultSorter (tez-runtime-library/.../output/OrderedPartitionedKVOutput.java:116-160).  Everything
 * else of the plugin -- events, counters, file names, the KeyValuesWriter -- is the reference's own code.
 *
 * NOT COMPILED IN THIS REPOSITORY: the build image has no JDK (java, javac and mvn are absent).  The C side of every
 * native method below is jni/tezgpu_jni.c; both follow include/tezgpu.h, which IS built and tested here through ctypes.
 */
package org.apache.tez.runtime.library.common.sort.impl;

import java.io.IOException;
import java.nio.ByteBuffer;
import java.nio.ByteOrder;
import java.nio.IntBuffer;

import org.apache.hadoop.conf.Configuration;
import org.apache.hadoop.fs.Path;
import org.apache.hadoop.io.BytesWritable;
import org.apache.hadoop.io.IntWritable;
import org.apache.hadoop.io.LongWritable;
import org.apache.hadoop.io.RawComparator;
import org.apache.hadoop.io.SequenceFile;
import org.apache.hadoop.io.Text;
import org.apache.hadoop.io.compress.CompressionCodec;
import org.apache.hadoop.io.compress.DefaultCodec;
import org.apache.hadoop.io.compress.Lz4Codec;
import org.apache.hadoop.io.compress.ZStandardCodec;
import org.apache.hadoop.io.serializer.SerializationFactory;
import org.apache.hadoop.io.serializer.Serializer;
import org.apache.hadoop.mapreduce.lib.partition.TotalOrderPartitioner;
import org.apache.hadoop.util.ReflectionUtils;
import org.apache.tez.runtime.api.OutputContext;
import org.apache.tez.runtime.library.api.TezRuntimeConfiguration;
import org.apache.tez.runtime.library.common.ConfigUtils;
import org.apache.tez.runtime.library.common.comparator.TezBytesComparator;
import org.apache.tez.runtime.library.partitioner.HashPartitioner;

/** Replaces PipelinedSorter.collect / sort / spill / flush (PipelinedSorter.java:387-466, 558-859). */
public class GpuSorter extends ExternalSorter {
  static {
    System.loadLibrary("tezgpu_jni"); // jni/tezgpu_jni.c, linked against libtezgpu.so
  }

  // ids of include/tezgpu.h
  static final int CMP_BYTES = 0, CMP_TEXT = 1, CMP_BYTESWRITABLE = 2, CMP_INT = 3, CMP_LONG = 4;
  static final int PART_GIVEN = 0, PART_HASH = 1, PART_TOTAL_ORDER = 2;
  static final String TOTAL_ORDER_NEW = "org.apache.hadoop.mapreduce.lib.partition.TotalOrderPartitioner";
  static final String TOTAL_ORDER_OLD = "org.apache.hadoop.mapred.lib.TotalOrderPartitioner";
  static final String MR_PARTITIONER = "org.apache.tez.mapreduce.partition.MRPartitioner";
  static final int COMBINE_NONE = 0, COMBINE_SUM_INT = 1, COMBINE_SUM_LONG = 2;
  static final int CODEC_NONE = 0, CODEC_DEFAULT = 1, CODEC_LZ4 = 2, CODEC_ZSTD = 3;
  static final int SORTER_UNORDERED = 2;
  private static final int BATCH_BYTES = 32 << 20;
  private static final int BATCH_RECORDS = 1 << 20;

  private long handle; // tezgpu_sorter*
  // the batch being serialised; a record larger than BATCH_BYTES is staged alone in a buffer sized for it
  private ByteBuffer kv = ByteBuffer.allocateDirect(BATCH_BYTES).order(ByteOrder.nativeOrder());
  private final IntBuffer keyOff = direct(BATCH_RECORDS), valOff = direct(BATCH_RECORDS), valLen = direct(BATCH_RECORDS),
      part = direct(BATCH_RECORDS);
  private final boolean devicePartitioner; // HashPartitioner or TotalOrderPartitioner: write() passes no partition
  private final BatchOutputStream sink = new BatchOutputStream();
  private int n;
  private int recStart; // offset in kv of the record being serialised
  private long collectedBytes;
  private boolean lastSpillRle;
  private final boolean unordered;

  private static IntBuffer direct(int ints) {
    return ByteBuffer.allocateDirect(4 * ints).order(ByteOrder.nativeOrder()).asIntBuffer();
  }

  public GpuSorter(OutputContext outputContext, Configuration conf, int numOutputs, long initialMemoryAvailable)
      throws IOException {
    this(outputContext, conf, numOutputs, initialMemoryAvailable, false);
  }

  /**
   * unordered: the writer behind UnorderedPartitionedKVOutput / UnorderedKVOutput (UnorderedPartitionedKVWriter): records
   * are only partitioned, no combiner runs, and the final merge over spills concatenates them (concatSpills).
   */
  public GpuSorter(OutputContext outputContext, Configuration conf, int numOutputs, long initialMemoryAvailable,
      boolean unordered) throws IOException {
    super(outputContext, conf, numOutputs, initialMemoryAvailable);
    this.unordered = unordered;
    final boolean deviceHash = partitioner instanceof HashPartitioner;
    final boolean totalOrder = totalOrderPartitioner(conf, numOutputs, unordered);
    devicePartitioner = deviceHash || totalOrder;
    // an unordered edge compares no keys; with TotalOrderPartitioner the split points are still checked in key order
    final int cmp = unordered && !totalOrder ? CMP_BYTES : comparatorId(comparator, conf);
    handle = nativeCreate(numOutputs, cmp, totalOrder ? PART_TOTAL_ORDER : deviceHash ? PART_HASH : PART_GIVEN,
        sendEmptyPartitionDetails, initialMemoryAvailable, /* CUDA ordinal, from the container's environment */
        Integer.parseInt(System.getenv().getOrDefault("TEZGPU_DEVICE", "0")), unordered ? SORTER_UNORDERED : 0);
    if (totalOrder) setSplitPoints(conf, cmp);
    keySerializer.open(sink);
    valSerializer.open(sink);
    // ExternalSorter.codec = CodecUtils.getCodec(conf): every spill and the final merge write through it
    final int c = codecId(codec);
    if (c != CODEC_NONE) nativeSetCodec(handle, c);
  }

  /**
   * The device writes and reads DefaultCodec (zlib), Lz4Codec and ZStandardCodec segments only.  The class must be one of them itself:
   * GzipCodec extends DefaultCodec but writes gzip members, so an instanceof test would be wrong.  Lz4Codec's
   * io.compression.codec.lz4.buffersize must lie in [TEZGPU_LZ4_CHUNK_BOUND, 262144] (tezgpu.h), as the plugin mirror
   * checks: Java readers decode the device's chunks into a buffer of that size, and the device reader takes chunks of
   * at most 262,144 bytes.  ZStandardCodec's io.compression.codec.zstd.level has no effect on the device writer.
   */
  static int codecId(CompressionCodec codec) throws IOException {
    if (codec == null) return CODEC_NONE;
    if (codec.getClass() == DefaultCodec.class) return CODEC_DEFAULT;
    if (codec.getClass() == Lz4Codec.class) return CODEC_LZ4;
    if (codec.getClass() == ZStandardCodec.class) return CODEC_ZSTD;
    throw new IOException("tez.runtime.compress.codec=" + codec.getClass().getName()
        + ": only org.apache.hadoop.io.compress.DefaultCodec, org.apache.hadoop.io.compress.Lz4Codec and"
        + " org.apache.hadoop.io.compress.ZStandardCodec are supported on the device path");
  }

  /**
   * Runs ExternalSorter's combiner on the device at every spill, when it is MRCombiner with IntSumReducer /
   * LongSumReducer (COMBINE_SUM_INT / COMBINE_SUM_LONG, chosen by the caller from the reducer and value classes).
   * Call before the first write.  Any other combiner is not run (a combiner may run zero times).
   */
  public void setCombiner(int combiner) throws IOException {
    nativeSetCombiner(handle, combiner);
  }

  /**
   * TotalOrderPartitioner (new or old API) is the output's partitioner: named as tez.runtime.partitioner.class, or
   * wrapped by MRPartitioner with more than one partition as mapreduce.job.partitioner.class (new API) /
   * mapred.partitioner.class (old API), as MRPartitioner picks it.  An unordered writer with one partition
   * (UnorderedKVOutput) runs no partitioner.  The plugin mirror decides the same way (tez_runtime_library.cc
   * total_order_partitioner).
   */
  static boolean totalOrderPartitioner(Configuration conf, int partitions, boolean unordered) {
    final String pc = conf.get(TezRuntimeConfiguration.TEZ_RUNTIME_PARTITIONER_CLASS, "");
    if (TOTAL_ORDER_NEW.equals(pc) || TOTAL_ORDER_OLD.equals(pc)) return !(unordered && partitions == 1);
    if (!MR_PARTITIONER.equals(pc) || partitions <= 1) return false;
    final String wrapped = conf.getBoolean("mapred.mapper.new-api", false) ? conf.get("mapreduce.job.partitioner.class", "")
        : conf.get("mapred.partitioner.class", "");
    return TOTAL_ORDER_NEW.equals(wrapped) || TOTAL_ORDER_OLD.equals(wrapped);
  }

  /**
   * TotalOrderPartitioner.setConf on the device: the split keys of TotalOrderPartitioner.getPartitionFile(conf)
   * (mapreduce.totalorderpartitioner.path, default _partition.lst; both APIs read the same key), read with
   * SequenceFile.Reader, serialized with the job's key serialization (what keySerializer writes for record keys) into
   * one direct buffer, and handed to tezgpu_sorter_set_split_points, which checks their count and order with Hadoop's
   * messages.  Search order: the content order of Text / BytesWritable keys with
   * mapreduce.totalorderpartitioner.naturalorder (default true), else the comparator's.
   */
  private void setSplitPoints(Configuration conf, int cmp) throws IOException {
    final Class<?> keyClass = ConfigUtils.getIntermediateOutputKeyClass(conf);
    final Path file = new Path(TotalOrderPartitioner.getPartitionFile(conf));
    final java.io.ByteArrayOutputStream bytes = new java.io.ByteArrayOutputStream();
    final java.util.ArrayList<Integer> lens = new java.util.ArrayList<>();
    @SuppressWarnings("unchecked")
    final Serializer<Object> ser = (Serializer<Object>) new SerializationFactory(conf).getSerializer(keyClass);
    ser.open(bytes);
    try (SequenceFile.Reader reader = new SequenceFile.Reader(conf, SequenceFile.Reader.file(file))) {
      Object key = ReflectionUtils.newInstance(keyClass, conf);
      while ((key = reader.next(key)) != null) {   // "wrong key class" comes from the reader, as in Hadoop
        final int before = bytes.size();
        ser.serialize(key);
        lens.add(bytes.size() - before);
      }
    } finally {
      ser.close();
    }
    final int n = lens.size();
    final ByteBuffer keys = ByteBuffer.allocateDirect(Math.max(1, bytes.size()));
    keys.put(bytes.toByteArray());
    final long[] off = new long[n];
    final int[] len = new int[n];
    for (int i = 0, at = 0; i < n; i++) {
      off[i] = at;
      len[i] = lens.get(i);
      at += len[i];
    }
    final boolean natural = conf.getBoolean(TotalOrderPartitioner.NATURAL_ORDER, true);
    final int order = natural && keyClass == Text.class ? CMP_TEXT
        : natural && keyClass == BytesWritable.class ? CMP_BYTESWRITABLE : cmp;
    // mapreduce.totalorderpartitioner.trie.maxdepth only shapes Java's index over the split points: nothing to pass
    nativeSetSplitPoints(handle, keys, off, len, n, order);
  }

  /** The device path supports a closed set of RawComparators; anything else keeps tez.runtime.sorter.class=PIPELINED. */
  static int comparatorId(RawComparator<?> c, Configuration conf) throws IOException {
    if (c instanceof TezBytesComparator) return CMP_BYTES;
    if (c instanceof Text.Comparator) return CMP_TEXT;
    if (c instanceof BytesWritable.Comparator) return CMP_BYTESWRITABLE;
    if (c instanceof IntWritable.Comparator) return CMP_INT;
    if (c instanceof LongWritable.Comparator) return CMP_LONG;
    throw new IOException("GpuSorter: no device comparator for " + c.getClass().getName()
        + " (supported: TezBytesComparator, Text, BytesWritable, IntWritable, LongWritable)");
  }

  @Override
  public void write(Object key, Object value) throws IOException {
    final int p = devicePartitioner ? -1 : partitioner.getPartition(key, value, partitions);
    if (!devicePartitioner && (p < 0 || p >= partitions)) {
      throw new IOException("Illegal partition for " + key + " (" + p + ")"); // PipelinedSorter.java:410-413
    }
    recStart = kv.position();
    keySerializer.serialize(key); // the same serializers PipelinedSorter.collect drives
    final int keyLen = kv.position() - recStart;
    valSerializer.serialize(value);
    // read after both serialisations: overflow() may have moved the record to the front of a new buffer
    keyOff.put(n, recStart);
    valOff.put(n, recStart + keyLen);
    valLen.put(n, kv.position() - recStart - keyLen);
    if (!devicePartitioner) part.put(n, p);
    mapOutputRecordCounter.increment(1);
    mapOutputByteCounter.increment(kv.position() - recStart);
    if (++n == BATCH_RECORDS || kv.remaining() < (BATCH_BYTES >> 3)) pushBatch();
    if (kv.capacity() > BATCH_BYTES) {
      pushBatch(); // the oversized record goes alone; the next batch takes a buffer of the usual size
      kv = ByteBuffer.allocateDirect(BATCH_BYTES).order(ByteOrder.nativeOrder());
    }
    // the granted sort memory bounds what one spill holds (ExternalSorter.getInitialMemoryRequirement, :330-347)
    if (collectedBytes + kv.position() > availableMemoryMb * 1024L * 1024L) {
      pushBatch();
      spill(false);
    }
  }

  /**
   * The record being serialised needs `more` bytes beyond the end of kv: push the records before it, then carry its
   * bytes so far to the front of kv, or of a new buffer sized for it when kv cannot hold it.
   */
  private void overflow(int more) throws IOException {
    final byte[] head = new byte[kv.position() - recStart];
    kv.position(recStart);
    kv.get(head);
    kv.position(recStart);
    pushBatch();
    kv.clear();
    final long need = (long) head.length + more;
    if (need > kv.capacity()) {
      if (need > Integer.MAX_VALUE - 8) throw new IOException("GpuSorter: record of " + need + " bytes or more");
      kv = ByteBuffer.allocateDirect((int) Math.min(Integer.MAX_VALUE - 8, Math.max(need, 2L * kv.capacity())))
          .order(ByteOrder.nativeOrder());
    }
    kv.put(head);
    recStart = 0;
  }

  private void pushBatch() throws IOException {
    if (n == 0) return;
    nativeCollect(handle, kv, kv.position(), keyOff, valOff, valLen, devicePartitioner ? null : part, n); // tezgpu_sorter_collect_batch
    collectedBytes += kv.position();
    kv.clear();
    n = 0;
  }

  private void spill(boolean last) throws IOException {
    final org.apache.hadoop.fs.Path out = mapOutputFile.getSpillFileForWrite(numSpills, collectedBytes);
    final org.apache.hadoop.fs.Path index = mapOutputFile.getSpillIndexFileForWrite(numSpills, partitions * 24L + 8);
    final long[] idx = new long[3 * partitions];
    final long[] counters = new long[8];
    nativeFlush(handle, out.toString(), index.toString(), idx, counters); // tezgpu_sorter_flush: file.out + file.out.index, 0640
    nativeReset(handle);
    lastSpillRle = counters[5] != 0;
    outputBytesWithOverheadCounter.increment(counters[0]);
    spilledRecordsCounter.increment(counters[2]);
    if (reportPartitionStats()) {
      for (int i = 0; i < partitions; i++) partitionStats[i] += idx[3 * i + 1]; // PipelinedSorter.java:631-633
    }
    numSpills++;
    collectedBytes = 0;
  }

  @Override
  public void flush() throws IOException {
    pushBatch();
    spill(true);
    numAdditionalSpills.increment(numSpills - 1);
    if (numSpills == 1 || !isFinalMergeEnabled()) {
      // single spill: sameVolRename to the final names (PipelinedSorter.java:730-756) -- unchanged reference code
      finishSingleSpillOrPipelined();
      return;
    }
    // final merge of all spills on the device, every partition at once (PipelinedSorter.java:774-836):
    // checkForSameKeys and the writer's rle are both needsRLE() of the LAST spill (:797-814)
    finalOutputFile = mapOutputFile.getOutputFileForWrite(0);
    finalIndexFile = mapOutputFile.getOutputIndexFileForWrite(0);
    if (unordered) {
      concatSpills(finalOutputFile.toString(), finalIndexFile.toString());
      numShuffleChunks.setValue(1);
      return;
    }
    GpuMergeIterator.mergeSpillsToFile(spillFilePaths(), spillIndexPaths(), partitions,
        comparatorId(comparator, conf), sendEmptyPartitionDetails, lastSpillRle, lastSpillRle, codecId(codec),
        finalOutputFile.toString(), finalIndexFile.toString());
    numShuffleChunks.setValue(1);
  }

  @Override
  public void close() throws IOException {
    super.close();
    if (handle != 0) nativeDestroy(handle);
    handle = 0;
  }

  /**
   * UnorderedPartitionedKVWriter.mergeAll (UnorderedPartitionedKVWriter.java:1058-1144) on the device: per partition the
   * current buffer (the spill flush() forced last) and then the spills in order, concatenated without run-length
   * encoding (tezgpu_concat_open + tezgpu_merge_write_partitions).  Partitions without records get no bytes and an
   * all-zero index entry.
   */
  private void concatSpills(String out, String index) throws IOException {
    final String[] files = spillFilePaths(), indexFiles = spillIndexPaths();
    final int s0 = numSpills;
    final ByteBuffer[] bytes = new ByteBuffer[s0];
    final TezSpillRecord[] records = new TezSpillRecord[s0];
    int nseg = 0;
    for (int s = 0; s < s0; s++) {
      try (java.nio.channels.FileChannel ch = java.nio.channels.FileChannel.open(java.nio.file.Paths.get(files[s]))) {
        bytes[s] = ByteBuffer.allocateDirect((int) ch.size());
        while (bytes[s].hasRemaining() && ch.read(bytes[s]) >= 0) { }
      }
      records[s] = new TezSpillRecord(new org.apache.hadoop.fs.Path(indexFiles[s]), conf);
      for (int p = 0; p < partitions; p++) if (records[s].getIndex(p).getPartLength() > 0) nseg++;
    }
    final long[] addresses = new long[nseg], lengths = new long[nseg], raws = new long[nseg];
    final int[] flags = new int[nseg], parts = new int[nseg];
    int i = 0;
    for (int p = 0; p < partitions; p++) {
      for (int k = 0; k < s0; k++) {
        final int s = k == 0 ? s0 - 1 : k - 1;
        final TezIndexRecord r = records[s].getIndex(p);
        if (r.getPartLength() == 0) continue;   // "Skip empty partitions within a spill" (:1108-1111)
        addresses[i] = GpuMergeIterator.nativeAddress(bytes[s]) + r.getStartOffset();
        lengths[i] = r.getPartLength();
        raws[i] = r.getRawLength();
        flags[i] = GpuMergeIterator.SEG_HAS_HEADER;
        parts[i++] = p;
      }
    }
    final GpuMergeIterator m = GpuMergeIterator.concat(addresses, lengths, flags, parts, partitions, raws, codecId(codec));
    try {
      m.writePartitions(out, index, partitions, false);
    } finally {
      m.close();
    }
  }

  // helpers a maintainer wires to the reference's own code (names as in PipelinedSorter)
  private void finishSingleSpillOrPipelined() throws IOException { /* PipelinedSorter.flush :730-772 */ }
  private String[] spillFilePaths() { return new String[numSpills]; }
  private String[] spillIndexPaths() { return new String[numSpills]; }

  // every native failure surfaces as IOException(tezgpu_last_error()), like the reference's own failures
  private static native long nativeCreate(int partitions, int comparator, int partitioner, boolean sendEmpty, long memory,
      int device, int sorterImpl) throws IOException;
  private static native void nativeCollect(long h, ByteBuffer kv, int bytes, IntBuffer keyOff, IntBuffer valOff,
      IntBuffer valLen, IntBuffer partition, int n) throws IOException;
  /** counters: [0] OUTPUT_BYTES_WITH_OVERHEAD [1] OUTPUT_BYTES_PHYSICAL [2] SPILLED_RECORDS [3] OUTPUT_RECORDS
   *  [4] OUTPUT_BYTES [5] rle used [6] adjacent equal keys [7] kernel launches */
  private static native void nativeFlush(long h, String out, String index, long[] idx, long[] counters) throws IOException;
  private static native void nativeReset(long h) throws IOException;
  private static native void nativeSetCombiner(long h, int combiner) throws IOException;
  private static native void nativeSetCodec(long h, int codec) throws IOException;
  /** tezgpu_sorter_set_split_points: split i = keys[off[i] .. off[i] + len[i]) */
  private static native void nativeSetSplitPoints(long h, ByteBuffer keys, long[] off, int[] len, int n, int order)
      throws IOException;
  private static native void nativeDestroy(long h);

  /** DataOutputStream target that appends to the direct batch buffer, making room through overflow(). */
  private final class BatchOutputStream extends java.io.OutputStream {
    @Override public void write(int v) throws IOException {
      if (!kv.hasRemaining()) overflow(1);
      kv.put((byte) v);
    }
    @Override public void write(byte[] a, int off, int len) throws IOException {
      if (kv.remaining() < len) overflow(len);
      kv.put(a, off, len);
    }
  }
}

/*
 * GpuMergeIterator -- TezMerger.merge(...) -> TezRawKeyValueIterator on the device (include/tezgpu.h, tezgpu_merge_*).
 *
 * Replaces the MergeQueue the reference builds at OG/MergeManager.java:804-811,899-903,1035-1041,1197-1199,1301-1319
 * and in PipelinedSorter.flush (:797-806).  NOT COMPILED IN THIS REPOSITORY (no JDK in the build image); the native side
 * is jni/tezgpu_jni.c.
 */
package org.apache.tez.runtime.library.common.sort.impl;

import java.io.IOException;
import java.nio.ByteBuffer;
import java.nio.ByteOrder;
import java.nio.IntBuffer;

import org.apache.hadoop.io.DataInputBuffer;
import org.apache.hadoop.util.Progress;

public final class GpuMergeIterator implements TezRawKeyValueIterator {
  static {
    System.loadLibrary("tezgpu_jni");
  }

  static final int SEG_HAS_HEADER = 1, SEG_DEVICE = 2, SEG_VERIFIED = 4;
  private static final int BATCH_BYTES = 8 << 20, BATCH_RECORDS = 1 << 16;

  private long handle; // tezgpu_merger*
  private long[] images; // decoded images of a budgeted merge (native memory, freed by close)
  // both grow to fit a record larger than BATCH_BYTES
  private ByteBuffer batch = ByteBuffer.allocateDirect(BATCH_BYTES).order(ByteOrder.nativeOrder());
  private final IntBuffer idx = ByteBuffer.allocateDirect(5 * 4 * BATCH_RECORDS).order(ByteOrder.nativeOrder()).asIntBuffer();
  private byte[] heap = new byte[BATCH_BYTES];   // DataInputBuffer wants a byte[]
  private final DataInputBuffer key = new DataInputBuffer(), value = new DataInputBuffer();
  private final Progress progress = new Progress();
  private int n, i = -1;

  /**
   * @param addresses  native addresses of the segments (in-memory byte[] pinned by the caller, or mapped file ranges)
   * @param lengths    segment lengths: header + body + 4 checksum bytes (partLength of the TezIndexRecord)
   * @param flags      SEG_HAS_HEADER for DiskSegments, 0 for InMemoryReader segments, | SEG_VERIFIED when the fetcher
   *                   already checked the CRC (IFile.Reader.readToMemory, IFile.java:764-809)
   * @param checkForSameKeys MergeQueue's constructor argument (TezMerger.java:560-573)
   */
  public GpuMergeIterator(long[] addresses, long[] lengths, int[] flags, int comparator, boolean checkForSameKeys)
      throws IOException {
    this(addresses, lengths, flags, null, GpuSorter.CODEC_NONE, comparator, checkForSameKeys);
  }

  /**
   * @param rawLengths rawLength of every segment (TezIndexRecord, or the ShuffleHeader's uncompressedLength); required
   *                   for the compressed ones ('T','I','F',1), may be null when none is compressed
   * @param codec      GpuSorter.codecId(CodecUtils.getCodec(conf)): CODEC_DEFAULT / CODEC_LZ4 / CODEC_ZSTD decompresses compressed segments on the
   *                   device, and writeFile then writes a compressed segment
   */
  public GpuMergeIterator(long[] addresses, long[] lengths, int[] flags, long[] rawLengths, int codec, int comparator,
      boolean checkForSameKeys) throws IOException {
    handle = nativeOpen(addresses, lengths, flags, null, 1, rawLengths, codec, comparator,
        Integer.parseInt(System.getenv().getOrDefault("TEZGPU_DEVICE", "0"))); // tezgpu_merge_open_codec
    if (!checkForSameKeys) nativeSetCheckForSameKeys(handle, false);
  }

  /**
   * MergeManager's final merge under tez.runtime.gpu.merge.device.budget.mb (INTEGRATION.md 2d): the merge holds at
   * most budgetBytes of device memory.  Compressed segments are first decoded on the device, in groups that fit the
   * budget, into native images of rawLength + 4 bytes that replace them (nativeDecodeSegments: tezgpu_decode_segments);
   * then every segment is merged in key-range steps (nativeOpenBounded: tezgpu_merge_open_bounded).  The segments must
   * be in host memory and stay valid until close(), which frees the images.
   */
  public GpuMergeIterator(long[] addresses, long[] lengths, int[] flags, long[] rawLengths, int codec, int comparator,
      boolean checkForSameKeys, long budgetBytes) throws IOException {
    final int device = Integer.parseInt(System.getenv().getOrDefault("TEZGPU_DEVICE", "0"));
    addresses = addresses.clone();
    lengths = lengths.clone();
    flags = flags.clone();
    images = new long[addresses.length];
    if (codec != GpuSorter.CODEC_NONE) {
      nativeDecodeSegments(addresses, lengths, flags, rawLengths, codec, budgetBytes, device, images);
      for (int s = 0; s < images.length; s++) {
        if (images[s] == 0) continue;
        addresses[s] = images[s];
        lengths[s] = rawLengths[s] + 4;
        flags[s] |= SEG_VERIFIED;   // the decode wrote the image's checksum from its bytes
      }
    }
    try {
      handle = nativeOpenBounded(addresses, lengths, flags, comparator, budgetBytes, device);
    } catch (IOException e) {
      nativeFreeImages(images);
      throw e;
    }
    if (!checkForSameKeys) nativeSetCheckForSameKeys(handle, false);
  }

  private GpuMergeIterator(long handle) {
    this.handle = handle;
  }

  /**
   * UnorderedPartitionedKVWriter.mergeAll (UnorderedPartitionedKVWriter.java:1058-1144) and UnorderedKVReader
   * (UnorderedKVReader.java:119-230): the segments concatenated, records in (segment, position) order, no comparator,
   * isSameKey() always false (tezgpu_concat_open).  partitions may be null for one partition.
   */
  public static GpuMergeIterator concat(long[] addresses, long[] lengths, int[] flags, int[] partitions, int numPartitions,
      long[] rawLengths, int codec) throws IOException {
    return new GpuMergeIterator(nativeConcatOpen(addresses, lengths, flags, partitions, numPartitions, rawLengths, codec,
        Integer.parseInt(System.getenv().getOrDefault("TEZGPU_DEVICE", "0"))));
  }

  /** file.out + file.out.index of every partition (tezgpu_merge_write_partitions); returns the 3 * P index triples. */
  public long[] writePartitions(String out, String index, int numPartitions, boolean writerRle) throws IOException {
    final long[] idx = new long[3 * numPartitions];
    nativeWritePartitions(handle, out, index, writerRle, idx);
    return idx;
  }

  /**
   * Combines the merged stream in writeIFile (PipelinedSorter's final merge from tez.runtime.combine.min.spills spills
   * on, PipelinedSorter.java:815-820); next() then fails: a combining merge has no record iterator.
   */
  public void setCombiner(int combiner) throws IOException {
    nativeSetCombiner(handle, combiner);
  }

  @Override
  public boolean next() throws IOException {
    if (++i >= n) {
      n = nativeNextBatch(handle, batch, batch.capacity(), idx, BATCH_RECORDS); // tezgpu_merge_next_batch
      if (n < 0) {
        // the next record alone needs -n bytes: grow both buffers and ask again (the stream has not moved)
        batch = ByteBuffer.allocateDirect(-n).order(ByteOrder.nativeOrder());
        heap = new byte[-n];
        n = nativeNextBatch(handle, batch, batch.capacity(), idx, BATCH_RECORDS);
      }
      i = 0;
      if (n > 0) {
        batch.position(0);
        batch.get(heap, 0, idx.get(5 * (n - 1) + 2) + idx.get(5 * (n - 1) + 3));
      }
    }
    return n > 0;
  }

  @Override public DataInputBuffer getKey() { key.reset(heap, idx.get(5 * i), idx.get(5 * i + 1)); return key; }
  @Override public DataInputBuffer getValue() { value.reset(heap, idx.get(5 * i + 2), idx.get(5 * i + 3)); return value; }
  @Override public boolean isSameKey() { return idx.get(5 * i + 4) != 0; }
  @Override public boolean hasNext() throws IOException { return i + 1 < n || nativeHasMore(handle); }
  @Override public Progress getProgress() { return progress; }

  /** TezMerger.writeFile(this, new IFile.Writer(..., rle)) collapses to one native call (TezMerger.java:215-245). */
  public long[] writeFile(String path, boolean writerRle) throws IOException {
    final long[] rawAndPart = new long[2];
    nativeWriteIFile(handle, path, writerRle, rawAndPart); // tezgpu_merge_write_ifile
    return rawAndPart;
  }

  @Override
  public void close() throws IOException {
    if (handle != 0) nativeClose(handle);
    if (images != null) nativeFreeImages(images);
    handle = 0;
    images = null;
  }

  /** PipelinedSorter.flush's final merge: all spills, all partitions, one device pass (PipelinedSorter.java:774-836). */
  static void mergeSpillsToFile(String[] spillFiles, String[] spillIndexFiles, int partitions, int comparator,
      boolean sendEmptyPartitionDetails, boolean checkForSameKeys, boolean writerRle, int codec, String out, String index)
      throws IOException {
    // tezgpu_merge_open_codec(P, the spills' rawLengths, codec) + set_check_for_same_keys + tezgpu_merge_write_partitions:
    // with CODEC_DEFAULT, CODEC_LZ4 or CODEC_ZSTD the compressed spills are read and file.out is written compressed
    nativeMergeSpills(spillFiles, spillIndexFiles, partitions, comparator, sendEmptyPartitionDetails, checkForSameKeys,
        writerRle, codec, out, index);
  }

  private static native long nativeOpen(long[] addresses, long[] lengths, int[] flags, int[] partitions, int numPartitions,
      long[] rawLengths, int codec, int comparator, int device) throws IOException;
  /** native address of a direct buffer (GetDirectBufferAddress), for the segment tables of the open calls */
  static native long nativeAddress(ByteBuffer direct);
  private static native long nativeOpenBounded(long[] addresses, long[] lengths, int[] flags, int comparator,
      long budgetBytes, int device) throws IOException;
  /** images[i] receives the native address of segment i's decoded image (malloc), 0 when it is not compressed */
  private static native void nativeDecodeSegments(long[] addresses, long[] lengths, int[] flags, long[] rawLengths,
      int codec, long budgetBytes, int device, long[] images) throws IOException;
  private static native void nativeFreeImages(long[] images);
  private static native long nativeConcatOpen(long[] addresses, long[] lengths, int[] flags, int[] partitions,
      int numPartitions, long[] rawLengths, int codec, int device) throws IOException;
  private static native void nativeWritePartitions(long h, String out, String index, boolean rle, long[] idx)
      throws IOException;
  private static native void nativeSetCheckForSameKeys(long h, boolean on) throws IOException;
  private static native void nativeSetCombiner(long h, int combiner) throws IOException;
  private static native int nativeNextBatch(long h, ByteBuffer out, int cap, IntBuffer idx, int idxCap) throws IOException;
  private static native boolean nativeHasMore(long h);
  private static native void nativeWriteIFile(long h, String path, boolean rle, long[] rawAndPart) throws IOException;
  private static native void nativeMergeSpills(String[] files, String[] indexFiles, int partitions, int comparator,
      boolean sendEmpty, boolean checkForSameKeys, boolean writerRle, int codec, String out, String index) throws IOException;
  private static native void nativeClose(long h);
}

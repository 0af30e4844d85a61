/*
 * GpuUnorderedKVReader -- UnorderedKVReader (RL/common/readers/UnorderedKVReader.java:119-230) over a concatenating
 * GpuMergeIterator (include/tezgpu.h, tezgpu_concat_open).
 *
 * Drop-in position: UnorderedKVInput.start() builds this reader instead of UnorderedKVReader once every input is
 * fetched; the fetched inputs (in-memory byte arrays or local file ranges) become the segment table of
 * GpuMergeIterator.concat in delivery order, the spills of one source in spill-id order.  The reference reads its
 * inputs in fetch-completion order, one at a time; the records of each input keep their order either way.
 * NOT COMPILED IN THIS REPOSITORY (no JDK in the build image); the native side is jni/tezgpu_jni.c.
 */
package org.apache.tez.runtime.library.common.readers;

import java.io.IOException;

import org.apache.hadoop.io.DataInputBuffer;
import org.apache.hadoop.io.serializer.Deserializer;
import org.apache.tez.runtime.library.api.KeyValueReader;
import org.apache.tez.runtime.library.common.sort.impl.GpuMergeIterator;

public class GpuUnorderedKVReader<K, V> extends KeyValueReader {
  private final GpuMergeIterator records;
  private final Deserializer<K> keyDeserializer;
  private final Deserializer<V> valDeserializer;
  private final DataInputBuffer keyIn = new DataInputBuffer(), valIn = new DataInputBuffer();
  private K key;
  private V value;
  private long numRecordsRead;

  /**
   * @param records         GpuMergeIterator.concat(...) over the fetched inputs, one partition
   * @param keyDeserializer / valDeserializer: opened on the reader's own buffers here, as UnorderedKVReader does (:88-96)
   */
  public GpuUnorderedKVReader(GpuMergeIterator records, Deserializer<K> keyDeserializer, Deserializer<V> valDeserializer)
      throws IOException {
    this.records = records;
    this.keyDeserializer = keyDeserializer;
    this.valDeserializer = valDeserializer;
    keyDeserializer.open(keyIn);
    valDeserializer.open(valIn);
  }

  /** KeyValueReader.next(): the next record of the concatenation (tezgpu_merge_next_batch, batched) */
  @Override
  public boolean next() throws IOException {
    if (!records.next()) {
      records.close();
      return false;
    }
    final DataInputBuffer k = records.getKey(), v = records.getValue();
    keyIn.reset(k.getData(), k.getPosition(), k.getLength() - k.getPosition());
    valIn.reset(v.getData(), v.getPosition(), v.getLength() - v.getPosition());
    key = keyDeserializer.deserialize(key);
    value = valDeserializer.deserialize(value);
    numRecordsRead++;   // INPUT_RECORDS_PROCESSED (UnorderedKVReader.next :107-110)
    return true;
  }

  @Override public Object getCurrentKey() { return key; }
  @Override public Object getCurrentValue() { return value; }
  public long getNumRecordsRead() { return numRecordsRead; }
}

/*
 * tez_runtime.h -- C API of the host-side mirror of the two Tez plugin classes that bound the hot path:
 *   OrderedPartitionedKVOutput  (RL/output/OrderedPartitionedKVOutput.java:91-218)
 *   OrderedGroupedKVInput       (RL/input/OrderedGroupedKVInput.java:95-317)
 * implemented in C++ (tez_b200/csrc/host/) on top of the tezgpu_* C ABI.  In a Tez deployment the unmodified Java
 * classes stay and only the ExternalSorter / TezMerger seam crosses JNI (INTEGRATION.md); this mirror exists because
 * the build image has no JVM, and lets the parity tests drive initialize/start/getWriter/close like the reference's
 * TestOnFileSortedOutput / TestOrderedGroupedKVInput do.  Same lifecycle, configuration keys
 * (RL/api/TezRuntimeConfiguration.java), file names (TezTaskOutputFiles), counters (TaskCounter) and event payloads
 * (ShufflePayloads.proto) as the reference.  Every function returns 0 or a TEZGPU_E_* code; tezrt_last_error() has
 * the message (the reference throws IOException / IllegalArgumentException at the same points).
 */
#ifndef TEZ_RUNTIME_H
#define TEZ_RUNTIME_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tezrt_output tezrt_output;
typedef struct tezrt_input tezrt_input;

const char *tezrt_last_error(void);

/* event types returned by close(): VertexManagerEvent / CompositeDataMovementEvent (ShuffleUtils.generateEventOnSpill, :409-441) */
#define TEZRT_EVENT_VERTEX_MANAGER 1
#define TEZRT_EVENT_COMPOSITE_DATA_MOVEMENT 2

/* ---- OutputContext + `new OrderedPartitionedKVOutput(outputContext, numPhysicalOutputs)` -------------------------
 * conf: newline separated key=value pairs (the UserPayload configuration, OrderedPartitionedKVOutput.java:93).
 * work_dir: OutputContext.getWorkDirs()[0]; unique_id: getUniqueIdentifier(); dest_vertex: getDestinationVertexName();
 * host/port: execution context host + shuffle service port; task_memory: getTotalMemoryAvailableToTask(). */
int32_t tezrt_output_create(const char *conf, const char *work_dir, const char *unique_id, const char *dest_vertex,
                            const char *host, int32_t shuffle_port, int64_t task_memory, int32_t num_physical_outputs,
                            int32_t device, tezrt_output **out);
/* `new UnorderedPartitionedKVOutput(outputContext, numPhysicalOutputs)` (partitioned = 1) or
 * `new UnorderedKVOutput(outputContext, numPhysicalOutputs)` (partitioned = 0: one writer partition,
 * RL/output/UnorderedKVOutput.java:107): the same output with the writer in TEZGPU_SORTER_UNORDERED mode
 * (RL/common/writers/UnorderedPartitionedKVWriter.java).  Every other tezrt_output_* call works on the handle.
 * initialize() requests tez.runtime.unordered.output.buffer.size-mb (> 0, :705-716); no combiner runs; close() writes
 * a single spill directly, concatenates several per partition with tezgpu_concat_open (current buffer first, then the
 * spills in order: mergeAll :1058-1144), or -- final merge off or tez.runtime.pipelined-shuffle.enabled -- sends one
 * event per spill with spill id and last-event flag (finalSpill :966-1006). */
int32_t tezrt_output_create_unordered(const char *conf, const char *work_dir, const char *unique_id, const char *dest_vertex,
                                      const char *host, int32_t shuffle_port, int64_t task_memory,
                                      int32_t num_physical_outputs, int32_t partitioned, int32_t device, tezrt_output **out);
/* initialize(): reads the configuration, requests the sort memory (requested = bytes passed to requestInitialMemory) */
int32_t tezrt_output_initialize(tezrt_output *o, int64_t *requested_memory);
/* MemoryUpdateCallback.memoryAssigned (the MemoryDistributor may grant less than requested) */
int32_t tezrt_output_memory_assigned(tezrt_output *o, int64_t granted);
/* start(): creates the sorter selected by tez.runtime.sorter.class (PIPELINED | LEGACY) */
int32_t tezrt_output_start(tezrt_output *o);
/* getWriter().write(key, value) with already serialized key / value bytes (KeyValuesWriter, :167-180).
 * partition < 0: the configured partitioner runs (HashPartitioner on the device); else the caller's Partitioner result. */
int32_t tezrt_output_write(tezrt_output *o, const uint8_t *key, uint32_t klen, const uint8_t *val, uint32_t vlen,
                           int32_t partition);
/* close(): flush + events. */
int32_t tezrt_output_close(tezrt_output *o, int32_t *num_events);
int32_t tezrt_output_event(tezrt_output *o, int32_t i, int32_t *type, const uint8_t **payload, uint64_t *payload_len,
                           int32_t *source_index_start, int32_t *count);
int64_t tezrt_output_counter(tezrt_output *o, const char *name);
int32_t tezrt_output_num_spills(tezrt_output *o);
/* The final merge over several spills, after close(): steps = 0 when none ran (one spill, or final merge off), 1 for a
 * one-step merge, else the key-range steps of the bounded merge; peak_device_bytes and h2d_bytes as
 * tezgpu_merge_bounded_info, 0 unless the merge ran under tez.runtime.gpu.merge.device.budget.mb.  That key (MiB; 0 or
 * unset: no budget; below 16: TEZGPU_E_INVALID at initialize) bounds the final merge of an ordered output without a
 * codec (tezgpu_merge_open_bounded); with a codec the final merge takes one step, as a bounded merge writes no
 * compressed output.  The unordered outputs concatenate and ignore it. */
int32_t tezrt_output_merge_info(tezrt_output *o, int32_t *steps, uint64_t *peak_device_bytes, uint64_t *h2d_bytes);
/* final file.out / file.out.index paths (ExternalSorter.getFinalOutputFile / getFinalIndexFile) */
const char *tezrt_output_file(tezrt_output *o);
const char *tezrt_output_index_file(tezrt_output *o);
int32_t tezrt_output_destroy(tezrt_output *o);

/* ---- InputContext + `new OrderedGroupedKVInput(inputContext, numPhysicalInputs)` ------------------------------- */
int32_t tezrt_input_create(const char *conf, const char *work_dir, const char *unique_id, int64_t task_memory,
                           int32_t num_physical_inputs, int32_t device, tezrt_input **out);
int32_t tezrt_input_initialize(tezrt_input *in, int64_t *requested_memory);
int32_t tezrt_input_start(tezrt_input *in);
/* handleEvents(DataMovementEvent) for a co-located producer: direct local-disk fetch of partition `partition` of the
 * producer's file.out through its index (OG/FetcherOrderedGrouped.java:697-771).  empty != 0: the producer reported
 * the partition empty in its event's bitmap (no fetch). */
int32_t tezrt_input_add_local_output(tezrt_input *in, int32_t source_index, const char *file_out,
                                     const char *index_file, int32_t partition, int32_t empty);
/* the same for a producer running with tez.runtime.enable.final-merge.in.output=false (pipelined shuffle): one event per
 * spill, carrying spill_id and last_event_flag (ShufflePayloads.proto DataMovementEventPayloadProto fields 9 and 8;
 * OG/ShuffleInputEventHandlerOrderedGrouped.java:225-240, OG/ShuffleScheduler.java:540-600).  The source counts as delivered once the event flagged last
 * and every spill id below it have arrived; duplicates are ignored. */
int32_t tezrt_input_add_local_spill(tezrt_input *in, int32_t source_index, const char *file_out, const char *index_file,
                                    int32_t partition, int32_t empty, int32_t spill_id, int32_t last_event);
/* waitForInputReady(): all physical inputs delivered -> final merge on the device */
int32_t tezrt_input_wait_ready(tezrt_input *in);
/* getReader(): KeyValuesReader.next() -> 1 when a new key group is available, 0 at the end */
int32_t tezrt_input_next(tezrt_input *in, const uint8_t **key, uint32_t *klen);
/* getCurrentValues() iteration: 1 and the next value of the current key, 0 when the group is exhausted */
int32_t tezrt_input_next_value(tezrt_input *in, const uint8_t **val, uint32_t *vlen);
/* ---- `new UnorderedKVInput(inputContext, numPhysicalInputs)` (RL/input/UnorderedKVInput.java): inputs are delivered
 * with tezrt_input_add_local_output / _add_local_spill; the first tezrt_input_next_kv (all inputs delivered) reads them
 * through tezgpu_concat_open in delivery order, the spills of one source in spill-id order (UnorderedKVReader reads
 * them in fetch-completion order, :119-230). */
int32_t tezrt_input_create_unordered(const char *conf, const char *work_dir, const char *unique_id, int64_t task_memory,
                                     int32_t num_physical_inputs, int32_t device, tezrt_input **out);
/* KeyValueReader.next() + getCurrentKey() / getCurrentValue(): 1 and the next record, 0 at the end */
int32_t tezrt_input_next_kv(tezrt_input *in, const uint8_t **key, uint32_t *klen, const uint8_t **val, uint32_t *vlen);
/* The merge behind the reader, after waitForInputReady: as tezrt_output_merge_info.  Under
 * tez.runtime.gpu.merge.device.budget.mb an OrderedGroupedKVInput decodes its compressed segments with
 * tezgpu_decode_segments, then merges every segment with tezgpu_merge_open_bounded under the same budget; the peak is
 * the larger of the two.  The stream and the counters are those of the merge without the key.  UnorderedKVInput
 * concatenates and ignores the key. */
int32_t tezrt_input_merge_info(tezrt_input *in, int32_t *steps, uint64_t *peak_device_bytes, uint64_t *h2d_bytes);
int64_t tezrt_input_counter(tezrt_input *in, const char *name);
int32_t tezrt_input_destroy(tezrt_input *in);

#ifdef __cplusplus
}
#endif
#endif

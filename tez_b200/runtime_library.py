"""Python face of the C++ host layer (tez_b200/csrc/host/, include/tez_runtime.h): the two plugin classes of the hot
path with the reference's names and lifecycle, so tests read like TestOnFileSortedOutput / TestOrderedGroupedKVInput.

    out = OrderedPartitionedKVOutput(OutputContext(...), numPhysicalOutputs)
    out.initialize(); out.start(); w = out.getWriter(); w.write(key_bytes, value_bytes); events = out.close()
    inp = OrderedGroupedKVInput(InputContext(...), numPhysicalInputs)
    inp.initialize(); inp.start(); inp.handleEvents([...]); r = inp.getReader()
    while r.next(): r.getCurrentKey(); list(r.getCurrentValues())

Keys / values are the serialized Writable bytes (serialization happens in the JVM in a real task).
"""
import ctypes as C
import zlib
from dataclasses import dataclass, field

from . import _lib
from ._lib import check_rt


def _merge_info(fn, h):
    steps, peak, h2d = C.c_int32(), C.c_uint64(), C.c_uint64()
    check_rt(fn(h, C.byref(steps), C.byref(peak), C.byref(h2d)))
    return steps.value, peak.value, h2d.value

TEXT = "org.apache.hadoop.io.Text"
INT_WRITABLE = "org.apache.hadoop.io.IntWritable"
LONG_WRITABLE = "org.apache.hadoop.io.LongWritable"
BYTES_WRITABLE = "org.apache.hadoop.io.BytesWritable"
TEZ_BYTES_COMPARATOR = "org.apache.tez.runtime.library.common.comparator.TezBytesComparator"
HASH_PARTITIONER = "org.apache.tez.runtime.library.partitioner.HashPartitioner"


def _conf_text(conf):
    return "\n".join("%s=%s" % (k, str(v).lower() if isinstance(v, bool) else v) for k, v in conf.items()).encode()


@dataclass
class OutputContext:
    """The slice of org.apache.tez.runtime.api.OutputContext the output uses."""
    conf: dict
    work_dir: str
    unique_identifier: str = "attempt_1_0001_1_00_000000_0_10001"
    destination_vertex_name: str = "consumer"
    host: str = "localhost"
    shuffle_port: int = 13562
    total_memory_available_to_task: int = 1 << 30
    device: int = 0
    memory_scale: float = 1.0        # MemoryDistributor may grant less than requested
    counters: dict = field(default_factory=dict)


@dataclass
class Event:
    type: str
    payload: bytes
    source_index_start: int = 0
    count: int = 0


def _varint(buf, pos):
    v = shift = 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        if b < 0x80:
            return v, pos
        shift += 7


def parse_proto(buf):
    """Minimal protobuf reader: {field: [values]} (varints as int, length-delimited as bytes)."""
    out, pos = {}, 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        f, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 2:
            n, pos = _varint(buf, pos)
            v = bytes(buf[pos:pos + n])
            pos += n
        else:
            raise ValueError("wire type %d" % wt)
        out.setdefault(f, []).append(v)
    return out


def empty_partitions_from_payload(payload, num_partitions):
    """DataMovementEventPayloadProto.empty_partitions -> set of partition ids (TezUtilsInternal.fromByteArray)."""
    p = parse_proto(payload)
    if 1 not in p:
        return set()
    bits = zlib.decompress(p[1][0], -15)
    n = len(bits)
    return {i for i in range(min(num_partitions, n * 8)) if bits[n - i // 8 - 1] >> (i % 8) & 1}


class KeyValuesWriter:
    def __init__(self, out):
        self._out = out

    def write(self, key, value_or_values, partition=-1):
        """write(key, value) / write(key, Iterable<value>) (KeyValuesWriter, OrderedPartitionedKVOutput.java:167-180)."""
        if isinstance(value_or_values, (bytes, bytearray)):
            value_or_values = (value_or_values,)
        L, h = self._out._L, self._out._h
        for v in value_or_values:
            check_rt(L.tezrt_output_write(h, key, len(key), v, len(v), partition))


class OrderedPartitionedKVOutput:
    def __init__(self, context, num_physical_outputs):
        self._L = _lib.load()
        self.context = context
        self.num_physical_outputs = num_physical_outputs
        self._h = C.c_void_p()
        c = context
        check_rt(self._create(_conf_text(c.conf), c.work_dir.encode(), c.unique_identifier.encode(),
                              c.destination_vertex_name.encode(), c.host.encode(), c.shuffle_port,
                              c.total_memory_available_to_task, num_physical_outputs, c.device, C.byref(self._h)))

    def _create(self, *args):
        return self._L.tezrt_output_create(*args)

    def initialize(self):
        req = C.c_int64()
        check_rt(self._L.tezrt_output_initialize(self._h, C.byref(req)))
        self.requested_memory = req.value
        # OutputContext.requestInitialMemory -> MemoryUpdateCallback.memoryAssigned
        check_rt(self._L.tezrt_output_memory_assigned(self._h, int(req.value * self.context.memory_scale)))
        return []

    def start(self):
        check_rt(self._L.tezrt_output_start(self._h))

    def getWriter(self):
        return KeyValuesWriter(self)

    def handleEvents(self, events):
        pass  # "Not expecting any events" (OrderedPartitionedKVOutput.java:183-186)

    def close(self):
        n = C.c_int32()
        check_rt(self._L.tezrt_output_close(self._h, C.byref(n)))
        events = []
        for i in range(n.value):
            t, p, ln, s, c = C.c_int32(), C.c_void_p(), C.c_uint64(), C.c_int32(), C.c_int32()
            check_rt(self._L.tezrt_output_event(self._h, i, C.byref(t), C.byref(p), C.byref(ln), C.byref(s), C.byref(c)))
            payload = C.string_at(p.value, ln.value) if ln.value else b""
            events.append(Event("VertexManagerEvent" if t.value == 1 else "CompositeDataMovementEvent", payload, s.value,
                                c.value))
        return events

    def counter(self, name):
        return self._L.tezrt_output_counter(self._h, name.encode())

    @property
    def num_spills(self):
        return self._L.tezrt_output_num_spills(self._h)

    def merge_info(self):
        """(steps, peak device bytes, bytes uploaded) of the final merge over the spills: steps 0 when none ran, 1 for a
        one-step merge; the bytes are 0 unless tez.runtime.gpu.merge.device.budget.mb bounded it."""
        return _merge_info(self._L.tezrt_output_merge_info, self._h)

    @property
    def final_output_file(self):
        return self._L.tezrt_output_file(self._h).decode()

    @property
    def final_index_file(self):
        return self._L.tezrt_output_index_file(self._h).decode()

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.tezrt_output_destroy(self._h)
            self._h = None


class UnorderedPartitionedKVOutput(OrderedPartitionedKVOutput):
    """The same output with the writer of UnorderedPartitionedKVWriter: partitioned, no key order, no combiner."""
    _partitioned = 1

    def _create(self, *args):
        return self._L.tezrt_output_create_unordered(*args[:-2], self._partitioned, *args[-2:])


class UnorderedKVOutput(UnorderedPartitionedKVOutput):
    """Broadcast / one-to-one output: one writer partition whatever numPhysicalOutputs is (UnorderedKVOutput.java:107)."""
    _partitioned = 0


@dataclass
class InputContext:
    conf: dict
    work_dir: str
    unique_identifier: str = "attempt_1_0001_1_01_000000_0_10002"
    total_memory_available_to_task: int = 1 << 30
    device: int = 0


@dataclass
class LocalOutput:
    """What a DataMovementEvent resolves to for a co-located producer (local-disk fetch)."""
    source_index: int
    file_out: str
    index_file: str
    partition: int
    empty: bool = False
    spill_id: int = -1          # >= 0: event of one spill of a producer without final merge (pipelined shuffle)
    last_event: bool = False


class KeyValuesReader:
    def __init__(self, inp):
        self._in = inp
        self._key = None

    def next(self):
        k, kl = C.c_void_p(), C.c_uint32()
        rc = self._in._L.tezrt_input_next(self._in._h, C.byref(k), C.byref(kl))
        if rc < 0:
            check_rt(rc)
        if rc == 0:
            return False
        self._key = C.string_at(k.value, kl.value) if kl.value else b""
        return True

    def getCurrentKey(self):
        return self._key

    def getCurrentValues(self):
        v, vl = C.c_void_p(), C.c_uint32()
        while True:
            rc = self._in._L.tezrt_input_next_value(self._in._h, C.byref(v), C.byref(vl))
            if rc < 0:
                check_rt(rc)
            if rc == 0:
                return
            yield C.string_at(v.value, vl.value) if vl.value else b""


class OrderedGroupedKVInput:
    def __init__(self, context, num_physical_inputs):
        self._L = _lib.load()
        self.context = context
        self._h = C.c_void_p()
        check_rt(self._create(_conf_text(context.conf), context.work_dir.encode(), context.unique_identifier.encode(),
                              context.total_memory_available_to_task, num_physical_inputs, context.device,
                              C.byref(self._h)))

    def _create(self, *args):
        return self._L.tezrt_input_create(*args)

    def initialize(self):
        req = C.c_int64()
        check_rt(self._L.tezrt_input_initialize(self._h, C.byref(req)))
        self.requested_memory = req.value
        return []

    def start(self):
        check_rt(self._L.tezrt_input_start(self._h))

    def handleEvents(self, local_outputs):
        for lo in local_outputs:
            spill_id = getattr(lo, "spill_id", -1)
            if spill_id is None or spill_id < 0:
                check_rt(self._L.tezrt_input_add_local_output(self._h, lo.source_index, lo.file_out.encode(),
                                                              lo.index_file.encode(), lo.partition, 1 if lo.empty else 0))
            else:   # pipelined shuffle: one event per spill of the producer
                check_rt(self._L.tezrt_input_add_local_spill(self._h, lo.source_index, lo.file_out.encode(),
                                                             lo.index_file.encode(), lo.partition, 1 if lo.empty else 0,
                                                             spill_id, 1 if getattr(lo, "last_event", False) else 0))

    def waitForInputReady(self):
        check_rt(self._L.tezrt_input_wait_ready(self._h))

    def getReader(self):
        self.waitForInputReady()
        return KeyValuesReader(self)

    def counter(self, name):
        return self._L.tezrt_input_counter(self._h, name.encode())

    def merge_info(self):
        """(steps, peak device bytes, bytes uploaded) of the merge behind the reader, after waitForInputReady; under
        tez.runtime.gpu.merge.device.budget.mb the peak covers the decode of compressed inputs too."""
        return _merge_info(self._L.tezrt_input_merge_info, self._h)

    def close(self):
        return []

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.tezrt_input_destroy(self._h)
            self._h = None


class KeyValueReader:
    """UnorderedKVReader: next() / getCurrentKey() / getCurrentValue(), every record in turn."""

    def __init__(self, inp):
        self._in = inp
        self._key = self._val = None

    def next(self):
        k, kl, v, vl = C.c_void_p(), C.c_uint32(), C.c_void_p(), C.c_uint32()
        rc = self._in._L.tezrt_input_next_kv(self._in._h, C.byref(k), C.byref(kl), C.byref(v), C.byref(vl))
        if rc < 0:
            check_rt(rc)
        if rc == 0:
            return False
        self._key = C.string_at(k.value, kl.value) if kl.value else b""
        self._val = C.string_at(v.value, vl.value) if vl.value else b""
        return True

    def getCurrentKey(self):
        return self._key

    def getCurrentValue(self):
        return self._val


class UnorderedKVInput(OrderedGroupedKVInput):
    """Reads every delivered input in turn, no merge: delivery order, the spills of one source in spill-id order."""

    def _create(self, *args):
        return self._L.tezrt_input_create_unordered(*args)

    def getReader(self):
        return KeyValueReader(self)

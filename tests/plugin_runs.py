"""Runs of the plugin classes the GPU tests share: one OrderedPartitionedKVOutput over a list of records, one
OrderedGroupedKVInput over producers' final outputs, and a file.out.index read back."""
import numpy as np

from tez_b200.runtime_library import (InputContext, LocalOutput, OrderedGroupedKVInput, OrderedPartitionedKVOutput,
                                      OutputContext, empty_partitions_from_payload)


def run_output(tmp, conf, records, P, uid="attempt_1_0001_1_00_000000_0_10001", mem=1 << 30):
    ctx = OutputContext(conf, str(tmp), unique_identifier=uid, total_memory_available_to_task=mem)
    out = OrderedPartitionedKVOutput(ctx, P)
    assert out.initialize() == []
    out.start()
    w = out.getWriter()
    for k, v in records:
        w.write(k, v)
    events = out.close()
    return out, events


def consume(tmp, conf, producers, partition, P):
    inp = OrderedGroupedKVInput(InputContext(conf, str(tmp)), len(producers))
    inp.initialize()
    inp.start()
    evs = []
    for i, (out, events) in enumerate(producers):
        empties = empty_partitions_from_payload(events[-1].payload, P)
        evs.append(LocalOutput(i, out.final_output_file, out.final_index_file, partition, empty=partition in empties))
    inp.handleEvents(evs)
    r = inp.getReader()
    groups = []
    while r.next():
        groups.append((r.getCurrentKey(), list(r.getCurrentValues())))
    return inp, groups


def read_index(path, P):
    return np.frombuffer(open(path, "rb").read()[:-8], dtype=">i8").reshape(P, 3)

"""Model of the device sampler for the tests: InputSampler.RandomSampler's contract as tezgpu_sample_keys states it, and
InputSampler.writePartitionFile's split rule (hadoop-mapreduce-client-core 3.4, restated from its public source, SURVEY
A.2), with Java's float arithmetic.

  sample   record i of a call has gid = gid_base + i and h = splitmix64(seed ^ gid) (& mask); it is a candidate when
           h < ceil(freq * 2^64) (every record at freq = 1); of more than max_samples candidates the max_samples smallest
           (h, gid) are kept, listed in gid order.
  select   the union of samples capped again to the max_samples smallest (h, gid), sorted under the comparator with ties
           by gid, then
             float stepSize = samples.length / (float) P;  int last = -1;
             for (int i = 1; i < P; ++i) {
               int k = Math.round(stepSize * i);
               while (last >= k && cmp(samples[last], samples[k]) == 0) ++k;
               emit samples[k];  last = k;
             }
           Math.round(float) is floor(x + 1/2) in exact arithmetic (halves toward +inf).  An empty sample with P > 1 or a
           k past the end raise SplitIndexError (Java: ArrayIndexOutOfBoundsException)."""
import math
from fractions import Fraction

import numpy as np

import sort_order_model as M

MASK64 = (1 << 64) - 1


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & MASK64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    return x ^ (x >> 31)


def threshold(freq):
    """None (every record) for freq = 1, else ceil(freq * 2^64) of the double freq, exactly."""
    assert 0.0 <= freq <= 1.0
    return None if freq == 1.0 else math.ceil(Fraction(freq) * (1 << 64))


def sample(n, seed, freq, max_samples, gid_base=0, mask=MASK64):
    """[(h, gid)] kept by one sample call, in gid order."""
    thr = threshold(freq)
    cand = []
    for i in range(n):
        g = gid_base + i
        h = splitmix64(seed ^ g) & mask
        if thr is None or h < thr:
            cand.append((h, g))
    if len(cand) > max_samples:
        cand = sorted(cand)[:max_samples]
    return sorted(cand, key=lambda t: t[1])


def java_round(x):
    """Math.round(float): the nearest integer, halves toward +inf (x: a float32 value)."""
    x = np.float32(x)
    f = math.floor(Fraction(float(x)))
    return f + (1 if Fraction(float(x)) - f >= Fraction(1, 2) else 0)


class SplitIndexError(IndexError):
    """writePartitionFile reading past the sample (ArrayIndexOutOfBoundsException)."""


def pick(sorted_content, P):
    """writePartitionFile's indices into a sorted sample; sorted_content[i] is the comparison key of sample i (equal
    comparison keys <=> cmp == 0)."""
    n = len(sorted_content)
    step = np.float32(np.float32(n) / np.float32(P))
    out, last = [], -1
    for i in range(1, P):
        k = java_round(np.float32(step * np.float32(i)))
        while last >= k and sorted_content[last] == sorted_content[k]:
            k += 1
        if k >= n:
            raise SplitIndexError("split %d reads sample %d of %d" % (i, k, n))
        out.append(k)
        last = k
    return out


def select(entries, P, max_samples, cmp):
    """entries: [(h, gid, key bytes)] of the union of samples.  Returns (split keys, chosen indices)."""
    if P == 1:
        return [], []
    kept = sorted(entries, key=lambda e: (e[0], e[1]))[:max_samples]
    kept.sort(key=lambda e: e[1])                                            # gid order: the stable sort's ties
    srt = sorted(kept, key=lambda e: M.content(cmp, e[2]))
    ks = pick([M.content(cmp, e[2]) for e in srt], P)
    return [srt[k][2] for k in ks], ks

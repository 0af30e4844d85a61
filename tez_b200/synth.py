"""Seeded, counter-based synthetic workloads (SURVEY.md 8d) generated directly with torch so that the benchmark
inputs can be produced in HBM (or pinned host memory) without shipping data.  Bit-identical to the oracle's
generators (tests/test_synth.py checks that on CPU)."""
import torch

_M1 = -0x61C8864680B583EB  # 0x9E3779B97F4A7C15 as int64
_M2 = -0x40A7B892E31B1A47  # 0xBF58476D1CE4E5B9
_M3 = -0x6B2FB644ECCEEE15  # 0x94D049BB133111EB


def _lsr(x, s):
    return (x >> s) & ((1 << (64 - s)) - 1)


def splitmix64(x):
    """x: int64 tensor (two's complement view of uint64). Wrap-around arithmetic == uint64 arithmetic."""
    x = x + _M1
    x = (x ^ _lsr(x, 30)) * _M2
    x = (x ^ _lsr(x, 27)) * _M3
    return x ^ _lsr(x, 31)


def _be_bytes(words):
    """int64 tensor [..., W] -> uint8 tensor [..., W*8] big-endian."""
    shifts = torch.arange(56, -8, -8, device=words.device, dtype=torch.int64)
    b = (words.unsqueeze(-1) >> shifts) & 0xFF
    return b.to(torch.uint8).reshape(*words.shape[:-1], -1)


def gen_c2(first_index, n, seed=2, device="cpu", out=None, chunk=1 << 22):
    """C2 records: 80 bytes = 16 B key (2 big-endian splitmix64 words) + 64 B value (8 words); word w of record i is
    splitmix64((seed << 56) ^ (16 * i + w)).  Returns a uint8 tensor of n*80 bytes."""
    if out is None:
        out = torch.empty(n * 80, dtype=torch.uint8, device=device)
    dev = out.device
    w = torch.arange(10, device=dev, dtype=torch.int64)
    sbits = (seed << 56)
    if sbits >= 1 << 63:
        sbits -= 1 << 64
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        i = torch.arange(first_index + s, first_index + s + m, device=dev, dtype=torch.int64)
        words = splitmix64((i.unsqueeze(1) * 16 + w) ^ sbits)
        out[s * 80:(s + m) * 80] = _be_bytes(words).reshape(-1)
    return out


def hash_bytes(keys):
    """WritableComparator.hashBytes over the rows of a uint8 tensor [n, L] -> int32-valued int64 tensor."""
    h = torch.ones(keys.shape[0], dtype=torch.int64, device=keys.device)
    sb = keys.to(torch.int64)
    sb = torch.where(sb > 127, sb - 256, sb)
    for j in range(keys.shape[1]):
        h = (h * 31 + sb[:, j]) & 0xFFFFFFFF
    return h


def hash_partition(keys, num_partitions):
    return (hash_bytes(keys) & 0x7FFFFFFF) % num_partitions


def zipf_ids(first_index, n, seed=5, s=1.1, num_ids=1 << 32, device="cpu"):
    """Record i -> an id in [0, num_ids) drawn Zipf(s) by inversion of the continuous approximation of the CDF
    (rank = (1 - u * (1 - N^(1-s)))^(1/(1-s)), u = splitmix64 counter in [0, 1)); int64 tensor.  Deterministic per device
    type; tests download the records they generated instead of re-deriving them on the host."""
    i = torch.arange(first_index, first_index + n, device=device, dtype=torch.int64)
    sbits = (seed << 56)
    if sbits >= 1 << 63:
        sbits -= 1 << 64
    u = (_lsr(splitmix64(i ^ sbits), 11)).to(torch.float64) * (1.0 / 9007199254740992.0)
    a = 1.0 - s
    rank = torch.pow(1.0 - u * (1.0 - float(num_ids) ** a), 1.0 / a)
    return torch.clamp(rank.to(torch.int64) - 1, 0, num_ids - 1)


WORD_MAX = 12
_WORD_REC = 1 + WORD_MAX + 4   # vint(length) + letters + IntWritable


def word_table(vocab, seed=7, s=1.1):
    """The vocabulary of gen_words, built on the host: (images uint8 [vocab, 17], lengths int64 [vocab], cdf int64
    [vocab]).  Word w has 3 + h_w % 10 lower-case letters, letter j = (splitmix64((seed << 56) ^ (16 * w + 1 + j)) >> 1) % 26
    with h_w the same hash at j = -1; its record image is the Text key (vint(length) + letters) followed by IntWritable(1).
    cdf[w] = floor(2^53 * sum_{v <= w} (v+1)^-s / sum_v (v+1)^-s): rank w is drawn with weight (w+1)^-s (Zipf)."""
    import numpy as np
    sbits = (seed << 56)
    if sbits >= 1 << 63:
        sbits -= 1 << 64
    w = torch.arange(vocab, dtype=torch.int64)
    j = torch.arange(WORD_MAX + 1, dtype=torch.int64)
    h = _lsr(splitmix64((w.unsqueeze(1) * 16 + j) ^ sbits), 1)
    lens = 3 + h[:, 0] % 10
    letters = (97 + h[:, 1:] % 26).to(torch.uint8)
    img = torch.zeros(vocab, _WORD_REC, dtype=torch.uint8)
    img[:, 0] = lens.to(torch.uint8)                  # vint of 3..12 is the byte itself
    pos = torch.arange(WORD_MAX, dtype=torch.int64)
    img[:, 1:1 + WORD_MAX] = torch.where(pos < lens.unsqueeze(1), letters, torch.zeros_like(letters))
    one = torch.tensor([0, 0, 0, 1], dtype=torch.uint8)
    for k in range(4):                                 # IntWritable(1) right behind the letters
        img[torch.arange(vocab), 1 + lens + k] = one[k]
    wt = (np.arange(1, vocab + 1, dtype=np.float64)) ** -s
    cdf = np.floor(np.cumsum(wt) / wt.sum() * float(1 << 53)).astype(np.int64)
    cdf[-1] = 1 << 53
    return img, lens + 5, torch.from_numpy(cdf)


def gen_words(first_index, n, seed=7, vocab=50000, device="cpu", s=1.1, table=None):
    """OrderedWordCount map output: record i is a Text key of the word of rank r_i (word_table) and IntWritable(1), where
    r_i = the first rank whose cdf exceeds splitmix64(((seed + 1) << 56) ^ i) >> 11 -- a Zipf(s) draw in integer
    arithmetic only, so the records are the same bytes on every device.  Records are packed back to back.  Returns
    (kv uint8, key_off int64, val_off int64, val_len int32) on `device`: the arrays GpuSorter.sort_device takes (the
    offsets are the uint64 values, the lengths the uint32 values), kv_bytes = kv.numel()."""
    img, rec_len, cdf = table if table is not None else word_table(vocab, seed, s)
    img, rec_len, cdf = img.to(device), rec_len.to(device), cdf.to(device)
    sbits = ((seed + 1) << 56) & ((1 << 64) - 1)
    if sbits >= 1 << 63:
        sbits -= 1 << 64
    i = torch.arange(first_index, first_index + n, device=device, dtype=torch.int64)
    u = _lsr(splitmix64(i ^ sbits), 11)
    rank = torch.clamp(torch.searchsorted(cdf, u, right=True), max=img.shape[0] - 1)
    size = rec_len[rank]
    key_off = torch.cumsum(size, 0) - size
    total = int(size.sum().item()) if n else 0
    kv = torch.empty(total, dtype=torch.uint8, device=device)
    for j in range(_WORD_REC):                         # byte j of every record that long
        m = size > j
        kv[(key_off + j)[m]] = img[rank[m], j]
    val_off = key_off + size - 4
    val_len = torch.full((n,), 4, dtype=torch.int32, device=device)
    return kv, key_off, val_off, val_len


def gen_c5(first_index, n, seed=5, val_len=4096, device="cpu", chunk=1 << 16):
    """BASELINE config 5 records (SURVEY 8d): key = 16 bytes rendered from a Zipf(1.1) id over 2^32 ids (two big-endian
    splitmix64 words of the id, so equal ids <=> equal keys and keys are spread over the partitions), value = val_len
    bytes, a pure function of the key.  Returns a uint8 tensor of n * (16 + val_len) bytes."""
    assert val_len % 8 == 0
    rec = 16 + val_len
    out = torch.empty(n * rec, dtype=torch.uint8, device=device)
    vw = torch.arange(val_len // 8, device=out.device, dtype=torch.int64)
    for s0 in range(0, n, chunk):
        m = min(chunk, n - s0)
        ids = zipf_ids(first_index + s0, m, seed=seed, device=out.device)
        k = torch.stack([splitmix64(ids * 2 + 0x1234567), splitmix64(ids * 2 + 0x7654321)], dim=1)
        v = splitmix64((ids.unsqueeze(1) << 10) ^ vw ^ 0x5A5A5A5A)
        view = out[s0 * rec:(s0 + m) * rec].view(m, rec)
        view[:, :16] = _be_bytes(k)
        view[:, 16:] = _be_bytes(v)
    return out

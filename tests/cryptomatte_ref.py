"""NumPy restatement of the Cryptomatte (include/vpt_b200.h: vpt_set_cryptomatte, vpt_cryptomatte_rank, vpt_cryptomatte_hash;
DESIGN.md section 8s).

State of one pixel: n (passes counted), overflow, and `capacity` entries (id, count).  Per pass at iteration it:
  1. it >= max_interactions: nothing changes (accum's gate);
  2. it == 0: the pixel is cleared first;
  3. n += 1;
  4. a sample with c = depth > 0 (NaN: false) adds its id to the entry that holds it (count > 0), else to the first entry with count 0,
     else to overflow.
Ranks: the non-empty entries by count descending, then instance index ascending, the sphere (SPHERE = 0xffffffff) last; rank r is
(id float, count / n) in float4 plane r // 2, components 2 (r % 2) and 2 (r % 2) + 1; ranks past the last entry and every rank of a pixel
with n == 0 are (0, 0)."""
import struct

import numpy as np

SPHERE = 0xFFFFFFFF
MAX_ENTRIES = 32


class PixelState:
    def __init__(self, capacity):
        assert 1 <= capacity <= MAX_ENTRIES
        self.capacity = capacity
        self.n = 0
        self.overflow = 0
        self.ids = [0] * capacity
        self.counts = [0] * capacity

    def clear(self):
        self.n = self.overflow = 0
        self.ids = [0] * self.capacity
        self.counts = [0] * self.capacity

    def add(self, sample_id):
        for j in range(self.capacity):
            if self.counts[j] > 0 and self.ids[j] == sample_id:
                self.counts[j] += 1
                return
        for j in range(self.capacity):
            if self.counts[j] == 0:
                self.ids[j], self.counts[j] = sample_id, 1
                return
        self.overflow += 1

    def words(self):
        """the 2 + 2 capacity state words of the pixel, in plane order"""
        w = [self.n, self.overflow]
        for j in range(self.capacity):
            w += [self.ids[j], self.counts[j]]
        return np.array(w, np.uint32)


def update(state, iteration, max_interactions, depths, ids):
    """a call at kp.iteration = `iteration` of len(depths) passes on one pixel: depths[p] the record's depth (0 for a pass that samples
    nothing or a culled pixel), ids[p] its id (read only where depth > 0)"""
    for p, d in enumerate(depths):
        it = iteration + p
        if it >= max_interactions:
            continue
        if it == 0:
            state.clear()
        state.n += 1
        if np.float32(d) > 0:
            state.add(int(ids[p]))
    return state


def rank_key(sample_id, count):
    """sort key: count descending, then instance index ascending, the sphere (the largest uint32) last"""
    return (-int(count), int(sample_id))


def ranks(state_words, capacity, id_table, sphere_id, n_ranks):
    """(n_ranks // 2, 4) float32 ranks of one pixel from its state words; id_table: float32 per instance"""
    assert n_ranks % 2 == 0 and 2 <= n_ranks <= 32
    w = np.asarray(state_words, np.uint32)
    n = int(w[0])
    out = np.zeros((n_ranks // 2, 4), np.float32)
    if n == 0:
        return out
    entries = [(int(w[2 + 2 * j]), int(w[3 + 2 * j])) for j in range(capacity) if int(w[3 + 2 * j]) > 0]
    entries.sort(key=lambda e: rank_key(*e))
    for r, (i, c) in enumerate(entries[:n_ranks]):
        if i == SPHERE:
            f = np.float32(sphere_id)
        elif i < len(id_table):
            f = np.float32(id_table[i])
        else:
            f = np.float32(0.0)
        out[r // 2, 2 * (r % 2)] = f
        out[r // 2, 2 * (r % 2) + 1] = np.float32(c) / np.float32(n)       # float32 division, rounded to nearest
    return out


def overflow_coverage(state_words):
    w = np.asarray(state_words, np.uint32)
    return np.float32(0.0) if int(w[0]) == 0 else np.float32(int(w[1])) / np.float32(int(w[0]))


def murmur3_32(data: bytes, seed=0):
    """MurmurHash3_x86_32 (Austin Appleby's public-domain algorithm)"""
    c1, c2, m = 0xCC9E2D51, 0x1B873593, 0xFFFFFFFF
    h = seed & m
    n4 = len(data) // 4
    for i in range(n4):
        k = int.from_bytes(data[4 * i:4 * i + 4], "little")
        k = (k * c1) & m
        k = ((k << 15) | (k >> 17)) & m
        k = (k * c2) & m
        h ^= k
        h = ((h << 13) | (h >> 19)) & m
        h = (h * 5 + 0xE6546B64) & m
    tail = data[4 * n4:]
    k = 0
    if len(tail) >= 3: k ^= tail[2] << 16
    if len(tail) >= 2: k ^= tail[1] << 8
    if len(tail) >= 1:
        k ^= tail[0]
        k = (k * c1) & m
        k = ((k << 15) | (k >> 17)) & m
        k = (k * c2) & m
        h ^= k
    h ^= len(data)
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & m
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & m
    h ^= h >> 16
    return h


def id_bits(h):
    """the Cryptomatte float's bits of hash h: bit 23 flipped when the exponent is 0 or 255 (no denormal, infinity or NaN)"""
    e = (h >> 23) & 0xFF
    return h ^ (1 << 23) if e in (0, 255) else h


def id_float(name: str):
    return struct.unpack("<f", struct.pack("<I", id_bits(murmur3_32(name.encode("utf-8")))))[0]


def manifest_hex(name: str):
    return "%08x" % id_bits(murmur3_32(name.encode("utf-8")))


def metadata_key(layer: str):
    """the <key> of the EXR header attributes cryptomatte/<key>/...: the first 7 hex digits of the layer name's hash"""
    return ("%08x" % murmur3_32(layer.encode("utf-8")))[:7]

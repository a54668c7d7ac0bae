"""CPU model of `mash sketch -r` as the streaming reads job computes it (DESIGN.md 2.6).

`ReferenceHeap` restates MinHashHeap (MinHashHeap.cpp:7-146) with its Bloom filter (bloom_filter.hpp as MinHashHeap constructs it:
one hash function, 8 b bits, one salt).  `sketch_reads_reference` pushes every k-mer of every kept record through it and applies the
stop test of Sketch.cpp:1258-1262 after each record; `sketch_reads_stretches` only replays the k-mers at or below the heap's top at
the start of each stretch of the k-mer stream, for arbitrary stretch boundaries -- the job's algorithm.  Both must agree.
"""
import hashlib
import heapq

import numpy as np

M32 = 0xFFFFFFFF
BLOOM_SALT = 0x9A0876E7
BLOOM_MAX_BITS = 1 << 32


def bloom_salt():
    """salt_[0] of bloom_filter(p) for one hash function and the default random_seed (bloom_filter.hpp:55, 183, 494-508)."""
    random_seed = (0xA5A5A5A55A5A5A5A * 0xA5A5A5A5 + 1) & 0xFFFFFFFFFFFFFFFF
    return (0xAAAAAAAA * 0xAAAAAAAA + random_seed) & M32


def hash_ap(key, use64, salt=BLOOM_SALT):
    """bloom_filter::hash_ap (bloom_filter.hpp:526-568) over the hash's 8 (use64) or 4 little-endian bytes."""
    h = salt
    if use64:
        i1, i2 = key & M32, (key >> 32) & M32
        h ^= ((h << 7) & M32) ^ ((i1 * (h >> 3)) & M32) ^ (~(((h << 11) + (i2 ^ (h >> 5))) & M32) & M32)
    else:
        h ^= ~(((h << 11) + ((key & M32) ^ (h >> 5))) & M32) & M32
    return h & M32


def bloom_bits(bloom_bytes):
    """Table size in bits: compute_optimal_parameters with false_positive_probability 0 ends at maximum_size = 8 b."""
    return 8 * bloom_bytes


def bloom_index(key, use64, bloom_bytes):
    """compute_indices: the 32-bit hash_ap modulo the table size (bloom_filter.hpp:443-447)."""
    return hash_ap(key, use64) % bloom_bits(bloom_bytes)


class ReferenceHeap:
    """MinHashHeap(use64, s, m, bloom_bytes).tryInsert, exactly (MinHashHeap.cpp:68-146)."""

    def __init__(self, s, m=1, bloom_bytes=0, use64=True):
        self.s, self.m, self.use64 = s, max(1, m), use64
        self.bloom_bytes = bloom_bytes
        self.bits = set() if bloom_bytes else None
        self.acc = {}                 # hashes with counts
        self.heap = []                # max-heap of acc (negated)
        self.pend = {}
        self.pheap = []               # max-heap of pending (negated), zombies included
        self.msum = 0

    def top(self):
        return -self.heap[0]

    def try_insert(self, h):
        if not (len(self.acc) < self.s or h < self.top()):
            return
        if h not in self.acc:
            if self.bits is not None:
                b = bloom_index(h, self.use64, self.bloom_bytes)
                if b in self.bits:
                    self.acc[h] = 2
                    heapq.heappush(self.heap, -h)
                    self.msum += 2
                else:
                    self.bits.add(b)
            elif self.m == 1 or self.pend.get(h, 0) == self.m - 1:
                self.acc[h] = self.m
                heapq.heappush(self.heap, -h)
                self.msum += self.m
                if self.m > 1:
                    self.pend.pop(h, None)
            else:
                if h not in self.pend:
                    heapq.heappush(self.pheap, -h)
                self.pend[h] = self.pend.get(h, 0) + 1
        else:
            self.acc[h] += 1
            self.msum += 1
        if len(self.acc) > self.s:
            t = self.top()
            self.msum -= self.acc.pop(t)
            while self.pheap and t < -self.pheap[0]:
                self.pend.pop(-self.pheap[0], None)
                heapq.heappop(self.pheap)
            heapq.heappop(self.heap)

    def gate(self):
        """Largest hash that can still pass the gate (2^64 - 1 while the heap is not full)."""
        return 0xFFFFFFFFFFFFFFFF if len(self.acc) < self.s else self.top()

    def stop(self, target_cov):
        return target_cov > 0 and len(self.acc) > 0 and self.msum / len(self.acc) >= target_cov

    def result(self):
        hs = np.array(sorted(self.acc), np.uint64)
        return hs, np.array([self.acc[int(h)] for h in hs], np.uint32)


def record_hashes(oracle, records, po):
    """getHash of every valid window of every kept record, in order (the records shorter than k are dropped)."""
    return [oracle.all_hashes(r, po) for r in records if len(r) >= po.kmer_size]


def sketch_reads_reference(hashes_per_record, s, m=1, bloom_bytes=0, target_cov=0.0, use64=True):
    """Every k-mer through the heap, the stop test after every record.  Returns (hashes, counts, records used)."""
    h = ReferenceHeap(s, m, bloom_bytes, use64)
    used = 0
    for hs in hashes_per_record:
        for x in hs.tolist():
            h.try_insert(x)
        used += 1
        if h.stop(target_cov):
            break
    return (*h.result(), used)


def sketch_reads_stretches(hashes_per_record, s, m=1, bloom_bytes=0, target_cov=0.0, use64=True, cuts=()):
    """The job's algorithm: the k-mer stream cut into stretches at the given k-mer indices; in each stretch only the k-mers at or
    below the gate as it stood at the stretch's start are events, replayed in order with the stop test due when an event that
    passes the gate falls into a later record, and at the end."""
    flat = np.concatenate(hashes_per_record) if hashes_per_record else np.zeros(0, np.uint64)
    rec = np.repeat(np.arange(len(hashes_per_record)), [x.size for x in hashes_per_record])
    bounds = [0] + sorted(c for c in set(cuts) if 0 < c < flat.size) + [flat.size]
    h = ReferenceHeap(s, m, bloom_bytes, use64)
    cur, events = None, 0
    for a, b in zip(bounds[:-1], bounds[1:]):
        sel = np.nonzero(flat[a:b] <= np.uint64(h.gate()))[0] + a
        events += sel.size
        for i in sel.tolist():
            x, r = int(flat[i]), int(rec[i])
            if not (len(h.acc) < h.s or x < h.top()):
                continue
            if cur is not None and r != cur:
                if h.stop(target_cov):
                    return (*h.result(), cur + 1, events)
            cur = r
            h.try_insert(x)
    if cur is not None and h.stop(target_cov):
        return (*h.result(), cur + 1, events)
    return (*h.result(), len(hashes_per_record), events)


def digest(hashes, counts, *extra):
    d = hashlib.sha256()
    d.update(np.ascontiguousarray(hashes, np.uint64).tobytes())
    d.update(np.ascontiguousarray(counts, np.uint32).tobytes())
    for e in extra:
        d.update(str(e).encode())
    return d.hexdigest()


def synth_reads(seed, genome_len, n_reads, read_len=150, err=0.01, n_frac=0.02):
    """Reads with substitutions (and the odd N) sampled from a seeded random genome."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    g = acgt[rng.integers(0, 4, genome_len)]
    starts = rng.integers(0, genome_len - read_len, n_reads)
    out = []
    for a in starts.tolist():
        r = g[a:a + read_len].copy()
        mk = rng.random(read_len) < err
        r[mk] = acgt[rng.integers(0, 4, int(mk.sum()))]
        if rng.random() < n_frac:
            r[int(rng.integers(0, read_len))] = ord("N")
        out.append(bytes(r))
    return out

"""CPU model of the best-hit protocol of dist (mash_b200/csrc/dist_best.cuh and mashgpu_dist_run_best_dev in dist.cu), step for
step in numpy: the streaming selection of dist_best_kernel's long-segment path, and the host's block-halving driver."""
import numpy as np

INF = (np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64(0xFFFFFFFF), np.int64(-1))
TILE = 1024
STEP = 256          # BEST_THREADS: candidates looked at between two looks at the tile's fill


def _less(da, ra, db, rb):
    return (da < db) | ((da == db) & (ra < rb))


class Keys:
    """An array of (distance bits, reference, index in the segment) keys, as the kernel's s_key."""

    def __init__(self, n):
        self.d = np.full(n, INF[0], np.uint64); self.r = np.full(n, INF[1], np.uint64); self.i = np.full(n, INF[2], np.int64)

    def cmpx(self, lo, hi, asc):
        """compare-exchange of the pairs (lo[t], hi[t]): afterwards lo <= hi where asc[t], lo >= hi elsewhere"""
        swap = _less(self.d[hi], self.r[hi], self.d[lo], self.r[lo]) == asc
        a, b = lo[swap], hi[swap]
        for arr in (self.d, self.r, self.i):
            arr[a], arr[b] = arr[b].copy(), arr[a].copy()


def _pairs(n, j):
    t = np.arange(n // 2)
    lo = ((t & ~(j - 1)) << 1) | (t & (j - 1))
    return lo, lo | j


def select_streaming(dbits, ref, n_best):
    """dist_best_kernel's CTA path on one segment.  Returns the segment indices of the n_best smallest (dbits, ref), in rank
    order, and the number of tile flushes."""
    cnt = dbits.size
    kw = 1
    while kw < n_best:
        kw <<= 1
    kept, tile = Keys(kw), Keys(TILE)
    thresh = (INF[0], INF[1])
    fill = flushes = 0
    for base in range(0, cnt, STEP):
        idx = np.arange(base, min(cnt, base + STEP))
        ok = _less(dbits[idx], ref[idx].astype(np.uint64), thresh[0], thresh[1])
        take = idx[ok]
        tile.d[fill:fill + take.size] = dbits[take]; tile.r[fill:fill + take.size] = ref[take]; tile.i[fill:fill + take.size] = take
        fill += take.size
        assert fill <= TILE
        if fill == 0 or (fill + STEP <= TILE and base + STEP < cnt):
            continue
        flushes += 1
        n2 = 2
        while n2 < fill:
            n2 <<= 1
        tile.d[fill:n2] = INF[0]; tile.r[fill:n2] = INF[1]; tile.i[fill:n2] = INF[2]
        k = 2
        while k <= n2:                                  # bitonic sort, descending
            j = k >> 1
            while j > 0:
                lo, hi = _pairs(n2, j)
                tile.cmpx(lo, hi, (lo & k) != 0)
                j >>= 1
            k <<= 1
        t = np.arange(kw)
        src = t + n2 - kw
        t, src = t[src >= 0], src[src >= 0]
        win = _less(tile.d[src], tile.r[src], kept.d[t], kept.r[t])
        kept.d[t[win]] = tile.d[src[win]]; kept.r[t[win]] = tile.r[src[win]]; kept.i[t[win]] = tile.i[src[win]]
        j = kw >> 1
        while j > 0:                                    # bitonic merge, ascending
            lo, hi = _pairs(kw, j)
            kept.cmpx(lo, hi, np.ones(lo.size, bool))
            j >>= 1
        thresh = (kept.d[n_best - 1], kept.r[n_best - 1])
        fill = 0
    return kept.i[:min(cnt, n_best)], flushes


def run_blocks(q_count, n_ref, capacity, block0, capture):
    """The host loop of mashgpu_dist_run_best_dev.  capture(q0, qn) -> number of hits of the queries [q0, q0 + qn).  Returns
    (blocks selected, in order; blocks discarded and split; blocks run)."""
    capacity = max(capacity, n_ref)
    todo = [(q * block0, min(block0, q_count - q * block0)) for q in reversed(range((q_count + block0 - 1) // block0))]
    done, splits, runs = [], 0, 0
    while todo:
        b0, bn = todo.pop()
        cap = min(capacity, bn * n_ref)
        n = capture(b0, bn)
        runs += 1
        if n > cap:
            assert bn >= 2
            splits += 1
            todo.append((b0 + bn // 2, bn - bn // 2))
            todo.append((b0, bn // 2))
            continue
        done.append((b0, bn))
    return done, splits, runs

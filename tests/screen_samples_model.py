"""numpy model of the screen's sparse finish (mashgpu_screen_finish_hits, DESIGN.md 4.3) next to the dense definition it must
equal (screen_reduce_kernel and the host-ordered -w of mashgpu_screen_finish).

A table is (ref, ref_n): row r holds ref_n[r] ascending hashes.  A sample is cnt: the hit counter of every distinct reference hash,
in ascending hash order (the job's counter layout)."""
import functools

import numpy as np


def pairs(ref, ref_n):
    """(distinct hashes ascending, sketch of every pair, distinct index of every pair), pairs in row-major order."""
    n = len(ref_n)
    pair_r = np.repeat(np.arange(n, dtype=np.int64), np.asarray(ref_n, np.int64))
    pair_h = np.concatenate([ref[r, :ref_n[r]] for r in range(n)]) if n else np.zeros(0, np.uint64)
    distinct = np.unique(pair_h)
    return distinct, pair_r, np.searchsorted(distinct, pair_h)


def identity_score(shared, n, k):
    """estimateIdentity as the host evaluates it for the -w order (C pow, as Python's float ** calls it)."""
    if shared == n:
        return 1.0
    if shared == 0:
        return 0.0
    return (shared / n) ** (1.0 / k)


def dense(ref, ref_n, cnt, k, winner=False, lengths=None):
    """Every sketch: shared, median as screen_reduce_kernel computes them (after the -w reallocation when winner)."""
    n = len(ref_n)
    distinct, pair_r, pair_d = pairs(ref, ref_n)
    c = np.asarray(cnt, np.int64)[pair_d]
    seen = c >= 1
    keep = seen
    if winner:
        lengths = np.zeros(n, np.uint64) if lengths is None else np.asarray(lengths, np.uint64)
        plain = np.bincount(pair_r[seen], minlength=n)
        score = [identity_score(int(plain[r]), int(ref_n[r]), k) for r in range(n)]
        order = sorted(range(n), key=lambda r: (-score[r], -int(lengths[r]), r))
        prio = np.empty(n, np.int64)
        prio[order] = np.arange(n)
        best = np.full(distinct.size, np.iinfo(np.int64).max)
        np.minimum.at(best, pair_d[seen], prio[pair_r[seen]])
        keep = seen & (best[pair_d] == prio[pair_r])
    shared = np.zeros(n, np.uint64)
    median = np.zeros(n, np.uint64)
    for r in range(n):
        depths = np.sort(c[keep & (pair_r == r)])
        shared[r] = depths.size
        median[r] = depths[depths.size // 2] if depths.size else 0
    return dict(shared=shared, median=median)


def build_index(ref, ref_n):
    """Inverted index: seg_ref[seg_start[d]:seg_start[d + 1]] = the sketches holding distinct hash d (a counting sort by d)."""
    distinct, pair_r, pair_d = pairs(ref, ref_n)
    seg_n = np.bincount(pair_d, minlength=distinct.size)
    seg_start = np.concatenate([[0], np.cumsum(seg_n)]).astype(np.int64)
    seg_ref = pair_r[np.argsort(pair_d, kind="stable")]
    return dict(distinct=distinct, seg_start=seg_start, seg_ref=seg_ref, n_ref=len(ref_n))


def exact_before(a, b, shared, n_hashes, lengths):
    """-w order of two hit sketches: shared / n descending by 64-bit cross-multiplication, then length descending, then index."""
    x, y = int(shared[a]) * int(n_hashes[b]), int(shared[b]) * int(n_hashes[a])
    if x != y:
        return -1 if x > y else 1
    if lengths[a] != lengths[b]:
        return -1 if lengths[a] > lengths[b] else 1
    return -1 if a < b else (1 if a > b else 0)


def sparse(index, cnt, ref_n, winner=False, lengths=None):
    """The rows of the sparse finish: sketches with shared >= 1 ascending, their shared and median, and the stats
    (hit hashes, expanded pairs)."""
    n = index["n_ref"]
    seg_start, seg_ref = index["seg_start"], index["seg_ref"]
    cnt = np.asarray(cnt, np.int64)
    hit = np.flatnonzero(cnt >= 1)
    seg_len = seg_start[hit + 1] - seg_start[hit]
    pair_r = np.concatenate([seg_ref[seg_start[d]:seg_start[d + 1]] for d in hit]) if hit.size else np.zeros(0, np.int64)
    pair_c = np.repeat(cnt[hit], seg_len)
    stats = dict(hit_hashes=int(hit.size), hit_pairs=int(pair_r.size))
    if winner:
        lengths = np.zeros(n, np.uint64) if lengths is None else np.asarray(lengths, np.uint64)
        plain = np.bincount(pair_r, minlength=n)
        hit_refs = np.flatnonzero(plain > 0)
        order = sorted(hit_refs.tolist(), key=functools.cmp_to_key(lambda a, b: exact_before(a, b, plain, ref_n, lengths)))
        prio = np.full(n, -1, np.int64)
        prio[order] = np.arange(len(order))
        best = np.array([prio[seg_ref[seg_start[d]:seg_start[d + 1]]].min() for d in hit], np.int64)
        assert np.all(best >= 0)                         # every sketch of a hit segment is ranked
        pair_r = np.asarray(order, np.int64)[best] if hit.size else np.zeros(0, np.int64)
        pair_c = cnt[hit]
    # counting sort of the pairs by sketch: per-sketch runs, each sorted for its median
    run_n = np.bincount(pair_r, minlength=n)
    rows = np.flatnonzero(run_n > 0)
    by_ref = pair_c[np.argsort(pair_r, kind="stable")]
    start = np.concatenate([[0], np.cumsum(run_n)])
    median = np.array([np.sort(by_ref[start[r]:start[r + 1]])[run_n[r] // 2] for r in rows], np.uint64)
    return dict(ref=rows, shared=run_n[rows].astype(np.uint64), median=median), stats

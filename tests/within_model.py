"""Checker for `mash within` (TEST INFRASTRUCTURE, never imported by the product).

  contain_closed_form  the rule the kernels implement (DESIGN.md 3.6), in numpy: containSketches(R, Q) of CommandContain.cpp:231-265
                       examines j_end = min(min(|R|, |Q|), #{t : Q[t] <= R[-1]}) query hashes (0 for an empty R) and counts
                       common = |Q[0 .. j_end) n R|; score = common / j_end, error = 1 / sqrt(j_end).
  RefContain           the reference's own containSketches (oracle/_ref/libmash_ref_contain.so, built in place by
                       oracle/contain.mk) over a query-major grid, on threads.
  edge_rows            hash rows that exercise every stop of the reference's loop.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libmash_ref_contain.so")
NEG_NAN = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]     # x86 result of 0.0 / 0 (sign bit set)

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)
f64p = C.POINTER(C.c_double)


def contain_closed_form(R, Q):
    """(common, examined) of containSketches(R, Q) for two ascending distinct hash arrays."""
    R = np.asarray(R, np.uint64)
    Q = np.asarray(Q, np.uint64)
    denom = min(R.size, Q.size)
    if R.size == 0 or denom == 0:
        return 0, 0
    j_end = min(denom, int(np.searchsorted(Q, R[-1], side="right")))
    common = int(np.isin(Q[:j_end], R, assume_unique=True).sum())
    return common, j_end


def score_error(common, examined):
    """The reference's doubles: score = common / j (the x86 NaN for j = 0), error = 1 / sqrt(j)."""
    common = np.asarray(common, np.float64)
    j = np.asarray(examined, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        score = np.where(j > 0, common / np.where(j > 0, j, 1), NEG_NAN)
        error = 1.0 / np.sqrt(j)
    return score, error


def grid_closed_form(ref, ref_n, qry, qry_n):
    """(common, examined) arrays of shape (n_qry, n_ref)."""
    nq, nr = len(qry_n), len(ref_n)
    common = np.zeros((nq, nr), np.uint32)
    examined = np.zeros((nq, nr), np.uint32)
    for q in range(nq):
        Q = qry[q, :qry_n[q]]
        for r in range(nr):
            common[q, r], examined[q, r] = contain_closed_form(ref[r, :ref_n[r]], Q)
    return common, examined


class RefContain:
    """The reference's own containSketches over a grid of pairs."""

    @staticmethod
    def available():
        return os.path.exists(REF_LIB)

    def __init__(self):
        self.lib = L = C.CDLL(REF_LIB)
        L.ref_contain_grid.restype = None
        L.ref_contain_grid.argtypes = [u64p, u32p, C.c_uint64, C.c_uint64, u64p, u32p, C.c_uint64, C.c_uint64,
                                       C.c_uint64, C.c_uint64, C.c_int, C.c_int, f64p, f64p]

    def grid(self, ref, ref_n, qry, qry_n, pair_begin=0, pair_count=None, use64=True, threads=1):
        """score, error of pairs [pair_begin, pair_begin + pair_count) of the query-major grid (p = q * n_ref + r)."""
        ref = np.ascontiguousarray(ref, np.uint64)
        qry = np.ascontiguousarray(qry, np.uint64)
        ref_n = np.ascontiguousarray(ref_n, np.uint32)
        qry_n = np.ascontiguousarray(qry_n, np.uint32)
        if ref.ndim == 1:
            ref = ref.reshape(-1, 1)
        if qry.ndim == 1:
            qry = qry.reshape(-1, 1)
        n_ref, n_qry = ref_n.size, qry_n.size
        if pair_count is None:
            pair_count = n_ref * n_qry - pair_begin
        score = np.zeros(pair_count, np.float64)
        error = np.zeros(pair_count, np.float64)
        self.lib.ref_contain_grid(ref.ctypes.data_as(u64p), ref_n.ctypes.data_as(u32p), ref.shape[1], n_ref,
                                  qry.ctypes.data_as(u64p), qry_n.ctypes.data_as(u32p), qry.shape[1], n_qry,
                                  pair_begin, pair_count, int(use64), int(threads), score.ctypes.data_as(f64p),
                                  error.ctypes.data_as(f64p))
        return score, error

    def pair(self, R, Q, use64=True):
        R = np.asarray(R, np.uint64)
        Q = np.asarray(Q, np.uint64)
        s, e = self.grid(np.pad(R, (0, 1)).reshape(1, -1), [R.size], np.pad(Q, (0, 1)).reshape(1, -1), [Q.size], use64=use64)
        return s[0], e[0]


def examined_from_error(error):
    """j from the reference's error = 1 / sqrt(j) (exact: j < 2^26); 0 where error is inf."""
    e = np.asarray(error, np.float64)
    with np.errstate(divide="ignore"):
        j = np.where(np.isinf(e), 0, np.rint(1.0 / (e * e)))
    return j.astype(np.int64)


def pack_rows(rows, stride=None):
    """list of 1-d hash arrays -> (n x stride) uint64 matrix (padding 2^64-1) and n_hashes."""
    n = np.array([len(r) for r in rows], np.uint32)
    stride = max(1, int(n.max()) if n.size else 1) if stride is None else stride
    H = np.full((len(rows), stride), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    for i, r in enumerate(rows):
        H[i, :len(r)] = np.asarray(r, np.uint64)
    return H, n


def edge_rows(rng, hi=2**64, size=40):
    """Rows covering each stop of the loop: empty, one hash, R below / above Q, ties at R's last hash, |R| > |Q| and < |Q|,
    identical rows, hashes 0 and 2^64-1 (hi = 2^32 for 32-bit lists)."""
    top = hi - 1

    def draw(m, lo=0, up=top):
        return np.unique(rng.integers(lo, up, m, dtype=np.uint64, endpoint=True))

    base = draw(size)
    rows = [
        np.zeros(0, np.uint64),                        # empty
        base[:1],                                      # one hash
        base.copy(),                                   # identical to base
        base[::2].copy(),                              # |R| < |Q| and a subset
        np.union1d(base, draw(size // 2)),             # |R| > |Q|
        draw(size, 0, hi // 8),                        # entirely low
        draw(size, hi - hi // 8, top),                 # entirely high
        np.union1d(draw(size // 2), np.array([0], np.uint64)),          # hash 0
        np.union1d(draw(size // 2), np.array([top], np.uint64)),        # hash 2^64-1 (or 2^32-1)
        np.union1d(base[: size // 3], draw(size // 3, hi // 2, top)),   # shares a prefix, then diverges
        base[base.size // 2:].copy(),                  # the upper half: R entirely above Q's first hashes
        np.union1d(draw(5), base[-1:]),                # a tie at the last hash of base
        np.array([0, top], np.uint64),                 # both extremes
        np.array([top], np.uint64),
        np.array([0], np.uint64),
    ]
    return rows

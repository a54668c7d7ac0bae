"""Greedy dereplication (mashgpu_dist_representatives, DESIGN.md 3.12) in numpy.

The graph is given as edges (i, j, d) with j < i: the pairs (q = i, r = j) of a self job with pass == 1 and numer > 0, at distance d.
- sequential(): the definition.  for v = 0 .. n-1, v is a representative iff no representative u < v has an edge {u, v}.
- device(): the device algorithm restated: sketch 0 first, then blocks of `block` rows from row 1; covered flags from the final status of
  earlier blocks, the block's own edges, and the rounds of Blelloch, Fineman and Shun, each reading the sets of the round before.
- assign(): every member's representative, the adjacent one with the least key (distance, min, max), the spanning forest's order.
"""
import numpy as np


def edges_from_grid(grid):
    """the graph of a dense grid of a self job (DistJob.run(0, n)): (i, j, distance) for j < i with pass and numer > 0"""
    hit = grid["pass"].astype(bool) & (grid["numer"] > 0)
    i, j = np.nonzero(hit)
    keep = j < i
    i, j = i[keep], j[keep]
    return i, j, grid["distance"][i, j]


def _earlier(n, i, j):
    """CSR of every row's earlier neighbours"""
    o = np.argsort(i, kind="stable")
    start = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(i, minlength=n), out=start[1:])
    return start, np.asarray(j)[o]


def sequential(n, i, j):
    """the representatives by the definition: a bool array of n"""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    start, nb = _earlier(n, i, j)
    is_rep = np.zeros(n, bool)
    for v in range(n):
        is_rep[v] = not is_rep[nb[start[v]:start[v + 1]]].any()
    return is_rep


def device(n, i, j, block=None):
    """the device algorithm with pass-1 blocks of `block` rows (None: all rows in one block).  Returns (is_rep, rounds per block)."""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    is_rep = np.zeros(n, bool)
    if n:
        is_rep[0] = True
    block = max(n - 1, 1) if block is None else block
    rounds = []
    for q0 in range(1, n, block):
        rows = min(block, n - q0)
        inside = (i >= q0) & (i < q0 + rows)
        bi, bj = i[inside], j[inside]
        covered = np.zeros(rows, bool)
        before = bj < q0
        covered[bi[before][is_rep[bj[before]]] - q0] = True
        a, b = bi[~before] - q0, bj[~before] - q0                  # bit (a, b) of the block's matrix, b < a
        state = np.where(covered, 2, 0)                             # 0 undecided, 1 in, 2 out
        r = 0
        while (state == 0).any():
            assert r < rows, "more rounds than rows"
            live = state[a] == 0
            la, lb = a[live], b[live]
            has_in = np.bincount(la, weights=state[lb] == 1, minlength=rows) > 0
            has_und = np.bincount(la, weights=state[lb] == 0, minlength=rows) > 0
            und = state == 0
            new = state.copy()
            new[und & has_in] = 2
            new[und & ~has_in & ~has_und] = 1
            state = new
            r += 1
        rounds.append(r)
        is_rep[q0:q0 + rows] = state == 1
    return is_rep, rounds


def assign(n, is_rep, i, j, d):
    """(rep, edge): rep[m] = the representative of member m, the adjacent one with the least (d, j, i); rep[v] = v for a representative.
    edge[m] = index of that edge in (i, j, d), -1 for a representative."""
    i, j, d = np.asarray(i, np.int64), np.asarray(j, np.int64), np.asarray(d, np.float64)
    rep, edge = np.arange(n, dtype=np.int64), np.full(n, -1, np.int64)
    cross = np.flatnonzero(is_rep[i] != is_rep[j])
    m = np.where(is_rep[i[cross]], j[cross], i[cross])
    o = np.lexsort((i[cross], j[cross], d[cross], m))               # by member, then the key
    m, e = m[o], cross[o]
    first = np.r_[True, m[1:] != m[:-1]] if m.size else np.zeros(0, bool)
    m, e = m[first], e[first]
    edge[m] = e
    rep[m] = np.where(i[e] == m, j[e], i[e])
    return rep, edge


def from_grid(grid, block=None):
    """the outputs of DistJob.representatives() from a dense grid of the same job, the device algorithm at `block`"""
    n = grid["numer"].shape[0]
    i, j, d = edges_from_grid(grid)
    is_rep, rounds = device(n, i, j, block)
    rep, edge = assign(n, is_rep, i, j, d)
    q, r = np.maximum(np.arange(n), rep), np.minimum(np.arange(n), rep)
    out = {"rep": rep.astype(np.uint32)}
    for k in ("numer", "denom", "distance", "pvalue"):
        v = grid[k][q, r].copy()
        v[is_rep] = 0
        out[k] = v
    out["n_reps"] = int(is_rep.sum())
    out["rounds"] = int(sum(rounds))
    return out

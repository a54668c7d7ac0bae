"""Models of the minimum spanning forest of dist (mashgpu_dist_spanning_forest, DESIGN.md 3.9).

Edges {row, col} (col < row) are ordered by the strict total order (distance, col, row).  `kruskal` is the definition; `boruvka` restates
the device rounds in numpy (per-component cheapest edge, the mutual-pick skip, the larger root hooked under the smaller one, then a
flatten) and counts them.  Both return edge indices in forest order."""
import numpy as np


def edge_order(row, col, dist):
    """edge indices sorted by (distance, col, row)"""
    return np.lexsort((np.asarray(row), np.asarray(col), np.asarray(dist, np.float64)))


def _find(parent, x):
    while parent[x] != x:
        parent[x] = parent[parent[x]]
        x = parent[x]
    return x


def kruskal(n, row, col, dist):
    parent = list(range(n))
    out = []
    for e in edge_order(row, col, dist):
        a, b = _find(parent, int(row[e])), _find(parent, int(col[e]))
        if a != b:
            parent[max(a, b)] = min(a, b)
            out.append(int(e))
    return np.array(out, np.int64)


def boruvka(n, row, col, dist):
    """(forest edge indices in forest order, rounds run) as the device computes them"""
    row = np.asarray(row, np.int64)
    col = np.asarray(col, np.int64)
    m = row.size
    rank = np.empty(m, np.int64)
    rank[edge_order(row, col, dist)] = np.arange(m)
    none = m
    label = np.arange(n)
    parent = list(range(n))
    picked, rounds = [], 0
    while n >= 2 and len(picked) < n - 1:
        a, b = label[row], label[col]
        live = a != b
        best = np.full(n, none, np.int64)
        np.minimum.at(best, a[live], rank[live])
        np.minimum.at(best, b[live], rank[live])
        by_rank = np.empty(m, np.int64)
        by_rank[rank] = np.arange(m)
        added = 0
        for v in np.flatnonzero((label == np.arange(n)) & (best != none)):
            e = by_rank[best[v]]
            o = label[col[e]] if label[row[e]] == v else label[row[e]]
            if o < v and best[o] == best[v]:
                continue                                        # a mutual pick: recorded by the smaller root
            picked.append(int(e))
            added += 1
            x, y = _find(parent, int(v)), _find(parent, int(o))
            assert x != y, "a picked edge closes a cycle"
            parent[max(x, y)] = min(x, y)
        label = np.array([_find(parent, i) for i in range(n)], np.int64)
        rounds += 1
        if added == 0:
            break
    picked = np.array(picked, np.int64)
    return picked[np.argsort(rank[picked], kind="stable")], rounds


def forest_labels(n, row, col):
    """label[i] = smallest vertex of i's tree"""
    parent = list(range(n))
    for a, b in zip(np.asarray(row).tolist(), np.asarray(col).tolist()):
        x, y = _find(parent, a), _find(parent, b)
        if x != y:
            parent[max(x, y)] = min(x, y)
    return np.array([_find(parent, i) for i in range(n)], np.int64)


def to_linkage(n, row, col, dist, join_at=1.0):
    """scipy linkage matrix of a forest given in forest order; separate trees are joined at `join_at` at the end"""
    parent = list(range(n))
    cluster = list(range(n))            # scipy cluster id of each root
    size = [1] * n
    z = []

    def join(a, b, d):
        x, y = _find(parent, a), _find(parent, b)
        z.append([min(cluster[x], cluster[y]), max(cluster[x], cluster[y]), d, size[x] + size[y]])
        r, s = min(x, y), max(x, y)
        parent[s] = r
        size[r] = size[x] + size[y]
        cluster[r] = n + len(z) - 1

    for a, b, d in zip(np.asarray(row).tolist(), np.asarray(col).tolist(), np.asarray(dist, np.float64).tolist()):
        join(a, b, d)
    roots = sorted({_find(parent, i) for i in range(n)})
    for r in roots[1:]:
        join(roots[0], r, join_at)
    return np.array(z, np.float64).reshape(-1, 4)

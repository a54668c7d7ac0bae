"""Model of the linkage cut per component (DESIGN.md 3.13, mashgpu_dist_linkage_cut).

threshold(t, n)                  T = t (1 + 8 n 2^-53), rounded up: no merge at height <= t joins two components at T.
components(D, T)                 labels[i] = smallest index of i's component in the graph of the pairs j < i with D(i, j) <= T; one
                                 component when T >= 1.  (The device takes the pairs within T that share a hash, plus the pairs of
                                 empty sketches, at distance 0: every other Mash pair without a shared hash is at distance 1.)
linkage_cut(D, method, t)        the per-component route: components at T, linkage_model.linkage_cached on each component's sub-grid
                                 (members in index order), and the cut of each.  Returns (labels, merges, n_components): labels[i] =
                                 smallest index of i's flat cluster; merges in the device's forest layout (leaves = indices, merge s =
                                 node n + s, grouped by component in order of smallest member).
whole_cut(D, method, t)          the same labels from the whole set's tree: cut(linkage_cached(D)).
clades_at_most(merges, n, t)     {frozenset of leaves: height bits} of the merges whose subtree's largest height is <= t; for a forest
                                 as for a tree.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from linkage_model import cut, linkage_cached, symmetric


def threshold(t, n):
    return float(np.nextafter(t * (1.0 + 8.0 * n * 2.0 ** -53), np.inf))


def smallest_labels(numbers):
    """cluster numbers (any ids) -> the smallest index with the same number"""
    first = {}
    return np.array([first.setdefault(int(c), i) for i, c in enumerate(numbers)], np.uint32)


def components(D, T):
    A = symmetric(D)
    n = len(A)
    if T >= 1:
        return np.zeros(n, np.uint32)
    i, j = np.tril_indices(n, -1)
    keep = A[i, j] <= T
    g = coo_matrix((np.ones(int(keep.sum())), (i[keep], j[keep])), shape=(n, n))
    return smallest_labels(connected_components(g, directed=False)[1])


def linkage_cut(D, method, t):
    A = symmetric(D)
    n = len(A)
    comp = components(A, threshold(t, n))
    labels = np.zeros(n, np.uint32)
    out = {"id_lo": [], "id_hi": [], "height": [], "size": []}
    roots = np.unique(comp)                         # ascending: the order of the components' smallest members
    for r in roots:
        mem = np.flatnonzero(comp == r)
        m = len(mem)
        if m == 1:
            labels[mem[0]] = mem[0]
            continue
        base = n + len(out["height"])
        merges, _, _ = linkage_cached(A[np.ix_(mem, mem)], method)
        labels[mem] = mem[smallest_labels(cut(merges, m, t))]
        glob = lambda x: int(mem[x]) if x < m else base + int(x) - m
        out["id_lo"] += [glob(x) for x in merges["id_lo"]]
        out["id_hi"] += [glob(x) for x in merges["id_hi"]]
        out["height"] += merges["height"].tolist()
        out["size"] += merges["size"].tolist()
    forest = {"id_lo": np.array(out["id_lo"], np.uint32), "id_hi": np.array(out["id_hi"], np.uint32),
              "height": np.array(out["height"], np.float64), "size": np.array(out["size"], np.uint32)}
    return labels, forest, len(roots)


def whole_cut(D, method, t):
    n = len(D)
    if n == 1:
        return np.zeros(1, np.uint32)
    return smallest_labels(cut(linkage_cached(D, method)[0], n, t))


def clades_at_most(merges, n, t):
    under = {i: frozenset([i]) for i in range(n)}
    worst = {i: 0.0 for i in range(n)}
    out = {}
    for s in range(len(merges["height"])):
        lo, hi, h = int(merges["id_lo"][s]), int(merges["id_hi"][s]), merges["height"][s]
        c = under[lo] | under[hi]
        w = max(h, worst[lo], worst[hi])
        under[n + s], worst[n + s] = c, w
        if w <= t:
            out[c] = np.float64(h).view(np.uint64)
    return out

"""Models of average and complete linkage (DESIGN.md 3.11).

linkage(D, method)         the definition: every step merges the least (D(a, b), b, a) over live slots a < b, found by a scan of
                           the whole lower triangle.  numpy float64, one operation at a time in the definition's order (numpy
                           never fuses), so its merges are mashgpu_linkage_matrix's bit for bit.
linkage_cached(D, method)  the device algorithm: per-row nearest-neighbour caches and their update rule.  Returns the same merges
                           (checked against linkage()), the rows rescanned as the device counts them, and the bytes those rescans
                           read.  O(n) numpy work per merge, so it reaches sizes the naive scan does not.
as_z(merges)               scipy's (n - 1, 4) Z.
cut(merges, n, t)          the clusters of `mash triangle -L <method> -d t`: scipy's fcluster(Z, t, "distance") (a maximal
                           subtree whose every merge has height <= t), numbered from 0 in the order of their first member.
tree(merges, n)            the rooted tree of `mash triangle -L` in nj_model's (parent, length) form: node height h_s * 0.5,
                           leaves 0, branch = height of the parent - height of the child; the root 2n - 2 has parent NONE.
Merges are dicts of arrays {"id_lo", "id_hi", "height", "size"}, the layout of Engine.linkage_matrix.
"""
import numpy as np

NONE = 0xFFFFFFFF
METHODS = ("average", "complete")


def symmetric(D):
    """the full matrix the device works on: the lower triangle mirrored, the diagonal 0 (the upper triangle of D is not read)"""
    A = np.tril(np.asarray(D, np.float64), -1).copy()
    iu = np.triu_indices(len(A), 1)
    A[iu] = A.T[iu]
    return A


def update(method, na, nb, da, db):
    """D(u, k) from D(a, k) and D(b, k), elementwise"""
    if method == "average":
        return (np.float64(na) * da + np.float64(nb) * db) / np.float64(na + nb)
    assert method == "complete"
    return np.where(db > da, db, da)


def _merges(n):
    m = max(n - 1, 0)
    return {"id_lo": np.zeros(m, np.uint32), "id_hi": np.zeros(m, np.uint32), "height": np.zeros(m, np.float64),
            "size": np.zeros(m, np.uint32)}


def _record(out, s, ids, a, b, h, size):
    out["id_lo"][s], out["id_hi"][s] = min(ids[a], ids[b]), max(ids[a], ids[b])
    out["height"][s], out["size"][s] = h, size


def linkage(D, method):
    A = symmetric(D)
    n = len(A)
    assert n >= 2
    M = A.copy()                                   # the search matrix: the lower triangle of live slots, +inf elsewhere
    M[np.triu_indices(n)] = np.inf
    size = np.ones(n, np.int64)
    ids = list(range(n))
    live = np.ones(n, bool)
    out = _merges(n)
    for s in range(n - 1):
        b, a = divmod(int(np.argmin(M)), n)        # first minimum in row-major order = least (D(a, b), b, a)
        h = M[b, a]
        na, nb = size[a], size[b]
        v = update(method, na, nb, A[a], A[b])
        _record(out, s, ids, a, b, h, na + nb)
        live[b] = False
        other = live.copy()
        other[a] = False
        A[a, other] = v[other]
        A[other, a] = v[other]
        M[a, :a] = np.where(other[:a], v[:a], np.inf)
        M[a + 1:, a] = np.where(other[a + 1:], v[a + 1:], np.inf)
        M[b, :] = np.inf
        M[:, b] = np.inf
        ids[a], size[a] = n + s, na + nb
    return out


def linkage_cached(D, method):
    """(merges, rows rescanned, bytes read by the rescans)"""
    A = symmetric(D)
    n = len(A)
    assert n >= 2
    cv = np.full(n, np.inf)
    cj = np.full(n, NONE, np.int64)
    live = np.ones(n, bool)
    size = np.ones(n, np.int64)
    ids = list(range(n))
    idx = np.arange(n)

    def rescan(i):                                  # dead columns hold NaN, which is never the least
        row = A[i, :i]
        if i == 0 or np.isnan(row).all():
            cv[i], cj[i] = np.inf, NONE
        else:
            j = int(np.nanargmin(row))
            cv[i], cj[i] = row[j], j

    for i in range(n):
        rescan(i)
    rows = read = 0
    out = _merges(n)
    for s in range(n - 1):
        cand = np.flatnonzero(cj != NONE)
        b = int(cand[np.argmin(cv[cand])])          # least (value, row): argmin takes the first of equal values
        a, h = int(cj[b]), cv[b]
        na, nb = size[a], size[b]
        v = update(method, na, nb, A[a], A[b])
        _record(out, s, ids, a, b, h, na + nb)
        live[b] = False
        other = live.copy()
        other[a] = False
        A[a, other] = v[other]
        A[other, a] = v[other]
        A[b + 1:, b] = np.nan
        K = idx[other & (idx > a)]
        vk, ck, jk = v[K], cv[K], cj[K]
        hit = (jk == a) | (jk == b)
        keep = hit & (vk <= ck)
        lower = ~hit & ((vk < ck) | ((vk == ck) & (a < jk)))
        cv[K[keep | lower]], cj[K[keep | lower]] = vk[keep | lower], a
        redo = [a] + K[hit & ~keep].tolist()
        cv[b], cj[b] = np.inf, NONE
        for i in redo:
            rescan(i)
        rows += len(redo)
        read += 8 * sum(redo)
        ids[a], size[a] = n + s, na + nb
    return out, rows, read


def as_z(merges):
    return np.column_stack([merges["id_lo"].astype(np.float64), merges["id_hi"].astype(np.float64), merges["height"],
                            merges["size"].astype(np.float64)])


def cut(merges, n, t):
    m = n - 1
    top = np.arange(2 * n - 1)
    worst = np.zeros(2 * n - 1)                     # the largest height in the subtree of each node
    for s in range(m):
        worst[n + s] = max(merges["height"][s], worst[merges["id_lo"][s]], worst[merges["id_hi"][s]])
    for s in range(m - 1, -1, -1):                  # from the root down: a child inherits its parent's cluster when it is cut below t
        u = n + s
        for c in (merges["id_lo"][s], merges["id_hi"][s]):
            top[c] = top[u] if worst[u] <= t else c
    number = {}
    return np.array([number.setdefault(int(top[i]), len(number)) for i in range(n)], np.int64)


def tree(merges, n):
    parent = np.full(2 * n - 1, NONE, np.uint32)
    height = np.zeros(2 * n - 1)
    height[n:] = merges["height"] * 0.5
    for s in range(n - 1):
        parent[merges["id_lo"][s]] = parent[merges["id_hi"][s]] = n + s
    length = np.zeros(2 * n - 1)
    for v in range(2 * n - 2):
        length[v] = height[parent[v]] - height[v]
    return parent, length


def ultrametric(n, rng, depth=12):
    """a random rooted binary tree with leaves 0..n-1 whose merge heights are distinct dyadic numbers, and its ultrametric matrix
    D(i, j) = height of the lowest common ancestor.  Returns (D, {frozenset of leaves: height} of every internal node)."""
    heights = np.sort(rng.choice(np.arange(1, 2 ** depth), n - 1, replace=False)) / 2.0 ** depth
    members = [[i] for i in rng.permutation(n)]
    D = np.zeros((n, n))
    clades = {}
    for h in heights:                               # merge two random clusters at each height, lowest first
        x, y = sorted(rng.choice(len(members), 2, replace=False))
        p, q = members[x], members[y]
        D[np.ix_(p, q)] = h
        D[np.ix_(q, p)] = h
        clades[frozenset(p + q)] = h
        members[x] = p + q
        del members[y]
    return D, clades


def clades(merges, n):
    """{frozenset of leaves: height} of every merge"""
    under = [frozenset([i]) for i in range(n)]
    out = {}
    for s in range(n - 1):
        c = under[merges["id_lo"][s]] | under[merges["id_hi"][s]]
        under.append(c)
        out[c] = merges["height"][s]
    return out

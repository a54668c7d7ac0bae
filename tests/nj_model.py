"""Models of neighbor joining (DESIGN.md 3.10).

nj(D)        numpy restatement of mashgpu_neighbor_joining_matrix, operation for operation: its parent and length are the device's
             bit for bit.  Every operation is one float64 numpy operation in the order of the definition (numpy never fuses).
nj_exact(D)  textbook NJ in fractions.Fraction, the row sums recomputed every step, ties broken the same way.
newick(parent, length, names)   the `mash triangle -N` line: children in ascending node id, lengths as `cout << v` prints them.
splits(parent, length, n)       the tree as an unrooted tree: {split: branch length}.
random_tree, TreeMatrix         trees with integer branch lengths and their path-length matrices (exactly additive).
"""
from collections import deque
from fractions import Fraction

import numpy as np

NONE = 0xFFFFFFFF


def symmetric(D):
    """the full matrix the device works on: the lower triangle mirrored, the diagonal 0 (the upper triangle of D is not read)"""
    A = np.tril(np.asarray(D, np.float64), -1).copy()
    iu = np.triu_indices(len(A), 1)
    A[iu] = A.T[iu]
    return A


def nj(D):
    A = symmetric(D)
    n = len(A)
    assert n >= 3
    parent = np.zeros(2 * n - 2, np.uint32)
    length = np.zeros(2 * n - 2, np.float64)
    r = np.cumsum(A, axis=1)[:, -1]                 # sequential over ascending k (np.sum would sum pairwise)
    ids = list(range(n))
    for s in range(n - 3):
        m = n - s
        # Q over the lower triangle of positions, row q, column p: ((m - 2) * D - r_p) - r_q
        Q = (np.float64(m - 2) * A - r[None, :]) - r[:, None]
        Q[np.triu_indices(m)] = np.inf
        t = int(np.argmin(Q))                        # first minimum in row-major order = least (Q, q, p)
        q, p = divmod(t, m)
        assert np.isfinite(Q[q, p])
        dab = A[q, p]
        la = dab * 0.5 + (r[p] - r[q]) / (2.0 * np.float64(m - 2))
        lb = dab - la
        u = n + s
        parent[ids[p]] = parent[ids[q]] = u
        length[ids[p]], length[ids[q]] = la, lb
        du = ((A[p] + A[q]) - dab) * 0.5
        rn = ((r - A[p]) - A[q]) + du
        rn[p] = ((r[p] + r[q]) - np.float64(m) * dab) * 0.5
        A[p, :] = du
        A[:, p] = du
        A[p, p] = 0.0
        keep = np.arange(m) != q
        A = A[keep][:, keep]
        r = rn[keep]
        ids[p] = u
        del ids[q]
    c = 2 * n - 3
    dxy, dxz, dyz = A[1, 0], A[2, 0], A[2, 1]
    for v, l in zip(ids, (((dxy + dxz) - dyz) * 0.5, ((dxy + dyz) - dxz) * 0.5, ((dxz + dyz) - dxy) * 0.5)):
        parent[v], length[v] = c, l
    parent[c], length[c] = NONE, 0.0
    return parent, length


def nj_exact(D):
    D = np.asarray(D)
    n = len(D)
    A = [[Fraction(0) if i == j else Fraction(float(D[max(i, j), min(i, j)])) for j in range(n)] for i in range(n)]
    live = list(range(n))                            # node ids in position order
    rows = list(range(n))                            # row of A of each position
    parent = [NONE] * (2 * n - 2)
    length = [Fraction(0)] * (2 * n - 2)
    for s in range(n - 3):
        m = len(live)
        R = [sum(A[rows[i]][rows[k]] for k in range(m)) for i in range(m)]
        best = None
        for q in range(1, m):
            for p in range(q):
                key = ((m - 2) * A[rows[q]][rows[p]] - R[p] - R[q], q, p)
                if best is None or key < best:
                    best = key
        _, q, p = best
        a, b = rows[p], rows[q]
        dab = A[a][b]
        la = dab / 2 + (R[p] - R[q]) / (2 * (m - 2))
        u = n + s
        parent[live[p]] = parent[live[q]] = u
        length[live[p]], length[live[q]] = la, dab - la
        for k in range(m):
            if k not in (p, q):
                A[a][rows[k]] = A[rows[k]][a] = (A[a][rows[k]] + A[b][rows[k]] - dab) / 2
        live[p] = u
        del live[q], rows[q]
    (x, y, z), (rx, ry, rz) = live, rows
    for v, l in ((x, (A[rx][ry] + A[rx][rz] - A[ry][rz]) / 2), (y, (A[rx][ry] + A[ry][rz] - A[rx][rz]) / 2),
                 (z, (A[rx][rz] + A[ry][rz] - A[rx][ry]) / 2)):
        parent[v], length[v] = 2 * n - 3, l
    return np.array(parent, np.uint32), length


def _bottom_up(parent):
    """node ids ordered so that every child comes before its parent"""
    parent = np.asarray(parent, np.int64)
    children = [[] for _ in range(len(parent))]
    roots = []
    for v, p in enumerate(parent):
        (roots if p == NONE else children[int(p)]).append(v)
    order = []
    stack = list(roots)
    while stack:
        v = stack.pop()
        order.append(v)
        stack.extend(children[v])
    return order[::-1]


def splits(parent, length, n):
    """the tree as an unrooted tree: {split: branch length}, a split being the XOR of random 64-bit leaf keys on the side of the
    branch without leaf 0 (so equal keys mean equal leaf sets, up to a 2^-64 chance)"""
    key = np.random.Generator(np.random.PCG64(12345)).integers(0, 2**63, n, dtype=np.int64).tolist()
    total = 0
    for k in key:
        total ^= k
    under = [0] * len(parent)
    for v in range(n):
        under[v] = key[v]
    has0 = [False] * len(parent)
    has0[0] = True
    out = {}
    for v in _bottom_up(parent):
        p = int(parent[v])
        if p == NONE:
            continue
        under[p] ^= under[v]
        has0[p] |= has0[v]
        out[total ^ under[v] if has0[v] else under[v]] = length[v]
    return out


def random_tree(n, kind, rng, max_length=9):
    """an unrooted binary tree with leaves 0..n-1 in the output format of nj (parent, length; the center has parent NONE) and integer
    branch lengths in [1, max_length].  kind: "random" (each leaf inserted on a random branch), "caterpillar" (on the last leaf's
    branch) or "balanced" (on the branches of the leaves in first-in first-out order).  Leaves are numbered in a random order."""
    nodes = 2 * n - 2
    center = nodes - 1
    parent = np.full(nodes, NONE, np.int64)
    parent[[0, 1, 2]] = center
    nxt = n
    fifo = deque([0, 1, 2])
    for x in range(3, n):
        if kind == "random":
            v = int(rng.integers(0, x + nxt - n))
            v = v if v < x else n + v - x
        elif kind == "caterpillar":
            v = x - 1
        else:
            v = fifo.popleft()
            fifo += [v, x]
        w = nxt
        nxt += 1
        parent[w] = parent[v]
        parent[v] = w
        parent[x] = w
    perm = rng.permutation(n)                        # leaf v becomes perm[v]
    relabel = np.concatenate([perm, np.arange(n, nodes)])
    out = np.full(nodes, NONE, np.int64)
    out[relabel] = np.where(parent == NONE, NONE, relabel[np.minimum(parent, nodes - 1)])
    length = rng.integers(1, max_length + 1, nodes).astype(np.float64)
    length[center] = 0.0
    return out.astype(np.uint32), length


class TreeMatrix:
    """rows of the path-length matrix of a tree in the format above, O(n) numpy work per row: the depth of the lowest common
    ancestor of two leaves is the least depth between them in a depth-first order of the leaves"""

    def __init__(self, parent, length, n):
        parent = np.asarray(parent, np.int64)
        children = [[] for _ in range(len(parent))]
        root = None
        for v, p in enumerate(parent):
            if p == NONE:
                root = v
            else:
                children[p].append(v)
        depth = np.zeros(len(parent))
        order, adj = [], []
        last_leaf_seen = False
        stack = [root]
        while stack:
            v = stack.pop()
            if v != root:
                depth[v] = depth[parent[v]] + length[v]
                if last_leaf_seen:
                    adj.append(depth[parent[v]])     # first node after a leaf: its parent is the two leaves' common ancestor
                    last_leaf_seen = False
            if v < n:
                order.append(v)
                last_leaf_seen = True
            stack.extend(reversed(children[v]))
        self.n = n
        self.depth = depth[:n]
        self.pos = np.empty(n, np.int64)
        self.pos[np.array(order)] = np.arange(n)
        self.adj = np.array(adj)

    def row(self, a):
        i = self.pos[a]
        lca = np.empty(self.n)
        lca[i] = self.depth[a]
        lca[i + 1:] = np.minimum.accumulate(self.adj[i:])
        if i:
            lca[:i] = np.minimum.accumulate(self.adj[:i][::-1])[::-1]
        d = (self.depth[a] + self.depth) - 2 * lca[self.pos]
        d[a] = 0.0
        return d

    def matrix(self):
        return np.stack([self.row(a) for a in range(self.n)])


def quote(name):
    if name == "" or any(ch in name for ch in " \t()[]':;,"):
        return "'" + name.replace("'", "''") + "'"
    return name


def fmt(v):
    """`cout << v` of a double (printf %g)"""
    return "%g" % v


def newick(parent, length, names):
    n = len(names)
    if n == 1:
        return quote(names[0]) + ";"
    if n == 2:
        x = fmt(float(length))                       # n = 2: `length` is the single branch D * 0.5
        return f"({quote(names[0])}:{x},{quote(names[1])}:{x});"
    children = [[] for _ in range(len(parent))]
    for v, p in enumerate(parent):                   # ascending ids, so every child list is ascending
        if p != NONE:
            children[int(p)].append(v)
    center = len(parent) - 1
    out = []
    stack = [("open", center)]
    while stack:                                     # iterative: a caterpillar is as deep as it is wide
        what, v = stack.pop()
        if what == "text":
            out.append(v)
        elif what == "open" and children[v]:
            out.append("(")
            tail = [("text", ")")]
            if v != center:
                tail.append(("text", ":" + fmt(length[v])))
            stack.extend(reversed(tail))
            for i, c in reversed(list(enumerate(children[v]))):
                stack.append(("open", c))
                if i:
                    stack.append(("text", ","))
        else:
            out.append(quote(names[v]) + ":" + fmt(length[v]))
    return "".join(out) + ";"

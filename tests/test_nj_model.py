"""CPU tests of the neighbor-joining models (tests/nj_model.py) and of the Newick writer of `mash triangle -N`
(mash_b200/host/newick.hpp, through tools/newick_test.cpp).  The models are what the GPU tests hold the device to."""
import os
import subprocess

import numpy as np
import pytest

from nj_model import NONE, TreeMatrix, newick, nj, nj_exact, random_tree, splits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind", ["random", "caterpillar", "balanced"])
def test_additive_trees_are_recovered_exactly(kind):
    """integer branch lengths >= 1: every D, Q, row sum and branch length is an exact integer or half-integer, so nj returns the
    true tree exactly (ties between cherries may rename internal nodes, so trees are compared by their splits)"""
    rng = np.random.Generator(np.random.PCG64(7))
    for n in list(range(3, 20)) + [25, 33, 47, 60]:
        parent, length = random_tree(n, kind, rng)
        D = TreeMatrix(parent, length, n).matrix()
        got_p, got_l = nj(D)
        assert splits(got_p, got_l, n) == splits(parent, length, n), (kind, n)
        assert got_p[-1] == NONE and got_l[-1] == 0.0


def test_tree_matrix_is_the_path_length_matrix():
    rng = np.random.Generator(np.random.PCG64(8))
    parent, length = random_tree(12, "random", rng)
    D = TreeMatrix(parent, length, 12).matrix()

    def path(v):
        out = []
        while v != NONE:
            out.append(v)
            v = int(parent[v])
        return out
    for a in range(12):
        for b in range(12):
            pa, pb = path(a), path(b)
            common = set(pa) & set(pb)
            want = sum(length[v] for v in pa + pb if v not in common)
            assert D[a, b] == want


def test_non_additive_matrices_against_exact_arithmetic():
    rng = np.random.Generator(np.random.PCG64(9))
    checked = 0
    for trial in range(80):
        n = int(rng.integers(3, 26)) if trial % 4 == 0 else int(rng.integers(3, 12))
        X = rng.random((n, n))
        D = np.tril(X + X.T, -1)
        D = D + D.T
        if not _clear_minimum(D):
            continue
        pe, le = nj_exact(D)
        pg, lg = nj(D)
        se, sg = splits(pe, le, n), splits(pg, lg, n)
        assert se.keys() == sg.keys()
        for k in se:
            assert abs(float(se[k]) - sg[k]) <= 1e-12
        checked += 1
    assert checked >= 30


def _clear_minimum(D):
    """every step's least Q beats the next by more than 1e-9 (exact arithmetic), so rounding cannot change the pair"""
    from fractions import Fraction
    n = len(D)
    A = [[Fraction(float(D[i, j])) for j in range(n)] for i in range(n)]
    live = list(range(n))
    while len(live) > 3:
        m = len(live)
        R = {i: sum(A[i][k] for k in live) for i in live}
        qs = sorted(((m - 2) * A[a][b] - R[a] - R[b], pa, pb) for pb, b in enumerate(live) for pa, a in enumerate(live[:pb]))
        _, pa, pb = qs[0]
        if m == 4:          # the two pairs of a quartet always tie, and either gives the same unrooted tree
            qs = [x for x in qs if {x[1], x[2]} & {pa, pb}]
        if qs[1][0] - qs[0][0] <= Fraction(1, 10**9):
            return False
        a, b = live[pa], live[pb]
        for k in live:
            if k not in (a, b):
                A[a][k] = A[k][a] = (A[a][k] + A[b][k] - A[a][b]) / 2
        del live[pb]
    return True


def test_all_equal_matrix_ties_give_the_documented_shape():
    """every Q ties at every step, so (q, p) = (1, 0) is joined each time: positions 0 and 1, then u (at position 0) with the next
    leaf, a caterpillar n0, n1 | n2 | ... whose last join and the last two leaves hang from the center"""
    n = 7
    parent, length = nj(np.ones((n, n)))
    assert list(parent[:n]) == [7, 7, 8, 9, 10, 11, 11]
    assert list(parent[n:]) == [8, 9, 10, 11, NONE]
    assert np.all(length[:n] == 0.5) and np.all(length[n:] == 0.0)
    assert newick(parent, length, [f"n{i}" for i in range(n)]) == "(n5:0.5,n6:0.5,(n4:0.5,(n3:0.5,(n2:0.5,(n0:0.5,n1:0.5):0):0):0):0);"


def test_row_sums_are_sequential():
    """row sums in ascending k (np.sum's pairwise order gives other bits for these values)"""
    D = np.zeros((40, 40))
    D[np.tril_indices(40, -1)] = np.random.Generator(np.random.PCG64(3)).random(780) * 1e-3 + 1.0
    D = D + D.T
    seq = np.cumsum(D, axis=1)[:, -1]
    want = np.array([_seq(row) for row in D])
    assert np.array_equal(seq, want)


def _seq(row):
    s = row[0]
    for x in row[1:]:
        s = s + x
    return s


@pytest.fixture(scope="module")
def newick_exe(tmp_path_factory):
    exe = str(tmp_path_factory.getbasetemp() / "newick_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "mash_b200", "host"), os.path.join(ROOT, "tools", "newick_test.cpp"),
                           "-o", exe])
    return exe


def cpp_newick(exe, parent, length, names):
    text = f"{len(names)}\n" + "".join(nm + "\n" for nm in names) + "".join(f"{int(p)} {float(l).hex()}\n" for p, l in zip(parent, length))
    return subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout.rstrip("\n")


def test_newick_quoting(newick_exe):
    names = ["plain", "with space", "tab\there", "o'brien", "", "a(b)", "x[1]", "c:d", "e;f", "g,h", "ok.fna"]
    n = len(names)
    parent, length = random_tree(n, "random", np.random.Generator(np.random.PCG64(4)))
    length = length / 7.0
    line = newick(parent, length, names)
    for q in ["'with space'", "'tab\there'", "'o''brien'", "''", "'a(b)'", "'x[1]'", "'c:d'", "'e;f'", "'g,h'", "plain:", "ok.fna:"]:
        assert q in line
    assert cpp_newick(newick_exe, parent, length, names) == line


def test_newick_small_trees(newick_exe):
    assert newick(None, None, ["a b"]) == "'a b';"
    assert newick(None, 0.0625, ["a", "b"]) == "(a:0.0625,b:0.0625);"
    parent, length = nj(np.array([[0, 0, 0], [1, 0, 0], [2, 3, 0]]))
    line = newick(parent, length, ["x", "y", "z"])
    assert line == "(x:0,y:1,z:2);"
    assert cpp_newick(newick_exe, parent, length, ["x", "y", "z"]) == line


def test_newick_deep_caterpillar(newick_exe):
    n = 5000
    parent, length = random_tree(n, "caterpillar", np.random.Generator(np.random.PCG64(5)))
    names = [f"leaf{i}" for i in range(n)]
    line = newick(parent, length, names)
    assert line.count("(") == line.count(")") == n - 2 and line.endswith(";")
    assert cpp_newick(newick_exe, parent, length, names) == line

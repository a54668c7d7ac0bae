"""tools/tree_ref.cpp from Python: the CPU reference of neighbor joining and average / complete linkage (mashgpu.h), a full
scan of the live lower triangle at every step.  Its outputs are in the layouts of Engine.neighbor_joining_matrix and
Engine.linkage_matrix, so they compare with the device's and the models' bit for bit.

build(directory)                   compiles the reference into directory and returns the executable's path.
trees(exe, D, methods, threads)    the trees of the lower triangle of D (n x n, or n x ld with junk past column n);
run(exe, D, method, threads)       one of them.
assert_nj_bits, assert_linkage_bits   two results equal bit for bit: ids and sizes equal, lengths and heights as uint64."""
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-O2", "-std=c++17", "-fopenmp", "-ffp-contract=off"]


def build(directory):
    exe = os.path.join(str(directory), "tree_ref")
    subprocess.check_call(["g++", *FLAGS, os.path.join(ROOT, "tools", "tree_ref.cpp"), "-o", exe])
    return exe


def trees(exe, D, methods, threads=None):
    """{method: tree} for each of methods ("nj", "average", "complete"), the matrix written once for all of them.  D: an (n, ld)
    float64 array, ld >= n; only the entries j < i of row i are read.  threads: OMP_NUM_THREADS (None: OpenMP's default)."""
    D = np.ascontiguousarray(D, np.float64)
    n, ld = D.shape
    env = dict(os.environ)
    if threads is not None:
        env["OMP_NUM_THREADS"] = str(threads)
    out = {}
    with tempfile.TemporaryDirectory(dir=os.path.dirname(exe)) as tmp:
        src, dst = os.path.join(tmp, "matrix"), os.path.join(tmp, "tree")
        D.tofile(src)
        for method in methods:
            subprocess.run([exe, method, str(n), str(ld), src, dst], env=env, check=True)
            out[method] = _read(open(dst, "rb").read(), method, n)
    return out


def run(exe, D, method, threads=None):
    """the tree of one method (see trees)"""
    return trees(exe, D, (method,), threads)[method]


def _read(raw, method, n):
    if method == "nj":
        m = 2 * n - 2
        return {"parent": np.frombuffer(raw, np.uint32, m).copy(), "length": np.frombuffer(raw, np.float64, m, 4 * m).copy()}
    m = n - 1
    u32 = np.frombuffer(raw, np.uint32, 3 * m)
    return {"id_lo": u32[:m].copy(), "id_hi": u32[m:2 * m].copy(), "size": u32[2 * m:].copy(),
            "height": np.frombuffer(raw, np.float64, m, 12 * m).copy()}


def assert_nj_bits(got, want):
    assert np.array_equal(got["parent"], want["parent"])
    assert np.array_equal(got["length"].view(np.uint64), want["length"].view(np.uint64))


def assert_linkage_bits(got, want):
    for key in ("id_lo", "id_hi", "size"):
        assert np.array_equal(got[key], want[key]), key
    assert np.array_equal(got["height"].view(np.uint64), want["height"].view(np.uint64))

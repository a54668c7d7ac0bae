"""`mash triangle -L average|complete` on the command line: average or complete linkage of every pair's distance.  Without -d the
stdout line must be the Newick writer of tests/nj_model.py over the rooted tree of tests/linkage_model.py; with -d t the clusters
must be the model's cut, and for average linkage also scipy's fcluster(Z, t, "distance") of scipy's own linkage, numbered in
first-member order.  (Complete linkage is not unique under ties, and Mash distances are full of them -- every unrelated pair is at
1 -- so scipy's merge order can give another complete-linkage tree.)  D is the distance grid of an in-process DistJob over the same
sketches (read from a .msh with tests/msh_reader.py), names from the sketches (comments with -C)."""
import shutil

import numpy as np
import pytest
from scipy.cluster.hierarchy import fcluster, linkage as scipy_linkage
from scipy.spatial.distance import squareform

from linkage_model import cut, linkage_cached, tree
from nj_model import newick
from test_gpu_cli_triangle_components import assert_refused, grid, sketch_msh, triangle, work  # noqa: F401  (the module fixture)

pytestmark = pytest.mark.gpu


def check_tree(work, method, args, msh, comment=False):
    out, err = triangle(work, "-L", method, *(["-C"] if comment else []), *args)
    names, D = grid(msh, comment)
    n = len(names)
    assert len(out) == 1
    if n == 1:
        assert out[0] == newick(None, None, names)
        rows = 0
    elif n == 2:                                   # the model's writer takes the one branch length for two leaves
        assert out[0] == newick(None, D[1, 0] * 0.5, names)
        rows = 1
    else:
        merges, rows, _ = linkage_cached(D, method)
        assert out[0] == newick(*tree(merges, n), names)
    assert f"Tree: {n} leaves, {n - 1} merges, {rows} rows rescanned" in err.splitlines()
    return out[0]


def check_clusters(work, method, t, args, msh, comment=False):
    out, err = triangle(work, "-L", method, "-d", t, *(["-C"] if comment else []), *args)
    names, D = grid(msh, comment)
    n = len(names)
    if n == 1:
        want = [0]
    else:
        want = cut(linkage_cached(D, method)[0], n, float(t)).tolist()
        if method == "average":
            f = fcluster(scipy_linkage(squareform(np.tril(D, -1) + np.tril(D, -1).T, checks=False), method=method), float(t), "distance")
            first = {}
            assert want == [first.setdefault(x, len(first)) for x in f]
    assert out == [f"{nm}\t{c}" for nm, c in zip(names, want)]
    assert f"Clusters: {max(want) + 1} at height <= {float(t):g}" in err.splitlines()
    return want


@pytest.mark.parametrize("method", ["average", "complete"])
def test_golden_genomes(work, method):
    msh = sketch_msh(work, "golden_l", "genome1.fna", "genome2.fna", "genome3.fna")
    line = check_tree(work, method, ["genome1.fna", "genome2.fna", "genome3.fna"], msh)
    assert line.startswith("(") and line.endswith(");") and line.count("(") == 2
    check_tree(work, method, ["-l", "genomes.txt"], msh)
    check_tree(work, method, ["golden_l.msh"], msh)
    check_clusters(work, method, "0.1", ["golden_l.msh"], msh)


@pytest.mark.parametrize("method", ["average", "complete"])
def test_synthetic_sketches_with_and_without_comments(work, method):
    check_tree(work, method, ["synth.msh"], work / "synth.msh")
    check_tree(work, method, ["synth.msh"], work / "synth.msh", comment=True)


@pytest.mark.parametrize("t", ["0.05", "0.1", "0.3", "1"])
def test_clusters_of_synthetic_sketches(work, t):
    want = check_clusters(work, "average", t, ["synth.msh"], work / "synth.msh")
    assert 1 < max(want) + 1 < 250 or t == "1"
    check_clusters(work, "complete", t, ["synth.msh"], work / "synth.msh")
    check_clusters(work, "average", t, ["-p", "4", "synth.msh"], work / "synth.msh")


def test_fasta_families(work):
    msh = sketch_msh(work, "fam_files_l", "-l", "families.txt")
    check_tree(work, "average", ["-l", "families.txt"], msh)
    check_tree(work, "complete", [f for f in (work / "families.txt").read_text().split()], msh)
    check_clusters(work, "average", "0.1", ["-l", "families.txt"], msh)
    msh = sketch_msh(work, "fam_records_l", "-i", "families.fa")
    check_tree(work, "average", ["families.fa"], msh)
    check_tree(work, "average", ["families.fa"], msh, comment=True)      # comments "family f" hold a blank: quoted
    check_clusters(work, "complete", "0.05", ["families.fa"], msh, comment=True)


def test_one_and_two_sketches_and_quoted_names(work):
    for name in ("o'brien.fna", "a,b.fna"):
        shutil.copy(work / "genome1.fna", work / name)
    msh = sketch_msh(work, "one_l", "o'brien.fna")
    assert check_tree(work, "average", ["one_l.msh"], msh) == "'o''brien.fna';"
    assert check_clusters(work, "average", "0.1", ["one_l.msh"], msh) == [0]
    msh = sketch_msh(work, "two_l", "o'brien.fna", "a,b.fna")
    assert check_tree(work, "complete", ["o'brien.fna", "a,b.fna"], msh) == "('o''brien.fna':0,'a,b.fna':0);"
    msh = sketch_msh(work, "two_more_l", "genome2.fna", "genome3.fna")
    names, D = grid(msh)
    line = check_tree(work, "average", ["genome2.fna", "genome3.fna"], msh)
    x = "%g" % (D[1, 0] * 0.5)
    assert line == f"(genome2.fna:{x},genome3.fna:{x});"
    assert check_clusters(work, "average", "0.5", ["genome2.fna", "genome3.fna"], msh) == [0, 0]
    assert check_clusters(work, "average", "0", ["genome2.fna", "genome3.fna"], msh) == [0, 1]


def test_refusals_usage_and_the_other_outputs(work):
    assert_refused(work, ["-L", "average"], (["-E"], ["-G"], ["-T"], ["-N"], ["-v", "0.5"]))
    out, err = triangle(work, "-L", "ward", "synth.msh", rc=1)
    assert out == [] and "ERROR" in err and "ward" in err
    _, usage = triangle(work, "-h")
    assert sum(line.lstrip().startswith("-L ") for line in usage.splitlines()) == 1
    m1, _ = triangle(work, "synth.msh")
    e1, _ = triangle(work, "-E", "-d", "0.1", "synth.msh")
    g1, _ = triangle(work, "-G", "-d", "0.1", "synth.msh")
    triangle(work, "-L", "average", "synth.msh")
    assert triangle(work, "synth.msh")[0] == m1
    assert triangle(work, "-E", "-d", "0.1", "synth.msh")[0] == e1
    assert triangle(work, "-G", "-d", "0.1", "synth.msh")[0] == g1

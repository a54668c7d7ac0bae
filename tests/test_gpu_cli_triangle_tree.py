"""`mash triangle -T` on the command line: the minimum spanning forest of the pairs that pass -d / -v and share a hash, as `-E` lines in
forest order.  Checked against the `mash triangle -E` output of the same inputs and cut-off: every forest line is one of its lines, the
forest spans its components, and its sorted distances are those of Kruskal's algorithm over it (printed distances are rounded, so
equal printed values need not be exact ties, but every minimum spanning forest has the same sorted weights).  `-E` and `-G` output
stay as they were."""
import numpy as np
import pytest

from forest_model import forest_labels, kruskal
from test_gpu_cli_triangle_components import clusters_from_edges, triangle, work  # noqa: F401  (the module fixture)
from test_shard_components_gloo import min_labels

pytestmark = pytest.mark.gpu


def check(work, cut, inputs, comment=False):
    names, _, _ = clusters_from_edges(work, cut, inputs, comment)
    index = {nm: i for i, nm in enumerate(names)}
    c = ["-C"] if comment else []
    edge_lines, _ = triangle(work, "-E", *c, *cut, *inputs)
    edge_lines = [l for l in edge_lines if not l.split("\t")[4].startswith("0/")]         # pairs without a shared hash are no edges
    out, err = triangle(work, "-T", *c, *cut, *inputs)
    n = len(names)
    assert set(out) <= set(edge_lines) and len(set(out)) == len(out)
    f = [l.split("\t") for l in out]
    row = np.array([index[x[0]] for x in f], np.int64)
    col = np.array([index[x[1]] for x in f], np.int64)
    dist = np.array([float(x[2]) for x in f])
    assert (row > col).all() and (np.diff(dist) >= 0).all()
    e = [l.split("\t") for l in edge_lines]
    er = np.array([index[x[0]] for x in e], np.int64)
    ec = np.array([index[x[1]] for x in e], np.int64)
    ed = np.array([float(x[2]) for x in e])
    labels = min_labels(n, np.stack([er, ec], 1))
    assert np.array_equal(forest_labels(n, row, col), labels)
    want = kruskal(n, er, ec, ed)
    assert len(out) == len(want) == n - len(np.unique(labels))
    assert np.array_equal(dist, ed[want])
    assert f"Forest: {len(out)} edges, {n - len(out)} trees in " in err
    return out


@pytest.mark.parametrize("cut", [[], ["-d", "0.05"], ["-d", "0.2"], ["-v", "1e-20"], ["-d", "0.3", "-v", "1e-10"]])
def test_forest_of_synthetic_sketches(work, cut):
    out = check(work, cut, ["synth.msh"])
    assert 0 < len(out) < 249


def test_forest_with_comments(work):
    check(work, ["-d", "0.1"], ["synth.msh"], comment=True)


@pytest.mark.parametrize("cut", [[], ["-d", "0.02"], ["-d", "0.06"]])
def test_forest_of_fasta_families(work, cut):
    check(work, cut, [f"{r}" for r in (work / "families.txt").read_text().split()])
    check(work, cut, ["-l", "families.txt"])
    check(work, cut, ["families.fa"])


def test_golden_genomes(work):
    out = check(work, [], ["genome1.fna", "genome2.fna", "genome3.fna"])
    assert len(out) == 2
    check(work, ["-d", "0.01"], ["-l", "genomes.txt"])


def test_cut_of_the_forest_is_the_clusters(work):
    out, _ = triangle(work, "-T", "synth.msh")
    names, _, _ = clusters_from_edges(work, [], ["synth.msh"])
    index = {nm: i for i, nm in enumerate(names)}
    for t in ("0.02", "0.05", "0.1"):
        g, _ = triangle(work, "-G", "-d", t, "synth.msh")
        want = [int(l.split("\t")[1]) for l in g]
        keep = [l.split("\t") for l in out if float(l.split("\t")[2]) <= float(t)]
        lab = forest_labels(len(names), [index[x[0]] for x in keep], [index[x[1]] for x in keep])
        number = {}
        assert [number.setdefault(x, len(number)) for x in lab] == want, t


def test_refusals_usage_and_the_other_outputs(work):
    for other in ("-E", "-G"):
        out, err = triangle(work, "-T", other, "synth.msh", rc=1)
        assert out == [] and "-T" in err and other in err
    _, usage = triangle(work, "-h")
    assert "-T " in usage
    # -E, -G and the matrix do not depend on -T being there: the same lines as a run with the other options only
    e1, _ = triangle(work, "-E", "-d", "0.1", "synth.msh")
    g1, _ = triangle(work, "-G", "-d", "0.1", "synth.msh")
    m1, _ = triangle(work, "synth.msh")
    triangle(work, "-T", "-d", "0.1", "synth.msh")
    assert triangle(work, "-E", "-d", "0.1", "synth.msh")[0] == e1
    assert triangle(work, "-G", "-d", "0.1", "synth.msh")[0] == g1
    assert triangle(work, "synth.msh")[0] == m1
    assert len(e1) > 0 and len(g1) == 250 and len(m1) == 251

"""`mash triangle -L average|complete -d t` on the command line goes through the linkage cut per component (DESIGN.md 3.13).  Its
stdout must be DistJob.linkage_cut()'s clusters and tests/linkage_cut_model.py's over run()'s grid, numbered from 0 in first-member
order, with and without -C and -p; on the fixture sets it must also be the cut of the dense route (DistJob.linkage()), computed here.
stderr keeps the `Clusters:` line and adds the component count."""
import json
import os
import subprocess

import numpy as np
import pytest

import mash_b200
from fixtures import GOLDEN
from linkage_cut_model import linkage_cut
from linkage_model import cut
from msh_reader import read_msh
from test_gpu_cli_triangle_components import MASH, sketch_msh, triangle, work  # noqa: F401  (the module fixture)
from test_gpu_dist_linkage_cut import families

pytestmark = pytest.mark.gpu


def load(msh, comment=False):
    m = read_msh(str(msh))
    refs = m["references"]
    s, k = m["sketchSize"], m["kmer"]
    hs = [np.array(r["hashes64"] or r["hashes32"] or [], np.uint64) for r in refs]
    n = len(refs)
    H = np.full((n, s), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    N = np.array([len(h) for h in hs], np.uint32)
    for i, h in enumerate(hs):
        H[i, :len(h)] = h
    L = np.array([r["length"] for r in refs], np.uint64)
    return [r["comment"] if comment else r["name"] for r in refs], H, N, L, s, k


def numbered(labels):
    first = {}
    return [first.setdefault(int(x), len(first)) for x in labels]


def wants(msh, method, ts, comment=False, dense=True):
    """per t: the clusters of linkage_cut(), after checking them against the model and (dense) the dense route's cut"""
    names, H, N, L, s, k = load(msh, comment)
    n = len(names)
    out = {}
    eng = mash_b200.Engine(0)
    try:
        job = eng.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
        try:
            D = job.run(0, n, outputs=("distance",))["distance"] if n > 1 else None
            whole = job.linkage(method) if dense and n > 1 else None
            for t in ts:
                got = job.linkage_cut(method, float(t))
                if n > 1:
                    labels, _, _ = linkage_cut(D, method, float(t))
                    assert np.array_equal(got["labels"], labels)
                    if dense:
                        assert numbered(got["labels"]) == cut(whole, n, float(t)).tolist()
                out[t] = (numbered(got["labels"]), got["n_components"], got["largest_component"])
        finally:
            job.close()
    finally:
        eng.close()
    return names, out


def check(work, method, ts, args, msh, comment=False, dense=True):
    names, want = wants(msh, method, ts, comment, dense)
    for t in ts:
        for extra in ([], ["-p", "4"]):
            out, err = triangle(work, "-L", method, "-d", t, *(["-C"] if comment else []), *extra, *args)
            clusters, comps, largest = want[t]
            assert out == [f"{nm}\t{c}" for nm, c in zip(names, clusters)]
            lines = err.splitlines()
            at = lines.index(f"Clusters: {max(clusters) + 1} at height <= {float(t):g}")
            assert lines[at + 1] == f"Components: {comps} linked, the largest of {largest} sketches"


@pytest.fixture(scope="module")
def families_msh(work):
    """1 200 sketches in families of 1 to 300 members (every tier), as a .msh"""
    H, N, L = families([1] * 30 + [2] * 20 + [4] * 10 + [9, 17, 33, 60, 120, 239, 300, 310], 1000, seed=21)
    g = json.load(open(os.path.join(GOLDEN, "ref_genomes.json")))
    g["sketches"] = [dict(name=f"f{i}", length=int(L[i]), comment=f"member {i}", hashes=[int(x) for x in H[i, :N[i]]]) for i in range(len(N))]
    (work / "families_cut.json").write_text(json.dumps(g, indent=1, separators=(",", " : ")))
    subprocess.run([MASH, "import-json", "families_cut.json", "families_cut.msh"], cwd=work, check=True, capture_output=True)
    return work / "families_cut.msh"


@pytest.mark.parametrize("method", ["average", "complete"])
def test_families_at_several_heights(work, families_msh, method):
    check(work, method, ["0", "0.005", "0.02", "0.05"], ["families_cut.msh"], families_msh, dense=False)
    check(work, method, ["0.02"], ["families_cut.msh"], families_msh, comment=True, dense=False)


@pytest.mark.parametrize("method", ["average", "complete"])
def test_fixture_sets_equal_the_dense_route(work, method):
    check(work, method, ["0.05", "0.1", "0.3", "1"], ["synth.msh"], work / "synth.msh")
    check(work, method, ["0.1"], ["synth.msh"], work / "synth.msh", comment=True)
    msh = sketch_msh(work, "golden_cut", "genome1.fna", "genome2.fna", "genome3.fna")
    check(work, method, ["0", "0.1", "0.5"], ["golden_cut.msh"], msh)
    msh = sketch_msh(work, "fam_records_cut", "-i", "families.fa")
    check(work, method, ["0.02", "0.05"], ["families.fa"], msh)
    check(work, method, ["0.05"], ["families.fa"], msh, comment=True)


def test_usage_names_the_component_limit(work):
    _, usage = triangle(work, "-h")
    assert "with -d the limit is the largest component" in usage

"""`mash triangle -G` on the command line: per sketch its cluster, the connected component of the pairs that pass -d / -v and
share a hash.  Checked against the clusters computed here from `mash triangle -E` with the same cut-off (edges with a shared
hash only), numbered from 0 in the order of their first member, and against the stderr summary."""
import gzip
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import mash_b200
from fixtures import GOLDEN, mutate, synth_genome, synth_sketches
from msh_reader import read_msh
from test_shard_components_gloo import min_labels

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("triangle_g")
    assert os.path.exists(MASH), "build the host shim first (__graft_entry__.build())"
    for f in ("genome1.fna", "genome2.fna", "genome3.fna"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    (d / "genomes.txt").write_text("genome1.fna\ngenome2.fna\ngenome3.fna\n")
    # synthetic FASTA families: three founders, each with mutated descendants, in one multi-record file and one file each
    recs = []
    for f in range(3):
        g = synth_genome(40 + f, 50_000)
        for m in range(6):
            recs.append((f"f{f}m{m}", f"family {f}", g))
            g = mutate(g, 0.01 * (m + 1), 1000 * f + m)
    order = np.random.Generator(np.random.PCG64(3)).permutation(len(recs))
    with open(d / "families.fa", "w") as fa:
        for i in order:
            name, comment, g = recs[i]
            fa.write(f">{name} {comment}\n{bytes(g).decode()}\n")
            (d / f"{name}.fa").write_text(f">{name} {comment}\n{bytes(g).decode()}\n")
    (d / "families.txt").write_text("".join(f"{recs[i][0]}.fa\n" for i in order))
    # a few hundred synthetic sketches in families, some ragged or empty
    g = json.load(open(os.path.join(GOLDEN, "ref_genomes.json")))
    H, N, L = synth_sketches(250, 1000, seed=5, n_families=8, ragged=True)
    N[[4, 9]] = 0
    g["sketches"] = [dict(name=f"s{i}", length=int(L[i]), comment=f"c{i}", hashes=[int(x) for x in H[i, :N[i]]]) for i in range(250)]
    (d / "synth.json").write_text(json.dumps(g, indent=1, separators=(",", " : ")))
    subprocess.run([MASH, "import-json", "synth.json", "synth.msh"], cwd=d, check=True, capture_output=True)
    return d


def triangle(work, *args, rc=0):
    p = subprocess.run([MASH, "triangle", *args], cwd=work, capture_output=True, text=True)
    assert p.returncode == rc, p.stderr
    return p.stdout.splitlines(), p.stderr


def sketch_msh(work, out, *args):
    subprocess.run([MASH, "sketch", "-o", out, *args], cwd=work, check=True, capture_output=True)
    return work / (out + ".msh")


def grid(msh, comment=False):
    """names and the distance grid of run() over the sketches of msh"""
    m = read_msh(str(msh))
    refs = m["references"]
    s, k = m["sketchSize"], m["kmer"]
    hs = [np.array(r["hashes64"] or r["hashes32"] or [], np.uint64) for r in refs]      # empty sketches have neither list
    n = len(refs)
    H = np.full((n, s), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    N = np.array([len(h) for h in hs], np.uint32)
    for i, h in enumerate(hs):
        H[i, :len(h)] = h
    L = np.array([r["length"] for r in refs], np.uint64)
    names = [r["comment"] if comment else r["name"] for r in refs]
    if n == 1:
        return names, np.zeros((1, 1))
    eng = mash_b200.Engine(0)
    try:
        job = eng.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
        try:
            D = job.run(0, n, outputs=("distance",))["distance"]
        finally:
            job.close()
    finally:
        eng.close()
    return names, D


def assert_refused(work, mode, others):
    """the output mode (its arguments) with each of the others is refused: nothing on stdout, an error naming both options"""
    for other in others:
        out, err = triangle(work, *mode, *other, "synth.msh", rc=1)
        assert out == [] and "ERROR" in err and mode[0] in err and other[0] in err


def clusters_from_edges(work, cut, inputs, comment=False):
    """names in input order, cluster per name, edge count: from `mash triangle -E` with the same cut-off"""
    matrix, _ = triangle(work, *(["-C"] if comment else []), *inputs)
    names = [l.split("\t")[0] for l in matrix[1:]]           # one row per sketch after the count line, the name first
    index = {nm: i for i, nm in enumerate(names)}
    assert len(index) == len(names)
    lines, _ = triangle(work, "-E", *(["-C"] if comment else []), *cut, *inputs)
    edges = [(index[f[0]], index[f[1]]) for f in (l.split("\t") for l in lines) if not f[4].startswith("0/")]
    labels = min_labels(len(names), edges)
    number = {}
    clusters = [number.setdefault(x, len(number)) for x in labels]
    return names, clusters, len(edges)


def check(work, cut, inputs, extra=(), comment=False):
    names, clusters, n_edges = clusters_from_edges(work, cut, inputs, comment)
    out, err = triangle(work, "-G", *(["-C"] if comment else []), *extra, *cut, *inputs)
    assert out == [f"{nm}\t{c}" for nm, c in zip(names, clusters)]
    assert f"Clusters: {max(clusters) + 1} from {n_edges} edges" in err.splitlines()
    return clusters


@pytest.mark.parametrize("cut", [[], ["-d", "0.05"], ["-d", "0.2"], ["-v", "1e-20"], ["-d", "0.3", "-v", "1e-10"]])
@pytest.mark.parametrize("extra", [[], ["-p", "4"]])
def test_clusters_of_synthetic_sketches(work, cut, extra):
    clusters = check(work, cut, ["synth.msh"], extra)
    assert 1 < max(clusters) + 1 < 250 or cut == []


def test_clusters_with_comments(work):
    check(work, ["-d", "0.1"], ["synth.msh"], comment=True)


@pytest.mark.parametrize("cut", [[], ["-d", "0.02"], ["-d", "0.06"]])
def test_clusters_of_fasta_families(work, cut):
    # one file per genome, and a list of them
    check(work, cut, [f"{r}" for r in (work / "families.txt").read_text().split()])
    check(work, cut, ["-l", "families.txt"])


def test_single_file_one_sketch_per_record(work):
    clusters = check(work, ["-d", "0.06"], ["families.fa"])
    assert len(clusters) == 18 and max(clusters) + 1 >= 3


def test_golden_genomes(work):
    check(work, [], ["genome1.fna", "genome2.fna", "genome3.fna"])
    check(work, ["-d", "0.01"], ["-l", "genomes.txt"])


def test_refusal_and_usage(work):
    out, err = triangle(work, "-G", "-E", "synth.msh", rc=1)
    assert out == [] and "-G" in err and "-E" in err
    _, usage = triangle(work, "-h")
    assert "-G " in usage

"""`mash dist -B N` on the command line: per query its N nearest references that share a hash with it, in the five columns of
plain `mash dist`.  Checked against the plain output of the same sketches; the exact order among equal distances is pinned at the
C ABI (tests/test_gpu_dist_best.py), where the doubles are visible, not through six printed digits."""
import gzip
import json
import os
import shutil
import subprocess
from collections import Counter, defaultdict

import pytest

from fixtures import GOLDEN, synth_sketches

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("dist_best")
    assert os.path.exists(MASH), "build the host shim first (__graft_entry__.build())"
    for f in ("genome1.fna", "genome2.fna", "genome3.fna"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    subprocess.run([MASH, "sketch", "-o", "g", "genome1.fna", "genome2.fna", "genome3.fna"], cwd=d, check=True, capture_output=True)
    (d / "queries.txt").write_text("genome2.fna\ngenome3.fna\n")
    # a few hundred synthetic sketches in families, some ragged or empty
    g = json.load(open(os.path.join(GOLDEN, "ref_genomes.json")))
    for name, n, seed in (("refs", 300, 5), ("qrys", 60, 6)):
        H, N, L = synth_sketches(n, 1000, seed=seed, n_families=6, ragged=True)
        if name == "qrys":
            Hr, Nr, _ = synth_sketches(300, 1000, seed=5, n_families=6, ragged=True)
            H[:30], N[:30] = Hr[:30], Nr[:30]
        g["sketches"] = [dict(name=f"{name}{i}", length=int(L[i]), comment=f"c{i}", hashes=[int(x) for x in H[i, :N[i]]]) for i in range(n)]
        (d / f"{name}.json").write_text(json.dumps(g, indent=1, separators=(",", " : ")))
        subprocess.run([MASH, "import-json", f"{name}.json", f"{name}.msh"], cwd=d, check=True, capture_output=True)
    return d


def dist(work, *args, rc=0):
    p = subprocess.run([MASH, "dist", *args], cwd=work, capture_output=True, text=True)
    assert p.returncode == rc, p.stderr
    return p.stdout.splitlines(), p.stderr


def by_query(lines):
    out = defaultdict(list)
    for l in lines:
        out[l.split("\t")[1]].append(l)
    return out


def check_best(best, plain, n_best):
    hits = {q: [l for l in ls if not l.split("\t")[4].startswith("0/")] for q, ls in by_query(plain).items()}
    got = by_query(best)
    assert [l.split("\t")[1] for l in best] == [q for q in dict.fromkeys(l.split("\t")[1] for l in plain) for _ in got.get(q, [])]     # query order
    for q, all_hits in hits.items():
        mine = got.get(q, [])
        assert len(mine) == min(n_best, len(all_hits)), q
        assert not Counter(mine) - Counter(all_hits)                # every line occurs in the plain output
        d = [float(l.split("\t")[2]) for l in mine]
        assert d == sorted(d)
        left = Counter(all_hits) - Counter(mine)
        assert all(float(l.split("\t")[2]) >= d[-1] for l in left) if mine else not left
    assert set(got) <= set(hits)


@pytest.mark.parametrize("extra", [[], ["-d", "0.1"], ["-v", "1e-20", "-d", "0.3"], ["-C"], ["-p", "4"]])
@pytest.mark.parametrize("n_best", [1, 5, 1024])
def test_best_lines_are_the_nearest_of_the_plain_output(work, n_best, extra):
    plain, _ = dist(work, *extra, "refs.msh", "qrys.msh")
    best, _ = dist(work, "-B", str(n_best), *extra, "refs.msh", "qrys.msh")
    check_best(best, plain, n_best)
    if n_best >= 300:
        assert Counter(best) == Counter(l for l in plain if not l.split("\t")[4].startswith("0/"))


def test_best_on_genomes_with_a_query_list(work):
    plain, _ = dist(work, "-l", "g.msh", "queries.txt")
    for n_best in (1, 2, 3):
        best, _ = dist(work, "-B", str(n_best), "-l", "g.msh", "queries.txt")
        check_best(best, plain, n_best)
    assert len(plain) == 6


def test_best_refuses_a_table_and_bad_counts(work):
    out, err = dist(work, "-B", "3", "-t", "refs.msh", "qrys.msh", rc=1)
    assert out == [] and "-B" in err and "-t" in err
    for bad in ("0", "1025", "2.5"):
        out, err = dist(work, "-B", bad, "refs.msh", "qrys.msh", rc=1)
        assert out == [] and "-B" in err
    _, usage = dist(work, "-h")
    assert "-B <int>" in usage

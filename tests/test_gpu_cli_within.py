"""`mash within` on the command line: stdout byte-identical to what the reference's containSketches values print through
CommandContain::writeOutput (score, error, reference name, query name; pairs with error <= (float)e; query-major order)."""
import gzip
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import msh_reader
import within_model as wm
from fixtures import GOLDEN, fmt_g

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


@pytest.fixture(scope="module")
def ref():
    if not wm.RefContain.available():
        pytest.skip("oracle/_ref/libmash_ref_contain.so not built")
    return wm.RefContain()


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("within")
    for f in ("genome1.fna", "genome2.fna", "genome3.fna"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    with open(d / "multi.fna", "wb") as o:                  # two records: two reference sketches with -i
        for f in ("genome1.fna", "genome2.fna"):
            o.write(open(d / f, "rb").read())
    assert os.path.exists(MASH), "build the host shim first (__graft_entry__.build())"
    for args in (["-o", "g1", "genome1.fna"], ["-o", "g23", "genome2.fna", "genome3.fna"], ["-s", "500", "-o", "g23s500", "genome2.fna", "genome3.fna"],
                 ["-s", "2000", "-o", "g23s2000", "genome2.fna", "genome3.fna"], ["-i", "-o", "multi", "multi.fna"],
                 ["-i", "-o", "g3i", "genome3.fna"]):
        subprocess.run([MASH, "sketch", *args], cwd=d, check=True, capture_output=True)
    (d / "queries.txt").write_text("genome2.fna\ngenome3.fna\n")
    return d


def run(work, *args, rc=0):
    p = subprocess.run([MASH, "within", *args], cwd=work, capture_output=True, text=True)
    assert p.returncode == rc, p.stderr
    return p.stdout, p.stderr


def sketches(path, s=None):
    m = msh_reader.read_msh(str(path))
    rows, names = [], []
    for r in m["references"]:
        h = np.array(r["hashes64"] if r["hashes64"] else (r["hashes32"] or []), np.uint64)
        rows.append(h[:s] if s else h)
        names.append(r["name"])
    return rows, names


def expected(ref, rrows, rnames, qrows, qnames, e=0.05):
    R, Rn = wm.pack_rows(rrows)
    Q, Qn = wm.pack_rows(qrows)
    score, error = ref.grid(R, Rn, Q, Qn, threads=8)
    lim = float(np.float32(e))
    out = []
    for k in range(len(score)):
        if error[k] <= lim:
            q, r = divmod(k, len(rrows))
            sc = "-nan" if np.isnan(score[k]) else fmt_g(score[k])
            out.append(f"{sc}\t{fmt_g(error[k])}\t{rnames[r]}\t{qnames[q]}\n")
    return "".join(out)


def test_fasta_reference_and_queries(work, ref):
    got, err = run(work, "genome1.fna", "genome2.fna", "genome3.fna")
    assert err == 'Sketching genome1.fna (provide sketch file made with "mash sketch" to skip)...done.\n'
    r, rn = sketches(work / "g1.msh")
    q, qn = sketches(work / "g23.msh")
    want = expected(ref, r, rn, q, qn)
    assert got == want and want.count("\n") >= 1
    assert run(work, "-p", "8", "genome1.fna", "genome2.fna", "genome3.fna")[0] == want
    assert run(work, "-p", "1", "-l", "genome1.fna", "queries.txt")[0] == want
    assert run(work, "g1.msh", "genome2.fna", "genome3.fna") == (want, "")
    assert run(work, "g1.msh", "g23.msh")[0] == want
    assert run(work, "-e", "0", "genome1.fna", "genome2.fna", "genome3.fna")[0] == ""


def test_individual_reference(work, ref):
    got, _ = run(work, "-i", "multi.fna", "genome3.fna")
    r, rn = sketches(work / "multi.msh")
    q, qn = sketches(work / "g3i.msh")
    assert len(rn) == 2
    assert got == expected(ref, r, rn, q, qn, e=0.05)
    assert run(work, "-i", "-e", "1", "multi.fna", "genome3.fna")[0] == expected(ref, r, rn, q, qn, e=1)


def test_query_sketch_sizes(work, ref):
    """contain = true: a query .msh with a smaller s is used as it is; a larger one is reduced with the usual warning."""
    r, rn = sketches(work / "g1.msh")
    q, qn = sketches(work / "g23s500.msh")
    got, err = run(work, "-e", "1", "g1.msh", "g23s500.msh")
    assert got == expected(ref, r, rn, q, qn, e=1) and got.count("\n") == 2 and "skipped" not in err
    q, qn = sketches(work / "g23s2000.msh", s=1000)
    got, err = run(work, "-e", "1", "g1.msh", "g23s2000.msh")
    assert got == expected(ref, r, rn, q, qn, e=1) and "Its sketches will be reduced." in err


def test_sketch_reference_options(work):
    want, _ = run(work, "g1.msh", "genome2.fna", "genome3.fna")
    for opt in ("-k", "-n"):
        args = [opt, "21"] if opt == "-k" else [opt]
        got, err = run(work, *args, "g1.msh", "genome2.fna", rc=1)
        assert got == "" and err == f"ERROR: The option {opt[1]} cannot be used when a sketch is provided; it is inherited from the sketch.\n"
    for opt in (["-a"], ["-z", "ACGT"]):
        got, err = run(work, *opt, "g1.msh", "genome2.fna", "genome3.fna")
        assert err == f"ERROR: The option {opt[0][1]} cannot be used when a sketch is provided; it is inherited from the sketch.\n"
        assert got == want


def _import(work, name, rows, s=1000):
    g = json.load(open(os.path.join(GOLDEN, "ref_genomes.json")))
    g["sketchSize"] = s
    g["sketches"] = [dict(name=f"{name}{i}", length=1000, comment="", hashes=[int(x) for x in r]) for i, r in enumerate(rows)]
    (work / f"{name}.json").write_text(json.dumps(g, indent=1, separators=(",", " : ")))
    subprocess.run([MASH, "import-json", f"{name}.json", f"{name}.msh"], cwd=work, check=True, capture_output=True)


def test_nothing_examined_prints_nan_inf(work, ref):
    """An empty reference sketch and one entirely below the query: j = 0, printed as -nan / inf under -e inf only."""
    _import(work, "low", [[5, 7], []])
    r, rn = sketches(work / "low.msh")
    q, qn = sketches(work / "g23.msh")
    got, _ = run(work, "-e", "inf", "low.msh", "g23.msh")
    assert got == expected(ref, r, rn, q, qn, e=float("inf"))
    assert got.count("-nan\tinf\t") == 4
    assert run(work, "-e", "1e30", "low.msh", "g23.msh")[0] == ""


def test_several_blocks_on_one_job(work, ref):
    """4100 x 4100 sketches: more than 2^24 pairs, so two blocks run on one job.  Most sketches hold 20 hashes (error > 0.05,
    nothing printed); a few hold 600, in both blocks (query rows 4092 and up are the second)."""
    rng = np.random.Generator(np.random.PCG64(9))
    big = np.unique(rng.integers(1, 2**63, 700, dtype=np.uint64))[:600]

    def rows(picks):
        out = [np.unique(rng.integers(1, 2**63, 20, dtype=np.uint64)) for _ in range(4100)]
        for i in picks:
            keep = big[rng.random(big.size) < 0.9]
            out[i] = np.union1d(keep, rng.integers(1, 2**63, 60, dtype=np.uint64))[:600]
        return out

    rr, qr = rows([0, 17, 4099]), rows([3, 4091, 4092, 4099])
    _import(work, "manyr", rr)
    _import(work, "manyq", qr)
    got, _ = run(work, "-p", "4", "manyr.msh", "manyq.msh")
    r, rn = sketches(work / "manyr.msh")
    q, qn = sketches(work / "manyq.msh")
    sel_r, sel_q = [0, 17, 4099], [3, 4091, 4092, 4099]
    lines = expected(ref, [r[i] for i in sel_r], [rn[i] for i in sel_r], [q[i] for i in sel_q], [qn[i] for i in sel_q])
    assert got == lines and got.count("\n") == 12

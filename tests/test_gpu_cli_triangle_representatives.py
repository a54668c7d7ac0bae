"""`mash triangle -R length|input` on the command line: greedy representatives in priority order (longest first, or input order) and
every other sketch's nearest representative.  Checked against the sequential model (tests/representatives_model.py) applied to the
same inputs' `mash triangle -E` lines, in the priority order that `mash info -t`'s lengths give, with the engine's exact distances
for the assignment key, and against the stderr summary."""
import subprocess

import numpy as np
import pytest

from fixtures import fmt_g
from representatives_model import assign, sequential
from test_gpu_cli_triangle_components import MASH, assert_refused, grid, sketch_msh, triangle, work  # noqa: F401 (work: the fixture)

pytestmark = pytest.mark.gpu


def info_lengths(work, msh):
    p = subprocess.run([MASH, "info", "-t", str(msh)], cwd=work, capture_output=True, text=True, check=True)
    rows = [l.split("\t") for l in p.stdout.splitlines() if l and not l.startswith("#")]
    return [r[2] for r in rows], np.array([int(r[1]) for r in rows], np.int64)


def expected(work, msh, order_kind, cut, comment=False):
    """the -R lines and the representative count, from the -E lines of the same cut-off"""
    names, D = grid(msh, comment)
    ids, lengths = info_lengths(work, msh)
    assert ids == grid(msh)[0]
    n = len(names)
    index = {nm: t for t, nm in enumerate(names)}
    assert len(index) == n
    lines, _ = triangle(work, "-E", *(["-C"] if comment else []), *cut, str(msh))
    pairs = np.array([(index[f[0]], index[f[1]]) for f in (l.split("\t") for l in lines) if not f[4].startswith("0/")], np.int64).reshape(-1, 2)
    order = np.argsort(-lengths, kind="stable") if order_kind == "length" else np.arange(n)
    pos = np.empty(n, np.int64)
    pos[order] = np.arange(n)
    a, b = pos[pairs[:, 0]], pos[pairs[:, 1]]
    i, j = np.maximum(a, b), np.minimum(a, b)
    d = D[np.maximum(pairs[:, 0], pairs[:, 1]), np.minimum(pairs[:, 0], pairs[:, 1])]
    is_rep = sequential(n, i, j)
    rep, edge = assign(n, is_rep, i, j, d)
    rep_of, dist_of = np.empty(n, np.int64), np.zeros(n)
    rep_of[order] = order[rep]
    dist_of[order] = np.where(edge >= 0, d[np.maximum(edge, 0)] if len(d) else 0.0, 0.0)
    return [f"{names[x]}\t{names[rep_of[x]]}\t{fmt_g(dist_of[x])}" for x in range(n)], int(is_rep.sum())


def check(work, msh, order_kind, cut, comment=False, extra=()):
    want, reps = expected(work, msh, order_kind, cut, comment)
    out, err = triangle(work, "-R", order_kind, *(["-C"] if comment else []), *extra, *cut, str(msh))
    assert out == want
    summary = [l for l in err.splitlines() if l.startswith("Representatives: ")]
    assert len(summary) == 1 and summary[0].startswith(f"Representatives: {reps} of {len(want)} sketches in ")
    return reps


@pytest.mark.parametrize("order_kind", ["length", "input"])
@pytest.mark.parametrize("cut", [[], ["-d", "0.05"], ["-d", "0.2"], ["-v", "1e-20"], ["-d", "0.3", "-v", "1e-10"]])
def test_synthetic_sketches(work, order_kind, cut):
    reps = check(work, work / "synth.msh", order_kind, cut)
    assert 1 < reps < 250


@pytest.mark.parametrize("order_kind", ["length", "input"])
def test_golden_genomes_and_fasta_families(work, order_kind):
    genomes = sketch_msh(work, "genomes", "genome1.fna", "genome2.fna", "genome3.fna")
    for cut in ([], ["-d", "0.05"]):
        check(work, genomes, order_kind, cut)
    families = sketch_msh(work, "families_each", *(work / "families.txt").read_text().split())
    for cut in ([], ["-d", "0.02"], ["-d", "0.06"]):
        check(work, families, order_kind, cut, extra=["-p", "4"])


def test_comments(work):
    check(work, work / "synth.msh", "length", ["-d", "0.1"], comment=True)


def test_refusals(work):
    assert_refused(work, ["-R", "length"], [["-E"], ["-G"], ["-T"], ["-N"], ["-L", "average"]])
    out, err = triangle(work, "-R", "longest", "synth.msh", rc=1)
    assert out == [] and "ERROR: The argument to -R must be length or input (longest given)." in err
    out, err = triangle(work, "-R", "quality", "-E", "synth.msh", rc=1)     # the argument is checked first, as -L's is
    assert "The argument to -R" in err

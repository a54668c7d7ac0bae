"""`mash triangle -N` on the command line: the neighbor-joining tree of every pair's distance as one Newick line.  Checked against
tests/nj_model.py: stdout must be newick(nj(D)) with D the distance grid of an in-process DistJob over the same sketches (read
from a .msh with tests/msh_reader.py), names from the sketches (comments with -C)."""
import shutil

import pytest

from msh_reader import read_msh
from nj_model import newick, nj
from test_gpu_cli_triangle_components import assert_refused, grid, sketch_msh, triangle, work  # noqa: F401  (the module fixture)

pytestmark = pytest.mark.gpu


def want_line(msh, comment=False):
    names, D = grid(msh, comment)
    if len(names) == 1:
        return newick(None, None, names)
    if len(names) == 2:
        return newick(None, D[1, 0] * 0.5, names)
    return newick(*nj(D), names)


def check(work, args, msh, comment=False):
    out, err = triangle(work, "-N", *(["-C"] if comment else []), *args)
    assert len(out) == 1
    assert out[0] == want_line(msh, comment)
    n = len(read_msh(str(msh))["references"])
    assert f"Tree: {n} leaves, {max(n - 3, 0)} joins" in err
    return out[0]


def leaves(line):
    """leaf labels of a Newick line (unquoted names only), read with a small stack parser"""
    depth, names, tok = 0, [], ""
    for ch in line:
        if ch in "(),;":
            if tok and ":" in tok:
                name = tok.split(":")[0]
                if name:
                    names.append(name)
            tok = ""
            depth += (ch == "(") - (ch == ")")
        else:
            tok += ch
    assert depth == 0
    return names


def test_golden_genomes(work):
    msh = sketch_msh(work, "golden_nj", "genome1.fna", "genome2.fna", "genome3.fna")
    line = check(work, ["genome1.fna", "genome2.fna", "genome3.fna"], msh)
    assert sorted(leaves(line)) == ["genome1.fna", "genome2.fna", "genome3.fna"]
    assert line.startswith("(") and line.endswith(");")
    check(work, ["-l", "genomes.txt"], msh)
    check(work, ["golden_nj.msh"], msh)


def test_synthetic_sketches_with_and_without_comments(work):
    check(work, ["synth.msh"], work / "synth.msh")
    check(work, ["synth.msh"], work / "synth.msh", comment=True)


def test_fasta_families(work):
    msh = sketch_msh(work, "fam_files", "-l", "families.txt")
    check(work, ["-l", "families.txt"], msh)
    check(work, [f for f in (work / "families.txt").read_text().split()], msh)
    msh = sketch_msh(work, "fam_records", "-i", "families.fa")
    check(work, ["families.fa"], msh)
    check(work, ["families.fa"], msh, comment=True)         # comments "family f" hold a blank: quoted


def test_one_and_two_sketches_and_quoted_names(work):
    for name in ("o'brien.fna", "a,b.fna"):
        shutil.copy(work / "genome1.fna", work / name)
    msh = sketch_msh(work, "one", "o'brien.fna")
    assert check(work, ["one.msh"], msh) == "'o''brien.fna';"
    msh = sketch_msh(work, "two", "o'brien.fna", "a,b.fna")
    line = check(work, ["o'brien.fna", "a,b.fna"], msh)
    assert line == "('o''brien.fna':0,'a,b.fna':0);"
    msh = sketch_msh(work, "two_more", "genome2.fna", "genome3.fna")
    line = check(work, ["genome2.fna", "genome3.fna"], msh)
    assert line.startswith("(genome2.fna:") and ",genome3.fna:" in line


def test_refusals_usage_and_the_other_outputs(work):
    assert_refused(work, ["-N"], (["-E"], ["-G"], ["-T"], ["-d", "0.1"], ["-v", "0.5"]))
    _, usage = triangle(work, "-h")
    assert "-N " in usage
    m1, _ = triangle(work, "synth.msh")
    e1, _ = triangle(work, "-E", "-d", "0.1", "synth.msh")
    triangle(work, "-N", "synth.msh")
    assert triangle(work, "synth.msh")[0] == m1
    assert triangle(work, "-E", "-d", "0.1", "synth.msh")[0] == e1

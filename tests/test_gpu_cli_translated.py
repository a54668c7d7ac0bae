"""`mash screen` with a protein sketch through the command-line front end: the mixture is translated in six frames
(CommandScreen.cpp:120, 484-599).  There is no reference golden for this mode; the rows are checked against the restatement of the reference's
translated hashSequence in tests/translated_screen_oracle.py."""
import gzip
import os
import shutil
import subprocess

import numpy as np
import pytest

import msh_reader
from fixtures import GOLDEN, fmt_g
import translated_screen_oracle as tso
from oracle.pyoracle import ALPHABET_PROTEIN
from test_translate_model import revcomp, translate

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


@pytest.fixture(scope="module")
def work(tmp_path_factory, golden):
    d = tmp_path_factory.mktemp("mashcli_trans")
    for f in ("reads1.fastq", "reads2.fastq"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    assert os.path.exists(MASH), "build the host shim first (__graft_entry__.build())"
    # translated regions of genome1..3: frame 0 of the forward strand and frame 1 of the reverse strand, 60 columns per line
    with open(d / "prot.faa", "wb") as f:
        for i, (_, recs) in enumerate(golden.genomes):
            seq = recs[0][2]
            for name, prot in ((f"g{i + 1}_fwd", translate(seq[:45_000])), (f"g{i + 1}_rev", translate(revcomp(seq[1000:31_001])[1:]))):
                f.write(b">%s genome%d region\n" % (name.encode(), i + 1))
                for a in range(0, len(prot), 60):
                    f.write(prot[a:a + 60] + b"\n")
    subprocess.run([MASH, "sketch", "-a", "-i", "-o", "prot", "prot.faa"], cwd=d, check=True, capture_output=True)
    return d


def test_translated_screen_cli(work, oracle, golden):
    pr = subprocess.run([MASH, "screen", "prot.msh", "reads1.fastq", "reads2.fastq"], cwd=work, check=True, capture_output=True, text=True)
    d = msh_reader.read_msh(str(work / "prot.msh"))
    assert d["kmer"] == 9 and d["alphabet"] == ALPHABET_PROTEIN and d["noncanonical"]
    refs = d["references"]
    s = d["sketchSize"]
    ref = np.full((len(refs), s), np.uint64(2**64 - 1)); ref_n = np.zeros(len(refs), np.uint32)
    for i, r in enumerate(refs):
        ref[i, :len(r["hashes64"])] = r["hashes64"]; ref_n[i] = len(r["hashes64"])
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    reads = [r for r in golden.reads_round_robin() if len(r) >= 9]
    want = tso.screen(oracle, ref, ref_n, [b"".join(b"*" + r for r in reads)], po, s=s)
    rows = [i for i in range(len(refs)) if want["shared"][i] != 0]
    assert len(rows) >= 3
    got = [l.split("\t") for l in pr.stdout.splitlines()]
    assert len(got) == len(rows)
    for line, i in zip(got, rows):
        assert line == [fmt_g(want["identity"][i]), f"{want['shared'][i]}/{ref_n[i]}", str(want["median"][i]), fmt_g(want["pvalue"][i]),
                        refs[i]["name"], refs[i]["comment"]]
    assert "Translating from 2 inputs..." in pr.stderr
    assert f"Estimated distinct (translated) k-mers in mixture: {want['set_size']}" in pr.stderr

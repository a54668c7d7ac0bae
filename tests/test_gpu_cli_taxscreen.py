"""`mash taxscreen` through the command-line front end: stdout byte-identical to the checker's report (the reference's own
fold, roll-up and writeReport, tests/taxscreen_oracle.py), stderr lines as the reference prints them, taxIDs from the
sketch comments and from a mapping file (-m), and the exit status when the dumps are missing."""
import gzip
import os
import shutil
import subprocess

import numpy as np
import pytest

import msh_reader
import taxscreen_oracle as txo
from fixtures import GOLDEN, mutate

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not txo.available(), reason="oracle/_ref/taxdb_ref not built")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


@pytest.fixture(scope="module")
def work(tmp_path_factory, golden):
    d = tmp_path_factory.mktemp("mashcli_tax")
    for f in ("reads1.fastq", "reads2.fastq"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    tax = txo.make_taxonomy(str(d / "tax"), seed=21, n_nodes=500, n_extra_roots=1, chain=80)
    known = sorted(tax.parent)
    rng = np.random.Generator(np.random.PCG64(4))
    # the golden genomes (which share most of their k-mers) and mutated copies; taxIDs in the comments: species of the deepest
    # inner node under taxID 1 with two or more children, one sketch with a taxID outside the taxonomy, one with none
    children = {}
    for t in known:
        if tax.parent[t] != t:
            children.setdefault(tax.parent[t], []).append(t)
    depth, root = {}, {}
    for t in known:
        u, n = t, 0
        while tax.parent[u] != u:
            u, n = tax.parent[u], n + 1
        depth[t], root[t] = n, u
    # the report walks down from taxID 1 only
    genus = max((t for t, c in children.items() if len(c) >= 2 and root[t] == 1), key=lambda t: (depth[t], t))
    kids = children[genus]
    entries = []
    for i, (_, recs) in enumerate(golden.genomes):
        seq = np.frombuffer(b"".join(r[2] for r in recs), np.uint8)
        for j, rate in enumerate((0.0, 0.002, 0.01, 0.04)):
            taxid = None if (i, j) == (1, 1) else 7_000_000 + i if (i, j) == (2, 3) else kids[int(rng.integers(0, len(kids)))]
            comment = f"genome{i + 1} variant {j}" + (f" taxid {taxid}" if taxid is not None else "")
            entries.append((f"g{i + 1}v{j}", comment, mutate(seq, rate, 10 * i + j).tobytes() if rate else seq.tobytes(), taxid))
    with open(d / "refs.fna", "wb") as f:
        for name, comment, seq, _ in entries:
            f.write(f">{name} {comment}\n".encode())
            for a in range(0, len(seq), 80):
                f.write(seq[a:a + 80] + b"\n")
    subprocess.run([MASH, "sketch", "-i", "-o", "refs", "refs.fna"], cwd=d, check=True, capture_output=True)
    # mapping file: taxIDs for the sketches that have none in their comment, and a line for a name that is not there
    with open(d / "map.txt", "w") as f:
        f.write("12345\tnot_a_sketch\n")
        for name, _, _, taxid in entries:
            if taxid is None:
                f.write(f"{known[int(rng.integers(0, len(known)))]}\t{name}\n")
    return d, tax, entries


def expected(work_dir, oracle, golden, ref_taxid, no_taxid_names):
    d = msh_reader.read_msh(str(work_dir / "refs.msh"))
    refs = d["references"]
    s = d["sketchSize"]
    ref = np.full((len(refs), s), np.uint64(2**64 - 1)); ref_n = np.zeros(len(refs), np.uint32)
    for i, r in enumerate(refs):
        ref[i, :len(r["hashes64"])] = r["hashes64"]; ref_n[i] = len(r["hashes64"])
    reads = [r for r in golden.reads_round_robin() if len(r) >= d["kmer"]]
    want = txo.taxscreen(oracle, txo.RefTaxDB(str(work_dir / "tax")), ref, ref_n, [b"".join(b"*" + r for r in reads)],
                         oracle.params(k=d["kmer"]), ref_taxid, s=s)
    outside = [int(r[0]) for r in want["rows"] if int(r[0]) == 0 or int(r[0]) >= 7_000_000]
    lines = ["Loading taxonomy files ..."]
    lines += [f"Entry for {9_000_000 + i} does not exist - it should!" for i in range(3)]
    lines += [None, "Reading mapping file ..."]           # None: "   N distinct taxa", filled in by check_stderr
    lines += [f"Could not find taxID for reference {n} in comment field or mapping file!" for n in no_taxid_names]
    lines += ["Loading refs.msh...", f"   {want['keys'].size} distinct hashes.", "Streaming from 2 inputs...",
              f"   Estimated distinct k-mers in pool: {want['set_size']}", "Assigning LCA taxIDs to hashes ..."]
    lines += [f"Couldn't find tax entry with taxID {t}" for t in outside]
    lines += ["Writing output..."]
    return want, lines, [r["name"] for r in refs]


def run_cli(work_dir, *args):
    return subprocess.run([MASH, "taxscreen", *args], cwd=work_dir, capture_output=True)


def check_stderr(stderr, lines, n_taxa):
    got = [l for l in stderr.decode().splitlines() if not (l.startswith("TaxID ") and l.endswith("not in database - ignoring it."))]
    want = [l if l is not None else f"   {n_taxa} distinct taxa" for l in lines]
    assert got == want


def test_taxscreen_cli_comments(work, oracle, golden):
    d, tax, entries = work
    pr = run_cli(d, "-t", "tax", "refs.msh", "reads1.fastq", "reads2.fastq")
    assert pr.returncode == 0, pr.stderr.decode()
    ref_taxid = np.array([t or 0 for _, _, _, t in entries], np.uint64)
    no_taxid = [n for n, _, _, t in entries if t is None]
    want, lines, names = expected(d, oracle, golden, ref_taxid, no_taxid)
    assert names == [e[0] for e in entries]
    assert pr.stdout == want["report"]
    assert pr.stdout.count(b"\n") > 2
    check_stderr(pr.stderr, lines, len(tax.parent))


def test_taxscreen_cli_mapping_file(work, oracle, golden):
    d, tax, entries = work
    pr = run_cli(d, "-m", "map.txt", "-t", "tax", "-p", "2", "-i", "0.5", "-v", "0.1", "refs.msh", "reads1.fastq", "reads2.fastq")
    assert pr.returncode == 0, pr.stderr.decode()
    mapping = {}
    for line in open(d / "map.txt"):
        t, name = line.rstrip("\n").split("\t")
        mapping.setdefault(name, int(t))
    ref_taxid = np.array([mapping.get(n) or t or 0 for n, _, _, t in entries], np.uint64)
    want, lines, _ = expected(d, oracle, golden, ref_taxid, [])
    assert pr.stdout == want["report"]
    check_stderr(pr.stderr, lines, len(tax.parent))


def test_taxscreen_cli_missing_dump(work, tmp_path):
    d, _, _ = work
    pr = run_cli(d, "-t", str(tmp_path), "refs.msh", "reads1.fastq")
    assert pr.returncode == 1
    assert pr.stderr.decode().startswith(f"Could not find a file names.dmp or nodes.dmp in directory {tmp_path}\n")
    assert pr.stdout == b""

"""`mash taxscreen` without a GPU: the order-free LCA rule against the reference's own fold, the engine's dump parser against
the reference's TaxDB, and the engine's report writer against the reference's writeReport, byte for byte, on seeded
synthetic NCBI dumps (tests/taxscreen_oracle.py)."""
import os
import subprocess

import numpy as np
import pytest

import taxscreen_oracle as txo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")

needs_ref = pytest.mark.skipif(not txo.available(), reason="oracle/_ref/taxdb_ref not built (reference sources absent)")

SHAPES = [dict(seed=1, n_nodes=300, n_extra_roots=0, chain=10),
          dict(seed=2, n_nodes=500, n_extra_roots=3, chain=400),       # forest with a deep chain
          dict(seed=3, n_nodes=40, n_extra_roots=5, chain=0, dup_scientific=0.5)]


@pytest.fixture(scope="module", params=range(len(SHAPES)))
def taxonomy(request, tmp_path_factory):
    d = str(tmp_path_factory.mktemp(f"tax{request.param}"))
    tax = txo.make_taxonomy(d, **SHAPES[request.param])
    ref = txo.RefTaxDB(d) if txo.available() else None
    yield d, tax, ref
    if ref:
        ref.close()


def random_multisets(tax, rng, n):
    known = sorted(tax.parent)
    roots = [t for t in known if tax.parent[t] == t]
    unknown = [7_000_001, 7_000_002, 7_000_003]
    for _ in range(n):
        m = int(rng.choice([1, 2, 2, 3, 4, 8, 20, 45]))
        pick = []
        for _ in range(m):
            u = rng.random()
            if u < 0.08:
                pick.append(0)
            elif u < 0.16:
                pick.append(int(rng.choice(unknown)))
            elif u < 0.26:
                pick.append(int(rng.choice(roots)))
            elif u < 0.32 and pick:
                pick.append(pick[int(rng.integers(0, len(pick)))])      # repeated taxID
            elif u < 0.66:
                # members of one small clade: a node and some of its descendants' relatives
                t = int(rng.choice(known))
                for _ in range(int(rng.integers(0, 4))):
                    t = tax.parent[t]
                pick.append(t)
            else:
                pick.append(int(rng.choice(known)))
        yield pick


@needs_ref
def test_fold_rule_matches_reference_fold(taxonomy):
    _, tax, ref = taxonomy
    rng = np.random.Generator(np.random.PCG64(11))
    sets = list(random_multisets(tax, rng, 600))
    sets += [[1, 1], [7_000_001, 7_000_001], [7_000_001], [0, 0, 7_000_002], [0], [], [1], [1, 0, 0]]
    sets += [[r, r] for r in tax.parent if tax.parent[r] == r] + [[r] for r in tax.parent if tax.parent[r] == r]
    taxids, seg, want = [], [0], []
    for m in sets:
        for _ in range(5):
            taxids += [int(x) for x in rng.permutation(np.array(m, np.int64))]
            seg.append(len(taxids))
            want.append(tax.fold_rule(m))
    got = ref.fold(np.array(taxids, np.uint64), np.array(seg, np.uint64))
    assert [int(x) for x in got] == want
    # the rule does say something: all four kinds of result occur
    kinds = {0 if w == 0 else 1 if w == 1 else 2 if w in tax.parent else 3 for w in want}
    assert kinds == {0, 1, 2, 3}


@needs_ref
def test_parser_matches_reference(taxonomy):
    d, tax, ref = taxonomy
    pr = subprocess.run([MASH, "tax-dump", d], capture_output=True, check=True)
    assert pr.stdout == ref.dump()
    lines = pr.stdout.decode().splitlines()
    assert len(lines) == len(tax.parent)
    for line in lines:
        t, p, rank, name = line.split("\t")
        assert int(p) == tax.parent[int(t)] and rank == tax.rank[int(t)] and name == tax.name[int(t)]
    assert f"   {len(tax.parent)} distinct taxa\n" in pr.stderr.decode()
    assert pr.stderr.decode().count("does not exist - it should!") == 3


def random_counts(tax, rng, n_taxa, big=False):
    known = sorted(tax.parent)
    taxa = set(int(t) for t in rng.choice(known, min(n_taxa, len(known)), replace=False))
    taxa |= {7_000_001, 0} if rng.random() < 0.7 else set()
    taxa = sorted(taxa)
    thc = rng.integers(1, 50, len(taxa)).astype(np.uint64)
    tc = (thc * rng.random(len(taxa))).astype(np.uint64)
    tc[rng.random(len(taxa)) < 0.3] = 0
    if big:
        thc[len(taxa) // 2] = 3_000_000_000
        tc[len(taxa) // 2] = 50_000_000               # 100 * count wraps in 32 bits above 42 949 672
    return np.array(taxa, np.uint64), tc, thc


def engine_report(d, rows, totals, tmp_path):
    f = tmp_path / "rows.txt"
    with open(f, "w") as fh:
        fh.write(f"{totals[0]} {totals[1]}\n")
        for r in rows:
            fh.write(" ".join(str(int(x)) for x in r) + "\n")
    return subprocess.run([MASH, "tax-report", d, str(f)], capture_output=True, check=True).stdout


@needs_ref
@pytest.mark.parametrize("case", range(6))
def test_report_matches_reference(taxonomy, case, tmp_path):
    d, tax, ref = taxonomy
    rng = np.random.Generator(np.random.PCG64(100 + case))
    taxa, tc, thc = random_counts(tax, rng, [5, 30, 120, 400, 60, 200][case], big=case == 4)
    want, rows, totals = ref.report(taxa, tc, thc)
    assert want.startswith(b"%\thashes\ttaxHashes")
    assert engine_report(d, rows, totals, tmp_path) == want


@needs_ref
def test_report_ties_beyond_insertion_sort(tmp_path):
    """A node with 40 children of equal clade counts: std::sort switches from insertion sort to introsort above 16
    elements, and the tie order of the report follows it."""
    d = str(tmp_path / "wide")
    os.makedirs(d)
    kids = [int(x) for x in np.random.Generator(np.random.PCG64(5)).choice(np.arange(100, 100_000), 40, replace=False)]
    with open(os.path.join(d, "nodes.dmp"), "w") as f:
        f.write("1\t|\t1\t|\tno rank\t|\n2\t|\t1\t|\tgenus\t|\n")
        for k in kids:
            f.write(f"{k}\t|\t2\t|\tspecies\t|\n")
    with open(os.path.join(d, "names.dmp"), "w") as f:
        f.write("1\t|\troot\t|\t\t|\tscientific name\t|\n2\t|\tWide genus\t|\t\t|\tscientific name\t|\n")
        for k in kids:
            f.write(f"{k}\t|\tSpecies number {k}\t|\t\t|\tscientific name\t|\n")
    ref = txo.RefTaxDB(d)
    try:
        counts = np.array([3] * 30 + [5] * 5 + [1] * 5, np.uint64)
        want, rows, totals = ref.report(np.array(kids, np.uint64), counts, counts + 1)
    finally:
        ref.close()
    assert want.count(b"\n") == 1 + 2 + 40
    assert engine_report(d, rows, totals, tmp_path) == want

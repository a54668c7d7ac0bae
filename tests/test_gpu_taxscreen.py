"""GPU parity tests of the taxonomy step of `mash taxscreen` (mashgpu_screen_taxonomy) through the C ABI: per-hash LCA taxIDs,
the rows of the counts map and the totals, against the checker built on the reference's own fold, roll-up and report
(tests/taxscreen_oracle.py), on the golden genomes and reads and on fuzzed tables."""
import numpy as np
import pytest

import taxscreen_oracle as txo
from fixtures import mutate, synth_genome
from oracle.pyoracle import ALPHABET_PROTEIN
from test_gpu_screen_translated import joined, protein_refs, reads_from

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not txo.available(), reason="oracle/_ref/taxdb_ref not built")]

UNKNOWN = [7_000_001, 7_000_002, 7_000_003]


@pytest.fixture(scope="module")
def tx(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("taxgpu"))
    tax = txo.make_taxonomy(d, seed=7, n_nodes=600, n_extra_roots=2, chain=150)
    return tax, txo.RefTaxDB(d)


@pytest.fixture(scope="module")
def gtax(gpu, tx):
    parent, tids = tx[0].dense()
    t = gpu.taxonomy_open(parent, tids)
    yield t
    t.close()


def assign_taxids(tax, rng, n, mode="mixed"):
    """Sketch taxIDs: leaves and inner nodes, roots (1 among them), taxIDs outside the taxonomy, 0, repeats; mode "clade":
    members of one deep clade only."""
    known = sorted(tax.parent)
    if mode == "clade":
        deep = max(known, key=lambda t: len(_path(tax, t)))
        clade = _path(tax, deep)[:6]
        return np.array([clade[int(rng.integers(0, len(clade)))] for _ in range(n)], np.uint64)
    roots = [t for t in known if tax.parent[t] == t]
    out = []
    for _ in range(n):
        u = rng.random()
        out.append(0 if u < 0.1 else int(rng.choice(UNKNOWN)) if u < 0.18 else int(rng.choice(roots)) if u < 0.24 else
                   out[int(rng.integers(0, len(out)))] if u < 0.4 and out else int(rng.choice(known)))
    return np.array(out, np.uint64)


def _path(tax, t):
    p = [t]
    while tax.parent[p[-1]] != p[-1]:
        p.append(tax.parent[p[-1]])
    return p


def run_tax(gpu, gtax, tax, ref, ref_n, p, chunks, ref_taxid, feed="host"):
    job = gpu.screen_open(ref, ref_n, p)
    try:
        if feed == "dev":
            import torch
            for c in chunks:
                dev = torch.from_numpy(np.frombuffer(c + b"\0" * 16, np.uint8).copy()).cuda()
                torch.cuda.synchronize()
                job.feed_dev(dev.data_ptr(), len(c))
        else:
            for c in chunks:
                job.feed(c)
        code, unknown = txo.ref_codes(tax, ref_taxid)
        return job.taxonomy(gtax, code, unknown, hash_taxid=True), unknown
    finally:
        job.close()


def check(res, want):
    assert np.array_equal(res["hash_taxid"], want["hash_taxid"])
    rows = np.stack([res["rows"][f] for f in ("taxid", "tax_count", "tax_hash_count", "clade_count", "clade_hash_count")], 1) \
        if res["rows"].size else np.zeros((0, 5), np.uint64)
    rows = rows[np.argsort(rows[:, 0], kind="stable")]
    assert np.array_equal(rows, want["rows"].astype(np.uint64))
    assert (res["total_count"], res["total_hash_count"]) == want["totals"]


def test_golden_genomes_and_reads(gpu, oracle, golden, tx, gtax):
    tax, reftax = tx
    k, s = 21, 1000
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    units = []
    for i, (_, recs) in enumerate(golden.genomes):
        seqs = [np.frombuffer(r[2], np.uint8) for r in recs]
        units.append(seqs)
        for j, rate in enumerate((0.001, 0.005, 0.01, 0.03, 0.1)):
            units.append([mutate(q, rate, 100 * i + j) for q in seqs])
    ref = np.full((len(units), s), np.uint64(2**64 - 1)); ref_n = np.zeros(len(units), np.uint32)
    for u, seqs in enumerate(units):
        h, _, _ = oracle.sketch_unit([q.tobytes() for q in seqs], po, s=s)
        ref[u, :h.size] = h; ref_n[u] = h.size
    reads = [r for r in golden.reads_round_robin() if len(r) >= k]
    chunk = b"".join(b"*" + r for r in reads)
    rng = np.random.Generator(np.random.PCG64(3))
    for mode in ("mixed", "clade"):
        ref_taxid = assign_taxids(tax, rng, len(units), mode)
        want = txo.taxscreen(oracle, reftax, ref, ref_n, [chunk], po, ref_taxid, s=s)
        assert int((want["counts"] >= 1).sum()) > 20
        res, _ = run_tax(gpu, gtax, tax, ref, ref_n, p, [chunk], ref_taxid)
        check(res, want)


def fuzz_table(oracle, po, seed, n_ref=1100, stride=64):
    """Rows of a genome's k-mer hashes: 8 hashes in every sketch (> 1024 holders), 8 in 40 sketches, pairs, and hashes of
    their own, plus fresh random hashes; reads of that genome hit a good part of them."""
    rng = np.random.Generator(np.random.PCG64(seed))
    g = synth_genome(seed, 300_000)
    H = np.unique(oracle.all_hashes(g.tobytes(), po))
    H = H[rng.permutation(H.size)]
    every, forty, pairs, own = H[:8], H[8:16], H[16:16 + n_ref], H[16 + n_ref:]
    ref = np.full((n_ref, stride), np.uint64(2**64 - 1)); ref_n = np.zeros(n_ref, np.uint32)
    o = 0
    for r in range(n_ref):
        row = list(every) + (list(forty) if r < 40 else []) + [pairs[r], pairs[r ^ 1]]
        m = int(rng.integers(0, stride - len(row) + 1))
        row += list(own[o:o + m // 2]) + list(rng.integers(0, 2**63, m - m // 2, dtype=np.uint64))
        o += m // 2
        if r % 97 == 5:
            row = []                                   # empty sketch
        row = np.unique(np.array(row, np.uint64))
        ref[r, :row.size] = row; ref_n[r] = row.size
    reads = []
    for _ in range(30_000):
        a = int(rng.integers(0, g.size - 150))
        reads.append(g[a:a + 150].tobytes())
    return ref, ref_n, reads


@pytest.mark.parametrize("feed,mode", [("joined", "mixed"), ("pipelined", "mixed"), ("dev", "clade"), ("pipelined", "clade")])
def test_fuzzed_tables(gpu, oracle, tx, gtax, feed, mode):
    tax, reftax = tx
    k, s = 21, 64
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    ref, ref_n, reads = fuzz_table(oracle, po, 40 + len(feed))
    chunks = joined(reads, 1000) if feed == "joined" else [b"".join(b"*" + r for r in reads)]
    assert feed == "joined" or len(chunks[0]) >= 4 << 20         # one host chunk large enough for the pipelined path
    ref_taxid = assign_taxids(tax, np.random.Generator(np.random.PCG64(9)), ref.shape[0], mode)
    want = txo.taxscreen(oracle, reftax, ref, ref_n, chunks, po, ref_taxid, s=s)
    res, unknown = run_tax(gpu, gtax, tax, ref, ref_n, p, chunks, ref_taxid, feed="dev" if feed == "dev" else "host")
    check(res, want)
    if mode == "mixed":
        assert res["unknown_in_lca"].any()             # unknown taxIDs meet others on the hashes held by every sketch


def test_no_taxids_and_empty_table(gpu, oracle, tx, gtax):
    tax, reftax = tx
    k, s = 21, 64
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    ref, ref_n, reads = fuzz_table(oracle, po, 77, n_ref=50)
    chunk = b"".join(b"*" + r for r in reads[:3000])
    zero = np.zeros(ref.shape[0], np.uint64)
    want = txo.taxscreen(oracle, reftax, ref, ref_n, [chunk], po, zero, s=s)
    res, _ = run_tax(gpu, gtax, tax, ref, ref_n, p, [chunk], zero)
    check(res, want)
    assert res["rows"]["taxid"].tolist() == [0]
    empty_n = np.zeros_like(ref_n)
    res, _ = run_tax(gpu, gtax, tax, ref, empty_n, p, [chunk], assign_taxids(tax, np.random.Generator(np.random.PCG64(1)), ref.shape[0]))
    assert res["rows"].size == 0 and res["total_count"] == 0 and res["total_hash_count"] == 0 and res["hash_taxid"].size == 0


def test_protein_table(gpu, oracle, tx, gtax):
    tax, reftax = tx
    k, s = 9, 1000
    p = gpu.params(k=k, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=k, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    ref, ref_n, _ = protein_refs(oracle, po, s)
    chunks = joined(reads_from(12, 4000), 500)
    ref_taxid = np.array([sorted(tax.parent)[5], sorted(tax.parent)[5], UNKNOWN[0], 0, 1], np.uint64)
    want = txo.taxscreen(oracle, reftax, ref, ref_n, chunks, po, ref_taxid, s=s)
    assert int((want["counts"] >= 1).sum()) > 0
    res, _ = run_tax(gpu, gtax, tax, ref, ref_n, p, chunks, ref_taxid)
    check(res, want)


def test_taxonomy_cycle_is_refused(gpu):
    import mash_b200
    with pytest.raises(mash_b200.MashGpuError, match="cycle"):
        gpu.taxonomy_open(np.array([0, 2, 3, 1], np.uint32), np.array([1, 10, 11, 12], np.uint64))

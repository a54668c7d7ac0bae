"""Checker for `mash taxscreen` (TEST INFRASTRUCTURE, never imported by the product).

Restates CommandTaxScreen.cpp:98-475 on top of the screen checkers (Oracle.screen, or tests/translated_screen_oracle.py for
protein sketches: the distinct reference hashes `keys` and their hit `counts`) and the reference's own taxonomy code
(taxdb.hpp, compiled in place into the tool oracle/_ref/taxdb_ref by oracle/taxdb.mk):

  RefTaxDB        the reference's parser (TaxDB(names, nodes)), getLowestCommonAncestor folded over a hash's sketches as
                  :420-424 folds it, and the roll-up of :442-471 followed by its writeReport, through that tool.
  taxscreen       per distinct hash: the fold over the sketches that hold it; counts[taxon] as :433-439 leaves them; then
                  roll-up, rows and the report from the tool.
  fold_rule       the order-free form of the fold (DESIGN.md 4.2), which the GPU implements; tests/test_taxscreen_model.py
                  pins it to the reference's own fold.
  make_taxonomy   seeded synthetic NCBI dumps: forests, deep chains, names with spaces, several name classes per taxID.
"""
import os
import subprocess
import tempfile

import numpy as np

import translated_screen_oracle as tso

HERE = os.path.dirname(os.path.abspath(__file__))
REF_TOOL = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "taxdb_ref")


def available():
    return os.path.exists(REF_TOOL)


class RefTaxDB:
    """The reference's TaxDB over one names.dmp / nodes.dmp pair (oracle/_ref/taxdb_ref, a process per call)."""

    def __init__(self, taxdir):
        self.dir = taxdir

    def close(self):
        pass

    def _run(self, *args, stdin=b""):
        return subprocess.run([REF_TOOL, self.dir, *args], input=stdin, capture_output=True, check=True)

    def dump(self):
        return self._run("dump").stdout

    def fold(self, taxids, seg_start):
        """Fold of getLowestCommonAncestor over each segment taxids[seg_start[s]:seg_start[s+1]], in that order."""
        t = [str(int(x)) for x in np.asarray(taxids, np.uint64)]
        ss = [int(x) for x in seg_start]
        text = "".join(" ".join(t[ss[i]:ss[i + 1]]) + "\n" for i in range(len(ss) - 1))
        out = self._run("fold", stdin=text.encode()).stdout.split()
        return np.array([int(x) for x in out], np.uint64)

    def report(self, taxid, tax_count, tax_hash_count):
        """counts[taxid] = (taxCount, taxHashCount) -> (report bytes, rows (n, 5): taxid, taxCount, taxHashCount, cladeCount,
        cladeHashCount ascending taxid, (totalCount, totalHashCount))."""
        text = "".join(f"{int(a)} {int(b)} {int(c)}\n" for a, b, c in zip(taxid, tax_count, tax_hash_count))
        with tempfile.TemporaryDirectory() as d:
            rows_path = os.path.join(d, "rows.txt")
            report = self._run("report", rows_path, stdin=text.encode()).stdout
            lines = open(rows_path).read().split("\n")
        totals = tuple(int(x) for x in lines[0].split())
        rows = np.array([[int(x) for x in l.split()] for l in lines[1:] if l], np.uint64).reshape(-1, 5)
        return report, rows, totals


# ---- synthetic NCBI dumps ------------------------------------------------------------------------------------------------
RANKS = ["no rank", "superkingdom", "phylum", "class", "order", "family", "genus", "species", "species group", "strain"]
WORDS = ["Escherichia", "coli", "str.", "K-12", "substr.", "MG1655", "Bacillus", "subtilis", "virus", "phage", "sp.", "group",
         "uncultured", "bacterium", "Candidatus", "Homo", "sapiens", "clade", "alpha", "beta"]


class Taxonomy:
    """taxid -> parent taxid, rank, name of a synthetic dump (roots are their own parent)."""

    def __init__(self):
        self.parent, self.rank, self.name = {}, {}, {}

    def dense(self):
        """(parent index array, taxid array) in ascending taxid order, for mashgpu_taxonomy_open."""
        tids = np.array(sorted(self.parent), np.uint64)
        idx = {int(t): i for i, t in enumerate(tids)}
        return np.array([idx[self.parent[int(t)]] for t in tids], np.uint32), tids

    def is_lca_root(self, t):
        return self.parent[t] == t or t <= 1

    def fold_rule(self, taxids):
        """The order-free form of the fold of CommandTaxScreen.cpp:420-424 (DESIGN.md 4.2)."""
        nz = [int(t) for t in taxids if t != 0]
        if not nz:
            return 0
        if len(nz) == 1:
            return nz[0]
        if any(t not in self.parent for t in nz):
            return 1
        paths = []
        for t in set(nz):
            p = [t]
            while not self.is_lca_root(p[-1]):
                p.append(self.parent[p[-1]])
            paths.append(p)
        common = set(paths[0]).intersection(*map(set, paths[1:]))
        if not common:
            return 1
        lca = next(t for t in paths[0] if t in common)       # the deepest common node
        return 1 if self.is_lca_root(lca) else lca


def make_taxonomy(taxdir, seed, n_nodes=400, n_extra_roots=2, chain=60, dup_scientific=0.05, missing_name_entries=3):
    """Write nodes.dmp / names.dmp for a random forest under taxID 1 plus n_extra_roots more roots, with a chain of `chain`
    nodes, names with spaces and several name classes per taxID.  Lines are shuffled (parents may follow children).  Returns
    the Taxonomy the reference's parser must read (the last scientific name of a taxID wins)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    tax = Taxonomy()
    ids = [1] + [int(x) for x in rng.choice(np.arange(2, 3_000_000), n_nodes + n_extra_roots + chain, replace=False)]
    roots = ids[:1 + n_extra_roots]
    for r in roots:
        tax.parent[r] = r
    rest = ids[1 + n_extra_roots:]
    placed = list(roots)
    for t in rest[:n_nodes]:
        # favour recent nodes so that depth grows, but keep some wide fan-outs
        p = placed[int(rng.integers(max(0, len(placed) - 30), len(placed)))] if rng.random() < 0.6 else placed[int(rng.integers(0, len(placed)))]
        tax.parent[t] = p
        placed.append(t)
    prev = placed[int(rng.integers(0, len(placed)))]
    for t in rest[n_nodes:]:
        tax.parent[t] = prev
        prev = t
    node_lines, name_lines = [], []
    for t, p in tax.parent.items():
        tax.rank[t] = RANKS[int(rng.integers(0, len(RANKS)))]
        node_lines.append(f"{t}\t|\t{p}\t|\t{tax.rank[t]}\t|\tEC\t|\t{int(rng.integers(0, 12))}\t|\t1\t|\t11\t|\t1\t|\t0\t|\t1\t|\t0\t|\t0\t|\t\t|\n")
        names = [(" ".join(rng.choice(WORDS, int(rng.integers(1, 5)))) + f" {t}", "scientific name")]
        if rng.random() < dup_scientific:
            names.append((f"Renamed taxon {t}", "scientific name"))
        for cls in ("synonym", "authority", "genbank common name", "includes"):
            if rng.random() < 0.3:
                names.insert(int(rng.integers(0, len(names) + 1)), (" ".join(rng.choice(WORDS, 2)) + f" {cls} {t}", cls))
        for nm, cls in names:
            uniq = f"{nm} <{cls}>" if rng.random() < 0.2 else ""
            name_lines.append((t, f"{t}\t|\t{nm}\t|\t{uniq}\t|\t{cls}\t|\n"))
            if cls == "scientific name":
                tax.name[t] = nm
    for i in range(missing_name_entries):            # names of taxIDs that nodes.dmp lacks ("Entry for ... does not exist")
        name_lines.append((0, f"{9_000_000 + i}\t|\tGhost {i}\t|\t\t|\tscientific name\t|\n"))
    rng.shuffle(node_lines)
    # names keep their per-taxID order (it decides which scientific name wins) but taxa are interleaved at random
    order = rng.permutation(len(name_lines))
    by_t = {}
    for t, line in name_lines:
        by_t.setdefault(t, []).append(line)
    queues = {t: list(v) for t, v in by_t.items()}
    keys = [name_lines[i][0] for i in order]
    out_names = [queues[t].pop(0) for t in keys]
    os.makedirs(taxdir, exist_ok=True)
    with open(os.path.join(taxdir, "nodes.dmp"), "w") as f:
        f.writelines(node_lines)
    with open(os.path.join(taxdir, "names.dmp"), "w") as f:
        f.writelines(out_names)
    return tax


# ---- the checker -------------------------------------------------------------------------------------------------------
def segments(ref, ref_n, keys):
    """(d per (sketch, hash) pair sorted by d, sketch of each pair, seg_start (n_keys + 1))."""
    rows = np.repeat(np.arange(ref.shape[0]), ref_n.astype(np.int64))
    cols = np.concatenate([np.arange(n) for n in ref_n.astype(np.int64)] + [np.zeros(0, np.int64)])
    d = np.searchsorted(keys, ref[rows, cols]) if rows.size else np.zeros(0, np.int64)
    order = np.argsort(d, kind="stable")
    return d[order], rows[order], np.searchsorted(d[order], np.arange(keys.size + 1)).astype(np.uint64)


def taxscreen(oracle, reftax, ref, ref_n, chunks, po, ref_taxid, s=1000):
    """Everything `mash taxscreen` computes after the taxonomy and the sketch taxIDs are known: dict(keys, counts, set_size,
    hash_taxid (per key, ascending), rows (n, 5), totals, report)."""
    ref = np.ascontiguousarray(ref, np.uint64); ref_n = np.ascontiguousarray(ref_n, np.uint32)
    if tso.is_translated(po):
        scr = tso.screen(oracle, ref, ref_n, chunks, po, s=s)
    else:
        scr = oracle.screen(ref, ref_n, chunks, po, s=s)
    keys, counts = scr["keys"], scr["counts"][:scr["keys"].size]
    _, pair_ref, seg = segments(ref, ref_n, keys)
    hash_taxid = reftax.fold(np.asarray(ref_taxid, np.uint64)[pair_ref], seg)
    taxa, inv = np.unique(hash_taxid, return_inverse=True)
    thc = np.bincount(inv, minlength=taxa.size).astype(np.uint64)
    tc = np.bincount(inv, weights=(counts >= 1), minlength=taxa.size).astype(np.uint64)
    report, rows, totals = reftax.report(taxa, tc, thc)
    return dict(keys=keys, counts=counts, set_size=scr["set_size"], hash_taxid=hash_taxid, rows=rows, totals=totals, report=report)


def ref_codes(tax, ref_taxid):
    """(ref_code, unknown taxIDs) for mashgpu_screen_taxonomy: node index in Taxonomy.dense() order, a slot per distinct
    taxID outside the taxonomy, or TAX_NONE for taxID 0."""
    _, tids = tax.dense()
    idx = {int(t): i for i, t in enumerate(tids)}
    unknown = sorted({int(t) for t in ref_taxid if t != 0 and int(t) not in idx})
    uidx = {t: tids.size + u for u, t in enumerate(unknown)}
    code = [0xFFFFFFFF if t == 0 else idx.get(int(t), uidx.get(int(t))) for t in ref_taxid]
    return np.array(code, np.uint32), np.array(unknown, np.uint64)

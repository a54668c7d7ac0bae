#!/usr/bin/env python
"""Cost of the taxonomy step of `mash taxscreen` next to the screen pass it follows, on one GPU.

    python tools/taxscreen_bench.py [--sketches 100000] [--nodes 2700000] [--reads 10000000]

Workload: a 100 000-sketch nucleotide table (k=21, s=1000) of 2 000 families that share hashes (members keep 90-99 % of
their family's base sketch), an NCBI-sized synthetic taxonomy (2.7 M nodes, 28 levels below the root) with each family mapped
to a species and one member in ten to another species, and 150 bp random reads in '*'-joined chunks of 2 M reads resident in
HBM.  Timed: the screen pass (feed_dev of every chunk + finish), mashgpu_screen_taxonomy (wall clock and the device time of
its kernels, mashgpu_stats.taxonomy_ms), and on the host the dump parse and the report writer (`mash tax-report`).  The CPU
arm (the reference's TaxDB fold over this table on one thread) is not run here.  Prints one JSON line with the card name and
its power limit.  Writes only to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from translated_screen_bench import card_and_power_limit   # noqa: E402

MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


def taxonomy(rng, n_nodes, levels=28):
    """parent (dense indices, root 0 = taxID 1) and distinct taxIDs of a tree of `levels` levels growing geometrically."""
    sizes = np.maximum(1, np.round(np.geomspace(3, n_nodes / 4, levels))).astype(np.int64)
    sizes[-1] += n_nodes - 1 - sizes.sum()
    parent = [np.zeros(1, np.int64)]
    start = [0, 1]
    for sz in sizes:
        prev_lo, prev_hi = start[-2], start[-1]
        parent.append(rng.integers(prev_lo, prev_hi, sz))
        start.append(start[-1] + sz)
    parent = np.concatenate(parent).astype(np.uint32)
    taxid = np.concatenate([[1], rng.choice(np.arange(2, 4 * n_nodes), n_nodes - 1, replace=False)]).astype(np.uint64)
    return parent, taxid, start


def write_dump(d, parent, taxid):
    ranks = np.array(["no rank", "genus", "species"])
    with open(os.path.join(d, "nodes.dmp"), "w") as f:
        f.writelines(f"{t}\t|\t{taxid[p]}\t|\t{ranks[i % 3]}\t|\tEC\t|\t0\t|\t1\t|\t11\t|\t1\t|\t0\t|\t1\t|\t0\t|\t0\t|\t\t|\n"
                     for i, (t, p) in enumerate(zip(taxid.tolist(), parent.tolist())))
    with open(os.path.join(d, "names.dmp"), "w") as f:
        f.writelines(f"{t}\t|\tTaxon number {t}\t|\t\t|\tscientific name\t|\n{t}\t|\tsynonym of {t}\t|\t\t|\tsynonym\t|\n" for t in taxid.tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sketches", type=int, default=100_000)
    ap.add_argument("--families", type=int, default=2_000)
    ap.add_argument("--nodes", type=int, default=2_700_000)
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    import torch
    import mash_b200
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    rng = np.random.Generator(np.random.PCG64(args.seed))
    s, k = 1000, 21
    hi = int(2**64 * s / 5_000_000)
    base = np.sort(rng.integers(0, hi, (args.families, s), dtype=np.uint64), axis=1)
    fam = rng.integers(0, args.families, args.sketches)
    keep = rng.random((args.sketches, s)) < rng.uniform(0.90, 0.99, (args.sketches, 1))
    ref = np.where(keep, base[fam], rng.integers(0, hi, (args.sketches, s), dtype=np.uint64))
    ref.sort(axis=1)
    ref_n = np.full(args.sketches, s, np.uint32)
    parent, taxid, start = taxonomy(rng, args.nodes)
    leaves = np.arange(start[-2], start[-1])
    species = rng.choice(leaves, args.families)
    code = species[fam].astype(np.uint32)
    other = rng.random(args.sketches) < 0.1
    code[other] = rng.choice(leaves, int(other.sum()))
    eng = mash_b200.Engine(0)
    eng.set_timing(True)
    p = eng.params(k=k, s=s)
    # reads: 150 bp random, '*'-joined, chunks of 2 M reads in device memory
    per = 2_000_000
    n_chunks = max(1, args.reads // per)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    gen = torch.Generator(device=dev).manual_seed(args.seed)
    chunks = []
    for _ in range(n_chunks):
        c = acgt[torch.randint(0, 4, (per, 151), device=dev, generator=gen)]
        c[:, 0] = ord("*")
        chunks.append(torch.cat([c.reshape(-1), torch.zeros(16, dtype=torch.uint8, device=dev)]))
    tax = eng.taxonomy_open(parent, taxid)
    results = []
    for rep in range(3):                                   # the first repetition warms every shape up
        job = eng.screen_open(ref, ref_n, p)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c in chunks:
            job.feed_dev(c.data_ptr(), c.numel() - 16)
        job.finish()
        t1 = time.perf_counter()
        eng.stats(reset=True)
        out = job.taxonomy(tax, code)
        t2 = time.perf_counter()
        st = eng.stats(reset=True)
        job.close()
        results.append(dict(screen_s=t1 - t0, taxonomy_wall_ms=(t2 - t1) * 1e3, taxonomy_device_ms=st["taxonomy_ms"],
                            rows=int(out["rows"].size), distinct_hashes=int(out["total_hash_count"])))
    tax.close()
    with tempfile.TemporaryDirectory() as d:
        write_dump(d, parent, taxid)
        rows = os.path.join(d, "rows.txt")
        with open(rows, "w") as f:
            f.write("0 0\n")
        t0 = time.perf_counter()
        subprocess.run([MASH, "tax-report", d, rows], check=True, capture_output=True)
        parse_s = time.perf_counter() - t0
        with open(rows, "w") as f:                     # the last pass's rows, with every seen count set so the whole tree prints
            f.write(f"{out['total_hash_count']} {out['total_hash_count']}\n")
            f.writelines(f"{r['taxid']} {r['tax_hash_count']} {r['tax_hash_count']} {r['clade_hash_count']} {r['clade_hash_count']}\n"
                         for r in out["rows"])
        t0 = time.perf_counter()
        rep_out = subprocess.run([MASH, "tax-report", d, rows], check=True, capture_output=True).stdout
        report_s = time.perf_counter() - t0 - parse_s
    last = results[1:]
    print(json.dumps(dict(card=card, power_limit_w=limit, sketches=args.sketches, nodes=args.nodes, reads=n_chunks * per,
                          screen_s=[round(r["screen_s"], 4) for r in last],
                          taxonomy_device_ms=[round(r["taxonomy_device_ms"], 3) for r in last],
                          taxonomy_wall_ms=[round(r["taxonomy_wall_ms"], 3) for r in last],
                          taxonomy_share_of_screen=[round(r["taxonomy_wall_ms"] / 1e3 / r["screen_s"], 4) for r in last],
                          rows=last[-1]["rows"], distinct_hashes=last[-1]["distinct_hashes"],
                          host_parse_s=round(parse_s, 3), host_report_s=round(report_s, 3), report_lines=rep_out.count(b"\n"),
                          cpu_reference_fold="not measured")))


if __name__ == "__main__":
    main()

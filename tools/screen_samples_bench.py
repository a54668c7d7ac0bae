#!/usr/bin/env python
"""Per-sample cost of screening a cohort against one table, on one GPU: a fresh job per sample against one resident job with
the dense finish or the sparse finish (mashgpu_screen_finish_hits), reset between samples.

    python tools/screen_samples_bench.py [--sketches 100000] [--small 40] [--large 3]

Workload: a 100 000-sketch s=1000 k=21 table from bench.py's make_sketches_device, in which 2 000 rows are replaced by the
sketches of 40 genomes of 1 Mbp from bench.py's make_genomes_device (50 rows per genome, so each of their hashes is held by 50
sketches).  Samples are 150 bp reads drawn from those genomes, '*'-joined in chunks of up to 2 M reads resident in HBM (fed
with feed_dev, so no host parse is timed): `--small` samples of 10^4 reads and `--large` samples of 10^7 reads.  Routes per sample:
  fresh   open, feed, finish, close (what one process per sample pays on the GPU, without the process and context start-up)
  dense   one job: feed, finish, reset
  sparse  one job: feed, finish_hits, reset (the index is built on a warm-up sample first and reported on its own)
Per route: wall time per sample (host clock around work that ends in a device synchronise) and the finish's time (wall clock
of finish(), which ends in a synchronise, or the CUDA-event device time of finish_hits).  The three routes' outputs are checked
to be identical on every timed sample.  Prints one JSON line with the card name and its power limit.  Writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import make_genomes_device, make_sketches_device   # noqa: E402
from translated_screen_bench import card_and_power_limit      # noqa: E402

READ = 150
PER_CHUNK = 2_000_000


def make_sample(torch, dev, stream, n_units, span, glen, n_reads, gen):
    """'*'-joined reads of READ bases from random genomes and offsets, as device chunks (each padded by 16 bytes)."""
    chunks = []
    for r0 in range(0, n_reads, PER_CHUNK):
        m = min(PER_CHUNK, n_reads - r0)
        u = torch.randint(0, n_units, (m,), device=dev, generator=gen)
        a = torch.randint(0, glen - READ, (m,), device=dev, generator=gen)
        c = torch.empty((m, READ + 1), dtype=torch.uint8, device=dev)
        c[:, 0] = ord("*")
        for b0 in range(0, m, 500_000):
            b1 = min(m, b0 + 500_000)
            idx = (u[b0:b1] * span + a[b0:b1])[:, None] + torch.arange(READ, device=dev)[None, :]
            c[b0:b1, 1:] = stream[idx]
            del idx
        chunks.append(torch.cat([c.reshape(-1), torch.zeros(16, dtype=torch.uint8, device=dev)]))
    return chunks


def feed(job, chunks):
    for c in chunks:
        job.feed_dev(c.data_ptr(), c.numel() - 16)


def run_routes(torch, eng, ref, ref_n, p, samples):
    """Times the three routes over the samples; returns per-route lists and the outputs for the cross-check."""
    res = {"fresh": [], "dense": [], "sparse": []}
    out = {"fresh": [], "dense": [], "sparse": []}
    for smp in samples:                                        # fresh job per sample
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        job = eng.screen_open(ref, ref_n, p)
        feed(job, smp)
        t1 = time.perf_counter()
        f = job.finish()
        t2 = time.perf_counter()
        job.close()
        t3 = time.perf_counter()
        res["fresh"].append(dict(wall_ms=(t3 - t0) * 1e3, finish_ms=(t2 - t1) * 1e3))
        out["fresh"].append(f)
    for route in ("dense", "sparse"):
        job = eng.screen_open(ref, ref_n, p)
        feed(job, samples[0][:1])
        if route == "sparse":
            job.finish_hits()                                  # builds the index
            index_ms = job.hits_stats()["index_ms"]
        else:
            job.finish()
        job.reset()
        for smp in samples:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            feed(job, smp)
            t1 = time.perf_counter()
            f = job.finish() if route == "dense" else job.finish_hits()
            t2 = time.perf_counter()
            job.reset()
            t3 = time.perf_counter()
            r = dict(wall_ms=(t3 - t0) * 1e3, finish_ms=(t2 - t1) * 1e3)
            if route == "sparse":
                st = job.hits_stats()
                r.update(finish_device_ms=st["finish_ms"], hit_hashes=st["hit_hashes"], hit_pairs=st["hit_pairs"], rows=int(f["ref"].size))
            res[route].append(r)
            out[route].append(f)
        job.close()
    for fr, de, sp in zip(out["fresh"], out["dense"], out["sparse"]):
        for key in ("shared", "median", "identity", "pvalue"):
            assert np.array_equal(fr[key], de[key]), key
            rows = np.flatnonzero(fr["shared"] >= 1)
            assert np.array_equal(sp["ref"], rows.astype(np.uint32)) and np.array_equal(sp[key], fr[key][rows]), key
        assert fr["set_size"] == de["set_size"] == sp["set_size"]
    return res, index_ms


def summary(rows, key):
    v = np.array([r[key] for r in rows], np.float64)
    return dict(median=round(float(np.median(v)), 3), min=round(float(v.min()), 3), max=round(float(v.max()), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sketches", type=int, default=100_000)
    ap.add_argument("--genomes", type=int, default=40)
    ap.add_argument("--small", type=int, default=40)
    ap.add_argument("--large", type=int, default=3)
    ap.add_argument("--small-reads", type=int, default=10_000)
    ap.add_argument("--large-reads", type=int, default=10_000_000)
    ap.add_argument("--seed", type=int, default=3)
    args = ap.parse_args()
    import torch
    import mash_b200
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    s, k, glen, copies = 1000, 21, 1_000_000, 50
    eng = mash_b200.Engine(0)
    p = eng.params(k=k, s=s)
    H, N, _ = make_sketches_device(torch, dev, args.sketches, s, args.seed)
    ref = H.cpu().numpy().view(np.uint64)
    ref_n = N.cpu().numpy().astype(np.uint32)
    del H, N
    stream, unit_start = make_genomes_device(torch, dev, args.genomes, glen, args.seed + 1)
    span = glen + 1
    host = stream[:args.genomes * span].cpu().numpy()
    gh, gn, _ = eng.sketch([host[u * span:u * span + glen].tobytes() for u in range(args.genomes)], p)
    for u in range(args.genomes):                              # 50 rows per genome, spread over the table
        rows = np.arange(copies) * (args.sketches // copies) + u
        ref[rows] = np.uint64(2**64 - 1)
        ref[rows, :gn[u]] = gh[u, :gn[u]]
        ref_n[rows] = gn[u]
    gen = torch.Generator(device=dev).manual_seed(args.seed + 2)
    out = dict(card=card, power_limit_w=limit, sketches=args.sketches, s=s, k=k, genome_rows=args.genomes * copies)
    for name, n_samples, n_reads in (("small", args.small, args.small_reads), ("large", args.large, args.large_reads)):
        samples = [make_sample(torch, dev, stream, args.genomes, span, glen, n_reads, gen) for _ in range(n_samples)]
        res, index_ms = run_routes(torch, eng, ref, ref_n, p, samples)
        d = dict(samples=n_samples, reads_per_sample=n_reads, index_build_ms=round(index_ms, 3))
        for route, rows in res.items():
            d[route] = dict(wall_ms=summary(rows, "wall_ms"), finish_ms=summary(rows, "finish_ms"),
                            window_s=round(sum(r["wall_ms"] for r in rows) / 1e3, 3))
        sp = res["sparse"]
        d["sparse"].update(finish_device_ms=summary(sp, "finish_device_ms"), hit_hashes=summary(sp, "hit_hashes"),
                           hit_pairs=summary(sp, "hit_pairs"), rows=summary(sp, "rows"))
        d["outputs_identical"] = True
        out[name] = d
        del samples
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Best hits of dist (DistJob.run_best) on one GPU, next to what a caller did without it: the dense grid to the host, then numpy.

    python tools/dist_best_bench.py [--refs 100000] [--queries 10000] [--s 1000] [--n-best 10] [--dense-queries 2000]
                                    [--family 20000] [--repeats 3] [--out DIR]

Sets: bench.make_sketches_device (the configs[2] generator: 100 families stored family by family).  Fails without a GPU.
  search   `queries` sketches (every (refs/queries)-th of the set, so each has its family among the references) against `refs`
           references: wall clock and pairs/s of run_best over all queries, candidates per query, block splits, and the CUDA-event
           time of grouping + dist_best_kernel as a share of the run
  compare  the first `dense-queries` of them both ways, alternated `repeats` times: run_best, and run (dense numer / distance /
           pass on the host, in blocks of 500 queries) followed by numpy.argpartition and a sort of the kept few; both must
           return the same lists
  self     the `refs` x `refs` self job (short segments: ~refs/100 hits per query)
  family   a one-family set of `family` sketches against itself: every pair is a hit (long segments, blocks split)
Prints one JSON line with the card name and its power limit read in the same run (and writes OUT/dist_best_bench.json).
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
import bench                                                # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402


def timed_best(torch, job, q0, qn, n_best):
    before = job.best_stats()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = job.run_best(q0, qn, n_best)
    dt = time.perf_counter() - t0
    after = job.best_stats()
    d = {k: after[k] - before[k] for k in after}
    return res, dict(seconds=dt, pairs_per_s=qn * job.n_ref / dt, candidates_per_query=d["candidates"] / max(1, qn), blocks_run=d["blocks_run"],
                     blocks_split=d["blocks_split"], select_ms=d["select_ms"], select_share=d["select_ms"] / 1e3 / dt)


def dense_then_numpy(job, q0, qn, n_best, block=500):
    """the caller's way without run_best: dense outputs to the host, argpartition per row, sort of the kept entries"""
    t0 = time.perf_counter()
    refs, dists = [], []
    for b in range(q0, q0 + qn, block):
        g = job.run(b, min(block, q0 + qn - b), outputs=("numer", "distance", "pass"))
        d = np.where(g["pass"] & (g["numer"] > 0), g["distance"], np.inf)
        kth = min(n_best, d.shape[1] - 1)
        part = np.argpartition(d, kth, axis=1)[:, :n_best]        # unordered n_best smallest; ties at the cut are broken below
        for i in range(d.shape[0]):
            cut = np.sort(d[i, part[i]])[-1]
            cand = np.flatnonzero(d[i] <= cut)
            cand = cand[np.lexsort((cand, d[i, cand]))][:n_best]
            cand = cand[np.isfinite(d[i, cand])]
            refs.append(cand); dists.append(d[i, cand])
    return refs, dists, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--refs", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--n-best", type=int, default=10)
    ap.add_argument("--dense-queries", type=int, default=2000)
    ap.add_argument("--family", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    if not torch.cuda.is_available():
        sys.exit("dist_best_bench: no CUDA device (the measurement does not fall back to anything)")
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    eng = mash_b200.Engine(0)
    eng.set_timing(True)
    n, s, nb = args.refs, args.s, args.n_best
    out = dict(card=card, power_limit_w=limit, n_best=nb, s=s)
    H, N, L = bench.make_sketches_device(torch, dev, n, s, 1)
    pick = torch.arange(0, n, max(1, n // args.queries), device=dev)[:args.queries]
    Hq, Nq, Lq = H[pick].contiguous(), N[pick].contiguous(), L[pick].contiguous()
    torch.cuda.synchronize()
    ref = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=n, stride=s)
    qry = _Set(Hq.data_ptr(), Nq.data_ptr(), Lq.data_ptr(), on_device=True, n=pick.numel(), stride=s)
    kspace = 4.0 ** 21

    job = eng.dist_open(ref, None, None, qry, None, None, sketch_size=s, k=21, kmer_space=kspace)
    nq = job.n_qry
    job.run_best(0, nq, nb)                                     # warm-up: buffers grown, modules loaded
    runs = [timed_best(torch, job, 0, nq, nb)[1] for _ in range(args.repeats)]
    out["search"] = dict(queries=nq, refs=n, runs=runs, seconds_min=min(r["seconds"] for r in runs), seconds_max=max(r["seconds"] for r in runs))
    dq = min(args.dense_queries, nq)
    dense_then_numpy(job, 0, min(dq, 500), nb)                  # warm-up
    cmp_best, cmp_dense, same = [], [], True
    for _ in range(args.repeats):
        res, st = timed_best(torch, job, 0, dq, nb)
        refs, dists, dt = dense_then_numpy(job, 0, dq, nb)
        cmp_best.append(st["seconds"]); cmp_dense.append(dt)
        for i in range(dq):
            h = res["n_hits"][i]
            same &= h == refs[i].size and np.array_equal(res["ref"][i, :h], refs[i]) and np.array_equal(res["distance"][i, :h], dists[i])
    out["compare"] = dict(queries=dq, refs=n, run_best_seconds=cmp_best, dense_numpy_seconds=cmp_dense, same_lists=bool(same),
                          speedup_min=min(cmp_dense) / max(cmp_best), speedup_max=max(cmp_dense) / min(cmp_best))
    job.close()

    job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=kspace)
    job.run_best(0, min(n, 20_000), nb)
    runs = [timed_best(torch, job, 0, n, nb)[1] for _ in range(args.repeats)]
    out["self"] = dict(n=n, runs=runs)
    job.close()
    del H, N, L, Hq, Nq, Lq
    torch.cuda.empty_cache()

    m = args.family
    H, N, L = bench.make_sketches_device(torch, dev, m, s, 3, n_families=1)
    torch.cuda.synchronize()
    fam = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=m, stride=s)
    job = eng.dist_open(fam, None, None, sketch_size=s, k=21, kmer_space=kspace)
    job.run_best(0, m, nb)
    runs = [timed_best(torch, job, 0, m, nb)[1] for _ in range(args.repeats)]
    # the same run when nothing is discarded: a capacity that holds every hit of the set
    job.set_best_capacity(m * m)
    job.run_best(0, m, nb)
    runs_fit = [timed_best(torch, job, 0, m, nb)[1] for _ in range(args.repeats)]
    out["family"] = dict(n=m, runs=runs, runs_capacity_fits=runs_fit)
    job.close()

    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_best_bench.json"), "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

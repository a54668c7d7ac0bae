#!/usr/bin/env python
"""Connected components of dist (DistJob.components) on one GPU, next to what a caller did without it: the pass list of the lower
triangle to the host (DistJob.run_list), then scipy.sparse.csgraph.connected_components on the same edges.

    python tools/dist_components_bench.py [--n 100000] [--s 1000] [--cuts 0.05,0.3] [--family 20000] [--big 0] [--repeats 3]
                                          [--out DIR]

Sets: bench.make_sketches_device (the configs[2] generator: 100 families stored family by family).  Fails without a GPU.
  cut      for each -d cut-off: components() and run_list + scipy, alternated `repeats` times; both must give the same labels
  family   a one-family set of `family` sketches: every pair that shares a hash is an edge (contention on few roots)
  big      (if --big > 0) components() on a set of that many sketches, 1000 per family (the dist5 set of bench.py at 10^6)
Reports wall clock and edges absorbed per second, with the card name and its power limit read in the same run, as one JSON line
(and OUT/dist_components_bench.json).
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


def timed_components(torch, job):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    labels, n_edges = job.components()
    dt = time.perf_counter() - t0
    return labels, n_edges, dt


def list_then_scipy(job, n, block=10_000, capacity=1 << 25):
    """the caller's way without components(): passing pairs of the lower triangle to the host, then scipy"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t0 = time.perf_counter()
    job.set_triangle(True)
    qs, rs = [], []
    for q0 in range(0, n, block):
        qn = min(block, n - q0)
        cap = capacity
        while True:
            n_pass, lst = job.run_list(q0, qn, cap)
            if n_pass <= cap:
                break
            cap = int(n_pass * 1.1) + 1
        keep = lst["numer"] > 0
        idx = lst["index"][keep]
        qs.append(q0 + idx // n); rs.append(idx % n)
    job.set_triangle(False)
    q = np.concatenate(qs).astype(np.int64); r = np.concatenate(rs).astype(np.int64)
    t1 = time.perf_counter()
    g = coo_matrix((np.ones(q.size, np.int8), (q, r)), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    first = np.full(comp.max() + 1, n, np.int64)
    np.minimum.at(first, comp, np.arange(n))
    labels = first[comp]
    t2 = time.perf_counter()
    return labels, q.size, t2 - t0, t1 - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--cuts", default="0.05,0.3")
    ap.add_argument("--family", type=int, default=20_000)
    ap.add_argument("--big", type=int, default=0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    if not torch.cuda.is_available():
        sys.exit("dist_components_bench: no CUDA device (the measurement does not fall back to anything)")
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    eng = mash_b200.Engine(0)
    n, s = args.n, args.s
    kspace = 4.0 ** 21
    out = dict(card=card, power_limit_w=limit, n=n, s=s)
    H, N, L = bench.make_sketches_device(torch, dev, n, s, 1)
    torch.cuda.synchronize()
    ref = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=n, stride=s)
    out["cuts"] = []
    for cut in (float(x) for x in args.cuts.split(",")):
        job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=kspace, max_distance=cut)
        timed_components(torch, job)                        # warm-up: buffers grown, modules loaded
        gpu_s, host_s, list_s, same = [], [], [], True
        for _ in range(args.repeats):
            labels, n_edges, dt = timed_components(torch, job)
            want, e_host, dt_host, dt_list = list_then_scipy(job, n)
            gpu_s.append(dt); host_s.append(dt_host); list_s.append(dt_list)
            same &= bool(np.array_equal(labels, want)) and n_edges == e_host
        job.close()
        out["cuts"].append(dict(max_distance=cut, edges=n_edges, clusters=int(np.unique(labels).size), components_seconds=gpu_s,
                                list_scipy_seconds=host_s, list_part_seconds=list_s, same_labels=same,
                                edges_per_s=n_edges / min(gpu_s), speedup_min=min(host_s) / max(gpu_s), speedup_max=max(host_s) / min(gpu_s)))
    del H, N, L
    torch.cuda.empty_cache()

    m = args.family
    H, N, L = bench.make_sketches_device(torch, dev, m, s, 3, n_families=1)
    torch.cuda.synchronize()
    fam = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=m, stride=s)
    job = eng.dist_open(fam, None, None, sketch_size=s, k=21, kmer_space=kspace)
    timed_components(torch, job)
    runs = [timed_components(torch, job) for _ in range(args.repeats)]
    job.close()
    out["family"] = dict(n=m, edges=runs[0][1], clusters=int(np.unique(runs[0][0]).size), seconds=[r[2] for r in runs],
                         edges_per_s=runs[0][1] / min(r[2] for r in runs), repeatable=all(np.array_equal(r[0], runs[0][0]) for r in runs))
    del H, N, L
    torch.cuda.empty_cache()

    if args.big > 0:
        m = args.big
        H, N, L = bench.make_sketches_device(torch, dev, m, s, 5, n_families=max(1, m // 1000))
        torch.cuda.synchronize()
        big = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=m, stride=s)
        job = eng.dist_open(big, None, None, sketch_size=s, k=21, kmer_space=kspace, max_distance=0.05)
        labels, n_edges, dt = timed_components(torch, job)
        job.close()
        out["big"] = dict(n=m, max_distance=0.05, edges=n_edges, clusters=int(np.unique(labels).size), seconds=dt, edges_per_s=n_edges / dt,
                          pairs_per_s=m * (m - 1) / 2 / dt)

    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_components_bench.json"), "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

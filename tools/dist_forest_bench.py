#!/usr/bin/env python
"""Minimum spanning forest of dist (DistJob.spanning_forest) on one GPU, with DistJob.components on the same set beside it.

    python tools/dist_forest_bench.py [--n 100000] [--s 1000] [--cuts 1.0,0.05] [--family 20000] [--repeats 3] [--out DIR]

Sets: bench.make_sketches_device (the configs[2] generator: 100 families stored family by family).  Fails without a GPU.
  cut      for each -d cut-off: spanning_forest() and components(), alternated `repeats` times; the forest must span the components
  family   a one-family set of `family` sketches, where most pairs share a hash (contention of the 128-bit CAS on few slots).  Also
           the dense distance grid to the host and Prim's algorithm there, over all pairs: a pair without a shared hash has distance 1,
           so Prim's sorted weights must be the forest's plus one 1.0 per join of two trees.
Reports the wall clock of the whole call, the Boruvka rounds and the mean time per round (the call does not time its rounds one by
one), with the card name and its power limit read in the same run, as one JSON line (and OUT/dist_forest_bench.json).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench                                                # noqa: E402
from forest_model import forest_labels                      # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t0


def host_prim_weights(job, n, block=2000):
    """sorted weights of a minimum spanning tree of the complete graph of distances: the dense distance grid to the host, then Prim's
    algorithm there"""
    t0 = time.perf_counter()
    d = np.empty((n, n), np.float64)
    for q0 in range(0, n, block):
        d[q0:q0 + block] = job.run(q0, min(block, n - q0), outputs=("distance",))["distance"]
    t1 = time.perf_counter()
    key = d[0].copy()
    in_tree = np.zeros(n, bool)
    in_tree[0] = True
    key[0] = np.inf
    w = np.empty(n - 1)
    for t in range(n - 1):
        v = int(np.argmin(key))
        w[t] = key[v]
        in_tree[v] = True
        np.minimum(key, d[v], out=key)
        key[in_tree] = np.inf
    return np.sort(w), t1 - t0, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--cuts", default="1.0,0.05")
    ap.add_argument("--family", type=int, default=20_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    if not torch.cuda.is_available():
        sys.exit("dist_forest_bench: no CUDA device (the measurement does not fall back to anything)")
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
    for cut in (float(x) for x in args.cuts.split(",") if x):
        job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=kspace, max_distance=cut)
        job.spanning_forest()                               # warm-up: modules loaded
        job.components()
        f_s, cc_s, same = [], [], True
        for _ in range(args.repeats):
            f, dt = timed(torch, job.spanning_forest)
            (labels, n_edges), dc = timed(torch, job.components)
            f_s.append(dt); cc_s.append(dc)
            same &= bool(np.array_equal(forest_labels(n, f["row"], f["col"]), labels))
        job.close()
        out["cuts"].append(dict(max_distance=cut, graph_edges=n_edges, forest_edges=int(len(f["row"])), trees=n - int(len(f["row"])),
                                rounds=f["rounds"], forest_seconds=f_s, seconds_per_round=min(f_s) / max(f["rounds"], 1),
                                components_seconds=cc_s, forest_spans_the_components=same))
    del H, N, L
    torch.cuda.empty_cache()

    m = args.family
    H, N, L = bench.make_sketches_device(torch, dev, m, s, 3, n_families=1)
    torch.cuda.synchronize()
    fam = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=m, stride=s)
    job = eng.dist_open(fam, None, None, sketch_size=s, k=21, kmer_space=kspace)
    job.spanning_forest()
    runs = [timed(torch, job.spanning_forest) for _ in range(args.repeats)]
    (labels, n_edges), dc = timed(torch, job.components)
    f = runs[0][0]
    w, grid_s, host_s = host_prim_weights(job, m)
    job.close()
    out["family"] = dict(n=m, graph_edges=n_edges, forest_edges=int(len(f["row"])), rounds=f["rounds"], forest_seconds=[r[1] for r in runs],
                         seconds_per_round=min(r[1] for r in runs) / max(f["rounds"], 1), components_seconds=dc,
                         repeatable=all(all(np.array_equal(r[0][k], f[k]) for k in ("row", "col", "distance")) for r in runs),
                         grid_to_host_seconds=grid_s, grid_and_host_prim_seconds=host_s, same_weights_as_host=bool(np.array_equal(w, np.sort(np.concatenate([f["distance"], np.ones(m - 1 - len(f["row"]))])))))
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_forest_bench.json"), "w") as fo:
            fo.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

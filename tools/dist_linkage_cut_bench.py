#!/usr/bin/env python
"""The linkage cut per component (DESIGN.md 3.13) on one GPU: device time per phase and component sizes.

    python tools/dist_linkage_cut_bench.py [--sizes 100000,30000] [--ts 0.05,0.1] [--s 1000] [--family 20000] [--dense-max 30000]
                                           [--out DIR]

Sets: bench.make_sketches_device (the configs[2] generator: 100 families stored family by family).  Fails without a GPU.
  size    for each n, method and t: DistJob.linkage_cut end to end (wall clock with a device synchronise around it, after a warm-up
          call) and its four phases (DistJob.linkage_cut_stats: components, grouping, CTA tier, matrix tier, CUDA events), the
          component count, the largest component and a histogram of component sizes; with n <= --dense-max also the dense route
          (DistJob.linkage then the cut), timed, and whether it gives the same labels.
  family  one family of --family sketches (one large component at every t), against DistJob.linkage.
Prints one JSON line (and OUT/dist_linkage_cut_bench.json) with the card name and its power limit read in the same run.
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
from linkage_cut_model import smallest_labels              # noqa: E402
from linkage_model import METHODS, cut                      # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402

EDGES = [1, 2, 3, 5, 9, 17, 33, 65, 129, 239, 513, 1025, 4097, 16385, 1 << 62]


def timed(torch, f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def histogram(labels_of_components):
    sizes = np.bincount(np.unique(labels_of_components, return_inverse=True)[1])
    h, _ = np.histogram(sizes, bins=EDGES)
    return {f"{lo}-{hi - 1}" if hi - 1 > lo else str(lo): int(c) for lo, hi, c in zip(EDGES[:-1], EDGES[1:], h) if c}


def run_set(torch, job, n, ts, dense, out_list, what):
    job.linkage_cut("average", ts[0])                     # warm-up: modules loaded, every kernel of the path run once
    for method in METHODS:
        whole = whole_s = None
        if dense:
            whole, whole_s = timed(torch, lambda: job.linkage(method))
        for t in ts:
            got, dt = timed(torch, lambda: job.linkage_cut(method, t))
            e = dict(set=what, n=n, method=method, t=t, seconds=dt, phases_ms=job.linkage_cut_stats(), n_components=got["n_components"],
                     largest_component=got["largest_component"], n_clusters=got["n_clusters"])
            if dense:
                e["dense_seconds"] = whole_s
                e["dense_equal_labels"] = bool(np.array_equal(smallest_labels(cut(whole, n, t)), got["labels"]))
            out_list.append(e)
    return job


def component_histogram(eng, ref, s, n, t, kmer_space):
    from linkage_cut_model import threshold
    job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=kmer_space, max_distance=threshold(t, n), max_pvalue=1.0)
    try:
        return histogram(job.components()[0])
    finally:
        job.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", default="100000,30000")
    ap.add_argument("--ts", default="0.05,0.1")
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--family", type=int, default=20000)
    ap.add_argument("--dense-max", type=int, default=30000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    if not torch.cuda.is_available():
        sys.exit("dist_linkage_cut_bench: no CUDA device (the measurement does not fall back to anything)")
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    eng = mash_b200.Engine(0)
    s, ts, ks = args.s, [float(x) for x in args.ts.split(",")], 4.0 ** 21
    out = dict(card=card, power_limit_w=limit, s=s, runs=[], histograms=[])
    for n in (int(x) for x in args.sizes.split(",") if x):
        H, N, L = bench.make_sketches_device(torch, dev, n, s, 1)
        torch.cuda.synchronize()
        ref = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=n, stride=s)
        job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=ks)
        run_set(torch, job, n, ts, n <= args.dense_max, out["runs"], "configs2")
        job.close()
        for t in ts:
            out["histograms"].append(dict(set="configs2", n=n, t=t, sizes=component_histogram(eng, ref, s, n, t, ks)))
        del H, N, L, ref
        torch.cuda.empty_cache()
    if args.family:
        n = args.family
        H, N, L = bench.make_sketches_device(torch, dev, n, s, 2, n_families=1)
        torch.cuda.synchronize()
        ref = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=n, stride=s)
        job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=ks)
        run_set(torch, job, n, ts, True, out["runs"], "one_family")
        job.close()
        for t in ts:
            out["histograms"].append(dict(set="one_family", n=n, t=t, sizes=component_histogram(eng, ref, s, n, t, ks)))
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_linkage_cut_bench.json"), "w") as fo:
            fo.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Average and complete linkage of dist (DESIGN.md 3.11) on one GPU: the matrix fill and the merges timed apart.

    python tools/dist_linkage_bench.py [--sizes 10000,30000] [--s 1000] [--repeats 2] [--cpu] [--out DIR]

Sets: bench.make_sketches_device (the configs[2] generator: 100 families stored family by family).  Fails without a GPU.
  size   for each n and method: the lower triangle of the self job's distances into an n x n device matrix (DistJob.run_dev,
         distance only) and Engine.linkage_matrix on it, each timed with a device synchronise around it, `repeats` times after a
         warm-up (the merges overwrite the matrix, so every repeat refills it); then DistJob.linkage end to end once, which must
         give the same merges bit for bit.  Rows rescanned are the device's count; the bytes they read are at most 8 (n - 1) per
         row, and exactly the cache model's count (tests/linkage_model.py, replayed on the host) on the first set.
  cpu    on the first set: the dense grid to the host, squareform and scipy's linkage, against the GPU merges: the same fcluster
         partitions at t = 0.05 and 0.1 and cophenetic distances within 1e-12; both clocks.
Prints one JSON line (and OUT/dist_linkage_bench.json) with the card name and its power limit read in the same run.
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
from dist_nj_bench import fill, timed                       # noqa: E402
from linkage_model import METHODS, linkage_cached           # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402


def same(x, y):
    return all(np.array_equal(x[k], y[k]) for k in ("id_lo", "id_hi", "size")) and \
        np.array_equal(x["height"].view(np.uint64), y["height"].view(np.uint64)) and x.get("rows_rescanned") == y.get("rows_rescanned")


def same_partition(a, b):
    return len(set(zip(a.tolist(), b.tolist()))) == len(set(a.tolist())) == len(set(b.tolist()))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", default="10000,30000")
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--cpu", action="store_true", help="the scipy arm and the model's byte count on the first set")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    if not torch.cuda.is_available():
        sys.exit("dist_linkage_bench: no CUDA device (the measurement does not fall back to anything)")
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    eng = mash_b200.Engine(0)
    s = args.s
    out = dict(card=card, power_limit_w=limit, s=s, sizes=[])
    for i, n in enumerate(int(x) for x in args.sizes.split(",") if x):
        H, N, L = bench.make_sketches_device(torch, dev, n, s, 1)
        torch.cuda.synchronize()
        ref = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=n, stride=s)
        job = eng.dist_open(ref, None, None, sketch_size=s, k=21, kmer_space=4.0 ** 21)
        job.set_triangle(True)
        M = torch.empty((n, n), dtype=torch.float64, device=dev)
        small = min(n, 200)                               # warm-up: modules loaded, every kernel run once
        for method in METHODS:
            fill(torch, job, M, small)
            eng.linkage_matrix(M, small, ld=n, method=method)
        entry = dict(n=n, merges=n - 1, methods={})
        for method in METHODS:
            fill_s, link_s, first, repeatable = [], [], None, True
            for _ in range(args.repeats):
                _, dt = timed(torch, lambda: fill(torch, job, M, n))
                fill_s.append(dt)
                eng.stats(reset=True)
                r, dt = timed(torch, lambda: eng.linkage_matrix(M, n, method=method))
                launches = eng.stats()["kernel_launches"]
                link_s.append(dt)
                repeatable &= first is None or same(r, first)
                first = first or r
            rows = first["rows_rescanned"]
            entry["methods"][method] = dict(fill_seconds=fill_s, linkage_seconds=link_s, repeatable=bool(repeatable), rows_rescanned=rows,
                                            rows_per_merge=rows / (n - 1), rescan_bytes_at_most=8.0 * (n - 1) * rows,
                                            launches_per_merge=(launches - 3) / (n - 1),
                                            last_height_below_an_earlier=bool((np.diff(first["height"]) < 0).any()))
            entry["methods"][method]["_merges"] = first
        del M
        torch.cuda.empty_cache()
        for method in METHODS:
            whole, whole_s = timed(torch, lambda: job.linkage(method))
            e = entry["methods"][method]
            e["job_seconds"] = whole_s
            e["job_equals_matrix_entry"] = bool(same(whole, e["_merges"]))
        if i == 0 and args.cpu:
            D = job.run(0, n, outputs=("distance",))["distance"]
            from scipy.cluster.hierarchy import cophenet, fcluster, linkage
            from scipy.spatial.distance import squareform
            t0 = time.perf_counter()
            D2 = job.run(0, n, outputs=("distance",))["distance"]
            cond = squareform(np.tril(D2, -1) + np.tril(D2, -1).T, checks=False)
            to_host_s = time.perf_counter() - t0
            cpu = dict(n=n, grid_to_host_and_squareform_seconds=to_host_s, methods={})
            for method in METHODS:
                t0 = time.perf_counter()
                Z = linkage(cond, method=method)
                scipy_s = time.perf_counter() - t0
                g = entry["methods"][method]["_merges"]
                ours = mash_b200.linkage_z(g)
                model, rows, read = linkage_cached(D, method)
                entry["methods"][method]["rescan_bytes"] = read
                cpu["methods"][method] = dict(
                    scipy_linkage_seconds=scipy_s,
                    gpu_job_seconds=entry["methods"][method]["job_seconds"],
                    same_fcluster_005=same_partition(fcluster(Z, 0.05, "distance"), fcluster(ours, 0.05, "distance")),
                    same_fcluster_01=same_partition(fcluster(Z, 0.1, "distance"), fcluster(ours, 0.1, "distance")),
                    cophenet_max_abs_diff=float(np.abs(cophenet(Z) - cophenet(ours)).max()),
                    model_equals_gpu=bool(same(dict(model, rows_rescanned=rows), g)))
            out["cpu"] = cpu
        for method in METHODS:
            del entry["methods"][method]["_merges"]
        out["sizes"].append(entry)
        job.close()
        del H, N, L
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_linkage_bench.json"), "w") as fo:
            fo.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

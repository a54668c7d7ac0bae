#!/usr/bin/env python
"""Neighbor joining of dist (DESIGN.md 3.10) on one GPU: the matrix fill and the joins timed apart.

    python tools/dist_nj_bench.py [--sizes 10000,30000] [--s 1000] [--cpu 2000] [--repeats 2] [--out DIR]

Sets: bench.make_sketches_device (the configs[2] generator: 100 families stored family by family).  Fails without a GPU.
  size   for each n: the lower triangle of the self job's distances into an n x n device matrix (DistJob.run_dev, distance only,
         lower triangle) and Engine.neighbor_joining_matrix on it, each timed with a device synchronise around it, `repeats`
         times (the joins overwrite the matrix, so every repeat refills it); then DistJob.neighbor_joining end to end once, which
         must give the same tree bit for bit.  Bytes scanned are those of the live lower triangle, 8 * m (m - 1) / 2 per step over
         m = n .. 4 (the least any scan reads), and their rate is compared with the 3.35 TB/s of the H100 SXM data sheet.
  cpu    the numpy model (tests/nj_model.py) against the GPU on the first `cpu` sketches of the first set: same tree, both clocks.
Prints one JSON line (and OUT/dist_nj_bench.json) with the card name and its power limit read in the same run.
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
from nj_model import nj                                     # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def scanned_bytes(n):
    m = np.arange(4, n + 1, dtype=np.float64)
    return float((4.0 * m * (m - 1)).sum())


def fill(torch, job, M, n):
    """the lower triangle of the job's distances into M (rows of n doubles), blocks of 2^27 pairs"""
    block = max(1, (1 << 27) // n)
    for q0 in range(1, n, block):
        job.run_dev(q0, min(block, n - q0), d_distance=M[q0].data_ptr())


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", default="10000,30000")
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--cpu", type=int, default=2000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    if not torch.cuda.is_available():
        sys.exit("dist_nj_bench: no CUDA device (the measurement does not fall back to anything)")
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
        fill(torch, job, M, small)
        eng.neighbor_joining_matrix(M, small, ld=n)
        fill_s, nj_s, tree, same = [], [], None, True
        for _ in range(args.repeats):
            _, dt = timed(torch, lambda: fill(torch, job, M, n))
            fill_s.append(dt)
            t, dt = timed(torch, lambda: eng.neighbor_joining_matrix(M, n))
            nj_s.append(dt)
            same &= tree is None or (np.array_equal(t["parent"], tree["parent"]) and np.array_equal(t["length"].view(np.uint64), tree["length"].view(np.uint64)))
            tree = t if tree is None else tree
        del M
        torch.cuda.empty_cache()
        whole, whole_s = timed(torch, job.neighbor_joining)
        same_whole = np.array_equal(whole["parent"], tree["parent"]) and np.array_equal(whole["length"].view(np.uint64), tree["length"].view(np.uint64))
        b = scanned_bytes(n)
        best = min(nj_s)
        out["sizes"].append(dict(n=n, steps=n - 3, fill_seconds=fill_s, nj_seconds=nj_s, job_seconds=whole_s, repeatable=bool(same),
                                 job_equals_matrix_entry=bool(same_whole), bytes_scanned=b, bytes_per_second=b / best,
                                 share_of_hbm=b / best / HBM_BYTES_PER_S, negative_lengths=int((tree["length"] < 0).sum())))
        if i == 0 and args.cpu:
            m = min(args.cpu, n)
            sub = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=m, stride=s)
            jb = eng.dist_open(sub, None, None, sketch_size=s, k=21, kmer_space=4.0 ** 21)
            gpu_tree, gpu_s = timed(torch, jb.neighbor_joining)
            D = jb.run(0, m, outputs=("distance",))["distance"]
            jb.close()
            t0 = time.perf_counter()
            cpu_p, cpu_l = nj(D)
            cpu_s = time.perf_counter() - t0
            out["cpu"] = dict(n=m, gpu_job_seconds=gpu_s, numpy_model_seconds=cpu_s,
                              same_tree=bool(np.array_equal(gpu_tree["parent"], cpu_p) and np.array_equal(gpu_tree["length"].view(np.uint64), cpu_l.view(np.uint64))))
        job.close()
        del H, N, L
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_nj_bench.json"), "w") as fo:
            fo.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

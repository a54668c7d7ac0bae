#!/usr/bin/env python
"""Rates of `mash within` (mashgpu_within_*) on one GPU, next to dist's merge-every-pair rate and the reference on the CPU.

    python tools/within_bench.py [--n 100000] [--s 1000] [--n2 10000] [--s2 10000] [--sub 4000] [--threads N] [--out DIR]

Workloads (bench.make_sketches_device, the configs[2] generator: 100 families stored family by family):
  grid1   n x n sketches of s = 1000, all against all: the tiled lockstep kernel
  grid2   n2 x n2 sketches of s = 10000, all against all: the warp-per-pair kernel
For each grid, the within job's run_dev writes all five outputs (common, examined, score, error, pass) in query blocks of at
most 2^27 pairs to device buffers, timed with CUDA events after one warm-up block; dist's run_dev with the prefilter off (every
pair merged) runs on the same set, same blocking, same timing.  CPU arm: the reference's own containSketches
(oracle/_ref/libmash_ref_contain.so) on a sub x sub subset of grid1 on `threads` cores, wall clock.  Check: a seeded sample of
pairs of the last timed block of each grid against the reference, bit for bit.  Prints one JSON line with the card name and its
power limit (and writes it to OUT/within_bench.json when --out is given).
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
import within_model as wm                                   # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402

F32_005 = float(np.float32(0.05))


def grid(torch, dev, eng, n, s, seed, ref, rng):
    from mash_b200._capi import _Set
    H, N, L = bench.make_sketches_device(torch, dev, n, s, seed)
    torch.cuda.synchronize()
    st = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=n, stride=s)
    qb = max(1, min(n, (1 << 27) // n))
    outs = dict(common=torch.empty(qb * n, dtype=torch.int32, device=dev), examined=torch.empty(qb * n, dtype=torch.int32, device=dev),
                score=torch.empty(qb * n, dtype=torch.float64, device=dev), error=torch.empty(qb * n, dtype=torch.float64, device=dev),
                passed=torch.empty(qb * n, dtype=torch.uint8, device=dev))
    ptrs = [outs[k].data_ptr() for k in ("common", "examined", "score", "error", "passed")]
    ts = torch.cuda.Stream()            # the runs and the events on one stream (the legacy default stream would mean the context's)
    stream = ts.cuda_stream
    res = {}

    def timed(run):
        run(0, qb)                                          # warm-up block
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(ts)
        q0 = 0
        for q0 in range(0, n, qb):
            run(q0, min(qb, n - q0))
        b.record(ts)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / 1e3, q0

    job = eng.within_open(st, None, max_error=F32_005)
    sec, last = timed(lambda q, c: job.run_dev(q, c, *ptrs, stream=stream))
    res["within_s"] = sec
    res["within_pairs_per_s"] = n * n / sec
    # seeded sample of the last timed block against the reference's own containSketches
    nb = min(qb, n - last)
    got = {k: v[:nb * n].cpu().numpy() for k, v in outs.items()}
    Hh = H.cpu().numpy().view(np.uint64)
    Nh = N.cpu().numpy().astype(np.uint32)
    sample = rng.integers(0, nb * n, 2000)
    bad = 0
    for k in sample:
        q, r = last + int(k) // n, int(k) % n
        sc, er = ref.grid(Hh[r:r + 1], Nh[r:r + 1], Hh[q:q + 1], Nh[q:q + 1])
        j = int(wm.examined_from_error(er)[0])
        ok = (got["score"][k].tobytes() == sc[0].tobytes() and got["error"][k].tobytes() == er[0].tobytes()
              and int(got["examined"][k]) == j and bool(got["passed"][k]) == bool(er[0] <= F32_005)
              and int(got["common"][k]) == (int(np.rint(sc[0] * j)) if j else 0))
        bad += not ok
    res["checked_pairs"] = int(sample.size)
    res["mismatches"] = bad
    res["passing_share_last_block"] = float(got["passed"].mean())
    res["mean_examined_last_block"] = float(got["examined"].view(np.uint32).mean())
    job.close()
    del outs

    douts = dict(numer=torch.empty(qb * n, dtype=torch.int32, device=dev), denom=torch.empty(qb * n, dtype=torch.int32, device=dev),
                 distance=torch.empty(qb * n, dtype=torch.float64, device=dev), pvalue=torch.empty(qb * n, dtype=torch.float64, device=dev),
                 passed=torch.empty(qb * n, dtype=torch.uint8, device=dev))
    dptrs = [douts[k].data_ptr() for k in ("numer", "denom", "distance", "pvalue", "passed")]
    kspace = 4.0 ** 21
    dj = eng.dist_open(st, None, None, sketch_size=s, k=21, kmer_space=kspace)
    dj.set_prefilter(0)
    sec, _ = timed(lambda q, c: dj.run_dev(q, c, *dptrs, stream=stream))
    dj.close()
    res["dist_merge_all_s"] = sec
    res["dist_merge_all_pairs_per_s"] = n * n / sec
    del douts
    return res, (H, N)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--n2", type=int, default=10_000)
    ap.add_argument("--s2", type=int, default=10_000)
    ap.add_argument("--sub", type=int, default=4000)
    ap.add_argument("--threads", type=int, default=len(os.sched_getaffinity(0)))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    dev = torch.device("cuda:0")
    card, limit = card_and_power_limit(torch, dev)
    eng = mash_b200.Engine(0)
    ref = wm.RefContain()
    rng = np.random.Generator(np.random.PCG64(2024))
    out = dict(card=card, power_limit_w=limit)
    r1, (H, N) = grid(torch, dev, eng, args.n, args.s, 1, ref, rng)
    out["grid1"] = dict(n=args.n, s=args.s, **r1)
    # CPU arm: the reference on a sub x sub subset of grid1
    m = min(args.sub, args.n)
    Hh = H[:m].cpu().numpy().view(np.uint64)
    Nh = N[:m].cpu().numpy().astype(np.uint32)
    del H, N
    t0 = time.perf_counter()
    ref.grid(Hh, Nh, Hh, Nh, threads=args.threads)
    dt = time.perf_counter() - t0
    out["cpu_reference"] = dict(n=m, s=args.s, threads=args.threads, seconds=dt, pairs_per_s=m * m / dt)
    torch.cuda.empty_cache()
    r2, _ = grid(torch, dev, eng, args.n2, args.s2, 2, ref, rng)
    out["grid2"] = dict(n=args.n2, s=args.s2, **r2)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "within_bench.json"), "w") as f:
            f.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Greedy dereplication (DistJob.representatives) on one GPU, with today's route beside it: the pass list to the host, then the
sequential definition and the nearest-representative assignment in numpy (tests/representatives_model.py).

    python tools/dist_representatives_bench.py [--n 100000] [--s 1000] [--cuts 1.0,0.05] [--family 20000] [--chain 33000]
                                               [--chain-cut 0.01] [--repeats 3] [--out DIR]

Sets:
  cut      bench.make_sketches_device (the configs[2] generator) at each -d cut-off
  family   a one-family set of `family` sketches: every pair shares a hash, one representative
  chain    an in-order mutation chain of `chain` 20 kb genomes (each one mutates the one before at 0.4 %) at -d chain-cut: sketch i
           is near only the few sketches just before it, the long dependency chain that makes the resolve rounds many; the chain is
           longer than one default block
For each set: the wall clock of the call (`repeats` times), the pass-1 blocks, the resolve rounds and the representatives, and from
a separate profiled call the device time of pass 1's runs, of the resolves and of pass 2 (the runs after the last resolve plus the
values).  The host route is timed where its edge list fits the host (not for the family: every pair is an edge).  Every call must
give the host route's result, or the first call's.  The card name and power limit are read in the same run; one JSON line (and
OUT/dist_representatives_bench.json).  Fails without a GPU.
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
from representatives_model import assign, sequential       # noqa: E402
from translated_screen_bench import card_and_power_limit   # noqa: E402


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t0


def host_route(job, n, capacity=1 << 23, rows=None):
    """pass lists of the lower triangle to the host, then the model: (rep, seconds for the lists, seconds in total)"""
    t0 = time.perf_counter()
    job.set_triangle(True)
    rows = rows or max(1, (1 << 28) // n)
    ii, jj, dd = [], [], []
    for q0 in range(1, n, rows):
        qc = min(rows, n - q0)
        m, lst = job.run_list(q0, qc, capacity)
        assert m <= capacity, "pass list over capacity"
        keep = lst["numer"] > 0
        idx = lst["index"][keep].astype(np.int64)
        ii.append(q0 + idx // n); jj.append(idx % n); dd.append(lst["distance"][keep])
    job.set_triangle(False)
    i, j, d = (np.concatenate(x) if x else np.zeros(0) for x in (ii, jj, dd))
    t1 = time.perf_counter()
    is_rep = sequential(n, i, j)
    rep, _ = assign(n, is_rep, i, j, d)
    return rep.astype(np.uint32), int(len(i)), t1 - t0, time.perf_counter() - t0


def phases(torch, job):
    """device seconds of pass 1's runs, the resolves and pass 2 (runs after the last resolve, and the values) in one profiled call"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        job.representatives()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if str(e.device_type).endswith("CUDA") and e.device_time_total > 0]
    last = max((e.time_range.end for e in ev if "greedy_resolve" in e.name), default=-1)
    out = {"pass1": 0.0, "resolve": 0.0, "pass2": 0.0}
    for e in ev:
        kind = "resolve" if "greedy_resolve" in e.name else ("pass1" if e.time_range.start < last else "pass2")
        out[kind] += e.device_time_total * 1e-6
    return out


def measure(torch, job, n, repeats, host=True):
    job.representatives()                                       # warm-up: modules loaded
    runs = [timed(torch, job.representatives) for _ in range(repeats)]
    r = runs[0][0]
    block = min((1 << 31) // n, 32768, max(n - 1, 1))
    rec = dict(n=n, seconds=[x[1] for x in runs], blocks=(n - 1 + block - 1) // block, block_rows=block, rounds=r["rounds"],
               representatives=r["n_reps"], repeatable=all(np.array_equal(x[0]["rep"], r["rep"]) and x[0]["rounds"] == r["rounds"] for x in runs))
    try:
        rec["device_seconds"] = phases(torch, job)
    except Exception as e:                                      # the profiler's event API differs between torch versions
        rec["device_seconds"] = f"not measured ({type(e).__name__}: {e})"
    if host:
        rep, edges, list_s, host_s = host_route(job, n)
        rec.update(host_edges=edges, host_lists_seconds=list_s, host_route_seconds=host_s, same_as_host=bool(np.array_equal(rep, r["rep"])))
    else:
        rec["host_route_seconds"] = "not measured"
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--cuts", default="1.0,0.05")
    ap.add_argument("--family", type=int, default=20_000)
    ap.add_argument("--chain", type=int, default=33_000)
    ap.add_argument("--chain-cut", type=float, default=0.01)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mash_b200
    from mash_b200._capi import _Set
    from fixtures import mutate, synth_genome
    if not torch.cuda.is_available():
        sys.exit("dist_representatives_bench: no CUDA device (the measurement does not fall back to anything)")
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
        rec = measure(torch, job, n, args.repeats, host=cut < 1.0)          # at -d 1 the pass list is every pair
        (_, n_edges), cc = timed(torch, job.components)
        rec.update(max_distance=cut, graph_edges=n_edges, components_seconds=cc)
        job.close()
        if cut < 1.0:                                           # `triangle -R length`: the job over the sketches longest first
            order = torch.argsort(-L, stable=True)
            Hp, Np, Lp = H[order].contiguous(), N[order].contiguous(), L[order].contiguous()
            torch.cuda.synchronize()
            job = eng.dist_open(_Set(Hp.data_ptr(), Np.data_ptr(), Lp.data_ptr(), on_device=True, n=n, stride=s), None, None, sketch_size=s,
                                k=21, kmer_space=kspace, max_distance=cut)
            r = job.representatives()
            rep, _, _, _ = host_route(job, n)
            rec["length_order"] = dict(representatives=r["n_reps"], rounds=r["rounds"], same_as_host=bool(np.array_equal(rep, r["rep"])))
            job.close()
            del Hp, Np, Lp
        out["cuts"].append(rec)
    del H, N, L
    torch.cuda.empty_cache()

    m = args.family
    H, N, L = bench.make_sketches_device(torch, dev, m, s, 3, n_families=1)
    torch.cuda.synchronize()
    fam = _Set(H.data_ptr(), N.data_ptr(), L.data_ptr(), on_device=True, n=m, stride=s)
    job = eng.dist_open(fam, None, None, sketch_size=s, k=21, kmer_space=kspace)
    out["family"] = measure(torch, job, m, args.repeats, host=False)
    job.close()
    del H, N, L
    torch.cuda.empty_cache()

    c = args.chain
    g = [synth_genome(11, 20_000)]
    for i in range(1, c):
        g.append(mutate(g[-1], 0.004, 100 + i))
    p = eng.params(k=21, s=s)
    Hc, Nc, Lc = eng.sketch([bytes(x) for x in g], p)
    del g
    job = eng.dist_open(Hc, Nc, Lc, sketch_size=s, k=21, kmer_space=p.kmer_space, max_distance=args.chain_cut)
    out["chain"] = measure(torch, job, c, args.repeats)
    out["chain"]["max_distance"] = args.chain_cut
    job.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_representatives_bench.json"), "w") as fo:
            fo.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()

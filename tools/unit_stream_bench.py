"""Measurements of the streaming unit job (mashgpu_unit_*, DESIGN.md 2.7).  Prints one JSON line per measurement.

  python tools/unit_stream_bench.py [--gbp 5 20] [--huge-gbp 100] [--cli-gb 3] [--parent-mash PATH]

1. One unit that fits, through the job and through mashgpu_sketch_batch (results must be identical), with the job's feed rate as
   a fraction of a plain pinned host-to-device copy of the same bytes, measured in the same run.
2. A generator-fed unit larger than the device (records are slices of a random pool), Gbp/s inside the feed calls and peak device
   bytes, and the same unit under a second feed split.
3. DESIGN.md 2.6's worst case (30 kb x 10^4 error-free reads, -r, m = 1) through mashgpu_sketch_reads with streaming forced,
   against the reads job's replay.
4. `mash sketch` on a generated FASTA from a file and from stdin: wall time and peak RSS (and the parent build's, if given).
The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mash_b200  # noqa: E402

REC = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else "unknown"


def pool(n, seed):
    return np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(seed).integers(0, 4, n)]


def records(pl, total, seed):
    """Slices of the pool (1 Mbp records at random offsets): no copies, any total."""
    rng = np.random.default_rng(seed)
    n = total // REC
    offs = rng.integers(0, pl.size - REC, n)
    return [pl[o:o + REC] for o in offs.tolist()]


def copy_rate(nbytes):
    import torch
    h = torch.empty(min(nbytes, 1 << 30), dtype=torch.uint8).pin_memory()
    d = torch.empty_like(h, device="cuda")
    d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    t = time.perf_counter()
    done = 0
    while done < nbytes:
        d.copy_(h, non_blocking=True)
        done += h.numel()
    torch.cuda.synchronize()
    return done / (time.perf_counter() - t)


def job_run(eng, p, feeds):
    job = eng.unit_open(p)
    try:
        t = time.perf_counter()
        for f in feeds:
            job.feed(f)
        feed_s = time.perf_counter() - t
        out = job.finish()
        total_s = time.perf_counter() - t
    finally:
        job.close()
    return out, feed_s, total_s


def fits(eng, gbp_list, pl):
    p = eng.params(k=21, s=1000)
    for gbp in gbp_list:
        recs = records(pl, int(gbp * 1e9), int(gbp * 10))
        nbytes = sum(r.size for r in recs)
        eng.sketch(recs[:4], p, unit_of_record=[0] * 4, n_units=1)          # warm-up
        t = time.perf_counter()
        h, n, length, c = eng.sketch(recs, p, unit_of_record=[0] * len(recs), n_units=1, counts=True)
        batch_s = time.perf_counter() - t
        (jh, jc, jl, _), feed_s, job_s = job_run(eng, p, [recs[i:i + 256] for i in range(0, len(recs), 256)])
        same = bool(np.array_equal(h[0, :n[0]], jh) and np.array_equal(c[0, :n[0]], jc) and jl == length[0])
        cr = copy_rate(nbytes)
        print(json.dumps({"what": "job_vs_batch", "gbp": nbytes / 1e9, "identical": same, "batch_s": round(batch_s, 3),
                          "job_s": round(job_s, 3), "job_feed_GBps": round(nbytes / feed_s / 1e9, 2),
                          "pinned_copy_GBps": round(cr / 1e9, 2), "job_over_copy": round(nbytes / job_s / cr, 3)}), flush=True)


def huge(eng, gbp, pl):
    p = eng.params(k=21, s=1000)
    total = int(gbp * 1e9)
    recs = records(pl, total, 99)
    out = []
    for step in (64, 97):
        eng.stats(reset=True)
        (h, c, length, _), feed_s, job_s = job_run(eng, p, (recs[i:i + step] for i in range(0, len(recs), step)))
        st = eng.stats()
        out.append((h, c, length, feed_s, job_s, st))
    h0, c0, l0, feed_s, job_s, st = out[0]
    same = bool(np.array_equal(h0, out[1][0]) and np.array_equal(c0, out[1][1]) and l0 == out[1][2])
    print(json.dumps({"what": "generator_fed", "gbp": l0 / 1e9, "feed_Gbp_per_s": round(l0 / feed_s / 1e9, 2), "job_s": round(job_s, 2),
                      "stages": st["unit_stages"], "peak_device_bytes": st["unit_peak_device_bytes"], "second_split_identical": same}),
          flush=True)


def worst_case(eng):
    g = pool(30_000, 7).tobytes()
    rng = np.random.default_rng(8)
    reads = []
    for _ in range(10_000):
        a = int(rng.integers(0, 30_000 - 30_000 // 2))
        reads.append(g[a:] + g[:a])                  # 30 kb error-free reads of a circular 30 kb genome
    p = eng.params(k=21, s=1000)
    t = time.perf_counter()
    job = eng.reads_open(p)
    job.feed(reads)
    rh, rc, _ = job.finish()
    job.close()
    replay_s = time.perf_counter() - t
    os.environ["MASHGPU_UNIT_STREAM_BYTES"] = "1"
    eng.stats(reset=True)
    t = time.perf_counter()
    h, c, used = eng.sketch_reads(reads, p, counts=True)
    unit_s = time.perf_counter() - t
    st = eng.stats()
    del os.environ["MASHGPU_UNIT_STREAM_BYTES"]
    print(json.dumps({"what": "worst_case_reads_m1", "gbp": 0.3, "replay_s": round(replay_s, 3), "unit_job_s": round(unit_s, 3),
                      "identical": bool(np.array_equal(h, rh) and np.array_equal(c, rc)), "reads_events": st["reads_events"]}), flush=True)


def cli(gb, parent):
    d = tempfile.mkdtemp(prefix="unit_cli_")
    fa = os.path.join(d, "in.fna")
    pl = pool(64 << 20, 5).tobytes()
    rng = np.random.default_rng(6)
    with open(fa, "wb") as f:
        for i in range(int(gb * 1e9) // REC):
            a = int(rng.integers(0, len(pl) - REC))
            f.write(b">r%d\n%s\n" % (i, pl[a:a + REC]))
    code = ("import resource, subprocess, sys, time; t = time.perf_counter(); "
            "subprocess.run(sys.argv[2:], check=True, capture_output=True, stdin=open(sys.argv[1], 'rb')); "
            "print(time.perf_counter() - t, resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss)")
    builds = [("this", os.path.join(ROOT, "mash_b200", "host", "mash"))] + ([("parent", parent)] if parent else [])
    for name, exe in builds:
        for src in ("file", "stdin"):
            args = [exe, "sketch", "-o", os.path.join(d, "o"), fa if src == "file" else "-"]
            out = subprocess.run([sys.executable, "-c", code, fa if src == "stdin" else os.devnull] + args, check=True,
                                 capture_output=True, text=True).stdout.split()
            print(json.dumps({"what": "cli_sketch", "build": name, "input": src, "gb": gb, "wall_s": round(float(out[0]), 2),
                              "peak_rss_MB": round(int(out[1]) / 1024, 1)}), flush=True)
    os.remove(fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, nargs="*", default=[5, 20])
    ap.add_argument("--huge-gbp", type=float, default=100)
    ap.add_argument("--cli-gb", type=float, default=3)
    ap.add_argument("--parent-mash", default="")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    eng = mash_b200.Engine(0)
    pl = pool(1 << 30, 1)
    if a.gbp:
        fits(eng, a.gbp, pl)
    if a.huge_gbp:
        huge(eng, a.huge_gbp, pl)
    worst_case(eng)
    if a.cli_gb:
        cli(a.cli_gb, a.parent_mash)


if __name__ == "__main__":
    main()

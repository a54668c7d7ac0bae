"""Reads mode (`mash sketch -r`) on the GPU: the streaming reads job against a build of the previous engine, in one call.

    python tools/reads_stream_bench.py --parent-lib DIR/libmashgpu.so --parent-mash DIR/host/mash --out OUTDIR [--parts ...]

Parts (all by default):
  memory  mashgpu_sketch_reads on in-memory read sets (150 bp, 1 % substitutions, seeded genomes: 5 Mbp at 100x and 100 Mbp at
          30x), parent and this build alternating, -m 1 / -m 2 / -m 2 -c / -b 100M (-b: this build only, the parent refuses it):
          wall time, results equal, events and replay ms
  worst   error-free reads of a 30 kb genome at 10^4x: events and replay ms (every read repeats k-mers the heap holds)
  large   --large-gbp Gbp fed through one job from a seeded generator (never held in memory), twice with different feed
          splits: Gbp/s, reads_peak_device_bytes, results equal
  cli     `mash sketch -r -m 2` on a gzipped FASTQ of --cli-gb GB: wall time and peak RSS, parent and this build alternating

Prints one JSON line per measurement with the card's name and power limit, and writes them to OUTDIR/reads_stream_bench.json.
Temporary files go to a temporary directory; nothing is written to the source tree.
"""
import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mash_b200._capi import SketchParams, Stats  # noqa: E402

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)
ACGT = np.frombuffer(b"ACGT", np.uint8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return {"card": name, "power_limit": power, "sm_clock_max": clock}


class Lib:
    """One libmashgpu.so through ctypes (the parent's struct is a prefix of this build's: extra fields are not read)."""

    def __init__(self, path):
        self.L = L = C.CDLL(path)
        L.mashgpu_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.mashgpu_set_alphabet.argtypes = [C.POINTER(SketchParams), C.c_char_p]
        L.mashgpu_sketch_reads.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.c_uint64, C.c_void_p, u64p, u64p, u32p, u32p, u64p]
        L.mashgpu_last_error.restype = C.c_char_p
        L.mashgpu_last_error.argtypes = [C.c_void_p]
        L.mashgpu_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats), C.c_int]
        L.mashgpu_set_timing.argtypes = [C.c_void_p, C.c_int]
        self.h = C.c_void_p()
        assert L.mashgpu_create(0, C.byref(self.h)) == 0
        self.has_job = hasattr(L, "mashgpu_reads_open")
        if self.has_job:
            L.mashgpu_reads_open.argtypes = [C.c_void_p, C.POINTER(SketchParams), C.POINTER(C.c_void_p)]
            L.mashgpu_reads_feed.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, u64p, C.POINTER(C.c_int)]
            L.mashgpu_reads_finish.argtypes = [C.c_void_p, u64p, u32p, u32p, u64p]
            L.mashgpu_reads_close.argtypes = [C.c_void_p]

    def check(self, rc):
        if rc:
            raise RuntimeError(f"mashgpu error {rc}: {self.L.mashgpu_last_error(self.h).decode()}")

    def params(self, m=1, c=0.0, b=0, k=21, s=1000):
        p = SketchParams()
        p.kmer_size, p.sketch_size, p.seed, p.min_copies, p.target_cov, p.bloom_bytes = k, s, 42, m, c, b
        self.L.mashgpu_set_alphabet(C.byref(p), b"ACGT")
        return p

    def stats(self, reset=False):
        st = Stats()
        self.check(self.L.mashgpu_get_stats(self.h, C.byref(st), int(reset)))
        return {f: getattr(st, f) for f, _ in Stats._fields_}

    def sketch_reads(self, reads, p):
        """reads: (n, L) uint8 array.  Returns (hashes, counts, used, seconds)."""
        n, rl = reads.shape
        ptrs = (reads.ctypes.data + np.arange(n, dtype=np.uint64) * np.uint64(rl)).astype(np.uint64)
        lens = np.full(n, rl, np.uint64)
        out = np.zeros(p.sketch_size, np.uint64); cnt = np.zeros(p.sketch_size, np.uint32)
        nn = C.c_uint32(0); used = C.c_uint64(0)
        t = time.perf_counter()
        self.check(self.L.mashgpu_sketch_reads(self.h, C.byref(p), n, ptrs.ctypes.data, lens.ctypes.data_as(u64p),
                                               out.ctypes.data_as(u64p), cnt.ctypes.data_as(u32p), C.byref(nn), C.byref(used)))
        dt = time.perf_counter() - t
        return out[:nn.value].copy(), cnt[:nn.value].copy(), used.value, dt


def sample_reads(rng, genome, n, rl=150, err=0.01):
    starts = rng.integers(0, genome.size - rl, n)
    reads = np.lib.stride_tricks.sliding_window_view(genome, rl)[starts]
    if err > 0:
        n_err = rng.binomial(n * rl, err)
        flat = reads.reshape(-1)
        flat[rng.integers(0, flat.size, n_err)] = ACGT[rng.integers(0, 4, n_err)]
    return reads


def emit(rows, row, info):
    row = {**row, **info}
    rows.append(row)
    print(json.dumps(row), flush=True)


def part_memory(new, old, info, rows, reps):
    for glen, cov in [(5_000_000, 100), (100_000_000, 30)]:
        rng = np.random.default_rng(glen)
        genome = ACGT[rng.integers(0, 4, glen)]
        reads = sample_reads(rng, genome, glen * cov // 150)
        gbp = reads.size / 1e9
        for name, kw in [("-m 1", dict(m=1)), ("-m 2", dict(m=2)), (f"-m 2 -c {cov // 5}", dict(m=2, c=float(cov // 5))),
                         ("-b 100M", dict(b=100_000_000))]:
            t_new, t_old, same = [], [], True
            for _ in range(reps):
                if "b" not in kw:
                    ho, co, uo, dt = old.sketch_reads(reads, old.params(**kw))
                    t_old.append(dt)
                hn, cn, un, dt = new.sketch_reads(reads, new.params(**kw))
                t_new.append(dt)
                if "b" not in kw:
                    same = same and np.array_equal(ho, hn) and np.array_equal(co, cn) and uo == un
            new.L.mashgpu_set_timing(new.h, 1)
            new.stats(reset=True)
            _, _, used, _ = new.sketch_reads(reads, new.params(**kw))
            st = new.stats(reset=True)
            new.L.mashgpu_set_timing(new.h, 0)
            emit(rows, {"part": "memory", "reads": f"{glen / 1e6:g} Mbp x {cov}", "gbp": round(gbp, 3), "options": name,
                        "new_s": [round(x, 4) for x in t_new], "parent_s": [round(x, 4) for x in t_old] or "refused by the parent",
                        "same_result": same if t_old else None, "reads_used": used, "events": st["reads_events"],
                        "replay_ms": round(st["reads_replay_ms"], 2), "peak_device_bytes": st["reads_peak_device_bytes"]}, info)
        del reads


def part_worst(new, old, info, rows):
    rng = np.random.default_rng(30_000)
    genome = ACGT[rng.integers(0, 4, 30_000)]
    reads = sample_reads(rng, genome, 30_000 * 10_000 // 150, err=0.0)
    ho, co, uo, t_old = old.sketch_reads(reads, old.params())
    new.L.mashgpu_set_timing(new.h, 1)
    new.stats(reset=True)
    hn, cn, un, t_new = new.sketch_reads(reads, new.params())
    st = new.stats(reset=True)
    new.L.mashgpu_set_timing(new.h, 0)
    emit(rows, {"part": "worst", "reads": "30 kb x 10^4, error-free", "gbp": round(reads.size / 1e9, 3), "options": "-m 1",
                "new_s": round(t_new, 3), "parent_s": round(t_old, 3),
                "same_result": bool(np.array_equal(ho, hn) and np.array_equal(co, cn) and uo == un),
                "events": st["reads_events"], "replay_ms": round(st["reads_replay_ms"], 2)}, info)


def part_large(new, info, rows, gbp):
    glen, rl = 100_000_000, 150
    genome = ACGT[np.random.default_rng(7).integers(0, 4, glen)]
    total_reads = int(gbp * 1e9) // rl
    results = []
    for batch in (1_000_000, 700_001):
        rng = np.random.default_rng(8)               # same reads in the same order, cut into different feeds
        p = new.params(m=2)
        job = C.c_void_p()
        new.stats(reset=True)
        new.check(new.L.mashgpu_reads_open(new.h, C.byref(p), C.byref(job)))
        done, t_feed, gen_chunk = 0, 0.0, 1_000_000
        pending = np.zeros((0, rl), np.uint8)
        t0 = time.perf_counter()
        while done < total_reads or pending.shape[0]:
            while pending.shape[0] < batch and done < total_reads:
                g = min(gen_chunk, total_reads - done)
                pending = np.concatenate([pending, sample_reads(rng, genome, g, rl)])
                done += g
            feed, pending = pending[:batch], pending[batch:]
            n = feed.shape[0]
            ptrs = (feed.ctypes.data + np.arange(n, dtype=np.uint64) * np.uint64(rl)).astype(np.uint64)
            lens = np.full(n, rl, np.uint64)
            st = C.c_int(0)
            t = time.perf_counter()
            new.check(new.L.mashgpu_reads_feed(job, n, ptrs.ctypes.data, lens.ctypes.data_as(u64p), C.byref(st)))
            t_feed += time.perf_counter() - t
        out = np.zeros(1000, np.uint64); cnt = np.zeros(1000, np.uint32); nn = C.c_uint32(0); used = C.c_uint64(0)
        new.check(new.L.mashgpu_reads_finish(job, out.ctypes.data_as(u64p), cnt.ctypes.data_as(u32p), C.byref(nn), C.byref(used)))
        wall = time.perf_counter() - t0
        new.L.mashgpu_reads_close(job)
        s = new.stats()
        results.append((out[:nn.value].copy(), cnt[:nn.value].copy(), used.value))
        emit(rows, {"part": "large", "gbp": round(total_reads * rl / 1e9, 2), "options": "-m 2", "feed_reads": batch,
                    "wall_s": round(wall, 1), "gbp_per_s_incl_generator": round(total_reads * rl / 1e9 / wall, 2),
                    "gbp_per_s_in_feed_calls": round(total_reads * rl / 1e9 / t_feed, 2), "events": s["reads_events"],
                    "peak_device_bytes": s["reads_peak_device_bytes"], "reads_used": used.value}, info)
    a, b = results
    emit(rows, {"part": "large", "same_result_for_both_feed_splits": bool(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2])}, info)


def part_cli(new_mash, old_mash, info, rows, gb, reps, tmp):
    rng = np.random.default_rng(11)
    genome = ACGT[rng.integers(0, 4, 5_000_000)]
    fq = os.path.join(tmp, "reads.fastq.gz")
    n_total = int(gb * 1e9) // 310
    with gzip.open(fq, "wb", compresslevel=1) as f:
        for a in range(0, n_total, 200_000):
            reads = sample_reads(rng, genome, min(200_000, n_total - a))
            f.write(b"".join(b"@r\n%s\n+\n%s\n" % (r.tobytes(), b"I" * 150) for r in reads))
    code = ("import resource, subprocess, sys, time; t = time.perf_counter(); subprocess.run(sys.argv[1:], check=True, capture_output=True); "
            "print(time.perf_counter() - t, resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss)")
    res = {"new": [], "parent": []}
    for _ in range(reps):
        for name, exe in (("parent", old_mash), ("new", new_mash)):
            out = subprocess.run([sys.executable, "-c", code, exe, "sketch", "-r", "-m", "2", "-o", os.path.join(tmp, name), fq],
                                 check=True, capture_output=True, text=True).stdout.split()
            res[name].append((round(float(out[0]), 2), int(out[1]) * 1024))
    same = open(os.path.join(tmp, "new.msh"), "rb").read() == open(os.path.join(tmp, "parent.msh"), "rb").read()
    emit(rows, {"part": "cli", "command": "mash sketch -r -m 2 reads.fastq.gz", "fastq_gb": gb, "gz_bytes": os.path.getsize(fq),
                "new_wall_s_and_peak_rss": res["new"], "parent_wall_s_and_peak_rss": res["parent"], "same_msh": same}, info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True)
    ap.add_argument("--parent-mash", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--parts", default="memory,worst,large,cli")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--large-gbp", type=float, default=100.0)
    ap.add_argument("--cli-gb", type=float, default=2.0)
    a = ap.parse_args()
    info = card()
    parts = a.parts.split(",")
    new = Lib(os.path.join(ROOT, "mash_b200", "libmashgpu.so"))
    old = Lib(a.parent_lib) if ("memory" in parts or "worst" in parts) else None
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        if "memory" in parts:
            part_memory(new, old, info, rows, a.reps)
        if "worst" in parts:
            part_worst(new, old, info, rows)
        if "large" in parts:
            part_large(new, info, rows, a.large_gbp)
        if "cli" in parts:
            part_cli(os.path.join(ROOT, "mash_b200", "host", "mash"), a.parent_mash, info, rows, a.cli_gb, a.reps, tmp)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "reads_stream_bench.json"), "a") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()

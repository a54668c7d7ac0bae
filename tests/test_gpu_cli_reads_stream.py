"""`mash sketch -r` through the host shim with the streaming reads job: -b (the reference's Bloom filter) with and without -c,
the "[N seqs]" comment of a -c stop, and a peak host memory that does not grow with the read set."""
import gzip
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import reads_stream_model as M
from fixtures import GOLDEN, fmt_g

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("mashcli_reads")
    for f in ("reads1.fastq", "reads2.fastq"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    return d


def _dump(work, msh):
    text = subprocess.run([MASH, "info", "-d", msh], cwd=work, check=True, capture_output=True, text=True).stdout
    return json.loads(text.replace(']\n\t\t\t"counts" :', '],\n\t\t\t"counts" :'))["sketches"][0]


@pytest.mark.parametrize("b,bytes_", [("1k", 1000), ("10M", 10_000_000)])
@pytest.mark.parametrize("c", [0.0, 2.0])
def test_bloom_option_through_the_cli(work, oracle, golden, b, bytes_, c):
    msh = f"bloom_{b}_{c}.msh"
    args = [MASH, "sketch", "-r", "-b", b] + (["-c", str(c)] if c > 0 else []) + ["-o", msh, "reads1.fastq", "reads2.fastq"]
    env = dict(os.environ, MASHGPU_READS_STAGE_BYTES="200000")          # several stages and stretches
    pr = subprocess.run(args, cwd=work, check=True, capture_output=True, text=True, env=env)
    reads = golden.reads_round_robin()
    po = oracle.params(k=21)
    h, cnt, used = M.sketch_reads_reference(M.record_hashes(oracle, reads, po), 1000, bloom_bytes=bytes_, target_cov=c)
    sk = _dump(work, msh)
    assert sk["hashes"] == [int(x) for x in h] and sk["counts"] == [int(x) for x in cnt]
    size = 2.0 ** 64 * len(h) / float(h[-1])
    assert sk["length"] == int(size)
    assert f"Estimated genome size: {fmt_g(size)}" in pr.stderr
    assert f"Estimated coverage:    {fmt_g(float(cnt.sum()) / len(cnt))}" in pr.stderr
    kept = len([r for r in reads if len(r) >= 21])
    if c > 0:
        assert f"Reads used:            {used}" in pr.stderr
        assert 0 < used < kept
        assert sk["comment"].startswith(f"[{used} seqs] ") == (used > 1)          # the reference writes the count from 2 records on
    else:
        assert used == kept and "Reads used" not in pr.stderr


def test_target_coverage_comment_counts_the_reads_used(work, oracle, golden):
    # with -c the record loop ends at the stopping read, so the comment's "[N seqs]" is the number of reads used
    pr = subprocess.run([MASH, "sketch", "-r", "-m", "2", "-c", "1.5", "-o", "cov.msh", "reads1.fastq", "reads2.fastq"], cwd=work,
                        check=True, capture_output=True, text=True)
    reads = golden.reads_round_robin()
    _, _, _, used = oracle.sketch_unit_mc(reads, oracle.params(k=21), s=1000, min_copies=2, target_cov=1.5, counts=True)
    assert f"Reads used:            {used}" in pr.stderr
    assert 0 < used < len(reads) - 1
    assert _dump(work, "cov.msh")["comment"].startswith(f"[{used} seqs] ")


def _write_fastq(path, n_reads, seed):
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    g = acgt[rng.integers(0, 4, 5_000_000)]
    with open(path, "wb") as f:
        done = 0
        while done < n_reads:
            n = min(100_000, n_reads - done)
            starts = rng.integers(0, g.size - 150, n)
            reads = g[starts[:, None] + np.arange(150)[None, :]]
            err = rng.random(reads.shape) < 0.01
            reads[err] = acgt[rng.integers(0, 4, int(err.sum()))]
            lines = []
            for i in range(n):
                lines.append(b"@r%d\n%s\n+\n%s\n" % (done + i, reads[i].tobytes(), b"I" * 150))
            f.write(b"".join(lines))
            done += n


def test_host_memory_does_not_grow_with_the_read_set(tmp_path):
    # the parent held every read on the host; the job holds one feed
    rss = []
    for n in (130_000, 1_300_000):                                      # ~40 MB and ~400 MB of FASTQ
        fq = tmp_path / f"r{n}.fastq"
        _write_fastq(fq, n, n)
        code = ("import resource, subprocess, sys; subprocess.run(sys.argv[1:], check=True, capture_output=True); "
                "print(resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss)")
        out = subprocess.run([sys.executable, "-c", code, MASH, "sketch", "-r", "-m", "2", "-o", str(tmp_path / f"r{n}"), str(fq)],
                             check=True, capture_output=True, text=True).stdout
        rss.append(int(out.strip()) * 1024)
        os.remove(fq)
    assert rss[1] - rss[0] < 128 << 20, rss                            # the larger set has ~175 MB more sequence

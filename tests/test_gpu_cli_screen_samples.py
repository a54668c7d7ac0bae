"""CLI tests of `mash screen -I`: each sample's rows equal a `mash screen` run over that sample alone, prefixed by the sample."""
import gzip
import os
import shutil
import subprocess

import pytest

from fixtures import GOLDEN
from test_gpu_cli import MASH, out, work  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def samples(work):  # noqa: F811
    with open(work / "reads1.fastq", "rb") as src, gzip.open(work / "reads2.fastq.gz", "wb") as dst:
        shutil.copyfileobj(src, dst)
    (work / "empty.fastq").write_bytes(b"")
    # genome 3's own sequence as one read set: a sample with other hits than the read files
    (work / "genome3_reads.fa").write_bytes(open(work / "genome3.fna", "rb").read())
    return work


def prefixed(work, sample, opts):
    return "".join(f"{sample}\t{line}\n" for line in out(work, "screen", *opts, "genomes.msh", sample).splitlines())


@pytest.mark.parametrize("opts", [[], ["-w"], ["-i", "0.9"], ["-v", "1e-10"], ["-i", "-1"], ["-w", "-i", "-1"]])
def test_samples_equal_one_screen_per_sample(samples, opts):
    names = ["reads1.fastq", "reads2.fastq", "reads2.fastq.gz", "genome3_reads.fa"]
    got = out(samples, "screen", "-I", *opts, "genomes.msh", *names)
    assert got == "".join(prefixed(samples, n, opts) for n in names)
    assert got


def test_sample_without_records_is_skipped(samples):
    r = subprocess.run([MASH, "screen", "-I", "genomes.msh", "reads1.fastq", "empty.fastq", "reads2.fastq"], cwd=samples,
                       capture_output=True, text=True)
    assert r.returncode == 0
    assert "empty.fastq" in r.stderr and "WARNING" in r.stderr
    assert r.stdout == prefixed(samples, "reads1.fastq", []) + prefixed(samples, "reads2.fastq", [])
    assert "Estimated distinct k-mers in reads2.fastq" in r.stderr


def test_stdin_only_as_first_sample(samples):
    r = subprocess.run([MASH, "screen", "-I", "genomes.msh", "reads1.fastq", "-"], cwd=samples, capture_output=True, text=True)
    assert r.returncode == 1 and "'-' for stdin must be first query" in r.stderr
    with open(samples / "reads2.fastq", "rb") as f:
        r = subprocess.run([MASH, "screen", "-I", "genomes.msh", "-", "reads1.fastq"], cwd=samples, stdin=f, capture_output=True, check=True)
    want = "".join(f"-\t{line}\n" for line in out(samples, "screen", "genomes.msh", "reads2.fastq").splitlines())
    assert r.stdout.decode() == want + prefixed(samples, "reads1.fastq", [])


def test_pooled_screen_unchanged(samples):
    assert out(samples, "screen", "genomes.msh", "reads1.fastq", "reads2.fastq") == open(os.path.join(GOLDEN, "ref_screen")).read()

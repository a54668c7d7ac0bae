"""`mash sketch` / `mash dist` through the host shim with file-mode units streamed through the unit job: with a low
MASHGPU_CLI_STREAM_BYTES the .msh files are byte-identical to the default run (one file, several, `-p 4` with large and small files,
`-M`, stdin, gzip); `mash sketch -r` without -m/-c/-b (now the unit job) equals the golden sketch and the heap model; a streamed
query gives the same `mash dist` output; peak host memory does not grow with the size of a unit."""
import gzip
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import reads_stream_model as M
from fixtures import GOLDEN, synth_genome

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASH = os.path.join(ROOT, "mash_b200", "host", "mash")
STREAM = {"MASHGPU_CLI_STREAM_BYTES": "100000", "MASHGPU_UNIT_STAGE_BYTES": "1000000"}


def _fasta(path, recs, seed):
    with open(path, "wb") as f:
        for i, r in enumerate(recs):
            f.write(b">rec%d_%d some comment\n" % (seed, i))
            for a in range(0, len(r), 80):
                f.write(r[a:a + 80] + b"\n")


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("mashcli_unit")
    for f in ("genome1.fna", "genome2.fna", "genome3.fna", "reads1.fastq", "reads2.fastq"):
        with gzip.open(os.path.join(GOLDEN, f + ".gz"), "rb") as src, open(d / f, "wb") as dst:
            shutil.copyfileobj(src, dst)
    # units of a few MB (handed over at the end of parsing) and of 19 MB (handed over in 16 MiB pieces while parsing), many stages
    _fasta(d / "big1.fna", [bytes(synth_genome(70 + i, n, n_runs=3, lower_frac=0.02)) for i, n in enumerate([2_500_000, 10, 700_000, 1_800_000])], 1)
    _fasta(d / "big2.fna", [bytes(synth_genome(80, 18_000_000))] + [bytes(synth_genome(81 + i, 4000)) for i in range(300)], 2)
    with open(d / "big1.fna", "rb") as src, gzip.open(d / "big1.fna.gz", "wb", compresslevel=1) as dst:
        shutil.copyfileobj(src, dst)
    return d


def _run(work, args, env=None, stdin=None):
    e = dict(os.environ, **(env or {}))
    with open(work / stdin, "rb") if stdin else open(os.devnull, "rb") as f:
        return subprocess.run([MASH] + args, cwd=work, check=True, capture_output=True, env=e, stdin=f)


def _same_msh(work, name, args, stdin=None):
    _run(work, ["sketch", "-o", f"{name}_default"] + args, stdin=stdin)
    _run(work, ["sketch", "-o", f"{name}_stream"] + args, env=STREAM, stdin=stdin)
    a = (work / f"{name}_default.msh").read_bytes()
    b = (work / f"{name}_stream.msh").read_bytes()
    assert a == b


CASES = {
    "one": ["big1.fna"],
    "several": ["genome1.fna", "big1.fna", "genome2.fna", "big2.fna", "genome3.fna"],
    "p4": ["-p", "4", "genome1.fna", "big1.fna", "genome2.fna", "big2.fna", "genome3.fna", "big1.fna.gz"],
    "counts": ["-M", "big2.fna", "genome1.fna", "big1.fna"],
    "gzip": ["big1.fna.gz", "genome2.fna"],
    "k16_s5000": ["-k", "16", "-s", "5000", "big2.fna", "big1.fna"],
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_streamed_sketch_files_are_byte_identical(work, case):
    _same_msh(work, case, CASES[case])


def test_streamed_stdin_is_byte_identical(work):
    _same_msh(work, "stdin", ["-"], stdin="big1.fna")


def test_plain_reads_mode_uses_the_unit_job(work, oracle, golden):
    # `mash sketch -r` without -m > 1, -c or -b: order-independent, so the parallel unit job; same sketch as the golden file and the
    # heap model, same stderr lines
    pr = _run(work, ["sketch", "-r", "-o", "plain", "reads1.fastq", "reads2.fastq"], env={"MASHGPU_UNIT_STAGE_BYTES": "200000"})
    text = _run(work, ["info", "-d", "plain.msh"]).stdout.decode()
    sk = json.loads(text.replace(']\n\t\t\t"counts" :', '],\n\t\t\t"counts" :'))["sketches"][0]
    gh, glen = golden.golden_reads_sketch()
    assert sk["hashes"] == [int(x) for x in gh] and sk["length"] == glen
    reads = golden.reads_round_robin()
    h, c, _ = M.sketch_reads_reference(M.record_hashes(oracle, reads, oracle.params(k=21)), 1000)
    assert sk["hashes"] == [int(x) for x in h] and sk["counts"] == [int(x) for x in c]
    err = pr.stderr.decode()
    assert "Estimated genome size:" in err and "Estimated coverage:" in err and "Reads used" not in err


def test_dist_with_a_streamed_query(work):
    args = ["dist", "genome1.fna", "big1.fna", "genome2.fna", "big2.fna"]
    a = _run(work, args).stdout
    b = _run(work, args, env=STREAM).stdout
    assert a == b and a.count(b"\n") == 3


def test_host_memory_does_not_grow_with_the_unit(tmp_path):
    # 1 Mbp records; both units stream (a low threshold and 16 MiB stages), so the larger one adds no host memory
    rng = np.random.default_rng(3)
    pool = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 8_000_000)].tobytes()
    rss = []
    for n_rec in (40, 1000):                                             # ~40 MB and ~1 GB of FASTA
        fa = tmp_path / f"u{n_rec}.fna"
        with open(fa, "wb") as f:
            for i in range(n_rec):
                a = int(rng.integers(0, len(pool) - 1_000_000))
                f.write(b">r%d\n%s\n" % (i, pool[a:a + 1_000_000]))
        code = ("import resource, subprocess, sys; subprocess.run(sys.argv[1:], check=True, capture_output=True); "
                "print(resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss)")
        env = dict(os.environ, MASHGPU_CLI_STREAM_BYTES="1000000", MASHGPU_UNIT_STAGE_BYTES=str(16 << 20))
        out = subprocess.run([sys.executable, "-c", code, MASH, "sketch", "-o", str(tmp_path / f"u{n_rec}"), str(fa)],
                             check=True, capture_output=True, text=True, env=env).stdout
        rss.append(int(out.strip()) * 1024)
        os.remove(fa)
    assert rss[1] - rss[0] < 128 << 20, rss

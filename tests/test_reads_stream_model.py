"""CPU checks of the streaming reads job's model (no GPU): the Bloom filter of `mash sketch -r -b` restated against the reference's
header, the Bloom branch of the heap against the reference's object code, and the per-stretch gate bound of DESIGN.md 2.6 --
replaying only the k-mers at or below the heap's top at the start of each stretch, for any stretch boundaries, gives the heap
that every k-mer gives."""
import json
import os

import numpy as np
import pytest

import reads_stream_model as M

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# (seed, k, s, bloom_bytes, genome length, reads): Bloom heaps whose digests the reference's object code produced (ref_bloom.json)
BLOOM_CASES = [(11, 21, 200, 1000, 20_000, 1500), (12, 21, 300, 65_536, 30_000, 2000), (13, 15, 150, 1000, 10_000, 1200),
               (14, 15, 200, 16 << 20, 20_000, 1500), (15, 32, 100, 4096, 15_000, 1000)]


def _kat():
    with open(os.path.join(GOLDEN, "bloom_kat.json")) as f:
        return json.load(f)["cases"]


def test_bloom_parameters_match_the_reference_header():
    # bloom_filter(p) as MinHashHeap builds it (false_positive_probability 0): one hash function, 8 b bits, one salt from the
    # default random_seed -- also above 2^29 bytes, where the 32-bit index reaches only the first 2^32 bits
    cases = _kat()
    assert any(c["bytes"] > (1 << 29) for c in cases)
    for c in cases:
        assert c["hashes"] == 1
        assert c["bits"] == M.bloom_bits(c["bytes"])
        assert c["salt"] == M.bloom_salt() == M.BLOOM_SALT


@pytest.mark.parametrize("use64", [True, False])
def test_bloom_index_matches_the_reference_header(use64):
    # compute_indices(hash_ap(key, 8 or 4 little-endian bytes, salt)) of the reference header, compiled as MinHashHeap uses it
    for c in _kat():
        for key, idx in c["idx64" if use64 else "idx32"]:
            assert M.bloom_index(key, use64, c["bytes"]) == idx


def _case_hashes(oracle, seed, k, genome_len, n_reads):
    reads = M.synth_reads(seed, genome_len, n_reads)
    po = oracle.params(k=k)
    return reads, po, M.record_hashes(oracle, reads, po)


@pytest.mark.parametrize("case", BLOOM_CASES, ids=[f"k{c[1]}-b{c[3]}" for c in BLOOM_CASES])
def test_bloom_heap_matches_reference_object_code(oracle, case):
    seed, k, s, b, glen, n = case
    reads, po, hs = _case_hashes(oracle, seed, k, glen, n)
    h, c, used = M.sketch_reads_reference(hs, s, bloom_bytes=b, use64=bool(po.use64))
    with open(os.path.join(GOLDEN, "ref_bloom.json")) as f:
        want = json.load(f)[f"{seed}-{k}-{s}-{b}-{glen}-{n}"]
    assert M.digest(h, c) == want
    assert (c == 2).any() and used == n


@pytest.mark.parametrize("case", BLOOM_CASES[:3], ids=[f"k{c[1]}-b{c[3]}" for c in BLOOM_CASES[:3]])
def test_bloom_golden_digests_come_from_the_reference(oracle, reflib, case):
    seed, k, s, b, glen, n = case
    reads, po, _ = _case_hashes(oracle, seed, k, glen, n)
    rh, rc, _ = reflib.sketch_unit_m(reads, po, s=s, bloom_bytes=b, counts=True)
    with open(os.path.join(GOLDEN, "ref_bloom.json")) as f:
        assert M.digest(rh, rc) == json.load(f)[f"{seed}-{k}-{s}-{b}-{glen}-{n}"]


@pytest.mark.parametrize("m,c", [(1, 0.0), (2, 0.0), (3, 0.0), (1, 2.0), (2, 3.0), (3, 1e9)])
def test_reference_heap_matches_the_checker(oracle, m, c):
    # the Python heap against the C restatement (itself pinned to the reference's object code by test_oracle_vs_ref.py)
    reads, po, hs = _case_hashes(oracle, 40 + m, 21, 20_000, 1500)
    h, cnt, used = M.sketch_reads_reference(hs, 200, m=m, target_cov=c)
    oh, oc, _, ou = oracle.sketch_unit_mc(reads, po, s=200, min_copies=m, target_cov=c, counts=True)
    assert used == ou and np.array_equal(h, oh) and np.array_equal(cnt, oc)


@pytest.mark.parametrize("k", [15, 21, 32])
@pytest.mark.parametrize("m,b,c", [(1, 0, 0.0), (2, 0, 0.0), (3, 0, 0.0), (1, 0, 2.5), (2, 0, 3.0), (1, 1000, 0.0), (1, 65_536, 0.0),
                                   (1, 1000, 2.2), (1, 65_536, 1e9)])
def test_stretch_replay_equals_the_reference_heap(oracle, k, m, b, c):
    _, po, hs = _case_hashes(oracle, 70 + k + m, k, 12_000, 1000)
    use64 = bool(po.use64)
    want = M.sketch_reads_reference(hs, 150, m=m, bloom_bytes=b, target_cov=c, use64=use64)
    total = sum(x.size for x in hs)
    rng = np.random.default_rng(k * 100 + m)
    for cuts in [(), tuple(range(1000, total, 1000)), tuple(rng.integers(0, total, 40).tolist()), tuple(range(1, total, 97))]:
        h, cnt, used, events = M.sketch_reads_stretches(hs, 150, m=m, bloom_bytes=b, target_cov=c, use64=use64, cuts=cuts)
        assert used == want[2]
        assert np.array_equal(h, want[0]) and np.array_equal(cnt, want[1])
        if cuts:
            assert events < total          # the gate bound really thins the stream


def test_bloom_kat_regenerates_from_the_reference_header(tmp_path):
    # tests/golden/bloom_kat.cpp compiles the reference's bloom_filter.hpp in place; where those sources are present the committed
    # known answers must come out again (tables up to 200 MB; the larger ones only differ in size)
    import subprocess
    ref = os.environ.get("REF", "/root/reference/src/mash")
    if not os.path.exists(os.path.join(ref, "bloom_filter.hpp")):
        pytest.skip("reference sources absent")
    exe = str(tmp_path / "kat")
    subprocess.check_call(["g++", "-O2", "-I", ref, os.path.join(GOLDEN, "bloom_kat.cpp"), "-o", exe])
    got = json.loads(subprocess.check_output([exe, str(200_000_000)]))["cases"]
    want = [c for c in _kat() if c["bytes"] <= 200_000_000]
    assert got == want and len(got) == 4

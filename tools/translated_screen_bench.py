#!/usr/bin/env python
"""Rate of the translated screen (protein sketches) on one GPU, with the translation kernel's share from CUDA events.

    python tools/translated_screen_bench.py [--reads 50000000] [--dump DIR]

Workload, shaped like bench.py's configs[3] screen: 50 synthetic 5 Mbp source genomes (bench.py's genome generator), 150 bp
reads sampled from them (0.5 % substitutions, 0.1 % N) in '*'-joined chunks of 2 M reads resident in HBM, screened against a
100 000-sketch protein table: the frame-0 translations of the 50 source genomes sketched at k=9 s=1000 through the library,
plus synthetic protein sketches.  Each chunk is translated in six frames on the device and its amino-acid k-mers are screened;
finish() is inside the timed pass.  Prints one JSON line (with the card name and its power limit); --dump DIR writes the
outputs (float64 .npy) for comparing two builds.  Writes nothing else.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# standard genetic code, index 16 b0 + 4 b1 + b2 with A0 C1 G2 T3 ('*' = stop); only used to build the protein table
CODON_AA = b"KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF"


def translate_frame0_device(torch, seq):
    """Frame-0 translation of a uint8 device tensor (case folded); stops and codons with other bytes as '*'."""
    dev = seq.device
    code = torch.full((256,), 4, dtype=torch.int64, device=dev)
    for c, v in zip(b"ACGTacgt", (0, 1, 2, 3, 0, 1, 2, 3)):
        code[c] = v
    aa = torch.tensor(list(CODON_AA) + [ord("*")], dtype=torch.uint8, device=dev)
    m = seq.numel() // 3
    c = code[seq[:3 * m].view(m, 3).long()]
    idx = torch.where((c == 4).any(dim=1), torch.full_like(c[:, 0], 64), c[:, 0] * 16 + c[:, 1] * 4 + c[:, 2])
    return aa[idx]


def card_and_power_limit(torch, dev):
    """Name and enforced power limit of the device (read-only nvidia-smi query; None where it cannot be read)."""
    name, limit = torch.cuda.get_device_name(dev), None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(dev.index or 0)],
                           capture_output=True, text=True, timeout=20)
        f = [x.strip() for x in r.stdout.strip().split(",")]
        if r.returncode == 0 and len(f) == 2:
            name, limit = f[0], float(f[1])
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=50_000_000)
    ap.add_argument("--sources", type=int, default=50)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--sketches", type=int, default=100_000)
    ap.add_argument("--dump", metavar="DIR", default=None)
    args = ap.parse_args()

    import torch
    import mash_b200
    from bench import make_genomes_device, make_sketches_device, u64_halves, dump_outputs
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    eng = mash_b200.Engine(0)
    ks, s, glen, n_src = 9, 1000, args.genome_len, args.sources
    pp = eng.params(k=ks, s=s, alphabet=mash_b200._capi.ALPHABET_PROTEIN, noncanonical=True)

    src, _ = make_genomes_device(torch, dev, n_src, glen, seed=20260923)
    # the protein table: frame-0 translations of the sources, sketched through the library, + synthetic protein sketches
    peps = [translate_frame0_device(torch, src[i * (glen + 1): i * (glen + 1) + glen]) for i in range(n_src)]
    starts = np.zeros(n_src + 1, np.uint64)
    starts[1:] = np.cumsum([q.numel() + 1 for q in peps])
    pstream = torch.zeros(int(starts[-1]) + 16, dtype=torch.uint8, device=dev)
    for i, q in enumerate(peps):
        pstream[int(starts[i]):int(starts[i]) + q.numel()] = q
    del peps
    src_h = torch.zeros((n_src, s), dtype=torch.int64, device=dev)
    src_n = torch.zeros(n_src, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    eng.sketch_stream_dev(pp, pstream.data_ptr(), starts, src_h.data_ptr(), src_n.data_ptr())
    del pstream
    SH, SN, SL = make_sketches_device(torch, dev, args.sketches - n_src, s, seed=7007, length=glen // 3)
    PH = torch.cat([src_h, SH]); PN = torch.cat([src_n, SN]); PL = torch.cat([torch.full((n_src,), glen // 3, dtype=SL.dtype, device=dev), SL])
    del SH, SN, SL

    # reads: '*' + 150 bases drawn from the source genomes, resident in HBM
    read_len, chunk_reads = 150, min(args.reads, 2_000_000)
    n_chunks = max(1, args.reads // chunk_reads)
    span_r = read_len + 1
    chunk_bytes = chunk_reads * span_r
    chunk_pitch = (chunk_bytes + 64 + 255) // 256 * 256
    chunks = torch.zeros((n_chunks, chunk_pitch), dtype=torch.uint8, device=dev)
    g = torch.Generator(device=dev); g.manual_seed(4242)
    lut = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    idx = torch.arange(read_len, device=dev)[None, :]
    for c in range(n_chunks):
        st = torch.randint(0, src.numel() - read_len, (chunk_reads,), generator=g, device=dev)
        body = src[st[:, None] + idx]
        err = torch.rand((chunk_reads, read_len), generator=g, device=dev) < 0.005
        body = torch.where(err, lut[torch.randint(0, 4, (chunk_reads, read_len), generator=g, device=dev, dtype=torch.uint8).long()], body)
        body = torch.where(torch.rand((chunk_reads, read_len), generator=g, device=dev) < 0.001, torch.full_like(body, ord("N")), body)
        v = chunks[c, :chunk_bytes].view(chunk_reads, span_r)
        v[:, 0] = ord("*")
        v[:, 1:] = body
    del src
    torch.cuda.synchronize()              # the inputs are written on torch's stream, the engine reads them on its own

    pset = mash_b200._capi._Set(PH.data_ptr(), PN.data_ptr(), PL.data_ptr(), on_device=True, n=PH.shape[0], stride=s)
    wjob = mash_b200._capi.ScreenJob(eng, pset, None, pp)                  # warm-up (peptide buffers, first-use costs)
    for c in range(min(2, n_chunks)):
        wjob.feed_dev(chunks[c].data_ptr(), chunk_bytes)
    wjob.close()
    torch.cuda.synchronize()
    job = mash_b200._capi.ScreenJob(eng, pset, None, pp)
    eng.set_timing(True); eng.stats(reset=True)
    t0 = time.perf_counter()
    for c in range(n_chunks):
        job.feed_dev(chunks[c].data_ptr(), chunk_bytes)
    res = job.finish()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    st = eng.stats(reset=True)
    eng.set_timing(False)
    job.close()
    bases = n_chunks * chunk_reads * read_len
    card, limit = card_and_power_limit(torch, dev)
    if args.dump:
        out = dict(shared=res["shared"], median=res["median"], identity=res["identity"], pvalue=res["pvalue"], set_size=np.array([res["set_size"]]))
        out["mixture_hi"], out["mixture_lo"] = u64_halves(res["mixture"])
        dump_outputs(args.dump, out)
    print(json.dumps({
        "metric": "Gbp_per_s_screened_translated", "value": bases / dt / 1e9, "unit": "Gbp/s (nucleotides of the mixture)",
        "workload": f"{n_chunks} '*'-joined chunks of {chunk_reads} 150 bp reads ({bases} bases, resident in HBM) vs {PH.shape[0]} protein sketches "
                    f"(k={ks}, s={s}): frame-0 translations of the {n_src} source genomes sketched through the library + synthetic protein sketches; "
                    "six-frame translation on the device, finish() included",
        "ms_total": dt * 1e3, "translate_kernel_ms": st["translate_kernel_ms"], "scan_kernel_ms": st["scan_kernel_ms"],
        "translate_share_of_pass": st["translate_kernel_ms"] / (dt * 1e3), "translate_launches": int(st["translate_kernel_launches"]),
        "exact_reruns": int(st["exact_reruns"]), "set_size": int(res["set_size"]),
        "source_shared": [int(x) for x in res["shared"][:n_src]], "source_sketch_n": [int(x) for x in src_n.cpu().numpy()],
        "synthetic_references_hit": int((res["shared"][n_src:] > 0).sum()),
        "card": card, "power_limit_w": limit}))


if __name__ == "__main__":
    main()

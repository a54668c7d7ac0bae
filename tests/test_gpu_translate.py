"""Byte-exact tests of the six-frame translation kernel (translate.cu) through mashgpu_translate6: every output byte of a
chunk against the checker's six_frames (translated_screen_oracle.py, pinned by test_translate_model.py), with '*' written
as 0 and one 0 after each frame.  The cases aim at the kernel's own edges: every length mod 3, 16 and 48 inside one CTA,
the CTA boundaries (12 288 bases), every byte triple in every frame, the 16-byte vector path and the byte-load path, bytes
past the end of the input, bytes outside the output, and a chunk above 2^31 bases."""
import numpy as np
import pytest

import translated_screen_oracle as tso

CTA = 256 * 48       # bases per CTA of translate6_kernel
CANARY = 0xA5        # never an amino acid or 0: an output byte left unwritten shows
MARGIN = 64          # canary bytes checked before and after the output
DIRTY = np.frombuffer(b"ACGTacgtACGTacgtUuNnRYKMSWBDHVXx*-.\x00\x01\x7f\x80\xc1\xff", np.uint8)


def translated_length(n):
    return sum(2 * ((n - f) // 3 + 1) if n > f else 2 for f in range(3))


def expected(seq, preserve_case):
    """The kernel's output for one chunk: six_frames with '*' as 0, each frame followed by one 0 byte."""
    out = []
    for fr in tso.six_frames(np.asarray(seq, np.uint8), preserve_case):
        out += [np.where(fr == ord("*"), 0, fr).astype(np.uint8), np.zeros(1, np.uint8)]
    return np.concatenate(out)


def dirty(seed, n, p_dirty=0.15):
    """Mostly A/C/G/T in both cases, with U/u, N, IUPAC letters, '*', 0 and bytes >= 0x80 mixed in."""
    rng = np.random.Generator(np.random.PCG64(seed))
    acgt = np.frombuffer(b"ACGTACGTacgt", np.uint8)[rng.integers(0, 12, n)]
    return np.where(rng.random(n) < p_dirty, DIRTY[rng.integers(0, DIRTY.size, n)], acgt).astype(np.uint8)


class Translator:
    """Device buffers reused across calls.  The input sits at a chosen offset from a 512-byte aligned allocation, with 'A'
    bytes before it and everywhere past its end (at least to its end rounded up to 16); the output sits between canary
    margins."""

    def __init__(self, gpu, max_len):
        import torch
        self.gpu, self.torch = gpu, torch
        self.d_in = torch.empty(max_len + 64, dtype=torch.uint8, device="cuda")
        self.d_out = torch.empty(translated_length(max_len) + 2 * MARGIN, dtype=torch.uint8, device="cuda")
        assert self.d_in.data_ptr() % 512 == 0

    def run(self, seq, preserve_case, offset=0):
        torch = self.torch
        seq = np.asarray(seq, np.uint8)
        n, t = seq.size, translated_length(seq.size)
        self.d_in.fill_(ord("A"))
        if n:
            self.d_in[offset:offset + n].copy_(torch.from_numpy(seq.copy()))
        self.d_out[:t + 2 * MARGIN].fill_(CANARY)
        torch.cuda.synchronize()
        self.gpu.translate6(self.d_in.data_ptr() + offset, n, preserve_case, self.d_out.data_ptr() + MARGIN)
        return self.d_out[:t + 2 * MARGIN].cpu().numpy()

    def check(self, seq, preserve_case, offset=0):
        got = self.run(seq, preserve_case, offset)
        want = expected(seq, preserve_case)
        assert (got[:MARGIN] == CANARY).all() and (got[-MARGIN:] == CANARY).all(), (len(seq), offset, "write outside the output")
        inner = got[MARGIN:-MARGIN]
        if not np.array_equal(inner, want):
            bad = np.flatnonzero(inner != want)
            pytest.fail(f"len {len(seq)} offset {offset} preserve_case {preserve_case}: {bad.size} bytes differ, first at {bad[0]} "
                        f"(got {inner[bad[0]]}, want {want[bad[0]]})")


@pytest.fixture(scope="module")
def tr(gpu):
    return Translator(gpu, 7 * CTA + 64)


def test_expected_layout():
    # the checker's layout on a hand-made chunk: ATGGCCTAAG -> forward frames ATG GCC TAA | TGG CCT AAG | GGC CTA, reverse
    # complement CTTAGGCCAT -> CTT AGG CCA | TTA GGC CAT | TAG GCC; a stop is 0 and each frame ends in 0
    want = b"MA\0\0" + b"WPK\0" + b"GL\0" + b"LRP\0" + b"LGH\0" + b"\0A\0"
    assert bytes(expected(np.frombuffer(b"ATGGCCTAAG", np.uint8), False)) == want
    for n in range(0, 60):
        assert expected(dirty(n, n), False).size == translated_length(n)
    assert translated_length(0) == 6 and translated_length(1) == 6 and translated_length(3) == 8


@pytest.mark.gpu
@pytest.mark.parametrize("preserve_case", [False, True])
def test_every_length_inside_one_cta(tr, preserve_case):
    # lengths 0..400: every len mod 3, 16 and 48; on the vector path (offset 0) and on the byte-load path
    src = dirty(11 + preserve_case, 401 + 400)
    for n in range(401):
        seq = src[n:2 * n]
        tr.check(seq, preserve_case, 0)
        tr.check(seq, preserve_case, 1 + n % 15)


@pytest.mark.gpu
@pytest.mark.parametrize("preserve_case", [False, True])
def test_cta_boundaries(tr, preserve_case):
    # len = 12288 m + d: the last CTA is nearly full, nearly empty or exactly full, with every len mod 3 around it
    src = dirty(21 + preserve_case, 7 * CTA + 64)
    ds = list(range(-6, 7)) + [-49, -48, -47, 47, 48, 49]
    for m in (1, 2, 3, 7):
        for d in ds:
            n = CTA * m + d
            seq = src[:n]
            tr.check(seq, preserve_case, 0)
            tr.check(seq, preserve_case, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", list(range(16)))
def test_alignment_and_bounds(tr, offset):
    # the input at every offset mod 16 (vector loads only at 0), 'A' past its end, canaries around the output
    src = dirty(31 + offset, 3 * CTA + 64, p_dirty=0.05)
    lens = [1, 2, 3, 4, 15, 16, 17, 31, 32, 33, 46, 47, 48, 49, 50, 51, 95, 96, 97, 98, CTA - 2, CTA - 1, CTA, CTA + 1, CTA + 2,
            CTA + 16, CTA + 17, 2 * CTA + 50, 3 * CTA - 15, 3 * CTA + 31]
    for n in lens:
        seq = src[:n].copy()
        seq[-min(n, 4):] = np.frombuffer(b"CCGT", np.uint8)[:min(n, 4)]      # an 'A' read past the end would change a codon
        tr.check(seq, offset % 2 == 1, offset)


@pytest.mark.gpu
@pytest.mark.parametrize("ab", [(0, 0), (1, 2), (2, 1)])
@pytest.mark.parametrize("preserve_case", [False, True])
def test_every_codon_in_every_frame(gpu, ab, preserve_case):
    # all 256^3 byte triples back to back after a prefix of a bytes and before a suffix of b bytes: triple i is codon i of
    # forward frame a and codon N - 1 - i of reverse frame b, so the three (a, b) put every triple in all six frames
    import torch
    a, b = ab
    t = np.arange(1 << 24, dtype=np.uint32)
    triples = np.stack([(t >> 16) & 255, (t >> 8) & 255, t & 255], axis=1).astype(np.uint8).reshape(-1)
    del t
    seq = np.concatenate([np.frombuffer(b"GA"[:a], np.uint8), triples, np.frombuffer(b"CT"[:b], np.uint8)])
    del triples
    n = seq.size
    d_in = torch.full((n + 16,), ord("A"), dtype=torch.uint8, device="cuda")
    d_in[:n].copy_(torch.from_numpy(seq))
    tl = translated_length(n)
    d_out = torch.full((tl + 2 * MARGIN,), CANARY, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    gpu.translate6(d_in.data_ptr(), n, preserve_case, d_out.data_ptr() + MARGIN)
    got = d_out.cpu().numpy()
    del d_in, d_out
    assert (got[:MARGIN] == CANARY).all() and (got[-MARGIN:] == CANARY).all()
    want = expected(seq, preserve_case)
    assert np.array_equal(got[MARGIN:-MARGIN], want)


def _fold(x, preserve_case):
    x = np.asarray(x, np.uint8).copy()
    if not preserve_case:
        low = (x > 96) & (x < 123)
        x[low] -= 32
    return x


def _aa(b0, b1, b2):
    """Amino acid of codons (b0, b1, b2) of folded bytes, 0 for a stop or a byte outside {A,C,G,T}."""
    c = np.stack([tso._BASE[b0], tso._BASE[b1], tso._BASE[b2]])
    aa = tso._AA[np.where((c == 4).any(axis=0), 64, 16 * c[0] + 4 * c[1] + c[2])]
    return np.where(aa == ord("*"), 0, aa).astype(np.uint8)


def frame_window(get, n, preserve_case, frame, lo, hi):
    """Codons of one frame (0..2 forward, 3..5 reverse) whose bases all lie in [lo, hi), computed from get(a, b) = seq[a:b]:
    forward codon i of frame f covers bases 3i+f..3i+f+2, reverse codon j of frame r bases n-3-(3j+r)..n-1-(3j+r), read
    backwards and complemented.  Returns (first codon index, amino acids)."""
    x = _fold(get(lo, hi), preserve_case)
    f = frame % 3
    if frame < 3:
        i0 = max(0, -(-(lo - f) // 3))
        i1 = (hi - 3 - f) // 3 + 1
        p = 3 * np.arange(i0, i1) + f - lo
        return i0, _aa(x[p], x[p + 1], x[p + 2])
    j0 = max(0, -(-(n - hi - f) // 3))           # smallest j with n-1-(3j+r) < hi
    j1 = (n - 3 - f - lo) // 3 + 1                 # past the largest j with n-3-(3j+r) >= lo
    p = n - 3 - (3 * np.arange(j0, j1) + f) - lo
    comp = tso._COMPLEMENT
    return j0, _aa(comp[x[p + 2]], comp[x[p + 1]], comp[x[p]])


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5, 29, 30, 31, 100, 101, 102])
def test_frame_window_equals_six_frames(n):
    # the windowed expectation of the large-chunk test, against six_frames on whole small chunks
    seq = dirty(500 + n, n)
    for pc in (False, True):
        frames = tso.six_frames(seq, pc)
        for fr in range(6):
            for lo, hi in ((0, n), (1, n), (0, max(0, n - 2)), (n // 3, n - n // 4), (7, 40)):
                lo, hi = min(lo, n), max(min(hi, n), min(lo, n))
                i0, got = frame_window(lambda a, b: seq[a:b], n, pc, fr, lo, hi)
                w = frames[fr][i0:i0 + got.size]
                assert np.array_equal(got, np.where(w == ord("*"), 0, w)), (n, pc, fr, lo, hi)
                inside = [i for i in range(frames[fr].size)
                          if (lo <= 3 * i + fr % 3 and 3 * i + fr % 3 + 3 <= hi if fr < 3 else
                              lo <= n - 3 - (3 * i + fr % 3) and n - (3 * i + fr % 3) <= hi)]
                assert list(range(i0, i0 + got.size)) == inside, (n, fr, lo, hi)


@pytest.mark.gpu
def test_chunk_above_2_pow_31_bases(gpu):
    # ~2.2 GB in, ~4.3 GB out: codon indices and output offsets past 2^31 (and past 2^32 in the reverse frames' output)
    import torch
    n = (1 << 31) + 3 * CTA * 1000 + 20_000
    n += (2 - n % 3) % 3                                  # len mod 3 == 2
    period = (1 << 20) + 7
    pattern = torch.from_numpy(dirty(41, period, p_dirty=0.05))
    reps = -(-(n + 16) // period)
    d_in = pattern.cuda().repeat(reps)                    # readable well past n rounded up to 16
    windows = [(0, 20_000), (n // 2 - 5000, n // 2 + 5000), ((1 << 31) - 30_000, (1 << 31) + 30_000), (n - 20_000, n)]
    for w, (lo, hi) in enumerate(windows):                # fresh bytes in every compared window
        d_in[lo:hi].copy_(torch.from_numpy(dirty(42 + w, hi - lo)))
    tl = translated_length(n)
    d_out = torch.full((tl + 2 * MARGIN,), CANARY, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for pc in (False, True):
        gpu.translate6(d_in.data_ptr(), n, pc, d_out.data_ptr() + MARGIN)
        torch.cuda.synchronize()
        assert (d_out[:MARGIN] == CANARY).all().item() and (d_out[-MARGIN:] == CANARY).all().item()
        nf = [(n - f) // 3 for f in range(3)]
        base = np.cumsum([0] + [nf[s % 3] + 1 for s in range(6)])
        assert base[6] == tl
        term = d_out[MARGIN + torch.tensor(base[1:] - 1, device="cuda")].cpu().numpy()
        assert (term == 0).all()
        get = lambda a, b: d_in[a:b].cpu().numpy()
        for lo, hi in windows:
            for fr in range(6):
                i0, want = frame_window(get, n, pc, fr, lo, hi)
                assert want.size > 0
                o = MARGIN + int(base[fr]) + i0
                got = d_out[o:o + want.size].cpu().numpy()
                assert np.array_equal(got, want), (pc, fr, lo, hi)
    del d_in, d_out


@pytest.mark.gpu
def test_translate6_refuses_null(gpu):
    import torch
    import mash_b200
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    for args in ((None, 10, 0, d.data_ptr()), (d.data_ptr(), 10, 0, None), (None, 0, 0, None)):
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.translate6(*args)
        assert e.value.code == 1 and "NULL" in str(e.value)          # MASHGPU_ERR_INVALID

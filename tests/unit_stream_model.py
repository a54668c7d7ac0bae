"""CPU model of the streaming unit job (mashgpu_unit_*, DESIGN.md 2.7): one sketch unit cut into stages, merged into a running
bottom-s with summed counts and one extra number -- the count of the current top at positions <= t*.

`sketch_unit_stages` restates, in the order the job does it, what each stage contributes: its own bottom-s distinct hashes with
count, first and last position, merged into the running set.  A stage changes the set only when a hash first seen in it enters;
t* (the latest first occurrence among the set's hashes) then lies in that stage, and the top's count at positions <= t* is its
total before the stage plus its occurrences in the stage up to t*.  The result must equal MinHashHeap with m = 1
(reads_stream_model.ReferenceHeap) fed every hash in order, for any stage boundaries.

`unit_merge` in sketch.cu is the device code's one copy of this rule: the unit job applies it per stage, and the exact re-run of a
flagged unit applies it once, as a merge into an empty state (with m > 1, the promoting m-th occurrence stands for the first).
"""
import numpy as np

EMPTY = 0xFFFFFFFFFFFFFFFF


def stage_candidates(seg, base, s):
    """The stage's s smallest distinct hashes, ascending: (hash, count, first position, last position), positions global."""
    out = {}
    for i, h in enumerate(seg.tolist()):
        if h in out:
            c, f, _ = out[h]
            out[h] = (c + 1, f, base + i)
        else:
            out[h] = (1, base + i, base + i)
    return [(h, *out[h]) for h in sorted(out)[:s]]


def top_count_to(seg, base, top, cand, tstar):
    """Occurrences of `top` in the stage at positions <= t*: decided by its first / last position in the stage, else counted over
    [stage start, t*] of the still-resident stage (the job's SCAN_COUNT recount)."""
    if cand is None:
        return 0, False
    _, c, f, l = cand
    if l <= tstar:
        return c, False
    if f > tstar:
        return 0, False
    if f == tstar:
        return 1, False
    return int(np.count_nonzero(seg[:tstar - base + 1] == np.uint64(top))), True


def sketch_unit_stages(flat, s, cuts=()):
    """The k-mer hash stream `flat` (uint64, stream order) cut into stages at the given indices.  Returns (hashes ascending, counts,
    recounts) with the reference heap's counts (top-of-heap quirk included)."""
    flat = np.ascontiguousarray(flat, np.uint64)
    bounds = [0] + sorted(c for c in set(cuts) if 0 < c < flat.size) + [flat.size]
    keys, tot = [], []            # the running bottom-s and the total count of each
    top_at_tstar = 0              # the current top's count at positions <= t*
    recounts = 0
    for a, b in zip(bounds[:-1], bounds[1:]):
        seg = flat[a:b]
        cand = stage_candidates(seg, a, s)
        i = j = 0
        nk, nt, src = [], [], []
        tstar = None
        while len(nk) < s and (i < len(keys) or j < len(cand)):
            if j == len(cand) or (i < len(keys) and keys[i] < cand[j][0]):
                nk.append(keys[i]); nt.append(tot[i]); src.append((i, None)); i += 1
            elif i == len(keys) or cand[j][0] < keys[i]:
                nk.append(cand[j][0]); nt.append(cand[j][1]); src.append((None, j))
                tstar = cand[j][2] if tstar is None else max(tstar, cand[j][2])      # entered in this stage
                j += 1
            else:
                nk.append(keys[i]); nt.append(tot[i] + cand[j][1]); src.append((i, j)); i += 1; j += 1
        if tstar is not None and nk[-1] != EMPTY:
            ri, cj = src[-1]
            before = tot[ri] if ri is not None else 0
            part, rec = top_count_to(seg, a, nk[-1], cand[cj] if cj is not None else None, tstar)
            top_at_tstar = before + part
            recounts += rec
        keys, tot = nk, nt
    counts = list(tot)
    if len(keys) == s and keys[-1] != EMPTY:
        counts[-1] = top_at_tstar
    return np.array(keys, np.uint64), np.array(counts, np.uint32), recounts
